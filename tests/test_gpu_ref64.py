"""The fused joint and the loss op against the chunked float64 reference (tests/joint_ref64.py, CUDA float64) at the
sizes where nothing else holds them to the truth:

  * BASELINE C3 at full size (B=32 T=512 U=128 V=1024 H=640): the tensor-core path in keep and recompute mode, the fp32
    exact path, and FastEmit at lambda = 0.01 on both paths;
  * BASELINE C5 at full size (bench.py's generator and seed: B=64, T_b up to 1600, U_b up to 200, V=4096): the tensor-core
    path with valid_tiles (one chunk, keep) and without (several chunks, recompute), and the fp32 exact path;
  * the tensor-core path at V = 8192, 16384, 32768 (H = 640) and V = 32768 (H = 128), where the dW kernel runs unsplit
    (S = 1: one fp32 accumulation chain over every lattice row of the batch): 524 288 valid rows, blank = V - 1, labels in
    the last 64-column chunk, and rows whose dominant column lies in the last chunk (so the forward's reference is raised
    after V/64 - 1 chunks were kept); keep mode and the recompute mode that the batch takes by itself over the 16 GiB
    chunk budget, and the fp32 exact path at V = 32768;
  * the loss op on fp32, fp16 and bf16 logits at V = 8192 and 32768 (two-pass kernels), ragged, with lattices of more
    than 500 wavefront steps.

Tolerances are DESIGN.md 4's: tensor-core path costs rtol 2e-4, gradients 1e-2·max|g| element-wise, relative Frobenius
error below 5e-3 and at least half the reference's norm; fp32 paths rtol 1e-4; 16-bit loss op the fp32 bounds widened by
its unit roundoff, against the reference run on the rounded logits.  On these long lattices every path also carries the
round-off of its fp32 alpha/beta (`ab_cell`, `ab_norm` below: the C oracle run in fp32 on one C3 utterance is itself
2.6e-3 relative, 6.6e-7·|cost|, from its float64 run), which DESIGN.md 4 states as a limit.  Every case prints its measured errors
(lines starting with "ref64"), so that a marginal pass is visible.  The reference runs before the path it checks and its
device memory is released in between, so each case fits one 80 GB card.
"""
import time

import numpy as np
import pytest
import torch

import joint_ref64 as r64
from conftest import assert_close
from test_gpu_fastemit import run_joint
from test_gpu_joint import synth
from test_gpu_large_offsets import UNIT, dev, op16_backward, op16_forward, op_fp32

pytestmark = pytest.mark.gpu

NAMES = ("d_enc", "d_pred", "dW", "db")
TC_COST = dict(rtol=2e-4, atol=1e-3)
CHUNK_BUDGET = 16 << 30                        # bytes of kept numerators per workspace chunk (joint_tc.cuh)
TC_SMS = 132


def dw_splits(H, V):
    """The dW kernel's lattice-row splits (dw_geometry in csrc/joint_bwd.cuh)."""
    return max(1, min(64, 4 * TC_SMS // (-(-V // 128) * (H // 128 + 1))))


def padded_rows(T, U):
    """Kept rows of one utterance of a padded (T, U) lattice: 16 x 8 tiles of 128 rows."""
    return -(-T // 16) * -(-U // 8) * 128


@pytest.fixture(scope="module", autouse=True)
def _wall_and_peak():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    print("\nref64 file: %.0f s wall, peak torch.cuda.max_memory_allocated %.1f GB"
          % (time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 1e9))


@pytest.fixture(autouse=True)
def _release_device_memory():
    yield
    torch.cuda.empty_cache()


def reference(k, gs, lam=0.0):
    """tests/joint_ref64.py on the device, results on the host."""
    t = time.perf_counter()
    out = r64.joint_loss_grad(*(dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")), k["labels"],
                              k["input_lengths"], k["label_lengths"], int(k["blank"]), grad_scale=gs, fastemit_lambda=lam)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    print("\nref64 reference: %d valid rows, V=%d, %.1f s" % (int(np.sum(k["input_lengths"] * (k["label_lengths"] + 1))),
                                                             k["W"].shape[1], time.perf_counter() - t))
    return out


def errors(costs, grads, want):
    """Measured errors, as printed: costs' max relative error, and per gradient the relative Frobenius error and the
    largest element-wise error over max|g|."""
    parts = ["costs %.2e" % np.max(np.abs(costs - want["costs"]) / np.abs(want["costs"]))]
    for g, n in zip(grads, NAMES):
        w = want[n]
        parts.append("%s frob %.2e max %.2e" % (n, np.linalg.norm(g - w) / np.linalg.norm(w),
                                                np.max(np.abs(g - w)) / np.max(np.abs(w))))
    return ", ".join(parts)


def ab_cell(cmax):
    """Per-cell floor of the fp32 alpha/beta round-off on lattices of hundreds of wavefront steps (DESIGN.md 4):
    alpha, beta and the log-likelihood are fp32 numbers of magnitude |cost|, so every occupancy exp(alpha + beta + lp - ll)
    carries a few eps32·|cost| of relative error.  Measured up to 2e-6·|cost| (1024 x 40 lattice), 1.4e-6·|cost| here."""
    return 1e-6 + 2e-6 * cmax


def ab_norm(cmax):
    """The same round-off in a reduced gradient (d_enc, d_pred, dW, db), relative to max|g|.  Measured on the fp32 exact
    path at C3, which has no 16-bit operand: 4.9e-7·|cost| element-wise, 3.5e-7·|cost| Frobenius.  Both joint paths
    compute alpha and beta in fp32, so the term is added to each path's own bound."""
    return 6e-7 * cmax


def check_tc(costs, grads, want, what):
    """DESIGN.md 4's tensor-core bounds plus the fp32 alpha/beta term: costs rtol 2e-4; no gradient below half the
    reference's norm; element-wise (1e-2 + ab)·max|g|; relative Frobenius error below 5e-3 + ab."""
    ab = ab_norm(float(np.abs(want["costs"]).max()))
    print("ref64 %s: %s (alpha/beta term %.2e)" % (what, errors(costs, grads, want), ab))
    assert np.all(np.isfinite(costs)), what
    assert_close(costs, want["costs"], what=what + " costs", **TC_COST)
    for g, n in zip(grads, NAMES):
        w = want[n]
        assert np.all(np.isfinite(g)), (what, n)
        ng, no = np.linalg.norm(g), np.linalg.norm(w)
        assert ng >= 0.5 * no, "%s %s: |g| = %.4g is less than half the reference's %.4g" % (what, n, ng, no)
        assert_close(g, w, rtol=0, atol=0, ntol=1e-2 + ab, what="%s %s" % (what, n))
        assert np.linalg.norm(g - w) / no < 5e-3 + ab, (what, n)


def check_fp32(costs, grads, want, gs, what):
    """fp32 bounds: costs rtol 1e-5; gradients rtol 1e-4, the per-cell floor and the norm-wise alpha/beta term."""
    cmax = float(np.abs(want["costs"]).max())
    print("ref64 %s: %s (alpha/beta term %.2e)" % (what, errors(costs, grads, want), ab_norm(cmax)))
    assert_close(costs, want["costs"], rtol=1e-5, atol=1e-3, what=what + " costs")
    for g, n in zip(grads, NAMES):
        assert_close(g, want[n], rtol=1e-4, atol=ab_cell(cmax) * np.max(np.abs(gs)),
                     ntol=max(1e-5, ab_norm(cmax)), what="%s %s" % (what, n))


def kernel_names(fn):
    """fn() with the library's kernel timing on: (fn's result, the set of kernel names it launched)."""
    from rnnt_speech_recognition_b200 import _lib
    _lib.set_timing(True)
    try:
        out = fn()
        torch.cuda.synchronize()
        names = {n for n, _ in _lib.get_timings()}
    finally:
        _lib.set_timing(False)
    return out, names


def assert_mode(names, keep, what):
    """keep: one keeping forward and nothing recomputed; otherwise a costs-only forward and recomputing forwards."""
    s = " ".join(sorted(names))
    if keep:
        assert "<fwd+keep>" in s and "<fwd>" not in s, (what, s)
    else:
        assert "<fwd>" in s and "<fwd+keep>" in s, (what, s)


# --------------------------------------------------------------------------------------------------- C3, full size
C3 = dict(B=32, T=512, U=128, V=1024, H=640)


@pytest.fixture(scope="module")
def c3():
    """tests/test_gpu_fullsize.py's inputs and their float64 reference at the upstream gradient 1/B."""
    k = synth(C3["B"], C3["T"], C3["U"], C3["V"], C3["H"], 2026, ragged=False)
    gs = np.full(C3["B"], 1.0 / C3["B"])
    return k, gs, reference(k, gs)


@pytest.mark.parametrize("keep", [True, False])
def test_c3_tensor_core_vs_float64(c3, keep):
    k, gs, want = c3
    (costs, grads), names = kernel_names(lambda: run_joint(k, "bf16", gs, keep=keep))
    assert_mode(names, keep, "C3")
    check_tc(costs, grads, want, "C3 bf16 %s" % ("keep" if keep else "recompute"))


def test_c3_fp32_exact_vs_float64(c3):
    k, gs, want = c3
    costs, grads = run_joint(k, "fp32", gs)
    check_fp32(costs, grads, want, gs, "C3 fp32 exact")


def test_c3_fastemit_vs_float64(c3):
    """lambda = 0.01 on both paths against the reference with every label arc's gradient scaled by 1.01.  The change
    FastEmit makes here (about 2e-3 of |g|) is of the order of both paths' fp32 alpha/beta round-off (the fp32 path's
    error is 0.8 to 4 times it), so whether lambda is applied at all is left to tests/test_gpu_fastemit.py, whose
    second difference at this size cancels the round-off common to the three runs; the printed ratios show it."""
    k, gs, want0 = c3
    lam = 0.01
    want = reference(k, gs, lam)
    costs, grads = run_joint(k, "fp32", gs, fastemit_lambda=lam)
    check_fp32(costs, grads, want, gs, "C3 fp32 exact, lambda 0.01")
    for g, n in zip(grads, NAMES):
        err, change = np.linalg.norm(g - want[n]), np.linalg.norm(want[n] - want0[n])
        print("ref64 C3 fp32 %s: |err| / |g(0.01) - g(0)| = %.2e" % (n, err / change))
    costs, grads = run_joint(k, "bf16", gs, fastemit_lambda=lam)
    check_tc(costs, grads, want, "C3 bf16, lambda 0.01")


# --------------------------------------------------------------------------------------------------- C5, full size
@pytest.fixture(scope="module")
def c5():
    """bench.py's C5 batch (its generator, seed 1234) as numpy, and its float64 reference at 1/B."""
    import bench
    cfg = bench.WORKLOADS["c5"]
    d = bench.synth(cfg, 1234, "cpu")
    k = dict(enc=d["enc"].numpy(), pred=d["pred"].numpy(), W=d["W"].numpy(), b=d["b"].numpy(),
             labels=d["labels"].numpy(), input_lengths=d["il"].numpy(), label_lengths=d["ll"].numpy(), blank=np.int32(0))
    il, ll = k["input_lengths"], k["label_lengths"]
    assert k["enc"].shape == (64, 1600, 640) and k["W"].shape == (640, 4096)
    assert (il[0], ll[0], il[1], ll[1]) == (1600, 199, 100, 9)
    assert il.min() >= 100 and ll.min() >= 9 and ll.max() <= 199
    gs = np.full(64, 1.0 / 64)
    return k, gs, reference(k, gs)


@pytest.mark.parametrize("valid_tiles", [True, False])
def test_c5_tensor_core_vs_float64(c5, valid_tiles):
    """valid_tiles: the batch is one compact chunk and the forward keeps its numerators (as bench.py runs C5); without
    it the padded batch exceeds the chunk budget and the backward recomputes chunk by chunk."""
    import rnnt_speech_recognition_b200 as rb
    k, gs, want = c5
    il, ll = k["input_lengths"], k["label_lengths"]
    vt = rb.valid_tile_count(il, ll) if valid_tiles else None
    assert 64 * padded_rows(1600, 200) * (2 * 4096 + 8) > CHUNK_BUDGET
    (costs, grads), names = kernel_names(lambda: run_joint(k, "bf16", gs, valid_tiles=vt))
    assert_mode(names, valid_tiles, "C5")
    check_tc(costs, grads, want, "C5 bf16 %s" % ("valid_tiles keep" if valid_tiles else "multi-chunk recompute"))
    for b in range(64):
        assert not grads[0][b, il[b]:].any() and not grads[1][b, ll[b] + 1:].any()


def test_c5_fp32_exact_vs_float64(c5):
    """The fp32 exact path on the same batch: its error is the fp32 alpha/beta round-off of lattices of up to 1799
    wavefront steps, without any 16-bit operand."""
    k, gs, want = c5
    costs, grads = run_joint(k, "fp32", gs)
    check_fp32(costs, grads, want, gs, "C5 fp32 exact")


# ------------------------------------------------------------------------------------------------------- large V
LARGE_V = [(8192, 640), (16384, 640), (32768, 640), (32768, 128)]
LV = dict(B=8, T=512, U=128)                   # 524 288 valid lattice rows
LV_PLANT = dict(b=5, u=77, nats=60.0)


def large_v_case(V, H):
    """synth's distributions at (8, 512, 128, V, H); blank = V - 1; labels in the last 64-column chunk; hidden unit H-1 is
    0 except pred[5, 77] = 10 and W[H-1, V-23] = 60, so in utterance 5's rows at u = 77 column V-23 lies about 60 nats
    above the rest (tests/test_gpu_numerics.py's dominant column) and the forward raises those rows' reference at the
    last chunk, rescaling the numerators it kept for all V/64 - 1 earlier chunks."""
    k = synth(LV["B"], LV["T"], LV["U"], V, H, V + H, ragged=False)
    rng = np.random.default_rng(V - H)
    col = V - 23
    k["blank"] = np.int32(V - 1)
    k["labels"] = rng.integers(V - 64, V - 1, k["labels"].shape).astype(np.int32)
    k["labels"][k["labels"] == col] = V - 64
    h = H - 1
    k["enc"][:, :, h] = 0.0
    k["pred"][:, :, h] = 0.0
    k["pred"][LV_PLANT["b"], LV_PLANT["u"], h] = 10.0
    k["W"][h] = 0.0
    k["W"][h, col] = LV_PLANT["nats"]
    return k


@pytest.mark.parametrize("V,H", LARGE_V)
def test_large_v_tensor_core_vs_float64(V, H):
    """Keep mode (V = 8192: by default; larger V: with valid_tiles, one compact chunk) and recompute mode (V = 8192:
    keep_activations=False; larger V: by default, the batch being over the chunk budget)."""
    import rnnt_speech_recognition_b200 as rb
    k = large_v_case(V, H)
    gs = np.full(LV["B"], 1.0 / LV["B"])
    want = reference(k, gs)
    over = V > 8192
    vt = rb.valid_tile_count(k["input_lengths"], k["label_lengths"])
    for mode, kw in (("keep", dict(valid_tiles=vt) if over else dict(keep=True)),
                     ("recompute", dict() if over else dict(keep=False))):
        (costs, grads), names = kernel_names(lambda: run_joint(k, "bf16", gs, **kw))
        assert_mode(names, mode == "keep", (V, H, mode))
        check_tc(costs, grads, want, "V=%d H=%d bf16 %s" % (V, H, mode))
        torch.cuda.empty_cache()


def test_large_v_fp32_exact_vs_float64():
    V, H = 32768, 640
    k = large_v_case(V, H)
    gs = np.full(LV["B"], 1.0 / LV["B"])
    want = reference(k, gs)
    costs, grads = run_joint(k, "fp32", gs)
    check_fp32(costs, grads, want, gs, "V=%d H=%d fp32 exact" % (V, H))


# ----------------------------------------------------------------------------------------------- loss op, large V
OP_LENGTHS = ((520, 32), (37, 9), (505, 20))    # (T_b, U_b): 551 and 524 wavefront steps
OP_DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


@pytest.mark.parametrize("V", [8192, 32768])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_op_large_v_vs_float64(V, dt):
    """Logits 2·N(0, 1) drawn in their own dtype; the reference reads them through a callback as the kernels do (16-bit
    values exactly widened) and hands each chunk of its logits gradient to a device-side comparison."""
    dtype = OP_DT[dt]
    B, maxT, maxU = len(OP_LENGTHS), max(T for T, _ in OP_LENGTHS), max(U for _, U in OP_LENGTHS)
    g = torch.Generator(device="cuda").manual_seed(V + len(dt))
    x = torch.empty(B, maxT, maxU, V, dtype=dtype, device="cuda")
    for b in range(B):
        x[b].normal_(0.0, 2.0, generator=g)
    rng = np.random.default_rng(V)
    labels = rng.integers(0, V, (B, maxU - 1)).astype(np.int32)
    labels[:, ::5] = 0                          # some labels equal to blank
    il = np.array([T for T, _ in OP_LENGTHS], np.int32)
    ll = np.array([U - 1 for _, U in OP_LENGTHS], np.int32)
    d = dict(lab=dev(labels), il=dev(il), ll=dev(ll))
    if dtype == torch.float32:
        gs = np.linspace(0.5, 1.5, B) * np.array([1.0, -1.0, 1.0])
        costs, grad = op_fp32(x, d, "rnntb200_loss_device", gs)
        u = 0.0
    else:
        gs = np.full(B, 1.0 / B)
        costs, ws = op16_forward(x, d)
        grad = op16_backward(x, d, ws, gs)
        del ws
        u = UNIT[dtype]
    torch.cuda.empty_cache()

    excess = []                                 # per chunk and utterance: max over its cells of |err| - rtol·|want|
    rtol = 1e-4 * (1 + u) + u
    gs_dev = dev(gs, torch.float64)

    def sink(bi, ti, ui, want):
        err = (grad[bi, ti, ui].double() - want).abs_().sub_(rtol * want.abs()).amax(dim=1)
        excess.append((bi.cpu().numpy(), err.cpu().numpy()))

    t = time.perf_counter()
    want_costs, _ = r64.op_loss_grad(lambda b, t_, u_: x[b, t_, u_].double(), tuple(x.shape), labels, il, ll, 0, gs,
                                     device="cuda", on_grad=sink)
    torch.cuda.synchronize()
    elapsed = time.perf_counter() - t
    atol = np.abs(gs) * ab_cell(np.abs(want_costs).max()) * (1 + u) + (2.0 ** -25 if dtype == torch.float16 else 0.0)
    bi = np.concatenate([e[0] for e in excess])
    ex = np.concatenate([e[1] for e in excess])
    assert len(bi) == int(np.sum(il * (ll + 1)))
    ratio = np.max(ex / atol[bi])
    print("\nref64 op %s V=%d: costs max rel %.2e, max (|err| - rtol|g|)/atol %.2e, reference %.1f s"
          % (dt, V, np.max(np.abs(costs - want_costs) / np.abs(want_costs)), ratio, elapsed))
    assert_close(costs, want_costs, rtol=1e-4 if u else 1e-5, atol=1e-4 if not u else 1e-5, what="costs")
    assert ratio <= 1.0, ("gradients out of tolerance", ratio)
    for b in range(B):                          # padded cells exactly zero (NaN-prefilled buffer: unwritten ones fail)
        T, U = int(il[b]), int(ll[b]) + 1
        assert not grad[b, T:].ne(0).any() and not grad[b, :T, U:].ne(0).any(), b
