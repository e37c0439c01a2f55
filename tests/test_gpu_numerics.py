"""Value coverage of the loss, against the fp64 oracle: logits far from the ordinary few-nat spread of a row, upstream
gradient scales far from 1, labels equal to blank, garbage in padded activations, and the loss op's kernel-selection
boundaries (V around 1024, unaligned buffers, maxU = 1024, long T, the fp64 entry).

The 16-bit path keeps each row's softmax numerators as bf16 E[row, v] = 2^(y_v - ref_row) against one fp32 reference
per row (DESIGN.md 3.4).  Its gradients are right only where the reference sits close enough to the row maximum, so
these cases move the row maximum far away from the logits the reference starts from: the first 32 logits pushed far
down (`suppressed`), or one column late in the row pushed far up (`dominant`).  Every 16-bit case also checks that
no gradient lost more than half its norm, so that rows dropped from the backward fail with a message saying so."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import assert_close, fp32_tol
from test_gpu_joint import run_joint, synth

pytestmark = pytest.mark.gpu

NAMES = ("d_enc", "d_pred", "dW", "db")
TC_COST_RTOL = 2e-4
PATHS = ("bf16-keep", "bf16-recompute", "fp32")
RNNT_STATUS_INVALID_VALUE = 2


# ---------------------------------------------------------------------------------------------------------- helpers
def oracle_of(oracle, k, gs):
    return oracle.joint_loss_grad(*(k[n].astype(np.float64) for n in ("enc", "pred", "W", "b")), k["labels"],
                                  k["input_lengths"], k["label_lengths"], int(k["blank"]), grad_scale=gs)


def run_path(k, path, gs):
    if path == "fp32":
        return run_joint(k, "fp32", scale=gs)
    return run_joint(k, "bf16", scale=gs, keep=(path == "bf16-keep"))


def check_tc(costs, grads, o):
    """The 16-bit path against the oracle (DESIGN.md 4): costs rtol 2e-4, gradients 1e-2 * max|g| element-wise and
    relative Frobenius error < 5e-3; first, no gradient may have lost half its norm (dropped rows)."""
    assert np.all(np.isfinite(costs)), costs
    assert_close(costs, o["costs"], rtol=TC_COST_RTOL, atol=1e-3, what="costs")
    for g, n in zip(grads, NAMES):
        assert np.all(np.isfinite(g)), n + " is not finite"
        ng, no = np.linalg.norm(g), np.linalg.norm(o[n])
        assert ng >= 0.5 * no, "%s: |g| = %.4g is less than half the oracle's %.4g: rows are missing" % (n, ng, no)
        assert_close(g, o[n], rtol=0, atol=0, ntol=1e-2, what=n)
        rel = np.linalg.norm(g - o[n]) / no
        assert rel < 5e-3, (n, rel)


def check_fp32(costs, grads, o, gs):
    """The fp32 fused path at the tolerances of test_gpu_joint.test_fp32_vs_oracle; the absolute floor follows the
    upstream gradient's scale, and the norm-wise floor the cost's magnitude (conftest.fp32_tol)."""
    cmax = float(np.abs(o["costs"]).max())
    assert_close(costs, o["costs"], rtol=1e-5, atol=1e-4, what="costs")
    for g, n in zip(grads, NAMES):
        assert_close(g, o[n], rtol=1e-4, atol=1e-6 * float(np.abs(gs).max()), ntol=max(1e-5, 2e-7 * cmax), what=n)


def check(path, costs, grads, o, gs):
    if path == "fp32":
        check_fp32(costs, grads, o, gs)
    else:
        check_tc(costs, grads, o)


_CACHE = {}


def cached_oracle(oracle, key, k, gs):
    if key not in _CACHE:
        _CACHE[key] = oracle_of(oracle, k, gs)
    return _CACHE[key]


def suppressed(V, delta, blank, B=2, seed=101):
    """synth() with the first 32 logits of every row pushed delta nats down (b[0:32] -= delta).  With blank = V-1 the
    labels come from [32, V-1), so the lattice itself stays ordinary; with blank = 0 the blank is among them."""
    k = synth(B, 24, 12, V, 128, seed, ragged=True)
    if blank != 0:
        k["labels"] = np.random.default_rng(seed + 1).integers(32, V - 1, k["labels"].shape).astype(np.int32)
    k["blank"] = np.int32(blank)
    k["b"] = k["b"].copy()
    k["b"][:32] -= np.float32(delta)
    return k


BLANKS = {"first": lambda V: 0, "last": lambda V: V - 1}


# ------------------------------------------------------------------- (a) the reference far below the row maximum
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("blank", ["first", "last"])
@pytest.mark.parametrize("V", [128, 1024])
@pytest.mark.parametrize("delta", [0, 30, 50, 75, 100])
def test_first_logits_far_below_row_max(oracle, delta, V, blank, path):
    """The row's first 32 logits, from which the 16-bit forward takes its reference, lie delta nats below the rest."""
    bl = BLANKS[blank](V)
    k = suppressed(V, delta, bl)
    gs = np.linspace(0.5, 1.5, 2)
    o = cached_oracle(oracle, ("a", delta, V, bl), k, gs)
    costs, grads = run_path(k, path, gs)
    check(path, costs, grads, o, gs)


# ------------------------------------------------------------------------- (b) one dominant column late in the row
def dominant(V, delta, variant, seed=202):
    """synth() with one bias column raised by delta nats: a plain column of the last 64-column chunk, a column of that
    chunk that is also the label at every third position, the blank as the last column, or the blank as column 0."""
    k = synth(2, 24, 12, V, 128, seed, ragged=True)
    col = {"plain": V - 23, "label": V - 41, "blank-last": V - 1, "blank-first": 0}[variant]
    k["labels"] = np.random.default_rng(seed + 1).integers(1, V - 64, k["labels"].shape).astype(np.int32)
    if variant == "label":
        k["labels"][:, ::3] = col
    k["blank"] = np.int32(V - 1 if variant == "blank-last" else 0)
    k["b"] = k["b"].copy()
    k["b"][col] += np.float32(delta)
    return k


@pytest.mark.parametrize("V,delta,variant,path", [
    (V, d, var, p) for var in ("plain", "label", "blank-last", "blank-first") for d in (40, 80, 100) for p in PATHS
    for V in (1024,)] + [(4096, 80, "label", "bf16-keep")])
def test_dominant_column(oracle, V, delta, variant, path):
    """One column delta nats above the rest of its row: far above the row's reference when it sits in the last chunk,
    far above the other three lanes of its quad when it is column 0."""
    k = dominant(V, delta, variant)
    gs = np.linspace(0.5, 1.5, 2)
    o = cached_oracle(oracle, ("b", V, delta, variant), k, gs)
    costs, grads = run_path(k, path, gs)
    check(path, costs, grads, o, gs)


def staircase(seed=212):
    """Logits close to the bias, in octaves (log2 units): columns 0-31 (the reference's source) at 0, columns 32-63 at
    61, one column of the second chunk at 66.5, all others at 0.  The forward's reference then stays put through chunk 0
    (61 < 64 above it) and is raised at chunk 1 (66.5 > 64), so the numerators kept for chunk 0 are rescaled after they
    were stored, and they still carry about 40 % of every row's softmax.  Blank and labels lie in columns 32-63."""
    V = 256
    k = synth(2, 24, 12, V, 128, seed, ragged=True)
    k["W"] = (0.1 * k["W"]).astype(np.float32)
    lvl = np.zeros(V)
    lvl[32:64], lvl[69] = 61.0, 66.5
    k["b"] = (lvl * np.log(2.0) + 0.1 * k["b"]).astype(np.float32)
    k["blank"] = np.int32(33)
    k["labels"] = np.random.default_rng(seed + 1).integers(34, 64, k["labels"].shape).astype(np.int32)
    return k


@pytest.mark.parametrize("path", PATHS)
def test_reference_raised_after_earlier_chunks_were_kept(oracle, path):
    """The reference is raised at chunk 1 while chunk 0 holds a large share of the row: a wrong rescale of the numerators
    already kept for chunk 0 shows in every gradient."""
    k = staircase()
    y2 = oracle.joint_forward(*(k[n].astype(np.float64) for n in ("enc", "pred", "W", "b"))) / np.log(2.0)
    ref0 = y2[..., :32].max(-1)
    assert (y2[..., :64].max(-1) - ref0 < 62.5).all() and (y2[..., 64:128].max(-1) - ref0 > 65.5).all()
    p = np.exp2(y2 - y2.max(-1, keepdims=True))
    assert (p[..., 32:64].sum(-1) / p.sum(-1) > 0.3).all()
    gs = np.linspace(0.5, 1.5, 2)
    o = cached_oracle(oracle, ("staircase",), k, gs)
    costs, grads = run_path(k, path, gs)
    check(path, costs, grads, o, gs)


# --------------------------------------------------------------------------------- (c) upstream gradient scale
SCALES = {"1e-6": [1e-6, 1e-6, 1e-6], "2^16": [65536.0, 65536.0, 65536.0], "mixed-sign": [1.0, -0.7, 0.4],
          "one-zero": [0.8, 0.0, 1.2]}


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("delta", [0, 50])
@pytest.mark.parametrize("scale", list(SCALES))
def test_upstream_gradient_scale(oracle, scale, delta, path):
    """Per-utterance upstream gradients far from 1 (a tiny loss weight, fp16-style loss scaling, signs, a zero)."""
    V = 256
    k = suppressed(V, delta, V - 1, B=3, seed=111)
    gs = np.array(SCALES[scale])
    o = cached_oracle(oracle, ("c", scale, delta), k, gs)
    costs, grads = run_path(k, path, gs)
    check(path, costs, grads, o, gs)
    for b in np.flatnonzero(gs == 0):          # a zero upstream gradient contributes exactly nothing
        assert not grads[0][b].any() and not grads[1][b].any()


# ------------------------------------------------------------------------------------- (d) labels equal to blank
@pytest.mark.parametrize("path", PATHS + ("op-fp32", "op-fp64"))
@pytest.mark.parametrize("blank", [0, 5, 127])
def test_labels_equal_to_blank(oracle, blank, path):
    """About a third of the labels are the blank index: the blank's two outgoing arcs then share one logit."""
    B, T, U, V, H = 3, 16, 10, 128, 64
    k = synth(B, T, U, V, H, 404, ragged=True)
    rng = np.random.default_rng(405)
    lab = rng.integers(0, V, (B, U - 1)).astype(np.int32)
    lab[rng.random(lab.shape) < 1 / 3] = blank
    k["labels"], k["blank"] = lab, np.int32(blank)
    assert (lab[0] == blank).sum() >= 2
    gs = np.linspace(0.5, 1.5, B)
    if path.startswith("op"):
        acts = oracle.joint_forward(*(k[n].astype(np.float64) for n in ("enc", "pred", "W", "b")))
        if path == "op-fp64":
            oc, og = oracle.rnnt_logits_grad(acts, lab, k["input_lengths"], k["label_lengths"], blank)
            st, costs, g = abi_loss(acts, lab, k["input_lengths"], k["label_lengths"], blank, fp64=True)
            assert st == 0
            assert_close(costs, oc, rtol=1e-10, atol=0, what="costs")
            assert_close(g, og, rtol=1e-10, atol=1e-10, what="grads")
        else:
            a32 = acts.astype(np.float32)
            oc, og = oracle.rnnt_logits_grad(a32.astype(np.float64), lab, k["input_lengths"], k["label_lengths"], blank)
            st, costs, g = abi_loss(a32, lab, k["input_lengths"], k["label_lengths"], blank)
            assert st == 0
            assert_close(costs, oc, rtol=1e-5, atol=1e-4, what="costs")
            assert_close(g, og, what="grads", **fp32_tol(oc))
        return
    o = oracle_of(oracle, k, gs)
    costs, grads = run_path(k, path, gs)
    check(path, costs, grads, o, gs)


# --------------------------------------------------------------------------------- (e) padded content does not leak
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("garbage", ["pm1e4", "normal100"])
def test_padding_content_does_not_leak(garbage, path):
    """enc[b, T_b:] and pred[b, U_b + 1:] are never part of the loss: large finite values there change nothing."""
    B, T, U, V, H = 3, 24, 12, 256, 128
    k = synth(B, T, U, V, H, 303, ragged=True)
    k["input_lengths"] = np.array([T, 15, 7], np.int32)
    k["label_lengths"] = np.array([U - 1, 6, 3], np.int32)
    rng = np.random.default_rng(304)
    clean, dirty = dict(k), dict(k)
    for n, lens in (("enc", k["input_lengths"]), ("pred", k["label_lengths"] + 1)):
        c, d = k[n].copy(), k[n].copy()
        for b in range(B):
            c[b, lens[b]:] = 0
            shape = d[b, lens[b]:].shape
            d[b, lens[b]:] = (rng.choice([-1e4, 1e4], shape) if garbage == "pm1e4" else 100 * rng.standard_normal(shape))
        clean[n], dirty[n] = c, d.astype(np.float32)
    gs = np.linspace(0.5, 1.5, B)
    c0, g0 = run_path(clean, path, gs)
    c1, g1 = run_path(dirty, path, gs)
    assert np.all(np.isfinite(c1))
    for b in range(B):
        assert not g1[0][b, k["input_lengths"][b]:].any() and not g1[1][b, k["label_lengths"][b] + 1:].any()
    if path == "fp32":                           # dW and d_pred are summed with atomics: not bit-reproducible
        assert_close(c1, c0, rtol=1e-6, atol=0, what="costs")
        for a, b_, n in zip(g1, g0, NAMES):
            assert np.linalg.norm(a - b_) <= 1e-6 * np.linalg.norm(b_), n
    else:
        assert np.array_equal(c1, c0)
        for a, b_, n in zip(g1, g0, NAMES):
            assert np.array_equal(a, b_), n


# ----------------------------------------------------------------------- (f) the loss op's boundaries, via the C ABI
def abi_loss(acts, labels, il, ll, blank=0, fp64=False, offset=0):
    """compute_rnnt_loss[_fp64] as test_gpu_loss_op.c_abi_loss calls it, with acts and grads placed `offset` elements
    past a fresh allocation (offset 1 at fp32: 4 bytes past a 16-byte boundary).  Returns (status, costs, grads)."""
    from rnnt_speech_recognition_b200 import _lib
    L = _lib.load()
    dt = torch.float64 if fp64 else torch.float32
    B, T, U, V = acts.shape
    n = acts.size
    x = torch.empty(n + 16, dtype=dt, device="cuda")[offset:offset + n].view(acts.shape)
    x.copy_(torch.as_tensor(np.ascontiguousarray(acts), dtype=dt))
    g = torch.full((n + 16,), float("nan"), dtype=dt, device="cuda")[offset:offset + n].view(acts.shape)
    if offset:
        assert x.data_ptr() % 16 != 0 and g.data_ptr() % 16 != 0
    lab = torch.as_tensor(np.ascontiguousarray(labels), dtype=torch.int32).cuda() if np.size(labels) else \
        torch.zeros(1, dtype=torch.int32).cuda()
    d_il = torch.as_tensor(np.asarray(il), dtype=torch.int32).cuda()
    d_ll = torch.as_tensor(np.asarray(ll), dtype=torch.int32).cuda()
    sz = C.c_size_t(0)
    assert L.get_workspace_size(T, U, B, True, C.byref(sz), 8 if fp64 else 4) == 0
    ws = torch.empty(sz.value, dtype=torch.uint8, device="cuda")
    costs = np.zeros(B, np.float64 if fp64 else np.float32)
    opt = _lib.RnntOptions(_lib.RNNT_GPU, 0, torch.cuda.current_stream().cuda_stream, blank, T, U, True)
    fn = L.compute_rnnt_loss_fp64 if fp64 else L.compute_rnnt_loss
    st = fn(x.data_ptr(), g.data_ptr(), lab.data_ptr(), d_ll.data_ptr(), d_il.data_ptr(), V, B, costs.ctypes.data,
            ws.data_ptr(), opt)
    torch.cuda.synchronize()
    return st, costs, g.cpu().numpy()


def random_case(B, T, U, V, seed, spread=2.0):
    rng = np.random.default_rng(seed)
    acts = (spread * rng.standard_normal((B, T, U, V))).astype(np.float32)
    labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
    il, ll = rng.integers(1, T + 1, B).astype(np.int32), rng.integers(0, U, B).astype(np.int32)
    il[0], ll[0] = T, U - 1
    return acts, labels, il, ll


def check_op(oracle, acts, labels, il, ll, blank=0, **kw):
    oc, og = oracle.rnnt_logits_grad(acts.astype(np.float64), labels, il, ll, blank)
    st, costs, g = abi_loss(acts, labels, il, ll, blank, **kw)
    assert st == 0
    assert_close(costs, oc, rtol=1e-5, atol=1e-4, what="costs")
    assert_close(g, og, what="grads", **fp32_tol(oc))
    for b in range(acts.shape[0]):                                  # padded cells exactly 0
        assert not g[b, il[b]:].any() and not g[b, :, ll[b] + 1:].any()
    return costs, g


@pytest.mark.parametrize("V", [1024, 1028, 2048, 4096])
def test_op_vocabulary_around_the_register_path(oracle, V):
    """V <= 1024 keeps a row in registers, V > 1024 takes the two-pass kernels."""
    check_op(oracle, *random_case(2, 10, 7, V, 500 + V))


@pytest.mark.parametrize("V", [128, 2048])
def test_op_unaligned_buffers(oracle, V):
    """acts and grads 4 bytes past a 16-byte boundary with V % 4 == 0: the scalar kernels, against the oracle and
    against the vectorised kernels of the aligned call."""
    case = random_case(3, 12, 9, V, 600 + V)
    c0, g0 = check_op(oracle, *case)
    c1, g1 = check_op(oracle, *case, offset=1)
    assert_close(c1, c0, rtol=1e-5, atol=1e-4, what="costs")
    assert_close(g1, g0, what="grads", **fp32_tol(c0))


def test_op_max_label_positions(oracle):
    """maxU = 1024, the documented limit of the alpha/beta wavefront (32 warps), ragged label lengths."""
    B, T, U, V = 3, 6, 1024, 64
    acts, labels, _, _ = random_case(B, T, U, V, 700, spread=1.0)
    check_op(oracle, acts, labels, np.array([T, 4, 5], np.int32), np.array([1023, 500, 0], np.int32))


@pytest.mark.parametrize("keep", [True, False])
def test_fused_max_label_positions(oracle, keep):
    B, T, U, V, H = 3, 6, 1024, 64, 64
    k = synth(B, T, U, V, H, 701, ragged=False)
    k["input_lengths"] = np.array([T, 4, 5], np.int32)
    k["label_lengths"] = np.array([1023, 500, 0], np.int32)
    gs = np.linspace(0.5, 1.5, B)
    o = cached_oracle(oracle, ("maxU", 1024), k, gs)
    costs, grads = run_joint(k, "bf16", scale=gs, keep=keep)
    check_tc(costs, grads, o)


def test_op_rejects_more_than_1024_label_positions():
    acts = np.zeros((1, 2, 1025, 4), np.float32)
    st, _, _ = abi_loss(acts, np.ones((1, 1024), np.int32), [2], [1024])
    assert st == RNNT_STATUS_INVALID_VALUE


def test_op_long_input(oracle):
    """T = 2000, U = 40: many macro steps of the wavefront."""
    check_op(oracle, *random_case(2, 2000, 40, 16, 800))


def test_fp64_entry_wide_ragged(oracle):
    """compute_rnnt_loss_fp64 at U = 257 (nine warps of the wavefront), ragged, against the fp64 oracle."""
    rng = np.random.default_rng(900)
    B, T, U, V = 3, 20, 257, 10
    acts = 2 * rng.standard_normal((B, T, U, V))
    labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
    il, ll = np.array([T, 13, 7], np.int32), np.array([256, 100, 31], np.int32)
    oc, og = oracle.rnnt_logits_grad(acts, labels, il, ll)
    st, costs, g = abi_loss(acts, labels, il, ll, fp64=True)
    assert st == 0
    assert_close(costs, oc, rtol=1e-10, atol=0, what="costs")
    assert_close(g, og, rtol=1e-10, atol=1e-10, what="grads")


@pytest.mark.parametrize("blank", ["first", "last"])
@pytest.mark.parametrize("delta", [0, 100])
def test_op_on_suppressed_logits(oracle, delta, blank):
    """Section (a)'s logits, materialised: the op's max-subtracted fp32 softmax has no reference to lose."""
    V = 1024
    bl = BLANKS[blank](V)
    k = suppressed(V, delta, bl)
    acts = oracle.joint_forward(*(k[n].astype(np.float64) for n in ("enc", "pred", "W", "b"))).astype(np.float32)
    check_op(oracle, acts, k["labels"], k["input_lengths"], k["label_lengths"], bl)
