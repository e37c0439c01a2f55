"""The loss paths past 2^31-element buffers, and the fp32 exact joint path across its row chunks.

Production batches (BASELINE C5, V = 4096) hold far more than 2^31 logits, logit gradients or kept numerators per
buffer.  The big buffers here are mostly padding and every valid lattice is small enough for the float64 references:
  * a small valid lattice is placed so that some of its cells lie past element 2^31, or a row-chunk boundary of the fp32
    exact joint path falls inside it; host-side geometry checks assert that placement (`test_placement_geometry` runs
    them without a GPU, and every GPU case repeats its own);
  * only each utterance's valid [:T_b, :U_b] block goes to the host, against the float64 oracle (`oracle`,
    `fastemit_ref`, `align_ref`) or against a run of the same utterances in a buffer below 2^31;
  * gradient buffers are NaN-prefilled through the C ABI, so a row the kernels never write fails, and padded cells
    are checked to be exactly zero on the device.
Tolerances are those of DESIGN.md 4 for each path.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import align_ref as ar
import fastemit_ref as fr
from conftest import ROOT, assert_close, fp32_tol
from test_gpu_align import OP_TOL, check as align_check

TWO31 = 2 ** 31
NAN = float("nan")
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
NAMES = ("d_enc", "d_pred", "dW", "db")


# ------------------------------------------------------------------------------------------------ placement on the host
def cell_offset(b, t, u, maxT, maxU, V):
    """Element offset of the first logit of lattice cell (b, t, u) in a (B, maxT, maxU, V) buffer."""
    return ((b * maxT + t) * maxU + u) * V


def crossing_frame(maxT, maxU, V, lengths):
    """Where the LAST utterance of a (B, maxT, maxU, V) buffer crosses element 2^31.  Asserts that the earlier
    utterances' valid cells lie below it, and that the last utterance's lattice straddles it: frame 0 lies wholly below
    2^31 and every frame from t0 on wholly past it, with 0 < t0 < T_b - 1 (the wavefront crosses it mid-lattice).
    Returns t0."""
    B = len(lengths)
    assert all(T <= maxT and U <= maxU for T, U in lengths)
    for b, (T, U) in enumerate(lengths[:-1]):
        assert cell_offset(b, T - 1, U - 1, maxT, maxU, V) + V <= TWO31, b
    b, (T, U) = B - 1, lengths[-1]
    assert cell_offset(b, 0, U - 1, maxT, maxU, V) + V <= TWO31
    past = [t for t in range(T) if cell_offset(b, t, 0, maxT, maxU, V) >= TWO31]
    assert past, "utterance %d lies wholly below 2^31" % b
    t0 = past[0]
    assert 0 < t0 < T - 1, (t0, T)
    return t0


def kept_row_offset(lengths, maxT, maxU, V, subsets):
    """Case C's placement.  The keeping forward ranks the valid 16 x 8 tiles in utterance order, 128 rows of V numerators
    each, so the last utterance's first kept numerator sits at element valid_tile_count(earlier utterances) * 128 * V of
    E.  Asserts that this is >= 2^31, and that each sub-batch in `subsets` (the reference runs) keeps fewer than 2^31
    numerators.  Returns the offset."""
    import rnnt_speech_recognition_b200 as rb
    il, ll = [T for T, _ in lengths], [U - 1 for _, U in lengths]
    first = rb.valid_tile_count(il[:-1], ll[:-1]) * 128 * V
    assert first >= TWO31, first
    for idx in subsets:
        assert rb.valid_tile_count([il[i] for i in idx], [ll[i] for i in idx]) * 128 * V <= TWO31, idx
    return first


def exact_chunk_rows(H, V, N):
    """Lattice rows per chunk of the fp32 exact joint path (JointWs: Z, L and dZ of a chunk in 1 GiB, >= 256 rows)."""
    return min(N, max(256, 2 ** 30 // ((2 * H + V) * 4)))


def chunk_boundaries(H, V, maxT, maxU, lengths):
    """The fp32 exact path's row-chunk boundaries of a batch.  Asserts that there is at least one and that each falls
    strictly inside a valid lattice: cell (b, t, u) with 0 < t < T_b - 1 and 0 < u < U_b - 1.  Returns (rows per chunk,
    boundary cells)."""
    N = len(lengths) * maxT * maxU
    rows = exact_chunk_rows(H, V, N)
    cells = []
    for r in range(rows, N, rows):
        b, rem = divmod(r, maxT * maxU)
        t, u = divmod(rem, maxU)
        T, U = lengths[b]
        assert 0 < t < T - 1 and 0 < u < U - 1, ("chunk boundary outside a valid lattice", r, b, t, u, T, U)
        cells.append((b, t, u))
    assert cells, "the batch is one chunk"
    return rows, cells


# The lattices that cross 2^31 or a chunk boundary are kept to about a hundred wavefront steps: there the fp32 paths hold
# the tolerances of DESIGN.md 4.  (On a 1024 x 40 lattice of random logits, cost ~9e3, fp32 round-off of alpha and beta
# reaches about 2e-6 * |cost| per gradient entry, twice the per-cell floor; that is a limit of fp32, not of the offsets.)
# So the padding in front of them is spread over more utterances instead.

# Case A: B = 11, maxT = 1024, maxU * V ~ 209 000 (2.35e9 logits).  Utterances 0-9 are short; utterance 10 (T = 48,
# U = 40: two warps of the wavefront) starts below element 2^31 and crosses it at frame 41 (31 at V = 1025).
OP_MAXT = 1024
OP_MAXU = {1024: 204, 1025: 204, 4096: 51}
OP_LENGTHS = {V: ((61, 9), (23, 34), (5, 1), (40, 12), (1, 7), (17, 3), (64, 33), (9, 20), (33, 2), (12, 15), (48, 40))
              for V in OP_MAXU}
LOGITS_FRAMES = 940                      # case B compares utterance 2's frames from here on

# Case C: 8 full utterances fill exactly 2^31 kept numerators; every kept row of utterance 8 lies past them.
TC = dict(maxT=512, maxU=128, V=4096, H=640)
TC_LENGTHS = ((512, 128),) * 8 + ((150, 30),)
TC_SUBSETS = (range(0, 4), range(4, 8), range(8, 9))
PLANT = dict(u=13, col=TC["V"] - 23, nats=60.0)

# Case D: two row chunks, the boundary inside the last utterance's lattice; sgemm128_kernel, and the generic sgemm_kernel
# at V % 4 != 0.  Short utterances in front, as many as put the boundary there.
EXACT = {"sgemm128": dict(H=256, V=1024, maxT=32, maxU=32, B=171, last=(24, 14)),
         "sgemm": dict(H=70, V=130, maxT=64, maxU=64, B=243, last=(48, 32))}


def exact_lengths(layout):
    e = EXACT[layout]
    rng = np.random.default_rng(e["B"])
    T = rng.integers(1, e["maxT"] // 4 + 1, e["B"] - 1)
    U = rng.integers(1, e["maxU"] // 8 + 1, e["B"] - 1)
    return tuple((int(t), int(u)) for t, u in zip(T, U)) + (e["last"],)


def exact_boundaries(layout):
    e = EXACT[layout]
    return chunk_boundaries(e["H"], e["V"], e["maxT"], e["maxU"], exact_lengths(layout))


def test_placement_geometry():
    """The host-side placement checks of the GPU cases below, with the numbers they are built around."""
    assert {V: crossing_frame(OP_MAXT, OP_MAXU[V], V, OP_LENGTHS[V]) for V in OP_MAXU} == {1024: 41, 1025: 31, 4096: 41}
    full = ((OP_MAXT, 700),) * 2 + ((OP_MAXT, 1),)
    assert LOGITS_FRAMES < crossing_frame(OP_MAXT, 700, 1024, full)
    assert kept_row_offset(TC_LENGTHS, TC["maxT"], TC["maxU"], TC["V"], TC_SUBSETS) == TWO31
    assert exact_boundaries("sgemm128") == (174762, [(170, 21, 10)])
    assert exact_boundaries("sgemm") == (994205, [(242, 46, 29)])
    # a placement that stops testing what it claims fails the check
    with pytest.raises(AssertionError):
        crossing_frame(OP_MAXT, 204, 1024, OP_LENGTHS[1024][:-1] + ((40, 40),))     # the last utterance wholly below 2^31
    with pytest.raises(AssertionError):
        kept_row_offset(((512, 128),) * 7 + ((150, 30),), 512, 128, 4096, ())      # 7 full utterances: below 2^31
    short = exact_lengths("sgemm128")[:-1]
    with pytest.raises(AssertionError):
        chunk_boundaries(256, 1024, 32, 32, short + ((22, 14),))                    # boundary on the last frame
    with pytest.raises(AssertionError):
        chunk_boundaries(256, 1024, 32, 32, short + ((24, 11),))                    # boundary on the last label position


# ------------------------------------------------------------------------------------------------------------ helpers
@pytest.fixture(autouse=True)
def _release_device_memory():
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def dev(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def lengths_of(lengths):
    return np.array([T for T, _ in lengths], np.int32), np.array([U - 1 for _, U in lengths], np.int32)


def check_alignment(al, log_probs_of, labels, il, ll, blank, tol):
    """test_gpu_align's score criterion and path identity, one utterance at a time on its valid block."""
    for b in range(len(il)):
        U = int(ll[b]) + 1
        one = type(al)(al.label_frames[b:b + 1, :U - 1], al.best_logp[b:b + 1], al.costs[b:b + 1])
        align_check(one, log_probs_of(b), labels[b:b + 1, :U - 1], il[b:b + 1], ll[b:b + 1], blank, tol)


# --------------------------------------------------------------------------------- A. the loss op past 2^31 logits
def op_case(V, dtype, seed):
    """(11, 1024, maxU, V) logits, 2 * N(0, 1) drawn on the device in the logits' own dtype (padded cells included), and
    the lengths of OP_LENGTHS."""
    B, maxU = len(OP_LENGTHS[V]), OP_MAXU[V]
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.empty(B, OP_MAXT, maxU, V, dtype=dtype, device="cuda")
    for b in range(B):
        x[b].normal_(0.0, 2.0, generator=g)
    labels = np.random.default_rng(seed).integers(1, V, (B, maxU - 1)).astype(np.int32)
    il, ll = lengths_of(OP_LENGTHS[V])
    return x, labels, il, ll


def op_workspace(x):
    from rnnt_speech_recognition_b200 import _lib
    B, T, U, _ = x.shape
    sz = C.c_size_t(0)
    assert _lib.load().get_workspace_size(T, U, B, True, C.byref(sz), 4) == 0
    return torch.empty(sz.value, dtype=torch.uint8, device="cuda")


def op_options(x, blank=0):
    from rnnt_speech_recognition_b200 import _lib
    return _lib.RnntOptions(_lib.RNNT_GPU, 0, torch.cuda.current_stream().cuda_stream, blank, x.shape[1], x.shape[2], True)


def op_fp32(x, d, entry, gs=None):
    """fp32 logits through compute_rnnt_loss (host costs) or rnntb200_loss_device (device costs, upstream gradients gs),
    with a NaN-prefilled gradient buffer.  Returns (costs, gradients)."""
    from rnnt_speech_recognition_b200 import _lib
    L, p = _lib.load(), _lib.ptr
    B, _, _, V = x.shape
    ws, g = op_workspace(x), torch.full_like(x, NAN)
    if entry == "compute_rnnt_loss":
        costs = np.zeros(B, np.float32)
        st = L.compute_rnnt_loss(p(x), p(g), p(d["lab"]), p(d["ll"]), p(d["il"]), V, B, costs.ctypes.data, p(ws),
                                 op_options(x))
    else:
        c = torch.full((B,), NAN, device="cuda")
        st = L.rnntb200_loss_device(p(x), p(g), p(d["lab"]), p(d["ll"]), p(d["il"]), p(dev(gs, torch.float32)), V, B,
                                    p(c), p(ws), op_options(x))
        costs = c.cpu().numpy()
    _lib.check(st, entry)
    torch.cuda.synchronize()
    return costs, g


def op16_forward(x, d):
    from rnnt_speech_recognition_b200 import _lib
    L, p = _lib.load(), _lib.ptr
    B, _, _, V = x.shape
    ws, c = op_workspace(x), torch.full((B,), NAN, device="cuda")
    kind = _lib.LOGITS_F16 if x.dtype == torch.float16 else _lib.LOGITS_BF16
    _lib.check(L.rnntb200_loss16_forward(p(x), kind, p(d["lab"]), p(d["ll"]), p(d["il"]), V, B, p(c), p(ws), op_options(x)),
               "rnntb200_loss16_forward")
    return c.cpu().numpy(), ws


def op16_backward(x, d, ws, gs, fastemit_lambda=0.0):
    """The 16-bit backward into a NaN-prefilled gradient buffer, from the workspace of op16_forward (read only)."""
    from rnnt_speech_recognition_b200 import _lib
    L, p = _lib.load(), _lib.ptr
    B, _, _, V = x.shape
    g = torch.full_like(x, NAN)
    kind = _lib.LOGITS_F16 if x.dtype == torch.float16 else _lib.LOGITS_BF16
    _lib.check(L.rnntb200_loss16_backward_fastemit(p(x), kind, p(d["lab"]), p(d["ll"]), p(d["il"]), p(dev(gs, torch.float32)),
                                                   V, B, p(g), p(ws), op_options(x), fastemit_lambda),
               "rnntb200_loss16_backward_fastemit")
    torch.cuda.synchronize()
    return g


def valid_blocks(x, il, ll):
    """Each utterance's valid logits block (1, T_b, U_b, V), exactly widened to float64 on the host."""
    return [x[b:b + 1, :int(il[b]), :int(ll[b]) + 1].cpu().double().numpy() for b in range(x.shape[0])]


def oracle_per_utterance(oracle, blocks, labels, il, ll):
    """float64 costs (B,) and logits gradients (one (1, T_b, U_b, V) array per utterance) of the valid blocks."""
    costs, grads = [], []
    for b, xb in enumerate(blocks):
        oc, og = oracle.rnnt_logits_grad(xb, labels[b:b + 1, :int(ll[b])], il[b:b + 1], ll[b:b + 1])
        costs.append(oc[0])
        grads.append(og)
    return np.array(costs), grads


def check_blocks(g, wants, il, ll, rtol, atols, what):
    """The valid block of each utterance of the device gradient g against wants[b] (host copy of that block only), and
    every padded cell exactly zero (on the device: NaN counts as non-zero, so an unwritten padded row fails too)."""
    for b, want in enumerate(wants):
        T, U = int(il[b]), int(ll[b]) + 1
        got = g[b:b + 1, :T, :U].float().cpu().numpy()
        assert_close(got, want, rtol=rtol, atol=atols[b], what="%s, utterance %d" % (what, b))
        assert not g[b, T:].ne(0).any() and not g[b, :T, U:].ne(0).any(), "%s: padded cells of utterance %d" % (what, b)


def alone(x, labels, il, ll):
    """The last utterance alone, in a buffer of its own valid extent (below 2^31), with its device labels / lengths, and
    its block of a gradient of the whole batch."""
    b = x.shape[0] - 1
    T, U = int(il[b]), int(ll[b]) + 1
    return (x[b:, :T, :U].contiguous(), dict(lab=dev(labels[b:, :U - 1]), il=dev(il[b:]), ll=dev(ll[b:])),
            lambda g: g[b, :T, :U])


def mixed_signs(B):
    return np.linspace(0.5, 1.5, B) * np.where(np.arange(B) % 3 == 1, -1.0, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1024, 4096, 1025])
def test_op_fp32_past_2_31(oracle, V):
    """compute_rnnt_loss and rnntb200_loss_device on 2.35e9 fp32 logits: the register (V = 1024), two-pass (4096) and
    scalar (1025) kernels, gradients and alignment of cells past element 2^31 against the float64 references."""
    import rnnt_speech_recognition_b200 as rb
    crossing_frame(OP_MAXT, OP_MAXU[V], V, OP_LENGTHS[V])
    x, labels, il, ll = op_case(V, torch.float32, seed=V)
    B = x.shape[0]
    d = dict(lab=dev(labels), il=dev(il), ll=dev(ll))
    blocks = valid_blocks(x, il, ll)
    oc, og = oracle_per_utterance(oracle, blocks, labels, il, ll)
    atol = fp32_tol(oc)["atol"]

    costs, g = op_fp32(x, d, "compute_rnnt_loss")
    assert_close(costs, oc, rtol=1e-5, atol=1e-4, what="costs")
    check_blocks(g, og, il, ll, 1e-4, [atol] * B, "compute_rnnt_loss grads")
    del g
    gs = mixed_signs(B)
    dcosts, g = op_fp32(x, d, "rnntb200_loss_device", gs)
    assert np.array_equal(dcosts, costs)
    check_blocks(g, [s * o for s, o in zip(gs, og)], il, ll, 1e-4, [abs(s) * atol for s in gs], "rnntb200_loss_device grads")

    x2, d2, block = alone(x, labels, il, ll)   # bit for bit: every cell's arithmetic is independent of its place
    c2, g2 = op_fp32(x2, d2, "rnntb200_loss_device", gs[-1:])
    assert c2[0] == dcosts[-1]
    assert torch.equal(g2[0], block(g))
    del g, g2

    al = rb.rnnt_align(x, d["lab"], d["il"], d["ll"])
    assert np.array_equal(al.costs.cpu().numpy(), dcosts)
    check_alignment(al, lambda b: ar.log_probs(blocks[b]), labels, il, ll, 0, OP_TOL)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1024, 4096, 1025])
@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_op16_past_2_31(oracle, dt, V):
    """rnntb200_loss16_forward / _backward on 2.35e9 16-bit logits at upstream gradients 1/B and 2^16/B (bf16 at V = 1024
    also with FastEmit lambda = 0.5), and rnnt_align, against the float64 references on the 16-bit values.  Tolerances
    of tests/test_gpu_mixed_precision.py (DESIGN.md 4)."""
    import rnnt_speech_recognition_b200 as rb
    dtype = DT[dt]
    u = UNIT[dtype]
    crossing_frame(OP_MAXT, OP_MAXU[V], V, OP_LENGTHS[V])
    x, labels, il, ll = op_case(V, dtype, seed=V + len(dt))
    B = x.shape[0]
    d = dict(lab=dev(labels), il=dev(il), ll=dev(ll))
    blocks = valid_blocks(x, il, ll)
    oc, og = oracle_per_utterance(oracle, blocks, labels, il, ll)
    costs, ws = op16_forward(x, d)
    assert_close(costs, oc, rtol=1e-4, atol=1e-5, what="costs")
    rtol = 1e-4 * (1 + u) + u

    def atols(gs):
        return [abs(s) * fp32_tol(oc)["atol"] * (1 + u) + (2.0 ** -25 if dtype == torch.float16 else 0) for s in gs]

    x2, d2, block = alone(x, labels, il, ll)
    c2, ws2 = op16_forward(x2, d2)
    assert c2[0] == costs[-1]
    for name, gs in (("1/B", np.full(B, 1 / B)), ("2^16/B", np.full(B, 2.0 ** 16 / B))):
        g = op16_backward(x, d, ws, gs)
        check_blocks(g, [s * o for s, o in zip(gs, og)], il, ll, rtol, atols(gs), "grads at " + name)
        g2 = op16_backward(x2, d2, ws2, gs[-1:])
        assert torch.equal(g2[0], block(g))
        del g, g2
    if dt == "bf16" and V == 1024:
        gs, lam = np.full(B, 1 / B), 0.5
        g = op16_backward(x, d, ws, gs, lam)
        want = [fr.logits_grad(xb, labels[b:b + 1, :int(ll[b])], il[b:b + 1], ll[b:b + 1], 0, lam, gs[b:b + 1])[1]
                for b, xb in enumerate(blocks)]
        check_blocks(g, want, il, ll, rtol, atols(gs), "grads at lambda = 0.5")
        del g

    al = rb.rnnt_align(x, d["lab"], d["il"], d["ll"])
    assert np.array_equal(al.costs.cpu().numpy(), costs)
    check_alignment(al, lambda b: ar.log_probs(blocks[b]), labels, il, ll, 0, OP_TOL)


# ------------------------------------------------------------------------------- B. joint_logits past 2^31 outputs
@pytest.mark.gpu
def test_joint_logits_past_2_31():
    """rnntb200_joint_logits into a NaN-prefilled (3, 1024, 700, 1024) buffer: every logit is written, and utterance 2's
    frames 940..1023 (the last 2^31 boundary crossing at frame 948) match float64 tanh(enc + pred) @ W + b."""
    from rnnt_speech_recognition_b200 import _lib, joint as J
    B, maxT, maxU, V, H = 3, OP_MAXT, 700, 1024, 64
    assert LOGITS_FRAMES < crossing_frame(maxT, maxU, V, ((maxT, maxU),) * 2 + ((maxT, 1),))
    rng = np.random.default_rng(77)
    enc, pred = rng.standard_normal((B, maxT, H)).astype(np.float32), rng.standard_normal((B, maxU, H)).astype(np.float32)
    W, bias = (rng.standard_normal((H, V)) / np.sqrt(H)).astype(np.float32), (0.1 * rng.standard_normal(V)).astype(np.float32)
    t = [dev(a) for a in (enc, pred, W, bias)]
    desc = J._desc(B, maxT, maxU, H, V, 0, "fp32")
    ws = J._workspace(desc, "cuda")
    out = torch.full((B, maxT, maxU, V), NAN, device="cuda")
    _lib.check(_lib.load().rnntb200_joint_logits(C.byref(desc), *map(_lib.ptr, t), _lib.ptr(out), _lib.ptr(ws)),
               "rnntb200_joint_logits")
    assert not torch.isnan(out).any()
    us = [0, 1, 31, 32, 350, 697, 698, 699]
    got = out[2, LOGITS_FRAMES:][:, us].cpu().numpy()
    z = np.tanh(enc[2, LOGITS_FRAMES:, None, :].astype(np.float64) + pred[2][us][None].astype(np.float64))
    assert_close(got, z @ W.astype(np.float64) + bias, rtol=1e-5, atol=2e-5, what="logits")


# ------------------------------------------------------------------------- C/D. the joint paths through the C ABI
def synth_case(lengths, maxT, maxU, V, H, seed):
    """tests/test_gpu_joint.synth's distributions at the given lengths."""
    B = len(lengths)
    rng = np.random.default_rng(seed)
    il, ll = lengths_of(lengths)
    return dict(enc=rng.standard_normal((B, maxT, H)).astype(np.float32),
                pred=rng.standard_normal((B, maxU, H)).astype(np.float32),
                W=(rng.standard_normal((H, V)) / np.sqrt(H)).astype(np.float32),
                b=(0.1 * rng.standard_normal(V)).astype(np.float32),
                labels=rng.integers(1, V, (B, maxU - 1)).astype(np.int32), blank=np.int32(0),
                input_lengths=il, label_lengths=ll)


def sub(k, idx):
    o = dict(k)
    for n in ("enc", "pred", "labels", "input_lengths", "label_lengths"):
        o[n] = np.ascontiguousarray(k[n][list(idx)])
    return o


def joint_abi(k, precision, gs=None, keep=True, valid_tiles=None, fastemit_lambda=0.0):
    """rnntb200_joint_loss_forward, then (gs given) rnntb200_joint_loss_backward_fastemit into NaN-prefilled d_enc,
    d_pred, dW, db.  Returns costs and the four gradients (None without gs) as numpy."""
    from rnnt_speech_recognition_b200 import _lib, joint as J
    L, p = _lib.load(), _lib.ptr
    t = [dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    (B, maxT, H), (maxU, V) = t[0].shape, (t[1].shape[1], t[2].shape[1])
    desc = J._desc(B, maxT, maxU, H, V, int(k["blank"]), precision, keep, valid_tiles)
    ws = J._workspace(desc, "cuda")
    args = [p(a) for a in t + [lab, ll, il]]
    costs = torch.full((B,), NAN, device="cuda")
    _lib.check(L.rnntb200_joint_loss_forward(C.byref(desc), *args, p(costs), p(ws)), "rnntb200_joint_loss_forward")
    grads = None
    if gs is not None:
        g = [torch.full_like(a, NAN) for a in t]
        _lib.check(L.rnntb200_joint_loss_backward_fastemit(C.byref(desc), *args, p(dev(gs, torch.float32)), *map(p, g), p(ws),
                                                           float(fastemit_lambda)), "rnntb200_joint_loss_backward_fastemit")
        grads = [a.cpu().numpy() for a in g]
    torch.cuda.synchronize()
    return costs.cpu().numpy(), grads


def joint_reference(oracle, k, gs, fastemit_lambda=0.0):
    """The float64 reference of a batch from one call per utterance on its valid block: costs, d_enc / d_pred (zero in
    the padding), dW and db summed over the utterances.  lambda > 0: tests/fastemit_ref.py, else the C oracle."""
    B, maxT, H = k["enc"].shape
    maxU, V = k["pred"].shape[1], k["W"].shape[1]
    out = dict(costs=np.zeros(B), d_enc=np.zeros((B, maxT, H)), d_pred=np.zeros((B, maxU, H)), dW=np.zeros((H, V)),
               db=np.zeros(V))
    W, bias = k["W"].astype(np.float64), k["b"].astype(np.float64)
    for b in range(B):
        T, U = int(k["input_lengths"][b]), int(k["label_lengths"][b]) + 1
        args = (k["enc"][b:b + 1, :T].astype(np.float64), k["pred"][b:b + 1, :U].astype(np.float64), W, bias,
                k["labels"][b:b + 1, :U - 1], k["input_lengths"][b:b + 1], k["label_lengths"][b:b + 1], int(k["blank"]))
        if fastemit_lambda:
            r = fr.joint_loss_grad(*args, grad_scale=gs[b:b + 1], fastemit_lambda=fastemit_lambda)
        else:
            r = oracle.joint_loss_grad(*args, grad_scale=gs[b:b + 1])
        out["costs"][b] = r["costs"][0]
        out["d_enc"][b, :T], out["d_pred"][b, :U] = r["d_enc"][0], r["d_pred"][0]
        out["dW"] += r["dW"]
        out["db"] += r["db"]
    return out


def assert_padding_zero(k, grads, what):
    for b in range(len(k["input_lengths"])):
        assert not grads[0][b, k["input_lengths"][b]:].any(), (what, "d_enc", b)
        assert not grads[1][b, k["label_lengths"][b] + 1:].any(), (what, "d_pred", b)


# ------------------------------------------------------------- C. tensor-core joint, kept numerators past 2^31
def tc_case():
    """B = 9 at maxT = 512, maxU = 128, V = 4096, H = 640: utterances 0-7 full, utterance 8 T = 150, U = 30.  Hidden unit
    H-1 is 0 in enc and pred except pred[8, 13] = 10, and W[H-1] is 0 except W[H-1, V-23] = 60: so in utterance 8's rows
    at u = 13 (and nowhere else) column V-23 of the last 64-column chunk lies 60 nats above the row's first 32 logits
    (tests/test_gpu_numerics.py's dominant column), and the forward rescales numerators it stored past 2^31."""
    k = synth_case(TC_LENGTHS, TC["maxT"], TC["maxU"], TC["V"], TC["H"], 808)
    h, col = TC["H"] - 1, PLANT["col"]
    k["enc"][:, :, h] = 0.0
    k["pred"][:, :, h] = 0.0
    k["pred"][8, PLANT["u"], h] = 10.0
    k["W"][h] = 0.0
    k["W"][h, col] = PLANT["nats"]
    k["labels"][k["labels"] == col] = 1
    return k


@pytest.fixture(scope="module")
def tc(oracle):
    """Case C's inputs, the float64 reference of utterance 8, and the keep-mode runs of the sub-batches {0-3}, {4-7}, {8}
    (each below 2^31 kept numerators)."""
    kept_row_offset(TC_LENGTHS, TC["maxT"], TC["maxU"], TC["V"], TC_SUBSETS)
    k = tc_case()
    B = len(TC_LENGTHS)
    gs = np.full(B, 1.0 / B)
    ref8 = joint_reference(oracle, sub(k, [8]), gs[8:])
    subs = [(idx,) + joint_abi(sub(k, idx), "bf16", gs[list(idx)]) for idx in TC_SUBSETS]
    return k, gs, ref8, subs


_C5_CHILD = r"""
import sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import rnnt_speech_recognition_b200 as rb
from rnnt_speech_recognition_b200 import _lib
from test_gpu_large_offsets import joint_abi
k = dict(np.load(sys.argv[3]))
_lib.set_timing(True)
costs, grads = joint_abi(k, "bf16", k["gs"], keep=True, valid_tiles=rb.valid_tile_count(k["input_lengths"], k["label_lengths"]))
np.savez(sys.argv[4], costs=costs, d_enc=grads[0], d_pred=grads[1], dW=grads[2], db=grads[3],
         kernels=np.array(sorted({n for n, _ in _lib.get_timings()})))
"""


def c5_mode(tmp_path, k, gs):
    """The batch as BASELINE C5 runs it, in a child process (the chunk budget is read once per process): a 1 GiB chunk
    budget, which the padded batch exceeds, and valid_tiles = valid_tile_count(lengths), which makes it one compact chunk
    in keep mode."""
    inp, out = str(tmp_path / "c5_in.npz"), str(tmp_path / "c5_out.npz")
    np.savez(inp, gs=gs, **k)
    subprocess.run([sys.executable, "-c", _C5_CHILD, ROOT, os.path.join(ROOT, "tests"), inp, out], check=True,
                   env=dict(os.environ, RNNTB200_CHUNK_MB="1024"), timeout=600)
    o = dict(np.load(out))
    kernels = " ".join(str(n) for n in o["kernels"])
    assert "<fwd+keep>" in kernels and "<fwd>" not in kernels, kernels       # one keeping forward, nothing recomputed
    return o["costs"], [o[n] for n in NAMES]


def check_tc_tolerance(got, want, what):
    """The tensor-core path against the float64 oracle (DESIGN.md 4): no gradient may lose half its norm, then 1e-2 *
    max|g| element-wise and relative Frobenius error < 5e-3."""
    assert np.all(np.isfinite(got)), what
    ng, no = np.linalg.norm(got), np.linalg.norm(want)
    assert ng >= 0.5 * no, "%s: |g| = %.4g is less than half the oracle's %.4g" % (what, ng, no)
    assert_close(got, want, rtol=0, atol=0, ntol=1e-2, what=what)
    assert np.linalg.norm(got - want) / no < 5e-3, what


@pytest.mark.gpu
def test_tc_kept_numerators_past_2_31(tc, tmp_path):
    """The tensor-core joint at V = 4096, H = 640 with utterance 8's kept numerators all past element 2^31, in keep mode,
    recompute mode and C5's one-chunk valid_tiles mode: utterance 8 against the float64 oracle and against a run of it
    alone, dW / db against the sum of the sub-batch runs, costs bit-identical across the modes."""
    k, gs, ref8, subs = tc
    T8, U8 = TC_LENGTHS[8]
    dW_sum = sum(s[2][2].astype(np.float64) for s in subs)
    db_sum = sum(s[2][3].astype(np.float64) for s in subs)
    alone_grads = subs[-1][2]
    runs = {"keep": joint_abi(k, "bf16", gs, keep=True), "recompute": joint_abi(k, "bf16", gs, keep=False),
            "valid-tiles": c5_mode(tmp_path, k, gs)}
    for mode, (costs, grads) in runs.items():
        for g, n in zip(grads, NAMES):
            assert np.all(np.isfinite(g)), (mode, n)                         # NaN-prefilled: every entry was written
        assert_padding_zero(k, grads, mode)
        assert_close(costs[8:], ref8["costs"], rtol=2e-4, atol=1e-3, what=mode + " costs[8]")
        check_tc_tolerance(grads[0][8:], ref8["d_enc"], mode + " d_enc[8]")
        check_tc_tolerance(grads[1][8:], ref8["d_pred"], mode + " d_pred[8]")
        # batch additivity (tests/test_gpu_fullsize.py's tolerances): the sub-batches keep fewer than 2^31 numerators
        for idx, c, g in subs:
            assert_close(costs[list(idx)], c, rtol=1e-6, atol=1e-3, what="%s costs of %s" % (mode, idx))
        assert_close(grads[0][8:], alone_grads[0], rtol=1e-4, atol=0, ntol=1e-4, what=mode + " d_enc[8] alone")
        assert_close(grads[1][8:], alone_grads[1], rtol=1e-4, atol=0, ntol=1e-4, what=mode + " d_pred[8] alone")
        assert_close(grads[2], dW_sum, rtol=0, atol=0, ntol=5e-4, what=mode + " dW additivity")
        assert_close(grads[3], db_sum, rtol=0, atol=0, ntol=5e-4, what=mode + " db additivity")
    assert np.array_equal(runs["keep"][0], runs["recompute"][0])
    assert np.array_equal(runs["keep"][0], runs["valid-tiles"][0])


# ---------------------------------------------------------------------------- D. fp32 exact joint across row chunks
@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(EXACT))
def test_exact_joint_across_row_chunks(oracle, layout):
    """The fp32 exact joint path over two row chunks whose boundary lies inside the last utterance's lattice: the chunk
    count of a forward-only call, costs and the four gradients at lambda = 0 and 0.5, and joint_rnnt_align, against the
    float64 references.  fp32 tolerances of DESIGN.md 4: costs rtol 1e-5; gradients rtol 1e-4, the per-cell floor
    |g|·(1e-6 + 1e-6·max|cost|) and the cost-scaled norm-wise term of
    tests/test_gpu_joint_bf16.py::test_c2_full_size_vs_oracle, max(1e-5, 2e-7·max|cost|)."""
    import rnnt_speech_recognition_b200 as rb
    from rnnt_speech_recognition_b200 import _lib
    e = EXACT[layout]
    rows, cells = exact_boundaries(layout)
    k = synth_case(exact_lengths(layout), e["maxT"], e["maxU"], e["V"], e["H"], 900 + e["H"])
    il, ll = k["input_lengths"], k["label_lengths"]
    _lib.set_timing(True)
    try:
        costs0, _ = joint_abi(k, "fp32")
        chunks = sum(n == "sgemm L=Z.W+b" for n, _ in _lib.get_timings())
    finally:
        _lib.set_timing(False)
    assert chunks == -(-e["B"] * e["maxT"] * e["maxU"] // rows) == len(cells) + 1

    gs = np.linspace(0.5, 1.5, e["B"])
    for lam in (0.0, 0.5):
        want = joint_reference(oracle, k, gs, lam)
        costs, grads = joint_abi(k, "fp32", gs, fastemit_lambda=lam)
        assert np.array_equal(costs, costs0)
        cmax = float(np.abs(want["costs"]).max())
        assert_close(costs, want["costs"], rtol=1e-5, atol=1e-4, what="costs")
        for g, n in zip(grads, NAMES):
            assert_close(g, want[n], rtol=1e-4, atol=fp32_tol(want["costs"])["atol"] * gs.max(),
                         ntol=max(1e-5, 2e-7 * cmax), what="%s at lambda = %g" % (n, lam))
        assert_padding_zero(k, grads, "lambda = %g" % lam)

    t = [dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")]
    al = rb.joint_rnnt_align(*t, dev(k["labels"]), dev(il), dev(ll), precision="fp32")
    assert np.array_equal(al.costs.cpu().numpy(), costs0)

    def log_probs(b):
        T, U = int(il[b]), int(ll[b]) + 1
        return ar.joint_log_probs(k["enc"][b:b + 1, :T], k["pred"][b:b + 1, :U], k["W"], k["b"])

    check_alignment(al, log_probs, k["labels"], il, ll, 0, OP_TOL)
