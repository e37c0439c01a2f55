"""Pruned RNN-T on the H100: the simple loss (`simple_rnnt_loss`, rnntb200_simple_*) and its band.

* The simple loss against the float64 reference (tests/pruned_ref.py) at the fp32 path's DESIGN §4 tolerances for
  reduced gradients, from tiny edge lattices to V = 4096, T = 2000, maxU = 1024 and a full C3-shaped batch; upstream
  gradients of several scales and signs; padded rows; agreement with the fp32 loss op on the materialised am + lm logits.
* The underflow fallback: am / lm peaked in disjoint columns 60, 100 and 150 nats above the rest.
* Determinism, CUDA-graph replay of forward + windows + backward, 16-bit inputs.
* The band: equal to the reference's on inputs whose score margins exceed 1e-3; its properties and feasibility rule on
  random inputs; end to end on the tensor-core joint.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import pruned_ref as pr
import window_ref as wr
from conftest import assert_close
from test_gpu_fastemit import dev
from test_gpu_joint import synth
from test_gpu_ref64 import ab_cell, ab_norm

pytestmark = pytest.mark.gpu


def run_simple(am, lm, labels, il, ll, blank=0, gs=None, dtype=torch.float32, s_range=None):
    """(costs, d_am, d_lm[, (t_lo, t_hi)]) on the host; gradients as float64."""
    import rnnt_speech_recognition_b200 as rb
    a = dev(am, torch.float32).to(dtype).requires_grad_()
    m = dev(lm, torch.float32).to(dtype).requires_grad_()
    B = am.shape[0]
    gs = np.full(B, 1.0 / B) if gs is None else gs
    out = rb.simple_rnnt_loss(a, m, dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32), blank,
                              s_range=s_range)
    costs = out[0] if s_range else out
    da, dl = torch.autograd.grad(costs, (a, m), grad_outputs=dev(gs, torch.float32))
    assert da.dtype == dtype and dl.dtype == dtype
    res = (costs.detach().cpu().numpy(), da.double().cpu().numpy(), dl.double().cpu().numpy())
    if s_range:
        res += (tuple(w.cpu().numpy() for w in out[1]),)
    return res


def check(got, want, gs, what):
    """fp32 bounds for reduced gradients (DESIGN §4): costs rtol 1e-5; gradients rtol 1e-4 plus the per-cell alpha/beta
    floor and the norm-wise term max(1e-5, alpha/beta)."""
    costs, d_am, d_lm = got
    cmax = float(np.abs(want[0]).max())
    assert_close(costs, want[0], rtol=1e-5, atol=1e-4, what=what + " costs")
    for g, w, n in ((d_am, want[1], "d_am"), (d_lm, want[2], "d_lm")):
        assert_close(g, w, rtol=1e-4, atol=ab_cell(cmax) * np.max(np.abs(gs)), ntol=max(1e-5, ab_norm(cmax)),
                     what="%s %s" % (what, n))


CASES = [  # (B, T, U, V, blank, label_blank, scale)
    (3, 6, 4, 5, 0, False, 2.0), (4, 9, 5, 6, 5, False, 2.0), (2, 7, 3, 7, 6, False, 2.0), (3, 1, 4, 5, 0, False, 2.0),
    (3, 5, 1, 4, 0, False, 2.0), (2, 4, 3, 5, 2, True, 2.0), (4, 33, 17, 24, 0, False, 3.0),
    (3, 40, 20, 1024, 1023, False, 3.0), (3, 37, 21, 1028, 0, False, 3.0), (2, 30, 12, 4096, 7, False, 3.0)]


@pytest.mark.parametrize("case", CASES)
def test_simple_loss_vs_reference(case):
    B, T, U, V, blank, lb, scale = case
    rng = np.random.default_rng(sum(case[:5]))
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, blank, scale=scale, label_blank=lb)
    gs = np.full(B, 1.0 / B)
    want = pr.simple_loss_grad_f64(am, lm, labels, il, ll, blank, gs, device="cuda")
    check(run_simple(am, lm, labels, il, ll, blank, gs), want, gs, "case %s" % (case,))


@pytest.mark.parametrize("T,U,V", [(2000, 8, 64), (40, 1024, 64)])
def test_simple_loss_long_lattices(T, U, V):
    rng = np.random.default_rng(T + U)
    am, lm, labels, il, ll = pr.random_case(rng, 2, T, U, V, 0, scale=1.0)
    gs = np.full(2, 0.5)
    want = pr.simple_loss_grad_f64(am, lm, labels, il, ll, 0, gs, device="cuda")
    check(run_simple(am, lm, labels, il, ll, 0, gs), want, gs, "T=%d U=%d" % (T, U))


def test_maxu_1025_is_rejected():
    import rnnt_speech_recognition_b200 as rb
    am, lm = torch.zeros(1, 3, 8, device="cuda"), torch.zeros(1, 1025, 8, device="cuda")
    i = torch.ones(1, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="invalid value"):
        rb.simple_rnnt_loss(am, lm, torch.zeros(1, 1024, dtype=torch.int32, device="cuda"), i, i)


def test_simple_loss_c3_batch():
    """A full C3-shaped batch (B=32, T=512, U=128, V=1024)."""
    B, T, U, V = 32, 512, 128, 1024
    rng = np.random.default_rng(2026)
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, 0, scale=1.0, ragged=False)
    am, lm = am.astype(np.float32), lm.astype(np.float32)
    gs = np.full(B, 1.0 / B)
    want = pr.simple_loss_grad_f64(am, lm, labels, il, ll, 0, gs, device="cuda")
    check(run_simple(am, lm, labels, il, ll, 0, gs), want, gs, "C3")


@pytest.mark.parametrize("kind", ["1/B", "2^16/B", "mixed", "zero"])
def test_upstream_gradients(kind):
    B, T, U, V = 4, 20, 9, 40
    rng = np.random.default_rng(5)
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, 3, scale=2.0)
    gs = {"1/B": np.full(B, 1.0 / B), "2^16/B": np.full(B, 2.0 ** 16 / B), "mixed": np.array([0.5, -1.5, 2.0, -0.25]),
          "zero": np.zeros(B)}[kind]
    got = run_simple(am, lm, labels, il, ll, 3, gs)
    if kind == "zero":
        assert not got[1].any() and not got[2].any()
        return
    check(got, pr.simple_loss_grad_f64(am, lm, labels, il, ll, 3, gs, device="cuda"), gs, kind)


def test_padded_rows_are_zero_and_ignored():
    """Rows past the lengths get exactly 0, and large finite values in them change nothing, bit for bit."""
    B, T, U, V = 4, 15, 8, 33
    rng = np.random.default_rng(9)
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, 0, scale=2.0)
    il[1], ll[2] = 3, 0
    labels[:, :] = np.where(np.arange(U - 1)[None, :] < ll[:, None], labels, 0)
    base = run_simple(am, lm, labels, il, ll, 0, s_range=3)
    am2, lm2, lab2 = am.copy(), lm.copy(), labels.copy()
    for b in range(B):
        am2[b, il[b]:] = 3e4 * rng.standard_normal((T - il[b], V))
        lm2[b, ll[b] + 1:] = -3e4 * rng.standard_normal((U - ll[b] - 1, V))
        lab2[b, ll[b]:] = V - 1
    other = run_simple(am2, lm2, lab2, il, ll, 0, s_range=3)
    for x, y in zip(base[:3], other[:3]):
        assert np.array_equal(x, y)
    assert all(np.array_equal(x, y) for x, y in zip(base[3], other[3]))
    for b in range(B):
        assert not base[1][b, il[b]:].any() and not base[2][b, ll[b] + 1:].any()


def test_agrees_with_loss_op_on_materialised_logits():
    import rnnt_speech_recognition_b200 as rb
    B, T, U, V = 3, 24, 10, 48
    rng = np.random.default_rng(12)
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, 0, scale=2.0)
    gs = np.full(B, 1.0 / B)
    costs, d_am, d_lm = run_simple(am, lm, labels, il, ll, 0, gs)
    x = (dev(am, torch.float32)[:, :, None, :] + dev(lm, torch.float32)[:, None, :, :]).contiguous().requires_grad_()
    oc = rb.rnnt_loss(x, dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32), 0)
    (g,) = torch.autograd.grad(oc, x, grad_outputs=dev(gs, torch.float32))
    g = g.double().cpu().numpy()
    check((costs, d_am, d_lm), (oc.detach().cpu().numpy(), g.sum(axis=2), g.sum(axis=1)), gs, "vs loss op")


@pytest.mark.parametrize("gap", [60.0, 100.0, 150.0])
def test_underflow_fallback(gap):
    """am's rows peak in the lower half of the vocabulary and lm's in the upper half, `gap` nats above the rest: the
    factorised normaliser is about 2 exp(-gap) (0 in fp32 at 150 nats), so these cells take the direct log-sum-exp."""
    B, T, U, V = 3, 7, 5, 16
    rng = np.random.default_rng(int(gap))
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, 0, scale=0.5)
    am[np.arange(B)[:, None], np.arange(T)[None, :], rng.integers(0, V // 2, (B, T))] += gap
    lm[np.arange(B)[:, None], np.arange(U)[None, :], rng.integers(V // 2, V, (B, U))] += gap
    gs = np.full(B, 1.0 / B)
    got = run_simple(am, lm, labels, il, ll, 0, gs)
    assert np.all(np.isfinite(got[0])) and np.all(np.isfinite(got[1])) and np.all(np.isfinite(got[2]))
    check(got, pr.simple_loss_grad(am, lm, labels, il, ll, 0, gs), gs, "gap %g" % gap)


def _c_entries(am, lm, lab, il, ll, V, B, T, U, S):
    """The C entries on preallocated buffers: fn() runs forward + windows + backward and returns the outputs."""
    from rnnt_speech_recognition_b200 import _lib
    L = _lib.load()
    sz = C.c_size_t(0)
    _lib.check(L.rnntb200_simple_workspace_size(B, T, U, V, C.byref(sz)), "ws")
    ws = torch.empty(sz.value, dtype=torch.uint8, device="cuda")
    costs = torch.empty(B, device="cuda")
    lo, hi = (torch.empty(B, U, dtype=torch.int32, device="cuda") for _ in range(2))
    d_am, d_lm = torch.empty_like(am), torch.empty_like(lm)
    gs = torch.full((B,), 1.0 / B, device="cuda")
    p = _lib.ptr

    def fn():
        opt = _lib.RnntOptions(_lib.RNNT_GPU, 0, _lib.stream().value, 0, T, U, True)
        assert L.rnntb200_simple_loss_forward(p(am), p(lm), p(lab), p(ll), p(il), V, B, p(costs), p(ws), opt) == 0
        assert L.rnntb200_simple_prune_windows(p(ll), p(il), B, S, p(lo), p(hi), p(ws), opt) == 0
        assert L.rnntb200_simple_loss_backward(p(am), p(lm), p(lab), p(ll), p(il), V, B, p(gs), p(d_am), p(d_lm), p(ws),
                                               opt) == 0
        return costs, lo, hi, d_am, d_lm
    return fn


def test_determinism_and_cuda_graph_replay():
    B, T, U, V, S = 4, 60, 20, 72, 4
    rng = np.random.default_rng(21)
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, 0, scale=2.0)
    am[0, :, :V // 2] += 70.0                                            # some cells take the fallback
    lm[0, :, V // 2:] += 70.0
    args = [dev(am, torch.float32), dev(lm, torch.float32), dev(labels, torch.int32), dev(il, torch.int32),
            dev(ll, torch.int32)]
    fn = _c_entries(*args, V, B, T, U, S)
    first = [x.clone() for x in fn()]
    second = [x.clone() for x in fn()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = fn()
    for o in outs:
        o.fill_(7)
    g.replay()
    torch.cuda.synchronize()
    for a, b, c in zip(first, second, outs):
        assert torch.equal(a, b) and torch.equal(a, c)
    assert torch.isfinite(first[0]).all()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_16bit_inputs_match_upcast_fp32(dtype):
    B, T, U, V = 3, 18, 7, 40
    rng = np.random.default_rng(4)
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, 0, scale=2.0)
    am16 = torch.as_tensor(am, dtype=torch.float32).to(dtype).float().numpy()
    lm16 = torch.as_tensor(lm, dtype=torch.float32).to(dtype).float().numpy()
    c16, a16, l16, w16 = run_simple(am, lm, labels, il, ll, dtype=dtype, s_range=3)
    c32, a32, l32, w32 = run_simple(am16, lm16, labels, il, ll, s_range=3)
    cast = lambda x: torch.as_tensor(x).float().to(dtype).double().numpy()
    assert np.array_equal(c16, c32)
    assert np.array_equal(a16, cast(a32)) and np.array_equal(l16, cast(l32))
    assert all(np.array_equal(x, y) for x, y in zip(w16, w32))


def _planted(S, tries=400):
    """Random inputs whose every frame's best raw start wins by more than 1e-3 (rejection sampling)."""
    for seed in range(tries):
        rng = np.random.default_rng(1000 + seed)
        am, lm, labels, il, ll = pr.random_case(rng, 3, 12, 7, 9, 0, scale=2.5)
        if pr.score_margins(am, lm, labels, il, ll, S).min() > 1e-3:
            return am, lm, labels, il, ll
    raise AssertionError("no planted case found")


@pytest.mark.parametrize("S", [2, 3, 4])
def test_windows_equal_reference_on_planted_inputs(S):
    am, lm, labels, il, ll = _planted(S)
    lo, hi, _ = pr.band(am, lm, labels, il, ll, S)
    got = run_simple(am, lm, labels, il, ll, s_range=S)[3]
    assert np.array_equal(got[0], lo) and np.array_equal(got[1], hi), (got, lo, hi)


@pytest.mark.parametrize("S", [2, 4, 5, 16])
def test_windows_properties_on_random_inputs(S):
    B, T, U, V = 16, 40, 30, 32
    rng = np.random.default_rng(S)
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, 0, scale=2.0)
    il[1], ll[1] = 3, 29                         # (S-1) T_b < U_b - 1 for S < 11: infeasible
    lo, hi = run_simple(am, lm, labels, il, ll, s_range=S)[3]
    lp = wr.log_softmax(pr.logits(am, lm))
    lpb, lpl, _ = wr.arc_logprobs(lp, labels, 0)
    costs = wr.masked_dp(lpb, lpl, il, ll, (lo, hi))[0]
    for b in range(B):
        Tn, Un = int(il[b]), int(ll[b]) + 1
        assert np.all(lo[b, Un:] == 0) and np.all(hi[b, Un:] == -1)
        # recover s_t from the windows: the band of frame t is the columns whose window holds t
        inb = (lo[b, :Un, None] <= np.arange(Tn)[None, :]) & (np.arange(Tn)[None, :] <= hi[b, :Un, None])
        for t in range(Tn):
            cols = np.flatnonzero(inb[:, t])
            assert len(cols) == min(S, Un) and cols[-1] - cols[0] == len(cols) - 1, (b, t, cols)
        s = inb.argmax(axis=0)
        assert s[0] == 0 and np.all(np.diff(s) >= 0) and np.all(np.diff(s) <= S - 1)
        assert np.isfinite(costs[b]) == ((S - 1) * Tn >= Un - 1), (b, Tn, Un, costs[b])
        if S >= Un:
            assert np.all(lo[b, :Un] == 0) and np.all(hi[b, :Un] == Tn - 1)


def _joint_loss(k, am, lm, S, valid_tiles=None, windows=None, gs=None):
    import rnnt_speech_recognition_b200 as rb
    t = [dev(k[n], torch.float32).requires_grad_() for n in ("enc", "pred", "W", "b")]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    if windows is None and S is not None:
        _, windows = rb.simple_rnnt_loss(dev(am, torch.float32), dev(lm, torch.float32), lab, il, ll, s_range=S)
    costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision="bf16", windows=windows, valid_tiles=valid_tiles)
    B = costs.shape[0]
    gs = np.full(B, 1.0 / B) if gs is None else gs
    grads = torch.autograd.grad(costs, t, grad_outputs=dev(gs, torch.float32))
    hw = None if windows is None else tuple(w.cpu().numpy() for w in windows)
    return costs.detach().cpu().numpy(), [x.cpu().numpy() for x in grads], hw


def test_large_s_range_is_the_unrestricted_joint_loss():
    B, T, U, V, H = 3, 40, 12, 128, 64
    k = synth(B, T, U, V, H, 3)
    rng = np.random.default_rng(3)
    am, lm = rng.standard_normal((B, T, V)), rng.standard_normal((B, U, V))
    full = _joint_loss(k, am, lm, None)
    pruned = _joint_loss(k, am, lm, U)
    assert np.array_equal(full[0], pruned[0])
    assert all(np.array_equal(a, b) for a, b in zip(full[1], pruned[1]))


def test_pruned_joint_loss_matches_window_reference():
    from test_gpu_ref64 import check_tc
    B, T, U, V, H = 3, 50, 20, 128, 64
    k = synth(B, T, U, V, H, 8)
    rng = np.random.default_rng(8)
    am, lm = 2 * rng.standard_normal((B, T, V)), 2 * rng.standard_normal((B, U, V))
    costs, grads, hw = _joint_loss(k, am, lm, 4)
    want = wr.joint_loss_grad(dev(k["enc"]), dev(k["pred"]), dev(k["W"]), dev(k["b"]), k["labels"], k["input_lengths"],
                              k["label_lengths"], 0, hw, np.full(B, 1.0 / B))
    check_tc(costs, grads, want, "pruned S=4")


def test_c3_pruned_step():
    """C3 with S = 5: finite costs no smaller than the unrestricted ones; valid_tile_count of host copies of the windows
    is accepted as valid_tiles (bit-identical to the call without it)."""
    import rnnt_speech_recognition_b200 as rb
    B, T, U, V, H = 32, 512, 128, 1024, 640
    k = synth(B, T, U, V, H, 77, ragged=False)
    rng = np.random.default_rng(77)
    am, lm = rng.standard_normal((B, T, V)).astype(np.float32), rng.standard_normal((B, U, V)).astype(np.float32)
    full = _joint_loss(k, am, lm, None)[0]
    costs, grads, hw = _joint_loss(k, am, lm, 5)
    assert np.all(np.isfinite(costs)) and np.all(costs >= full - 1e-5 * np.abs(full)), (costs - full).min()
    vt = rb.valid_tile_count(k["input_lengths"], k["label_lengths"], hw)
    assert vt < rb.valid_tile_count(k["input_lengths"], k["label_lengths"])
    win = tuple(dev(w, torch.int32) for w in hw)
    c2, g2, _ = _joint_loss(k, am, lm, None, valid_tiles=vt, windows=win)
    assert np.array_equal(costs, c2) and all(np.array_equal(a, b) for a, b in zip(grads, g2))
