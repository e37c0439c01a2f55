"""Alignment-restricted loss, host side (no GPU): the float64 reference tests/window_ref.py pinned by exhaustive path
enumeration, central differences, the oracle (full windows) and the best path (left = right = 0); `alignment_windows` and the
windowed `valid_tile_count` against brute force over cells; the windowed entries' argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

import align_ref
import fastemit_ref
import window_ref as wr
import rnnt_speech_recognition_b200 as rb
from rnnt_speech_recognition_b200 import _lib
from rnnt_speech_recognition_b200.windows import check_windows


def _case(rng, B, T, U, V, ragged=True):
    acts = rng.standard_normal((B, T, U, V)) * 2
    labels = rng.integers(0, V, (B, max(U - 1, 1))).astype(np.int32)
    il = rng.integers(max(1, T // 2), T + 1, B).astype(np.int32) if ragged else np.full(B, T, np.int32)
    ll = rng.integers(0, U, B).astype(np.int32) if ragged else np.full(B, U - 1, np.int32)
    il[0], ll[0] = T, U - 1
    return acts, labels, il, ll


def _full(il, B, U):
    return np.zeros((B, U), np.int32), np.broadcast_to((il - 1)[:, None], (B, U)).astype(np.int32)


@pytest.mark.parametrize("seed", range(4))
def test_reference_equals_path_enumeration(seed):
    rng = np.random.default_rng(seed)
    B, T, U, V = 3, 5, 4, 6
    acts, labels, il, ll = _case(rng, B, T, U, V)
    lo, hi = wr.random_feasible_windows(rng, il, ll, U, slack=1)
    lo[2], hi[2] = 1, 0                                             # utterance 2: no cell allowed
    lp = wr.log_softmax(acts)
    lpb, lpl, _ = wr.arc_logprobs(lp, labels, 2)
    costs, gb, gl = wr.masked_dp(lpb, lpl, il, ll, (lo, hi))
    ok = wr.allowed_mask((lo, hi), il, ll, T, U)
    for b in range(B):
        want = wr.enumerate_cost(lpb[b], lpl[b], int(il[b]), int(ll[b]) + 1, ok[b])
        assert costs[b] == want or abs(costs[b] - want) < 1e-12 * abs(want)
    assert costs[2] == np.inf and not gb[2].any() and not gl[2].any()
    assert not gb[~ok].any() and not gl[~ok].any()


def test_reference_gradient_is_the_central_difference():
    rng = np.random.default_rng(7)
    B, T, U, V = 2, 6, 4, 5
    acts, labels, il, ll = _case(rng, B, T, U, V)
    win = wr.random_feasible_windows(rng, il, ll, U, slack=1)
    costs, dx = wr.logits_grad(acts, labels, il, ll, 1, win)
    ok = wr.allowed_mask(win, il, ll, T, U)
    assert not dx[~ok].any()
    h = 1e-6
    for _ in range(40):
        i = tuple(rng.integers(0, n) for n in acts.shape)
        ap, am = acts.copy(), acts.copy()
        ap[i] += h
        am[i] -= h
        num = (wr.logits_grad(ap, labels, il, ll, 1, win)[0][i[0]] - wr.logits_grad(am, labels, il, ll, 1, win)[0][i[0]]) / (2 * h)
        assert abs(num - dx[i]) < 1e-7, (i, num, dx[i])


@pytest.mark.parametrize("lam", [0.0, 0.5])
def test_full_windows_equal_the_oracle(oracle, lam):
    rng = np.random.default_rng(3)
    B, T, U, V = 3, 9, 6, 8
    acts, labels, il, ll = _case(rng, B, T, U, V)
    gs = rng.uniform(0.5, 2, B)
    for win in (None, _full(il, B, U)):
        costs, dx = wr.logits_grad(acts, labels, il, ll, 3, win, lam, gs)
        want_c, want_dx = fastemit_ref.logits_grad(acts, labels, il, ll, 3, lam, gs)
        np.testing.assert_allclose(costs, want_c, rtol=1e-12)
        np.testing.assert_allclose(dx, want_dx, rtol=1e-9, atol=1e-13)


def test_joint_reference_with_full_windows_equals_the_unwindowed_one():
    import joint_ref64
    rng = np.random.default_rng(5)
    B, T, U, V, H = 2, 7, 5, 8, 6
    enc, pred = rng.standard_normal((B, T, H)), rng.standard_normal((B, U, H))
    W, bias = rng.standard_normal((H, V)), rng.standard_normal(V)
    labels = rng.integers(0, V, (B, U - 1)).astype(np.int32)
    il, ll = np.array([T, T - 2], np.int32), np.array([U - 1, U - 3], np.int32)
    want = joint_ref64.joint_loss_grad(enc, pred, W, bias, labels, il, ll, 1, fastemit_lambda=0.25, chunk_rows=11)
    got = wr.joint_loss_grad(enc, pred, W, bias, labels, il, ll, 1, _full(il, B, U), fastemit_lambda=0.25, chunk_rows=13)
    for k in want:
        np.testing.assert_allclose(got[k], want[k], rtol=1e-9, atol=1e-13, err_msg=k)
    # and, with real windows, the chunked joint chain equals the dense logits gradient chained by hand
    win = wr.random_feasible_windows(rng, il, ll, U, slack=1)
    got = wr.joint_loss_grad(enc, pred, W, bias, labels, il, ll, 1, win, chunk_rows=7)
    z = np.tanh(enc[:, :, None] + pred[:, None])
    costs, dl = wr.logits_grad(z @ W + bias, labels, il, ll, 1, win)
    np.testing.assert_allclose(got["costs"], costs, rtol=1e-12)
    np.testing.assert_allclose(got["dW"], np.einsum("btuh,btuv->hv", z, dl), rtol=1e-9, atol=1e-13)
    np.testing.assert_allclose(got["d_enc"], ((dl @ W.T) * (1 - z * z)).sum(2), rtol=1e-9, atol=1e-13)


def _best_path(acts, labels, il, ll, blank):
    """(label_frames (B,U-1) with -1 padding, best_logp (B,)) of tests/align_ref.py's Viterbi."""
    return align_ref.viterbi(wr.log_softmax(acts), labels, il, ll, blank)[:2]


def test_zero_width_windows_admit_the_best_path_only():
    rng = np.random.default_rng(11)
    B, T, U, V = 4, 10, 6, 7
    acts, labels, il, ll = _case(rng, B, T, U, V)
    frames, best = _best_path(acts, labels, il, ll, 0)
    lo, hi = rb.alignment_windows(torch.tensor(frames), torch.tensor(il), torch.tensor(ll), 0, 0)
    costs, _ = wr.logits_grad(acts, labels, il, ll, 0, (lo.numpy(), hi.numpy()))
    np.testing.assert_allclose(costs, -np.asarray(best), rtol=1e-12)
    plain, _ = wr.logits_grad(acts, labels, il, ll, 0, None)
    wide, _ = wr.logits_grad(acts, labels, il, ll, 0, tuple(w.numpy() for w in rb.alignment_windows(
        torch.tensor(frames), torch.tensor(il), torch.tensor(ll), 2, 1)))
    assert (plain <= wide + 1e-12).all() and (wide <= costs + 1e-12).all()


@pytest.mark.parametrize("T,U", [(1, 1), (1, 4), (9, 1), (40, 19), (33, 9)])
@pytest.mark.parametrize("left,right", [(0, 0), (2, 5), (100, 100)])
def test_alignment_windows_and_tile_count_against_brute_force(T, U, left, right):
    rng = np.random.default_rng(T * 131 + U)
    B = 4
    il = rng.integers(1, T + 1, B).astype(np.int32)
    ll = rng.integers(0, U, B).astype(np.int32)
    il[0], ll[0] = T, U - 1
    frames = np.full((B, U - 1), -1, np.int32)
    for b in range(B):
        frames[b, :ll[b]] = np.sort(rng.integers(0, il[b], ll[b]))
    lo, hi = (w.numpy() for w in rb.alignment_windows(torch.tensor(frames), torch.tensor(il), torch.tensor(ll), left, right))
    assert lo.dtype == np.int32 and lo.shape == (B, U) == hi.shape
    tiles = 0
    for b in range(B):
        a = np.concatenate([[0], frames[b, :ll[b]], [il[b] - 1]])          # a_{-1}, a_0 .., a_{U_b-1}
        for u in range(ll[b] + 1):
            assert lo[b, u] == max(0, a[u] - left) and hi[b, u] == min(il[b] - 1, a[u + 1] + right)
        # label j may be emitted exactly at [a_j - left, a_j + right] (clipped to the utterance)
        for j in range(ll[b]):
            emit = [t for t in range(il[b]) if lo[b, j] <= t <= hi[b, j] and lo[b, j + 1] <= t <= hi[b, j + 1]]
            assert emit == list(range(max(0, frames[b, j] - left), min(il[b] - 1, frames[b, j] + right) + 1))
        ok = wr.allowed_mask((lo, hi), il, ll, T, U)[b]
        for t0 in range(0, T, 16):
            for u0 in range(0, U, 8):
                tiles += bool(ok[t0:t0 + 16, u0:u0 + 8].any())
    assert rb.valid_tile_count(il, ll, (lo, hi)) == tiles
    assert rb.valid_tile_count(il, ll, _full(il, B, U)) == rb.valid_tile_count(il, ll)


def test_tile_count_of_a_straight_alignment_at_benchmark_size():
    T, U = 512, 128
    a = np.round(np.linspace(0, T - 1, U + 1)[1:-1]).astype(np.int32)[None]
    il, ll = torch.tensor([T], dtype=torch.int32), torch.tensor([U - 1], dtype=torch.int32)
    counts = [rb.valid_tile_count([T], [U - 1], tuple(w.numpy() for w in rb.alignment_windows(torch.tensor(a), il, ll, r, r)))
              for r in (64, 16, 4, 0)]
    assert counts == [163, 77, 62, 47] and rb.valid_tile_count([T], [U - 1]) == 512


def test_infeasible_windows_in_the_reference():
    rng = np.random.default_rng(2)
    B, T, U, V = 2, 6, 4, 5
    acts, labels, il, ll = _case(rng, B, T, U, V, ragged=False)
    lo, hi = _full(il, B, U)
    lo, hi = lo.copy(), hi.copy()
    lo[1, 2], hi[1, 2] = 4, 3                                       # an empty column cuts every path of utterance 1
    costs, dx = wr.logits_grad(acts, labels, il, ll, 0, (lo, hi), 0.5)
    ref, rdx = wr.logits_grad(acts[:1], labels[:1], il[:1], ll[:1], 0, None, 0.5)
    assert costs[1] == np.inf and not dx[1].any() and np.isfinite(dx).all()
    assert costs[0] == ref[0] and (dx[0] == rdx[0]).all()


def test_window_argument_checks():
    dev = torch.device("cpu")
    lo, hi = torch.zeros(2, 3, dtype=torch.int32), torch.zeros(2, 3, dtype=torch.int32)
    assert check_windows(None, 2, 3, dev) == (None, None)
    with pytest.raises(TypeError):
        check_windows((lo, None), 2, 3, dev)
    with pytest.raises(TypeError):
        check_windows((lo.long(), hi), 2, 3, dev)
    with pytest.raises(ValueError):
        check_windows((lo,), 2, 3, dev)
    with pytest.raises(RuntimeError):
        check_windows((lo, hi), 2, 3, dev)                          # CPU tensors: the library has no CPU path
    with pytest.raises(ValueError):
        rb.alignment_windows(torch.zeros(2, 3, dtype=torch.int32), torch.ones(2, dtype=torch.int32),
                             torch.ones(2, dtype=torch.int32), -1, 0)


def test_one_null_window_is_rejected_before_any_device_work():
    """Exactly one of t_lo / t_hi NULL -> RNNT_STATUS_INVALID_VALUE; no device is touched (this runs without a GPU)."""
    L = _lib.load()
    p = C.c_void_p(0x1000)                                          # never dereferenced: the check comes first
    opt = _lib.RnntOptions(_lib.RNNT_GPU, 0, None, 0, 4, 3, True)
    desc = _lib.JointDesc(1, 4, 3, 64, 64, 0, _lib.BF16_TC, None, 0, 0)
    for lo, hi in ((p, None), (None, p)):
        assert L.rnntb200_loss_device_windowed(p, p, p, p, p, None, lo, hi, 8, 1, p, p, opt, 0.0) == 2
        assert L.rnntb200_loss16_forward_windowed(p, _lib.LOGITS_F16, p, p, p, lo, hi, 8, 1, p, p, opt) == 2
        assert L.rnntb200_loss16_backward_windowed(p, _lib.LOGITS_BF16, p, p, p, lo, hi, p, 8, 1, p, p, opt, 0.0) == 2
        assert L.rnntb200_joint_loss_forward_windowed(C.byref(desc), p, p, p, p, p, p, p, lo, hi, p, p) == 2
        assert L.rnntb200_joint_loss_backward_windowed(C.byref(desc), p, p, p, p, p, p, p, lo, hi, p, p, p, p, p, p, 0.0) == 2
