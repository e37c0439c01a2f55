"""Pruned RNN-T, host side (no GPU): the float64 reference tests/pruned_ref.py pinned by the oracle on materialised
am + lm logits and by central differences; the band policy pinned by exhaustive path enumeration (its score, its
properties, window <-> band equivalence, feasibility iff (S-1) T_b >= U_b - 1, full windows for S >= U_b); the simple
entries' argument checks."""
import ctypes as C

import numpy as np
import pytest

import pruned_ref as pr
import window_ref as wr
from conftest import load
from rnnt_speech_recognition_b200 import _lib


CASES = [  # (B, T, U, V, blank, label_blank)
    (3, 6, 4, 5, 0, False), (4, 7, 5, 6, 5, False), (2, 5, 3, 7, 6, False), (3, 1, 4, 5, 0, False),
    (3, 5, 1, 4, 0, False), (2, 4, 3, 5, 2, True)]


@pytest.mark.parametrize("case", CASES)
def test_simple_reference_equals_oracle(case, oracle):
    B, T, U, V, blank, lb = case
    rng = np.random.default_rng(sum(case[:5]))
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, blank, scale=2.0, label_blank=lb)
    costs, d_am, d_lm = pr.simple_loss_grad(am, lm, labels, il, ll, blank)
    oc, og = oracle.rnnt_logits_grad(pr.logits(am, lm), labels[:, :max(U - 1, 1)], il, ll, blank)
    np.testing.assert_allclose(costs, oc, rtol=1e-12)
    np.testing.assert_allclose(d_am, og.sum(axis=2), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(d_lm, og.sum(axis=1), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("case", CASES)
def test_factorised_reference_equals_materialised(case):
    """simple_loss_grad_f64 (no (B,T,U,V) tensor: the full-size GPU tests use it) against simple_loss_grad."""
    B, T, U, V, blank, lb = case
    rng = np.random.default_rng(11 + sum(case[:5]))
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, blank, scale=3.0, label_blank=lb)
    gs = np.linspace(-1.0, 2.0, B)
    want = pr.simple_loss_grad(am, lm, labels, il, ll, blank, grad_scale=gs)
    got = pr.simple_loss_grad_f64(am, lm, labels, il, ll, blank, grad_scale=gs)
    for g, w in zip(got, want):
        np.testing.assert_allclose(g, w, rtol=1e-11, atol=1e-13)


def test_simple_reference_on_golden_lengths(oracle):
    """The golden ragged case's labels and lengths (B=5, T=12, U=7, V=11) with random am / lm."""
    g = load("logits_ragged_B5_T12_U7_V11.npz")
    B, T, U, V = g["acts"].shape
    rng = np.random.default_rng(7)
    am, lm = rng.standard_normal((B, T, V)) * 2, rng.standard_normal((B, U, V)) * 2
    args = (g["labels"], g["input_lengths"], g["label_lengths"], int(g["blank"]))
    costs, d_am, d_lm = pr.simple_loss_grad(am, lm, *args)
    oc, og = oracle.rnnt_logits_grad(pr.logits(am, lm), *args)
    np.testing.assert_allclose(costs, oc, rtol=1e-12)
    np.testing.assert_allclose(d_am, og.sum(axis=2), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(d_lm, og.sum(axis=1), rtol=1e-10, atol=1e-12)
    il, ll = g["input_lengths"], g["label_lengths"]
    for b in range(B):                                    # rows past the lengths: exactly 0
        assert not d_am[b, il[b]:].any() and not d_lm[b, ll[b] + 1:].any()


def test_simple_reference_central_differences():
    rng = np.random.default_rng(3)
    B, T, U, V, blank = 2, 4, 3, 5, 1
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, V, blank)
    gs = np.array([0.7, -1.3])
    _, d_am, d_lm = pr.simple_loss_grad(am, lm, labels, il, ll, blank, grad_scale=gs)
    f = lambda a, l: float((pr.simple_loss_grad(a, l, labels, il, ll, blank)[0] * gs).sum())
    h = 1e-6
    for x, d in ((am, d_am), (lm, d_lm)):
        num = np.zeros_like(x)
        for i in np.ndindex(x.shape):
            xp, xm = x.copy(), x.copy()
            xp[i] += h
            xm[i] -= h
            num[i] = (f(xp, lm) - f(xm, lm)) / (2 * h) if x is am else (f(am, xp) - f(am, xm)) / (2 * h)
        np.testing.assert_allclose(d, num, rtol=1e-6, atol=1e-8)


def _utt(rng, T, U, V=4, scale=1.5):
    am, lm, labels, il, ll = pr.random_case(rng, 1, T, U, V, 0, scale=scale, ragged=False)
    return am, lm, labels, il, ll


@pytest.mark.parametrize("seed", range(6))
def test_score_equals_enumerated_probabilities(seed):
    """score(t,s) = P(s <= entry, exit < s+S) - P(entry < s, exit >= s+S) over every path of the lattice."""
    rng = np.random.default_rng(seed)
    T, U, S = int(rng.integers(2, 6)), int(rng.integers(2, 6)), int(rng.integers(2, 4))
    am, lm, labels, il, ll = _utt(rng, T, U)
    _, gB, gL = pr.occupancies(am, lm, labels, il, ll)
    lp = wr.log_softmax(pr.logits(am, lm))
    lpb, lpl, _ = wr.arc_logprobs(lp, labels, 0)
    paths = pr.enumerate_paths(lpb[0], lpl[0], T, U)
    Z = sum(p for p, _ in paths)
    sc = pr.scores(gB[0], gL[0], T, U, S)
    for t in range(T - 1):
        for s in range(sc.shape[1]):
            want = sum(p * ((s <= e and x < s + S) - (e < s and x >= s + S)) for p, seg in paths for e, x in [seg[t]]) / Z
            assert abs(sc[t, s] - want) < 1e-12, (t, s, sc[t, s], want)


@pytest.mark.parametrize("seed", range(40))
def test_band_properties_and_windows(seed):
    rng = np.random.default_rng(100 + seed)
    B, T, U, S = 3, int(rng.integers(1, 9)), int(rng.integers(1, 9)), int(rng.integers(2, 5))
    am, lm, labels, il, ll = pr.random_case(rng, B, T, U, 5, 0, scale=2.0)
    lo, hi, starts = pr.band(am, lm, labels, il, ll, S)
    for b in range(B):
        Tn, Un, s = int(il[b]), int(ll[b]) + 1, starts[b]
        assert s[0] == 0 and np.all(np.diff(s) >= 0) and np.all(np.diff(s) <= S - 1), s
        assert np.all(s <= max(0, Un - S)) and np.all(s >= 0)
        # window <-> band, cell by cell, and (0, -1) past U_b
        for u in range(U):
            for t in range(T):
                in_band = t < Tn and u < Un and s[t] <= u < s[t] + S
                assert in_band == (lo[b, u] <= t <= hi[b, u]), (b, t, u)
            if u >= Un:
                assert (lo[b, u], hi[b, u]) == (0, -1)
        # feasibility iff (S-1) T_b >= U_b - 1, through the windowed loss; S >= U_b: full windows
        lp = wr.log_softmax(pr.logits(am[b:b + 1], lm[b:b + 1]))
        lpb, lpl, _ = wr.arc_logprobs(lp, labels[b:b + 1], 0)
        cost = wr.masked_dp(lpb, lpl, il[b:b + 1], ll[b:b + 1], (lo[b:b + 1], hi[b:b + 1]))[0][0]
        assert np.isfinite(cost) == ((S - 1) * Tn >= Un - 1), (Tn, Un, S, cost)
        if S >= Un:
            assert np.all(lo[b, :Un] == 0) and np.all(hi[b, :Un] == Tn - 1)


def test_infeasible_band_is_an_inf_cost():
    """S = 2, T_b = 2, U_b = 4: (S-1) T_b = 2 < 3, so the band admits no path."""
    rng = np.random.default_rng(0)
    am, lm, labels, il, ll = _utt(rng, 2, 4)
    lo, hi, _ = pr.band(am, lm, labels, il, ll, 2)
    lp = wr.log_softmax(pr.logits(am, lm))
    lpb, lpl, _ = wr.arc_logprobs(lp, labels, 0)
    assert wr.masked_dp(lpb, lpl, il, ll, (lo, hi))[0][0] == np.inf


def test_simple_entries_reject_bad_arguments():
    """Argument errors come back as RNNT_STATUS_INVALID_VALUE before any device work (no GPU needed)."""
    L = _lib.load()
    p = C.c_void_p(16)
    opt = lambda blank=0, T=4, U=3: _lib.RnntOptions(_lib.RNNT_GPU, 0, None, blank, T, U, True)
    sz = C.c_size_t(0)
    assert L.rnntb200_simple_workspace_size(2, 4, 3, 8, C.byref(sz)) == 0 and sz.value > 0
    first = sz.value
    assert L.rnntb200_simple_workspace_size(2, 4, 3, 8, C.byref(sz)) == 0 and sz.value == first
    assert L.rnntb200_simple_workspace_size(2, 4, 1025, 8, C.byref(sz)) == 2
    assert L.rnntb200_simple_workspace_size(0, 4, 3, 8, C.byref(sz)) == 2
    assert L.rnntb200_simple_workspace_size(2, 4, 3, 8, None) == 2
    fwd = L.rnntb200_simple_loss_forward
    assert fwd(None, p, p, p, p, 8, 2, p, p, opt()) == 2
    assert fwd(p, p, p, p, p, 8, 2, None, p, opt()) == 2
    assert fwd(p, p, p, p, p, 8, 2, p, p, opt(U=1025)) == 2
    assert fwd(p, p, p, p, p, 8, 2, p, p, opt(blank=8)) == 2
    assert fwd(p, p, p, p, p, 8, 2, p, p, opt(blank=-1)) == 2
    bwd = L.rnntb200_simple_loss_backward
    assert bwd(p, p, p, p, p, 8, 2, None, None, p, p, opt()) == 2
    assert bwd(p, p, p, p, p, 8, 2, None, p, p, None, opt()) == 2
    assert bwd(p, p, p, p, p, 8, 2, None, p, p, p, opt(U=1025)) == 2
    win = L.rnntb200_simple_prune_windows
    assert win(p, p, 2, 1, p, p, p, opt()) == 2
    assert win(p, p, 2, 4, None, p, p, opt()) == 2
    assert win(p, p, 2, 4, p, p, p, opt(U=1025)) == 2
    assert win(p, p, 0, 4, p, p, p, opt()) == 2


@pytest.mark.parametrize("bad", [1, 0, -3, 2.5, True])
def test_simple_rnnt_loss_rejects_bad_s_range(bad):
    import torch
    import rnnt_speech_recognition_b200 as rb
    z = torch.zeros(1, 2, 3)
    i = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(ValueError):
        rb.simple_rnnt_loss(z, z, torch.zeros(1, 1, dtype=torch.int32), i, i, s_range=bad)
