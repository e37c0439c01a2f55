"""CPU checks of forced alignment: the float64 reference (tests/align_ref.py) against exhaustive enumeration of every
path, its tie rule and its bounds against the oracle's cost, and the argument checks of the three C entries (which must
bail out before any device work, so no GPU is needed)."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest

import align_ref as ar
from oracle import oracle as _oracle


def enumerate_paths(lp, labels, T, U, blank):
    """Every alignment of one utterance as (frames, score): label j at frame f_j with f non-decreasing in [0, T)."""
    lab = np.asarray(labels[:U - 1], np.int64)
    out = []
    for f in itertools.combinations_with_replacement(range(T), U - 1):
        s = sum(lp[t, j, lab[j]] for j, t in enumerate(f))
        u = 0
        for t in range(T):
            while u < U - 1 and f[u] <= t:
                u += 1
            s += lp[t, u, blank]
        out.append((np.array(f, np.int32), s))
    return out


def small_case(seed, B, T, U, V, blank=0, ragged=True, label_is_blank=False, scale=2.0):
    rng = np.random.default_rng(seed)
    acts = scale * rng.standard_normal((B, T, U, V))
    labels = rng.choice([v for v in range(V) if v != blank], size=(B, max(U - 1, 0))).astype(np.int32)
    if label_is_blank:
        labels[rng.random(labels.shape) < 0.4] = blank
    il, ll = np.full(B, T, np.int32), np.full(B, U - 1, np.int32)
    if ragged:
        il, ll = rng.integers(1, T + 1, B).astype(np.int32), rng.integers(0, U, B).astype(np.int32)
        il[0], ll[0] = T, U - 1
    return acts, labels, il, ll


CASES = [dict(seed=0, B=4, T=6, U=5, V=7), dict(seed=1, B=5, T=5, U=4, V=6, blank=3),
         dict(seed=2, B=3, T=1, U=5, V=6, ragged=False), dict(seed=3, B=3, T=6, U=1, V=5, ragged=False),
         dict(seed=4, B=4, T=4, U=5, V=5, blank=4, label_is_blank=True), dict(seed=5, B=4, T=6, U=3, V=9, scale=0.3),
         dict(seed=6, B=3, T=1, U=1, V=4, ragged=False)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "seed%d_T%d_U%d" % (c["seed"], c["T"], c["U"]))
def test_reference_against_enumeration(case):
    blank = case.get("blank", 0)
    acts, labels, il, ll = small_case(**case)
    lp = ar.log_probs(acts)
    frames, best, gap = ar.viterbi(lp, labels, il, ll, blank)
    ar.check_frames(frames, il, ll)
    assert np.allclose(ar.path_score(lp, labels, frames, il, ll, blank), best, rtol=0, atol=1e-12)
    for b in range(acts.shape[0]):
        T, U = int(il[b]), int(ll[b]) + 1
        paths = enumerate_paths(lp[b], labels[b], T, U, blank)
        scores = np.array([s for _, s in paths])
        order = np.argsort(-scores, kind="stable")
        assert abs(best[b] - scores[order[0]]) <= 1e-12
        assert np.array_equal(frames[b, :U - 1], paths[order[0]][0])
        assert len(paths) == math.comb(T + U - 2, U - 1)
        if len(paths) == 1:
            assert gap[b] == np.inf
        else:
            assert abs(gap[b] - (scores[order[0]] - scores[order[1]])) <= 1e-9


@pytest.mark.parametrize("T,U,V,blank", [(6, 5, 7, 0), (4, 4, 5, 2), (1, 4, 3, 0), (5, 1, 3, 1)])
def test_ties_take_the_earliest_emission(T, U, V, blank):
    """Uniform logits: every path scores the same (bit for bit), and the blank-wins-ties rule emits every label at
    frame 0.  The enumeration confirms those frames are element-wise the earliest among the optimal paths."""
    acts = np.zeros((2, T, U, V))
    labels = np.full((2, U - 1), (blank + 1) % V, np.int32)
    labels[1, ::2] = blank                                        # labels equal to blank tie the same way
    il, ll = np.full(2, T, np.int32), np.full(2, U - 1, np.int32)
    lp = ar.log_probs(acts)
    frames, best, gap = ar.viterbi(lp, labels, il, ll, blank)
    assert not frames.any()
    assert np.all(gap == (np.inf if min(T, U) == 1 else 0.0))
    for b in range(2):
        paths = enumerate_paths(lp[b], labels[b], T, U, blank)
        top = max(s for _, s in paths)
        for f, s in paths:
            if s == top:
                assert np.all(frames[b, :U - 1] <= f)


@pytest.mark.parametrize("case", CASES[:5], ids=lambda c: "seed%d" % c["seed"])
def test_bounds_against_the_cost(case):
    """best_logp <= -cost (one path against the sum over all) and >= -cost - log(#paths) (the best of n paths holds at
    least 1/n of their total)."""
    blank = case.get("blank", 0)
    acts, labels, il, ll = small_case(**case)
    costs, _ = _oracle.rnnt_logits_grad(acts, labels if labels.size else np.zeros((acts.shape[0], 1), np.int32), il, ll,
                                        blank, want_grad=False)
    _, best, _ = ar.viterbi(ar.log_probs(acts), labels, il, ll, blank)
    npaths = np.array([math.comb(int(t) + int(u) - 1, int(u)) for t, u in zip(il, ll)], np.float64)
    assert np.all(best <= -costs + 1e-12)
    assert np.all(best >= -costs - np.log(npaths) - 1e-12)


@pytest.fixture(scope="module")
def L():
    from rnnt_speech_recognition_b200 import _lib
    return _lib.load()


def test_align_argument_checks_without_gpu(L):
    """Every call below fails in its argument checks: status 2 (RNNT_STATUS_INVALID_VALUE) and no kernel launched."""
    from rnnt_speech_recognition_b200 import _lib
    one = C.c_void_p(16)           # never dereferenced
    n0 = L.rnntb200_launch_count()

    def opt(blank=0, T=4, U=3):
        return _lib.RnntOptions(_lib.RNNT_GPU, 0, None, blank, T, U, True)

    for fn, pre in ((L.rnntb200_align_device, ()), (L.rnntb200_align16, (_lib.LOGITS_BF16,))):
        def call(acts=one, V=5, B=1, costs=one, best=one, frames=one, o=None, logit_type=None):
            p = pre if logit_type is None else (logit_type,)
            return fn(acts, *p, one, one, one, V, B, costs, best, frames, one, o or opt())
        assert call(acts=None) == 2
        assert call(V=0) == 2
        assert call(B=0) == 2
        assert call(costs=None) == 2
        assert call(best=None) == 2
        assert call(frames=None) == 2                             # maxU = 3: label_frames is required
        assert call(o=opt(T=0)) == 2
        assert call(o=opt(U=0)) == 2
        assert call(o=opt(U=1025)) == 2
        assert call(o=opt(blank=5)) == 2
        assert call(o=opt(blank=-1)) == 2
        if pre:
            assert call(logit_type=7) == 2
    d = _lib.JointDesc(2, 4, 3, 64, 128, 0, 0, None)
    args = [one] * 11
    assert L.rnntb200_joint_align(None, *args) == 2
    for i in range(11):                                           # enc, pred, W, b, labels, lengths, costs, best, frames, ws
        bad = list(args)
        bad[i] = None
        assert L.rnntb200_joint_align(C.byref(d), *bad) == 2, i
    for kw in (dict(V=0), dict(blank_label=128), dict(maxU=1025), dict(precision=5), dict(B=0)):
        bd = _lib.JointDesc(2, 4, 3, 64, 128, 0, 0, None)
        for k, v in kw.items():
            setattr(bd, k, v)
        assert L.rnntb200_joint_align(C.byref(bd), *args) == 2, kw
    assert L.rnntb200_launch_count() == n0


def test_align_rejects_other_dtypes_before_the_device():
    import torch
    from rnnt_speech_recognition_b200 import rnnt_align
    z = torch.zeros(1, 2, 2, 3, dtype=torch.float64)
    lab, n = torch.zeros(1, 1, dtype=torch.int32), torch.ones(1, dtype=torch.int32)
    with pytest.raises(TypeError):
        rnnt_align(z, lab, n, n)
