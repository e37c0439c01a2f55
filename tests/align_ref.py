"""Forced-alignment reference for the tests (float64, CPU): the Viterbi recurrence of DESIGN §1 in numpy.

    delta(0,0) = 0
    delta(t,u) = max(delta(t-1,u) + lpb(t-1,u), delta(t,u-1) + lpl(t,u-1))     (a predecessor outside the lattice: -inf)
    best_logp  = delta(T-1,U-1) + lpb(T-1,U-1)

The label arc wins only when strictly greater; on the lattice's edges the only predecessor is taken.  Log-probs come
from `oracle.log_softmax` / `oracle.joint_forward`.  Besides the frames and the score, `viterbi` returns the gap to the
second-best path: the smallest decision margin along the best path (every other path leaves the best one at some cell,
walking back, and loses at least that cell's margin; leaving it at the cell of smallest margin loses exactly that).
"""
import numpy as np

from oracle import oracle as _oracle


def log_probs(acts):
    """Log-softmax of raw logits in float64 (softmax inside, as the loss op)."""
    return _oracle.log_softmax(np.ascontiguousarray(acts, np.float64))


def joint_log_probs(enc, pred, W, b):
    return log_probs(_oracle.joint_forward(*(np.asarray(a, np.float64) for a in (enc, pred, W, b))))


def _arcs(lp, labels, b, T, U, blank):
    lpb = lp[b, :T, :U, blank]
    lpl = np.full((T, U), -np.inf)
    if U > 1:
        lab = np.asarray(labels[b][:U - 1], np.int64)
        lpl[:, :U - 1] = np.take_along_axis(lp[b, :T, :U - 1], np.broadcast_to(lab[None, :, None], (T, U - 1, 1)),
                                            axis=-1)[..., 0]
    return lpb, lpl


def viterbi(lp, labels, input_lengths, label_lengths, blank=0):
    """lp (B,maxT,maxU,V) float64 log-probs.  Returns label_frames (B, maxU-1) int32 (-1 padded), best_logp (B,) and
    gap (B,) (inf when the lattice holds a single path)."""
    lp = np.asarray(lp, np.float64)
    B, _, maxU, _ = lp.shape
    frames = np.full((B, max(maxU - 1, 0)), -1, np.int32)
    best, gap = np.empty(B), np.empty(B)
    for b in range(B):
        T, U = int(input_lengths[b]), int(label_lengths[b]) + 1
        lpb, lpl = _arcs(lp, labels, b, T, U, blank)
        delta = np.full((T, U), -np.inf)
        lab = np.zeros((T, U), bool)
        margin = np.full((T, U), np.inf)
        delta[0, 0] = 0.0
        for n in range(1, T + U - 1):                         # anti-diagonals: each depends on the previous one only
            u = np.arange(max(0, n - T + 1), min(n, U - 1) + 1)
            t = n - u
            tb, ul = np.maximum(t - 1, 0), np.maximum(u - 1, 0)
            nb = np.where(t > 0, delta[tb, u] + lpb[tb, u], -np.inf)
            nl = np.where(u > 0, delta[t, ul] + lpl[t, ul], -np.inf)
            take = (nl > nb) | (t == 0)
            delta[t, u] = np.where(take, nl, nb)
            lab[t, u] = take
            both = (t > 0) & (u > 0)
            margin[t, u] = np.where(both, np.abs(nl - nb), np.inf)
        best[b] = delta[T - 1, U - 1] + lpb[T - 1, U - 1]
        t, u, g = T - 1, U - 1, np.inf
        while t > 0 or u > 0:
            g = min(g, margin[t, u])
            if u > 0 and lab[t, u]:
                u -= 1
                frames[b, u] = t
            else:
                t -= 1
        gap[b] = g
    return frames, best, gap


def path_score(lp, labels, frames, input_lengths, label_lengths, blank=0):
    """float64 log-probability (B,) of the alignments `frames` (label j emitted at frame frames[b, j])."""
    lp = np.asarray(lp, np.float64)
    B = lp.shape[0]
    out = np.empty(B)
    for b in range(B):
        T, U = int(input_lengths[b]), int(label_lengths[b]) + 1
        lpb, lpl = _arcs(lp, labels, b, T, U, blank)
        f = np.asarray(frames[b][:U - 1], np.int64)
        u_at = np.searchsorted(f, np.arange(T), side="right")     # labels emitted by the end of frame t
        out[b] = lpl[f, np.arange(U - 1)].sum() + lpb[np.arange(T), u_at].sum()
    return out


def check_frames(frames, input_lengths, label_lengths):
    """Padding exactly -1; per utterance non-decreasing and within [0, T_b)."""
    frames = np.asarray(frames)
    for b in range(frames.shape[0]):
        n = int(label_lengths[b])
        f = frames[b, :n]
        assert np.all(frames[b, n:] == -1), (b, frames[b, n:])
        assert np.all(f >= 0) and np.all(f < int(input_lengths[b])) and np.all(np.diff(f) >= 0), (b, f)
