"""Float64 reference of pruned RNN-T (TEST INFRASTRUCTURE), written for this purpose: the trivial joiner's simple loss and
the band policy of DESIGN §1.

  * `simple_loss_grad`  costs, d_am, d_lm of the RNN-T loss on the materialised logits am[:,:,None] + lm[:,None]
                        (tests/window_ref.py's float64 loss, softmax inside), times grad_scale;
  * `occupancies`       gamma_B, gamma_L (B,T,U): blank- and label-arc occupancies of the simple lattice;
  * `scores`            score(t,s) of one utterance, by direct windowed sums;
  * `band`              the raw argmax, the two scans over t and the per-column windows (t_lo, t_hi), (B,U) int32;
  * `enumerate_paths`   every path of a small lattice with its probability (pins the band's statements).
"""
import itertools

import numpy as np

import window_ref as wr


def random_case(rng, B, T, U, V, blank=0, scale=1.0, ragged=True, label_blank=False):
    """am (B,T,V), lm (B,U,V) float64, labels (B, max(U-1,1)) int32, lengths; utterance 0 spans (T, U).  label_blank: every
    label equals blank."""
    am, lm = rng.standard_normal((B, T, V)) * scale, rng.standard_normal((B, U, V)) * scale
    labels = rng.integers(0, V, (B, max(U - 1, 1))).astype(np.int32)
    if label_blank:
        labels[:] = blank
    il = rng.integers(1, T + 1, B).astype(np.int32) if ragged else np.full(B, T, np.int32)
    ll = rng.integers(0, U, B).astype(np.int32) if ragged else np.full(B, U - 1, np.int32)
    il[0], ll[0] = T, U - 1
    return am, lm, labels, il, ll


def logits(am, lm):
    return np.asarray(am, np.float64)[:, :, None, :] + np.asarray(lm, np.float64)[:, None, :, :]


def simple_loss_grad(am, lm, labels, input_lengths, label_lengths, blank=0, grad_scale=None):
    costs, dx = wr.logits_grad(logits(am, lm), labels, input_lengths, label_lengths, blank, grad_scale=grad_scale)
    return costs, dx.sum(axis=2), dx.sum(axis=1)


def simple_loss_grad_f64(am, lm, labels, input_lengths, label_lengths, blank=0, grad_scale=None, device="cpu"):
    """simple_loss_grad without the (B,T,U,V) tensor, for full-size batches: torch float64 on `device`, the normaliser as
    ma + ml + log(exp(am - ma) . exp(lm - ml)^T) (exact in float64 down to gaps of ~700 nats), window_ref's masked_dp for
    the lattice, and the gradients from the cell occupancy gamma = gamma_B + gamma_L:
        d_am[t] = sum_u g (gamma p - gamma_B e_blank - gamma_L e_{y_u}),   d_lm[u] likewise over t.
    Returns numpy costs, d_am, d_lm."""
    import torch
    f = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float64, device=device)
    am, lm = f(am), f(lm)
    B, T, V = am.shape
    U = lm.shape[1]
    il, ll = np.asarray(input_lengths, np.int64), np.asarray(label_lengths, np.int64)
    ma, ml = am.max(dim=2, keepdim=True).values, lm.max(dim=2, keepdim=True).values
    Ea, El = torch.exp(am - ma), torch.exp(lm - ml)
    rel = torch.log(torch.bmm(Ea, El.transpose(1, 2)))                 # lse - ma - ml, (B,T,U)
    lse = rel + ma + ml.transpose(1, 2)
    lpb = am[:, :, blank][:, :, None] + lm[:, :, blank][:, None, :] - lse
    lab = torch.as_tensor(np.asarray(labels, np.int64).reshape(B, -1)[:, :max(U - 1, 0)], device=device)
    lpl = torch.zeros_like(lpb)
    if U > 1:
        am_y = torch.gather(am, 2, lab[:, None, :].expand(B, T, U - 1))
        lm_y = torch.gather(lm[:, :U - 1], 2, lab[:, :, None])[..., 0]
        lpl[:, :, :U - 1] = am_y + lm_y[:, None, :] - lse[:, :, :U - 1]
    costs, gb, gl = wr.masked_dp(lpb.cpu().numpy(), lpl.cpu().numpy(), il, ll)
    gs = np.ones(B) if grad_scale is None else np.asarray(grad_scale, np.float64)
    gB, gL = f(-gb * gs[:, None, None]), f(-gl * gs[:, None, None])
    G = (gB + gL) * torch.exp(-rel)
    G = torch.where(torch.isfinite(G), G, torch.zeros_like(G))
    d_am = Ea * torch.bmm(G, El)
    d_lm = El * torch.bmm(G.transpose(1, 2), Ea)
    d_am[:, :, blank] -= gB.sum(dim=2)
    d_lm[:, :, blank] -= gB.sum(dim=1)
    if U > 1:
        d_am.scatter_add_(2, lab[:, None, :].expand(B, T, U - 1), -gL[:, :, :U - 1])
        d_lm[:, :U - 1].scatter_add_(2, lab[:, :, None], -gL[:, :, :U - 1].sum(dim=1)[:, :, None])
    for b in range(B):
        d_am[b, il[b]:] = 0
        d_lm[b, ll[b] + 1:] = 0
    return costs, d_am.cpu().numpy(), d_lm.cpu().numpy()


def occupancies(am, lm, labels, input_lengths, label_lengths, blank=0):
    lp = wr.log_softmax(logits(am, lm))
    lpb, lpl, _ = wr.arc_logprobs(lp, labels, blank)
    costs, gb, gl = wr.masked_dp(lpb, lpl, input_lengths, label_lengths)
    return costs, -gb, -gl


def scores(gB, gL, Tn, Un, S):
    """score(t,s) (T_b - 1, max(0, U_b - S) + 1) of one utterance: sum_{u=s}^{min(s+S,U_b)-1} gB(t,u) - gL(t,s-1)."""
    smax = max(0, Un - S)
    sc = np.zeros((max(Tn - 1, 0), smax + 1))
    for t in range(Tn - 1):
        for s in range(smax + 1):
            sc[t, s] = gB[t, s:min(s + S, Un)].sum() - (gL[t, s - 1] if s > 0 else 0.0)
    return sc


def band_starts(gB, gL, Tn, Un, S):
    """s_t (T_b,) of one utterance after the raw argmax, the monotone scan and the bounded-step scan."""
    sc = scores(gB, gL, Tn, Un, S)
    s = np.zeros(Tn, np.int64)
    if Tn > 1:
        s[:Tn - 1] = np.argmax(sc, axis=1)                     # the smallest argmax
    s[Tn - 1] = max(0, Un - S)
    s = np.minimum.accumulate(s[::-1])[::-1]
    t = np.arange(Tn)
    q = np.maximum.accumulate((s - (S - 1) * t)[::-1])[::-1]   # max_{t' >= t} (s_t' - (S-1) t')
    return np.minimum((S - 1) * t, (S - 1) * t + q)


def windows_of_starts(starts, Un, S, U):
    """(t_lo, t_hi) (U,) of one utterance: the frames whose band [s_t, s_t + S) holds column u; (0, -1) when none."""
    lo, hi = np.zeros(U, np.int32), np.full(U, -1, np.int32)
    for u in range(Un):
        ts = [t for t, s in enumerate(starts) if s <= u < s + S]
        if ts:
            lo[u], hi[u] = min(ts), max(ts)
    return lo, hi


def band(am, lm, labels, input_lengths, label_lengths, S, blank=0):
    """The band of a batch: (t_lo, t_hi) (B,U) int32 and the per-utterance starts."""
    _, gB, gL = occupancies(am, lm, labels, input_lengths, label_lengths, blank)
    B, U = len(input_lengths), np.asarray(lm).shape[1]
    lo, hi, starts = np.zeros((B, U), np.int32), np.zeros((B, U), np.int32), []
    for b in range(B):
        Tn, Un = int(input_lengths[b]), int(label_lengths[b]) + 1
        st = band_starts(gB[b], gL[b], Tn, Un, S)
        starts.append(st)
        lo[b], hi[b] = windows_of_starts(st, Un, S, U)
    return lo, hi, starts


def score_margins(am, lm, labels, input_lengths, label_lengths, S, blank=0):
    """Per utterance, the smallest gap over frames t < T_b - 1 between the best score and the best other start (inf when
    a frame has a single start): where it exceeds the GPU's round-off, the GPU must pick the same raw starts."""
    _, gB, gL = occupancies(am, lm, labels, input_lengths, label_lengths, blank)
    out = []
    for b in range(len(input_lengths)):
        Tn, Un = int(input_lengths[b]), int(label_lengths[b]) + 1
        sc = scores(gB[b], gL[b], Tn, Un, S)
        m = np.inf
        if sc.shape[1] > 1:
            srt = np.sort(sc, axis=1)
            m = float((srt[:, -1] - srt[:, -2]).min()) if len(sc) else np.inf
        out.append(m)
    return np.asarray(out)


def enumerate_paths(lpb, lpl, Tn, Un):
    """Every path (0,0) -> terminating blank of one utterance as (probability, segments), segments[t] = (entry, exit): the
    label positions the path visits at frame t."""
    out = []
    for ups in itertools.combinations(range(Tn + Un - 2), Un - 1):       # positions of the label arcs among the moves
        ups = set(ups)
        t = u = 0
        lp, seg = 0.0, [[0, 0] for _ in range(Tn)]
        for i in range(Tn + Un - 2):
            if i in ups:
                lp += lpl[t, u]
                u += 1
            else:
                lp += lpb[t, u]
                t += 1
                seg[t][0] = u
            seg[t][1] = u
        lp += lpb[Tn - 1, Un - 1]
        out.append((np.exp(lp), [tuple(s) for s in seg]))
    return out
