"""Float64 reference of the alignment-restricted RNN-T loss (TEST INFRASTRUCTURE), written for this purpose.

Definition (DESIGN §1): per utterance b and lattice column u an inclusive frame window [t_lo[b,u], t_hi[b,u]]; cell (t,u)
is allowed iff t_lo <= t <= t_hi and t < T_b; both arcs leaving a cell that is not allowed have log-probability -inf, as
does the terminating blank if the last cell is not allowed.  cost = -log sum P(path) over the paths through allowed cells.

  * `allowed_mask`      the definition, cell by cell;
  * `masked_dp`         alpha / beta over the masked arc log-probs (numpy float64, whole batch per anti-diagonal):
                        costs and the arc gradients G_blank = d cost / d lp_blank(t,u), G_label = d cost / d lp_label(t,u)
                        (minus the arc occupancies).  Windows that admit no path: cost +inf, gradients 0;
  * `enumerate_cost`    -log of the sum over every admitted path, by recursion (tiny lattices: pins masked_dp);
  * `logits_grad`       costs and the dense gradient w.r.t. raw logits (softmax inside), FastEmit's (1 + lambda) on label arcs;
  * `joint_loss_grad`   the fused path, chunked over lattice rows with tests/joint_ref64.py's two passes.
"""
import numpy as np
import torch

import joint_ref64 as R

NEG = -np.inf


def allowed_mask(windows, input_lengths, label_lengths, T, U):
    """bool (B,T,U): inside the utterance's lattice and, with windows, inside the column's window."""
    il = np.asarray(input_lengths, np.int64).reshape(-1)
    ll = np.asarray(label_lengths, np.int64).reshape(-1)
    t = np.arange(T)[None, :, None]
    u = np.arange(U)[None, None, :]
    ok = (t < il[:, None, None]) & (u <= ll[:, None, None])
    if windows is not None:
        lo, hi = (np.asarray(w, np.int64)[:, None, :] for w in windows)
        ok &= (t >= lo) & (t <= hi)
    return ok


def _lse(a, b):
    m = np.maximum(a, b)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = m + np.log(np.exp(a - m) + np.exp(b - m))
    return np.where(np.isneginf(m), NEG, r)


def masked_dp(lpb, lpl, input_lengths, label_lengths, windows=None):
    """lpb, lpl (B,T,U): log-probs of the blank / label arc leaving each cell.  Returns costs (B,), G_blank, G_label (B,T,U)."""
    lpb, lpl = np.asarray(lpb, np.float64), np.asarray(lpl, np.float64)
    B, T, U = lpb.shape
    il = np.asarray(input_lengths, np.int64).reshape(-1)
    ll = np.asarray(label_lengths, np.int64).reshape(-1)
    ok = allowed_mask(windows, il, ll, T, U)
    u_idx = np.arange(U)[None, None, :]
    mb = np.where(ok, lpb, NEG)
    ml = np.where(ok & (u_idx < ll[:, None, None]), lpl, NEG)
    bi = np.arange(B)
    term = np.full((B, T, U), NEG)                    # the terminating blank, leaving (T_b-1, U_b-1)
    term[bi, il - 1, ll] = mb[bi, il - 1, ll]
    # blank arcs that stay inside the lattice: from t < T_b - 1 (padded cells are -inf already)
    mb_in = np.where(np.arange(T)[None, :, None] < il[:, None, None] - 1, mb, NEG)
    alpha = np.full((B, T + 1, U + 1), NEG)
    beta = np.full((B, T + 1, U + 1), NEG)
    alpha[:, 0, 0] = 0.0
    for n in range(1, T + U - 1):
        u = np.arange(max(0, n - T + 1), min(U - 1, n) + 1)
        t = n - u
        up = np.where(t > 0, alpha[:, t - 1, u] + mb_in[:, np.maximum(t - 1, 0), u], NEG)
        left = np.where(u > 0, alpha[:, t, u - 1] + ml[:, t, np.maximum(u - 1, 0)], NEG)
        alpha[:, t, u] = _lse(up, left)
    for n in range(T + U - 2, -1, -1):
        u = np.arange(max(0, n - T + 1), min(U - 1, n) + 1)
        t = n - u
        beta[:, t, u] = _lse(_lse(beta[:, t + 1, u] + mb_in[:, t, u], beta[:, t, u + 1] + ml[:, t, u]), term[:, t, u])
    a, bt = alpha[:, :T, :U], beta
    llf = a[bi, il - 1, ll] + mb[bi, il - 1, ll]
    feas = np.isfinite(llf)
    z = np.where(feas, llf, 0.0)[:, None, None]
    with np.errstate(invalid="ignore"):
        gb = -(np.exp(a + mb_in + bt[:, 1:, :U] - z) + np.exp(a + term - z))
        gl = -np.exp(a + ml + bt[:, :T, 1:] - z)
    gb = np.where(feas[:, None, None] & np.isfinite(gb), gb, 0.0)
    gl = np.where(feas[:, None, None] & np.isfinite(gl), gl, 0.0)
    return np.where(feas, -llf, np.inf), gb, gl


def enumerate_cost(lpb, lpl, T, U, allowed):
    """One utterance (lpb, lpl, allowed: (>=T, >=U)): -log sum over every path (0,0) -> terminating blank that visits allowed
    cells only, each path's log-probability summed arc by arc."""
    paths = []

    def walk(t, u, lp):
        if not allowed[t, u]:
            return
        if t == T - 1 and u == U - 1:
            paths.append(lp + lpb[t, u])
        if t < T - 1:
            walk(t + 1, u, lp + lpb[t, u])
        if u < U - 1:
            walk(t, u + 1, lp + lpl[t, u])

    walk(0, 0, 0.0)
    if not paths:
        return np.inf
    p = np.asarray(paths)
    return -(p.max() + np.log(np.exp(p - p.max()).sum()))


def log_softmax(x):
    x = np.asarray(x, np.float64)
    m = x.max(axis=-1, keepdims=True)
    return x - (m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True)))


def arc_logprobs(lp, labels, blank):
    """(B,T,U,V) log-probs -> lpb, lpl (B,T,U) (lpl of the last column: 0, masked by the DP)."""
    B, T, U, V = lp.shape
    lab = np.zeros((B, U), np.int64)
    if U > 1:
        lab[:, :U - 1] = np.asarray(labels, np.int64).reshape(B, -1)[:, :U - 1]
    lpl = np.take_along_axis(lp, np.broadcast_to(lab[:, None, :, None], (B, T, U, 1)), axis=-1)[..., 0]
    return lp[..., blank], lpl, lab


def logits_grad(acts, labels, input_lengths, label_lengths, blank=0, windows=None, fastemit_lambda=0.0, grad_scale=None):
    """GPU-op semantics: raw logits in, costs (B,) and d costs / d logits (B,T,U,V) out (times grad_scale[b]); 0 in padded
    and not-allowed cells."""
    lp = log_softmax(acts)
    B, T, U, V = lp.shape
    lpb, lpl, lab = arc_logprobs(lp, labels, blank)
    costs, gb, gl = masked_dp(lpb, lpl, input_lengths, label_lengths, windows)
    gl = (1.0 + fastemit_lambda) * gl
    dlp = np.zeros((B, T, U, V))
    dlp[..., blank] = gb
    np.add.at(dlp, (np.arange(B)[:, None, None], np.arange(T)[None, :, None], np.arange(U)[None, None, :], lab[:, None, :]), gl)
    dx = dlp - np.exp(lp) * dlp.sum(axis=-1, keepdims=True)
    if grad_scale is not None:
        dx *= np.asarray(grad_scale, np.float64)[:, None, None, None]
    return costs, dx


def joint_loss_grad(enc, pred, W, bias, labels, input_lengths, label_lengths, blank=0, windows=None, grad_scale=None,
                    fastemit_lambda=0.0, chunk_rows=None, device=None):
    """The fused path in float64 with windows: dict(costs, d_enc, d_pred, dW, db) as numpy; joint_ref64.joint_loss_grad with
    the arc gradients of masked_dp in place of the oracle's."""
    if device is None:
        device = enc.device if isinstance(enc, torch.Tensor) else torch.device("cpu")
    enc, pred, W, bias = (R._f64(a, device) for a in (enc, pred, W, bias))
    B, maxT, H = enc.shape
    maxU, V = pred.shape[1], W.shape[1]
    rows = chunk_rows or R.default_chunk_rows(V)
    host = lambda x: x.cpu().numpy() if isinstance(x, torch.Tensor) else x
    labels, input_lengths, label_lengths = host(labels), host(input_lengths), host(label_lengths)
    if windows is not None:
        windows = tuple(host(w) for w in windows)
    cells = R.Cells(labels, input_lengths, label_lengths, maxT, maxU, blank, device)

    def logits_of(sl):
        z = torch.tanh(enc[cells.b[sl], cells.t[sl]] + pred[cells.b[sl], cells.u[sl]])
        return torch.addmm(bias, z, W), z

    lpb, lpl, lse = R._pass1(cells, logits_of, rows)
    idx = (cells.b_host, cells.t_host, cells.u_host)
    pb, pl = np.zeros((B, maxT, maxU)), np.zeros((B, maxT, maxU))
    pb[idx], pl[idx] = lpb.cpu().numpy(), lpl.cpu().numpy()
    costs, gb, gl = masked_dp(pb, pl, input_lengths, label_lengths, windows)
    gb, gl = R._scaled_arcs(cells, torch.as_tensor(gb[idx], device=device), torch.as_tensor(gl[idx], device=device),
                            grad_scale, fastemit_lambda)
    d_enc, d_pred = torch.zeros(B * maxT, H, dtype=R.F64, device=device), torch.zeros(B * maxU, H, dtype=R.F64, device=device)
    dW, db = torch.zeros(H, V, dtype=R.F64, device=device), torch.zeros(V, dtype=R.F64, device=device)

    def consume(sl, dl, z):
        dW.addmm_(z.T, dl)
        db.add_(dl.sum(dim=0))
        dpre = (dl @ W.T).mul_(1.0 - z * z)
        d_enc.index_add_(0, cells.b[sl] * maxT + cells.t[sl], dpre)
        d_pred.index_add_(0, cells.b[sl] * maxU + cells.u[sl], dpre)

    R._pass2(cells, logits_of, lse, gb, gl, rows, consume)
    return dict(costs=costs, d_enc=d_enc.view(B, maxT, H).cpu().numpy(), d_pred=d_pred.view(B, maxU, H).cpu().numpy(),
                dW=dW.cpu().numpy(), db=db.cpu().numpy())


def random_feasible_windows(rng, input_lengths, label_lengths, U, slack=3):
    """Windows around a random monotone path per utterance, widened by up to `slack` frames on either side: always feasible.
    Returns int32 (t_lo, t_hi) of shape (B, U)."""
    B = len(input_lengths)
    lo, hi = np.zeros((B, U), np.int32), np.full((B, U), -1, np.int32)
    for b, (T, yl) in enumerate(zip(input_lengths, label_lengths)):
        T, Un = int(T), int(yl) + 1
        a = np.sort(rng.integers(0, T, Un - 1)) if Un > 1 else np.zeros(0, np.int64)
        prev = np.concatenate([[0], a])
        nxt = np.concatenate([a, [T - 1]])
        lo[b, :Un] = np.maximum(0, prev - rng.integers(0, slack + 1, Un))
        hi[b, :Un] = np.minimum(T - 1, nxt + rng.integers(0, slack + 1, Un))
    return lo, hi
