"""Float64 reference of the fused joint + loss and of the loss op that scales to full benchmark sizes (TEST
INFRASTRUCTURE).  Plain torch on whatever device its tensors are on: CUDA float64 in the GPU tests, CPU in the host test.

The O(N·V) work runs in chunks of valid lattice rows (cells (b, t, u) with t < T_b, u <= U_b), in two passes:

  1. logits of the chunk (joint: `z = tanh(enc[b,t] + pred[b,u])`, `z·W + b`; op: a caller's callback), their
     log-softmax, and of it only `lp_blank(t,u)` and `lp_label(t,u)` (plus the row's log-normaliser for pass 2);
  2. the costs and the arc gradients `G_blank = ∂cost/∂lp_blank`, `G_label = ∂cost/∂lp_label` from the C oracle's
     dynamic program run on a two-column log-prob plane (column 0 the blank arcs, column 1 the label arcs, every label 1,
     blank 0): O(B·T·U) data.  A label equal to blank needs no special case, as the two arcs have columns of their own.
     FastEmit multiplies `G_label` by (1 + λ);
  3. the chunk's logits again, the logits gradient `g_b·[G_b·δ(v,blank) + G_l·δ(v,label_u) − (G_b + G_l)·p_v]` (the chain
     rule of tests/fastemit_ref.py's log-prob gradient through the softmax), and from it (joint) `dW += zᵀ·dlogit`,
     `db += Σ dlogit`, `dZ = dlogit·Wᵀ` and the u- and t-sums of `dZ·(1 − z²)` into `d_enc` and `d_pred`; (op) the
     chunk's logits gradient to the caller.

Padded cells are never formed, so they contribute nothing.  Nothing of the kernels' closed forms is used.
tests/test_joint_ref64_host.py pins this module to the oracle and tests/fastemit_ref.py at the 1e-12 level.
"""
import numpy as np
import torch

from oracle import oracle as _oracle

F64 = torch.float64


def default_chunk_rows(V):
    """About 64 k lattice rows, at most 2^31 logits (16 GiB of float64) per chunk."""
    return max(1, min(65536, (1 << 31) // V))


class Cells:
    """The valid lattice cells of a batch in (b, t, u) order, as int64 tensors on `device`, with each cell's label
    (blank on the last row u = U_b - 1, which has no label arc)."""

    def __init__(self, labels, input_lengths, label_lengths, maxT, maxU, blank, device):
        il = np.asarray(input_lengths, np.int64).reshape(-1)
        ll = np.asarray(label_lengths, np.int64).reshape(-1)
        lab = np.asarray(labels, np.int64).reshape(len(il), -1)
        b, t, u = [], [], []
        for i, (T, U) in enumerate(zip(il, ll + 1)):
            tt, uu = np.meshgrid(np.arange(T), np.arange(U), indexing="ij")
            b.append(np.full(T * U, i))
            t.append(tt.reshape(-1))
            u.append(uu.reshape(-1))
        b, t, u = (np.concatenate(x) if x else np.zeros(0, np.int64) for x in (b, t, u))
        has_label = u < ll[b]
        cell_lab = np.full(len(b), blank, np.int64)
        cell_lab[has_label] = lab[b[has_label], u[has_label]]
        self.B, self.maxT, self.maxU, self.blank = len(il), int(maxT), int(maxU), int(blank)
        self.il, self.ll, self.N = il, ll, len(b)
        self.b_host, self.t_host, self.u_host = b, t, u
        self.b, self.t, self.u, self.lab = (torch.as_tensor(x, device=device) for x in (b, t, u, cell_lab))

    def chunks(self, rows):
        for r0 in range(0, self.N, rows):
            yield slice(r0, min(self.N, r0 + rows))


def _pass1(cells, logits_of, rows):
    """Per valid cell: log-softmax at the blank and at the cell's label, and the row's log-normaliser."""
    dev = cells.b.device
    lpb, lpl, lse = (torch.empty(cells.N, dtype=F64, device=dev) for _ in range(3))
    for sl in cells.chunks(rows):
        x = logits_of(sl)[0]
        xb = x[:, cells.blank].clone()
        xl = x.gather(1, cells.lab[sl, None])[:, 0]
        m = x.max(dim=1).values
        x.sub_(m[:, None]).exp_()                  # in place: one (rows, V) buffer per chunk
        lse[sl] = m + x.sum(dim=1).log()
        lpb[sl], lpl[sl] = xb - lse[sl], xl - lse[sl]
        del x
    return lpb, lpl, lse


def _arc_grads(cells, lpb, lpl):
    """costs (B,) float64 numpy and G_blank, G_label per valid cell (tensors on the cells' device), from the C oracle on
    the two-column plane."""
    B, maxT, maxU = cells.B, cells.maxT, cells.maxU
    plane = np.zeros((B, maxT, maxU, 2))
    idx = (cells.b_host, cells.t_host, cells.u_host)
    plane[idx + (0,)] = lpb.cpu().numpy()
    plane[idx + (1,)] = lpl.cpu().numpy()
    ones = np.ones((B, max(maxU - 1, 1)), np.int32)
    costs, g = _oracle.rnnt_cost_and_grad(plane, ones, cells.il.astype(np.int32), cells.ll.astype(np.int32), 0)
    dev = cells.b.device
    gb = torch.as_tensor(g[idx + (0,)], device=dev)
    gl = torch.as_tensor(g[idx + (1,)], device=dev)
    return costs, gb, gl


def _pass2(cells, logits_of, lse, gb, gl, rows, consume):
    """The logits gradient of each chunk (gb, gl already carry the upstream gradient and FastEmit) to consume(sl, dl, ctx)."""
    for sl in cells.chunks(rows):
        x, ctx = logits_of(sl)
        x.sub_(lse[sl, None]).exp_()               # p
        x.mul_(-(gb[sl] + gl[sl])[:, None])
        x[:, cells.blank] += gb[sl]
        x.scatter_add_(1, cells.lab[sl, None], gl[sl, None])
        consume(sl, x, ctx)
        del x, ctx


def _scaled_arcs(cells, gb, gl, grad_scale, fastemit_lambda):
    dev = gb.device
    g = torch.ones(cells.B, dtype=F64, device=dev) if grad_scale is None else \
        torch.as_tensor(np.asarray(grad_scale, np.float64).reshape(-1), device=dev)
    gc = g[cells.b]
    return gb * gc, gl * ((1.0 + fastemit_lambda) * gc)


def _f64(a, device):
    if isinstance(a, torch.Tensor):
        return a.detach().to(device=device, dtype=F64)
    return torch.as_tensor(np.asarray(a, np.float64), device=device)


def joint_loss_grad(enc, pred, W, bias, labels, input_lengths, label_lengths, blank=0, grad_scale=None,
                    fastemit_lambda=0.0, chunk_rows=None, device=None):
    """The fused path in float64: dict(costs, d_enc, d_pred, dW, db) as numpy, as oracle.joint_loss_grad (and
    fastemit_ref.joint_loss_grad for lambda > 0).  Inputs are numpy arrays or tensors; the work runs on `device`
    (default: enc's device when it is a tensor, else the CPU)."""
    if device is None:
        device = enc.device if isinstance(enc, torch.Tensor) else torch.device("cpu")
    enc, pred, W, bias = (_f64(a, device) for a in (enc, pred, W, bias))
    B, maxT, H = enc.shape
    maxU, V = pred.shape[1], W.shape[1]
    rows = chunk_rows or default_chunk_rows(V)
    cells = Cells(labels.cpu().numpy() if isinstance(labels, torch.Tensor) else labels,
                  *(x.cpu().numpy() if isinstance(x, torch.Tensor) else x for x in (input_lengths, label_lengths)),
                  maxT, maxU, blank, device)

    def logits_of(sl):
        z = torch.tanh(enc[cells.b[sl], cells.t[sl]] + pred[cells.b[sl], cells.u[sl]])
        return torch.addmm(bias, z, W), z

    lpb, lpl, lse = _pass1(cells, logits_of, rows)
    costs, gb, gl = _arc_grads(cells, lpb, lpl)
    gb, gl = _scaled_arcs(cells, gb, gl, grad_scale, fastemit_lambda)
    d_enc, d_pred = torch.zeros(B * maxT, H, dtype=F64, device=device), torch.zeros(B * maxU, H, dtype=F64, device=device)
    dW, db = torch.zeros(H, V, dtype=F64, device=device), torch.zeros(V, dtype=F64, device=device)

    def consume(sl, dl, z):
        dW.addmm_(z.T, dl)
        db.add_(dl.sum(dim=0))
        dpre = (dl @ W.T).mul_(1.0 - z * z)
        d_enc.index_add_(0, cells.b[sl] * maxT + cells.t[sl], dpre)
        d_pred.index_add_(0, cells.b[sl] * maxU + cells.u[sl], dpre)

    _pass2(cells, logits_of, lse, gb, gl, rows, consume)
    return dict(costs=costs, d_enc=d_enc.view(B, maxT, H).cpu().numpy(), d_pred=d_pred.view(B, maxU, H).cpu().numpy(),
                dW=dW.cpu().numpy(), db=db.cpu().numpy())


def op_loss_grad(logits_of, shape, labels, input_lengths, label_lengths, blank=0, grad_scale=None, fastemit_lambda=0.0,
                 chunk_rows=None, device="cpu", on_grad=None):
    """The loss op in float64 on materialised logits of `shape` = (B, maxT, maxU, V), read through the callback
    `logits_of(b, t, u)` -> (rows, V) float64 tensor of those cells' logits (a fresh tensor: it is overwritten).

    Returns the costs (B,) and, without `on_grad`, the dense logits gradient (B, maxT, maxU, V) as numpy (0 in padded
    cells).  With `on_grad`, each chunk's gradient goes to `on_grad(b, t, u, dlogits)` instead and None is returned in
    its place: the caller keeps the block it wants."""
    B, maxT, maxU, V = shape
    rows = chunk_rows or default_chunk_rows(V)
    cells = Cells(labels, input_lengths, label_lengths, maxT, maxU, blank, device)

    def logits_of_chunk(sl):
        return logits_of(cells.b[sl], cells.t[sl], cells.u[sl]), None

    lpb, lpl, lse = _pass1(cells, logits_of_chunk, rows)
    costs, gb, gl = _arc_grads(cells, lpb, lpl)
    gb, gl = _scaled_arcs(cells, gb, gl, grad_scale, fastemit_lambda)
    dense = None
    if on_grad is None:
        dense = torch.zeros(B, maxT, maxU, V, dtype=F64, device=device)

        def on_grad(b, t, u, dl):
            dense[b, t, u] = dl

    _pass2(cells, logits_of_chunk, lse, gb, gl, rows,
           lambda sl, dl, _: on_grad(cells.b[sl], cells.t[sl], cells.u[sl], dl))
    return costs, (None if dense is None else dense.cpu().numpy())
