"""Alignment-restricted RNN-T (Mahadeokar et al., "Alignment Restricted Streaming Recurrent Neural Network Transducer",
SLT 2021): per-label time windows for the loss.

The loss entries take ``windows=(t_lo, t_hi)``: two int32 CUDA tensors (B, U), U = max label length + 1.  Cell (t, u) of
utterance b is allowed iff ``t_lo[b,u] <= t <= t_hi[b,u]`` (and t < T_b); both arcs leaving any other cell have
log-probability -inf, so ``costs[b] = -log sum P(path)`` over the paths that visit allowed cells only (DESIGN §1,
include/rnnt_b200.h).  Nothing is clamped: an empty or out-of-range window is an empty column; windows that admit no path
give a cost of +inf and zero gradients.  ``alignment_windows`` is the Ar-RNN-T policy on top of that: windows around a
reference alignment such as ``rnnt_align`` / ``joint_rnnt_align`` return.
"""
import numpy as np
import torch

__all__ = ["alignment_windows", "valid_tile_count"]


def alignment_windows(label_frames, input_lengths, label_lengths, left, right):
    """Windows that let label j be emitted exactly at the frames ``[a_j - left, a_j + right]`` around the reference
    alignment ``a = label_frames`` ((B, U-1) int32, ``Alignment.label_frames`` with its -1 padding): with a_{-1} = 0 and
    a_{U_b-1} = T_b - 1,

        t_lo[b,u] = max(0, a_{u-1} - left),    t_hi[b,u] = min(T_b - 1, a_u + right).

    The reference path itself is always admitted (the cost is finite); ``left = right = 0`` admits that path only.
    Device tensors in, ``(t_lo, t_hi)`` int32 (B, U) on the same device out, no host synchronisation.  Columns past an
    utterance's U_b hold the empty window (0, -1); the library ignores them."""
    left, right = int(left), int(right)
    if left < 0 or right < 0:
        raise ValueError("left and right must be >= 0")
    if label_frames.dim() != 2 or input_lengths.shape != (label_frames.shape[0],) or label_lengths.shape != input_lengths.shape:
        raise ValueError("expected label_frames (B, U-1) and a length per example")
    B, U = label_frames.shape[0], label_frames.shape[1] + 1
    dev = label_frames.device
    frames = label_frames.to(torch.int64)
    zero = torch.zeros(B, 1, dtype=torch.int64, device=dev)
    u = torch.arange(U, device=dev).unsqueeze(0)
    last = (input_lengths.to(torch.int64) - 1).unsqueeze(1)                 # T_b - 1
    ylen = label_lengths.to(torch.int64).unsqueeze(1)
    a_u = torch.where(u < ylen, torch.cat([frames, zero], 1), last)         # a_u, a_{U_b-1} = T_b - 1
    a_prev = torch.cat([zero, frames], 1)                                   # a_{u-1}, a_{-1} = 0
    t_lo = torch.clamp(a_prev - left, min=0)
    t_hi = torch.minimum(a_u + right, last)
    pad = u > ylen
    t_lo = torch.where(pad, torch.zeros_like(t_lo), t_lo)
    t_hi = torch.where(pad, torch.full_like(t_hi, -1), t_hi)
    return t_lo.to(torch.int32).contiguous(), t_hi.to(torch.int32).contiguous()


def check_windows(windows, B, U, device):
    """``windows`` of a loss call as the C entries take them: (None, None), or two contiguous int32 CUDA tensors (B, U)."""
    if windows is None:
        return None, None
    try:
        t_lo, t_hi = windows
    except (TypeError, ValueError):
        raise ValueError("windows must be a pair (t_lo, t_hi)") from None
    for t, n in ((t_lo, "t_lo"), (t_hi, "t_hi")):
        if not isinstance(t, torch.Tensor):
            raise TypeError("windows: %s must be a tensor (both bounds are required)" % n)
    for t, n in ((t_lo, "t_lo"), (t_hi, "t_hi")):
        if t.dtype != torch.int32:
            raise TypeError("windows: %s must be torch.int32" % n)
        if not t.is_cuda or t.device != device:
            raise RuntimeError("windows: %s must be a CUDA tensor on the device of the inputs" % n)
        if tuple(t.shape) != (B, U):
            raise ValueError("windows: %s must be (B, U) = (%d, %d), got %s" % (n, B, U, tuple(t.shape)))
    return t_lo.contiguous(), t_hi.contiguous()


def valid_tile_count(input_lengths, label_lengths, windows=None):
    """Number of 16 x 8 lattice tiles of a batch that are valid, from HOST copies of the lengths (lists, numpy arrays or
    CPU tensors): the value ``joint_rnnt_loss(..., valid_tiles=...)`` / ``rnntb200JointDesc.valid_tile_bound`` expects.
    Without windows a tile is valid iff it intersects the utterance's T_b x U_b lattice; with ``windows=(t_lo, t_hi)``
    (host copies, (B, U)) iff in addition some column u of its 8 (u < U_b) has [t_lo, t_hi] meet its 16 frames -- the
    rule of the library's tile compaction.  A data loader has the lengths on the host anyway; the library itself never
    reads device memory back."""
    if windows is None:
        return int(sum(((int(t) + 15) // 16) * ((int(u) + 1 + 7) // 8) for t, u in zip(input_lengths, label_lengths)))
    t_lo, t_hi = (np.asarray(w).astype(np.int64) for w in windows)
    total = 0
    for b, (T, ylen) in enumerate(zip(input_lengths, label_lengths)):
        T, Un = int(T), int(ylen) + 1
        nTb = (T + 15) // 16
        if nTb <= 0:
            continue
        lo, hi = t_lo[b, :Un], t_hi[b, :Un]
        t0 = 16 * np.arange(nTb)[:, None]
        hit = (lo <= hi)[None, :] & (lo[None, :] < t0 + 16) & (hi[None, :] >= t0)          # (t-block, column)
        for u0 in range(0, Un, 8):
            total += int(hit[:, u0:u0 + 8].any(axis=1).sum())
    return total
