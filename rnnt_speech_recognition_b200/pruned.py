"""Pruned RNN-T (Kuang, Guo, Kang, Lin, Povey, "Pruned RNN-T for fast, memory-efficient ASR training", Interspeech 2022).

A *trivial joiner* scores lattice cell (t,u) with the logits ``am[b,t,:] + lm[b,u,:]`` (no tanh, no H x V projection per
cell).  Its RNN-T loss, the "simple" loss, is cheap because the log-softmax normaliser factorises into a GEMM over the
vocabulary; it is trained as an auxiliary term, and its arc occupancies choose, per frame, the ``s_range`` label positions
the full joint is evaluated on.  That band is handed to the full joint as per-column frame windows (windows.py), so the
pruned loss is the existing windowed loss::

    simple, windows = simple_rnnt_loss(am_proj(enc), lm_proj(pred), labels, enc_lens, label_lens, s_range=5)
    pruned = joint.loss(enc, pred, labels, enc_lens, label_lens, windows=windows)
    loss = (0.5 * simple + pruned).sum() / B

The caller owns the two ``Linear(., V)`` projections that make ``am`` and ``lm``.  Band policy and C entries: DESIGN §1,
include/rnnt_b200.h (part 3).
"""
import ctypes as C

import torch

from . import _lib
from .joint import _f32

__all__ = ["simple_rnnt_loss"]

_ptr = _lib.ptr


def _check(am, lm, labels, input_lengths, label_lengths):
    for t, n in ((am, "am"), (lm, "lm")):
        if not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor: rnnt_b200 has no CPU path" % n)
        if t.dtype != torch.float32:
            raise TypeError("%s must be float32, float16 or bfloat16" % n)
    for t, n in ((labels, "labels"), (input_lengths, "input_lengths"), (label_lengths, "label_lengths")):
        if t.dtype != torch.int32:
            raise TypeError("%s must be torch.int32" % n)
        if not t.is_cuda or t.device != am.device:
            raise RuntimeError("%s must be a CUDA tensor on the device of am" % n)
    if am.dim() != 3 or lm.dim() != 3 or lm.shape[0] != am.shape[0] or lm.shape[2] != am.shape[2] or lm.device != am.device:
        raise ValueError("expected am (B, T, V) and lm (B, U, V) on one device")
    B, U = am.shape[0], lm.shape[1]
    if labels.dim() != 2 or labels.shape[0] != B or (labels.shape[1] != U - 1 and U > 1):
        raise ValueError("labels must be (B, U-1)")
    if input_lengths.shape != (B,) or label_lengths.shape != (B,):
        raise ValueError("must have a length per example.")


class _SimpleRNNT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, am, lm, labels, input_lengths, label_lengths, blank, s_range):
        L = _lib.load()
        B, T, V = am.shape
        U = lm.shape[1]
        dev = am.device
        lab = labels if labels.numel() else torch.zeros(1, dtype=torch.int32, device=dev)
        sz = C.c_size_t(0)
        _lib.check(L.rnntb200_simple_workspace_size(B, T, U, V, C.byref(sz)), "rnntb200_simple_workspace_size")
        ws = torch.empty(sz.value, dtype=torch.uint8, device=dev)
        costs = torch.empty(B, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            opt = _lib.RnntOptions(_lib.RNNT_GPU, 0, _lib.stream().value, int(blank), T, U, True)
            _lib.check(L.rnntb200_simple_loss_forward(_ptr(am), _ptr(lm), _ptr(lab), _ptr(label_lengths),
                                                      _ptr(input_lengths), V, B, _ptr(costs), _ptr(ws), opt),
                       "rnntb200_simple_loss_forward")
            if s_range is not None:
                t_lo = torch.empty(B, U, dtype=torch.int32, device=dev)
                t_hi = torch.empty(B, U, dtype=torch.int32, device=dev)
                _lib.check(L.rnntb200_simple_prune_windows(_ptr(label_lengths), _ptr(input_lengths), B, s_range,
                                                           _ptr(t_lo), _ptr(t_hi), _ptr(ws), opt),
                           "rnntb200_simple_prune_windows")
        ctx.save_for_backward(am, lm, lab, input_lengths, label_lengths)
        ctx.ws, ctx.blank = ws, int(blank)
        if s_range is None:
            return costs
        ctx.mark_non_differentiable(t_lo, t_hi)
        return costs, t_lo, t_hi

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_costs, *_):
        L = _lib.load()
        am, lm, lab, input_lengths, label_lengths = ctx.saved_tensors
        B, T, V = am.shape
        U = lm.shape[1]
        g = grad_costs.to(torch.float32).contiguous()
        d_am, d_lm = torch.empty_like(am), torch.empty_like(lm)
        with torch.cuda.device(am.device):
            opt = _lib.RnntOptions(_lib.RNNT_GPU, 0, _lib.stream().value, ctx.blank, T, U, True)
            _lib.check(L.rnntb200_simple_loss_backward(_ptr(am), _ptr(lm), _ptr(lab), _ptr(label_lengths),
                                                       _ptr(input_lengths), V, B, _ptr(g), _ptr(d_am), _ptr(d_lm),
                                                       _ptr(ctx.ws), opt),
                       "rnntb200_simple_loss_backward")
        return d_am, d_lm, None, None, None, None, None


def simple_rnnt_loss(am, lm, labels, input_lengths, label_lengths, blank=0, s_range=None):
    """The trivial joiner's RNN-T loss: per-utterance costs (B,) float32 of the logits ``am[:,:,None,:] + lm[:,None,:,:]``
    (softmax inside), without that (B,T,U,V) tensor ever being formed.  ``am`` (B,T,V), ``lm`` (B,U,V) CUDA tensors,
    float32, float16 or bfloat16 (cast to float32 at the boundary; each gradient comes back in its input's dtype), U <= 1024;
    ``labels`` (B,U-1), lengths (B,) int32.  Differentiable in ``am`` and ``lm``; rows past an utterance's lengths get
    exactly zero gradient.
    ``s_range`` (int >= 2): also return the pruning band of this forward as ``windows=(t_lo, t_hi)`` (int32 (B,U), not
    differentiable) for the windowed loss entries: ``(costs, (t_lo, t_hi))``.  The band admits a path iff
    ``(s_range - 1) * T_b >= U_b - 1`` (otherwise the windowed cost is +inf); ``s_range >= U_b`` gives full windows."""
    if s_range is not None:
        if isinstance(s_range, bool) or int(s_range) != s_range or int(s_range) < 2:
            raise ValueError("s_range must be an int >= 2, got %r" % (s_range,))
        s_range = int(s_range)
    am, lm = _f32(am).contiguous(), _f32(lm).contiguous()
    labels, input_lengths, label_lengths = (t.contiguous() for t in (labels, input_lengths, label_lengths))
    _check(am, lm, labels, input_lengths, label_lengths)
    out = _SimpleRNNT.apply(am, lm, labels, input_lengths, label_lengths, blank, s_range)
    if s_range is None:
        return out
    return out[0], (out[1], out[2])
