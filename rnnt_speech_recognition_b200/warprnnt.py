"""RNN-T loss op on materialised logits -- the reference's op-level surface on torch tensors.

Mirrors, name for name:
  * ``warprnnt_tensorflow.rnnt_loss(acts, labels, input_lengths, label_lengths, blank_label=0)``
    (warp-transducer/tensorflow_binding/warprnnt_tensorflow/__init__.py:9-42): per-utterance costs
    ``(B,)``, differentiable w.r.t. ``acts`` with gradient ``grad_loss[:,None,None,None] * grads``.
  * ``warprnnt_pytorch.rnnt_loss / RNNTLoss`` with reductions and ``certify_inputs``
    (warp-transducer/pytorch_binding/warprnnt_pytorch/__init__.py:10-140) -> ``torch_rnnt_loss``,
    ``RNNTLoss``.

Differences from the reference bindings, all deliberate:
  * costs stay on the device (the reference copies them to host and synchronises the stream
    every call, gpu_rnnt.h:209-213; the torch binding builds a CPU tensor, __init__.py:27);
  * CUDA tensors only: the reference's CPU branch is not reproduced (no CPU fallback);
  * gradients of padded cells are written by the gradient kernel itself (no memset pass);
  * float16 / bfloat16 logits are accepted natively (the reference's op is float32-only): fp32 arithmetic, costs
    float32, gradients formed in the backward pass in the logits' dtype with the upstream gradient folded in;
  * ``fastemit_lambda`` (FastEmit, Yu et al. 2021; default 0 = the plain loss): the gradient of every label-emission
    log-probability is scaled by (1 + lambda).  Costs stay -log p(y|x), not (1 + lambda) times it, so loss curves
    compare across lambda.
"""
import ctypes as C

import torch

from . import _lib
from .windows import check_windows

__all__ = ["rnnt_loss", "torch_rnnt_loss", "RNNTLoss", "certify_inputs"]

_ptr = _lib.ptr


def check_type(var, t, name):
    if var.dtype is not t:
        raise TypeError("{} must be {}".format(name, t))


def check_contiguous(var, name):
    if not var.is_contiguous():
        raise ValueError("{} must be contiguous".format(name))


def check_dim(var, dim, name):
    if len(var.shape) != dim:
        raise ValueError("{} must be {}D".format(name, dim))


def certify_inputs(log_probs, labels, lengths, label_lengths, check_max=True):
    """Same checks, messages and exception types as warprnnt_pytorch/__init__.py:115-140.
    ``check_max=False`` skips the two device-synchronising max() comparisons (used by the
    TF-flavoured entry, whose op only checks ranks: warprnnt_op.cc:51-86)."""
    check_type(labels, torch.int32, "labels")
    check_type(label_lengths, torch.int32, "label_lengths")
    check_type(lengths, torch.int32, "lengths")
    check_contiguous(log_probs, "log_probs")
    check_contiguous(labels, "labels")
    check_contiguous(label_lengths, "label_lengths")
    check_contiguous(lengths, "lengths")
    if lengths.shape[0] != log_probs.shape[0]:
        raise ValueError("must have a length per example.")
    if label_lengths.shape[0] != log_probs.shape[0]:
        raise ValueError("must have a label length per example.")
    check_dim(log_probs, 4, "log_probs")
    check_dim(labels, 2, "labels")
    check_dim(lengths, 1, "lenghts")
    check_dim(label_lengths, 1, "label_lenghts")
    if check_max:
        max_T = torch.max(lengths)
        max_U = torch.max(label_lengths)
        T, U = log_probs.shape[1:3]
        if T != max_T:
            raise ValueError("Input length mismatch")
        if U != max_U + 1:
            raise ValueError("Output length mismatch")


def workspace_bytes(maxT, maxU, B, dtype_size=4):
    sz = C.c_size_t(0)
    _lib.check(_lib.load().get_workspace_size(maxT, maxU, B, True, C.byref(sz), dtype_size), "get_workspace_size")
    return sz.value


def _prepare(acts, labels, act_lens, label_lens, float32_only=False):
    """The checks and buffers of every call on materialised logits: all tensors on the device, (for the float32-only op,
    warprnnt_op.cc:15) float32 logits, labels (B, U-1); then the loss workspace, and a 1-element stand-in for labels
    with no elements (U == 1).  Returns (B, T, U, V), workspace, labels."""
    for t, n in ((acts, "acts"), (labels, "labels"), (act_lens, "input_lengths"), (label_lens, "label_lengths")):
        if not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor: rnnt_b200 has no CPU path (no fallback by design)" % n)
    if float32_only and acts.dtype != torch.float32:
        raise TypeError("acts must be torch.float32")
    B, T, U, V = acts.shape
    if labels.shape[1] != U - 1 and not (U == 1 and labels.shape[1] == 0):
        raise ValueError("labels must be (B, U-1)")
    ws = torch.empty(workspace_bytes(T, U, B), dtype=torch.uint8, device=acts.device)
    lab = labels if labels.numel() else torch.zeros(1, dtype=torch.int32, device=acts.device)
    return (B, T, U, V), ws, lab


def _options(blank, T, U):
    # (call inside `with torch.cuda.device(...)`: the stream must be the current stream OF THE TENSORS' DEVICE)
    return _lib.RnntOptions(_lib.RNNT_GPU, 0, _lib.stream().value, int(blank), T, U, True)


class _RNNTOp(torch.autograd.Function):
    """WarpRNNT op + _RNNTLossGrad: gradients are computed eagerly in forward and cached, exactly
    as both reference bindings do (warprnnt_op.cc:100-137, warprnnt_pytorch/__init__.py:24-42)."""

    @staticmethod
    def forward(ctx, acts, labels, act_lens, label_lens, blank, fastemit_lambda=0.0, t_lo=None, t_hi=None):
        L = _lib.load()
        (B, T, U, V), ws, lab = _prepare(acts, labels, act_lens, label_lens, float32_only=True)
        grads = torch.empty_like(acts) if acts.requires_grad else None
        costs = torch.empty(B, dtype=torch.float32, device=acts.device)
        with torch.cuda.device(acts.device):
            st = L.rnntb200_loss_device_windowed(_ptr(acts), _ptr(grads), _ptr(lab), _ptr(label_lens), _ptr(act_lens),
                                                 None, _ptr(t_lo), _ptr(t_hi), V, B, _ptr(costs), _ptr(ws),
                                                 _options(blank, T, U), fastemit_lambda)
        _lib.check(st, "rnntb200_loss_device_windowed")
        ctx.grads = grads
        return costs

    @staticmethod
    def backward(ctx, grad_costs):
        g = ctx.grads
        ctx.grads = None
        return (g.mul_(grad_costs.view(-1, 1, 1, 1).to(g)),) + (None,) * 7


_LOGIT_TYPE = {torch.float16: _lib.LOGITS_F16, torch.bfloat16: _lib.LOGITS_BF16}


class _RNNTOp16(torch.autograd.Function):
    """The op on float16 / bfloat16 logits (mixed-precision training).  The forward computes costs only and keeps the
    fp32 workspace; the backward forms the 16-bit gradient in one pass with ``grad_costs`` multiplied in before its
    single rounding, so a loss-scaled fp16 gradient does not underflow and no fp32 (B,T,U,V) tensor ever exists."""

    @staticmethod
    def forward(ctx, acts, labels, act_lens, label_lens, blank, fastemit_lambda=0.0, t_lo=None, t_hi=None):
        L = _lib.load()
        (B, T, U, V), ws, lab = _prepare(acts, labels, act_lens, label_lens)
        costs = torch.empty(B, dtype=torch.float32, device=acts.device)
        with torch.cuda.device(acts.device):
            st = L.rnntb200_loss16_forward_windowed(_ptr(acts), _LOGIT_TYPE[acts.dtype], _ptr(lab), _ptr(label_lens),
                                                    _ptr(act_lens), _ptr(t_lo), _ptr(t_hi), V, B, _ptr(costs), _ptr(ws),
                                                    _options(blank, T, U))
        _lib.check(st, "rnntb200_loss16_forward_windowed")
        if acts.requires_grad:
            ctx.windows = (t_lo, t_hi)
            ctx.save_for_backward(acts, lab, act_lens, label_lens)
            ctx.ws, ctx.blank, ctx.fastemit_lambda = ws, int(blank), fastemit_lambda
        return costs

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_costs):
        L = _lib.load()
        acts, lab, act_lens, label_lens = ctx.saved_tensors
        B, T, U, V = acts.shape
        g = grad_costs.to(torch.float32).contiguous()
        grads = torch.empty_like(acts)
        with torch.cuda.device(acts.device):
            st = L.rnntb200_loss16_backward_windowed(_ptr(acts), _LOGIT_TYPE[acts.dtype], _ptr(lab), _ptr(label_lens),
                                                     _ptr(act_lens), *map(_ptr, ctx.windows), _ptr(g), V, B, _ptr(grads),
                                                     _ptr(ctx.ws), _options(ctx.blank, T, U), ctx.fastemit_lambda)
        _lib.check(st, "rnntb200_loss16_backward_windowed")
        ctx.ws = None
        return (grads,) + (None,) * 7


def _op(acts):
    """float16 / bfloat16 logits take the native 16-bit op; everything else the float32 op (which rejects other types)."""
    return _RNNTOp16 if acts.dtype in _LOGIT_TYPE else _RNNTOp


def rnnt_loss(acts, labels, input_lengths, label_lengths, blank_label=0, fastemit_lambda=0.0, windows=None):
    """TF-binding signature (warprnnt_tensorflow/__init__.py:9): per-utterance costs (B,).
    ``acts`` are raw logits (B,T,U,V) float32, float16 or bfloat16 -- the softmax is performed inside, as the
    reference's GPU op does; costs are float32 and ``acts.grad`` has ``acts.dtype``.  ``labels`` (B,U-1) int32 zero
    padded; lengths (B,) int32.  ``fastemit_lambda`` >= 0 (finite; ValueError otherwise): FastEmit regularisation of
    the gradient, costs unchanged.  ``windows``: optional ``(t_lo, t_hi)`` int32 CUDA tensors (B,U), the
    alignment-restricted loss (windows.py): only paths inside the per-column frame windows count, the gradients of cells
    outside them are exactly 0 and their logits are not read; windows that admit no path give a cost of +inf."""
    lam = _lib.fastemit_lambda(fastemit_lambda)
    acts = acts.contiguous()
    certify_inputs(acts, labels, input_lengths, label_lengths, check_max=False)
    t_lo, t_hi = check_windows(windows, acts.shape[0], acts.shape[2], acts.device)
    return _op(acts).apply(acts, labels, input_lengths, label_lengths, blank_label, lam, t_lo, t_hi)


def torch_rnnt_loss(acts, labels, act_lens, label_lens, blank=0, reduction="mean", fastemit_lambda=0.0, windows=None):
    """warprnnt_pytorch.rnnt_loss (pytorch_binding/warprnnt_pytorch/__init__.py:53-70):
    reduction in {'none','sum','mean'}; 'mean' divides the summed cost by the batch size.  ``acts`` float32, float16
    or bfloat16 (costs float32 either way).  ``fastemit_lambda``, ``windows``: as in ``rnnt_loss``."""
    lam = _lib.fastemit_lambda(fastemit_lambda)
    certify_inputs(acts, labels, act_lens, label_lens, check_max=True)
    t_lo, t_hi = check_windows(windows, acts.shape[0], acts.shape[2], acts.device)
    costs = _op(acts).apply(acts, labels, act_lens, label_lens, blank, lam, t_lo, t_hi)
    if reduction in ("sum", "mean"):
        costs = costs.sum().unsqueeze(-1)
        if reduction == "mean":
            costs = costs / acts.size(0)
    elif reduction != "none":
        raise ValueError("reduction must be 'none', 'sum' or 'mean'")
    return costs


class RNNTLoss(torch.nn.Module):
    """warprnnt_pytorch.RNNTLoss (pytorch_binding/warprnnt_pytorch/__init__.py:73-100)."""

    def __init__(self, blank=0, reduction="mean", fastemit_lambda=0.0):
        super().__init__()
        self.blank = blank
        self.reduction = reduction
        self.fastemit_lambda = _lib.fastemit_lambda(fastemit_lambda)

    def forward(self, acts, labels, act_lens, label_lens, windows=None):
        return torch_rnnt_loss(acts, labels, act_lens, label_lens, self.blank, self.reduction, self.fastemit_lambda,
                               windows)
