"""Fused joint network + RNN-T loss (the north-star path): torch surface over
``rnntb200_joint_loss_forward/backward`` (include/rnnt_b200.h).

Reference being replaced (file:line under /root/reference):
  model.py:158-166      joint_inp = enc[:,:,None,:] + pred[:,None,:,:]; Dense(tanh); Dense(vocab)
  utils/loss.py:24-36   loss adapter -> warprnnt_tensorflow.rnnt_loss
  run_rnnt.py:269-284   model(...) -> loss_fn(...) -> tape.gradient

``enc_acts`` / ``pred_acts`` are the Dense-1 projections hoisted out of the lattice
(W1^T(f_t+g_u)+b1 = (W1^T f_t + b1) + W1^T g_u, SURVEY 8a2): the (B,T,U,*) tensors of the
reference never exist here, in either direction.
"""
import ctypes as C
import os

import torch

from . import _lib
from .loss import encoder_lengths
from .windows import check_windows, valid_tile_count

__all__ = ["joint_rnnt_loss", "joint_logits", "joint_step", "Joint", "get_fused_loss_fn"]

_PREC = {"fp32": _lib.FP32_EXACT, "bf16": _lib.BF16_TC, _lib.FP32_EXACT: _lib.FP32_EXACT, _lib.BF16_TC: _lib.BF16_TC}

_ptr = _lib.ptr


def _desc(B, T, U, H, V, blank, precision, keep=False, tile_bound=0):
    # (call inside `with torch.cuda.device(...)`: the stream is the CURRENT stream of the tensors' device)
    return _lib.JointDesc(B, T, U, H, V, int(blank), _PREC[precision], _lib.stream().value, int(tile_bound or 0),
                          1 if keep else 0)


def _workspace(desc, device):
    sz = C.c_size_t(0)
    _lib.check(_lib.load().rnntb200_joint_workspace_size(C.byref(desc), C.byref(sz)), "rnntb200_joint_workspace_size")
    return torch.empty(sz.value, dtype=torch.uint8, device=device)


def _f32(t):
    """Mixed-precision inputs (float16 / bfloat16, e.g. under torch.autocast) are cast to float32 at the boundary; the
    kernels then run exactly as on float32 inputs, and autograd returns each gradient in its input's dtype.  Any other
    dtype passes through (and is rejected by the checks)."""
    return t.float() if t is not None and t.dtype in (torch.float16, torch.bfloat16) else t


def _check(enc, pred, W, b, labels, input_lengths, label_lengths):
    for t, n in ((enc, "enc_acts"), (pred, "pred_acts"), (W, "W"), (b, "b")):
        if not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor: rnnt_b200 has no CPU path" % n)
        if t.dtype != torch.float32:
            raise TypeError("%s must be torch.float32" % n)
    for t, n in ((labels, "labels"), (input_lengths, "input_lengths"), (label_lengths, "label_lengths")):
        if t.dtype != torch.int32:
            raise TypeError("%s must be torch.int32" % n)
        if not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor (device-resident lengths/labels, warprnnt_op.cc:88-94)" % n)
    if enc.dim() != 3 or pred.dim() != 3 or W.dim() != 2 or b.dim() != 1:
        raise ValueError("expected enc (B,T,H), pred (B,U,H), W (H,V), b (V)")
    B, T, H = enc.shape
    if pred.shape[0] != B or pred.shape[2] != H or W.shape[0] != H or b.shape[0] != W.shape[1]:
        raise ValueError("inconsistent shapes")
    U = pred.shape[1]
    if labels.dim() != 2 or labels.shape[0] != B or (labels.shape[1] != U - 1 and U > 1):
        raise ValueError("labels must be (B, U-1)")
    if input_lengths.shape != (B,) or label_lengths.shape != (B,):
        raise ValueError("must have a length per example.")


def _joint_setup(enc, pred, W, b, labels, input_lengths, label_lengths, blank, precision, keep, valid_tiles):
    """What the joint loss and alignment calls do before their call: contiguous operands and their checks, a 1-element
    stand-in for labels with no elements (U == 1), the descriptor and its workspace.  Returns the operands in the order
    of the C entries (enc, pred, W, b, labels, label_lengths, input_lengths), the descriptor and the workspace."""
    enc, pred, W, b = (t.contiguous() for t in (enc, pred, W, b))
    labels, input_lengths, label_lengths = (t.contiguous() for t in (labels, input_lengths, label_lengths))
    _check(enc, pred, W, b, labels, input_lengths, label_lengths)
    B, T, H = enc.shape
    U, V = pred.shape[1], W.shape[1]
    lab = labels if labels.numel() else torch.zeros(1, dtype=torch.int32, device=enc.device)
    with torch.cuda.device(enc.device):
        desc = _desc(B, T, U, H, V, blank, precision, keep, valid_tiles)
    return (enc, pred, W, b, lab, label_lengths, input_lengths), desc, _workspace(desc, enc.device)


class _JointRNNT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, enc, pred, W, b, labels, input_lengths, label_lengths, blank, precision, compact, keep=None, valid_tiles=None,
                fastemit_lambda=0.0, t_lo=None, t_hi=None):
        L = _lib.load()
        # a backward will follow: let the forward keep its softmax numerators / tanh outputs in the workspace
        keep = any(ctx.needs_input_grad[:4]) if keep is None else keep
        args, desc, ws = _joint_setup(enc, pred, W, b, labels, input_lengths, label_lengths, blank, precision, keep,
                                      valid_tiles)
        device = args[0].device
        costs = torch.empty(desc.B, dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            st = L.rnntb200_joint_loss_forward_windowed(C.byref(desc), *map(_ptr, args), _ptr(t_lo), _ptr(t_hi), _ptr(costs),
                                                        _ptr(ws))
        _lib.check(st, "rnntb200_joint_loss_forward_windowed")
        ctx.save_for_backward(*args)
        ctx.windows = (t_lo, t_hi)
        ctx.ws, ctx.desc, ctx.fastemit_lambda = ws, desc, fastemit_lambda
        return costs

    @staticmethod
    def backward(ctx, grad_costs):
        L = _lib.load()
        args = ctx.saved_tensors
        g = grad_costs.to(torch.float32).contiguous()
        d_enc, d_pred, dW, db = (torch.empty_like(t) for t in args[:4])
        with torch.cuda.device(args[0].device):
            desc = ctx.desc
            desc.stream = _lib.stream().value          # the forward's descriptor, on the backward's current stream
            st = L.rnntb200_joint_loss_backward_windowed(C.byref(desc), *map(_ptr, args), *map(_ptr, ctx.windows), _ptr(g),
                                                         _ptr(d_enc), _ptr(d_pred), _ptr(dW), _ptr(db), _ptr(ctx.ws),
                                                         ctx.fastemit_lambda)
        _lib.check(st, "rnntb200_joint_loss_backward_windowed")
        ctx.ws = None
        return (d_enc, d_pred, dW, db) + (None,) * 11


def joint_rnnt_loss(enc_acts, pred_acts, W, b, labels, input_lengths, label_lengths, blank=0, precision="bf16",
                    compact=True, keep_activations=None, valid_tiles=None, fastemit_lambda=0.0, windows=None):
    """Per-utterance RNN-T NLL (B,) of logits = tanh(enc_acts[:,:,None]+pred_acts[:,None]) @ W + b,
    differentiable w.r.t. enc_acts, pred_acts, W, b -- without ever materialising (B,T,U,V).
    precision: 'bf16' = the tensor-core path (wgmma, 16-bit operands, fp32 accumulate) or 'fp32' (exact CUDA-core path).
    compact: accepted for compatibility and ignored -- ragged batches are compacted on the device, the library never
    synchronises with the host.
    keep_activations: None = automatically when a gradient is required (the forward then leaves its softmax
    numerators (bf16, 2 bytes per logit) in the workspace and the backward is two fused GEMM kernels);
    False = nothing of size O(B*T*U*V) survives the forward call; the backward re-runs the projection chunk by chunk
    (one more tensor-core pass).
    valid_tiles: optional promise `valid_tile_count(host lengths)` (rnntb200JointDesc.valid_tile_bound): sizes the workspace
    for the batch's valid lattice tiles instead of the padded (T,U) lattice, so that large ragged batches stay one chunk and
    keep their numerators; a broken promise yields NaN costs and a device-side message, never an out-of-bounds write.
    float16 / bfloat16 inputs are cast to float32 first (costs float32, each gradient in its input's dtype).
    fastemit_lambda: FastEmit regularisation (Yu et al. 2021), a finite float >= 0 (ValueError otherwise): the gradient
    of every label-emission log-probability is scaled by (1 + lambda); the costs stay -log p(y|x).  0 = the plain loss,
    bit for bit.
    windows: optional ``(t_lo, t_hi)``, int32 CUDA tensors (B, U): the alignment-restricted loss (windows.py), summed over
    the paths inside the per-column frame windows only; lattice tiles outside them are never computed.  With windows,
    ``valid_tiles`` is ``valid_tile_count(host lengths, windows=host windows)``: the workspace then holds the band only.
    Windows that admit no path give a cost of +inf and zero gradients; full windows are the plain loss, bit for bit."""
    lam = _lib.fastemit_lambda(fastemit_lambda)
    t_lo, t_hi = check_windows(windows, enc_acts.shape[0], pred_acts.shape[1], enc_acts.device)
    return _JointRNNT.apply(_f32(enc_acts), _f32(pred_acts), _f32(W), _f32(b), labels, input_lengths, label_lengths, blank,
                            precision, compact, keep_activations, valid_tiles, lam, t_lo, t_hi)


def joint_logits(enc_acts, pred_acts, W, b):
    """model.py:158-166's literal output: logits (B,T,U,V) float32, materialised (not differentiable;
    use joint_rnnt_loss for training).  For callers that want the reference's tensor itself.  float16 / bfloat16
    inputs are cast to float32; the logits are float32 either way."""
    L = _lib.load()
    enc, pred, W, b = (_f32(t).contiguous() for t in (enc_acts, pred_acts, W, b))
    B, T, H = enc.shape
    U, V = pred.shape[1], W.shape[1]
    with torch.cuda.device(enc.device):
        desc = _desc(B, T, U, H, V, 0, "fp32")
        ws = _workspace(desc, enc.device)
        out = torch.empty(B, T, U, V, dtype=torch.float32, device=enc.device)
        st = L.rnntb200_joint_logits(C.byref(desc), _ptr(enc), _ptr(pred), _ptr(W), _ptr(b), _ptr(out), _ptr(ws))
    _lib.check(st, "rnntb200_joint_logits")
    return out


def joint_step(f, g, K1, b1, K2, b2, want_logits=True, want_best=False):
    """``rnntb200_joint_step``: logits (B,V) of ONE lattice cell per batch row, tanh((f+g) @ K1 + b1) @ K2 + b2, and/or
    its argmax + log-softmax value.  ``f``, ``g``: (B,P) float32 CUDA views whose last dimension is contiguous (row
    strides are passed through, so ``encoded[:, i, :]`` / ``pred_out[:, -1, :]`` are not copied).  Not differentiable
    (inference).  float16 / bfloat16 arguments are cast to float32 (outputs float32).
    Returns (logits | None, best | None, best_logp | None)."""
    L = _lib.load()
    f, g, K1, b1, K2, b2 = (_f32(t) for t in (f, g, K1, b1, K2, b2))
    for t, n in ((f, "f"), (g, "g"), (K2, "K2")):
        if not t.is_cuda or t.dtype != torch.float32:
            raise TypeError("%s must be a float32 CUDA tensor (rnnt_b200 has no CPU path)" % n)
    if f.dim() != 2 or g.shape != f.shape or f.stride(1) != 1 or g.stride(1) != 1:
        raise ValueError("f and g must be (B,P) with a contiguous last dimension")
    B, P = f.shape
    K1c = K1.detach().contiguous() if K1 is not None else None
    K2c = K2.detach().contiguous()
    H, V = K2c.shape
    b1c = b1.detach().contiguous() if b1 is not None else None
    b2c = b2.detach().contiguous() if b2 is not None else None
    with torch.cuda.device(f.device):
        logits = torch.empty(B, V, dtype=torch.float32, device=f.device) if want_logits else None
        best = torch.empty(B, dtype=torch.int32, device=f.device) if want_best else None
        logp = torch.empty(B, dtype=torch.float32, device=f.device) if want_best else None
        st = L.rnntb200_joint_step(_ptr(f.detach()), f.stride(0), _ptr(g.detach()), g.stride(0), _ptr(K1c), _ptr(b1c), _ptr(K2c),
                                   _ptr(b2c), B, P, H, V, _ptr(logits), _ptr(best), _ptr(logp),
                                   _lib.stream())
    _lib.check(st, "rnntb200_joint_step")
    return logits, best, logp


class _Dense1(torch.autograd.Function):
    """Keras Dense-1 of the joint (model.py:162-163) on the UN-broadcast inputs: ``x (..., P) @ K1 (P,H) [+ b1]`` and its three
    gradients through ``rnntb200_dense1_forward / _backward`` (the library's own fp32 kernels; SURVEY 8 f1)."""

    @staticmethod
    def forward(ctx, x, K1, b1):
        L = _lib.load()
        if not x.is_cuda or x.dtype != torch.float32 or K1.dtype != torch.float32:
            raise TypeError("dense1: float32 CUDA tensors required (rnnt_b200 has no CPU path)")
        P, H = K1.shape
        if x.shape[-1] != P:
            raise ValueError("dense1: x (..., %d) against a (%d, %d) kernel" % (x.shape[-1], P, H))
        xc, Kc = x.detach().contiguous(), K1.detach().contiguous()
        bc = b1.detach().contiguous() if b1 is not None else None
        rows = xc.numel() // P
        with torch.cuda.device(x.device):
            out = torch.empty(*x.shape[:-1], H, dtype=torch.float32, device=x.device)
            st = L.rnntb200_dense1_forward(_ptr(xc), rows, P, _ptr(Kc), _ptr(bc), H, _ptr(out),
                                           _lib.stream())
        _lib.check(st, "rnntb200_dense1_forward")
        ctx.save_for_backward(xc, Kc)
        ctx.has_bias = b1 is not None
        return out

    @staticmethod
    def backward(ctx, d_out):
        L = _lib.load()
        xc, Kc = ctx.saved_tensors
        P, H = Kc.shape
        rows = xc.numel() // P
        dA = d_out.contiguous()
        need_x, need_k, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.has_bias and ctx.needs_input_grad[2]
        with torch.cuda.device(xc.device):
            dX = torch.empty_like(xc) if need_x else None
            dK = torch.zeros_like(Kc) if need_k else None          # the entry accumulates
            db = torch.zeros(H, dtype=torch.float32, device=xc.device) if need_b else None
            st = L.rnntb200_dense1_backward(_ptr(xc), _ptr(dA), _ptr(Kc), rows, P, H, _ptr(dX), _ptr(dK), _ptr(db),
                                            _lib.stream())
        _lib.check(st, "rnntb200_dense1_backward")
        return dX, dK, db


def dense1(x, K1, b1=None):
    """``x @ K1 (+ b1)`` through the extension (differentiable in x, K1, b1).  float16 / bfloat16 arguments are cast to
    float32 (output float32, each gradient in its argument's dtype)."""
    return _Dense1.apply(_f32(x), _f32(K1), _f32(b1))


class Joint(torch.nn.Module):
    """The joint network of model.py:158-166 with Keras-layout parameters:
    dense_1 kernel (P,H) + bias (H) with tanh, dense_2 kernel (H,V) + bias (V).

    ``forward(inp_enc, pred_outputs)`` returns the reference's logits tensor (drop-in for the Keras
    model output); ``loss(...)`` runs the fused path where that tensor never exists, with FastEmit regularisation of
    strength ``fastemit_lambda`` (0: none; see ``joint_rnnt_loss``)."""

    def __init__(self, proj_size, joint_net_size, vocab_size, precision="bf16", blank=0, fastemit_lambda=0.0):
        super().__init__()
        self.kernel_1 = torch.nn.Parameter(torch.empty(proj_size, joint_net_size))
        self.bias_1 = torch.nn.Parameter(torch.zeros(joint_net_size))
        self.kernel_2 = torch.nn.Parameter(torch.empty(joint_net_size, vocab_size))
        self.bias_2 = torch.nn.Parameter(torch.zeros(vocab_size))
        torch.nn.init.xavier_uniform_(self.kernel_1)   # Keras Dense default glorot_uniform
        torch.nn.init.xavier_uniform_(self.kernel_2)
        self.precision, self.blank = precision, blank
        self.fastemit_lambda = _lib.fastemit_lambda(fastemit_lambda)

    def hoist(self, inp_enc, pred_outputs):
        """Dense-1 is linear before its tanh, so it is applied to the (B,T,P) and (B,U,P) inputs instead of the (B,T,U,P)
        lattice (SURVEY 8 a2), by the extension's own kernels (`dense1`: rnntb200_dense1_forward / _backward, SURVEY 8 f1)."""
        return dense1(inp_enc, self.kernel_1, self.bias_1), dense1(pred_outputs, self.kernel_1, None)

    def forward(self, inp_enc, pred_outputs):
        enc_acts, pred_acts = self.hoist(inp_enc, pred_outputs)
        return joint_logits(enc_acts, pred_acts, self.kernel_2, self.bias_2)

    def step(self, f, g):
        """Greedy-decode joint, utils/decoding.py:6-18: ``joint(model, f, g)`` adds ``f`` (B,T,P) to the LAST
        prediction-network frame ``g[:, -1, :]`` and returns ``outputs[:, 0, 0, :]`` -- the (B,V) logits of frame 0.
        One launch of the library's decode kernel (both Dense layers fused, fp32)."""
        return joint_step(f[:, 0, :], g[:, -1, :], self.kernel_1, self.bias_1, self.kernel_2, self.bias_2)[0]

    def greedy_step(self, f, g):
        """The decode step of utils/decoding.py:69-78 in one launch: ``preds = log_softmax(joint(model, f, g))``,
        ``predicted_id = argmax(preds)``.  Returns (predicted_id (B,) int32, its log-probability (B,) float32); the
        (B,V) logits are not written at all."""
        _, best, logp = joint_step(f[:, 0, :], g[:, -1, :], self.kernel_1, self.bias_1, self.kernel_2, self.bias_2,
                                   want_logits=False, want_best=True)
        return best, logp

    def loss(self, inp_enc, pred_outputs, labels, input_lengths, label_lengths, windows=None, valid_tiles=None):
        """``windows`` / ``valid_tiles``: the alignment-restricted loss, as in ``joint_rnnt_loss``."""
        enc_acts, pred_acts = self.hoist(inp_enc, pred_outputs)
        return joint_rnnt_loss(enc_acts, pred_acts, self.kernel_2, self.bias_2, labels, input_lengths, label_lengths,
                               self.blank, self.precision, valid_tiles=valid_tiles, fastemit_lambda=self.fastemit_lambda,
                               windows=windows)

    @torch.no_grad()
    def align(self, inp_enc, pred_outputs, labels, input_lengths, label_lengths):
        """Forced alignment on the fused path (``joint_rnnt_align``): the frame at which the most likely path emits each
        label.  Returns ``Alignment(label_frames, best_logp, costs)``; the costs equal ``loss``'s.  FastEmit does not
        change it: lambda touches only gradients."""
        from .align import joint_rnnt_align
        enc_acts, pred_acts = self.hoist(inp_enc, pred_outputs)
        return joint_rnnt_align(enc_acts, pred_acts, self.kernel_2, self.bias_2, labels, input_lengths, label_lengths,
                                self.blank, self.precision)


def get_fused_loss_fn(reduction_factor, joint):
    """utils/loss.get_loss_fn-shaped adapter for the fused path: the returned function takes the joint
    network's INPUTS in place of y_pred (run_rnnt.py:269-273 collapsed into one call)."""
    _lib.load()

    def _loss_fn(y_true, inp_enc, pred_outputs, spec_lengths, label_lengths, windows=None):
        y_true = y_true.to(torch.int32).contiguous()
        enc_lengths = encoder_lengths(spec_lengths, reduction_factor).contiguous()
        kw = {} if windows is None else {"windows": windows}
        return joint.loss(inp_enc, pred_outputs, y_true, enc_lengths, label_lengths.to(torch.int32).contiguous(), **kw)

    return _loss_fn
