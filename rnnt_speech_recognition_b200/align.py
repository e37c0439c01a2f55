"""RNN-T forced alignment: the single most likely path (Viterbi) through the lattice the loss sums over, per utterance.

The path gives the frame at which each label is emitted: the emission delay that FastEmit trains down, word
timestamps, and a filter for badly transcribed training data.  Definition (DESIGN §1, include/rnnt_b200.h), with
T = input_lengths[b], U = label_lengths[b] + 1 and the loss's log-probs lpb(t,u) at blank and lpl(t,u) at labels[b][u]:

    delta(0,0) = 0
    delta(t,u) = max(delta(t-1,u) + lpb(t-1,u), delta(t,u-1) + lpl(t,u-1))     (a predecessor outside the lattice: -inf)
    best_logp  = delta(T-1,U-1) + lpb(T-1,U-1)  <=  -cost

On an exact tie the blank predecessor wins, so among equally scoring paths the one that emits every label earliest is
returned.  ``label_frames[b, j]`` is the frame that emits ``labels[b, j]`` (non-decreasing, in [0, T)), -1 for
j >= label_lengths[b].  A frame index times the encoder's time reduction factor times the feature frame shift is the
emission time in seconds.

Nothing here is differentiable: every call runs under ``torch.no_grad``.  The joint path computes the alignment without
materialising the (B,T,U,V) logits, exactly where ``joint_rnnt_loss`` computes the loss.
"""
import collections
import ctypes as C

import torch

from . import _lib
from .joint import _check, _desc, _f32, _workspace
from .warprnnt import _LOGIT_TYPE, _ptr, _require_cuda, _stream, certify_inputs, workspace_bytes

__all__ = ["Alignment", "rnnt_align", "joint_rnnt_align"]

Alignment = collections.namedtuple("Alignment", ["label_frames", "best_logp", "costs"])
Alignment.__doc__ = """label_frames int32 (B, maxU-1), best_logp float32 (B,), costs float32 (B,) (= the loss's costs)."""


def _outputs(B, U, device):
    return (torch.empty(B, max(U - 1, 0), dtype=torch.int32, device=device),
            torch.empty(B, dtype=torch.float32, device=device), torch.empty(B, dtype=torch.float32, device=device))


@torch.no_grad()
def rnnt_align(acts, labels, act_lens, label_lens, blank=0):
    """Forced alignment on materialised logits ``acts`` (B,T,U,V) -- float32, float16 or bfloat16, softmax inside, as
    ``rnnt_loss`` takes them.  ``labels`` (B,U-1) int32, lengths (B,) int32.  Returns ``Alignment``; its costs equal
    ``rnnt_loss``'s bit for bit."""
    if acts.dtype != torch.float32 and acts.dtype not in _LOGIT_TYPE:
        raise TypeError("acts must be torch.float32, torch.float16 or torch.bfloat16")
    L = _lib.load()
    acts = acts.contiguous()
    certify_inputs(acts, labels, act_lens, label_lens, check_max=False)
    for t, n in ((acts, "acts"), (labels, "labels"), (act_lens, "input_lengths"), (label_lens, "label_lengths")):
        _require_cuda(t, n)
    B, T, U, V = acts.shape
    if labels.shape[1] != U - 1 and not (U == 1 and labels.shape[1] == 0):
        raise ValueError("labels must be (B, U-1)")
    frames, best, costs = _outputs(B, U, acts.device)
    ws = torch.empty(workspace_bytes(T, U, B), dtype=torch.uint8, device=acts.device)
    lab = labels if labels.numel() else torch.zeros(1, dtype=torch.int32, device=acts.device)
    with torch.cuda.device(acts.device):
        opt = _lib.RnntOptions(_lib.RNNT_GPU, 0, _stream().value, int(blank), T, U, True)
        if acts.dtype == torch.float32:
            name = "rnntb200_align_device"
            st = L.rnntb200_align_device(_ptr(acts), _ptr(lab), _ptr(label_lens), _ptr(act_lens), V, B, _ptr(costs),
                                         _ptr(best), _ptr(frames), _ptr(ws), opt)
        else:
            name = "rnntb200_align16"
            st = L.rnntb200_align16(_ptr(acts), _LOGIT_TYPE[acts.dtype], _ptr(lab), _ptr(label_lens), _ptr(act_lens), V,
                                    B, _ptr(costs), _ptr(best), _ptr(frames), _ptr(ws), opt)
    _lib.check(st, name)
    return Alignment(frames, best, costs)


@torch.no_grad()
def joint_rnnt_align(enc_acts, pred_acts, W, b, labels, input_lengths, label_lengths, blank=0, precision="bf16",
                     valid_tiles=None):
    """Forced alignment on the fused joint path: the lattice of logits = tanh(enc_acts[:,:,None] + pred_acts[:,None]) @ W
    + b, never materialised.  Arguments as ``joint_rnnt_loss`` (float16 / bfloat16 inputs are cast to float32; a broken
    ``valid_tiles`` promise gives NaN costs and best_logp and frames of -1).  Returns ``Alignment``; its costs equal
    those of ``joint_rnnt_loss`` with the same precision, bit for bit."""
    L = _lib.load()
    enc, pred, W, b = (_f32(t).contiguous() for t in (enc_acts, pred_acts, W, b))
    labels, input_lengths, label_lengths = (t.contiguous() for t in (labels, input_lengths, label_lengths))
    _check(enc, pred, W, b, labels, input_lengths, label_lengths)
    B, T, H = enc.shape
    U, V = pred.shape[1], W.shape[1]
    lab = labels if labels.numel() else torch.zeros(1, dtype=torch.int32, device=enc.device)
    with torch.cuda.device(enc.device):
        desc = _desc(B, T, U, H, V, blank, precision, False, valid_tiles)
        ws = _workspace(desc, enc.device)
        frames, best, costs = _outputs(B, U, enc.device)
        st = L.rnntb200_joint_align(C.byref(desc), _ptr(enc), _ptr(pred), _ptr(W), _ptr(b), _ptr(lab),
                                    _ptr(label_lengths), _ptr(input_lengths), _ptr(costs), _ptr(best), _ptr(frames),
                                    _ptr(ws))
    _lib.check(st, "rnntb200_joint_align")
    return Alignment(frames, best, costs)
