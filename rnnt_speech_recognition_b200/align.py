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
from ._lib import ptr as _ptr
from .joint import _f32, _joint_setup
from .warprnnt import _LOGIT_TYPE, _options, _prepare, certify_inputs

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
    (B, T, U, V), ws, lab = _prepare(acts, labels, act_lens, label_lens)
    frames, best, costs = _outputs(B, U, acts.device)
    with torch.cuda.device(acts.device):
        opt = _options(blank, T, U)
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
    args, desc, ws = _joint_setup(_f32(enc_acts), _f32(pred_acts), _f32(W), _f32(b), labels, input_lengths, label_lengths,
                                  blank, precision, False, valid_tiles)
    device = args[0].device
    frames, best, costs = _outputs(desc.B, desc.maxU, device)
    with torch.cuda.device(device):
        st = L.rnntb200_joint_align(C.byref(desc), *map(_ptr, args), _ptr(costs), _ptr(best), _ptr(frames), _ptr(ws))
    _lib.check(st, "rnntb200_joint_align")
    return Alignment(frames, best, costs)
