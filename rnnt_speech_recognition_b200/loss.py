"""Loss adapter -- torch mirror of the reference's ``utils/loss.py`` (get_loss_fn, :12-38).

Same name, argument order and semantics; what changes is what sits underneath:
``rnnt_loss`` is the B200 CUDA op of this package instead of warp-transducer, and the silent
``_fallback_loss`` of utils/loss.py:14-22 (returns y_pred when the binding is missing) is
deliberately NOT reproduced: a missing CUDA library raises at get_loss_fn() time.
"""
import torch

from . import _lib
from .warprnnt import rnnt_loss


def encoder_lengths(spec_lengths, reduction_factor):
    """T_b = ceil(spec_len_b / reduction_factor) as int32 -- utils/loss.py:31-33
    (tf.math.ceil of a true division, i.e. computed in floating point)."""
    return torch.ceil(spec_lengths.to(torch.float64) / reduction_factor).to(torch.int32)


def get_loss_fn(reduction_factor, fastemit_lambda=0.0):
    """``fastemit_lambda`` >= 0: FastEmit regularisation of the gradient (``rnnt_loss``); the costs are unchanged."""
    lam = _lib.fastemit_lambda(fastemit_lambda)
    _lib.load()  # fail loudly here, not with a fallback later

    def _loss_fn(y_true, y_pred, spec_lengths, label_lengths, windows=None):
        """y_true (B,U-1) int labels; y_pred (B,T,U,V) float32 / float16 / bfloat16 logits; spec_lengths (B,) pre-reduction
        frame counts; label_lengths (B,) -> per-utterance NLL (B,).  utils/loss.py:24-36.  windows: optional (t_lo, t_hi) of
        the alignment-restricted loss (``rnnt_loss``)."""
        y_true = y_true.to(torch.int32).contiguous()                 # tf.cast(y_true, tf.int32)
        # GPU build: no explicit log_softmax (utils/loss.py:29-30 applies it only on CPU builds)
        enc_lengths = encoder_lengths(spec_lengths, reduction_factor).contiguous()
        return rnnt_loss(y_pred, y_true, enc_lengths, label_lengths.to(torch.int32).contiguous(), fastemit_lambda=lam,
                         windows=windows)

    return _loss_fn
