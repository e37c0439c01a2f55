"""rnnt_speech_recognition_b200 -- B200-native RNN-T loss hot path (joint forward, alpha/beta
dynamic program, gradients) behind the reference's own loss surface.

Public names follow the reference:
  get_loss_fn            utils/loss.py:12
  rnnt_loss              warprnnt_tensorflow/__init__.py:9   (per-utterance costs)
  torch_rnnt_loss, RNNTLoss, certify_inputs   warprnnt_pytorch/__init__.py:53-140
  Joint, joint_rnnt_loss model.py:158-166 fused with the loss (no (B,T,U,V) tensor)
  joint_train_step       run_rnnt.py:259-296 for the joint (loss/B scaling, one packed all-reduce, SGD step)
and, with no reference analogue, forced alignment: rnnt_align, joint_rnnt_align, Joint.align (align.py), and the
alignment-restricted loss: ``windows=`` on every loss entry, alignment_windows (windows.py), and pruned RNN-T:
simple_rnnt_loss (pruned.py), whose band is such windows.
"""
from .loss import encoder_lengths, get_loss_fn
from .warprnnt import RNNTLoss, certify_inputs, rnnt_loss, torch_rnnt_loss
from .joint import Joint, dense1, get_fused_loss_fn, joint_logits, joint_rnnt_loss, joint_step, valid_tile_count
from .align import Alignment, joint_rnnt_align, rnnt_align
from .windows import alignment_windows
from .pruned import simple_rnnt_loss
from .train import joint_train_step, make_optimizer

__all__ = ["get_loss_fn", "encoder_lengths", "rnnt_loss", "torch_rnnt_loss", "RNNTLoss", "certify_inputs", "Joint",
           "joint_rnnt_loss", "joint_logits", "joint_step", "dense1", "valid_tile_count", "get_fused_loss_fn", "joint_train_step", "make_optimizer",
           "rnnt_align", "joint_rnnt_align", "Alignment", "alignment_windows", "simple_rnnt_loss"]
