"""Training-step shim around the hot path (SURVEY 8f rank 3): what run_rnnt.py:259-296 does around the loss,
restated on torch for the part of the model this package owns -- the joint network -- so that a
run_rnnt.py-equivalent loop can run on the fused path.  The encoder / prediction networks stay the caller's:
their outputs come in as tensors and receive their gradients through autograd as usual.

  reference                                            here
  loss_fn(labels, model(...), spec_len, label_len)     joint.loss(...) via get_fused_loss_fn      run_rnnt.py:269-273
  loss = reduce_sum(rnnt_loss) * (1 / batch_size)      costs.sum() / global_batch_size            run_rnnt.py:278
  tape.gradient + MirroredStrategy all-reduce          backward + ONE packed all-reduce           run_rnnt.py:284-288
  strategy.reduce(MEAN, loss)                          same buffer carries the loss sum           run_rnnt.py:292-296
  optimizer.apply_gradients                            optimizer.step()                           run_rnnt.py:288
"""
import torch

from .distributed import allreduce_packed_
from .joint import get_fused_loss_fn


def make_optimizer(params, learning_rate=1e-4, momentum=0.9):
    """The reference trains with plain SGD + momentum 0.9 (run_rnnt.py:483-484)."""
    return torch.optim.SGD(params, lr=learning_rate, momentum=momentum)


def joint_train_step(joint, optimizer, inp_enc, pred_outputs, labels, spec_lengths, label_lengths, global_batch_size,
                     reduction_factor=2, group=None, scaler=None):
    """One optimisation step of `joint` on this rank's shard of the batch.

    inp_enc (B_local,T,P), pred_outputs (B_local,U,P): encoder / prediction-network outputs (may require grad: their
    .grad is filled for the caller's networks); labels (B_local,U-1); spec_lengths, label_lengths (B_local).
    Returns the mean per-utterance loss over the GLOBAL batch (a 0-dim tensor, identical on every rank).
    Cross-rank traffic: one all-reduce of [sum of costs | gradient of every joint parameter].

    scaler: optional torch.amp.GradScaler, the counterpart of the reference's LossScaleOptimizer(loss_scale='dynamic')
    under --fp16_run (run_rnnt.py:486-488).  The scaled loss is back-propagated, the joint's gradients are all-reduced
    while still scaled, and only then unscaled by scaler.step(optimizer): a non-finite gradient on any rank reaches
    every rank, so all ranks skip the step together and scaler.update() keeps their scales equal.  The gradients that
    reach inp_enc / pred_outputs (and the caller's networks) are scaled as well: scaler.step unscales every parameter
    of `optimizer`, so an optimizer that also holds those networks' parameters steps them consistently (their
    gradients are not part of the all-reduce).  The returned loss is unscaled."""
    loss_fn = get_fused_loss_fn(reduction_factor, joint)
    optimizer.zero_grad(set_to_none=True)
    costs = loss_fn(labels, inp_enc, pred_outputs, spec_lengths, label_lengths)        # (B_local,)
    loss = costs.sum() / float(global_batch_size)                                       # run_rnnt.py:278
    if scaler is None:
        loss.backward()
    else:
        scaler.scale(loss).backward()
    params = [p for p in joint.parameters() if p.grad is not None]
    loss_sum = costs.detach().sum().reshape(1)
    allreduce_packed_([loss_sum] + [p.grad for p in params], group=group)
    if scaler is None:
        optimizer.step()
    else:
        scaler.step(optimizer)
        scaler.update()
    return loss_sum[0] / float(global_batch_size)
