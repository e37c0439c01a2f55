"""FastEmit reference for the tests (float64, CPU): the defining form on top of the C oracle.

FastEmit (Yu et al., ICASSP 2021) with strength lambda >= 0 changes only the gradient: the gradient of every
label-emission log-probability lp_label(t,u) is multiplied by (1 + lambda), blank log-probabilities keep theirs, and the
costs stay -log p(y|x).  This module builds exactly that, and nothing of the kernels' closed form:

  * `arc_grads`: d cost / d lp_blank(t,u) and d cost / d lp_label(t,u) as two separate arc gradients, read from the
    oracle's log-prob gradient (`oracle.rnnt_cost_and_grad`).  A label equal to blank would share its log-prob column
    with the blank arc, so such labels are moved to one extra column holding a copy of the blank log-probs first.
  * `logprob_grad`: the label arcs' gradients scaled by (1 + lambda), added into a dense (B,T,U,V) log-prob gradient.
  * `logits_grad`: that gradient chained through the log-softmax (softmax inside, as the GPU op's logits).
  * `joint_loss_grad`: the joint network (oracle.joint_forward) with the logits gradient chained through Dense-2,
    tanh and the broadcast add.

At lambda = 0 these are the plain loss's gradients (tests/test_fastemit_host.py pins them to the oracle's own
entries, and the arc gradients to central differences of the cost).
"""
import numpy as np

from oracle import oracle as _oracle


def _labels(labels, B, U):
    lab = np.asarray(labels, np.int32).reshape(B, -1)[:, :max(U - 1, 0)]
    return np.ascontiguousarray(lab)


def arc_grads(log_probs, labels, input_lengths, label_lengths, blank=0):
    """costs (B,), G_blank (B,T,U), G_label (B,T,U): the gradients of the costs w.r.t. each blank arc and each label arc
    (0 where the arc does not exist)."""
    lp = np.ascontiguousarray(log_probs, np.float64)
    B, T, U, V = lp.shape
    lab = _labels(labels, B, U)
    lp_aug = np.concatenate([lp, lp[..., blank:blank + 1]], axis=-1)     # column V: a private copy of the blank log-probs
    lab_aug = np.where(lab == blank, V, lab).astype(np.int32)
    costs, g = _oracle.rnnt_cost_and_grad(lp_aug, lab_aug if lab_aug.size else np.zeros((B, 1), np.int32),
                                          input_lengths, label_lengths, blank)
    g_blank = g[..., blank].copy()
    g_label = np.zeros((B, T, U))
    if U > 1:
        idx = np.broadcast_to(lab_aug[:, None, :, None], (B, T, U - 1, 1))
        g_label[:, :, :U - 1] = np.take_along_axis(g[:, :, :U - 1], idx, axis=-1)[..., 0]
    return costs, g_blank, g_label


def logprob_grad(log_probs, labels, input_lengths, label_lengths, blank=0, fastemit_lambda=0.0):
    """costs (B,) and the dense gradient (B,T,U,V) w.r.t. the log-probs with every label arc's gradient scaled by
    (1 + lambda).  A label equal to blank receives both arcs' terms in its column."""
    lp = np.asarray(log_probs, np.float64)
    B, T, U, V = lp.shape
    costs, gb, gl = arc_grads(lp, labels, input_lengths, label_lengths, blank)
    grad = np.zeros((B, T, U, V))
    grad[..., blank] = gb
    if U > 1:
        lab = _labels(labels, B, U)
        gl_dense = np.zeros((B, T, U - 1, V))
        np.put_along_axis(gl_dense, np.broadcast_to(lab[:, None, :, None], (B, T, U - 1, 1)),
                          ((1.0 + fastemit_lambda) * gl[:, :, :U - 1])[..., None], axis=-1)
        grad[:, :, :U - 1] += gl_dense
    return costs, grad


def log_softmax(x):
    x = np.asarray(x, np.float64)
    m = x.max(axis=-1, keepdims=True)
    return x - (m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True)))


def logits_grad(acts, labels, input_lengths, label_lengths, blank=0, fastemit_lambda=0.0, grad_scale=None):
    """GPU-op semantics: raw logits in (softmax inside), costs (B,) and the gradient w.r.t. the logits out, times
    grad_scale[b] when given.  Padded cells are 0."""
    lp = log_softmax(acts)
    costs, dlp = logprob_grad(lp, labels, input_lengths, label_lengths, blank, fastemit_lambda)
    dx = dlp - np.exp(lp) * dlp.sum(axis=-1, keepdims=True)
    if grad_scale is not None:
        dx *= np.asarray(grad_scale, np.float64)[:, None, None, None]
    return costs, dx


def joint_loss_grad(enc, pred, W, bias, labels, input_lengths, label_lengths, blank=0, grad_scale=None,
                    fastemit_lambda=0.0):
    """Whole fused path in float64: dict(costs, d_enc, d_pred, dW, db), as oracle.joint_loss_grad."""
    enc, pred, W, bias = (np.asarray(a, np.float64) for a in (enc, pred, W, bias))
    logits = _oracle.joint_forward(enc, pred, W, bias)
    costs, dl = logits_grad(logits, labels, input_lengths, label_lengths, blank, fastemit_lambda, grad_scale)
    z = np.tanh(enc[:, :, None, :] + pred[:, None, :, :])
    dpre = (dl @ W.T) * (1.0 - z * z)
    return dict(costs=costs, d_enc=dpre.sum(axis=2), d_pred=dpre.sum(axis=1),
                dW=np.einsum("btuh,btuv->hv", z, dl), db=dl.sum(axis=(0, 1, 2)))
