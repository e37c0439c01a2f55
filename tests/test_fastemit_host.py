"""CPU checks of FastEmit: the float64 reference (tests/fastemit_ref.py) pinned by central differences of the cost and
by its own internal consistency, and the argument checks of the new C entries and torch keywords (no GPU needed: every
call below is rejected before any device work)."""
import ctypes as C

import numpy as np
import pytest
import torch

import fastemit_ref as fe

LAMBDAS = (0.0, 0.5, 2.0)
RNNT_STATUS_INVALID_VALUE = 2


def _cost(lpb, lpl, T, U):
    """-log p(y|x) of one lattice from its arc log-probs (lpb (T,U), lpl (T,U-1)): an independent float64 forward pass."""
    a = np.full((T, U), -np.inf)
    a[0, 0] = 0.0
    for t in range(T):
        for u in range(U):
            if t == 0 and u == 0:
                continue
            no_emit = a[t - 1, u] + lpb[t - 1, u] if t > 0 else -np.inf
            emit = a[t, u - 1] + lpl[t, u - 1] if u > 0 else -np.inf
            a[t, u] = np.logaddexp(no_emit, emit)
    return -(a[T - 1, U - 1] + lpb[T - 1, U - 1])


def _central_differences(lp, labels, il, ll, blank, h=1e-5):
    """d cost / d arc by central differences, per utterance: (B,T,U) for blank arcs and for label arcs."""
    B, T, U, V = lp.shape
    db, dl = np.zeros((B, T, U)), np.zeros((B, T, U))
    for b in range(B):
        Tb, Ub = int(il[b]), int(ll[b]) + 1
        lpb = lp[b, :Tb, :Ub, blank].copy()
        lpl = np.array([[lp[b, t, u, labels[b, u]] for u in range(Ub - 1)] for t in range(Tb)]).reshape(Tb, Ub - 1)
        for arcs, out in ((lpb, db), (lpl, dl)):
            for idx in np.ndindex(arcs.shape):
                keep = arcs[idx]
                arcs[idx] = keep + h
                cp = _cost(lpb, lpl, Tb, Ub)
                arcs[idx] = keep - h
                cm = _cost(lpb, lpl, Tb, Ub)
                arcs[idx] = keep
                out[b][idx] = (cp - cm) / (2 * h)
    return db, dl


def _case(name):
    rng = np.random.default_rng(CASES.index(name))
    B, T, U, V, blank = dict(ragged=(3, 6, 4, 5, 0), u1=(2, 5, 1, 4, 0), t1=(2, 1, 4, 5, 0), blank3=(2, 5, 4, 6, 3),
                             label_is_blank=(2, 5, 4, 5, 2))[name]
    acts = 1.5 * rng.standard_normal((B, T, U, V))
    cand = [v for v in range(V) if v != blank]
    labels = rng.choice(cand, size=(B, max(U - 1, 1))).astype(np.int32)
    il, ll = np.full(B, T, np.int32), np.full(B, U - 1, np.int32)
    if name == "ragged":
        il, ll = np.array([6, 3, 5], np.int32), np.array([3, 1, 0], np.int32)
    if name == "label_is_blank":
        labels[0, 1] = labels[1, 0] = labels[1, 2] = blank
    return fe.log_softmax(acts), labels, il, ll, blank


CASES = ("ragged", "u1", "t1", "blank3", "label_is_blank")


@pytest.mark.parametrize("lam", LAMBDAS)
@pytest.mark.parametrize("name", CASES)
def test_reference_pinned_by_central_differences(name, lam):
    """Label arcs: (1 + lambda) d cost / d lp_label; blank arcs: d cost / d lp_blank; a label equal to blank gets both."""
    lp, labels, il, ll, blank = _case(name)
    B, T, U, V = lp.shape
    costs, g = fe.logprob_grad(lp, labels, il, ll, blank, lam)
    cd_b, cd_l = _central_differences(lp, labels, il, ll, blank)
    for b in range(B):
        Tb, Ub = int(il[b]), int(ll[b]) + 1
        assert abs(costs[b] - _cost(lp[b, :Tb, :Ub, blank],
                                    np.array([[lp[b, t, u, labels[b, u]] for u in range(Ub - 1)] for t in range(Tb)]).reshape(Tb, Ub - 1),
                                    Tb, Ub)) < 1e-12
        for t in range(T):
            for u in range(U):
                want = np.zeros(V)
                if t < Tb and u < Ub:
                    want[blank] += cd_b[b, t, u]
                    if u < Ub - 1:
                        want[labels[b, u]] += (1 + lam) * cd_l[b, t, u]
                np.testing.assert_allclose(g[b, t, u], want, rtol=1e-6, atol=1e-8, err_msg=str((name, lam, b, t, u)))


@pytest.mark.parametrize("name", CASES)
def test_reference_at_lambda_zero_is_the_oracle(oracle, name):
    lp, labels, il, ll, blank = _case(name)
    c0, g0 = fe.logprob_grad(lp, labels, il, ll, blank, 0.0)
    co, go = oracle.rnnt_cost_and_grad(lp, labels, il, ll, blank)
    assert np.array_equal(c0, co)
    if not (labels[:, :lp.shape[2] - 1] == blank).any():     # the oracle's dense gradient keeps one term per column
        assert np.array_equal(g0, go)
    x = 2.0 * np.random.default_rng(1).standard_normal(lp.shape)
    cx, gx = fe.logits_grad(x, labels, il, ll, blank, 0.0)
    cxo, gxo = oracle.rnnt_logits_grad(x, labels, il, ll, blank)
    np.testing.assert_allclose(cx, cxo, rtol=1e-13)
    np.testing.assert_allclose(gx, gxo, rtol=0, atol=1e-13)


@pytest.mark.parametrize("lam", LAMBDAS)
@pytest.mark.parametrize("name", CASES)
def test_logits_variant_is_the_logprob_variant_through_log_softmax(name, lam):
    _, labels, il, ll, blank = _case(name)
    rng = np.random.default_rng(7)
    B, T, U, V = _case(name)[0].shape
    x = 2.0 * rng.standard_normal((B, T, U, V))
    gs = rng.uniform(0.5, 1.5, B)
    costs, dx = fe.logits_grad(x, labels, il, ll, blank, lam, grad_scale=gs)
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    lp = torch.log_softmax(xt, dim=-1)
    c2, dlp = fe.logprob_grad(lp.detach().numpy(), labels, il, ll, blank, lam)
    assert np.allclose(costs, c2, rtol=1e-14)
    (lp * torch.tensor(dlp * gs[:, None, None, None])).sum().backward()
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=0, atol=1e-14)
    assert np.abs(dx.sum(axis=-1)).max() < 1e-14                  # rows of a logit gradient sum to 0
    for b in range(B):
        assert not dx[b, il[b]:].any() and not dx[b, :, ll[b] + 1:].any()


@pytest.mark.parametrize("lam", LAMBDAS)
def test_joint_variant_is_the_torch_joint_through_the_logits_variant(lam):
    rng = np.random.default_rng(11)
    B, T, U, V, H = 3, 7, 5, 9, 6
    enc, pred = rng.standard_normal((B, T, H)), rng.standard_normal((B, U, H))
    W, bias = rng.standard_normal((H, V)) / np.sqrt(H), 0.1 * rng.standard_normal(V)
    labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
    il, ll = np.array([7, 4, 6], np.int32), np.array([4, 2, 0], np.int32)
    gs = np.array([0.5, 1.0, -0.3])
    o = fe.joint_loss_grad(enc, pred, W, bias, labels, il, ll, 0, gs, lam)
    t = [torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (enc, pred, W, bias)]
    logits = torch.tanh(t[0][:, :, None] + t[1][:, None]) @ t[2] + t[3]
    c, dl = fe.logits_grad(logits.detach().numpy(), labels, il, ll, 0, lam, grad_scale=gs)
    (logits * torch.tensor(dl)).sum().backward()
    np.testing.assert_allclose(o["costs"], c, rtol=1e-13)
    for x, n in zip(t, ("d_enc", "d_pred", "dW", "db")):
        np.testing.assert_allclose(o[n], x.grad.numpy(), rtol=1e-10, atol=1e-13, err_msg=n)
    if lam == 0:
        want = fe._oracle.joint_loss_grad(enc, pred, W, bias, labels, il, ll, 0, grad_scale=gs)
        for n in ("costs", "d_enc", "d_pred", "dW", "db"):
            np.testing.assert_allclose(o[n], want[n], rtol=1e-10, atol=1e-13, err_msg=n)


BAD = (-1e-3, -1.0, float("nan"), float("inf"), float("-inf"))


def test_new_c_entries_reject_bad_lambda_without_gpu():
    from rnnt_speech_recognition_b200 import _lib
    L = _lib.load()
    opt = _lib.RnntOptions(_lib.RNNT_GPU, 0, None, 0, 4, 3, True)
    one = C.c_void_p(16)  # never dereferenced
    d = _lib.JointDesc(2, 4, 3, 64, 128, 0, _lib.BF16_TC, None)
    for lam in BAD:
        assert L.rnntb200_loss_device_fastemit(one, one, one, one, one, None, 5, 1, one, one, opt, lam) == RNNT_STATUS_INVALID_VALUE
        for lt in (_lib.LOGITS_F16, _lib.LOGITS_BF16):
            assert L.rnntb200_loss16_backward_fastemit(one, lt, one, one, one, None, 5, 1, one, one, opt,
                                                       lam) == RNNT_STATUS_INVALID_VALUE
        for prec in (_lib.FP32_EXACT, _lib.BF16_TC):
            d.precision = prec
            assert L.rnntb200_joint_loss_backward_fastemit(C.byref(d), *([one] * 13), lam) == RNNT_STATUS_INVALID_VALUE
    # the usual argument checks still come first at a valid lambda
    assert L.rnntb200_loss_device_fastemit(None, None, one, one, one, None, 5, 1, one, one, opt, 0.5) == RNNT_STATUS_INVALID_VALUE
    assert L.rnntb200_joint_loss_backward_fastemit(C.byref(d), None, *([one] * 12), 0.5) == RNNT_STATUS_INVALID_VALUE


@pytest.mark.parametrize("lam", BAD + ("x", None))
def test_torch_entry_points_reject_bad_lambda(lam):
    import rnnt_speech_recognition_b200 as rb
    acts = torch.zeros(1, 2, 2, 3)
    lab, il, ll = torch.ones(1, 1, dtype=torch.int32), torch.tensor([2], dtype=torch.int32), torch.tensor([1], dtype=torch.int32)
    with pytest.raises(ValueError):
        rb.rnnt_loss(acts, lab, il, ll, fastemit_lambda=lam)
    with pytest.raises(ValueError):
        rb.torch_rnnt_loss(acts, lab, il, ll, fastemit_lambda=lam)
    with pytest.raises(ValueError):
        rb.RNNTLoss(fastemit_lambda=lam)
    with pytest.raises(ValueError):
        rb.get_loss_fn(2, fastemit_lambda=lam)
    with pytest.raises(ValueError):
        rb.joint_rnnt_loss(torch.zeros(1, 2, 4), torch.zeros(1, 2, 4), torch.zeros(4, 3), torch.zeros(3), lab, il, ll,
                           fastemit_lambda=lam)
    with pytest.raises(ValueError):
        rb.Joint(4, 4, 3, fastemit_lambda=lam)


def test_default_lambda_is_zero():
    import inspect
    import rnnt_speech_recognition_b200 as rb
    for f in (rb.rnnt_loss, rb.torch_rnnt_loss, rb.RNNTLoss.__init__, rb.get_loss_fn, rb.joint_rnnt_loss, rb.Joint.__init__):
        assert inspect.signature(f).parameters["fastemit_lambda"].default == 0.0, f
    assert rb.Joint(4, 4, 3).fastemit_lambda == 0.0 and rb.Joint(4, 4, 3, fastemit_lambda=0.01).fastemit_lambda == 0.01
