"""CPU-side checks of mixed-precision training: the argument checks of the 16-bit loss entries (no GPU needed, every
call below bails out before touching device memory) and loss scaling in joint_train_step with a pure-torch stub joint,
alone and in a gloo world of 2."""
import ctypes as C
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_dist_gloo import _StubJoint, _batch

RNNT_STATUS_INVALID_VALUE = 2


def test_loss16_argument_checks_without_gpu():
    from rnnt_speech_recognition_b200 import _lib
    L = _lib.load()
    opt = _lib.RnntOptions(_lib.RNNT_GPU, 0, None, 0, 4, 3, True)
    one = C.c_void_p(16)  # never dereferenced
    F16, BF16 = _lib.LOGITS_F16, _lib.LOGITS_BF16
    fwd = lambda acts, lt, lab, ll, il, V, B, costs, ws, o=opt: L.rnntb200_loss16_forward(acts, lt, lab, ll, il, V, B,
                                                                                          costs, ws, o)
    bwd = lambda acts, lt, lab, ll, il, gc, V, B, g, ws, o=opt: L.rnntb200_loss16_backward(acts, lt, lab, ll, il, gc, V, B,
                                                                                           g, ws, o)
    for lt in (F16, BF16):
        assert fwd(None, lt, one, one, one, 5, 1, one, one) == RNNT_STATUS_INVALID_VALUE
        assert fwd(one, lt, None, one, one, 5, 1, one, one) == RNNT_STATUS_INVALID_VALUE
        assert fwd(one, lt, one, None, one, 5, 1, one, one) == RNNT_STATUS_INVALID_VALUE
        assert fwd(one, lt, one, one, None, 5, 1, one, one) == RNNT_STATUS_INVALID_VALUE
        assert fwd(one, lt, one, one, one, 5, 1, None, one) == RNNT_STATUS_INVALID_VALUE
        assert fwd(one, lt, one, one, one, 5, 1, one, None) == RNNT_STATUS_INVALID_VALUE
        assert fwd(one, lt, one, one, one, 0, 1, one, one) == RNNT_STATUS_INVALID_VALUE
        assert fwd(one, lt, one, one, one, 5, 0, one, one) == RNNT_STATUS_INVALID_VALUE
        assert bwd(None, lt, one, one, one, None, 5, 1, one, one) == RNNT_STATUS_INVALID_VALUE
        assert bwd(one, lt, None, one, one, None, 5, 1, one, one) == RNNT_STATUS_INVALID_VALUE
        assert bwd(one, lt, one, one, one, None, 5, 1, None, one) == RNNT_STATUS_INVALID_VALUE
        assert bwd(one, lt, one, one, one, None, 5, 1, one, None) == RNNT_STATUS_INVALID_VALUE
        for bad in (_lib.RnntOptions(_lib.RNNT_GPU, 0, None, 0, 0, 3, True),       # maxT = 0
                    _lib.RnntOptions(_lib.RNNT_GPU, 0, None, 0, 4, 1025, True),    # maxU past the wavefront's 1024
                    _lib.RnntOptions(_lib.RNNT_GPU, 0, None, 5, 4, 3, True),       # blank == V
                    _lib.RnntOptions(_lib.RNNT_GPU, 0, None, -1, 4, 3, True)):
            assert fwd(one, lt, one, one, one, 5, 1, one, one, bad) == RNNT_STATUS_INVALID_VALUE
            assert bwd(one, lt, one, one, one, None, 5, 1, one, one, bad) == RNNT_STATUS_INVALID_VALUE
    for lt in (-1, 2, 7):                                                          # unknown logit type
        assert fwd(one, lt, one, one, one, 5, 1, one, one) == RNNT_STATUS_INVALID_VALUE
        assert bwd(one, lt, one, one, one, None, 5, 1, one, one) == RNNT_STATUS_INVALID_VALUE


B, T, U, P, V = 4, 6, 3, 8, 5


def _steps(joint, enc, pred, lab, sl, ll, scaler, n=3, group=None):
    from rnnt_speech_recognition_b200 import joint_train_step, make_optimizer
    opt = make_optimizer(joint.parameters(), learning_rate=0.1)
    return [joint_train_step(joint, opt, enc, pred, lab, sl, ll, global_batch_size=B, scaler=scaler, group=group).item()
            for _ in range(n)]


def test_scaled_step_matches_unscaled_step():
    """A power-of-two loss scale is exact in both directions: the scaled steps reproduce the unscaled ones."""
    enc, pred, lab, sl, ll = _batch(B, T, U, P)
    ref, scaled = _StubJoint(P, V), _StubJoint(P, V)
    want = _steps(ref, enc, pred, lab, sl, ll, None)
    scaler = torch.amp.GradScaler("cpu", init_scale=2.0 ** 16)
    got = _steps(scaled, enc, pred, lab, sl, ll, scaler)
    assert np.allclose(got, want, rtol=1e-6, atol=0)
    for a, b in zip(scaled.parameters(), ref.parameters()):
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-7)
    assert scaler.get_scale() == 2.0 ** 16                  # no overflow: the scale stays (growth after 2000 steps)


def _scaled_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from rnnt_speech_recognition_b200 import distributed as D
    enc, pred, lab, sl, ll = _batch(B, T, U, P)
    lo, hi = D.shard_bounds(B, world, rank)
    enc = enc[lo:hi].clone()
    if rank == 1:
        enc[0, 0, 0] = float("nan")          # a non-finite loss and gradient on this rank only
    joint = _StubJoint(P, V)
    scaler = torch.amp.GradScaler("cpu", init_scale=2.0 ** 16)
    _steps(joint, enc, pred[lo:hi], lab[lo:hi], sl[lo:hi], ll[lo:hi], scaler, n=1)
    out[rank] = (scaler.get_scale(), joint.kernel_2.detach().clone().numpy(), joint.bias_2.detach().clone().numpy())
    dist.destroy_process_group()


def test_nonfinite_gradient_on_one_rank_skips_the_step_on_every_rank():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with mp.Manager() as m:
        out = m.dict()
        mp.spawn(_scaled_worker, args=(2, port, out), nprocs=2, join=True)
        res = dict(out)
    init = _StubJoint(P, V)
    for r in range(2):
        scale, k2, b2 = res[r]
        assert scale == 2.0 ** 15, (r, scale)                               # both ranks backed off
        assert np.array_equal(k2, init.kernel_2.detach().numpy())           # and skipped the step
        assert np.array_equal(b2, init.bias_2.detach().numpy())
    assert np.array_equal(res[0][1], res[1][1]) and np.array_equal(res[0][2], res[1][2])
