"""Argument limits of the decode-step joint and of Dense-1 that the C entries enforce on the host, before any device work
(no GPU needed: the library loads without one).

`rnntb200_joint_step` keeps each CTA's eighth of the logits in shared memory, next to the input row and the hidden row:
joint_step_smem() = 4 (max(P, 256) + H + 256 + ceil(V / 8)) dynamic bytes, plus 96 static bytes (the cluster's
partial maxima, sums and indices).  Beyond 48 KB in all the kernel needs the opt-in, whose ceiling on sm_90 is 227 KB
(232 448 bytes) per block; so V <= 8 (58 088 - max(P, 256) - H - 256), and a larger V is an invalid argument.
"""
import ctypes as C

import pytest

from rnnt_speech_recognition_b200 import _lib

INVALID = 2                          # RNNT_STATUS_INVALID_VALUE
STEP_STATIC_SMEM = 8 * (4 + 4 + 4)   # part_m, part_s, part_i of joint_step_kernel
SMEM_DEFAULT = 48 * 1024 - STEP_STATIC_SMEM
SMEM_MAX = 232448 - STEP_STATIC_SMEM
INT_MAX = 2 ** 31 - 1


def step_smem(P, H, V):
    """joint_step_smem(): the dynamic shared memory of one CTA of the decode step, in bytes."""
    return 4 * (max(P, 256) + H + 256 + -(-V // 8))


def step_max_v(P, H):
    """The largest V whose step_smem fits the opt-in ceiling."""
    return 8 * (SMEM_MAX // 4 - max(P, 256) - H - 256)


# Never dereferenced: every call below must be rejected before it touches one of these.
ADDR = C.c_void_p(0x100000)


def joint_step(P, H, V, K1=ADDR, logits=ADDR, best=ADDR, best_logp=ADDR, B=1):
    return _lib.load().rnntb200_joint_step(ADDR, P, ADDR, P, K1, ADDR, ADDR, ADDR, B, P, H, V, logits, best, best_logp,
                                           None)


def test_step_max_v_is_the_shared_memory_bound():
    for P, H in ((64, 64), (1, 1), (256, 2048), (4096, 2048), (640, 640)):
        v = step_max_v(P, H)
        assert step_smem(P, H, v) <= SMEM_MAX < step_smem(P, H, v + 1)
    assert step_max_v(64, 64) == 460096 and step_max_v(4096, 2048) == 413504


@pytest.mark.parametrize("what,kw", [("P = 4097", dict(P=4097, H=64, V=100)),
                                     ("H = 2049", dict(P=64, H=2049, V=100)),
                                     ("K1 NULL with P != H", dict(P=64, H=32, V=100, K1=None)),
                                     ("no output", dict(P=64, H=64, V=100, logits=None, best=None, best_logp=None)),
                                     ("V past shared memory, P = H = 64", dict(P=64, H=64, V=step_max_v(64, 64) + 1)),
                                     ("V past shared memory, P = 4096, H = 2048",
                                      dict(P=4096, H=2048, V=step_max_v(4096, 2048) + 1)),
                                     ("V = 2^20", dict(P=64, H=64, V=2 ** 20))])
def test_joint_step_rejects(what, kw):
    assert joint_step(**kw) == INVALID, what


def test_dense1_rejects():
    L = _lib.load()
    assert L.rnntb200_dense1_forward(ADDR, INT_MAX + 1, 4, ADDR, ADDR, 4, ADDR, None) == INVALID
    assert L.rnntb200_dense1_backward(ADDR, ADDR, ADDR, INT_MAX + 1, 4, 4, ADDR, ADDR, ADDR, None) == INVALID
    assert L.rnntb200_dense1_backward(ADDR, ADDR, None, 16, 4, 4, ADDR, None, None, None) == INVALID     # dX without K1
    assert L.rnntb200_dense1_backward(None, ADDR, ADDR, 16, 4, 4, None, ADDR, None, None) == INVALID     # dK1 without X
