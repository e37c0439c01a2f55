"""ctypes binding of librnnt_b200.so (C ABI: include/rnnt_b200.h).

The product path FAILS LOUDLY when the CUDA library is missing or was not built: there is no
CPU or eager-PyTorch fallback anywhere behind these entry points.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.environ.get("RNNTB200_LIB") or os.path.join(HERE, "librnnt_b200.so")   # RNNTB200_LIB: A/B another build

RNNT_CPU, RNNT_GPU = 0, 1
FP32_EXACT, BF16_TC = 0, 1
LOGITS_F16, LOGITS_BF16 = 0, 1


class RnntOptions(C.Structure):
    """struct rnntOptions (include/rnnt_b200.h; reference rnnt.h:43-64), passed by value."""
    _fields_ = [("loc", C.c_int), ("num_threads", C.c_uint), ("stream", C.c_void_p), ("blank_label", C.c_int),
                ("maxT", C.c_int), ("maxU", C.c_int), ("batch_first", C.c_bool)]


class JointDesc(C.Structure):
    """rnntb200JointDesc (include/rnnt_b200.h)."""
    _fields_ = [("B", C.c_int), ("maxT", C.c_int), ("maxU", C.c_int), ("H", C.c_int), ("V", C.c_int),
                ("blank_label", C.c_int), ("precision", C.c_int), ("stream", C.c_void_p),
                ("valid_tile_bound", C.c_int), ("keep_activations", C.c_int)]


EXPORTS = ("get_warprnnt_version", "rnntGetStatusString", "get_workspace_size", "compute_rnnt_loss",
           "compute_rnnt_loss_fp64", "rnntb200_loss_device", "rnntb200_loss16_forward", "rnntb200_loss16_backward",
           "rnntb200_loss_device_fastemit", "rnntb200_loss16_backward_fastemit",
           "rnntb200_joint_workspace_size",
           "rnntb200_joint_loss_forward", "rnntb200_joint_loss_backward", "rnntb200_joint_loss_backward_fastemit",
           "rnntb200_loss_device_windowed", "rnntb200_loss16_forward_windowed", "rnntb200_loss16_backward_windowed",
           "rnntb200_joint_loss_forward_windowed", "rnntb200_joint_loss_backward_windowed",
           "rnntb200_align_device", "rnntb200_align16", "rnntb200_joint_align",
           "rnntb200_joint_logits", "rnntb200_joint_step",
           "rnntb200_dense1_forward", "rnntb200_dense1_backward",
           "rnntb200_simple_workspace_size", "rnntb200_simple_loss_forward", "rnntb200_simple_loss_backward",
           "rnntb200_simple_prune_windows",
           "rnntb200_launch_count", "rnntb200_build_info", "rnntb200_set_timing", "rnntb200_get_timing")

_lib = None


def load(build_if_missing=True):
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing and (not os.path.exists(SO) or os.environ.get("RNNTB200_AUTOBUILD") == "1"):
        # The in-tree .so is built by `__graft_entry__.build()` / `python -m rnnt_speech_recognition_b200.build`.
        # It is only compiled here when it is missing (or RNNTB200_AUTOBUILD=1 asks for a staleness check), so
        # that importing the package on a GPU box never spends a minute in nvcc because of snapshot mtimes.
        from . import build as _b
        try:
            if _b.is_stale():
                _b.build()
        except Exception:
            if not os.path.exists(SO):
                raise
    if not os.path.exists(SO):
        raise RuntimeError("librnnt_b200.so is missing: run `python -m rnnt_speech_recognition_b200.build` "
                           "(there is no CPU fallback)")
    L = C.CDLL(SO)
    vp, ci = C.c_void_p, C.c_int
    L.get_warprnnt_version.restype = ci
    L.rnntGetStatusString.restype = C.c_char_p
    L.rnntGetStatusString.argtypes = [ci]
    L.get_workspace_size.argtypes = [ci, ci, ci, C.c_bool, C.POINTER(C.c_size_t), C.c_size_t]
    L.compute_rnnt_loss.argtypes = [vp, vp, vp, vp, vp, ci, ci, vp, vp, RnntOptions]
    L.compute_rnnt_loss_fp64.argtypes = L.compute_rnnt_loss.argtypes
    L.rnntb200_loss_device.argtypes = [vp, vp, vp, vp, vp, vp, ci, ci, vp, vp, RnntOptions]
    L.rnntb200_loss16_forward.argtypes = [vp, ci, vp, vp, vp, ci, ci, vp, vp, RnntOptions]
    L.rnntb200_loss16_backward.argtypes = [vp, ci, vp, vp, vp, vp, ci, ci, vp, vp, RnntOptions]
    L.rnntb200_loss_device_fastemit.argtypes = L.rnntb200_loss_device.argtypes + [C.c_float]
    L.rnntb200_loss16_backward_fastemit.argtypes = L.rnntb200_loss16_backward.argtypes + [C.c_float]
    L.rnntb200_joint_workspace_size.argtypes = [C.POINTER(JointDesc), C.POINTER(C.c_size_t)]
    L.rnntb200_joint_loss_forward.argtypes = [C.POINTER(JointDesc)] + [vp] * 9
    L.rnntb200_joint_loss_backward.argtypes = [C.POINTER(JointDesc)] + [vp] * 13
    L.rnntb200_joint_loss_backward_fastemit.argtypes = L.rnntb200_joint_loss_backward.argtypes + [C.c_float]
    L.rnntb200_loss_device_windowed.argtypes = [vp] * 8 + [ci, ci, vp, vp, RnntOptions, C.c_float]
    L.rnntb200_loss16_forward_windowed.argtypes = [vp, ci] + [vp] * 5 + [ci, ci, vp, vp, RnntOptions]
    L.rnntb200_loss16_backward_windowed.argtypes = [vp, ci] + [vp] * 6 + [ci, ci, vp, vp, RnntOptions, C.c_float]
    L.rnntb200_joint_loss_forward_windowed.argtypes = [C.POINTER(JointDesc)] + [vp] * 11
    L.rnntb200_joint_loss_backward_windowed.argtypes = [C.POINTER(JointDesc)] + [vp] * 15 + [C.c_float]
    L.rnntb200_align_device.argtypes = [vp, vp, vp, vp, ci, ci, vp, vp, vp, vp, RnntOptions]
    L.rnntb200_align16.argtypes = [vp, ci, vp, vp, vp, ci, ci, vp, vp, vp, vp, RnntOptions]
    L.rnntb200_joint_align.argtypes = [C.POINTER(JointDesc)] + [vp] * 11
    L.rnntb200_joint_logits.argtypes = [C.POINTER(JointDesc)] + [vp] * 6
    L.rnntb200_joint_step.argtypes = [vp, C.c_longlong, vp, C.c_longlong, vp, vp, vp, vp, ci, ci, ci, ci, vp, vp, vp, vp]
    L.rnntb200_dense1_forward.argtypes = [vp, C.c_longlong, ci, vp, vp, ci, vp, vp]
    L.rnntb200_dense1_backward.argtypes = [vp, vp, vp, C.c_longlong, ci, ci, vp, vp, vp, vp]
    L.rnntb200_simple_workspace_size.argtypes = [ci, ci, ci, ci, C.POINTER(C.c_size_t)]
    L.rnntb200_simple_loss_forward.argtypes = [vp] * 5 + [ci, ci, vp, vp, RnntOptions]
    L.rnntb200_simple_loss_backward.argtypes = [vp] * 5 + [ci, ci, vp, vp, vp, vp, RnntOptions]
    L.rnntb200_simple_prune_windows.argtypes = [vp, vp, ci, ci, vp, vp, vp, RnntOptions]
    L.rnntb200_launch_count.restype = C.c_ulonglong
    L.rnntb200_build_info.restype = C.c_char_p
    L.rnntb200_set_timing.argtypes = [ci]
    L.rnntb200_set_timing.restype = None
    L.rnntb200_get_timing.argtypes = [ci, C.POINTER(C.c_char_p), C.POINTER(C.c_float)]
    _lib = L
    return L


def fastemit_lambda(value):
    """FastEmit's lambda as the library takes it: a finite float >= 0 (ValueError otherwise)."""
    try:
        lam = float(value)
    except (TypeError, ValueError):
        raise ValueError("fastemit_lambda must be a finite number >= 0, got %r" % (value,)) from None
    if not (0.0 <= lam < float("inf")):          # NaN fails the comparison too
        raise ValueError("fastemit_lambda must be a finite number >= 0, got %r" % (value,))
    return lam


def ptr(t):
    """A tensor's device address as the C ABI takes it (None: NULL)."""
    return C.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    """The current CUDA stream (of the current device: call inside ``with torch.cuda.device(...)``)."""
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(status, what):
    if status != 0:
        raise RuntimeError("%s failed: %s (status %d)" % (what, load().rnntGetStatusString(status).decode(), status))


def launch_count():
    return int(load().rnntb200_launch_count())


def set_timing(on):
    load().rnntb200_set_timing(int(bool(on)))


def get_timings():
    """[(kernel name, milliseconds)] recorded since set_timing(True); synchronise the stream first."""
    L, out, i = load(), [], 0
    name, ms = C.c_char_p(), C.c_float()
    while L.rnntb200_get_timing(i, C.byref(name), C.byref(ms)):
        out.append((name.value.decode(), ms.value))
        i += 1
    return out
