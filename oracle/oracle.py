"""ctypes front-end of the parity checker (TEST INFRASTRUCTURE, not product code).

Two back-ends, both CPU-only:

* ``liboracle.so``  -- the C restatement in ``oracle/rnnt_oracle.c`` (each C function cites
  the reference file:line it follows).
* ``oracle/_ref/libwarprnnt.so`` -- the UNMODIFIED reference library compiled by ``oracle/Makefile`` from the
  warp-transducer checkout that ``WARP_TRANSDUCER_DIR`` names (when it is set).  Its C ABI is
  ``warp-transducer/include/rnnt.h:16-143``; ``rnntOptions`` is passed by value.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / reference arm may
import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_REF = None


def build(force=False):
    """Compile liboracle.so (and oracle/_ref when WARP_TRANSDUCER_DIR names the reference sources)."""
    so = os.path.join(_HERE, "liboracle.so")
    src = [os.path.join(_HERE, f) for f in ("rnnt_oracle.c", "rnnt_oracle_impl.inc")]
    stale = (not os.path.exists(so)) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in src)
    if force or stale or (_ref_sources() and not os.path.exists(os.path.join(_HERE, "_ref", "libwarprnnt.so"))):
        subprocess.run(["make", "-C", _HERE, "all"], check=True, capture_output=True)
    return so


def _ref_sources():
    d = os.environ.get("WARP_TRANSDUCER_DIR")
    return bool(d) and os.path.isdir(os.path.join(d, "src"))


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def _p(a, ct):
    return None if a is None else a.ctypes.data_as(C.POINTER(ct))


def _f(dtype):
    return ("_f32", C.c_float) if dtype == np.float32 else ("_f64", C.c_double)


def log_softmax(x):
    x = np.ascontiguousarray(x)
    sfx, ct = _f(x.dtype)
    y = np.empty_like(x)
    V = x.shape[-1]
    fn = getattr(lib(), "oracle_log_softmax" + sfx)
    fn.restype = None
    fn(_p(x, ct), _p(y, ct), C.c_long(x.size // V), C.c_int(V))
    return y


def _ints(labels, label_lengths, input_lengths):
    return (np.ascontiguousarray(labels, dtype=np.int32), np.ascontiguousarray(label_lengths, dtype=np.int32),
            np.ascontiguousarray(input_lengths, dtype=np.int32))


def rnnt_cost_and_grad(log_probs, labels, input_lengths, label_lengths, blank=0, want_grad=True):
    """CPU-path semantics: LOG-PROBS in, costs (B,) and grads w.r.t. log-probs out."""
    lp = np.ascontiguousarray(log_probs)
    sfx, ct = _f(lp.dtype)
    B, T, U, V = lp.shape
    labels, label_lengths, input_lengths = _ints(labels, label_lengths, input_lengths)
    costs = np.zeros(B, lp.dtype)
    grads = np.zeros_like(lp) if want_grad else None
    rc = getattr(lib(), "oracle_rnnt_cost_and_grad" + sfx)(
        _p(lp, ct), _p(grads, ct), _p(labels, C.c_int), _p(label_lengths, C.c_int), _p(input_lengths, C.c_int),
        V, B, T, U, blank, _p(costs, ct))
    if rc:
        raise ValueError("oracle status %d" % rc)
    return costs, grads


def rnnt_logits_grad(acts, labels, input_lengths, label_lengths, blank=0, want_grad=True):
    """GPU-op semantics: raw LOGITS in, costs (B,) and grads w.r.t. logits out."""
    x = np.ascontiguousarray(acts)
    sfx, ct = _f(x.dtype)
    B, T, U, V = x.shape
    labels, label_lengths, input_lengths = _ints(labels, label_lengths, input_lengths)
    costs = np.zeros(B, x.dtype)
    grads = np.zeros_like(x) if want_grad else None
    rc = getattr(lib(), "oracle_rnnt_logits_grad" + sfx)(
        _p(x, ct), _p(grads, ct), _p(labels, C.c_int), _p(label_lengths, C.c_int), _p(input_lengths, C.c_int),
        V, B, T, U, blank, _p(costs, ct))
    if rc:
        raise ValueError("oracle status %d" % rc)
    return costs, grads


def joint_forward(enc, pred, W, bias):
    enc = np.ascontiguousarray(enc)
    sfx, ct = _f(enc.dtype)
    pred, W, bias = (np.ascontiguousarray(a, dtype=enc.dtype) for a in (pred, W, bias))
    B, T, H = enc.shape
    U = pred.shape[1]
    V = W.shape[1]
    out = np.empty((B, T, U, V), enc.dtype)
    fn = getattr(lib(), "oracle_joint_forward" + sfx)
    fn.restype = None
    fn(_p(enc, ct), _p(pred, ct), _p(W, ct), _p(bias, ct), B, T, U, H, V, _p(out, ct))
    return out


def joint_step(f, g, K1, b1, K2, b2):
    """Greedy-decode joint of ONE lattice cell per batch row in float64 numpy (utils/decoding.py:6-18 followed by the
    log_softmax + argmax of utils/decoding.py:69-78): returns (logits (B,V), argmax (B,), log-softmax value at the argmax (B,)).
    ``K1 is None``: f, g are already-projected activations."""
    x = np.asarray(f, np.float64) + np.asarray(g, np.float64)
    z = np.tanh(x @ np.asarray(K1, np.float64) + (0.0 if b1 is None else np.asarray(b1, np.float64))) if K1 is not None else np.tanh(x)
    y = z @ np.asarray(K2, np.float64) + (0.0 if b2 is None else np.asarray(b2, np.float64))
    m = y.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(y - m).sum(axis=1))
    best = y.argmax(axis=1)
    return y, best.astype(np.int32), y[np.arange(len(y)), best] - lse


def joint_loss_grad(enc, pred, W, bias, labels, input_lengths, label_lengths, blank=0, grad_scale=None,
                    want_grad=True):
    """Whole hot path: returns dict(costs, d_enc, d_pred, dW, db)."""
    enc = np.ascontiguousarray(enc)
    sfx, ct = _f(enc.dtype)
    pred, W, bias = (np.ascontiguousarray(a, dtype=enc.dtype) for a in (pred, W, bias))
    B, T, H = enc.shape
    U = pred.shape[1]
    V = W.shape[1]
    labels, label_lengths, input_lengths = _ints(labels, label_lengths, input_lengths)
    gs = None if grad_scale is None else np.ascontiguousarray(grad_scale, dtype=enc.dtype)
    costs = np.zeros(B, enc.dtype)
    out = dict(costs=costs)
    if want_grad:
        out.update(d_enc=np.zeros_like(enc), d_pred=np.zeros_like(pred), dW=np.zeros_like(W),
                   db=np.zeros_like(bias))
    rc = getattr(lib(), "oracle_joint_loss_grad" + sfx)(
        _p(enc, ct), _p(pred, ct), _p(W, ct), _p(bias, ct), _p(labels, C.c_int), _p(label_lengths, C.c_int),
        _p(input_lengths, C.c_int), _p(gs, ct), B, T, U, H, V, blank, _p(costs, ct), _p(out.get("d_enc"), ct),
        _p(out.get("d_pred"), ct), _p(out.get("dW"), ct), _p(out.get("db"), ct))
    if rc:
        raise ValueError("oracle status %d" % rc)
    return out


def get_workspace_size(maxT, maxU, minibatch, gpu, dtype_size=4):
    sz = C.c_size_t(0)
    rc = lib().oracle_get_workspace_size(maxT, maxU, minibatch, int(bool(gpu)), C.byref(sz), C.c_size_t(dtype_size))
    return rc, sz.value


# ----------------------------------------------------------------------------------------------
# The real reference library (oracle/_ref/libwarprnnt.so), C ABI of warp-transducer/include/rnnt.h
# ----------------------------------------------------------------------------------------------
class RnntOptions(C.Structure):
    """struct rnntOptions -- rnnt.h:43-64 (32 bytes on x86-64, passed BY VALUE)."""
    _fields_ = [("loc", C.c_int), ("num_threads", C.c_uint), ("stream", C.c_void_p), ("blank_label", C.c_int),
                ("maxT", C.c_int), ("maxU", C.c_int), ("batch_first", C.c_bool)]


def ref_path():
    return os.path.join(_HERE, "_ref", "libwarprnnt.so")


def have_ref():
    if not os.path.exists(ref_path()) and _ref_sources():
        build()
    return os.path.exists(ref_path())


def ref():
    global _REF
    if _REF is None:
        if not have_ref():
            raise FileNotFoundError("oracle/_ref/libwarprnnt.so not built (set WARP_TRANSDUCER_DIR at build time)")
        L = C.CDLL(ref_path())
        L.rnntGetStatusString.restype = C.c_char_p
        L.get_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_bool, C.POINTER(C.c_size_t), C.c_size_t]
        L.compute_rnnt_loss.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p, RnntOptions]
        _REF = L
    return _REF


def ref_cpu_cost_and_grad(log_probs, labels, input_lengths, label_lengths, blank=0, want_grad=True, num_threads=0):
    """compute_rnnt_loss(RNNT_CPU, batch_first) of the real reference: log-probs in,
    costs + grads w.r.t. log-probs out (rnnt_entrypoint.cpp:38-72)."""
    L = ref()
    lp = np.ascontiguousarray(log_probs, dtype=np.float32)
    B, T, U, V = lp.shape
    labels, label_lengths, input_lengths = _ints(labels, label_lengths, input_lengths)
    sz = C.c_size_t(0)
    assert L.get_workspace_size(T, U, B, False, C.byref(sz), 4) == 0
    ws = np.empty(sz.value, np.uint8)
    costs = np.zeros(B, np.float32)
    grads = np.zeros_like(lp) if want_grad else None
    opt = RnntOptions(0, num_threads, None, blank, T, U, True)
    rc = L.compute_rnnt_loss(lp.ctypes.data, None if grads is None else grads.ctypes.data, labels.ctypes.data,
                             label_lengths.ctypes.data, input_lengths.ctypes.data, V, B, costs.ctypes.data,
                             ws.ctypes.data, opt)
    if rc:
        raise ValueError(L.rnntGetStatusString(rc).decode())
    return costs, grads
