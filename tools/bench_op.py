"""Materialised-logits op (compute_rnnt_loss drop-in) on one H100: this library vs the reference's own SIMT CUDA
kernels (warp-transducer compiled unmodified for sm_90 into oracle/_ref/libwarprnnt_gpu.so).

  python tools/bench_op.py [B T U V]      default BASELINE C2 (16 256 64 256) and a larger (32 512 128 1024) case

Reports ms per call (loss + gradients w.r.t. logits), achieved GB/s on the algorithmic bytes of SURVEY 8(d)
(3*N*V*4 + 24*N) and agreement of the two results.  Secondary baseline only -- the headline bench is bench.py.
"""
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rnnt_speech_recognition_b200 import _lib  # noqa: E402


def run_lib(L, fn_name, x, g, lab, il, ll, ws, costs_host, opt_cls, iters=10):
    B, T, U, V = x.shape
    opt = opt_cls(1, 0, torch.cuda.current_stream().cuda_stream, 0, T, U, True)
    fn = getattr(L, fn_name)
    fn.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p, opt_cls]
    call = lambda: fn(x.data_ptr(), g.data_ptr(), lab.data_ptr(), ll.data_ptr(), il.data_ptr(), V, B,
                      costs_host.ctypes.data, ws.data_ptr(), opt)
    for _ in range(3):
        assert call() == 0
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        call()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    shapes = [tuple(int(v) for v in sys.argv[1:5])] if len(sys.argv) >= 5 else [(16, 256, 64, 256), (32, 512, 128, 1024)]
    for res in run_shapes(shapes):
        print(json.dumps(res))


def run_shapes(shapes):
    import numpy as np
    L = _lib.load()
    ref_path = os.path.join(ROOT, "oracle", "_ref", "libwarprnnt_gpu.so")
    R = C.CDLL(ref_path) if os.path.exists(ref_path) else None
    out = []
    for (B, T, U, V) in shapes:
        torch.manual_seed(0)
        x = torch.randn(B, T, U, V, device="cuda")
        lab = torch.randint(1, V, (B, U - 1), dtype=torch.int32, device="cuda")
        il = torch.full((B,), T, dtype=torch.int32, device="cuda")
        ll = torch.full((B,), U - 1, dtype=torch.int32, device="cuda")
        N = B * T * U
        byts = 3.0 * N * V * 4 + 24.0 * N
        res = {"shape": [B, T, U, V], "algorithmic_bytes": byts}
        sz = C.c_size_t(0)
        L.get_workspace_size(T, U, B, True, C.byref(sz), 4)
        ws = torch.empty(sz.value, dtype=torch.uint8, device="cuda")
        g1 = torch.empty_like(x)
        c1 = np.zeros(B, np.float32)
        ms = run_lib(L, "compute_rnnt_loss", x, g1, lab, il, ll, ws, c1, _lib.RnntOptions)
        res["rnnt_b200"] = {"ms": ms, "GBps": byts / ms / 1e6}
        if R is not None:
            R.get_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_bool, C.POINTER(C.c_size_t), C.c_size_t]
            R.get_workspace_size(T, U, B, True, C.byref(sz), 4)
            ws2 = torch.empty(sz.value, dtype=torch.uint8, device="cuda")
            g2 = torch.empty_like(x)
            c2 = np.zeros(B, np.float32)
            ms2 = run_lib(R, "compute_rnnt_loss", x, g2, lab, il, ll, ws2, c2, _lib.RnntOptions)
            res["reference_simt_sm90"] = {"ms": ms2, "GBps": byts / ms2 / 1e6}
            res["max_abs_grad_diff"] = (g1 - g2).abs().max().item()
            res["max_rel_cost_diff"] = float(np.abs(c1 - c2).max() / np.abs(c2).max())
            res["speedup"] = ms2 / ms
        out.append(res)
        del x, g1, ws
        torch.cuda.empty_cache()
    return out


if __name__ == "__main__":
    main()
