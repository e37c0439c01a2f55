"""Cost of the alignment-restricted loss on one GPU: `joint_rnnt_loss` with windows of several widths around each
utterance's own alignment, alternating with the call without windows in one process.

  python tools/bench_windows.py [rounds]       default 3 rounds

Workloads (forward + backward through the torch surface, tensor-core path, CUDA events around `iters` calls after a
warm-up of the same shape):
  * BASELINE C3 (B=32 T=512 U=128 V=1024 H=640);
  * a C5-shaped ragged batch (B=32, T up to 1200, U up to 160, same V and H), `valid_tiles` given in every variant.
Windows: `alignment_windows(joint_rnnt_align(same inputs).label_frames, ..., left, right)` for (left, right) in full,
(64,64), (16,16), (4,4); "full" covers the lattice (bit-identical to no windows).  Each round times none, then every
width, then none again, so drift shows as spread between the two unwindowed runs.  One JSON line per timing, then per
variant a summary: valid tiles, workspace bytes, median and spread of the step time, and the per-kernel times of one
instrumented step (`rnntb200_set_timing`, outside the timed region).  Every line carries the card's name and power
limit read in the same run.
"""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rnnt_speech_recognition_b200 as rb  # noqa: E402
from rnnt_speech_recognition_b200 import _lib  # noqa: E402
from rnnt_speech_recognition_b200.joint import _desc  # noqa: E402

WIDTHS = (None, "full", (64, 64), (16, 16), (4, 4))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q or "unavailable"}


def timed(fn, warmup=3, iters=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def workload(name):
    B, V, H = 32, 1024, 640
    g = torch.Generator().manual_seed(1234)
    if name == "C3":
        T, U = 512, 128
        il_h, ll_h = torch.full((B,), T, dtype=torch.int32), torch.full((B,), U - 1, dtype=torch.int32)
    else:
        T, U = 1200, 160
        il_h = torch.randint(300, T + 1, (B,), generator=g, dtype=torch.int32)
        ll_h = torch.randint(20, U, (B,), generator=g, dtype=torch.int32)
        il_h[0], ll_h[0] = T, U - 1
    t = [v.cuda().requires_grad_() for v in (
        torch.randn(B, T, H, generator=g), torch.randn(B, U, H, generator=g), torch.randn(H, V, generator=g) / H ** 0.5,
        torch.zeros(V))]
    lab = torch.randint(1, V, (B, U - 1), generator=g, dtype=torch.int32).cuda()
    il, ll = il_h.cuda(), ll_h.cuda()
    frames = rb.joint_rnnt_align(*t, lab, il, ll, precision="bf16",
                                 valid_tiles=rb.valid_tile_count(il_h, ll_h)).label_frames
    variants = {}
    for w in WIDTHS:
        if w is None:
            win, vt = None, rb.valid_tile_count(il_h, ll_h)
        else:
            lr = (T, T) if w == "full" else w
            win = rb.alignment_windows(frames, il, ll, *lr)
            vt = rb.valid_tile_count(il_h, ll_h, tuple(x.cpu().numpy() for x in win))
        sz = C.c_size_t(0)
        _lib.load().rnntb200_joint_workspace_size(C.byref(_desc(B, T, U, H, V, 0, "bf16", True, vt)), C.byref(sz))

        def step(win=win, vt=vt):
            costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision="bf16", windows=win, valid_tiles=vt)
            torch.autograd.grad(costs.sum() / B, t)
        variants["none" if w is None else ("full" if w == "full" else "%d,%d" % w)] = (step, vt, sz.value)
    return variants


def kernel_times(step):
    _lib.set_timing(True)
    step()
    torch.cuda.synchronize()
    out = {}
    for n, ms in _lib.get_timings():
        out[n] = round(out.get(n, 0.0) + ms, 3)
    _lib.set_timing(False)
    return out


def main():
    assert torch.cuda.is_available(), "bench_windows.py needs a GPU"
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    info = card()
    for name in ("C3", "C5-shaped ragged"):
        variants = workload(name)
        ms = {k: [] for k in variants}
        for r in range(rounds):
            for k in list(variants) + ["none"]:
                t = timed(variants[k][0])
                ms[k].append(t)
                print(json.dumps(dict(info, workload=name, round=r, windows=k, ms=round(t, 3))), flush=True)
        for k, (step, vt, ws) in variants.items():
            print(json.dumps(dict(info, workload=name, summary=True, windows=k, valid_tiles=vt, workspace_bytes=ws,
                                  median_ms=round(statistics.median(ms[k]), 3), spread_ms=round(max(ms[k]) - min(ms[k]), 3),
                                  runs=len(ms[k]), kernels_ms=kernel_times(step))), flush=True)
        del variants
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
