"""Cost of forced alignment on one GPU, against the costs-only forward of the same workload, alternating in one process.

  python tools/bench_align.py [rounds]       default 3 rounds

Workloads (CUDA events around `iters` calls after a warm-up, everything under torch.no_grad):
  * BASELINE C3: `joint_rnnt_align` against `joint_rnnt_loss` (B=32 T=512 U=128 V=1024 H=640, tensor-core path);
  * a C5-shaped ragged batch (B=64, T_b in [100, 1600], U_b in [10, 200], V=4096, H=640) with `valid_tiles`;
  * the materialised-logits op at (32, 512, 128, 1024), float32 and bfloat16 logits: `rnnt_align` against `rnnt_loss`.
Each round times align, then the forward, then align again.  Then one call of each with the library's per-kernel timing
on (`rnntb200_set_timing`), which reports `viterbi_kernel` and `backtrace_kernel` next to `alpha_beta_kernel`.  Every
JSON line carries the card's name and power limit, read in the same run.
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import rnnt_speech_recognition_b200 as rb  # noqa: E402
from rnnt_speech_recognition_b200 import _lib  # noqa: E402
from bench_fastemit import card, timed  # noqa: E402


def joint(B, lengths, V, H, seed, valid):
    g = torch.Generator().manual_seed(seed)
    if lengths:
        il = torch.randint(100, 1601, (B,), generator=g, dtype=torch.int32)
        ll = torch.randint(10, 201, (B,), generator=g, dtype=torch.int32)
        T, U = int(il.max()), int(ll.max()) + 1
    else:
        T, U = 512, 128
        il, ll = torch.full((B,), T, dtype=torch.int32), torch.full((B,), U - 1, dtype=torch.int32)
    t = [v.cuda() for v in (torch.randn(B, T, H, generator=g), torch.randn(B, U, H, generator=g),
                            torch.randn(H, V, generator=g) / H ** 0.5, torch.zeros(V))]
    lab = torch.randint(1, V, (B, U - 1), generator=g, dtype=torch.int32).cuda()
    vt = rb.valid_tile_count(il.tolist(), ll.tolist()) if valid else None
    il, ll = il.cuda(), ll.cuda()
    return (lambda: rb.joint_rnnt_align(*t, lab, il, ll, valid_tiles=vt),
            lambda: rb.joint_rnnt_loss(*t, lab, il, ll, valid_tiles=vt))


def op(dtype):
    B, T, U, V = 32, 512, 128, 1024
    torch.manual_seed(0)
    lab = torch.randint(1, V, (B, U - 1), dtype=torch.int32, device="cuda")
    il = torch.full((B,), T, dtype=torch.int32, device="cuda")
    ll = torch.full((B,), U - 1, dtype=torch.int32, device="cuda")
    x = torch.randn(B, T, U, V, device="cuda").to(dtype)
    return lambda: rb.rnnt_align(x, lab, il, ll), lambda: rb.rnnt_loss(x, lab, il, ll)


def kernel_ms(fn):
    fn()
    torch.cuda.synchronize()
    _lib.set_timing(True)
    fn()
    torch.cuda.synchronize()
    out = {}
    for name, ms in _lib.get_timings():
        out[name] = round(out.get(name, 0.0) + ms, 4)
    _lib.set_timing(False)
    return out


def main():
    assert torch.cuda.is_available(), "bench_align.py needs a GPU"
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    info = card()
    work = {"C3 joint bf16": lambda: joint(32, False, 1024, 640, 1234, False),
            "C5-shaped joint bf16 valid_tiles": lambda: joint(64, True, 4096, 640, 99, True),
            "op (32,512,128,1024) float32": lambda: op(torch.float32),
            "op (32,512,128,1024) bfloat16": lambda: op(torch.bfloat16)}
    with torch.no_grad():
        for name, make in work.items():
            align, fwd = make()
            ms = {"align": [], "forward": []}
            for r in range(rounds):
                for kind, fn in (("align", align), ("forward", fwd), ("align", align)):
                    t = timed(fn, warmup=2, iters=5)
                    ms[kind].append(t)
                    print(json.dumps(dict(info, workload=name, round=r, call=kind, ms=round(t, 3))), flush=True)
            print(json.dumps(dict(info, workload=name, summary=True, median_ms_align=round(statistics.median(ms["align"]), 3),
                                  median_ms_forward=round(statistics.median(ms["forward"]), 3),
                                  spread_ms_align=round(max(ms["align"]) - min(ms["align"]), 3),
                                  kernels_align=kernel_ms(align), kernels_forward=kernel_ms(fwd))), flush=True)
            del align, fwd
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
