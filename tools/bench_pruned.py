"""Cost of pruned RNN-T on one GPU against the unrestricted step and the align-then-restrict recipe, in one process.

  python tools/bench_pruned.py [rounds]       default 3 rounds

Workloads: BASELINE C3 (B=32 T=512 U=128 V=1024 H=640) and the C5-shaped ragged batch of tools/bench_windows.py (B=32,
T up to 1200, U up to 160), with random am (B,T,V) / lm (B,U,V) standing in for the trivial joiner's projections.
Variants, each a forward + backward through the torch surface (tensor-core joint, CUDA events around 10 steps after 3):
  * full      the unrestricted joint_rnnt_loss step;
  * S=4/5/8/16  simple_rnnt_loss(am, lm, ..., s_range=S) forward + windows + backward, then the windowed joint step, with
              the loss 0.5 * simple + pruned;
  * align+-16 joint_rnnt_align, alignment_windows(+-16) and the windowed joint step.
`valid_tiles` is `valid_tile_count` of host copies of the variant's windows, taken once before timing (the windows of
these fixed inputs do not change between steps).  Each round times every variant in turn; per variant a summary line
with the valid tiles, median and spread of the step time and the per-kernel times of one instrumented step.  Every line
carries the card's name and power limit read in the same run.
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
from bench_windows import card, kernel_times, timed  # noqa: E402

S_RANGES = (4, 5, 8, 16)


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
    am = torch.randn(B, T, V, generator=g).cuda().requires_grad_()
    lm = torch.randn(B, U, V, generator=g).cuda().requires_grad_()
    lab = torch.randint(1, V, (B, U - 1), generator=g, dtype=torch.int32).cuda()
    il, ll = il_h.cuda(), ll_h.cuda()
    vt_full = rb.valid_tile_count(il_h, ll_h)
    host = lambda win: tuple(x.cpu().numpy() for x in win)
    variants = {}

    def full():
        costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision="bf16", valid_tiles=vt_full)
        torch.autograd.grad(costs.sum() / B, t)
    variants["full"] = (full, vt_full)

    for S in S_RANGES:
        with torch.no_grad():
            _, win = rb.simple_rnnt_loss(am, lm, lab, il, ll, s_range=S)
        vt = rb.valid_tile_count(il_h, ll_h, host(win))

        def pruned(S=S, vt=vt):
            simple, win = rb.simple_rnnt_loss(am, lm, lab, il, ll, s_range=S)
            costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision="bf16", windows=win, valid_tiles=vt)
            torch.autograd.grad((0.5 * simple + costs).sum() / B, t + [am, lm])
        variants["S=%d" % S] = (pruned, vt)

    frames = rb.joint_rnnt_align(*t, lab, il, ll, precision="bf16", valid_tiles=vt_full).label_frames
    vt_al = rb.valid_tile_count(il_h, ll_h, host(rb.alignment_windows(frames, il, ll, 16, 16)))

    def aligned():
        fr = rb.joint_rnnt_align(*t, lab, il, ll, precision="bf16", valid_tiles=vt_full).label_frames
        win = rb.alignment_windows(fr, il, ll, 16, 16)
        costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision="bf16", windows=win, valid_tiles=vt_al)
        torch.autograd.grad(costs.sum() / B, t)
    variants["align+-16"] = (aligned, vt_al)
    return variants


def main():
    assert torch.cuda.is_available(), "bench_pruned.py needs a GPU"
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    info = card()
    for name in ("C3", "C5-shaped ragged"):
        variants = workload(name)
        ms = {k: [] for k in variants}
        for r in range(rounds):
            for k, (step, _) in variants.items():
                t = timed(step)
                ms[k].append(t)
                print(json.dumps(dict(info, workload=name, round=r, variant=k, ms=round(t, 3))), flush=True)
        for k, (step, vt) in variants.items():
            print(json.dumps(dict(info, workload=name, summary=True, variant=k, valid_tiles=vt,
                                  median_ms=round(statistics.median(ms[k]), 3), spread_ms=round(max(ms[k]) - min(ms[k]), 3),
                                  runs=len(ms[k]), kernels_ms=kernel_times(step))), flush=True)
        del variants
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
