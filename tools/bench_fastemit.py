"""Cost of FastEmit on one GPU: the same calls at fastemit_lambda = 0 and 0.01, alternating in one process.

  python tools/bench_fastemit.py [rounds]       default 3 rounds

Workloads (forward + backward through the torch surface, CUDA events around `iters` calls after a warm-up):
  * BASELINE C3 `joint_rnnt_loss` (B=32 T=512 U=128 V=1024 H=640, tensor-core path, bf16 inputs cast at the boundary);
  * the materialised-logits op at (32, 512, 128, 1024) with float32 and with bfloat16 logits.
Each round times every workload at lambda = 0, then 0.01, then 0 again, so drift shows up as spread between the two
lambda = 0 runs.  One JSON line per timing and a summary per workload (median of each lambda, and the run-to-run
spread of lambda = 0), each carrying the card's name and power limit read in the same run.
"""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rnnt_speech_recognition_b200 as rb  # noqa: E402

LAMBDA = 0.01


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
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


def joint_c3():
    B, T, U, V, H = 32, 512, 128, 1024, 640
    g = torch.Generator().manual_seed(1234)
    t = [v.to("cuda", torch.bfloat16).requires_grad_() for v in (
        torch.randn(B, T, H, generator=g), torch.randn(B, U, H, generator=g), torch.randn(H, V, generator=g) / H ** 0.5,
        torch.zeros(V))]
    lab = torch.randint(1, V, (B, U - 1), generator=g, dtype=torch.int32).cuda()
    il = torch.full((B,), T, dtype=torch.int32, device="cuda")
    ll = torch.full((B,), U - 1, dtype=torch.int32, device="cuda")

    def step(lam):
        costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision="bf16", fastemit_lambda=lam)
        torch.autograd.grad(costs.sum() / B, t)
    return step


def op(dtype):
    B, T, U, V = 32, 512, 128, 1024
    torch.manual_seed(0)
    lab = torch.randint(1, V, (B, U - 1), dtype=torch.int32, device="cuda")
    il = torch.full((B,), T, dtype=torch.int32, device="cuda")
    ll = torch.full((B,), U - 1, dtype=torch.int32, device="cuda")
    w = torch.full((B,), 1.0 / B, device="cuda")
    x = torch.randn(B, T, U, V, device="cuda").to(dtype).requires_grad_()

    def call(lam):
        costs = rb.rnnt_loss(x, lab, il, ll, fastemit_lambda=lam)
        torch.autograd.grad(costs, x, grad_outputs=w)
    return call


def main():
    assert torch.cuda.is_available(), "bench_fastemit.py needs a GPU"
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    info = card()
    work = {"joint_rnnt_loss C3 bf16": joint_c3, "op (32,512,128,1024) float32": lambda: op(torch.float32),
            "op (32,512,128,1024) bfloat16": lambda: op(torch.bfloat16)}
    for name, make in work.items():
        fn = make()
        ms = {0.0: [], LAMBDA: []}
        for r in range(rounds):
            for lam in (0.0, LAMBDA, 0.0):
                t = timed(lambda: fn(lam))
                ms[lam].append(t)
                print(json.dumps(dict(info, workload=name, round=r, fastemit_lambda=lam, ms=round(t, 3))), flush=True)
        z, f = ms[0.0], ms[LAMBDA]
        print(json.dumps(dict(info, workload=name, summary=True, median_ms_lambda0=round(statistics.median(z), 3),
                              median_ms_lambda=round(statistics.median(f), 3), fastemit_lambda=LAMBDA,
                              spread_ms_lambda0=round(max(z) - min(z), 3), spread_ms_lambda=round(max(f) - min(f), 3))),
              flush=True)
        del fn
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
