"""Mixed-precision cost of the loss on one GPU: the materialised-logits op on float16 / bfloat16 logits against the
float32 op, and the fused joint + loss step with bfloat16 against float32 inputs.

  python tools/bench_op16.py [B T U V]      default (16 256 64 256) and (32 512 128 1024)

Per shape and logits dtype: ms per forward + backward call through the torch surface (rnnt_loss, then the gradient
w.r.t. the logits for a per-utterance upstream gradient), achieved GB/s on the bytes each path has to move, and the
peak memory allocated during the call (logits included).  Bytes:
  float32 surface  5*N*V*4 + 24*N   the op's 3*N*V*4 (lse read, gradient read + write) + the backward's mul_ (read + write)
  16-bit op        6*N*V + 24*N     2 B read in the forward, 2 B read + 2 B write in the backward
Then one BASELINE C3 joint_rnnt_loss step (B=32 T=512 U=128 V=1024 H=640, tensor-core path) with enc / pred / W / b
given as bfloat16 (cast to float32 at the boundary) against float32.  One JSON line per result, each carrying the
card's name and power limit read in the same run.
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import rnnt_speech_recognition_b200 as rb  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
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


def peak_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated()


def op_shape(B, T, U, V, info):
    N = B * T * U
    torch.manual_seed(0)
    lab = torch.randint(1, V, (B, U - 1), dtype=torch.int32, device="cuda")
    il = torch.full((B,), T, dtype=torch.int32, device="cuda")
    ll = torch.full((B,), U - 1, dtype=torch.int32, device="cuda")
    w = torch.full((B,), 1.0 / B, device="cuda")
    out = []
    for dtype, byts in ((torch.float32, 5.0 * N * V * 4 + 24.0 * N), (torch.float16, 6.0 * N * V + 24.0 * N),
                        (torch.bfloat16, 6.0 * N * V + 24.0 * N)):
        torch.manual_seed(1)
        x = torch.randn(B, T, U, V, device="cuda").to(dtype).requires_grad_()

        def call():
            costs = rb.rnnt_loss(x, lab, il, ll)
            return torch.autograd.grad(costs, x, grad_outputs=w)[0]

        ms = timed(call)
        peak = peak_bytes(call)
        out.append(dict(info, shape=[B, T, U, V], logits=str(dtype).replace("torch.", ""), ms=round(ms, 3),
                        bytes=byts, GBps=round(byts / ms / 1e6, 1), peak_GB=round(peak / 1e9, 3)))
        del x
        torch.cuda.empty_cache()
    return out


def joint_c3(info, steps=10):
    B, T, U, V, H = 32, 512, 128, 1024, 640
    g = torch.Generator().manual_seed(1234)
    base = dict(enc=torch.randn(B, T, H, generator=g), pred=torch.randn(B, U, H, generator=g),
                W=torch.randn(H, V, generator=g) / H ** 0.5, b=torch.zeros(V))
    lab = torch.randint(1, V, (B, U - 1), generator=g, dtype=torch.int32).cuda()
    il = torch.full((B,), T, dtype=torch.int32, device="cuda")
    ll = torch.full((B,), U - 1, dtype=torch.int32, device="cuda")
    out = []
    for dtype in (torch.float32, torch.bfloat16, torch.float32, torch.bfloat16):     # alternating, two rounds each
        t = [v.to("cuda", dtype).requires_grad_() for v in base.values()]

        def step():
            costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision="bf16")
            torch.autograd.grad(costs.sum() / B, t)

        out.append(dict(info, workload="joint_rnnt_loss C3", inputs=str(dtype).replace("torch.", ""),
                        ms=round(timed(step, iters=steps), 3)))
        del t
        torch.cuda.empty_cache()
    return out


def main():
    assert torch.cuda.is_available(), "bench_op16.py needs a GPU"
    shapes = [tuple(int(v) for v in sys.argv[1:5])] if len(sys.argv) >= 5 else [(16, 256, 64, 256), (32, 512, 128, 1024)]
    info = card()
    for s in shapes:
        for r in op_shape(*s, info):
            print(json.dumps(r), flush=True)
    for r in joint_c3(info):
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
