"""Measured error of the bf16 tensor-core path and of the fp32 exact path against the chunked float64 reference
(tests/joint_ref64.py) at the benchmark configuration: costs and all four gradients, one JSON line per path.

  python tools/accuracy_c3.py                 # BASELINE C3 (bench.py's inputs, seed 1234)
  python tools/accuracy_c3.py c5              # BASELINE C5 (bf16 with valid_tiles, as bench.py runs it)
  python tools/accuracy_c3.py B T U V H       # another dense shape
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import bench  # noqa: E402
import joint_ref64 as r64  # noqa: E402
import rnnt_speech_recognition_b200 as rb  # noqa: E402

if len(sys.argv) >= 6:
    B, T, U, V, H = (int(x) for x in sys.argv[1:6])
    name, cfg = "custom", dict(B=B, T=T, U=U, V=V, H=H)
else:
    name = sys.argv[1] if len(sys.argv) > 1 else "c3"
    cfg = bench.WORKLOADS[name]
d = bench.synth(cfg, 1234, "cuda")
enc, pred, W, b, lab, il, ll = (d[n] for n in ("enc", "pred", "W", "b", "labels", "il", "ll"))
B = enc.shape[0]
vt = rb.valid_tile_count(il.tolist(), ll.tolist()) if cfg.get("ragged") else None

want = r64.joint_loss_grad(enc, pred, W, b, lab, il, ll, grad_scale=[1.0 / B] * B)
torch.cuda.empty_cache()


def run(prec):
    t = [x.clone().requires_grad_() for x in (enc, pred, W, b)]
    costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision=prec, valid_tiles=vt if prec == "bf16" else None)
    (costs.sum() / B).backward()
    torch.cuda.synchronize()
    out = costs.detach().double().cpu(), [x.grad.double().cpu() for x in t]
    del t, costs
    torch.cuda.empty_cache()
    return out


ref_costs = torch.as_tensor(want["costs"])
for prec in ("bf16", "fp32"):
    c, g = run(prec)
    out = {"config": name, "shape": [cfg[k] for k in "BTUVH"], "path": prec, "reference": "float64",
           "device": torch.cuda.get_device_name(), "cost_max": ref_costs.abs().max().item(),
           "cost_max_rel_err": ((c - ref_costs).abs() / ref_costs.abs()).max().item()}
    for n, a in zip(("d_enc", "d_pred", "dW", "db"), g):
        r = torch.as_tensor(want[n])
        out[n] = {"rel_frobenius": ((a - r).norm() / r.norm()).item(),
                  "max_abs_err_over_max": ((a - r).abs().max() / r.abs().max()).item()}
    print(json.dumps(out))
