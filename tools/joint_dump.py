"""Runs one synthetic joint_rnnt_loss forward+backward on the tensor-core path and saves costs + gradients to an .npz.
Used by tests that compare two PROCESS-level configurations of the library (environment switches are read once per
process), e.g. the multi-chunk backward (RNNTB200_CHUNK_MB) against the single-chunk one.

    python tools/joint_dump.py OUT.npz B T U V H seed ragged keep [bound [fastemit_lambda]]

bound: 0 = none, 1 = pass valid_tiles = valid_tile_count(host lengths), N > 1 = pass valid_tiles = N (a deliberately wrong promise).
fastemit_lambda: passed to joint_rnnt_loss when given (default: the keyword is not passed).
The .npz also records which forward kernels ran ("kernels"), so that a test can tell keep mode from the recomputing mode.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

if __name__ == "__main__":
    from test_gpu_joint import run_joint, synth
    out = sys.argv[1]
    B, T, U, V, H, seed, ragged, keep = (int(x) for x in sys.argv[2:10])
    bound = int(sys.argv[10]) if len(sys.argv) > 10 else 0
    extra = dict(fastemit_lambda=float(sys.argv[11])) if len(sys.argv) > 11 else {}
    k = synth(B, T, U, V, H, seed, bool(ragged))
    import rnnt_speech_recognition_b200 as rb
    from rnnt_speech_recognition_b200 import _lib
    vt = None if bound == 0 else (rb.valid_tile_count(k["input_lengths"], k["label_lengths"]) if bound == 1 else bound)
    _lib.set_timing(True)
    if extra:
        import torch
        from test_gpu_joint import dev
        t = [dev(k[n], torch.float32).requires_grad_() for n in ("enc", "pred", "W", "b")]
        lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
        c = rb.joint_rnnt_loss(*t, lab, il, ll, blank=int(k["blank"]), precision="bf16", keep_activations=bool(keep),
                               valid_tiles=vt, **extra)
        (c * torch.full((B,), 1.0 / B, device="cuda")).sum().backward()
        costs, grads = c.detach().cpu().numpy(), [x.grad.cpu().numpy() for x in t]
    else:
        costs, grads = run_joint(k, "bf16", keep=bool(keep), valid_tiles=vt)
    names = sorted({n for n, _ in _lib.get_timings()})
    np.savez(out, costs=costs, d_enc=grads[0], d_pred=grads[1], dW=grads[2], db=grads[3], kernels=np.array(names))
