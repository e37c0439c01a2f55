"""Writes tests/golden/ref_cases.npz: what the unmodified reference library (oracle/_ref, built with WARP_TRANSDUCER_DIR
set) returns for the inputs of tests/test_oracle.py's live-reference comparisons, so that those comparisons run without
the reference sources.

    WARP_TRANSDUCER_DIR=<warp-transducer checkout> python tests/golden/make_ref_cases.py

Inputs are regenerated from seeds by the functions below, which the tests import.
"""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_cases.npz")
N_CPU_CASES = 40
N_JOINT_CASES = 10


def live_case(oracle):
    rng = np.random.default_rng(99)
    B, T, U, V = 4, 13, 6, 9
    acts = rng.standard_normal((B, T, U, V)).astype(np.float32)
    labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
    il = np.array([13, 7, 1, 10], np.int32)
    ll = np.array([5, 2, 0, 4], np.int32)
    return oracle.log_softmax(acts), labels, il, ll


def cpu_case(oracle, i):
    """Random shape, ragged lengths, blank position and logit scale; case i of a fixed sequence."""
    p = np.random.default_rng(1000 + i)
    B, T, U, V = int(p.integers(1, 5)), int(p.integers(1, 13)), int(p.integers(1, 8)), int(p.integers(2, 12))
    scale = float(p.choice([0.3, 1.0, 6.0]))
    rng = np.random.default_rng(int(p.integers(0, 2 ** 31 - 1)))
    acts = (scale * rng.standard_normal((B, T, U, V))).astype(np.float32)
    blank = int(rng.integers(0, V))
    cand = np.array([v for v in range(V) if v != blank])
    labels = (rng.choice(cand, size=(B, U - 1)).astype(np.int32) if U > 1 else np.zeros((B, 0), np.int32))
    il = rng.integers(1, T + 1, B).astype(np.int32)
    ll = rng.integers(0, U, B).astype(np.int32)
    il[0], ll[0] = T, U - 1                       # the reference sizes its slabs by maxT / maxU
    return oracle.log_softmax(acts), labels, il, ll, blank


def joint_cases():
    """The torch-fp64 joint chained through the reference library's fp64 entry (make_golden.joint_case)."""
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    rng = np.random.default_rng(20260924)
    out = []
    for _ in range(N_JOINT_CASES):
        B, T, U = int(rng.integers(1, 4)), int(rng.integers(1, 9)), int(rng.integers(1, 6))
        V, H = int(rng.integers(2, 9)), int(rng.integers(1, 7))
        out.append(mg.joint_case(rng, B, T, U, V, H, blank=int(rng.integers(0, V)), ragged=bool(rng.integers(0, 2))))
    return out


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from oracle import oracle
    assert oracle.have_ref(), "set WARP_TRANSDUCER_DIR to a warp-transducer checkout"
    d = {}
    lp, labels, il, ll = live_case(oracle)
    d["live_costs"], d["live_grads"] = oracle.ref_cpu_cost_and_grad(lp, labels, il, ll, num_threads=2)
    s = C.c_size_t(0)
    assert oracle.ref().get_workspace_size(13, 6, 4, True, C.byref(s), 4) == 0
    d["live_ws_gpu"] = np.array(s.value, np.int64)
    for i in range(N_CPU_CASES):
        lp, labels, il, ll, blank = cpu_case(oracle, i)
        d["cpu%d_costs" % i], d["cpu%d_grads" % i] = oracle.ref_cpu_cost_and_grad(lp, labels, il, ll, blank=blank, num_threads=1)
    for i, k in enumerate(joint_cases()):
        for n, a in k.items():
            d["joint%d_%s" % (i, n)] = np.asarray(a)
    np.savez_compressed(OUT, **d)
    print(OUT, len(d), "arrays")
