"""BASELINE C3 at FULL size (B=32, T=512, U=128, V=1024, H=640: the configuration bench.py quotes).

The CPU oracle needs minutes per utterance there, so the bf16 tensor-core path is held to
  * the fp32 exact CUDA path on the same inputs (itself pinned to the oracle / the reference's KATs at small sizes), and
  * size-independent properties of the loss: softmax shift invariance (sum_v dlogits == 0 => sum_v db == 0 and
    sum_v dW[h,:] == 0; costs unchanged by a constant added to the bias), batch additivity (per-utterance costs and
    d_enc/d_pred do not depend on the rest of the batch; weight gradients of a batch are the sum over its parts) and
    permutation equivariance.
"""
import numpy as np
import pytest
import torch

from conftest import assert_close
from test_gpu_joint import run_joint, synth

pytestmark = pytest.mark.gpu

C3 = dict(B=32, T=512, U=128, V=1024, H=640)
NAMES = ("d_enc", "d_pred", "dW", "db")


@pytest.fixture(scope="module")
def c3():
    k = synth(C3["B"], C3["T"], C3["U"], C3["V"], C3["H"], 2026, ragged=False)
    costs, grads = run_joint(k, "bf16")
    return k, costs, grads


def sub(k, idx):
    o = dict(k)
    for n in ("enc", "pred", "labels", "input_lengths", "label_lengths"):
        o[n] = np.ascontiguousarray(k[n][idx])
    return o


def test_c3_bf16_vs_fp32_exact(c3):
    k, c16, g16 = c3
    c32, g32 = run_joint(k, "fp32")
    assert np.all(np.isfinite(c16))
    assert_close(c16, c32, rtol=2e-4, atol=1e-2, what="costs")
    for a, b, n in zip(g16, g32, NAMES):
        assert np.all(np.isfinite(a)), n
        rel = np.linalg.norm(a - b) / np.linalg.norm(b)
        assert rel < 5e-3, (n, rel)
    # kept-activation backward against the recomputing backward at full size: the same kernels on the same numerators
    c_re, g_re = run_joint(k, "bf16", keep=False)
    assert np.array_equal(c16, c_re)
    for a, b, n in zip(g16, g_re, NAMES):
        assert np.linalg.norm(a - b) <= 1e-6 * np.linalg.norm(b), n


def test_c3_softmax_shift_invariance(c3):
    k, costs, (d_enc, d_pred, dW, db) = c3
    assert abs(db.astype(np.float64).sum()) <= 1e-3 * np.abs(db).sum()
    rows = np.abs(dW.astype(np.float64).sum(axis=1))
    assert np.all(rows <= 1e-3 * np.abs(dW).sum(axis=1) + 1e-6)
    k2 = dict(k)
    k2["b"] = (k["b"] + np.float32(0.75)).astype(np.float32)
    c2, _ = run_joint(k2, "bf16")
    assert_close(c2, costs, rtol=1e-5, atol=1e-2, what="costs under a bias shift")


def test_c3_batch_additivity_and_permutation(c3):
    k, costs, grads = c3
    B = C3["B"]
    halves = [np.arange(0, B // 2), np.arange(B // 2, B)]
    dW_sum, db_sum = 0.0, 0.0
    for idx in halves:
        ch, gh = run_joint(sub(k, idx), "bf16", scale=np.full(len(idx), 1.0 / B))
        assert_close(ch, costs[idx], rtol=1e-6, atol=1e-3, what="costs of a sub-batch")
        assert_close(gh[0], grads[0][idx], rtol=1e-4, atol=0, ntol=1e-4, what="d_enc of a sub-batch")
        assert_close(gh[1], grads[1][idx], rtol=1e-4, atol=0, ntol=1e-4, what="d_pred of a sub-batch")
        dW_sum, db_sum = dW_sum + gh[2].astype(np.float64), db_sum + gh[3].astype(np.float64)
    # (split-K ranges differ between the full batch and its halves: fp32 tensor-core accumulation order, ~1e-4 relative on
    #  the largest entries -- db[blank] is a same-sign sum over 2 M rows)
    assert_close(dW_sum, grads[2], rtol=0, atol=0, ntol=5e-4, what="dW additivity")
    assert_close(db_sum, grads[3], rtol=0, atol=0, ntol=5e-4, what="db additivity")
    perm = np.random.default_rng(7).permutation(B)
    cp, gp = run_joint(sub(k, perm), "bf16")
    assert_close(cp, costs[perm], rtol=1e-6, atol=1e-3, what="permuted costs")
    assert_close(gp[2], grads[2], rtol=0, atol=0, ntol=5e-4, what="dW under permutation")


def test_c3_ragged_matches_fp32_exact():
    """Same shape, ragged lengths (device-ranked tiles + partially filled tiles at full width)."""
    k = synth(8, C3["T"], C3["U"], C3["V"], C3["H"], 2027, ragged=True)
    c32, g32 = run_joint(k, "fp32")
    for keep in (True, False):
        c16, g16 = run_joint(k, "bf16", keep=keep)
        assert_close(c16, c32, rtol=2e-4, atol=1e-2, what="costs")
        for a, b, n in zip(g16, g32, NAMES):
            rel = np.linalg.norm(a - b) / np.linalg.norm(b)
            assert rel < 5e-3, (n, rel, keep)
        for b in range(8):
            assert not g16[0][b, k["input_lengths"][b]:].any() and not g16[1][b, k["label_lengths"][b] + 1:].any()
