"""The dZ backward kernel (`bwd_dz_kernel`) of the tensor-core path at the run and pass geometries its epilogue has to
get right: one run = (utterance, 16-step time block) walking its u-blocks of 8 label positions, one pass = 128 columns
of H, the epilogue's enc / pred slice staged in shared memory by TMA per pass.  d_enc (sums over u, accumulated along a
run) and d_pred (sums over t, one partial plane per time block) are checked against the float64 oracle at the
tensor-core tolerances (DESIGN.md §4), and for bit-equality between keep and recompute mode and between one and several
workspace chunks (the same kernels on the same numerators)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, assert_close
from test_gpu_joint import run_joint, synth

pytestmark = pytest.mark.gpu

TC_COST_RTOL = 2e-4
TC_GRAD_NTOL = 1e-2
NAMES = ("d_enc", "d_pred", "dW", "db")


def oracle_of(oracle, k, gs):
    return oracle.joint_loss_grad(*(k[n].astype(np.float64) for n in ("enc", "pred", "W", "b")), k["labels"],
                                  k["input_lengths"], k["label_lengths"], 0, grad_scale=gs)


def check_vs_oracle(oracle, k):
    B = k["enc"].shape[0]
    gs = np.linspace(0.5, 1.5, B)
    o = oracle_of(oracle, k, gs)
    c_keep, g_keep = run_joint(k, "bf16", scale=gs, keep=True)
    c_re, g_re = run_joint(k, "bf16", scale=gs, keep=False)
    assert_close(c_keep, o["costs"], rtol=TC_COST_RTOL, atol=1e-3, what="costs")
    for g, n in zip(g_keep, NAMES):
        assert np.all(np.isfinite(g)), n
        assert_close(g, o[n], rtol=0, atol=0, ntol=TC_GRAD_NTOL, what=n)
        # a dropped tile, pass or row shows as a loss of norm, not only as an element-wise error
        assert np.linalg.norm(g) >= 0.5 * np.linalg.norm(o[n]), n
    assert np.array_equal(c_keep, c_re)
    for a, b_, n in zip(g_keep[:2], g_re[:2], NAMES):
        assert np.array_equal(a, b_), n
    for b in range(B):   # padded rows of d_enc / d_pred are exactly zero
        assert not g_keep[0][b, k["input_lengths"][b]:].any()
        assert not g_keep[1][b, k["label_lengths"][b] + 1:].any()


@pytest.mark.parametrize("B,T,U,V,H,seed", [
    (2, 20, 8, 128, 192, 0),      # one u-block per run, two passes (128 + 64 columns)
    (2, 20, 16, 128, 640, 1),     # two u-blocks per run, five passes
    (2, 18, 24, 128, 704, 2),     # three u-blocks, six passes, the last of 64 columns (H % 128 == 64)
    (1, 33, 40, 192, 640, 3),     # five u-blocks, three time blocks (the last partial)
    (1, 16, 128, 64, 192, 4),     # sixteen u-blocks, one K block of V
])
def test_u_blocks_per_run_vs_oracle(oracle, B, T, U, V, H, seed):
    check_vs_oracle(oracle, synth(B, T, U, V, H, seed, ragged=False))


@pytest.mark.parametrize("H", [192, 640, 704])
def test_ragged_runs_vs_oracle(oracle, H):
    """Utterances whose runs end at different u-blocks (1 to 5) and time blocks, partial last tiles in both directions."""
    k = synth(5, 37, 40, 128, H, 20 + H, ragged=False)
    k["input_lengths"] = np.array([37, 16, 5, 30, 17], np.int32)
    k["label_lengths"] = np.array([39, 0, 23, 8, 16], np.int32)
    for b in range(5):
        k["labels"][b, k["label_lengths"][b]:] = 0
    check_vs_oracle(oracle, k)


def dump(tmp_path, tag, args, env):
    f = str(tmp_path / (tag + ".npz"))
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "joint_dump.py"), f] + args,
                   check=True, env=dict(os.environ, **env), timeout=300)
    return dict(np.load(f))


def test_chunks_and_valid_tiles_bit_identical(tmp_path):
    """One workspace chunk, several chunks (keep and recompute) and a held `valid_tiles` bound give bit-identical costs,
    d_enc and d_pred (per-utterance quantities); a broken bound gives NaN costs and no fault."""
    base = ["6", "45", "40", "192", "640", "51", "1"]
    one = dump(tmp_path, "one", base + ["1"], {})
    chunked = dump(tmp_path, "chunked", base + ["1"], {"RNNTB200_CHUNK_MB": "1"})
    nokeep = dump(tmp_path, "nokeep", base + ["0"], {"RNNTB200_CHUNK_MB": "1"})
    bound = dump(tmp_path, "bound", base + ["1", "1"], {"RNNTB200_CHUNK_MB": "1"})
    broken = dump(tmp_path, "broken", base + ["1", "2"], {"RNNTB200_CHUNK_MB": "1"})
    assert "<fwd+keep>" in " ".join(str(x) for x in bound["kernels"])
    for o in (chunked, nokeep, bound):
        assert np.array_equal(o["costs"], one["costs"])
        for n in ("d_enc", "d_pred"):
            assert np.array_equal(o[n], one[n]), n
        for n in ("dW", "db"):                                  # summed over utterances in another order
            assert_close(o[n], one[n], rtol=0, atol=0, ntol=2e-5, what=n)
    assert np.isnan(broken["costs"]).all()


def test_common_voice_shaped_ragged_batch():
    """BASELINE C5's shape in miniature (V = 4096, H = 640, maxU = 200, ragged lengths that end inside time and label
    blocks): d_enc and d_pred against the fp32 exact path, and bit-equal between keep and recompute mode."""
    B, T, U, V, H = 4, 120, 200, 4096, 640
    k = synth(B, T, U, V, H, 61, ragged=False)
    k["input_lengths"] = np.array([120, 9, 77, 101], np.int32)
    k["label_lengths"] = np.array([199, 6, 130, 41], np.int32)
    for b in range(B):
        k["labels"][b, k["label_lengths"][b]:] = 0
    c32, g32 = run_joint(k, "fp32")
    c16, g16 = run_joint(k, "bf16", keep=True)
    c16r, g16r = run_joint(k, "bf16", keep=False)
    assert_close(c16, c32, rtol=TC_COST_RTOL, atol=1e-3, what="costs")
    for a, b_, n in zip(g16, g32, NAMES):
        assert np.all(np.isfinite(a)), n
        assert np.linalg.norm(a - b_) / np.linalg.norm(b_) < 5e-3, n
    assert np.array_equal(c16, c16r)
    for a, b_, n in zip(g16[:2], g16r[:2], NAMES):
        assert np.array_equal(a, b_), n
