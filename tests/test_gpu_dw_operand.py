"""The dW backward of the tensor-core path, whose A operand (the bf16 dW operand [rs * tanh(enc + pred), rs], one row per
kept lattice row) is written once by the dZ kernel's epilogue and read by the dW kernel's TMA on 128 h x 256 v tiles.
The cases sit where that split of work has edges:

  * H = 64, 128, 640, 768: one or six 128-row blocks, H % 128 == 64 (the last block holds rows H - 64 .. H, its second
    warpgroup reads column H and zero fill) and H % 128 == 0 (a block of its own holds only the db row);
  * V = 192, 1024, 1152: a last v-tile of 192 and of 128 columns (B boxes past V read as zeros), four full tiles;
  * ragged lengths, band windows (tiles without a slot, rows of rs = 0 inside slotted tiles), keep and recompute mode,
    several workspace chunks;
  * NaN in enc past T_b and in pred past U_b inside a tile: nothing of theirs may reach any gradient.

dW and db are held to tests/joint_ref64.py (float64) at DESIGN.md 4's tensor-core bounds, windowed runs to the fp32
exact path with the same windows; every run is checked for determinism, and one for CUDA-graph replay."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import joint_ref64 as r64
from conftest import ROOT, assert_close
from test_gpu_joint import dev, synth

pytestmark = pytest.mark.gpu

NAMES = ("d_enc", "d_pred", "dW", "db")
TC_COST = dict(rtol=2e-4, atol=1e-3)


def run(k, precision="bf16", keep=True, win=None, gs=None):
    import rnnt_speech_recognition_b200 as rb
    t = [dev(k[n], torch.float32).requires_grad_() for n in ("enc", "pred", "W", "b")]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    w = None if win is None else tuple(dev(x, torch.int32) for x in win)
    costs = rb.joint_rnnt_loss(*t, lab, il, ll, blank=int(k["blank"]), precision=precision, keep_activations=keep,
                               windows=w)
    B = costs.shape[0]
    gs = np.full(B, 1.0 / B) if gs is None else gs
    (costs * dev(gs, torch.float32)).sum().backward()
    return costs.detach().cpu().numpy(), [x.grad.cpu().numpy() for x in t]


def reference(k, gs):
    out = r64.joint_loss_grad(*(dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")), k["labels"],
                              k["input_lengths"], k["label_lengths"], int(k["blank"]), grad_scale=gs)
    torch.cuda.synchronize()
    return out


def check_grad(g, w, what, ntol=1e-2, frob=5e-3):
    """DESIGN.md 4's tensor-core bounds: element-wise ntol * max|g|, relative Frobenius error, no loss of norm."""
    assert np.all(np.isfinite(g)), what
    ng, no = np.linalg.norm(g), np.linalg.norm(w)
    assert ng >= 0.5 * no, "%s: |g| = %.4g is less than half the reference's %.4g" % (what, ng, no)
    assert_close(g, w, rtol=0, atol=0, ntol=ntol, what=what)
    assert np.linalg.norm(g - w) / no < frob, what


def ragged(B, T, U, V, H, seed):
    """Lengths that end inside time blocks of 16 and label blocks of 8, the longest utterance first."""
    k = synth(B, T, U, V, H, seed, ragged=False)
    rng = np.random.default_rng(seed + 1)
    k["input_lengths"] = np.concatenate([[T], rng.integers(3, T, B - 1)]).astype(np.int32)
    k["label_lengths"] = np.concatenate([[U - 1], rng.integers(0, U - 1, B - 1)]).astype(np.int32)
    for b in range(B):
        k["labels"][b, k["label_lengths"][b]:] = 0
    return k


@pytest.mark.parametrize("V", [192, 1024, 1152])
@pytest.mark.parametrize("H", [64, 128, 640, 768])
def test_dw_db_vs_float64(H, V):
    k = ragged(3, 45, 21, V, H, 7 * H + V)
    gs = np.array([0.5, 1.0, 1.5])
    want = reference(k, gs)
    costs, grads = run(k, keep=True, gs=gs)
    assert_close(costs, want["costs"], what="costs", **TC_COST)
    for g, n in zip(grads, NAMES):
        check_grad(g, want[n], "H=%d V=%d %s" % (H, V, n))
    costs2, grads2 = run(k, keep=True, gs=gs)                   # deterministic
    costs_re, grads_re = run(k, keep=False, gs=gs)              # the recomputing backward: the same kernels, the same bits
    for o_c, o_g in ((costs2, grads2), (costs_re, grads_re)):
        assert np.array_equal(o_c, costs)
        for a, b_, n in zip(o_g, grads, NAMES):
            assert np.array_equal(a, b_), n


def band_windows(il, ll, U, width):
    """Per label position u < U_b the frames [u T_b / U_b - width, (u + 1) T_b / U_b + width], clipped: a monotone band
    that admits paths and leaves most 16 x 8 tiles of a long lattice without a slot."""
    B = len(il)
    lo, hi = np.zeros((B, U), np.int32), np.zeros((B, U), np.int32)
    for b in range(B):
        T, Ub = int(il[b]), int(ll[b]) + 1
        for u in range(U):
            c = min(u, Ub - 1)
            lo[b, u] = max(0, c * T // Ub - width)
            hi[b, u] = min(T - 1, (c + 1) * T // Ub + width)
    return lo, hi


@pytest.mark.parametrize("keep", [True, False])
def test_windowed_dw_vs_fp32_exact(keep):
    """Band windows: tiles without a slot at the start and the end of a run, rows of rs = 0 inside slotted tiles."""
    k = ragged(3, 160, 40, 1152, 640, 31)
    win = band_windows(k["input_lengths"], k["label_lengths"], 40, 6)
    c32, g32 = run(k, "fp32", win=win)
    c16, g16 = run(k, "bf16", keep=keep, win=win)
    assert np.all(np.isfinite(c32))
    assert_close(c16, c32, what="costs", **TC_COST)
    for a, b_, n in zip(g16, g32, NAMES):
        check_grad(a, b_, "windowed %s" % n)
    c16b, g16b = run(k, "bf16", keep=keep, win=win)
    assert np.array_equal(c16, c16b)
    for a, b_, n in zip(g16, g16b, NAMES):
        assert np.array_equal(a, b_), n


def test_several_workspace_chunks_vs_float64(tmp_path):
    """RNNTB200_CHUNK_MB (read once per process) splits the batch into several chunks: the dW operand is rewritten per
    chunk and the dW planes accumulate across chunks."""
    args = ["5", "45", "40", "1152", "704", "77", "1"]
    outs = {}
    for tag, env in (("one", {}), ("chunked", {"RNNTB200_CHUNK_MB": "1"})):
        f = str(tmp_path / (tag + ".npz"))
        subprocess.run([sys.executable, os.path.join(ROOT, "tools", "joint_dump.py"), f] + args + ["1"],
                       check=True, env=dict(os.environ, **env), timeout=300)
        outs[tag] = dict(np.load(f))
    k = synth(5, 45, 40, 1152, 704, 77, ragged=True)
    want = reference(k, np.full(5, 1.0 / 5))
    for tag, o in outs.items():
        for n in NAMES:
            check_grad(o[n], want[n], "%s %s" % (tag, n))
    for n in ("dW", "db"):                                      # summed over utterances in another order
        assert_close(outs["chunked"][n], outs["one"][n], rtol=0, atol=0, ntol=2e-5, what=n)


def test_nan_padding_past_the_lengths_reaches_no_gradient():
    """enc rows t >= T_b and pred rows u > U_b inside the last tile of an utterance hold NaN: the results are those of
    zero padding, bit for bit (rows outside the lattice have rs = 0, and their dW operand is 0)."""
    k = ragged(3, 45, 21, 1152, 704, 5)
    k["input_lengths"] = np.array([45, 37, 20], np.int32)       # 37 % 16 and 20 % 16 end inside a time block
    k["label_lengths"] = np.array([20, 12, 9], np.int32)        # U_b = 13, 10 end inside a label block
    clean = run(k)
    for b in range(3):
        k["enc"][b, k["input_lengths"][b]:] = np.nan
        k["pred"][b, k["label_lengths"][b] + 1:] = np.nan
    dirty = run(k)
    assert np.array_equal(dirty[0], clean[0])
    for a, b_, n in zip(dirty[1], clean[1], NAMES):
        assert np.all(np.isfinite(a)), n
        assert np.array_equal(a, b_), n


def test_cuda_graph_replay():
    """The dZ kernel's operand store and the dW kernel's loads are stream-ordered: the backward replays in a CUDA graph
    on new inputs with the bits of an eager run."""
    import rnnt_speech_recognition_b200 as rb
    torch.manual_seed(0)
    B, T, U, V, H = 3, 64, 24, 1152, 768
    enc = torch.randn(B, T, H, device="cuda", requires_grad=True)
    pred = torch.randn(B, U, H, device="cuda", requires_grad=True)
    W = (torch.randn(H, V, device="cuda") / H ** 0.5).requires_grad_()
    b = torch.zeros(V, device="cuda", requires_grad=True)
    lab = torch.randint(1, V, (B, U - 1), dtype=torch.int32, device="cuda")
    il = torch.tensor([T, 37, 50], dtype=torch.int32, device="cuda")
    ll = torch.tensor([U - 1, 5, 17], dtype=torch.int32, device="cuda")

    def step():
        for t in (enc, pred, W, b):
            t.grad = None
        costs = rb.joint_rnnt_loss(enc, pred, W, b, lab, il, ll, precision="bf16")
        (costs.sum() / B).backward()
        return costs

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = step()
        grads = [t.grad for t in (enc, pred, W, b)]
    torch.cuda.current_stream().wait_stream(s)
    with torch.no_grad():
        enc.copy_(torch.randn_like(enc))
        pred.copy_(torch.randn_like(pred))
    g.replay()
    torch.cuda.synchronize()
    got_c, got_g = out.clone(), [x.clone() for x in grads]
    want_c = step().detach()
    torch.cuda.synchronize()
    assert torch.equal(got_c, want_c)
    for a, t in zip(got_g, (enc, pred, W, b)):
        assert torch.equal(a, t.grad)
