"""Alignment-restricted RNN-T (`windows=`) on the H100, on every numerical path: the fp32 loss op, the fp16 / bf16 loss op,
the fp32 exact joint and the tensor-core joint (keep, recompute, several workspace chunks, with and without `valid_tiles`).

* Against the float64 reference (tests/window_ref.py) at each path's DESIGN §4 tolerance, with random feasible windows and
  with `alignment_windows` of the GPU's own alignment; gradients of cells outside the windows exactly 0.
* Full windows are bit-identical to the call without windows; infeasible windows give +inf / zero gradients and leave the
  other utterances alone; large values in cells outside the windows change nothing.
* Tensor-core path: bands that start in a later u-block and leave whole time blocks empty (outputs NaN-prefilled through
  the C ABI), a broken windowed `valid_tiles` promise, determinism, CUDA-graph replay, full C3 size.
"""
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import window_ref as wr
from conftest import ROOT, assert_close, fp32_tol, load
from test_gpu_fastemit import UNIT, dev, op_tol
from test_gpu_joint import synth
from test_gpu_joint_bf16 import TC_COST_RTOL, TC_GRAD_NTOL
from test_gpu_ref64 import ab_cell, ab_norm, check_fp32

pytestmark = pytest.mark.gpu

NAMES = ("d_enc", "d_pred", "dW", "db")
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


def full_windows(il, B, U):
    return np.zeros((B, U), np.int32), np.broadcast_to((np.asarray(il) - 1)[:, None], (B, U)).astype(np.int32).copy()


def dwin(win):
    return None if win is None else tuple(dev(w, torch.int32) for w in win)


def run_op(acts, labels, il, ll, blank=0, gs=None, dtype=torch.float32, win=None, lam=0.0):
    import rnnt_speech_recognition_b200 as rb
    x = dev(acts, torch.float32).to(dtype).requires_grad_()
    B = acts.shape[0]
    gs = np.full(B, 1.0 / B) if gs is None else gs
    costs = rb.rnnt_loss(x, dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32), blank,
                         fastemit_lambda=lam, windows=dwin(win))
    (g,) = torch.autograd.grad(costs, x, grad_outputs=dev(gs, torch.float32))
    return costs.detach().cpu().numpy(), g.double().cpu().numpy()


def run_joint(k, precision, win=None, gs=None, keep=None, lam=0.0, valid_tiles=None):
    import rnnt_speech_recognition_b200 as rb
    t = [dev(k[n], torch.float32).requires_grad_() for n in ("enc", "pred", "W", "b")]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    costs = rb.joint_rnnt_loss(*t, lab, il, ll, blank=int(k["blank"]), precision=precision, keep_activations=keep,
                               fastemit_lambda=lam, windows=dwin(win), valid_tiles=valid_tiles)
    B = costs.shape[0]
    gs = np.full(B, 1.0 / B) if gs is None else gs
    grads = torch.autograd.grad(costs, t, grad_outputs=dev(gs, torch.float32))
    return costs.detach().cpu().numpy(), [g.double().cpu().numpy() for g in grads]


def joint_ref(k, win, gs, lam=0.0):
    return wr.joint_loss_grad(k["enc"], k["pred"], k["W"], k["b"], k["labels"], k["input_lengths"], k["label_lengths"],
                              int(k["blank"]), win, gs, lam)


def op_case(name):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    blank = 0
    if name.startswith("logits_"):
        k = load(name)
        return k["acts"], k["labels"], k["input_lengths"], k["label_lengths"], int(k["blank"])
    kind, V = name.split(":")
    V = int(V)
    B, T, U = {"wide": (3, 60, 45), "t1": (2, 1, 5), "u1": (2, 9, 1)}.get(kind, (3, 20, 9))
    acts = (2.0 * rng.standard_normal((B, T, U, V))).astype(np.float32)
    labels = rng.integers(0, V, (B, max(U - 1, 1))).astype(np.int32)[:, :max(U - 1, 0) or 1]
    il, ll = rng.integers(1, T + 1, B).astype(np.int32), rng.integers(0, U, B).astype(np.int32)
    il[0], ll[0] = T, U - 1
    if kind == "blank5":
        labels[rng.random(labels.shape) < 1 / 3] = 5
        blank = 5
    if kind == "blanklast":
        blank = V - 1
    if U == 1:
        labels = np.zeros((B, 0), np.int32)
    return acts, labels, il, ll, blank


OP_CASES = ["logits_ragged_B5_T12_U7_V11.npz", "logits_wide_U70_V40.npz", "wide:24", "v:1024", "v:1028", "v:4096",
            "blank5:128", "blanklast:64", "t1:32", "u1:32"]


@pytest.mark.parametrize("lam", [0.0, 0.5])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("name", OP_CASES)
def test_op_vs_reference(name, dt, lam):
    acts, labels, il, ll, blank = op_case(name)
    B, T, U, V = acts.shape
    dtype = DT[dt]
    x = dev(acts, torch.float32).to(dtype).double().cpu().numpy()          # the values the kernels see
    rng = np.random.default_rng(17)
    win = wr.random_feasible_windows(rng, il, ll, U, slack=2)
    gs = rng.uniform(0.5, 2.0, B)
    want_c, want_g = wr.logits_grad(x, labels, il, ll, blank, win, lam, gs)
    costs, g = run_op(acts, labels, il, ll, blank, gs, dtype, win, lam)
    assert np.isfinite(want_c).all()
    assert_close(costs, want_c, what="costs", **fp32_tol(want_c))
    rtol, atol = op_tol(want_c, dtype, gs)
    assert np.all(np.abs(g - want_g) <= atol + rtol * np.abs(want_g)), float(np.abs(g - want_g).max())
    assert not g[~wr.allowed_mask(win, il, ll, T, U)].any()                # padded and not-allowed cells: exactly 0
    plain, _ = run_op(acts, labels, il, ll, blank, gs, dtype, None, lam)
    assert (costs >= plain - 1e-4 * np.abs(plain)).all()


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("name", ["logits_wide_U70_V40.npz", "v:1024", "v:1028"])
def test_op_full_windows_are_bit_identical(name, dt):
    acts, labels, il, ll, blank = op_case(name)
    B, T, U, V = acts.shape
    for lam in (0.0, 0.5):
        c0, g0 = run_op(acts, labels, il, ll, blank, None, DT[dt], None, lam)
        lo, hi = full_windows(il, B, U)
        c1, g1 = run_op(acts, labels, il, ll, blank, None, DT[dt], (lo - 3, hi + 1000), lam)
        assert np.array_equal(c0, c1) and np.array_equal(g0, g1)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_op_infeasible_utterance_and_junk_outside_the_windows(dt):
    acts, labels, il, ll, blank = op_case("wide:24")
    B, T, U, V = acts.shape
    rng = np.random.default_rng(3)
    lo, hi = wr.random_feasible_windows(rng, il, ll, U, slack=2)
    c_ok, g_ok = run_op(acts, labels, il, ll, blank, None, DT[dt], (lo, hi), 0.5)
    lo2, hi2 = lo.copy(), hi.copy()
    lo2[1, 0], hi2[1, 0] = 5, 2                                            # utterance 1: column 0 empty, no path
    junk = acts.copy()
    junk[~wr.allowed_mask((lo2, hi2), il, ll, T, U)] = 3e4                 # large finite logits where nothing may be read
    for a in (acts, junk):
        c, g = run_op(a, labels, il, ll, blank, None, DT[dt], (lo2, hi2), 0.5)
        assert c[1] == np.inf and not g[1].any() and np.isfinite(g).all()
        keep = [b for b in range(B) if b != 1]
        assert np.array_equal(c[keep], c_ok[keep]) and np.array_equal(g[keep], g_ok[keep])


JOINT_CASES = [(3, 37, 19, 128, 64, 0, True), (2, 70, 45, 256, 192, 1, True), (2, 1, 6, 64, 64, 2, False),
               (2, 20, 1, 64, 64, 3, False)]


@pytest.mark.parametrize("lam", [0.0, 0.5])
@pytest.mark.parametrize("B,T,U,V,H,seed,ragged", JOINT_CASES)
def test_fp32_joint_vs_reference(B, T, U, V, H, seed, ragged, lam):
    k = synth(B, T, U, V, H, seed, ragged)
    if U == 1:
        k["labels"] = np.zeros((B, 0), np.int32)
    rng = np.random.default_rng(seed)
    win = wr.random_feasible_windows(rng, k["input_lengths"], k["label_lengths"], U, slack=2)
    gs = np.linspace(0.5, 1.5, B)
    want = joint_ref(k, win, gs, lam)
    costs, grads = run_joint(k, "fp32", win, gs, lam=lam)
    check_fp32(costs, grads, want, gs, "fp32 joint")              # DESIGN §4's fp32 bounds with the alpha/beta term


@pytest.mark.parametrize("keep", [True, False])
@pytest.mark.parametrize("lam", [0.0, 0.5])
@pytest.mark.parametrize("B,T,U,V,H,seed,ragged", JOINT_CASES)
def test_tc_joint_vs_reference(B, T, U, V, H, seed, ragged, lam, keep):
    import rnnt_speech_recognition_b200 as rb
    k = synth(B, T, U, V, H, seed, ragged)
    if U == 1:
        k["labels"] = np.zeros((B, 0), np.int32)
    rng = np.random.default_rng(seed)
    win = wr.random_feasible_windows(rng, k["input_lengths"], k["label_lengths"], U, slack=2)
    gs = np.linspace(0.5, 1.5, B)
    want = joint_ref(k, win, gs, lam)
    vt = rb.valid_tile_count(k["input_lengths"], k["label_lengths"], win)
    outs = [run_joint(k, "bf16", win, gs, keep, lam, v) for v in (None, vt)]
    for costs, grads in outs:
        assert_close(costs, want["costs"], rtol=TC_COST_RTOL, atol=1e-3, what="costs")
        for g, n in zip(grads, NAMES):
            assert_close(g, want[n], rtol=0, atol=0, ntol=TC_GRAD_NTOL, what=n)
    assert np.array_equal(outs[0][0], outs[1][0])                          # with / without valid_tiles
    for a, b_ in zip(outs[0][1], outs[1][1]):
        assert np.array_equal(a, b_)
    c2, g2 = run_joint(k, "bf16", win, gs, not keep, lam)                  # keep vs recompute: identical costs
    assert np.array_equal(c2, outs[0][0])
    for a, b_, n in zip(g2, outs[0][1], NAMES):
        assert_close(a, b_, rtol=0, atol=0, ntol=1e-6, what=n)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_joint_full_windows_equal_the_unwindowed_call(precision):
    k = synth(4, 70, 45, 256, 192, 31, ragged=True)
    B, U = 4, 45
    lo, hi = full_windows(k["input_lengths"], B, U)
    for keep in (True, False):
        for lam in (0.0, 0.5):
            c0, g0 = run_joint(k, precision, None, keep=keep, lam=lam)
            c1, g1 = run_joint(k, precision, (lo, hi + 7), keep=keep, lam=lam)
            assert np.array_equal(c0, c1)
            for a, b_, n in zip(g0, g1, NAMES):
                if precision == "bf16":
                    assert np.array_equal(a, b_), n
                else:       # float atomics: within the exact path's own run-to-run variation
                    assert_close(a, b_, rtol=0, atol=0, ntol=2e-5, what=n)


def _abi_joint(k, win, keep, prefill=float("nan")):
    """The windowed C entries called directly on the tensor-core path, every output and the workspace prefilled."""
    import rnnt_speech_recognition_b200 as rb
    from rnnt_speech_recognition_b200 import _lib
    from rnnt_speech_recognition_b200.joint import _joint_setup
    L = _lib.load()
    t = [dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")]
    ints = [dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths")]
    args, desc, ws = _joint_setup(*t, *ints, int(k["blank"]), "bf16", keep, None)
    ws[:ws.numel() // 4 * 4].view(torch.float32).fill_(prefill)
    lo, hi = dwin(win)
    B = desc.B
    costs = torch.full((B,), prefill, device="cuda")
    outs = [torch.full_like(x, prefill) for x in t]
    g = torch.full((B,), 1.0 / B, device="cuda")
    p = _lib.ptr
    assert L.rnntb200_joint_loss_forward_windowed(C.byref(desc), *map(p, args), p(lo), p(hi), p(costs), p(ws)) == 0
    assert L.rnntb200_joint_loss_backward_windowed(C.byref(desc), *map(p, args), p(lo), p(hi), p(g), *map(p, outs), p(ws), 0.0) == 0
    torch.cuda.synchronize()
    return costs.cpu().numpy(), [o.double().cpu().numpy() for o in outs]


@pytest.mark.parametrize("keep", [True, False])
def test_tc_band_that_skips_leading_u_blocks_and_whole_time_blocks(keep):
    """Utterance 0: a staircase whose band enters each time block in a later u-block.  Utterance 1: every label inside frames
    [64, 80), so the blank runs before and after leave most (time block, u-block) pairs without a slot.  Utterance 2: no path
    at all (infeasible): all its time blocks are empty."""
    B, T, U, V, H = 3, 128, 41, 128, 128
    k = synth(B, T, U, V, H, 9, ragged=False)
    il, ll = k["input_lengths"], k["label_lengths"]
    lo, hi = np.zeros((B, U), np.int32), np.zeros((B, U), np.int32)
    a = (np.arange(U) * 3).astype(np.int32)
    lo[0], hi[0] = np.maximum(a - 1, 0), np.minimum(a + 4, T - 1)
    lo[0, 0], hi[0, -1] = 0, T - 1
    lo[1], hi[1] = 64, 79
    lo[1, 0], hi[1, -1] = 0, T - 1
    lo[2], hi[2] = 10, 5
    win = (lo, hi)
    want = joint_ref(k, win, np.full(B, 1.0 / B))
    assert np.isfinite(want["costs"][:2]).all() and want["costs"][2] == np.inf
    costs, grads = _abi_joint(k, win, keep)
    assert costs[2] == np.inf
    assert_close(costs[:2], want["costs"][:2], rtol=TC_COST_RTOL, atol=1e-3, what="costs")
    for g, n in zip(grads, NAMES):
        assert np.isfinite(g).all(), n
        assert_close(g, want[n], rtol=0, atol=0, ntol=TC_GRAD_NTOL, what=n)
    ok = wr.allowed_mask(win, il, ll, T, U)
    d_enc, d_pred = grads[0], grads[1]
    assert not d_enc[~ok.any(axis=2)].any()            # frames with no allowed cell (whole empty time blocks among them)
    assert not d_pred[~ok.any(axis=1)].any()
    assert not d_enc[2].any() and not d_pred[2].any()
    # large finite junk in the inputs of frames / label positions no allowed cell uses changes nothing
    k2 = dict(k, enc=k["enc"].copy(), pred=k["pred"].copy())
    k2["enc"][~ok.any(axis=2)] = 50.0
    c2, g2 = _abi_joint(k2, win, keep, prefill=1e30)
    assert np.array_equal(c2, costs)
    for a_, b_, n in zip(g2, grads, NAMES):
        assert np.array_equal(a_, b_), n


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_joint_infeasible_utterance_leaves_the_others_alone(precision):
    k = synth(3, 40, 20, 128, 64, 4, ragged=True)
    B, U = 3, 20
    rng = np.random.default_rng(0)
    lo, hi = wr.random_feasible_windows(rng, k["input_lengths"], k["label_lengths"], U, slack=2)
    c_ok, g_ok = run_joint(k, precision, (lo, hi), lam=0.5)
    lo2, hi2 = lo.copy(), hi.copy()
    lo2[1, 0], hi2[1, 0] = 3, 1
    c, g = run_joint(k, precision, (lo2, hi2), lam=0.5)
    assert c[1] == np.inf and np.array_equal(c[[0, 2]], c_ok[[0, 2]])
    for a in g:
        assert np.isfinite(a).all()
    assert not g[0][1].any() and not g[1][1].any()
    k1 = {n: (v[[0, 2]] if n in ("enc", "pred", "labels", "input_lengths", "label_lengths") else v) for n, v in k.items()}
    want = joint_ref(k1, (lo[[0, 2]], hi[[0, 2]]), np.full(2, 1.0 / 3), 0.5)
    ab = ab_norm(float(want["costs"].max()))
    tol = dict(rtol=1e-4, atol=1e-6, ntol=max(1e-5, ab)) if precision == "fp32" else dict(rtol=0, atol=0, ntol=TC_GRAD_NTOL)
    assert_close(g[2], want["dW"], what="dW", **tol)
    assert_close(g[0][[0, 2]], want["d_enc"], what="d_enc", **tol)


@pytest.mark.parametrize("left,right", [(0, 0), (2, 3), (16, 16)])
def test_windows_from_the_gpus_own_alignment(left, right):
    import rnnt_speech_recognition_b200 as rb
    k = synth(4, 90, 40, 256, 128, 12, ragged=True)
    t = [dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    al = rb.joint_rnnt_align(*t, lab, il, ll, precision="bf16")
    win = rb.alignment_windows(al.label_frames, il, ll, left, right)
    hwin = tuple(w.cpu().numpy() for w in win)
    vt = rb.valid_tile_count(k["input_lengths"], k["label_lengths"], hwin)
    costs = rb.joint_rnnt_loss(*t, lab, il, ll, precision="bf16", windows=win, valid_tiles=vt).cpu().numpy()
    plain, best = al.costs.cpu().numpy(), al.best_logp.cpu().numpy()
    assert np.isfinite(costs).all()
    assert (costs >= plain - 1e-5 * np.abs(plain)).all() and (costs <= -best + 1e-5 * np.abs(best)).all()
    if (left, right) == (0, 0):
        np.testing.assert_allclose(costs, -best, rtol=1e-5)
    want = joint_ref(k, hwin, None)
    assert_close(costs, want["costs"], rtol=TC_COST_RTOL, atol=1e-3, what="costs")
    # the op on the materialised logits, same windows
    logits = rb.joint_logits(*t)
    c_op = rb.rnnt_loss(logits, lab, il, ll, windows=win).cpu().numpy()
    assert_close(c_op, want["costs"], what="op costs", **fp32_tol(want["costs"]))


def test_tc_windowed_runs_are_bit_identical_and_replay_in_a_cuda_graph():
    import rnnt_speech_recognition_b200 as rb
    torch.manual_seed(0)
    B, T, U, V, H = 4, 64, 32, 256, 128
    enc = torch.randn(B, T, H, device="cuda", requires_grad=True)
    pred = torch.randn(B, U, H, device="cuda", requires_grad=True)
    W = (torch.randn(H, V, device="cuda") / H ** 0.5).requires_grad_()
    b = torch.zeros(V, device="cuda", requires_grad=True)
    lab = torch.randint(1, V, (B, U - 1), dtype=torch.int32, device="cuda")
    il_h, ll_h = np.array([T, T - 7, 20, T], np.int32), np.array([U - 1, 5, U - 1, 12], np.int32)
    il, ll = dev(il_h), dev(ll_h)
    win = dwin(wr.random_feasible_windows(np.random.default_rng(1), il_h, ll_h, U, slack=3))

    def step():
        for t in (enc, pred, W, b):
            t.grad = None
        costs = rb.joint_rnnt_loss(enc, pred, W, b, lab, il, ll, precision="bf16", windows=win, fastemit_lambda=0.5)
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
    for _ in range(2):                                                     # eager, twice: bit-identical to the replay
        want_c = step().detach()
        torch.cuda.synchronize()
        assert torch.equal(got_c, want_c)
        for a, t in zip(got_g, (enc, pred, W, b)):
            assert torch.equal(a, t.grad)


_CHUNK_SCRIPT = """
import sys, numpy as np, torch
sys.path.insert(0, %r); sys.path.insert(0, %r)
import window_ref as wr
from test_gpu_joint import synth
from test_gpu_windows import run_joint
k = synth(5, 70, 45, 256, 192, 31, True)
win = wr.random_feasible_windows(np.random.default_rng(2), k["input_lengths"], k["label_lengths"], 45, slack=2)
import rnnt_speech_recognition_b200 as rb
vt = rb.valid_tile_count(k["input_lengths"], k["label_lengths"], win)
c, g = run_joint(k, "bf16", win, keep=bool(int(sys.argv[2])), lam=0.5, valid_tiles={"none": None, "exact": vt, "broken": vt - 1}[sys.argv[3]])
np.savez(sys.argv[1], costs=c, d_enc=g[0], d_pred=g[1], dW=g[2], db=g[3])
"""


def test_tc_windowed_multi_chunk_backward(tmp_path):
    """RNNTB200_CHUNK_MB=1 (read once per process, hence the child processes): 5 utterances in chunks of 1-2; with the
    windowed `valid_tiles` the band is one chunk again, and a promise one tile too small gives NaN costs."""
    outs = []
    small = {"RNNTB200_CHUNK_MB": "1"}
    for tag, env, keep, vt in (("one", {}, "1", "none"), ("chunked", small, "1", "none"), ("chunked_nokeep", small, "0", "none"),
                               ("bound", small, "1", "exact"), ("broken", small, "1", "broken")):
        f = str(tmp_path / (tag + ".npz"))
        subprocess.run([sys.executable, "-c", _CHUNK_SCRIPT % (ROOT, os.path.join(ROOT, "tests")), f, keep, vt], check=True,
                       env=dict(os.environ, **env), timeout=300)
        outs.append(dict(np.load(f)))
    assert np.isnan(outs.pop()["costs"]).all()
    for o in outs[1:]:
        assert np.array_equal(o["costs"], outs[0]["costs"])
        for n in ("d_enc", "d_pred"):
            assert_close(o[n], outs[0][n], rtol=0, atol=0, ntol=1e-6, what=n)
        for n in ("dW", "db"):
            assert_close(o[n], outs[0][n], rtol=0, atol=0, ntol=2e-5, what=n)


def test_op_limits_maxU_1024_and_T_2000():
    """One thread per label position at the 1024 limit, and a long utterance: costs against the reference's DP."""
    import rnnt_speech_recognition_b200 as rb
    rng = np.random.default_rng(8)
    for B, T, U, V in ((1, 40, 1024, 8), (1, 2000, 12, 8)):
        acts = rng.standard_normal((B, T, U, V)).astype(np.float32)
        labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
        il, ll = np.array([T], np.int32), np.array([U - 1], np.int32)
        win = wr.random_feasible_windows(rng, il, ll, U, slack=3)
        want_c, want_g = wr.logits_grad(acts, labels, il, ll, 0, win)
        costs, g = run_op(acts, labels, il, ll, 0, np.ones(B), torch.float32, win)
        assert_close(costs, want_c, what="costs", **fp32_tol(want_c))
        rtol, atol = op_tol(want_c, torch.float32, np.ones(B))
        rtol += ab_cell(float(want_c.max()))       # fp32 alpha/beta round-off over thousands of wavefront steps (DESIGN §4)
        assert np.all(np.abs(g - want_g) <= atol + rtol * np.abs(want_g))


def test_c3_full_size_band_of_16_frames():
    """BASELINE C3 (B=32 T=512 U=128 V=1024 H=640), windows of +-16 frames around each utterance's own alignment: against
    the chunked float64 reference with the alpha/beta term of tests/test_gpu_ref64.py; restricted costs lie between the
    unrestricted costs and -best_logp."""
    import rnnt_speech_recognition_b200 as rb
    from test_gpu_ref64 import check_tc
    B, T, U, V, H = 32, 512, 128, 1024, 640
    k = synth(B, T, U, V, H, 1234, ragged=False)
    t = [dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    al = rb.joint_rnnt_align(*t, lab, il, ll, precision="bf16")
    win = rb.alignment_windows(al.label_frames, il, ll, 16, 16)
    hwin = tuple(w.cpu().numpy() for w in win)
    vt = rb.valid_tile_count(k["input_lengths"], k["label_lengths"], hwin)
    assert vt < 0.3 * rb.valid_tile_count(k["input_lengths"], k["label_lengths"])
    del t
    costs, grads = run_joint(k, "bf16", hwin, valid_tiles=vt)
    plain, best = al.costs.cpu().numpy(), al.best_logp.cpu().numpy()
    assert (costs >= plain - 1e-5 * np.abs(plain)).all() and (costs <= -best + 1e-5 * np.abs(best)).all()
    want = wr.joint_loss_grad(dev(k["enc"]), dev(k["pred"]), dev(k["W"]), dev(k["b"]), k["labels"], k["input_lengths"],
                              k["label_lengths"], 0, hwin, np.full(B, 1.0 / B))
    check_tc(costs, grads, want, "C3 windows +-16")
