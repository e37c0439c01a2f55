"""Forced alignment (rnnt_align / joint_rnnt_align) on the H100, on every path: the fp32 loss op, the fp16 / bf16 loss
op, the fp32 exact joint and the tensor-core joint (one and several workspace chunks).

Score criterion (DESIGN §4), always required: the GPU's path, scored in float64 with the reference's log-probs, and the
reported best_logp are both within tol of the reference's best_logp, tol = rtol * |best_logp| + atol with the path's
cost tolerance.  Path identity: wherever the reference's gap to the second-best path exceeds 2 * tol, the frames equal
the reference's exactly (each side's score error is below tol, so the two paths cannot swap there).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import align_ref as ar
from conftest import golden_names, load
from test_gpu_joint import synth

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
OP_TOL = (1e-4, 1e-5)          # (rtol, atol): fp32 arithmetic on the logits as the kernels see them
TC_TOL = (2e-4, 1e-3)          # the tensor-core joint's cost tolerance


def dev(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def np_(t):
    return t.detach().cpu().numpy()


def check(al, lp, labels, il, ll, blank, tol, min_identical=0):
    """The score criterion, path identity where the gap allows it, and the frames' shape rules.  Returns how many
    utterances were held to path identity."""
    frames, best = np_(al.label_frames), np_(al.best_logp).astype(np.float64)
    ar.check_frames(frames, il, ll)
    rf, rb, gap = ar.viterbi(lp, labels, il, ll, blank)
    score = ar.path_score(lp, labels, frames, il, ll, blank)
    t = tol[0] * np.abs(rb) + tol[1]
    assert np.all(np.abs(score - rb) <= t), ("path score", score, rb, t)
    assert np.all(np.abs(best - rb) <= t), ("best_logp", best, rb, t)
    assert np.all(best <= -np_(al.costs) + t), ("best_logp above -cost", best, np_(al.costs))
    sure = gap > 2 * t
    for b in np.flatnonzero(sure):
        assert np.array_equal(frames[b], rf[b]), ("frames", b, frames[b], rf[b], gap[b], t[b])
    assert sure.sum() >= min_identical, (sure.sum(), gap, t)
    return int(sure.sum())


def arcs_only(lp_blank, lp_label):
    """A (B,T,U,2) log-prob tensor holding only the two arcs of each cell (column 0: blank, column 1: the label), with
    labels all 1 and blank 0: the reference then needs no (B,T,U,V) float64 tensor."""
    return np.stack([lp_blank, lp_label], axis=-1)


# ------------------------------------------------------------------------------------------------------ op path
def op_case(name):
    if name.startswith("logits_"):
        k = load(name)
        return k["acts"], k["labels"], k["input_lengths"], k["label_lengths"], int(k["blank"])
    kind, V = name.split(":")
    V = int(V)
    rng = np.random.default_rng(7 + V + len(kind))
    B, T, U = dict(ragged=(3, 40, 33), multiwarp=(3, 30, 200), t1=(3, 1, 9), u1=(3, 12, 1)).get(kind, (2, 10, 7))
    acts = (2.0 * rng.standard_normal((B, T, U, V))).astype(np.float32)
    blank = dict(blank5=5, blank_last=V - 1, label_is_blank=5).get(kind, 0)
    labels = rng.choice([v for v in range(V) if v != blank], size=(B, U - 1)).astype(np.int32)
    il, ll = rng.integers(1, T + 1, B).astype(np.int32), rng.integers(0, U, B).astype(np.int32)
    il[0], ll[0] = T, U - 1
    if kind == "label_is_blank":
        labels[rng.random(labels.shape) < 1 / 3] = blank
    return acts, labels, il, ll, blank


OP_CASES = golden_names("logits_") + ["ragged:50", "multiwarp:24", "t1:16", "u1:16", "blank5:32", "blank_last:40",
                                      "label_is_blank:128", "v:24", "v:1024", "v:1028", "v:4096"]


def run_op_align(acts, labels, il, ll, blank, dtype, garbage=None):
    import rnnt_speech_recognition_b200 as rb
    x = dev(acts, torch.float32).to(dtype)
    return rb.rnnt_align(x, dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32), blank)


def op_forward_costs(acts, labels, il, ll, blank, dtype):
    import rnnt_speech_recognition_b200 as rb
    with torch.no_grad():
        x = dev(acts, torch.float32).to(dtype)
        return np_(rb.rnnt_loss(x, dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32), blank))


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("name", OP_CASES)
def test_op_vs_reference(name, dt):
    """V = 24 / 1024 / 4096: register and two-pass lse kernels; 50, 1028 and the golden shapes: the scalar kernel."""
    dtype = DT[dt]
    acts, labels, il, ll, blank = op_case(name)
    x = torch.as_tensor(acts).to(dtype).double().numpy()           # the logits as the kernels see them
    al = run_op_align(acts, labels, il, ll, blank, dtype)
    assert np.array_equal(np_(al.costs), op_forward_costs(acts, labels, il, ll, blank, dtype))
    check(al, ar.log_probs(x), labels, il, ll, blank, OP_TOL)
    again = run_op_align(acts, labels, il, ll, blank, dtype)
    for a, b in zip(al, again):
        assert torch.equal(a, b)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_op_limits(dt):
    """maxU = 1024 (32 warps) and T = 2000; maxU = 1025 is rejected."""
    import rnnt_speech_recognition_b200 as rb
    dtype = DT[dt]
    for (B, T, U, V, seed) in ((2, 24, 1024, 16, 1), (2, 2000, 12, 24, 2)):
        rng = np.random.default_rng(seed)
        acts = (2.0 * rng.standard_normal((B, T, U, V))).astype(np.float32)
        labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
        il, ll = np.array([T, T - 5], np.int32), np.array([U - 1, U // 2], np.int32)
        al = run_op_align(acts, labels, il, ll, 0, dtype)
        x = torch.as_tensor(acts).to(dtype).double().numpy()
        check(al, ar.log_probs(x), labels, il, ll, 0, OP_TOL)
    x = torch.zeros(1, 2, 1025, 4, device="cuda", dtype=dtype)
    with pytest.raises(RuntimeError, match="invalid value"):
        rb.rnnt_align(x, torch.ones(1, 1024, dtype=torch.int32, device="cuda"), torch.tensor([2], dtype=torch.int32).cuda(),
                      torch.tensor([1024], dtype=torch.int32).cuda())


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_op_uniform_logits_emit_at_frame_zero(dt):
    acts = np.zeros((3, 9, 6, 40), np.float32)
    labels = np.full((3, 5), 3, np.int32)
    labels[1, ::2] = 0                                            # labels equal to blank tie the same way
    il, ll = np.array([9, 4, 1], np.int32), np.array([5, 3, 5], np.int32)
    al = run_op_align(acts, labels, il, ll, 0, DT[dt])
    f = np_(al.label_frames)
    ar.check_frames(f, il, ll)
    assert not np.where(f >= 0, f, 0).any()


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_op_garbage_in_padding_is_ignored(dt):
    dtype = DT[dt]
    acts, labels, il, ll, blank = op_case("ragged:64")
    want = run_op_align(acts, labels, il, ll, blank, dtype)
    big = 3.0e4 if dtype == torch.float16 else 1.0e30
    g = acts.copy()
    lab = labels.copy()
    for b in range(g.shape[0]):
        g[b, il[b]:] = big
        g[b, :, ll[b] + 1:] = -big
        lab[b, ll[b]:] = 7
    got = run_op_align(g, lab, il, ll, blank, dtype)
    for a, b in zip(got, want):
        assert torch.equal(a, b)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_op_planted_alignment_at_full_size(dt):
    """(32, 512, 128, 1024): label j dominates its cell at a chosen frame f_j and blank dominates every other cell, so
    the all-dominant path is the best one by a wide margin and its frames are exact."""
    import rnnt_speech_recognition_b200 as rb
    B, T, U, V = 32, 512, 128, 1024
    g = torch.Generator(device="cuda").manual_seed(11)
    lab = torch.randint(1, V, (B, U - 1), generator=g, device="cuda", dtype=torch.int32)
    il = torch.randint(T // 2, T + 1, (B,), generator=g, device="cuda", dtype=torch.int32)
    ll = torch.randint(U // 2, U, (B,), generator=g, device="cuda", dtype=torch.int32)
    il[0], ll[0] = T, U - 1
    frames = torch.sort(torch.randint(0, T, (B, U - 1), generator=g, device="cuda"), dim=1).values
    frames = torch.minimum(frames, (il - 1)[:, None].long())
    x = 0.1 * torch.randn(B, T, U, V, generator=g, device="cuda")
    x[..., 0] += 8.0                                              # blank dominates ...
    bi, ui = torch.meshgrid(torch.arange(B, device="cuda"), torch.arange(U - 1, device="cuda"), indexing="ij")
    m = ui < ll[:, None]                                          # ... except where label j < U_b - 1 is planted
    x[bi[m], frames[m], ui[m], 0] -= 8.0
    x[bi[m], frames[m], ui[m], lab.long()[m]] += 8.0
    x = x.to(DT[dt])
    al = rb.rnnt_align(x, lab, il, ll)
    want = torch.where(ui < ll[:, None], frames, -1).to(torch.int32)
    assert torch.equal(al.label_frames, want)
    with torch.no_grad():
        assert torch.equal(al.costs, rb.rnnt_loss(x, lab, il, ll))
    assert bool((al.best_logp <= -al.costs).all())


# ------------------------------------------------------------------------------------------------------ joint paths
def joint_case(name):
    if name.startswith("joint_"):
        return load(name)
    B, T, U, V, H, seed, ragged, blank = dict(
        small=(2, 20, 8, 64, 64, 0, False, 0), ragged=(3, 37, 19, 128, 128, 1, True, 0),
        wide=(2, 33, 40, 512, 640, 4, True, 0), multiwarp=(2, 12, 150, 64, 64, 8, True, 0),
        v1024=(2, 12, 9, 1024, 128, 5, True, 0), v4096=(2, 8, 6, 4096, 64, 6, True, 0),
        t1=(3, 1, 5, 64, 128, 21, False, 0), u1=(3, 9, 1, 64, 64, 25, False, 0),
        blank5=(2, 12, 6, 128, 64, 22, False, 5), blank_last=(2, 12, 6, 128, 64, 23, False, 127),
        label_is_blank=(2, 12, 6, 128, 64, 24, False, 5))[name]
    k = synth(B, T, U, V, H, seed, ragged)
    rng = np.random.default_rng(seed)
    k["W"] *= 3.0                                                 # sharper posteriors: most decisions far from a tie
    if blank or name == "t1":
        k["labels"] = rng.choice([v for v in range(V) if v != blank], size=(B, U - 1)).astype(np.int32)
        if name == "label_is_blank":
            k["labels"][rng.random(k["labels"].shape) < 1 / 3] = blank
        k["blank"] = np.int32(blank)
    return k


JOINT_CASES = ["small", "ragged", "wide", "multiwarp", "v1024", "v4096", "t1", "u1", "blank5", "blank_last",
               "label_is_blank"]


def run_joint_align(k, precision, valid_tiles=None):
    import rnnt_speech_recognition_b200 as rb
    t = [dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    al = rb.joint_rnnt_align(*t, lab, il, ll, blank=int(k["blank"]), precision=precision, valid_tiles=valid_tiles)
    with torch.no_grad():
        c = rb.joint_rnnt_loss(*t, lab, il, ll, blank=int(k["blank"]), precision=precision, valid_tiles=valid_tiles)
    return al, np_(c)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", golden_names("joint_") + JOINT_CASES)
def test_joint_vs_reference(name, precision):
    k = joint_case(name)
    if precision == "bf16" and k["W"].shape[1] % 64:
        pytest.skip("the tensor-core path needs V % 64 == 0")
    lp = ar.joint_log_probs(k["enc"], k["pred"], k["W"], k["b"])
    al, costs = run_joint_align(k, precision)
    assert np.array_equal(np_(al.costs), costs)
    n = check(al, lp, k["labels"], k["input_lengths"], k["label_lengths"], int(k["blank"]),
              OP_TOL if precision == "fp32" else TC_TOL)
    if name in ("ragged", "wide", "multiwarp", "small"):
        assert n >= 1                                             # the frames were held to the reference somewhere
    again, _ = run_joint_align(k, precision)
    for a, b in zip(al, again):
        assert torch.equal(a, b)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_joint_uniform_logits_emit_at_frame_zero(precision):
    k = synth(3, 20, 7, 64, 64, 3, ragged=True)
    k["W"][:] = 0.0
    k["b"][:] = 0.5
    al, _ = run_joint_align(k, precision)
    f = np_(al.label_frames)
    ar.check_frames(f, k["input_lengths"], k["label_lengths"])
    assert not np.where(f >= 0, f, 0).any()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_joint_garbage_in_padding_is_ignored(precision):
    k = joint_case("ragged")
    want, _ = run_joint_align(k, precision)
    g = {n: v.copy() for n, v in k.items()}
    for b in range(g["enc"].shape[0]):
        g["enc"][b, k["input_lengths"][b]:] = 1e30
        g["pred"][b, k["label_lengths"][b] + 1:] = -1e30
        g["labels"][b, k["label_lengths"][b]:] = 3
    got, _ = run_joint_align(g, precision)
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_joint_module_align():
    import rnnt_speech_recognition_b200 as rb
    torch.manual_seed(3)
    B, T, U, P, H, V = 3, 14, 5, 64, 64, 64
    joint = rb.Joint(P, H, V, precision="bf16", fastemit_lambda=0.5).cuda()
    enc, pred = torch.randn(B, T, P, device="cuda"), torch.randn(B, U, P, device="cuda")
    labels = torch.randint(1, V, (B, U - 1), device="cuda", dtype=torch.int32)
    il = torch.tensor([T, T - 3, 2], device="cuda", dtype=torch.int32)
    ll = torch.tensor([U - 1, 2, U - 1], device="cuda", dtype=torch.int32)
    al = joint.align(enc, pred, labels, il, ll)
    assert not al.label_frames.requires_grad and not al.best_logp.requires_grad
    with torch.no_grad():
        costs = joint.loss(enc, pred, labels, il, ll)
        e, p = joint.hoist(enc, pred)
        direct = rb.joint_rnnt_align(e, p, joint.kernel_2, joint.bias_2, labels, il, ll, precision="bf16")
    assert torch.equal(al.costs, costs)
    for a, b in zip(al, direct):
        assert torch.equal(a, b)
    # 16-bit inputs are cast at the boundary
    half = rb.joint_rnnt_align(e.bfloat16(), p.bfloat16(), joint.kernel_2, joint.bias_2, labels, il, ll)
    ar.check_frames(np_(half.label_frames), np_(il), np_(ll))


# ------------------------------------------------------------------------------------------------------ graphs, chunks, tile bound
def test_cuda_graph_replay_is_bit_identical():
    import rnnt_speech_recognition_b200 as rb
    acts, labels, il, ll, blank = op_case("ragged:64")
    x = dev(acts, torch.float32)
    lab, dil, dll = dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32)
    k = joint_case("ragged")
    t = [dev(k[n], torch.float32) for n in ("enc", "pred", "W", "b")]
    jl, jil, jll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))

    def step():
        return (rb.rnnt_align(x, lab, dil, dll, blank), rb.rnnt_align(x.bfloat16(), lab, dil, dll, blank),
                rb.joint_rnnt_align(*t, jl, jil, jll, precision="bf16"))

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = step()
    torch.cuda.current_stream().wait_stream(s)
    x.copy_(torch.randn_like(x) * 2)
    t[0].copy_(torch.randn_like(t[0]))
    g.replay()
    torch.cuda.synchronize()
    got = [[v.clone() for v in o] for o in out]
    want = step()
    torch.cuda.synchronize()
    for go, wo in zip(got, want):
        for a, b in zip(go, wo):
            assert torch.equal(a, b)


_CHILD = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
import rnnt_speech_recognition_b200 as rb
k = dict(np.load(sys.argv[2]))
t = [torch.as_tensor(k[n]).cuda() for n in ("enc", "pred", "W", "b")]
lab, il, ll = (torch.as_tensor(k[n]).cuda() for n in ("labels", "input_lengths", "label_lengths"))
vt = int(k["vt"]) or None
al = rb.joint_rnnt_align(*t, lab, il, ll, precision="bf16", valid_tiles=vt)
np.savez(sys.argv[3], label_frames=al.label_frames.cpu().numpy(), best_logp=al.best_logp.cpu().numpy(),
         costs=al.costs.cpu().numpy())
"""


def _child(tmp_path, k, vt, tag, env):
    import rnnt_speech_recognition_b200 as rb
    inp, out = str(tmp_path / "in.npz"), str(tmp_path / (tag + ".npz"))
    np.savez(inp, vt=np.int64(vt or 0), **{n: k[n] for n in ("enc", "pred", "W", "b", "labels", "input_lengths", "label_lengths")})
    subprocess.run([sys.executable, "-c", _CHILD, os.path.dirname(os.path.dirname(rb.__file__)), inp, out], check=True,
                   env=dict(os.environ, **env), timeout=300)
    return dict(np.load(out))


def test_multi_chunk_workspace_and_tile_bound(tmp_path):
    """RNNTB200_CHUNK_MB=1 (several workspace chunks, read once per process) gives the single-chunk results bit for
    bit, with and without a valid_tiles bound.  There the bound sizes the workspace (the padded batch does not fit one
    chunk), so a broken one gives NaN costs and best_logp and frames of -1."""
    import rnnt_speech_recognition_b200 as rb
    k = synth(5, 70, 45, 256, 192, 31, True)
    k["W"] *= 3.0
    al, _ = run_joint_align(k, "bf16")
    lp = ar.joint_log_probs(k["enc"], k["pred"], k["W"], k["b"])
    check(al, lp, k["labels"], k["input_lengths"], k["label_lengths"], 0, TC_TOL, min_identical=1)
    vt = rb.valid_tile_count(k["input_lengths"], k["label_lengths"])
    for env, bound in (({"RNNTB200_CHUNK_MB": "1"}, None), ({"RNNTB200_CHUNK_MB": "1"}, vt), ({}, vt)):
        got = _child(tmp_path, k, bound, "run", env)
        for n, v in zip(("label_frames", "best_logp", "costs"), al):
            assert np.array_equal(got[n], np_(v)), (env, bound, n)
    bad = _child(tmp_path, k, 1, "bad", {"RNNTB200_CHUNK_MB": "1"})
    assert np.isnan(bad["costs"]).all() and np.isnan(bad["best_logp"]).all()
    assert (bad["label_frames"] == -1).all()


def c5_like(B, V, H, seed):
    """Ragged batch of C5's shape family (BASELINE C5: T_b in [100, 1600], U_b in [10, 200], V = 4096, H = 640),
    scaled down in B and T so the float64 reference stays affordable."""
    rng = np.random.default_rng(seed)
    il = rng.integers(100, 400, B).astype(np.int32)
    ll = rng.integers(10, 120, B).astype(np.int32)
    T, U = int(il.max()), int(ll.max()) + 1
    k = dict(enc=rng.standard_normal((B, T, H)).astype(np.float32), pred=rng.standard_normal((B, U, H)).astype(np.float32),
             W=(3.0 * rng.standard_normal((H, V)) / np.sqrt(H)).astype(np.float32),
             b=(0.1 * rng.standard_normal(V)).astype(np.float32), labels=rng.integers(1, V, (B, U - 1)).astype(np.int32),
             blank=np.int32(0), input_lengths=il, label_lengths=ll)
    return k


def materialised_arcs(k, b):
    """float64 log-probs of utterance b's two arcs per cell, from its fp32 logits materialised by joint_logits."""
    import rnnt_speech_recognition_b200 as rb
    T, U = int(k["input_lengths"][b]), int(k["label_lengths"][b]) + 1
    with torch.no_grad():
        x = rb.joint_logits(dev(k["enc"][b:b + 1, :T]), dev(k["pred"][b:b + 1, :U]), dev(k["W"]), dev(k["b"]))[0]
        lse = torch.logsumexp(x.double(), dim=-1)
        blank = int(k["blank"])
        lpb = x[..., blank].double() - lse
        lab = dev(np.concatenate([k["labels"][b, :U - 1], [blank]]).astype(np.int64))
        lpl = torch.gather(x.double(), 2, lab[None, :, None].expand(T, U, 1))[..., 0] - lse
    return lpb.cpu().numpy(), lpl.cpu().numpy()


def check_against_materialised(k, als, utts):
    """Per utterance: both alignments against the Viterbi path of the fp32 materialised logits (arcs only), with the
    tensor-core tolerance.  Returns how many (utterance, path) pairs were held to path identity."""
    n = 0
    for b in utts:
        T, U = int(k["input_lengths"][b]), int(k["label_lengths"][b]) + 1
        lpb, lpl = materialised_arcs(k, b)
        lp = arcs_only(lpb, lpl)[None]
        lab, il, ll = np.ones((1, U - 1), np.int32), np.array([T], np.int32), np.array([U - 1], np.int32)
        for al in als:
            one = type(al)(al.label_frames[b:b + 1, :U - 1], al.best_logp[b:b + 1], al.costs[b:b + 1])
            n += check(one, lp, lab, il, ll, 0, TC_TOL)
    return n


def test_c5_shaped_ragged_batch_with_valid_tiles():
    import rnnt_speech_recognition_b200 as rb
    k = c5_like(6, 4096, 640, 55)
    vt = rb.valid_tile_count(k["input_lengths"], k["label_lengths"])
    al, costs = run_joint_align(k, "bf16", valid_tiles=vt)
    plain, _ = run_joint_align(k, "bf16")
    assert np.array_equal(np_(al.costs), costs)
    for a, b in zip(al, plain):
        assert torch.equal(a, b)
    ar.check_frames(np_(al.label_frames), k["input_lengths"], k["label_lengths"])
    check_against_materialised(k, [al], range(6))


def test_c3_full_size_tensor_core_against_fp32_exact():
    """B=32 T=512 U=128 V=1024 H=640: for a few utterances, the tensor-core and the fp32 exact alignments against the
    Viterbi path of that utterance's materialised fp32 logits, and against each other."""
    k = synth(32, 512, 128, 1024, 640, 2026, ragged=False)
    k["W"] *= 3.0
    tc, tc_costs = run_joint_align(k, "bf16")
    ex, ex_costs = run_joint_align(k, "fp32")
    assert np.array_equal(np_(tc.costs), tc_costs) and np.array_equal(np_(ex.costs), ex_costs)
    for al in (tc, ex):
        ar.check_frames(np_(al.label_frames), k["input_lengths"], k["label_lengths"])
    n = check_against_materialised(k, [tc, ex], (0, 13, 31))
    print("C3: %d of 6 (utterance, path) pairs held to path identity" % n)
