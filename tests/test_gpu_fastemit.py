"""FastEmit (`fastemit_lambda`) on the H100, on every numerical path: the fp32 loss op (vector and scalar gradient
kernels), the fp16 / bf16 loss op, the fp32 exact joint and the 16-bit tensor-core joint (keep, recompute and several
workspace chunks).

* lambda = 0 through the new C entries and keywords is bit-identical to the entries without FastEmit.
* lambda in {0.5, 2} against the float64 reference (tests/fastemit_ref.py) at each path's DESIGN §4 tolerance.  The
  same cases check sensitivity: the reference's g(lambda) - g(0) exceeds the path's tolerance at least 10-fold, and
  the GPU's g(lambda) - g(0) matches it, so a build that ignores lambda fails.
* Costs do not depend on lambda; upstream gradients are folded in; CUDA-graph replay; the train step; full C3 size.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import fastemit_ref as fe
from conftest import ROOT, assert_close, fp32_tol, golden_names, load
from test_gpu_joint import synth

pytestmark = pytest.mark.gpu

NAMES = ("d_enc", "d_pred", "dW", "db")
DT16 = {"f16": torch.float16, "bf16": torch.bfloat16}
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
LAMBDAS = (0.5, 2.0)


def dev(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


# ------------------------------------------------------------------------------------------------------ runners
def run_op(acts, labels, il, ll, blank=0, gs=None, dtype=torch.float32, offset=0, **kw):
    """rnnt_loss on `acts` (as `dtype`, placed `offset` elements past an allocation) with upstream gradients gs:
    (costs, acts.grad as float64) on the host.  kw: fastemit_lambda, when given."""
    import rnnt_speech_recognition_b200 as rb
    n = acts.size
    x = torch.empty(n + 16, dtype=dtype, device="cuda")[offset:offset + n].view(acts.shape)
    x.copy_(dev(acts, torch.float32))
    x.requires_grad_()
    B = acts.shape[0]
    gs = np.full(B, 1.0 / B) if gs is None else gs
    costs = rb.rnnt_loss(x, dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32), blank, **kw)
    (costs * dev(gs, torch.float32)).sum().backward()
    return costs.detach().cpu().numpy(), x.grad.double().cpu().numpy()


def run_joint(k, precision, gs=None, keep=None, **kw):
    import rnnt_speech_recognition_b200 as rb
    t = [dev(k[n], torch.float32).requires_grad_() for n in ("enc", "pred", "W", "b")]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    costs = rb.joint_rnnt_loss(*t, lab, il, ll, blank=int(k["blank"]), precision=precision, keep_activations=keep, **kw)
    B = costs.shape[0]
    gs = np.full(B, 1.0 / B) if gs is None else gs
    (costs * dev(gs, torch.float32)).sum().backward()
    return costs.detach().cpu().numpy(), [x.grad.double().cpu().numpy() for x in t]


def with_old_entries(fn):
    """fn() with the torch surface's calls of the three FastEmit entries routed to the entries without FastEmit
    (dropping the trailing lambda): what the library computed before FastEmit existed."""
    from rnnt_speech_recognition_b200 import _lib
    L = _lib.load()
    with pytest.MonkeyPatch.context() as mp:
        for new, old in (("rnntb200_loss_device_fastemit", L.rnntb200_loss_device),
                         ("rnntb200_loss16_backward_fastemit", L.rnntb200_loss16_backward),
                         ("rnntb200_joint_loss_backward_fastemit", L.rnntb200_joint_loss_backward)):
            mp.setattr(L, new, lambda *a, _old=old: _old(*a[:-1]))
        return fn()


# ------------------------------------------------------------------------------------------------------ tolerances
def op_tol(costs, dtype, gs):
    """(rtol, atol) of the loss op's gradients against gs * reference (DESIGN §4; tests/test_gpu_mixed_precision.py)."""
    t = fp32_tol(costs)
    if dtype == torch.float32:
        return t["rtol"], np.abs(gs)[:, None, None, None] * t["atol"]
    u = UNIT[dtype]
    return 1e-4 * (1 + u) + u, np.abs(gs)[:, None, None, None] * t["atol"] * (1 + u) + (2.0 ** -25 if dtype == torch.float16 else 0)


def check_sensitive(got, want, got0, want0, bound, what):
    """want - want0 (the reference's FastEmit change) exceeds the tolerance 10-fold somewhere, and got - got0 matches it
    at twice the tolerance (each side is within one tolerance of the reference).  bound(ref) -> element-wise bound."""
    ratio = max(np.max(np.abs(w - w0) / bound(w)) for w, w0 in zip(want, want0))
    assert ratio >= 10, (what, "FastEmit's change is not resolvable at this tolerance", ratio)
    for g, g0, w, w0, n in zip(got, got0, want, want0, what):
        d = np.abs((g - g0) - (w - w0))
        assert np.all(d <= 2 * bound(w)), (n, "g(lambda) - g(0) differs from the reference's", float(np.max(d / (2 * bound(w)))))


# ------------------------------------------------------------------------------------------------------ op cases
def op_case(name):
    if name.startswith("logits_"):
        k = load(name)
        return k["acts"], k["labels"], k["input_lengths"], k["label_lengths"], int(k["blank"])
    kind, V = name.split(":")
    V = int(V)
    rng = np.random.default_rng(31 + V)
    B, T, U = (3, 40, 33) if kind == "ragged" else (2, 10, 7)
    acts = (2.0 * rng.standard_normal((B, T, U, V))).astype(np.float32)
    labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
    il, ll = rng.integers(1, T + 1, B).astype(np.int32), rng.integers(0, U, B).astype(np.int32)
    il[0], ll[0] = T, U - 1
    if kind == "label_is_blank":
        labels[rng.random(labels.shape) < 1 / 3] = 5
        return acts, labels, il, ll, 5
    return acts, labels, il, ll, 0


OP_CASES = golden_names("logits_") + ["ragged:50", "label_is_blank:128", "v:24", "v:1024", "v:1028", "v:4096"]


@pytest.mark.parametrize("lam", LAMBDAS)
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("name", OP_CASES)
def test_op_vs_reference(name, dt, lam):
    """V = 24 / 1024 / 4096: register and two-pass vector kernels; 50, 1028 and fp32 golden shapes with V % 4 != 0:
    the scalar kernels."""
    dtype = torch.float32 if dt == "f32" else DT16[dt]
    acts, labels, il, ll, blank = op_case(name)
    B = acts.shape[0]
    x = torch.as_tensor(acts).to(dtype).double().numpy()          # the exact values the kernels see
    gs = np.linspace(0.5, 1.5, B) / B
    c, g = run_op(acts, labels, il, ll, blank, gs, dtype, fastemit_lambda=lam)
    c0, g0 = run_op(acts, labels, il, ll, blank, gs, dtype, fastemit_lambda=0.0)
    oc, og = fe.logits_grad(x, labels, il, ll, blank, lam, grad_scale=gs)
    _, og0 = fe.logits_grad(x, labels, il, ll, blank, 0.0, grad_scale=gs)
    assert np.array_equal(c, c0)                                  # the costs do not depend on lambda
    assert_close(c, oc, rtol=1e-4, atol=1e-5, what="costs")
    rtol, atol = op_tol(oc, dtype, gs)
    assert_close(g, og, rtol=rtol, atol=atol, what="grads")
    for b in range(B):
        assert not g[b, il[b]:].any() and not g[b, :, ll[b] + 1:].any()
    if not ll.any():                                              # no label arcs: FastEmit changes nothing
        assert np.array_equal(g, g0)
        return
    check_sensitive([g], [og], [g0], [og0], lambda w: atol + rtol * np.abs(w).max(), ["grads"])


@pytest.mark.parametrize("V", [64, 50])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_op_lambda_zero_is_bit_identical(dt, V):
    """The new entries at lambda = 0 (default keyword and explicit 0) against the entries without FastEmit; V = 50 and
    an unaligned buffer reach the scalar kernels."""
    dtype = torch.float32 if dt == "f32" else DT16[dt]
    acts, labels, il, ll, blank = op_case("ragged:%d" % V)
    for offset in (0, 1):
        want = with_old_entries(lambda: run_op(acts, labels, il, ll, blank, None, dtype, offset))
        got = run_op(acts, labels, il, ll, blank, None, dtype, offset)
        got0 = run_op(acts, labels, il, ll, blank, None, dtype, offset, fastemit_lambda=0.0)
        for a, b in ((got, want), (got0, want)):
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ------------------------------------------------------------------------------------------------------ joint cases
TC_COST_RTOL, TC_NTOL = 2e-4, 1e-2


def joint_case(name):
    if name.startswith("joint_"):
        return load(name)
    B, T, U, V, H, seed, ragged, blank = dict(
        small=(2, 20, 8, 64, 64, 0, False, 0), ragged=(3, 37, 19, 128, 128, 1, True, 0),
        wide=(2, 33, 40, 512, 640, 4, True, 0), v1024=(2, 12, 9, 1024, 128, 5, True, 0),
        v4096=(2, 8, 6, 4096, 64, 6, True, 0), t1=(3, 1, 5, 64, 128, 21, False, 0), blank5=(2, 12, 6, 128, 64, 22, False, 5),
        blank_last=(2, 12, 6, 128, 64, 23, False, 127), label_is_blank=(2, 12, 6, 128, 64, 24, False, 5))[name]
    k = synth(B, T, U, V, H, seed, ragged)
    rng = np.random.default_rng(seed)
    if blank or name == "t1":
        k["labels"] = rng.choice([v for v in range(V) if v != blank], size=(B, U - 1)).astype(np.int32)
        if name == "label_is_blank":
            k["labels"][rng.random(k["labels"].shape) < 1 / 3] = blank
        k["blank"] = np.int32(blank)
    return k


TC_CASES = ["small", "ragged", "wide", "v1024", "v4096", "t1", "blank5", "blank_last", "label_is_blank"]


def reference(k, gs, lam):
    return fe.joint_loss_grad(*(k[n].astype(np.float64) for n in ("enc", "pred", "W", "b")), k["labels"],
                              k["input_lengths"], k["label_lengths"], int(k["blank"]), gs, lam)


@pytest.mark.parametrize("lam", LAMBDAS)
@pytest.mark.parametrize("name", golden_names("joint_") + ["ragged", "label_is_blank"])
def test_fp32_joint_vs_reference(name, lam):
    k = joint_case(name)
    B = k["enc"].shape[0]
    gs = np.linspace(0.5, 1.5, B)
    c, g = run_joint(k, "fp32", gs, fastemit_lambda=lam)
    c0, g0 = run_joint(k, "fp32", gs, fastemit_lambda=0.0)
    o, o0 = reference(k, gs, lam), reference(k, gs, 0.0)
    assert np.array_equal(c, c0)
    assert_close(c, o["costs"], rtol=1e-5, atol=1e-4, what="costs")
    for x, n in zip(g, NAMES):
        assert_close(x, o[n], rtol=1e-4, atol=1e-6, ntol=1e-5, what=n)
    check_sensitive(g, [o[n] for n in NAMES], g0, [o0[n] for n in NAMES],
                    lambda w: 1e-6 + (1e-5 + 1e-4) * np.abs(w).max(), NAMES)


@pytest.mark.parametrize("keep", [True, False])
@pytest.mark.parametrize("lam", LAMBDAS)
@pytest.mark.parametrize("name", TC_CASES)
def test_tc_joint_vs_reference(name, lam, keep):
    k = joint_case(name)
    B = k["enc"].shape[0]
    gs = np.linspace(0.5, 1.5, B)
    c, g = run_joint(k, "bf16", gs, keep, fastemit_lambda=lam)
    c0, g0 = run_joint(k, "bf16", gs, keep, fastemit_lambda=0.0)
    o, o0 = reference(k, gs, lam), reference(k, gs, 0.0)
    assert np.array_equal(c, c0)
    assert_close(c, o["costs"], rtol=TC_COST_RTOL, atol=1e-3, what="costs")
    for x, n in zip(g, NAMES):
        assert_close(x, o[n], rtol=0, atol=0, ntol=TC_NTOL, what=n)
        assert np.linalg.norm(x) >= 0.5 * np.linalg.norm(o[n]), n
    for b in range(B):
        assert not g[0][b, k["input_lengths"][b]:].any() and not g[1][b, k["label_lengths"][b] + 1:].any()
    check_sensitive(g, [o[n] for n in NAMES], g0, [o0[n] for n in NAMES], lambda w: TC_NTOL * np.abs(w).max(), NAMES)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_empty_transcripts_are_unaffected(precision):
    """U = 1: no label arcs, so FastEmit changes nothing, bit for bit."""
    k = synth(3, 9, 2, 64, 64, 25, ragged=False)
    k["pred"], k["labels"], k["label_lengths"] = k["pred"][:, :1].copy(), np.zeros((3, 0), np.int32), np.zeros(3, np.int32)
    c0, g0 = run_joint(k, precision, fastemit_lambda=0.0)
    c1, g1 = run_joint(k, precision, fastemit_lambda=2.0)
    assert np.array_equal(c0, c1)
    if precision == "bf16":                   # the fp32 path sums with float atomics
        for a, b in zip(g0, g1):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("precision,keep", [("fp32", None), ("bf16", True), ("bf16", False)])
def test_joint_lambda_zero_is_bit_identical(precision, keep):
    k = joint_case("ragged")
    want = with_old_entries(lambda: run_joint(k, precision, keep=keep))
    got = run_joint(k, precision, keep=keep)
    got0 = run_joint(k, precision, keep=keep, fastemit_lambda=0.0)
    for a in (got, got0):
        assert np.array_equal(a[0], want[0])
        for x, y, n in zip(a[1], want[1], NAMES):
            if precision == "bf16":
                assert np.array_equal(x, y), n
            else:                             # d_enc / d_pred / dW of the fp32 path are float-atomic sums
                assert_close(x, y, rtol=1e-5, atol=1e-7, what=n)


def _dump(tmp_path, tag, env, *extra):
    f = str(tmp_path / (tag + ".npz"))
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "joint_dump.py"), f, "5", "70", "45", "256", "192", "31",
                    "1", "1"] + list(extra), check=True, env=dict(os.environ, **env), timeout=300)
    return dict(np.load(f))


def test_multi_chunk_backward(tmp_path):
    """Several workspace chunks (RNNTB200_CHUNK_MB=1, read once per process): lambda = 0 bit-identical to the plain call,
    and lambda = 0.5 equal to the single-chunk run up to the summation order of dW / db."""
    chunked = {"RNNTB200_CHUNK_MB": "1"}
    plain = _dump(tmp_path, "plain", chunked)
    zero = _dump(tmp_path, "zero", chunked, "0", "0.0")
    for n in ("costs",) + NAMES:
        assert np.array_equal(zero[n], plain[n]), n
    one = _dump(tmp_path, "one", {}, "0", "0.5")
    many = _dump(tmp_path, "many", chunked, "0", "0.5")
    assert np.array_equal(many["costs"], one["costs"]) and np.array_equal(many["costs"], plain["costs"])
    for n in ("d_enc", "d_pred"):
        assert_close(many[n], one[n], rtol=0, atol=0, ntol=1e-6, what=n)
    for n in ("dW", "db"):
        assert_close(many[n], one[n], rtol=0, atol=0, ntol=2e-5, what=n)
    k = synth(5, 70, 45, 256, 192, 31, True)
    o, o0 = reference(k, np.full(5, 0.2), 0.5), reference(k, np.full(5, 0.2), 0.0)
    got, got0 = [many[n].astype(np.float64) for n in NAMES], [plain[n].astype(np.float64) for n in NAMES]
    for x, n in zip(got, NAMES):
        assert_close(x, o[n], rtol=0, atol=0, ntol=TC_NTOL, what=n)
    check_sensitive(got, [o[n] for n in NAMES], got0, [o0[n] for n in NAMES], lambda w: TC_NTOL * np.abs(w).max(), NAMES)


# ------------------------------------------------------------------------------------------------------ upstream gradients, graphs, train step
@pytest.mark.parametrize("path", ["f32", "bf16-op", "fp32", "bf16"])
def test_mixed_sign_and_zero_upstream_gradients(path):
    gs = np.array([1.0, -0.7, 0.0])
    if path in ("f32", "bf16-op"):
        acts, labels, il, ll, blank = op_case("ragged:64")
        dtype = torch.float32 if path == "f32" else torch.bfloat16
        x = torch.as_tensor(acts).to(dtype).double().numpy()
        _, g = run_op(acts, labels, il, ll, blank, gs, dtype, fastemit_lambda=0.5)
        oc, og = fe.logits_grad(x, labels, il, ll, blank, 0.5, grad_scale=gs)
        rtol, atol = op_tol(oc, dtype, gs)
        assert_close(g, og, rtol=rtol, atol=atol, what="grads")
        assert not g[2].any()
        return
    k = joint_case("ragged")
    _, g = run_joint(k, path, gs, fastemit_lambda=0.5)
    o = reference(k, gs, 0.5)
    for x, n in zip(g, NAMES):
        if path == "fp32":
            assert_close(x, o[n], rtol=1e-4, atol=1e-6, ntol=1e-5, what=n)
        else:
            assert_close(x, o[n], rtol=0, atol=0, ntol=TC_NTOL, what=n)
    assert not g[0][2].any() and not g[1][2].any()


def test_cuda_graph_replay_of_the_16bit_backward():
    import rnnt_speech_recognition_b200 as rb
    acts, labels, il, ll, blank = op_case("ragged:64")
    x = dev(acts, torch.float32).to(torch.bfloat16).requires_grad_()
    lab, dil, dll = dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32)
    w = torch.full((x.shape[0],), 1.0 / x.shape[0], device="cuda")

    def step():
        x.grad = None
        costs = rb.rnnt_loss(x, lab, dil, dll, blank, fastemit_lambda=0.5)
        (costs * w).sum().backward()
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
        grad = x.grad
    torch.cuda.current_stream().wait_stream(s)
    with torch.no_grad():
        x.copy_(torch.randn_like(x, dtype=torch.float32).to(torch.bfloat16) * 2)
    g.replay()
    torch.cuda.synchronize()
    got_c, got_g = out.clone(), grad.clone()
    want_c = step().detach()
    torch.cuda.synchronize()
    assert torch.equal(got_c, want_c) and torch.equal(got_g, x.grad)


def test_train_step_matches_a_manual_step():
    import copy
    import rnnt_speech_recognition_b200 as rb
    torch.manual_seed(5)
    B, T, U, P, H, V, lam = 3, 14, 5, 64, 64, 64, 0.5
    joint = rb.Joint(P, H, V, precision="bf16", fastemit_lambda=lam).cuda()
    manual = copy.deepcopy(joint)
    enc, pred = torch.randn(B, T, P, device="cuda"), torch.randn(B, U, P, device="cuda")
    labels = torch.randint(1, V, (B, U - 1), device="cuda", dtype=torch.int32)
    spec_lengths = torch.tensor([2 * T, 2 * T - 3, 2 * T - 1], device="cuda", dtype=torch.int32)
    label_lengths = torch.tensor([U - 1, U - 2, U - 1], device="cuda", dtype=torch.int32)
    loss = rb.joint_train_step(joint, torch.optim.SGD(joint.parameters(), lr=0.1), enc, pred, labels, spec_lengths,
                               label_lengths, global_batch_size=B)
    opt = torch.optim.SGD(manual.parameters(), lr=0.1)
    enc_acts, pred_acts = manual.hoist(enc, pred)
    costs = rb.joint_rnnt_loss(enc_acts, pred_acts, manual.kernel_2, manual.bias_2, labels,
                               rb.encoder_lengths(spec_lengths, 2), label_lengths, precision="bf16", fastemit_lambda=lam)
    (costs.sum() / B).backward()
    opt.step()
    assert torch.allclose(loss, costs.detach().sum() / B, rtol=1e-6)
    for a, b in zip(joint.parameters(), manual.parameters()):     # (dense1's dK1 is a float-atomic sum)
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-7)
    # lambda reached the step: the same step without FastEmit lands elsewhere
    torch.manual_seed(5)
    ref = rb.Joint(P, H, V, precision="bf16").cuda()
    rb.joint_train_step(ref, torch.optim.SGD(ref.parameters(), lr=0.1), enc, pred, labels, spec_lengths, label_lengths,
                        global_batch_size=B)
    assert not torch.allclose(ref.kernel_2, joint.kernel_2, rtol=1e-4, atol=1e-6)


# ------------------------------------------------------------------------------------------------------ full C3 size
def test_c3_full_size():
    """B=32 T=512 U=128 V=1024 H=640, lambda = 0.01.  The primary check at this size is against the float64 reference
    (tests/test_gpu_ref64.py::test_c3_fastemit_vs_float64); these are its secondary properties: softmax shift invariance, linearity of
    the gradients in lambda, and the 16-bit path against the fp32 exact path at the same lambda.  Linearity is held on
    the fp32 path against |g(lambda) - g(0)|; on the 16-bit path the change at lambda = 0.01 (about 2e-3 of |g|) is of
    the order of its bf16 rounding, so there the second difference is held to the path's Frobenius tolerance."""
    k = synth(32, 512, 128, 1024, 640, 2026, ragged=False)
    lam = 0.01
    runs = {p: [run_joint(k, p, fastemit_lambda=x) for x in (0.0, lam, 2 * lam)] for p in ("bf16", "fp32")}
    msgs, bad = [], []
    for p, ((c0, g0), (c1, g1), (c2, g2)) in runs.items():
        assert np.array_equal(c0, c1) and np.array_equal(c0, c2), p
        for a, b, c, n in zip(g0, g1, g2, NAMES):
            step, curv, norm = np.linalg.norm(b - a), np.linalg.norm(c - 2 * b + a), np.linalg.norm(b)
            msgs.append("C3 %s %s: |g(l)-g(0)|/|g(l)| = %.2e, |g(2l)-2g(l)+g(0)|/|g(l)-g(0)| = %.2e"
                        % (p, n, step / norm, curv / step))
            if not (step > 0 and (curv <= 1e-2 * step if p == "fp32" else curv <= 5e-3 * norm)):
                bad.append((p, n))
    (c16, g16), (c32, g32) = runs["bf16"][1], runs["fp32"][1]
    d_enc, d_pred, dW, db = g16
    assert abs(db.sum()) <= 1e-3 * np.abs(db).sum()
    assert np.all(np.abs(dW.sum(axis=1)) <= 1e-3 * np.abs(dW).sum(axis=1) + 1e-6)
    assert_close(c16, c32, rtol=2e-4, atol=1e-2, what="costs")
    for a, b, n in zip(g16, g32, NAMES):
        rel = np.linalg.norm(a - b) / np.linalg.norm(b)
        msgs.append("C3 %s: bf16 vs fp32 exact at lambda %.2f: %.2e" % (n, lam, rel))
        if not (np.all(np.isfinite(a)) and rel < 5e-3):
            bad.append(("bf16 vs fp32", n))
    print("\n".join(msgs))
    assert not bad, bad
