"""Mixed-precision training on the H100: the native float16 / bfloat16 loss op against the fp64 oracle, its torch
surface and CUDA-graph capture, and 16-bit inputs on the joint path (cast to float32 at the boundary).

Tolerance of the 16-bit op (DESIGN.md 4).  Its arithmetic is the fp32 op's, run on the exactly widened 16-bit logits;
the only new error is the one rounding of each gradient to 16 bits, at most u = 2^-8 (bf16) or 2^-11 (fp16) relative,
or 2^-25 absolute among fp16 subnormals.  So against g_b times the oracle's gradient of the same 16-bit logits:
    rtol = 1e-4 (1 + u) + u,   atol = |g_b| fp32_tol(costs).atol (1 + u)  (+ 2^-25 for fp16),
costs rtol 1e-4, padded cells exactly 0."""

import numpy as np
import pytest
import torch

from conftest import assert_close, fp32_tol, golden_names, load

pytestmark = pytest.mark.gpu

DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}


def dev(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def to16(acts, dtype, offset=0):
    """16-bit device copy of `acts`, placed `offset` elements past a fresh allocation."""
    n = acts.size
    x = torch.empty(n + 16, dtype=dtype, device="cuda")[offset:offset + n].view(acts.shape)
    x.copy_(dev(acts, torch.float32))
    return x


def run16(x, labels, il, ll, blank, gs):
    """rnnt_loss on 16-bit x with upstream gradients gs: (costs, acts.grad) as numpy."""
    import rnnt_speech_recognition_b200 as rb
    x = x.detach().requires_grad_()
    costs = rb.rnnt_loss(x, dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32), blank)
    assert costs.dtype == torch.float32 and costs.shape == (x.shape[0],)
    (costs * dev(gs, torch.float32)).sum().backward()
    assert x.grad.dtype == x.dtype
    return costs.detach().cpu().numpy(), x.grad.float().cpu().numpy()


def check16(oracle, x, labels, il, ll, blank=0, gs=None):
    """The 16-bit op on x against the oracle on x's exact values; returns (costs, grads, oracle grads * gs)."""
    B = x.shape[0]
    gs = np.full(B, 1.0 / B) if gs is None else np.asarray(gs, np.float64)
    oc, og = oracle.rnnt_logits_grad(x.double().cpu().numpy(), labels, il, ll, blank)
    costs, g = run16(x, labels, il, ll, blank, gs)
    assert_close(costs, oc, rtol=1e-4, atol=1e-5, what="costs")
    u = UNIT[x.dtype]
    want = og * gs[:, None, None, None]
    atol = np.abs(gs)[:, None, None, None] * fp32_tol(oc)["atol"] * (1 + u) + (2.0 ** -25 if x.dtype == torch.float16 else 0)
    assert_close(g, want, rtol=1e-4 * (1 + u) + u, atol=atol, what="grads")
    for b in range(B):                                   # padded cells exactly 0
        assert not g[b, il[b]:].any() and not g[b, :, ll[b] + 1:].any()
    return costs, g, want


def random_case(B, T, U, V, seed, spread=2.0):
    rng = np.random.default_rng(seed)
    acts = (spread * rng.standard_normal((B, T, U, V))).astype(np.float32)
    labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
    il, ll = rng.integers(1, T + 1, B).astype(np.int32), rng.integers(0, U, B).astype(np.int32)
    il[0], ll[0] = T, U - 1
    return acts, labels, il, ll


# ------------------------------------------------------------------------------------- the 16-bit op vs the oracle
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("name", golden_names("logits_"))
def test_golden_logits(oracle, name, dt):
    """blank != 0, U = 1 and T = 1 among them."""
    k = load(name)
    check16(oracle, to16(k["acts"], DTYPES[dt]), k["labels"], k["input_lengths"], k["label_lengths"], int(k["blank"]))


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("B,T,U,V,seed", [(3, 40, 33, 50, 0), (2, 70, 130, 24, 1), (1, 5, 257, 16, 3)])
def test_ragged_multi_warp_wavefront(oracle, B, T, U, V, seed, dt):
    acts, labels, il, ll = random_case(B, T, U, V, seed)
    check16(oracle, to16(acts, DTYPES[dt]), labels, il, ll)


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("blank", [0, 5, 127])
def test_labels_equal_to_blank(oracle, blank, dt):
    acts, labels, il, ll = random_case(3, 16, 10, 128, 404)
    rng = np.random.default_rng(405)
    labels[rng.random(labels.shape) < 1 / 3] = blank
    assert (labels[0] == blank).sum() >= 2
    check16(oracle, to16(acts, DTYPES[dt]), labels, il, ll, blank)


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("V", [24, 50, 1024, 1028, 2048, 2056, 4096])
def test_vocabulary_sizes(oracle, V, dt):
    """50, 1028: the scalar kernels (V % 8 != 0); 24 ... 2048: rows held in registers; 2056, 4096: two passes."""
    acts, labels, il, ll = random_case(2, 10, 7, V, 500 + V)
    check16(oracle, to16(acts, DTYPES[dt]), labels, il, ll)


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("V", [128, 2048])
def test_unaligned_buffer(oracle, V, dt):
    """acts one element (2 bytes) past a 16-byte boundary: the scalar kernels, against the oracle and the aligned call."""
    acts, labels, il, ll = random_case(3, 12, 9, V, 600 + V)
    x0, x1 = to16(acts, DTYPES[dt]), to16(acts, DTYPES[dt], offset=1)
    assert x1.data_ptr() % 16 != 0 and torch.equal(x0, x1)
    c0, g0, _ = check16(oracle, x0, labels, il, ll)
    c1, g1, _ = check16(oracle, x1, labels, il, ll)
    assert_close(c1, c0, rtol=1e-5, atol=1e-4, what="costs")


SCALES = {"1/B": lambda B: np.full(B, 1.0 / B), "2^16/B": lambda B: np.full(B, 2.0 ** 16 / B),
          "mixed-sign": lambda B: np.array([1.0, -0.7, 0.4]), "one-zero": lambda B: np.array([0.8, 0.0, 1.2])}


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("scale", list(SCALES))
def test_upstream_gradients(oracle, scale, dt):
    acts, labels, il, ll = random_case(3, 20, 12, 512, 700, spread=4.0)
    gs = SCALES[scale](3)
    _, g, want = check16(oracle, to16(acts, DTYPES[dt]), labels, il, ll, gs=gs)
    for b in np.flatnonzero(gs == 0):                    # a zero upstream gradient gives exactly zero gradients
        assert not g[b].any()
    if dt == "f16" and scale == "2^16/B":
        # entries an unscaled (1/B) fp16 gradient would flush to 0 come out non-zero once the loss scale is folded in
        unscaled = np.abs(want) * 2.0 ** -16
        tiny = (unscaled < 2.0 ** -25) & (np.abs(want) > 2.0 ** -20)
        assert tiny.sum() > 100, tiny.sum()
        assert (g[tiny] != 0).all()


# ------------------------------------------------------------------------------------------------- torch surface
@pytest.mark.parametrize("dt", list(DTYPES))
def test_torch_surface(dt):
    """rnnt_loss, torch_rnnt_loss (none / sum / mean), RNNTLoss and get_loss_fn on 16-bit acts agree with the fp32 op on
    acts.float(); costs are float32 and acts.grad has acts' dtype."""
    import rnnt_speech_recognition_b200 as rb
    dtype = DTYPES[dt]
    acts, labels, il, ll = random_case(3, 16, 9, 256, 800)
    il[:], ll[:] = 16, 8                                 # torch_rnnt_loss checks max lengths against the shape
    x16 = to16(acts, dtype)
    lab, d_il, d_ll = dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32)
    u = UNIT[dtype]

    def compare(fn, reduction_scale):
        a = x16.detach().clone().requires_grad_()
        f = x16.detach().float().requires_grad_()
        c16, c32 = fn(a), fn(f)
        assert c16.dtype == torch.float32 and c16.shape == c32.shape
        c16.sum().backward()
        c32.sum().backward()
        assert a.grad.dtype == dtype
        assert_close(c16.detach().cpu().numpy(), c32.detach().cpu().numpy(), rtol=1e-4, atol=1e-5, what="costs")
        cref = fn(f.detach()).detach().cpu().numpy()
        atol = reduction_scale * fp32_tol(cref)["atol"] * (1 + u) + (2.0 ** -25 if dtype == torch.float16 else 0)
        assert_close(a.grad.float().cpu().numpy(), f.grad.cpu().numpy(), rtol=1e-4 * (1 + u) + u, atol=atol, what="grads")

    compare(lambda a: rb.rnnt_loss(a, lab, d_il, d_ll), 1.0)
    for red, s in (("none", 1.0), ("sum", 1.0), ("mean", 1.0 / 3)):
        compare(lambda a: rb.torch_rnnt_loss(a, lab, d_il, d_ll, reduction=red), s)
        compare(lambda a: rb.RNNTLoss(reduction=red)(a, lab, d_il, d_ll), s)
    loss_fn = rb.get_loss_fn(2)
    compare(lambda a: loss_fn(lab.long(), a, 2 * d_il, d_ll.long()), 1.0)


def test_other_dtypes_still_rejected():
    import rnnt_speech_recognition_b200 as rb
    lab = torch.ones(1, 2, dtype=torch.int32, device="cuda")
    il, ll = torch.tensor([2], dtype=torch.int32, device="cuda"), torch.tensor([2], dtype=torch.int32, device="cuda")
    with pytest.raises(TypeError):
        rb.rnnt_loss(torch.zeros(1, 2, 3, 4, dtype=torch.float64, device="cuda"), lab, il, ll)


@pytest.mark.parametrize("dt", list(DTYPES))
def test_cuda_graph_capture(dt):
    """Forward + backward of the 16-bit op captured into a CUDA graph and replayed: identical to eager runs, on the
    captured inputs and after new values are copied into them."""
    import rnnt_speech_recognition_b200 as rb
    dtype = DTYPES[dt]
    acts, labels, il, ll = random_case(2, 24, 12, 256, 900)
    acts2 = random_case(2, 24, 12, 256, 901)[0]
    lab, d_il, d_ll = dev(labels, torch.int32), dev(il, torch.int32), dev(ll, torch.int32)
    w = torch.tensor([0.5, 2.0], device="cuda")

    def step(x):
        costs = rb.rnnt_loss(x, lab, d_il, d_ll)
        gx, = torch.autograd.grad((costs * w).sum(), x)
        return costs, gx

    want1, want2 = (step(to16(a, dtype).requires_grad_()) for a in (acts, acts2))
    # the captured leaf is first used on the side stream, so its gradient accumulator belongs to the capture's stream
    x = to16(acts, dtype).requires_grad_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c_s, g_s = step(x)
    for a, (wc, wg) in ((acts, want1), (acts2, want2)):
        with torch.no_grad():
            x.copy_(to16(a, dtype))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(c_s, wc) and torch.equal(g_s, wg)


# ----------------------------------------------------------------------------------------------- the joint path
def synth(B, T, U, V, H, seed):
    from test_gpu_joint import synth as s
    return s(B, T, U, V, H, seed, ragged=True)


NAMES = ("enc", "pred", "W", "b")


def joint_run(k, precision, cast):
    """joint_rnnt_loss with the inputs named in `cast` given as (dtype) tensors; returns costs and the four gradients."""
    import rnnt_speech_recognition_b200 as rb
    t = [dev(k[n], torch.float32).to(cast.get(n, torch.float32)).requires_grad_() for n in NAMES]
    lab, il, ll = (dev(k[n], torch.int32) for n in ("labels", "input_lengths", "label_lengths"))
    costs = rb.joint_rnnt_loss(*t, lab, il, ll, blank=int(k["blank"]), precision=precision)
    assert costs.dtype == torch.float32
    (costs * torch.linspace(0.5, 1.5, costs.shape[0], device="cuda")).sum().backward()
    for x in t:
        assert x.grad.dtype == x.dtype
    return costs.detach(), [x.grad for x in t]


def ulp16_close(a, b, what):
    """Two 16-bit tensors from fp32 results that differ by float-atomic ordering: at most one 16-bit ulp apart, plus the
    fp32 path's norm-wise run-to-run variation (DESIGN.md 4: relative 1e-6)."""
    a, b = a.double(), b.double()
    ulp = b.abs() * (2.0 ** -7 if what[1] == torch.bfloat16 else 2.0 ** -10) + 2.0 ** -24
    bad = (a - b).abs() > 2 * ulp + 1e-6 * b.abs().max()
    assert not bad.any(), (what, int(bad.sum()))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("name", NAMES)
def test_joint_loss_16bit_input(name, dt, precision):
    """One input in 16 bits at a time, against the fp32 run on the same values upcast, each gradient cast to its input's
    dtype.  The tensor-core path is deterministic: bit-identical.  The fp32 path sums d_enc, d_pred, dW and db with float
    atomics: costs bit-identical, gradients within that run-to-run variation."""
    dtype = DTYPES[dt]
    k = synth(3, 20, 9, 128, 64, 11)
    k[name] = torch.as_tensor(k[name]).to(dtype).float().numpy()          # values exactly representable in 16 bits
    c16, g16 = joint_run(k, precision, {name: dtype})
    c32, g32 = joint_run(k, precision, {})
    want = [g.to(dtype) if n == name else g for g, n in zip(g32, NAMES)]
    assert torch.equal(c16, c32)
    for g, w, n in zip(g16, want, NAMES):
        assert g.dtype == w.dtype
        if precision == "bf16":
            assert torch.equal(g, w), n
        elif g.dtype == torch.float32:
            assert (g - w).norm() <= 1e-6 * w.norm(), n
        else:
            ulp16_close(g, w, (n, dtype))


@pytest.mark.parametrize("dt", list(DTYPES))
def test_dense1_logits_and_step_16bit_inputs(dt):
    """dense1 output and dX, joint_logits and joint_step: bit-identical to the upcast fp32 run; dense1's dK1 (float
    atomics) within one 16-bit ulp; db1 bit-identical."""
    import rnnt_speech_recognition_b200 as rb
    dtype = DTYPES[dt]
    torch.manual_seed(5)
    x32 = torch.randn(3, 7, 48, device="cuda").to(dtype).float()
    K32 = (torch.randn(48, 64, device="cuda") / 8).to(dtype).float()
    b32 = torch.randn(64, device="cuda").to(dtype).float()
    dout = torch.randn(3, 7, 64, device="cuda")
    res = {}
    for key, cast in (("16", dtype), ("32", torch.float32)):
        x, K, b = (t.to(cast).requires_grad_() for t in (x32, K32, b32))
        out = rb.dense1(x, K, b)
        assert out.dtype == torch.float32
        out.backward(dout)
        res[key] = (out.detach(), x.grad, K.grad, b.grad)
    (o16, dx16, dk16, db16), (o32, dx32, dk32, db32) = res["16"], res["32"]
    assert torch.equal(o16, o32) and torch.equal(dx16, dx32.to(dtype)) and torch.equal(db16, db32.to(dtype))
    assert dk16.dtype == dtype
    ulp16_close(dk16, dk32.to(dtype), ("dK1", dtype))

    enc, pred = torch.randn(2, 9, 64, device="cuda"), torch.randn(2, 5, 64, device="cuda")
    W, bias = torch.randn(64, 40, device="cuda") / 8, torch.randn(40, device="cuda")
    l16 = rb.joint_logits(enc.to(dtype), pred.to(dtype), W.to(dtype), bias.to(dtype))
    l32 = rb.joint_logits(*(t.to(dtype).float() for t in (enc, pred, W, bias)))
    assert l16.dtype == torch.float32 and torch.equal(l16, l32)

    j = rb.Joint(48, 64, 40, precision="fp32").cuda()
    f, g = torch.randn(2, 7, 48, device="cuda").to(dtype), torch.randn(2, 5, 48, device="cuda").to(dtype)
    s16 = j.step(f, g)
    s32 = j.step(f.float(), g.float())
    assert s16.dtype == torch.float32 and torch.equal(s16, s32)
    b16, lp16 = j.greedy_step(f, g)
    b32, lp32 = j.greedy_step(f.float(), g.float())
    assert torch.equal(b16, b32) and torch.equal(lp16, lp32)
    with torch.no_grad():
        assert torch.equal(j(f, g), j(f.float(), g.float()))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_autocast_lstm_end_to_end(precision):
    """Under torch.autocast(bfloat16), Joint.loss on the 16-bit outputs of nn.LSTM networks runs end to end, and every
    parameter and input gets a gradient of its own dtype."""
    import rnnt_speech_recognition_b200 as rb
    torch.manual_seed(7)
    B, T, U, P, H, V = 3, 16, 6, 64, 64, 64
    enc_net = torch.nn.LSTM(P, P, batch_first=True).cuda()
    pred_net = torch.nn.LSTM(P, P, batch_first=True).cuda()
    joint = rb.Joint(P, H, V, precision=precision).cuda()
    x = torch.randn(B, T, P, device="cuda", requires_grad=True)
    y = torch.randn(B, U, P, device="cuda", requires_grad=True)
    labels = torch.randint(1, V, (B, U - 1), dtype=torch.int32, device="cuda")
    il = torch.tensor([T, T - 2, T - 5], dtype=torch.int32, device="cuda")
    ll = torch.tensor([U - 1, U - 2, 2], dtype=torch.int32, device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        enc, _ = enc_net(x)
        pred, _ = pred_net(y)
        assert enc.dtype in (torch.float16, torch.bfloat16) and pred.dtype == enc.dtype    # cuDNN's LSTM may pick fp16
        costs = joint.loss(enc, pred, labels, il, ll)
    assert costs.dtype == torch.float32 and torch.isfinite(costs).all()
    (costs.sum() / B).backward()
    for m in (enc_net, pred_net, joint):
        for n, p in m.named_parameters():
            assert p.grad is not None and p.grad.dtype == p.dtype and torch.isfinite(p.grad).all(), n
    for t in (x, y):
        assert t.grad is not None and t.grad.dtype == t.dtype and torch.isfinite(t.grad).all()
