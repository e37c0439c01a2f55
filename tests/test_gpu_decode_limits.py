"""The decode-step joint (`rnntb200_joint_step`) and the hoisted Dense-1 (`rnntb200_dense1_forward / _backward`) at the
limits include/rnnt_b200.h states, against float64 references.

Decode step, against oracle.joint_step (float64 numpy):
  * shapes at the slice boundaries of the 8-CTA cluster (hidden slices of ceil(H/8) <= 256 units, vocabulary slices wider
    than the 256-thread block), P up to 4096, H up to 2048, B up to 1024, K1 given and NULL;
  * dynamic shared memory on both sides of the 48 KB opt-in threshold and at the largest V that fits (V one past it is
    refused; tests/test_decode_limits_host.py has the arithmetic);
  * logits within 2e-5 * max|y| where the FMA chains are <= 1024 long, and beyond that within `step_bound`, a float64
    bound of the fp32 round-off computed from the terms; argmax exact and best_logp within that bound wherever the two
    best logits are further apart than twice it;
  * rows independent of the batch, row-strided and broadcast (ldg = 0) inputs, every subset of the three outputs,
    CUDA-graph replay;
  * the argmax rules, exact by construction: with K2 = 0 the logits are b2 bit for bit, so ties within and across the
    CTA slices, rows of -inf and rows holding NaN have known answers.  A NaN outranks every number and the first NaN
    wins, as np.argmax and torch.argmax decide (what the reference's tf.argmax does with NaN is not pinned here); so
    0 <= best < V on every row.
Dense-1, against torch float64 on the device, through the C ABI and through `rb.dense1`:
  * the accumulation of dK1 / db1, each output NULL, each GEMM kernel choice (split-K, unsplit, the generic kernel
    through P % 4 != 0 and through a buffer 4 bytes off 16-byte alignment), row counts past the 65535 row tiles of
    either kernel's grid, X past 2^31 elements, CUDA-graph replay;
  * the fp32 exact joint path and joint_logits, which run on the same GEMM launcher, past 65535 row tiles.
Peak torch.cuda.max_memory_allocated of the file: about 10 GB (X past 2^31 elements).
"""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from conftest import assert_close, fp32_tol
from test_decode_limits_host import INVALID, SMEM_DEFAULT, step_max_v, step_smem
from test_gpu_large_offsets import NAMES, assert_padding_zero, exact_chunk_rows, joint_abi, joint_reference, synth_case

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
U32 = 2.0 ** -24                 # unit round-off of float32
TANH_ULPS = 4                    # tanhf is within 2 ulp (CUDA C Programming Guide); twice that
SENTINEL_F, SENTINEL_I = 12345.0, -7


@pytest.fixture(autouse=True)
def _release_device_memory():
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def lib():
    from rnnt_speech_recognition_b200 import _lib
    return _lib.load()


def ptr(t):
    from rnnt_speech_recognition_b200 import _lib
    return _lib.ptr(t)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ================================================================================================ decode step
def step_case(B, P, H, V, seed, k1=True):
    g = np.random.default_rng(seed)
    f = g.standard_normal((B, P)).astype(np.float32)
    q = g.standard_normal((B, P)).astype(np.float32)
    K1 = (g.standard_normal((P, H)) / np.sqrt(P)).astype(np.float32) if k1 else None
    b1 = (0.1 * g.standard_normal(H)).astype(np.float32) if k1 else None
    K2 = (g.standard_normal((H, V)) / np.sqrt(H)).astype(np.float32)
    b2 = (0.1 * g.standard_normal(V)).astype(np.float32)
    return f, q, K1, b1, K2, b2


def step(f, g, K1, b1, K2, b2, want=("logits", "best", "logp")):
    """rnntb200_joint_step through the C ABI on device tensors (f, g: (B, P) with unit column stride, any row stride).
    All three outputs are allocated and prefilled with sentinels; those not in `want` are passed as NULL.
    Returns (status, logits, best, best_logp)."""
    B, P = f.shape
    H, V = K2.shape
    logits = torch.full((B, V), SENTINEL_F, device="cuda")
    best = torch.full((B,), SENTINEL_I, dtype=torch.int32, device="cuda")
    logp = torch.full((B,), SENTINEL_F, device="cuda")
    outs = [t if n in want else None for t, n in ((logits, "logits"), (best, "best"), (logp, "logp"))]
    st = lib().rnntb200_joint_step(ptr(f), f.stride(0), ptr(g), g.stride(0), ptr(K1), ptr(b1), ptr(K2), ptr(b2), B, P, H, V,
                                   *map(ptr, outs), stream())
    torch.cuda.synchronize()
    return st, logits, best, logp


def gamma(n):
    return n * U32 / (1 - n * U32)


def step_bound(f, q, K1, b1, K2, b2):
    """Per-logit float64 bound of the kernel's fp32 round-off.  Stage 1 rounds x = f + g once, then each hidden unit is
    a chain of at most P FMAs plus up to 256 partial sums and b1: |ds| <= gamma(P + 258) (sum|x K1| + |b1|); tanhf adds
    a few ulp and passes |ds| on at most unchanged (|tanh'| <= 1).  Stage 2: |dy| <= sum_h |dz_h| |K2| + gamma(H + 258)
    (sum |z K2| + |b2|), with gamma(n) = n u / (1 - n u), u = 2^-24."""
    x = f.astype(np.float64) + q.astype(np.float64)
    if K1 is not None:
        b1a = 0.0 if b1 is None else np.abs(b1.astype(np.float64))
        s = x @ K1.astype(np.float64) + (0.0 if b1 is None else b1.astype(np.float64))
        ds = gamma(x.shape[1] + 258) * (np.abs(x) @ np.abs(K1.astype(np.float64)) + b1a)
    else:
        s, ds = x, U32 * np.abs(x)
    z = np.tanh(s)
    dz = ds + TANH_ULPS * np.spacing(np.abs(z).astype(np.float32)).astype(np.float64)
    aK2 = np.abs(K2.astype(np.float64))
    b2a = 0.0 if b2 is None else np.abs(b2.astype(np.float64))
    return dz @ aK2 + gamma(z.shape[1] + 258) * ((np.abs(z) + dz) @ aK2 + b2a)


def check_step(got, ref, args):
    """Logits, argmax and best_logp of one call against oracle.joint_step.  Logit tolerance: 2e-5 * max|y| where the
    chains are <= 1024 long, step_bound beyond.  Argmax exact and best_logp within 5e-5 + twice the row's bound on the
    rows whose two best logits are further apart than twice the bound."""
    logits, best, logp = (t.cpu().numpy() for t in got)
    y, ybest, ylogp = ref
    B, V = y.shape
    P, H = args[0].shape[1], args[4].shape[0]
    if max(P, H) <= 1024:
        tol = np.full_like(y, 2e-5 * max(1.0, np.abs(y).max()))
    else:
        tol = step_bound(*args)
    err = np.abs(logits.astype(np.float64) - y)
    assert np.all(err <= tol), "logits: worst %.3g at bound %.3g" % ((err - tol).max() + tol.max(), tol.max())
    assert np.all((best >= 0) & (best < V))
    rt = tol.max(axis=1)
    srt = np.sort(y, axis=1)
    clear = (srt[:, -1] - srt[:, -2]) > 2 * rt if V > 1 else np.ones(B, bool)
    assert clear.any()
    np.testing.assert_array_equal(best[clear], ybest[clear])
    assert np.all(np.abs(logp[clear] - ylogp[clear]) <= 5e-5 + 2 * rt[clear])


SWEEP = ([(3, 100, H, 777, True) for H in (7, 8, 9, 255, 256, 257, 2041, 2048)] +      # hidden slices; H = 2048: parts == 1
         [(3, 96, 200, V, True) for V in (1, 7, 9, 2047, 2049, 32000)] +               # vocabulary slices, several passes
         [(2, P, 300, 1500, True) for P in (1, 255, 257, 4096)] +
         [(3, 2048, 2048, 5000, True), (3, 2048, 2048, 5000, False),                   # K1 given / NULL at P = H = 2048
          (1, 4096, 2048, 32000, True), (1, 640, 640, 1024, True)])


@pytest.mark.parametrize("B,P,H,V,k1", SWEEP)
def test_step_shapes_vs_oracle(B, P, H, V, k1):
    from oracle import oracle
    args = step_case(B, P, H, V, seed=P * 7 + H * 3 + V, k1=k1)
    if max(P, H) > 1024:
        # step_bound is a worst case, far above the actual round-off (about 0.2 to 0.6 at P = 4096 or P = H = 2048 with
        # K1): raise one logit of b2 so that every row's maximum clears twice the bound and the argmax stays checked
        y, j = oracle.joint_step(*args)[0], 7 * V // 11
        args[5][j] += np.float32(y.max() - y[:, j].min() + 2 * step_bound(*args).max() + 0.1)
    st, *got = step(*map(dev, args))
    assert st == 0
    check_step(got, oracle.joint_step(*args), args)


def test_step_rows_independent_of_batch():
    """B = 1024 against the oracle, and every row bit-identical to a B = 1 call on that row."""
    from oracle import oracle
    args = step_case(1024, 320, 512, 1024, seed=1024)
    f, q, K1, b1, K2, b2 = map(dev, args)
    st, *got = step(f, q, K1, b1, K2, b2)
    assert st == 0
    check_step(got, oracle.joint_step(*args), args)
    for b in range(f.shape[0]):
        _, lg, bb, lp = step(f[b:b + 1], q[b:b + 1], K1, b1, K2, b2)
        assert torch.equal(lg[0], got[0][b]) and bb[0] == got[1][b] and torch.equal(lp[0], got[2][b]), b


def test_step_strided_and_broadcast_inputs():
    """f row-strided with ldf = P + 5 (not a multiple of 4) at an offset of 3 floats, g one row broadcast with expand
    (ldg = 0): against the oracle and bit-identical to a call on contiguous copies."""
    from oracle import oracle
    B, P, H, V = 6, 301, 256, 3000
    f0, q0, K1, b1, K2, b2 = step_case(B, P, H, V, seed=301)
    fbuf = torch.zeros(B, P + 5, device="cuda")
    fbuf[:, 3:3 + P] = dev(f0)
    f = fbuf[:, 3:3 + P]
    g = dev(q0[:1]).expand(B, P)
    assert f.stride(0) == P + 5 and (P + 5) % 4 and g.stride(0) == 0
    rest = [dev(a) for a in (K1, b1, K2, b2)]
    st, *got = step(f, g, *rest)
    assert st == 0
    q = np.repeat(q0[:1], B, axis=0)
    check_step(got, oracle.joint_step(f0, q, K1, b1, K2, b2), (f0, q, K1, b1, K2, b2))
    _, *want = step(f.contiguous(), g.contiguous(), *rest)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def smem_v(nbytes, P=64, H=64):
    """The largest V whose dynamic shared memory is at most nbytes."""
    return 8 * (nbytes // 4 - max(P, 256) - H - 256)


SMEM_CASES = {"largest without the opt-in": smem_v(SMEM_DEFAULT),
              "first with the opt-in": smem_v(SMEM_DEFAULT) + 1,
              "past 48 KB of dynamic memory": smem_v(48 * 1024) + 1,
              "largest that fits": step_max_v(64, 64)}


@pytest.mark.parametrize("what", list(SMEM_CASES))
def test_step_shared_memory(what):
    """P = H = 64 (K2 up to 118 MB) at V on both sides of the 48 KB threshold (static memory included) and at the
    largest V of the opt-in; one more V is refused before any device work, the outputs untouched."""
    from oracle import oracle
    V = SMEM_CASES[what]
    assert {"largest without the opt-in": step_smem(64, 64, V) <= SMEM_DEFAULT,
            "first with the opt-in": step_smem(64, 64, V) == SMEM_DEFAULT + 4,
            "past 48 KB of dynamic memory": step_smem(64, 64, V) == 48 * 1024 + 4,
            "largest that fits": step_smem(64, 64, V + 1) > step_smem(64, 64, V)}[what]
    args = step_case(2, 64, 64, V, seed=V)
    d = list(map(dev, args))
    st, *got = step(*d)
    assert st == 0
    check_step(got, oracle.joint_step(*args), args)
    if what == "largest that fits":
        K2 = torch.zeros(64, V + 1, device="cuda")
        st, lg, bb, lp = step(d[0], d[1], d[2], d[3], K2, None)
        assert st == INVALID
        assert bool((lg == SENTINEL_F).all()) and bool((bb == SENTINEL_I).all()) and bool((lp == SENTINEL_F).all())


def b2_call(b2, B=2, P=40, H=24):
    """A call whose logits are b2 bit for bit: K2 = 0 (every product and partial sum is +0), random f, g, K1, b1."""
    f, q, K1, b1, _, _ = step_case(B, P, H, 1, seed=len(b2))
    st, lg, bb, lp = step(*map(dev, (f, q, K1, b1)), torch.zeros(H, len(b2), device="cuda"), dev(b2.astype(np.float32)))
    assert st == 0
    return lg.cpu().numpy(), bb.cpu().numpy(), lp.cpu().numpy()


def log_softmax_at(y, i):
    m = y.max()
    return float(y[i] - (m + np.log(np.exp(y - m).sum())))


# V = 2049: slices of 257 entries (two passes of the block), CTA r owns [257 r, 257 r + 257), CTA 7 the 250 of
# [1799, 2049).  V = 32000: slices of 4000 (16 passes).
TIES = {"different CTAs": (2049, (1000, 300)),
        "first and last entry": (2049, (2048, 0)),
        "same CTA, different threads": (2049, (514 + 200, 514 + 5)),
        "same CTA and thread, two passes": (2049, (514 + 3 + 256, 514 + 3)),
        "last, partial slice": (2049, (1799 + 249, 1799 + 3)),
        "last slice and an earlier one": (2049, (2048, 1799 + 3, 5)),
        "three CTAs, 16 passes": (32000, (31999, 16000, 4001))}


@pytest.mark.parametrize("what", list(TIES))
def test_step_ties_take_the_smallest_index(what):
    V, planted = TIES[what]
    rng = np.random.default_rng(V + sum(planted))
    b2 = np.clip(0.5 * rng.standard_normal(V), -2.5, 2.5).astype(np.float32)
    b2[list(planted)] = 3.0
    lg, bb, lp = b2_call(b2)
    assert np.array_equal(lg, np.broadcast_to(b2, lg.shape))
    assert np.all(bb == min(planted))
    assert np.all(np.abs(lp - log_softmax_at(b2.astype(np.float64), min(planted))) <= 1e-5)


@pytest.mark.parametrize("V", [1, 9, 2049, 32000])
def test_step_all_equal_logits(V):
    lg, bb, lp = b2_call(np.full(V, 0.7, np.float32))
    assert np.all(lg == np.float32(0.7)) and np.all(bb == 0)
    assert np.all(np.abs(lp.astype(np.float64) + np.log(V)) <= 2 * np.spacing(np.float32(np.log(V))))


def nonfinite_rows():
    rng = np.random.default_rng(99)
    rows = {}
    for V in (7, 2049, 32000):
        finite = (0.5 * rng.standard_normal(V)).astype(np.float32)
        ninf = np.full(V, -INF, np.float32)
        rows[(V, "all -inf")] = ninf
        rows[(V, "all NaN")] = np.full(V, NAN, np.float32)
        last = finite.copy()
        last[V - 1] = NAN
        rows[(V, "NaN last")] = last
        two = finite.copy()
        two[[V - 1, V // 3]] = NAN
        rows[(V, "two NaN")] = two
        first = finite.copy()
        first[0] = NAN
        rows[(V, "NaN first")] = first
        mixed = ninf.copy()
        mixed[V - 2] = NAN
        rows[(V, "NaN among -inf")] = mixed
        one = ninf.copy()
        one[V // 2] = 1.5
        rows[(V, "one finite among -inf")] = one
    return rows


NONFINITE = nonfinite_rows()


@pytest.mark.parametrize("key", list(NONFINITE), ids=["V=%d, %s" % k for k in NONFINITE])
def test_step_nonfinite_rows(key):
    """best is np.argmax's answer (the first NaN if there is one, else the first maximum: 0 for a row of -inf), so it
    always lies in [0, V); best_logp is NaN exactly where float64 log_softmax is NaN."""
    b2 = NONFINITE[key]
    V = len(b2)
    lg, bb, lp = b2_call(b2)
    np.testing.assert_array_equal(lg, np.broadcast_to(b2, lg.shape))      # NaN compares equal to NaN here
    want = int(np.argmax(b2))
    assert np.all(bb == want), (bb, want)
    assert np.all((bb >= 0) & (bb < V))
    with np.errstate(invalid="ignore"):
        wl = log_softmax_at(b2.astype(np.float64), want)
    if np.isnan(wl):
        assert np.all(np.isnan(lp)), lp
    else:
        assert np.all(np.abs(lp - wl) <= 1e-6), (lp, wl)


def test_step_output_subsets():
    """Each non-empty subset of (logits, best, best_logp): the outputs asked for are bit-identical to those of the call
    that asks for all three, the buffers passed as NULL keep their sentinels."""
    args = list(map(dev, step_case(5, 200, 300, 3000, seed=5)))
    names = ("logits", "best", "logp")
    st, *full = step(*args)
    assert st == 0 and not bool((full[0] == SENTINEL_F).any()) and not bool((full[1] == SENTINEL_I).any())
    for n in range(1, 4):
        for want in itertools.combinations(names, n):
            st, *got = step(*args, want=want)
            assert st == 0
            for name, g, f, s in zip(names, got, full, (SENTINEL_F, SENTINEL_I, SENTINEL_F)):
                if name in want:
                    assert torch.equal(g, f), (want, name)
                else:
                    assert bool((g == s).all()), (want, name)


def test_step_cuda_graph_replay():
    """Capture rnntb200_joint_step (V past 48 KB of shared memory: the opt-in path) into a CUDA graph, replay it on new
    input values: bit-identical to an eager call on those values."""
    B, P, H, V = 4, 320, 512, 100000
    assert step_smem(P, H, V) > 48 * 1024
    a0 = step_case(B, P, H, V, seed=7)
    a1 = step_case(B, P, H, V, seed=8)
    f, q, K1, b1, K2, b2 = map(dev, a0)
    outs = (torch.empty(B, V, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda"), torch.empty(B, device="cuda"))

    def call():
        return lib().rnntb200_joint_step(ptr(f), P, ptr(q), P, ptr(K1), ptr(b1), ptr(K2), ptr(b2), B, P, H, V,
                                         *map(ptr, outs), stream())

    assert call() == 0                                   # eager first: the opt-in is set outside the capture
    torch.cuda.synchronize()
    first = [o.clone() for o in outs]
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        assert call() == 0
    for dst, src in zip((f, q, K1, b1, K2, b2), a1):
        dst.copy_(torch.from_numpy(src))
    gr.replay()
    torch.cuda.synchronize()
    st, *want = step(f, q, K1, b1, K2, b2)
    assert st == 0
    assert all(torch.equal(o, w) for o, w in zip(outs, want))
    assert not torch.equal(outs[0], first[0])


# ================================================================================================== Dense-1
def d1_forward(X, rows, P, K1, b1, H, out):
    return lib().rnntb200_dense1_forward(ptr(X), rows, P, ptr(K1), ptr(b1), H, ptr(out), stream())


def d1_backward(X, dA, K1, rows, P, H, dX, dK1, db1):
    return lib().rnntb200_dense1_backward(ptr(X), ptr(dA), ptr(K1), rows, P, H, ptr(dX), ptr(dK1), ptr(db1), stream())


def maxabs(t):
    return float(t.abs().max())


def within(got, ref, k, floor=0.0):
    """tests/test_gpu_decode.py's bound for a length-k fp32 reduction: 2e-6 * scale * sqrt(k), scale = max|ref| (at least
    `floor`)."""
    err = maxabs(got.double() - ref)
    bound = 2e-6 * max(floor, maxabs(ref)) * k ** 0.5
    assert err <= bound, (err, bound)          # NaN fails


def xt_da(X, dA, chunk=1 << 18):
    """X^T dA and the column sums of dA in float64 on the device, chunked over the rows."""
    dK = torch.zeros(X.shape[1], dA.shape[1], dtype=torch.float64, device="cuda")
    db = torch.zeros(dA.shape[1], dtype=torch.float64, device="cuda")
    for r in range(0, X.shape[0], chunk):
        d = dA[r:r + chunk].double()
        dK += X[r:r + chunk].double().T @ d
        db += d.sum(0)
    return dK, db


def x_k(X, K1, b1, chunk=1 << 18):
    """Generator of (row range, X K1 + b1 in float64) chunks."""
    for r in range(0, X.shape[0], chunk):
        y = X[r:r + chunk].double() @ K1.double()
        yield slice(r, r + chunk), (y + b1.double() if b1 is not None else y)


def d1_tensors(rows, P, H, seed, offset=0):
    """X (rows, P), dA (rows, H) and, with offset = 1, views 4 bytes past a 16-byte boundary; K1 (P, H), b1 (H)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.randn(rows * P + offset, generator=g, device="cuda")[offset:].view(rows, P)
    dA = torch.randn(rows * H + offset, generator=g, device="cuda")[offset:].view(rows, H)
    K1 = torch.randn(P, H, generator=g, device="cuda") / P ** 0.5
    b1 = 0.1 * torch.randn(H, generator=g, device="cuda")
    return X, dA, K1, b1


def nan_out(rows, n, offset=0):
    return torch.full((rows * n + offset,), NAN, device="cuda")[offset:].view(rows, n)


def check_dense1(X, dA, K1, b1, offset=0, want_dX=True):
    """Forward and the three gradients into NaN-prefilled out / dX and zeroed dK1 / db1, against float64."""
    rows, P = X.shape
    H = K1.shape[1]
    out = nan_out(rows, H, offset)
    assert d1_forward(X, rows, P, K1, b1, H, out) == 0
    for sl, ref in x_k(X, K1, b1):
        within(out[sl], ref, P, floor=1.0)
    del out
    dX = nan_out(rows, P, offset) if want_dX else None
    dK, db = torch.zeros(P, H, device="cuda"), torch.zeros(H, device="cuda")
    assert d1_backward(X, dA, K1, rows, P, H, dX, dK, db) == 0
    torch.cuda.synchronize()
    if want_dX:
        Kd = K1.double()
        for r in range(0, rows, 1 << 18):
            within(dX[r:r + (1 << 18)], dA[r:r + (1 << 18)].double() @ Kd.T, H)
    rK, rb = xt_da(X, dA)
    within(dK, rK, rows)
    within(db, rb, rows, floor=1.0)


KERNELS = {"split-K dK1 (fast kernel)": (8192, 256, 256, 0),      # dK1: 4 tiles < 132, K = rows >= 4096
           "unsplit (fast kernel)": (4095, 256, 256, 0),
           "generic kernel, P % 4 != 0": (5000, 77, 64, 0),
           "generic kernel, misaligned buffers": (5000, 64, 64, 1)}


@pytest.mark.parametrize("what", list(KERNELS))
def test_dense1_kernel_choices(what):
    rows, P, H, offset = KERNELS[what]
    X, dA, K1, b1 = d1_tensors(rows, P, H, seed=rows + P, offset=offset)
    assert (X.data_ptr() % 16 == 4) == bool(offset)
    check_dense1(X, dA, K1, b1, offset)


@pytest.mark.parametrize("rows,P,H", [(8388609, 4, 4),     # fast kernel: 65535 * 128 = 8388480 rows per launch
                                      (4194305, 3, 4)])    # generic kernel (P % 4 != 0): 65535 * 64 = 4194240
def test_dense1_past_the_grid_limit(rows, P, H):
    """Row counts past the 65535 row tiles one launch's gridDim.y holds: every row of out / dX written and within the
    bound (rows 65535 * tile - 1 and 65535 * tile are the first launch's last and the second's first), dK1 / db1 over all
    rows."""
    X, dA, K1, b1 = d1_tensors(rows, P, H, seed=rows)
    check_dense1(X, dA, K1, b1)


def test_dense1_x_past_2_31_elements():
    """X (8388609, 256): its last row lies past element 2^31.  Forward and dK1 / db1 (dX NULL keeps the peak near 10 GB)."""
    P, H = 256, 4
    rows = 2 ** 31 // P + 1
    X, dA, K1, b1 = d1_tensors(rows, P, H, seed=31)
    assert X.numel() > 2 ** 31
    check_dense1(X, dA, K1, b1, want_dX=False)


@pytest.mark.parametrize("P,H,Re,Rp", [(256, 256, 6000, 300), (77, 50, 5000, 130)])
def test_dense1_backward_accumulates(P, H, Re, Rp):
    """The documented pair of calls into one buffer: the encoder side with db1, the prediction side without, onto
    non-zero dK1 / db1 (split-K atomics on the 6000-row call): prefill + X_enc^T dA_enc + X_pred^T dA_pred."""
    Xe, dAe, K1, _ = d1_tensors(Re, P, H, seed=Re)
    Xp, dAp, _, _ = d1_tensors(Rp, P, H, seed=Rp)
    g = torch.Generator(device="cuda").manual_seed(3)
    preK, preb = torch.randn(P, H, generator=g, device="cuda"), torch.randn(H, generator=g, device="cuda")
    dK, db = preK.clone(), preb.clone()
    dXe, dXp = nan_out(Re, P), nan_out(Rp, P)
    assert d1_backward(Xe, dAe, K1, Re, P, H, dXe, dK, db) == 0
    assert d1_backward(Xp, dAp, K1, Rp, P, H, dXp, dK, None) == 0
    torch.cuda.synchronize()
    ke, be = xt_da(Xe, dAe)
    kp, _ = xt_da(Xp, dAp)
    within(dK, preK.double() + ke + kp, Re + Rp)
    within(db, preb.double() + be, Re, floor=1.0)
    within(dXe, dAe.double() @ K1.double().T, H)
    within(dXp, dAp.double() @ K1.double().T, H)

    # the same through rb.dense1 and autograd, onto existing .grad tensors
    import rnnt_speech_recognition_b200 as rb
    K = K1.clone().requires_grad_()
    b = torch.zeros(H, device="cuda", requires_grad=True)
    K.grad, b.grad = preK.clone(), preb.clone()
    xe, xp = Xe.clone().requires_grad_(), Xp.clone().requires_grad_()
    torch.autograd.backward([rb.dense1(xe, K, b), rb.dense1(xp, K, None)], [dAe, dAp])
    within(K.grad, preK.double() + ke + kp, Re + Rp)
    within(b.grad, preb.double() + be, Re, floor=1.0)
    assert torch.equal(xe.grad, dXe) and torch.equal(xp.grad, dXp)


@pytest.mark.parametrize("null", ["dX", "dK1", "db1"])
def test_dense1_backward_null_output(null):
    """One of dX, dK1, db1 NULL: the other two as in the call with all three (dX and db1 bit for bit, dK1 within the
    bound: its split-K atomics arrive in any order), and nothing written outside them.  The outputs are laid out in one
    sentinel-filled arena with 64-float guards; the NULL output's place in it keeps the sentinel."""
    rows, P, H, G = 5000, 128, 96, 64
    X, dA, K1, _ = d1_tensors(rows, P, H, seed=77)
    sizes = {"dX": rows * P, "dK1": P * H, "db1": H}
    arena = torch.full((sum(sizes.values()) + 4 * G,), SENTINEL_F, device="cuda")
    views, o = {}, G
    for n, s in sizes.items():
        views[n] = arena[o:o + s]
        o += s + G
    for n in ("dK1", "db1"):                    # accumulated into
        if n != null:
            views[n].zero_()
    ref ={"dX": nan_out(rows, P).view(-1), "dK1": torch.zeros(P * H, device="cuda"), "db1": torch.zeros(H, device="cuda")}
    assert d1_backward(X, dA, K1, rows, P, H, ref["dX"], ref["dK1"], ref["db1"]) == 0
    args = {n: (None if n == null else views[n]) for n in sizes}
    assert d1_backward(X if null != "dK1" else None, dA, K1, rows, P, H, args["dX"], args["dK1"], args["db1"]) == 0
    torch.cuda.synchronize()
    o = 0
    for n, s in sizes.items():
        assert bool((arena[o:o + G] == SENTINEL_F).all()), "guard in front of " + n
        o += G
        if n == null:
            assert bool((arena[o:o + s] == SENTINEL_F).all()), n
        elif n == "dK1":
            within(views[n], xt_da(X, dA)[0].view(-1), rows)
            within(views[n], ref[n].double(), rows)
        else:
            assert torch.equal(views[n], ref[n]), n
        o += s
    assert bool((arena[o:] == SENTINEL_F).all()), "guard at the end"


def test_dense1_cuda_graph_replay():
    """Forward and backward (zeroing dK1 / db1 first) captured into one CUDA graph and replayed on new X, dA: out, dX and
    db1 bit-identical to eager calls on the new values, dK1 (split-K atomics) within the bound of float64."""
    rows, P, H = 5000, 128, 96
    X, dA, K1, b1 = d1_tensors(rows, P, H, seed=1)
    X1, dA1, _, _ = d1_tensors(rows, P, H, seed=2)
    out, dX = torch.empty(rows, H, device="cuda"), torch.empty(rows, P, device="cuda")
    dK, db = torch.zeros(P, H, device="cuda"), torch.zeros(H, device="cuda")

    def run():
        assert d1_forward(X, rows, P, K1, b1, H, out) == 0
        dK.zero_()
        db.zero_()
        assert d1_backward(X, dA, K1, rows, P, H, dX, dK, db) == 0

    run()
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        run()
    X.copy_(X1)
    dA.copy_(dA1)
    gr.replay()
    torch.cuda.synchronize()
    got = [t.clone() for t in (out, dX, dK, db)]
    run()
    torch.cuda.synchronize()
    assert torch.equal(got[0], out) and torch.equal(got[1], dX) and torch.equal(got[3], db)
    within(got[2], xt_da(X1, dA1)[0], rows)
    within(got[0], X1.double() @ K1.double() + b1.double(), P, floor=1.0)


# ------------------------------------------------------------------- the fp32 exact joint past 65535 row tiles
# maxT = maxU = 64 (4096 lattice rows per utterance), one row chunk of the exact path for the whole batch.  Utterance c
# straddles the first launch's last row tile: T = 64, U = 8, its rows from frame t0 on lie past 65535 * tile.
# Utterance c + 2 lies wholly past it; all others are a few frames and labels: almost every row is padding.
EXACT_LIMIT = {"sgemm128": dict(H=4, V=16, tile=128), "sgemm": dict(H=4, V=15, tile=64)}     # V % 4 != 0: generic


def exact_limit_case(layout):
    e = EXACT_LIMIT[layout]
    maxT = maxU = 64
    limit = 65535 * e["tile"]
    c = limit // (maxT * maxU)
    B = c + 3
    rng = np.random.default_rng(c)
    lengths = [(int(t), int(u)) for t, u in zip(rng.integers(1, 5, B), rng.integers(1, 4, B))]
    lengths[c], lengths[c + 2] = (64, 8), (20, 10)
    N = B * maxT * maxU
    assert exact_chunk_rows(e["H"], e["V"], N) == N > limit                 # one chunk, taller than one launch
    first, last = c * maxT * maxU, c * maxT * maxU + (63 * maxU + 7)
    assert first < limit <= last and (c + 2) * maxT * maxU > limit
    return synth_case(tuple(lengths), maxT, maxU, e["V"], e["H"], 4242), limit


@pytest.mark.parametrize("layout", list(EXACT_LIMIT))
def test_exact_joint_past_the_grid_limit(oracle, layout):
    """rnntb200_joint_loss_forward / _backward (fp32) and rnntb200_joint_logits on 8.4 M (fast kernel) and 4.2 M (generic
    kernel) lattice rows: costs and the four gradients against the float64 oracle at the tolerances of
    tests/test_gpu_large_offsets.py::test_exact_joint_across_row_chunks, padded d_enc / d_pred rows exactly 0, and every
    logit of the utterances around and past the limit against float64."""
    from rnnt_speech_recognition_b200 import joint as J
    k, limit = exact_limit_case(layout)
    B = len(k["input_lengths"])
    gs = np.linspace(0.5, 1.5, B)
    want = joint_reference(oracle, k, gs)
    costs, grads = joint_abi(k, "fp32", gs)
    cmax = float(np.abs(want["costs"]).max())
    assert_close(costs, want["costs"], rtol=1e-5, atol=1e-4, what="costs")
    for g, n in zip(grads, NAMES):
        assert_close(g, want[n], rtol=1e-4, atol=fp32_tol(want["costs"])["atol"] * gs.max(), ntol=max(1e-5, 2e-7 * cmax),
                     what=n)
    assert_padding_zero(k, grads, layout)
    del grads

    t = [dev(k[n]) for n in ("enc", "pred", "W", "b")]
    (_, maxT, H), (maxU, V) = t[0].shape, (t[1].shape[1], t[2].shape[1])
    desc = J._desc(B, maxT, maxU, H, V, 0, "fp32")
    ws = J._workspace(desc, "cuda")
    out = torch.full((B, maxT, maxU, V), NAN, device="cuda")
    assert lib().rnntb200_joint_logits(C.byref(desc), *map(ptr, t), ptr(out), ptr(ws)) == 0
    torch.cuda.synchronize()
    assert not bool(torch.isnan(out).any())
    c = limit // (maxT * maxU)
    for b in (0, c - 1, c, c + 1, c + 2):
        z = torch.tanh(t[0][b].double()[:, None, :] + t[1][b].double()[None, :, :])
        ref = (z @ t[2].double() + t[3].double()).cpu().numpy()
        assert_close(out[b].cpu().numpy(), ref, rtol=1e-5, atol=2e-5, what="logits of utterance %d" % b)
