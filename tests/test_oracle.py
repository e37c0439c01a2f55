"""Pin the oracle (oracle/rnnt_oracle.c) against the reference's own known-answer tests, the
golden fixtures generated from the reference library (tests/golden/make_golden.py) and, when it
is present in this container, the unmodified reference library itself (oracle/_ref)."""
import numpy as np
import pytest

from conftest import GOLDEN, assert_close, fp32_tol, golden_names, load


def softmax_chain(lp_grads, log_probs):
    """grads wrt logits from grads wrt log-probs: g - P * sum_v g (autograd of log_softmax)."""
    P = np.exp(log_probs.astype(np.float64))
    return lp_grads - P * lp_grads.sum(-1, keepdims=True)


def test_kat_small(oracle):
    k = load("kat_small.npz")   # warp-transducer/tests/test_cpu.cpp:12-71, pytorch test.py:51-78
    acts = k["acts"].astype(np.float32)
    lp = oracle.log_softmax(acts)
    costs, _ = oracle.rnnt_cost_and_grad(lp, k["labels"], k["input_lengths"], k["label_lengths"], want_grad=False)
    assert abs(costs[0] - k["cost"]) < 1e-4            # eps of test_cpu.cpp:66
    c2, g = oracle.rnnt_logits_grad(acts, k["labels"], k["input_lengths"], k["label_lengths"])
    assert np.allclose(c2, k["cost"], rtol=1e-6)       # test.py:75
    assert np.allclose(g, k["logits_grads"])           # test.py:77 (default rtol 1e-5, atol 1e-8)


def test_kat_big_logprob_grads(oracle):
    k = load("kat_big.npz")     # options_test, test_cpu.cpp:73-179
    lp = oracle.log_softmax(k["acts_6dp"].astype(np.float32))
    costs, grads = oracle.rnnt_cost_and_grad(lp, k["labels"], k["input_lengths"], k["label_lengths"])
    assert np.all(np.abs(costs - k["costs"]) < 1e-4)
    assert np.all(np.abs(grads - k["logprob_grads"]) < 1e-4)


def test_kat_big_logits_grads(oracle):
    k = load("kat_big.npz")     # test_gpu.cu:96-224, test_warprnnt_op.py:52-87, test.py:80-160
    costs, grads = oracle.rnnt_logits_grad(k["acts"].astype(np.float32), k["labels"], k["input_lengths"],
                                           k["label_lengths"])
    assert np.allclose(costs, k["costs"], atol=1e-6, rtol=1e-6)
    assert np.allclose(grads, k["logits_grads"], atol=1e-6, rtol=1e-3)
    c64, g64 = oracle.rnnt_logits_grad(k["acts"], k["labels"], k["input_lengths"], k["label_lengths"])
    assert np.allclose(c64, k["costs"], atol=1e-12, rtol=1e-12)
    assert np.allclose(g64, k["logits_grads"], atol=2e-7)   # the KAT table itself was printed from an fp32 run


@pytest.mark.parametrize("name", golden_names("logits_"))
def test_logits_cases(oracle, name):
    k = load(name)
    blank = int(k["blank"])
    costs, grads = oracle.rnnt_logits_grad(k["acts"], k["labels"], k["input_lengths"], k["label_lengths"], blank)
    assert np.all(np.isfinite(costs)) and np.all(np.isfinite(grads))      # inf_test, test_cpu.cpp:181-240
    tol = fp32_tol(k["costs"])
    assert np.allclose(costs, k["costs"], rtol=1e-5, atol=1e-5)
    assert np.allclose(grads, k["logits_grads"], **tol)
    # CPU-path semantics against the fp32 run of the real reference
    lp = oracle.log_softmax(k["acts"])
    c32, g32 = oracle.rnnt_cost_and_grad(lp, k["labels"], k["input_lengths"], k["label_lengths"], blank)
    assert np.allclose(c32, k["costs_f32"], rtol=1e-5, atol=1e-5)
    assert np.allclose(g32, k["logprob_grads_f32"], **tol)
    # padded cells carry exactly zero gradient (gpu_rnnt.h:109, cpu_rnnt.h:155-158)
    for b in range(k["acts"].shape[0]):
        T, U = int(k["input_lengths"][b]), int(k["label_lengths"][b]) + 1
        assert not grads[b, T:].any() and not grads[b, :, U:].any()
    # f64 instantiation agrees with the f64 reference run to round-off
    c64, g64 = oracle.rnnt_logits_grad(k["acts"].astype(np.float64), k["labels"], k["input_lengths"],
                                       k["label_lengths"], blank)
    assert np.allclose(c64, k["costs"], rtol=1e-10) and np.allclose(g64, k["logits_grads"], atol=1e-10)


@pytest.mark.parametrize("name", golden_names("joint_"))
def test_joint_cases(oracle, name):
    k = load(name)
    B = k["enc"].shape[0]
    out = oracle.joint_loss_grad(k["enc"], k["pred"], k["W"], k["b"], k["labels"], k["input_lengths"],
                                 k["label_lengths"], int(k["blank"]), grad_scale=np.full(B, 1.0 / B))
    assert np.allclose(out["costs"], k["costs"], rtol=1e-5)
    for g in ("d_enc", "d_pred", "dW", "db"):
        assert_close(out[g], k[g], rtol=1e-4, atol=1e-6, ntol=1e-5, what=g)
    o64 = oracle.joint_loss_grad(*(k[n].astype(np.float64) for n in ("enc", "pred", "W", "b")), k["labels"],
                                 k["input_lengths"], k["label_lengths"], int(k["blank"]),
                                 grad_scale=np.full(B, 1.0 / B))
    for g in ("d_enc", "d_pred", "dW", "db"):
        assert np.allclose(o64[g], k[g], rtol=1e-9, atol=1e-11), g


def test_numeric_gradient(oracle):
    """Central-difference check, the property test of test_cpu.cpp:287-379 (eps 1e-2, rel-L2 < 1e-4),
    run in fp64 so the finite difference itself is trustworthy."""
    rng = np.random.default_rng(7)
    B, T, U, V = 2, 6, 4, 5
    acts = rng.uniform(0, 1, (B, T, U, V))
    labels = rng.integers(1, V, (B, U - 1)).astype(np.int32)
    il, ll = np.array([T, T - 2], np.int32), np.array([U - 1, U - 2], np.int32)
    _, g = oracle.rnnt_logits_grad(acts, labels, il, ll)
    num = np.zeros_like(acts)
    eps = 1e-4
    flat = acts.reshape(-1)
    for i in range(flat.size):
        old = flat[i]
        flat[i] = old + eps
        cp, _ = oracle.rnnt_logits_grad(acts, labels, il, ll, want_grad=False)
        flat[i] = old - eps
        cm, _ = oracle.rnnt_logits_grad(acts, labels, il, ll, want_grad=False)
        flat[i] = old
        num.reshape(-1)[i] = (cp.sum() - cm.sum()) / (2 * eps)
    rel = ((g - num) ** 2).sum() / (g ** 2).sum()     # rel_diff, tests/test.h:22-32
    assert rel < 1e-8


def ref_cases():
    """Outputs of the unmodified reference library for the inputs of tests/golden/make_ref_cases.py."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("make_ref_cases", os.path.join(GOLDEN, "make_ref_cases.py"))
    mrc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mrc)
    return mrc, load("ref_cases.npz")


def test_against_live_reference(oracle):
    """The restatement agrees with the unmodified reference library on random input: live when oracle/_ref is built,
    otherwise against the reference's stored outputs (tests/golden/ref_cases.npz)."""
    mrc, gold = ref_cases()
    lp, labels, il, ll = mrc.live_case(oracle)
    c, g = oracle.rnnt_cost_and_grad(lp, labels, il, ll)
    cr, gr, ws = gold["live_costs"], gold["live_grads"], int(gold["live_ws_gpu"])
    if oracle.have_ref():
        cr, gr = oracle.ref_cpu_cost_and_grad(lp, labels, il, ll, num_threads=2)
        import ctypes as C
        s = C.c_size_t(0)
        assert oracle.ref().get_workspace_size(13, 6, 4, True, C.byref(s), 4) == 0
        ws = s.value
    assert np.allclose(c, cr, rtol=1e-6) and np.allclose(g, gr, rtol=1e-5, atol=1e-7)
    rc, sz = oracle.get_workspace_size(13, 6, 4, True)
    assert rc == 0 and ws == sz


def test_invalid_arguments(oracle):
    assert oracle.get_workspace_size(0, 3, 2, False)[0] == 2    # rnnt_entrypoint.cpp:102-105
    assert oracle.get_workspace_size(4, 3, 2, False) == (0, 2 * 4 * 4 * 3 * 4)
    assert oracle.get_workspace_size(4, 3, 2, True) == (0, 2 * (3 * 4 * 3 + 2) * 4)


def test_against_live_reference_property(oracle):
    """On random shapes, ragged lengths, blank positions and logit scales (a fixed sequence of cases) the restatement and
    the unmodified reference library agree on costs and log-prob gradients (live, or its stored outputs)."""
    mrc, gold = ref_cases()
    for i in range(mrc.N_CPU_CASES):
        lp, labels, il, ll, blank = mrc.cpu_case(oracle, i)
        c, g = oracle.rnnt_cost_and_grad(lp, labels, il, ll, blank=blank)
        if oracle.have_ref():
            cr, gr = oracle.ref_cpu_cost_and_grad(lp, labels, il, ll, blank=blank, num_threads=1)
        else:
            cr, gr = gold["cpu%d_costs" % i], gold["cpu%d_grads" % i]
        assert np.allclose(c, cr, rtol=1e-5, atol=1e-6), (i, lp.shape)
        assert np.allclose(g, gr, rtol=1e-4, atol=1e-6), (i, lp.shape)


def test_joint_oracle_against_torch_fp64_chain_property(oracle):
    """The joint is parity-unpinned by the reference (TensorFlow arithmetic): its anchor is model.py:158-166 restated in
    torch fp64 and chained by autograd through log_softmax into the reference library's fp64 entry point
    (tests/golden/make_golden.py: joint_case).  Ten random shapes beyond the committed fixtures: generated live when
    oracle/_ref is built, otherwise the stored chain results."""
    mrc, gold = ref_cases()
    if oracle.have_ref():
        cases = mrc.joint_cases()
    else:
        cases = [{n[len("joint%d_" % i):]: gold[n] for n in gold if n.startswith("joint%d_" % i)}
                 for i in range(mrc.N_JOINT_CASES)]
    for k in cases:
        B = k["enc"].shape[0]
        o64 = oracle.joint_loss_grad(*(k[n].astype(np.float64) for n in ("enc", "pred", "W", "b")), k["labels"],
                                     k["input_lengths"], k["label_lengths"], int(k["blank"]), grad_scale=np.full(B, 1.0 / B))
        assert np.allclose(o64["costs"], k["costs"], rtol=1e-10), k["enc"].shape
        for g in ("d_enc", "d_pred", "dW", "db"):
            assert np.allclose(o64[g], k[g], rtol=1e-9, atol=1e-11), (g, k["enc"].shape)
