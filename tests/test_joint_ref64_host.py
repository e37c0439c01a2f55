"""tests/joint_ref64.py (the chunked float64 reference of the GPU parity tests at full size) pinned on the host to the
C oracle and to tests/fastemit_ref.py at the 1e-12 level: golden joint and logits fixtures, random ragged batches, U = 1,
T = 1, blank in {0, 5, V-1} with labels equal to blank, FastEmit lambda in {0, 0.5}, and chunks of 1 row, of a prime
number of rows, with a boundary inside an utterance, and of the whole batch."""
import numpy as np
import pytest

import fastemit_ref as fr
import joint_ref64 as r64
from conftest import assert_close, golden_names, load

REL = 1e-12
NAMES = ("d_enc", "d_pred", "dW", "db")


def pinned(got, want, what):
    """Costs and gradients within 1e-12 relative, element-wise plus a 1e-12·max|g| norm term (the two sides sum in
    different orders)."""
    assert_close(got["costs"], want["costs"], rtol=REL, atol=0, what=what + " costs")
    for n in NAMES:
        assert_close(got[n], want[n], rtol=REL, atol=0, ntol=REL, what="%s %s" % (what, n))


def joint_args(k):
    return [k[n].astype(np.float64) for n in ("enc", "pred", "W", "b")] + [k["labels"], k["input_lengths"],
                                                                          k["label_lengths"], int(k["blank"])]


def random_joint(B, T, U, V, H, seed, blank=0, label_is_blank=False):
    rng = np.random.default_rng(seed)
    il, ll = rng.integers(1, T + 1, B).astype(np.int32), rng.integers(0, U, B).astype(np.int32)
    il[0], ll[0] = T, U - 1
    labels = rng.integers(0, V, (B, U - 1)).astype(np.int32)
    if label_is_blank:
        labels[:, ::2] = blank
    return dict(enc=rng.standard_normal((B, T, H)), pred=rng.standard_normal((B, U, H)),
                W=rng.standard_normal((H, V)) / np.sqrt(H), b=0.1 * rng.standard_normal(V),
                labels=labels, input_lengths=il, label_lengths=ll, blank=np.int32(blank))


JOINT_CASES = {n: (lambda n=n: load(n)) for n in golden_names("joint_")}
JOINT_CASES.update({
    "ragged": lambda: random_joint(4, 11, 7, 13, 9, 1),
    "ragged_wide": lambda: random_joint(3, 6, 15, 40, 5, 2),
    "u1": lambda: random_joint(3, 8, 1, 6, 4, 3),
    "t1": lambda: random_joint(3, 1, 6, 7, 4, 4),
    "blank5_label_is_blank": lambda: random_joint(3, 9, 6, 11, 6, 5, blank=5, label_is_blank=True),
    "blank_last_label_is_blank": lambda: random_joint(3, 9, 6, 11, 6, 6, blank=10, label_is_blank=True),
    "blank0_label_is_blank": lambda: random_joint(2, 7, 5, 8, 3, 7, blank=0, label_is_blank=True),
})


@pytest.mark.parametrize("name", sorted(JOINT_CASES))
def test_joint_against_oracle_and_fastemit_ref(oracle, name):
    k = JOINT_CASES[name]()
    B = len(k["input_lengths"])
    gs = np.linspace(0.5, 1.5, B)
    args = joint_args(k)
    pinned(r64.joint_loss_grad(*args, grad_scale=gs), oracle.joint_loss_grad(*args, grad_scale=gs), name + " vs oracle")
    for lam in (0.0, 0.5):
        pinned(r64.joint_loss_grad(*args, grad_scale=gs, fastemit_lambda=lam),
               fr.joint_loss_grad(*args, grad_scale=gs, fastemit_lambda=lam), "%s vs fastemit_ref, lambda %g" % (name, lam))


def test_labels_equal_to_blank_are_separate_arcs():
    """With label == blank the two arcs share a logit column: the reference adds both arcs' terms there, which
    fastemit_ref reaches by moving such labels to a private column.  Check that it is the case being exercised."""
    k = random_joint(3, 9, 6, 11, 6, 5, blank=5, label_is_blank=True)
    used = [k["labels"][b, :k["label_lengths"][b]] for b in range(3)]
    assert any((u == 5).any() for u in used)
    args = joint_args(k)
    for lam in (0.0, 0.5):
        pinned(r64.joint_loss_grad(*args, fastemit_lambda=lam), fr.joint_loss_grad(*args, fastemit_lambda=lam),
               "lambda %g" % lam)


@pytest.mark.parametrize("name", golden_names("logits_"))
def test_op_against_oracle_and_fastemit_ref(oracle, name):
    k = load(name)
    x = k["acts"].astype(np.float64)
    blank = int(k["blank"])
    B = x.shape[0]
    gs = np.linspace(0.5, 1.5, B)
    lab, il, ll = k["labels"], k["input_lengths"], k["label_lengths"]
    xt = r64.torch.as_tensor(x)
    for lam in (0.0, 0.5):
        costs, g = r64.op_loss_grad(lambda b, t, u: xt[b, t, u].clone(), x.shape, lab, il, ll, blank, gs, lam)
        wc, wg = fr.logits_grad(x, lab, il, ll, blank, lam, gs)
        assert_close(costs, wc, rtol=REL, atol=0, what=name + " costs")
        assert_close(g, wg, rtol=REL, atol=0, ntol=REL, what="%s grads, lambda %g" % (name, lam))
    oc, og = oracle.rnnt_logits_grad(x, lab, il, ll, blank)
    costs, g = r64.op_loss_grad(lambda b, t, u: xt[b, t, u].clone(), x.shape, lab, il, ll, blank)
    assert_close(costs, oc, rtol=REL, atol=0, what=name + " costs vs oracle")
    assert_close(g, og, rtol=REL, atol=0, ntol=REL, what=name + " grads vs oracle")


def test_chunk_size_does_not_matter():
    """1 row, a prime number of rows, a chunk whose boundaries fall inside utterances, and the whole batch at once."""
    k = random_joint(5, 13, 9, 17, 8, 11)
    args = joint_args(k)
    cells = r64.Cells(k["labels"], k["input_lengths"], k["label_lengths"], 13, 9, 0, "cpu")
    first = int(k["input_lengths"][0]) * (int(k["label_lengths"][0]) + 1)
    inside = first + 5
    assert 0 < inside - first < int(k["input_lengths"][1]) * (int(k["label_lengths"][1]) + 1)
    want = r64.joint_loss_grad(*args, grad_scale=np.linspace(0.5, 1.5, 5), fastemit_lambda=0.5, chunk_rows=cells.N)
    for rows in (1, 7, inside):
        pinned(r64.joint_loss_grad(*args, grad_scale=np.linspace(0.5, 1.5, 5), fastemit_lambda=0.5, chunk_rows=rows),
               want, "%d rows per chunk" % rows)
    x = fr._oracle.joint_forward(*[a for a in args[:4]])
    xt = r64.torch.as_tensor(x)
    shape = x.shape
    lab, il, ll = k["labels"], k["input_lengths"], k["label_lengths"]
    wc, wg = r64.op_loss_grad(lambda b, t, u: xt[b, t, u].clone(), shape, lab, il, ll, chunk_rows=cells.N)
    for rows in (1, 7, inside):
        c, g = r64.op_loss_grad(lambda b, t, u: xt[b, t, u].clone(), shape, lab, il, ll, chunk_rows=rows)
        assert_close(c, wc, rtol=REL, atol=0, what="op costs, %d rows" % rows)
        assert_close(g, wg, rtol=REL, atol=0, ntol=REL, what="op grads, %d rows" % rows)


def test_large_v_geometry():
    """tests/test_gpu_ref64.py's large-V cases run the dW kernel unsplit, have at least 5e5 valid rows, and (but V =
    8192) exceed the kept-numerator chunk budget by themselves; its loss-op lattices have more than 500 wavefront
    steps."""
    import test_gpu_ref64 as g
    for V, H in g.LARGE_V:
        assert g.dw_splits(H, V) == 1, (V, H)
        assert g.LV["B"] * g.LV["T"] * g.LV["U"] >= 5e5
        over = g.LV["B"] * g.padded_rows(g.LV["T"], g.LV["U"]) * (2 * V + 8) > g.CHUNK_BUDGET
        assert over == (V > 8192), (V, H)
    assert g.dw_splits(640, 4096) == 2 and g.dw_splits(640, 1024) == 11
    assert sum(T + U - 1 > 500 for T, U in g.OP_LENGTHS) == 2


def test_on_grad_receives_every_valid_cell_once():
    k = random_joint(3, 7, 5, 6, 4, 12)
    x = fr._oracle.joint_forward(*joint_args(k)[:4])
    xt = r64.torch.as_tensor(x)
    lab, il, ll = k["labels"], k["input_lengths"], k["label_lengths"]
    _, dense = r64.op_loss_grad(lambda b, t, u: xt[b, t, u].clone(), x.shape, lab, il, ll)
    seen = np.zeros(x.shape[:3], np.int64)
    got = np.zeros_like(dense)

    def sink(b, t, u, dl):
        np.add.at(seen, (b.numpy(), t.numpy(), u.numpy()), 1)
        got[b.numpy(), t.numpy(), u.numpy()] = dl.numpy()

    c, none = r64.op_loss_grad(lambda b, t, u: xt[b, t, u].clone(), x.shape, lab, il, ll, chunk_rows=4, on_grad=sink)
    assert none is None
    valid = np.zeros_like(seen)
    for b in range(3):
        valid[b, :il[b], :ll[b] + 1] = 1
    assert np.array_equal(seen, valid)
    assert_close(got, dense, rtol=REL, atol=0, ntol=REL, what="chunked sink")
