import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load(name):
    return dict(np.load(os.path.join(GOLDEN, name)))


def golden_names(prefix):
    return sorted(os.path.basename(p) for p in glob.glob(os.path.join(GOLDEN, prefix + "*.npz")))


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    return o


def fp32_tol(costs):
    """Tolerance policy of the parity tests (DESIGN.md, "Tolerances").

    north_star: fp32 rtol = 1e-4.  The absolute floor scales with the cost because every gradient
    entry is exp(alpha + beta + lp - ll) minus (sometimes) another such exponential, and the fp32
    round-off of an exponent of magnitude O(|ll|) is a few eps32 * |ll|: the UNMODIFIED reference library
    run in fp32 is itself 3e-5 (|cost| ~ 310), 4.5e-5 (|cost| ~ 450) and 9.6e-4 (|cost| ~ 1540, T=300)
    away from its own fp64 run -- i.e. up to 6.2e-7 * |cost|; the floor below is 1e-6 * |cost|.
    """
    cmax = float(np.max(np.abs(costs))) if np.size(costs) else 0.0
    return dict(rtol=1e-4, atol=1e-6 + 1e-6 * cmax)


def assert_close(a, b, rtol=1e-4, atol=1e-6, ntol=0.0, what=""):
    """|a-b| <= atol + ntol*max|b| + rtol*|b| elementwise.  ntol is the norm-wise term used for
    REDUCED gradients (d_enc, d_pred, dW, db): an fp32 sum of n terms carries eps32*sum|terms| of
    round-off, which is bounded by the tensor's scale, not by each (possibly cancelling) entry."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    bound = atol + ntol * (np.max(np.abs(b)) if b.size else 0.0) + rtol * np.abs(b)
    err = np.abs(a - b)
    bad = ~(err <= bound)            # catches NaN too
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(bound, 1e-300), 0)), a.shape)
        raise AssertionError("%s: %d/%d out of tolerance; worst at %s got %r want %r (bound %.3g)" %
                             (what, bad.sum(), a.size, i, a[i], b[i], bound[i]))
