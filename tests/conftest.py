import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a machine that has one")


class _Golden(dict):
    @property
    def files(self):
        return list(self)


def golden(name):
    """The arrays of tests/golden/<name>.npz and of its continuation files <name>.1.npz, <name>.2.npz, ... (a golden
    set is split where one file would exceed 1 MB)."""
    out, k, path = _Golden(), 0, os.path.join(GOLDEN, name + ".npz")
    while os.path.exists(path):
        with np.load(path) as z:
            out.update((key, z[key]) for key in z.files)
        k += 1
        path = os.path.join(GOLDEN, "%s.%d.npz" % (name, k))
    return out


def assert_close_to_max(a, b, rel=1e-5, what=""):
    """max|a-b| <= rel * max|b| over the whole array (per-cell relative error is meaningless
    for near-cancelling +- cells); NaN patterns must agree."""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    na, nb = np.isnan(a), np.isnan(b)
    assert (na == nb).all(), what + ": NaN pattern differs"
    if nb.all():
        return
    scale = np.abs(b[~nb]).max()
    err = np.abs(a[~nb] - b[~nb]).max() if (~nb).any() else 0.0
    assert err <= rel * max(scale, 1e-30), "%s: max err %.3e vs scale %.3e (rel %.2e > %.1e)" % (
        what, err, scale, err / max(scale, 1e-30), rel)


@pytest.fixture(scope="session")
def oracle():
    from oracle import evk_oracle
    evk_oracle.build()
    return evk_oracle


def make_events(seed, n, H, W, frac=True, tscale=0.1, pol="pm1", dtype=np.float32):
    rng = np.random.default_rng(seed)
    xs = rng.random(n) * (W - 1) if frac else rng.integers(0, W, n).astype(np.float64)
    ys = rng.random(n) * (H - 1) if frac else rng.integers(0, H, n).astype(np.float64)
    ts = np.sort(rng.random(n)) * tscale
    if pol == "pm1":
        ps = rng.integers(0, 2, n) * 2.0 - 1.0
    elif pol == "ones":
        ps = np.ones(n)
    else:
        ps = rng.standard_normal(n)
    return tuple(a.astype(dtype) for a in (xs, ys, ts, ps))
