import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "oracle", "_ref")
if os.path.isdir(os.path.join(REF, "cornac")) and REF not in sys.path:
    sys.path.insert(0, REF)          # the unmodified reference install (git-ignored, built by oracle/build_ref.sh)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def have_cornac():
    try:
        import cornac  # noqa: F401
        return True
    except Exception:
        return False


needs_cornac = pytest.mark.skipif(not have_cornac(), reason="reference cornac install (oracle/_ref) not importable")


def rel_err(a, b):
    """norm-wise relative error (SURVEY.md 7: element-wise rel is meaningless near 0)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def synth_csr(n_users, n_items, nnz, seed, zipf=0.8):
    """Unique (u,i) pairs, Zipf-ish item popularity -> (indptr, indices) int32, sorted rows."""
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** zipf
    p /= p.sum()
    u = rng.randint(n_users, size=int(nnz * 1.3))
    i = rng.choice(n_items, size=len(u), p=p)
    key = np.unique(u.astype(np.int64) * n_items + i)
    if len(key) > nnz:
        key = np.sort(rng.choice(key, size=nnz, replace=False))
    u, i = key // n_items, key % n_items
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    np.add.at(indptr, u + 1, 1)
    indptr = np.cumsum(indptr).astype(np.int32)
    return indptr, i.astype(np.int32)
