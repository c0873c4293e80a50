"""EFM without a GPU: the host matrices against the compiled reference's _build_matrices, the C oracle of the fit against
the reference's fixtures, and the semantics of the rank queries."""
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import GOLDEN, golden, needs_cornac
from oracle import efm_oracle as EO

FACTORS = ("U1", "U2", "V", "H1", "H2")
CASES = ("efm_default", "efm_odd", "efm_nopop", "efm_lambdas", "efm_sparse", "efm_bign", "efm_tie", "efm_exact")
# Largest |oracle - reference| / max|reference| per factor matrix over every fixture and max_iter (up to 10), measured
# on x86-64 against the reference built with scipy's OpenBLAS: 5.2e-7 (efm_default, V after 10 iterations).  The
# reference's sdot order is unspecified, so the two differ by the rounding of the predictions, which the iterations
# carry forward.  Pinned with a 4x margin.
ORACLE_BOUND = 2e-6


def matrices(g):
    return tuple(sp.csr_matrix((g[m + "_data"], g[m + "_indices"], g[m + "_indptr"]), shape=shape)
                 for m, shape in (("A", (int(g["num_users"]), int(g["num_items"]))),
                                  ("X", (int(g["num_users"]), int(g["num_aspects"]))),
                                  ("Y", (int(g["num_items"]), int(g["num_aspects"])))))


def hyper(g):
    return {k: float(g[k]) for k in ("lambda_x", "lambda_y", "lambda_u", "lambda_h", "lambda_v")}


def fixture_helpers():
    """tests/golden/make_golden_efm.py, whose train_set / unpack_reviews rebuild a fixture's train set and reviews."""
    sys.path.insert(0, GOLDEN)
    try:
        import make_golden_efm
    finally:
        sys.path.remove(GOLDEN)
    return make_golden_efm


def train_set(g):
    return fixture_helpers().train_set(g)


def query_restatement(users, U1, H1, V, N, alpha, s):
    """b200_efm_queries in numpy: the top aspects by a stable sort on (-X_, id)."""
    E = U1.shape[1]
    acc = np.zeros((len(U1), len(V)))
    for f in range(E):                        # the defined dot: f64, index order
        acc = acc + U1[:, f:f + 1].astype(np.float64) * V[:, f].astype(np.float64)[None, :]
    X_ = acc.astype(np.float32)
    c, beta = alpha / (N * s), 1.0 - alpha
    out = []
    for u in users:
        top = np.lexsort((np.arange(len(V)), -X_[u].astype(np.float64)))[: min(N, len(V))]
        acc = np.zeros(E)
        for a in top:
            acc = acc + np.float64(X_[u, a]) * V[a].astype(np.float64)
        out.append(np.concatenate([(c * acc + beta * U1[u].astype(np.float64)).astype(np.float32),
                                   (beta * H1[u].astype(np.float64)).astype(np.float32)]))
    return np.stack(out)


@needs_cornac
@pytest.mark.parametrize("case", CASES + ("efm_experiment",))
def test_host_matrices_equal_reference(case):
    from cornac_b200.recom_efm import build_matrices
    g = golden(case)
    ts = train_set(g)
    if case == "efm_experiment":
        import cornac
        want = cornac.models.EFM(max_iter=0, seed=1).fit(ts)._build_matrices(ts)
        n_aspects = ts.sentiment.num_aspects
        s, pop = 5.0, True
    else:
        want = matrices(g)
        n_aspects, s, pop = int(g["num_aspects"]), float(g["rating_scale"]), bool(g["use_item_aspect_popularity"])
    got = build_matrices(ts, ts.num_users, ts.num_items, n_aspects, s, pop)
    for gm, wm in zip(got, want):
        assert gm.shape == wm.shape
        assert np.array_equal(gm.indptr, wm.indptr) and np.array_equal(gm.indices, wm.indices)
        assert gm.data.dtype == np.float32 and np.array_equal(gm.data, wm.data.astype(np.float32))


def test_fixture_edges():
    """The fixtures hold what they are meant to: empty X / Y rows, an aspect nobody mentions, a stored zero rating,
    N > n_aspects, long aspect columns."""
    A, X, Y = matrices(golden("efm_sparse"))
    assert np.any(np.diff(X.indptr) == 0) and np.any(np.diff(Y.indptr) == 0)
    assert np.any((X.getnnz(axis=0) + Y.getnnz(axis=0)) == 0)
    assert np.any(A.data == 0)
    g = golden("efm_bign")
    assert int(g["num_most_cared_aspects"]) > int(g["num_aspects"])
    A, X, Y = matrices(golden("efm_default"))
    assert (X.getnnz(axis=0) + Y.getnnz(axis=0)).max() > 64 and A.getnnz(axis=0).max() > 32


def test_oracle_exact_dot_equals_reference():
    """Dyadic start: every prediction is exact in any order, so one iteration of the oracle is the reference's, bit for
    bit -- the chain order, the lambda grouping and the f32 sqrt."""
    g = golden("efm_exact")
    fs = [g[f + "0"].copy() for f in FACTORS]
    EO.fit(*matrices(g), *fs, 1, **hyper(g))
    for f, x in zip(FACTORS, fs):
        assert np.array_equal(x, g[f + "_1"]), f


@pytest.mark.parametrize("case", CASES)
def test_oracle_within_bound_of_reference(case):
    g = golden(case)
    A, X, Y = matrices(g)
    for mi in g["max_iters"]:
        fs = [g[f + "0"].copy() for f in FACTORS]
        EO.fit(A, X, Y, *fs, int(mi), **hyper(g))
        for f, x in zip(FACTORS, fs):
            want = g["%s_%d" % (f, mi)]
            scale = max(float(np.max(np.abs(want))), 1e-30)
            assert float(np.max(np.abs(x - want))) <= ORACLE_BOUND * scale, (case, int(mi), f)
        if case == "efm_sparse":
            dead = (X.getnnz(axis=0) + Y.getnnz(axis=0)) == 0
            assert int(mi) == 0 or np.all(fs[2][dead] == 0)


def test_oracle_split_iterations():
    g = golden("efm_odd")
    A, X, Y = matrices(g)
    one = [g[f + "0"].copy() for f in FACTORS]
    EO.fit(A, X, Y, *one, 5, **hyper(g))
    two = [g[f + "0"].copy() for f in FACTORS]
    EO.fit(A, X, Y, *two, 2, **hyper(g))
    EO.fit(A, X, Y, *two, 3, **hyper(g))
    assert all(np.array_equal(a, b) for a, b in zip(one, two))


@pytest.mark.parametrize("n_aspects,N", [(30, 15), (10, 25), (0, 15), (12, 12), (6, 1)])
def test_query_semantics(n_aspects, N):
    rng = np.random.RandomState(n_aspects + N)
    U1 = rng.uniform(0, 1, (20, 7)).astype(np.float32)
    H1 = rng.uniform(0, 1, (20, 5)).astype(np.float32)
    V = rng.uniform(0, 1, (n_aspects, 7)).astype(np.float32)
    if n_aspects >= 4:                        # exact ties in X_: equal rows (the smaller id first)
        V[3] = V[1]
        V[2] = V[0]
    users = np.array([0, 3, 19, 3])
    got = EO.queries(users, U1, H1, V, N, 0.85, 5.0)
    assert np.array_equal(got, query_restatement(users, U1, H1, V, N, 0.85, 5.0))
    if n_aspects == 0:                        # no aspect: the query is (1 - alpha) times the user's factors
        assert np.array_equal(got[:, :7], ((1 - 0.85) * U1[users].astype(np.float64)).astype(np.float32))
