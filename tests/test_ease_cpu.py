"""EASE without a GPU: the committed fixtures against a fresh run of the reference, the ordered restatements of scipy's
Gram matrix and score rows that the kernels follow, the plug-in's constructor against the reference's, and the refusal of
the device entry points."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import golden, needs_cornac

CASES = ["ease_l500_pos", "ease_l500_all", "ease_l1_pos", "ease_l001_all", "ease_n1", "ease_n130", "ease_tie"]


def fixture_matrix(g):
    return sp.csr_matrix((g["X_data"], g["X_indices"], g["X_indptr"]), shape=(int(g["num_users"]), int(g["num_items"])))


def ordered_gram(X, lamb):
    """Sum over users in ascending order of X[u, a] * X[u, b], each product and sum rounded, then lamb on the diagonal."""
    X = X.tocsr()
    X.sort_indices()
    n = X.shape[1]
    G = np.zeros((n, n))
    for u in range(X.shape[0]):
        idx, val = X.indices[X.indptr[u]:X.indptr[u + 1]], X.data[X.indptr[u]:X.indptr[u + 1]]
        G[np.ix_(idx, idx)] = G[np.ix_(idx, idx)] + val[:, None] * val[None, :]
    G[np.diag_indices(n)] = G.diagonal() + lamb
    return G


def ordered_scores(X, B, users):
    """acc = +0.0, then acc = acc + x * B[i, :] over the stored (i, x) of the row, in stored order."""
    out = []
    for u in users:
        acc = np.zeros(B.shape[1])
        for p in range(X.indptr[u], X.indptr[u + 1]):
            acc = acc + X.data[p] * B[X.indices[p]]
        out.append(acc)
    return np.stack(out)


def non_dyadic(seed, n_users=120, n_items=70, density=0.15):
    rng = np.random.RandomState(seed)
    X = sp.random(n_users, n_items, density=density, random_state=rng, format="csr")
    X.data = rng.uniform(-2.0, 3.0, size=X.nnz) * np.pi
    return X


@needs_cornac
@pytest.mark.parametrize("name", CASES)
def test_fixtures_are_reproduced_by_the_reference(name):
    from cornac.data import Dataset
    from cornac.models import EASE
    g = golden(name)
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    m = EASE(lamb=float(g["lamb"]), posB=bool(g["posB"]), verbose=False).fit(Dataset.from_uir(data, seed=None))
    assert (m.U != fixture_matrix(g)).nnz == 0
    # np.linalg.inv's rounding depends on the BLAS kernels of the host: B to its rounding, the scores from it exactly
    assert np.max(np.abs(m.B - g["B"])) <= 1e-12 * max(np.max(np.abs(g["B"])), 1e-300)
    rows = np.stack([np.asarray(m.score(int(u))).ravel() for u in g["query_users"]])
    assert np.array_equal(rows.view(np.int64), ordered_scores(m.U, m.B, g["query_users"]).view(np.int64))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_ordered_gram_is_scipy(seed):
    X = non_dyadic(seed)
    want = X.T.dot(X).toarray()
    want[np.diag_indices(want.shape[0])] = want.diagonal() + 0.37
    assert np.array_equal(ordered_gram(X, 0.37), want)
    # the order matters: summing over users in descending order differs somewhere
    Xr = sp.csr_matrix(X.toarray()[::-1])
    assert not np.array_equal(ordered_gram(Xr, 0.37), want)


def test_ordered_scores_are_scipy():
    X = non_dyadic(4)
    B = np.random.RandomState(5).normal(size=(X.shape[1], X.shape[1]))
    users = np.arange(X.shape[0])
    assert np.array_equal(ordered_scores(X, B, users), X[users].dot(B))
    # rows whose only products are -0.0: scipy starts from +0.0, so they score +0.0 (a start from the first product: -0.0)
    Y = sp.csr_matrix((np.array([1.0, -1.0]), np.array([0, 1]), np.array([0, 1, 2])), shape=(2, 2))
    Bz = np.array([[-0.0, 1.0], [0.0, 1.0]])
    want = Y.dot(Bz)
    assert not np.signbit(want[0, 0]) and not np.signbit(want[1, 0])
    assert np.array_equal(ordered_scores(Y, Bz, [0, 1]).view(np.int64), want.view(np.int64))


@pytest.mark.parametrize("name", CASES)
def test_fixture_scores_follow_the_ordered_restatement(name):
    g = golden(name)
    X = fixture_matrix(g)
    got = ordered_scores(X, g["B"], g["query_users"])
    assert np.array_equal(got.view(np.int64), g["query_scores"].view(np.int64))


@needs_cornac
def test_constructor_matches_the_reference():
    from cornac.models import EASE as Ref
    from cornac_b200 import EASE
    ref, ours = Ref(), EASE()
    for a in ("name", "lamb", "posB", "trainable", "verbose", "seed", "B", "U"):
        assert getattr(ours, a) == getattr(ref, a), a
    m = EASE(name="x", lamb=3.5, posB=False, trainable=False, verbose=False, seed=4)
    c = m.clone()
    assert (c.name, c.lamb, c.posB, c.trainable, c.verbose, c.seed) == ("x", 3.5, False, False, False, 4)
    c2 = m.clone(dict(lamb=7))
    assert c2.lamb == 7 and c2.posB is False
    assert "_b200_dev" in m.ignored_attrs and "_b200_eval_cache" in m.ignored_attrs


def test_entry_points_refuse_without_a_gpu(monkeypatch):
    import torch
    from cornac_b200 import B200Error, engine
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    X = sp.random(10, 8, density=0.5, format="csr", random_state=0)
    with pytest.raises(B200Error):
        engine.ease_fit(X, 500.0, True)
    with pytest.raises(B200Error):
        engine.EaseRatings(X)
    with pytest.raises(B200Error):
        engine.ease_score(None, [0], None)
