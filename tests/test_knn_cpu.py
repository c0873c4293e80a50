"""UserKNN / ItemKNN without a GPU: the numpy oracle against the compiled reference's fixtures, the plug-ins' host
preprocessing against the reference's helpers, constructor validation, and the refusal of the device entry points."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import golden, needs_cornac
from oracle import knn_oracle as KO

CASES = ["knn_user_cosine_k20", "knn_user_pearson_idf_k10", "knn_item_cosine_bm25_k20", "knn_item_pearson_k5",
         "knn_item_implicit_k20", "knn_user_implicit_k20", "knn_item_tie_k3", "knn_user_tie_k3"]


def csr(g, p, n_cols):
    n = len(g[p + "indptr"]) - 1
    return sp.csr_matrix((g[p + "data"], g[p + "indices"], g[p + "indptr"]), shape=(n, n_cols))


def raw_similarity(g, n):
    """compute_similarity's own output (before the amplify map); stored only where amplify != 1, else it is sim_mat."""
    return csr(g, "raw_" if "raw_data" in g.files else "sim_", n)


def oracle_similarity(g, denominator="compiled"):
    return KO.similarity(g["w_indptr"], g["w_indices"], g["w_data"], int(g["w_cols"]), denominator)


def oracle_scores(g, users):
    """Score rows from the fixture's own sim_mat and the mean-centred rating matrix."""
    n_u, n_i = int(g["num_users"]), int(g["num_items"])
    X = csr(g, "", n_i)
    ui = X.copy()
    ui.data = ui.data - np.repeat(g["mean_arr"], np.diff(ui.indptr)) if float(X.data.min()) != float(X.data.max()) else ui.data
    ui.data[ui.data == 0] = 1e-8
    out = []
    if str(g["model"]) == "UserKNN":
        S = csr(g, "sim_", n_u).toarray()
        iu = ui.T.tocsr()
        for u in users:
            out.append(g["mean_arr"][u] + KO.score_row(True, S[u], iu.indptr, iu.indices, iu.data, int(g["k"])))
    else:
        S = csr(g, "sim_", n_i)
        for u in users:
            out.append(g["mean_arr"][u] + KO.score_row(False, ui[u].toarray().ravel(), S.indptr, S.indices, S.data, int(g["k"])))
    return np.stack(out)


@pytest.mark.parametrize("name", CASES)
def test_oracle_similarity_is_bit_identical_to_the_reference(name):
    g = golden(name)
    got = oracle_similarity(g)
    want = raw_similarity(g, got.shape[0]).toarray()
    assert np.array_equal(got, want)
    assert np.array_equal(got, got.T)
    amp = KO.amplify(got, float(g["amplify"]))
    np.testing.assert_allclose(amp, csr(g, "sim_", got.shape[0]).toarray(), rtol=1e-15, atol=0)


def test_compiled_reference_uses_the_fused_denominator():
    """-ffast-math turns sqrt(D1) * sqrt(D2) into sqrt(D1 * D2): on implicit data every similarity is then exactly 1.0,
    where the source formula gives 1 +- 1 ulp for some pairs."""
    g = golden("knn_item_implicit_k20")
    want = raw_similarity(g, int(g["num_items"])).toarray()
    assert set(np.unique(want[want != 0]).tolist()) == {1.0}
    assert not np.array_equal(oracle_similarity(g, "source"), want)


@pytest.mark.parametrize("name", CASES)
def test_oracle_scores_match_the_reference(name):
    g = golden(name)
    users = g["query_users"]
    got = oracle_scores(g, users)
    ref = g["query_scores"]
    assert np.all(np.abs(got - ref) <= 1e-12 * np.maximum(1.0, np.abs(ref)))


def test_tie_fixture_separates_tie_rules():
    """Keeping the largest values of a tie group instead of the reference's rule moves the tie case's scores far."""
    g = golden("knn_item_tie_k3")
    wrong = KO.select
    try:
        KO.select = lambda cand, k: sorted(cand, key=lambda p: (p[0], p[1]))[-k:]
        moved = oracle_scores(g, g["query_users"])
    finally:
        KO.select = wrong
    assert np.max(np.abs(moved - g["query_scores"])) > 1e-3


# ---- the plug-ins' host preprocessing ------------------------------------------------------------------------------
def _dataset(g):
    from cornac.data import Dataset
    X = csr(g, "", int(g["num_items"])).tocoo()
    return Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(X.row, X.col, X.data)], seed=None)


@needs_cornac
@pytest.mark.parametrize("name", CASES)
def test_host_preprocessing_matches_the_reference(name):
    from cornac.models import Recommender
    from cornac.models.knn import recom_knn as R
    from cornac_b200 import recom_knn as M
    g = golden(name)
    ds = _dataset(g)
    cls = getattr(M, str(g["model"]))
    kw = dict(k=int(g["k"]), similarity=str(g["similarity"]), mean_centered=bool(g["mean_centered"]),
              weighting=None if str(g["weighting"]) == "None" else str(g["weighting"]), amplify=float(g["amplify"]))
    m = cls(**kw)
    Recommender.fit(m, ds)
    seen = {}
    real = R.compute_similarity

    def spy(data_mat, **a):
        seen["w"] = data_mat.tocsr().copy()
        return real(data_mat, **a)

    R.compute_similarity = spy
    try:
        ref = getattr(R, str(g["model"]))(verbose=False, **kw).fit(ds)
    finally:
        R.compute_similarity = real
    m_w, m_ui, m_mean = m._host_prepare(ds)
    assert np.array_equal(m_mean, ref.mean_arr)
    ref_w = seen["w"]
    assert np.array_equal(m_w.indptr, ref_w.indptr) and np.array_equal(m_w.indices, ref_w.indices)
    assert np.array_equal(m_w.data, ref_w.data)
    m._keep_ratings(m_ui)
    kept = "iu_mat" if str(g["model"]) == "UserKNN" else "ui_mat"
    assert (getattr(m, kept) != getattr(ref, kept)).nnz == 0
    # the reference's own helpers on arbitrary float data (not only small integers)
    rng = np.random.RandomState(3)
    Y = sp.random(40, 30, density=0.3, random_state=rng, format="csr")
    Y.data = rng.normal(size=Y.nnz)
    a, ma = R._mean_centered(Y.copy())
    b, mb = M._mean_centered(Y.copy())
    assert np.array_equal(ma, mb) and np.array_equal(a.data, b.data)


@needs_cornac
def test_constructor_validation_matches_the_reference():
    from cornac.models import ItemKNN as RI, UserKNN as RU
    from cornac_b200 import ItemKNN, UserKNN
    for ours, ref in ((UserKNN, RU), (ItemKNN, RI)):
        for bad in (dict(similarity="jaccard"), dict(weighting="tfidf")):
            with pytest.raises(ValueError) as e_ref:
                ref(**bad)
            with pytest.raises(ValueError) as e_ours:
                ours(**bad)
            assert str(e_ours.value) == str(e_ref.value)
        for k in (0, -3):
            with pytest.raises(ValueError):
                ours(k=k)
        m = ours(k=7, similarity="pearson", mean_centered=True, weighting="bm25", amplify=1.5, seed=3)
        assert (m.k, m.similarity, m.mean_centered, m.weighting, m.amplify, m.num_threads) == (7, "pearson", True, "bm25", 1.5, 1)


def test_entry_points_refuse_without_a_gpu(monkeypatch):
    import torch
    from cornac_b200 import B200Error, engine
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    X = sp.random(10, 8, density=0.5, format="csr", random_state=0)
    with pytest.raises(B200Error):
        engine.knn_similarity(X, 1.0)
    with pytest.raises(B200Error):
        engine.knn_score(False, None, [0], None, 5)
    with pytest.raises(B200Error):
        engine.KnnRatings(X, np.zeros(10))
