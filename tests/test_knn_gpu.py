"""UserKNN / ItemKNN on the GPU: the similarity kernel bit for bit against the compiled reference, the score kernels
against the oracle and the fixtures, the plug-ins against the reference's classes."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import golden, needs_cornac, synth_csr
from oracle import knn_oracle as KO
from test_knn_cpu import CASES, csr, raw_similarity

pytestmark = pytest.mark.gpu

TOL = 1e-12


def close(got, ref):
    got, ref = np.asarray(got), np.asarray(ref)
    return bool(np.all(np.abs(got - ref) <= TOL * np.maximum(1.0, np.abs(ref))))


def _engine():
    from cornac_b200 import engine
    engine.require_cuda()
    return engine


def _ratings_of(g):
    """(user_mode, device rating matrix) the scores of fixture g read, built from its own data and mean_arr."""
    engine = _engine()
    X = csr(g, "", int(g["num_items"]))
    ui = X.copy()
    if float(X.data.min()) != float(X.data.max()):
        ui.data = ui.data - np.repeat(g["mean_arr"], np.diff(ui.indptr))
        ui.data[ui.data == 0] = 1e-8
    user_mode = str(g["model"]) == "UserKNN"
    return user_mode, engine.KnnRatings(ui.T.tocsr() if user_mode else ui, g["mean_arr"]), ui


@pytest.mark.parametrize("name", CASES)
def test_similarity_is_bit_identical_to_the_reference(name):
    engine = _engine()
    g = golden(name)
    W = csr(g, "w_", int(g["w_cols"]))
    S, sim = engine.knn_similarity(W, 1.0)
    want = raw_similarity(g, W.shape[0])
    D = S.cpu().numpy()
    assert np.array_equal(D, want.toarray())
    assert np.array_equal(D, D.T)
    assert np.array_equal(sim.indptr, want.indptr) and np.array_equal(sim.indices, want.indices)
    assert np.array_equal(sim.data, want.data)
    S2, _ = engine.knn_similarity(W, 1.0)
    assert np.array_equal(S2.cpu().numpy(), D)
    S3, sim3 = engine.knn_similarity(W, float(g["amplify"]))
    ref_amp = csr(g, "sim_", W.shape[0])
    assert np.array_equal(sim3.indices, ref_amp.indices) and close(sim3.data, ref_amp.data)


@needs_cornac
@pytest.mark.parametrize("shape", [(2000, 1500, 150000), (10000, 3000, 60000)])
@pytest.mark.parametrize("kind", ["cosine", "pearson"])
def test_similarity_matches_compiled_compute_similarity(shape, kind):
    """An ML-1M-shaped slice (shared-memory accumulators) and 10 000 rows (workspace accumulators)."""
    from cornac.models.knn.similarity import compute_similarity
    from cornac_b200.recom_knn import _mean_centered
    engine = _engine()
    n, m, nnz = shape
    indptr, indices = synth_csr(n, m, nnz, seed=5)
    rng = np.random.RandomState(6)
    W = sp.csr_matrix((rng.randint(1, 6, size=len(indices)).astype(np.float64), indices, indptr), shape=(n, m))
    if kind == "pearson":
        W, _ = _mean_centered(W)
    S, sim = engine.knn_similarity(W, 1.0)
    ref = compute_similarity(W, num_threads=0, verbose=False)
    assert np.array_equal(sim.indptr, ref.indptr) and np.array_equal(sim.indices, ref.indices)
    assert np.array_equal(sim.data, ref.data)
    D = S.cpu().numpy()
    assert np.array_equal(D, D.T)
    S2, _ = engine.knn_similarity(W, 1.0)
    assert np.array_equal(S2.cpu().numpy(), D)


@pytest.mark.parametrize("name", CASES)
def test_score_rows_match_the_fixtures(name):
    engine = _engine()
    g = golden(name)
    user_mode, R, _ = _ratings_of(g)
    n = int(g["num_users"] if user_mode else g["num_items"])
    S = engine.knn_dense(csr(g, "sim_", n))
    got = engine.knn_score(user_mode, S, g["query_users"], R, int(g["k"])).cpu().numpy()
    assert close(got, g["query_scores"])
    again = engine.knn_score(user_mode, S, g["query_users"], R, int(g["k"])).cpu().numpy()
    assert np.array_equal(again, got)


@pytest.mark.parametrize("name", ["knn_user_cosine_k20", "knn_item_pearson_k5", "knn_item_tie_k3", "knn_user_tie_k3"])
@pytest.mark.parametrize("k", [1, 2, 7, 400, 1024])
def test_score_rows_match_the_oracle_for_any_k(name, k):
    """k = 1, k above every stream length (400, 1024: the sum-everything path) and the kept-pair path in between;
    k = 1024 also runs with the kept pairs in the workspace."""
    engine = _engine()
    g = golden(name)
    user_mode, R, ui = _ratings_of(g)
    n = int(g["num_users"] if user_mode else g["num_items"])
    sim = csr(g, "sim_", n)
    users = g["query_users"][:8]
    got = engine.knn_score(user_mode, engine.knn_dense(sim), users, R, k).cpu().numpy()
    if user_mode:
        iu, D = ui.T.tocsr(), sim.toarray()
        want = [g["mean_arr"][u] + KO.score_row(True, D[u], iu.indptr, iu.indices, iu.data, k) for u in users]
    else:
        want = [g["mean_arr"][u] + KO.score_row(False, ui[u].toarray().ravel(), sim.indptr, sim.indices, sim.data, k)
                for u in users]
    assert close(got, np.stack(want))


def _dataset(g):
    from cornac.data import Dataset
    return Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])], seed=None)


def _model(g):
    import cornac_b200
    kw = dict(k=int(g["k"]), similarity=str(g["similarity"]), mean_centered=bool(g["mean_centered"]),
              weighting=None if str(g["weighting"]) == "None" else str(g["weighting"]), amplify=float(g["amplify"]))
    return getattr(cornac_b200, str(g["model"]))(verbose=False, **kw)


def _check_model(m, g):
    assert np.array_equal(m.mean_arr, g["mean_arr"])
    ref = csr(g, "sim_", m.sim_mat.shape[0])
    assert np.array_equal(m.sim_mat.indptr, ref.indptr) and np.array_equal(m.sim_mat.indices, ref.indices)
    assert close(m.sim_mat.data, ref.data)
    rows = np.stack([m.score(int(u)) for u in g["query_users"]])
    assert rows.dtype == np.float64 and close(rows, g["query_scores"])
    single = np.array([m.score(int(u), int(i)) for u, i in g["single_pairs"]])
    assert close(single, g["single_scores"])
    for q, u in enumerate(g["query_users"]):
        ids, scores = m.rank(int(u), k=10)
        ref_ids, ref_sc = g["top10"][q], g["top10_scores"][q]
        assert close(scores[ids[:10]], ref_sc)
        full = g["query_scores"][q]
        cut = np.sort(full)[::-1][9]
        top = ids[:10]
        assert np.array_equal(top, top[np.lexsort((top, -full[top]))])     # score desc, id asc
        if np.sort(full)[::-1][10] != cut:          # no tie across the cut: the same ids (the reference orders ties by id desc)
            assert np.array_equal(np.sort(top), np.sort(ref_ids))
        else:
            assert np.array_equal(np.sort(full[ids[:10]]), np.sort(ref_sc))


@needs_cornac
@pytest.mark.parametrize("name", CASES)
def test_plugins_match_the_fixtures(name):
    g = golden(name)
    m = _model(g).fit(_dataset(g))
    _check_model(m, g)


@needs_cornac
def test_save_load_round_trip(tmp_path):
    from cornac.models import Recommender
    for name in ("knn_user_pearson_idf_k10", "knn_item_cosine_bm25_k20"):
        g = golden(name)
        m = _model(g).fit(_dataset(g))
        path = m.save(str(tmp_path / name))
        loaded = Recommender.load(path)
        assert loaded._b200_dev is None if hasattr(loaded, "_b200_dev") else True
        _check_model(loaded, g)


@needs_cornac
def test_experiment_matches_the_reference_classes():
    """The eight variants of the reference's examples/knn_movielens.py on an ML-100K-shaped split."""
    import cornac
    import cornac_b200
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, MAE, NDCG, RMSE, Recall
    rng = np.random.RandomState(100)
    indptr, indices = synth_csr(943, 1682, 100000, seed=100)
    users = np.repeat(np.arange(943), np.diff(indptr))
    data = [(str(u), str(i), float(r)) for u, i, r in zip(users, indices, rng.randint(1, 6, size=len(indices)))]
    K = 50
    variants = [("UserKNN", dict(similarity="cosine")), ("UserKNN", dict(similarity="pearson")),
                ("UserKNN", dict(similarity="cosine", amplify=2.0)), ("UserKNN", dict(similarity="cosine", weighting="idf")),
                ("UserKNN", dict(similarity="cosine", weighting="bm25")), ("ItemKNN", dict(similarity="cosine")),
                ("ItemKNN", dict(similarity="pearson")), ("ItemKNN", dict(similarity="cosine", mean_centered=True))]
    results = {}
    for lib in (cornac.models, cornac_b200):
        rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123)
        models = [getattr(lib, c)(k=K, name="%s-%d" % (c, j), verbose=False, **kw) for j, (c, kw) in enumerate(variants)]
        exp = cornac.Experiment(eval_method=rs, models=models, metrics=[RMSE(), MAE(), Recall(k=10), NDCG(k=10), AUC()],
                                verbose=False)
        exp.run()
        results[lib.__name__] = {r.model_name: r.metric_avg_results for r in exp.result}
    ref, ours = results["cornac.models"], results["cornac_b200"]
    assert set(ref) == set(ours) and len(ref) == 8
    for name in ref:
        for metric, tol in (("RMSE", 1e-9), ("MAE", 1e-9), ("Recall@10", 1e-6), ("NDCG@10", 1e-6), ("AUC", 1e-6)):
            assert abs(ours[name][metric] - ref[name][metric]) <= tol, (name, metric, ours[name][metric], ref[name][metric])


def test_oversize_similarity_is_refused_before_allocating():
    import torch
    from cornac_b200 import B200Error
    engine = _engine()
    n = 200000                                          # 320 GB dense
    W = sp.csr_matrix((np.ones(3), np.array([0, 1, 2], np.int32), np.r_[[0, 1, 2, 3], np.full(n - 3, 3)].astype(np.int32)),
                      shape=(n, 4))
    before = torch.cuda.memory_allocated()
    with pytest.raises(B200Error, match=str(n * n * 8)):
        engine.knn_similarity(W, 1.0)
    assert torch.cuda.memory_allocated() == before
