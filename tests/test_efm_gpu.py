"""EFM on the GPU: the fit bit-identical to the C oracle, the exact-dot fixture equal to the compiled reference, the rank
queries equal to the oracle, the rank rows against the reference's EFM.rank, and the plug-in's scoring, ranking,
persistence and Experiment contract."""
import contextlib
import io

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import golden, needs_cornac
from oracle import efm_oracle as EO
from oracle import oracle as O
from test_efm_cpu import CASES, FACTORS, fixture_helpers, hyper, matrices, train_set

pytestmark = pytest.mark.gpu


def device(xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x).copy()).cuda() for x in xs]


def host(ds):
    return [d.cpu().numpy() for d in ds]


def gpu_fit(data, init, n_iter, g):
    from cornac_b200 import engine
    d = device(init)
    engine.efm_fit(data, *d, n_iter, **hyper(g))
    return host(d)


@pytest.mark.parametrize("case", CASES)
def test_fit_equals_oracle(case):
    from cornac_b200 import engine
    g = golden(case)
    A, X, Y = matrices(g)
    data = engine.EfmData(A, X, Y)
    init = [g[f + "0"] for f in FACTORS]
    for n_iter in sorted({1, 4, *[int(m) for m in g["max_iters"]]}):
        want = [x.copy() for x in init]
        EO.fit(A, X, Y, *want, n_iter, **hyper(g))
        got = gpu_fit(data, init, n_iter, g)
        for f, a, b in zip(FACTORS, got, want):
            assert np.array_equal(a, b), (case, n_iter, f)
    # two calls of 2 and 3 iterations are one call of 5
    d = device(init)
    engine.efm_fit(data, *d, 2, **hyper(g))
    engine.efm_fit(data, *d, 3, **hyper(g))
    assert all(np.array_equal(a, b) for a, b in zip(host(d), gpu_fit(data, init, 5, g)))


def test_long_chains_equal_oracle():
    """Rows and columns far longer than a warp: 2 000 users x 500 items x 40 aspects, E = 40, L = 60."""
    from cornac_b200 import engine
    rng = np.random.RandomState(7)

    def sparse(n_rows, n_cols, nnz):
        key = rng.choice(n_rows * n_cols, size=nnz, replace=False)
        return sp.csr_matrix((rng.uniform(1, 5, nnz).astype(np.float32), (key // n_cols, key % n_cols)),
                             shape=(n_rows, n_cols))

    A, X, Y = sparse(2000, 500, 40000), sparse(2000, 40, 20000), sparse(500, 40, 8000)
    init = [rng.uniform(0, 0.3, s).astype(np.float32) for s in ((2000, 40), (500, 40), (40, 40), (2000, 60), (500, 60))]
    g = dict(lambda_x=1.0, lambda_y=1.0, lambda_u=0.01, lambda_h=0.01, lambda_v=0.01)
    want = [x.copy() for x in init]
    EO.fit(A, X, Y, *want, 3, **g)
    got = gpu_fit(engine.EfmData(A, X, Y), init, 3, dict((k, np.array(v)) for k, v in g.items()))
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_exact_dot_equals_reference():
    from cornac_b200 import engine
    g = golden("efm_exact")
    got = gpu_fit(engine.EfmData(*matrices(g)), [g[f + "0"] for f in FACTORS], 1, g)
    for f, a in zip(FACTORS, got):
        assert np.array_equal(a, g[f + "_1"]), f


@pytest.mark.parametrize("case", CASES)
def test_queries_equal_oracle(case):
    import torch
    from cornac_b200 import engine
    g = golden(case)
    mi = int(g["max_iters"][-1])
    U1, H1, V = (g["%s_%d" % (f, mi)] for f in ("U1", "H1", "V"))
    N, alpha, s = int(g["num_most_cared_aspects"]), float(g["alpha"]), float(g["rating_scale"])
    users = np.arange(U1.shape[0])
    for n in (N, 1, V.shape[0] + 3):
        Q = engine.efm_queries(*device([U1, H1, V]), n, alpha, s)
        assert np.array_equal(Q.cpu().numpy(), EO.queries(users, U1, H1, V, n, alpha, s)), (case, n)
    sub = torch.tensor([3, 0, 3], dtype=torch.int64, device="cuda")
    Q = engine.efm_queries(*device([U1, H1, V]), N, alpha, s, user_idx=sub)
    assert np.array_equal(Q.cpu().numpy(), EO.queries([3, 0, 3], U1, H1, V, N, alpha, s))


def _model(g, mi=None):
    """The plug-in holding a fixture's factors after its last fit (no training)."""
    from cornac_b200 import EFM
    mi = int(g["max_iters"][-1]) if mi is None else mi
    kw = {k: g[k].item() for k in ("num_explicit_factors", "num_latent_factors", "num_most_cared_aspects",
                                   "rating_scale", "alpha")}
    model = EFM(trainable=False, init_params={f: g["%s_%d" % (f, mi)].copy() for f in FACTORS}, **kw)
    return model.fit(train_set(g))


@needs_cornac
@pytest.mark.parametrize("case", CASES)
def test_rank_rows_and_topk(case):
    g = golden(case)
    model = _model(g)
    U1, U2, V, H1, H2 = (np.asarray(getattr(model, f)) for f in FACTORS)
    Q = EO.queries(np.arange(U1.shape[0]), U1, H1, V, model.num_most_cared_aspects, model.alpha, model.rating_scale)
    W = np.concatenate([U2, H2], axis=1)
    rows = O.score_batch(Q, W)
    users = np.arange(U1.shape[0])
    ids, sc = model.rank_batch(users, 10)
    for q in users:
        wi, ws, _ = O.topk(rows[q], 10)
        assert np.array_equal(ids[q], wi) and np.array_equal(sc[q], ws), (case, q)
    # against the reference's EFM.rank: an f32 error bound from the magnitudes, and the top ids away from near-ties
    mag = np.abs(Q).astype(np.float64) @ np.abs(W).T.astype(np.float64)
    for q, u in enumerate(g["rank_users"]):
        ranked, scores = model.rank(int(u))
        want = g["rank_scores"][q]
        assert np.array_equal(scores, rows[u])
        assert np.all(np.abs(scores - want) <= 1e-5 * (mag[u] + np.abs(want)) + 1e-6), (case, u)
        order = np.lexsort((np.arange(len(want)), -want))
        gap = np.abs(np.diff(want[order[:11]]))
        if gap.min() > 1e-4 * np.max(np.abs(want)):
            assert np.array_equal(ranked[:10], order[:10]), (case, u)
        # score(u) is the plain row, not the rank row
        plain = model.score(int(u))
        assert np.array_equal(plain, O.score_batch(np.concatenate([U1, H1], axis=1)[u:u + 1], W)[0])
        assert np.max(np.abs(plain - g["score_rows"][q])) <= 1e-5 * np.max(np.abs(g["score_rows"][q]))
        assert not np.array_equal(plain, scores)
    with pytest.raises(IndexError):
        model.rank(U1.shape[0] + 5)


@needs_cornac
def test_plugin_contract(tmp_path):
    from cornac.exception import ScoreException
    from cornac_b200 import EFM
    g = golden("efm_odd")
    ts = train_set(g)
    kw = dict(num_explicit_factors=7, num_latent_factors=37, num_most_cared_aspects=4, max_iter=6)
    init = {f: g[f + "0"].copy() for f in FACTORS}
    with contextlib.redirect_stdout(io.StringIO()):
        model = EFM(init_params=init, **kw).fit(ts)
    # trained in place, equal to the oracle
    want = [g[f + "0"].copy() for f in FACTORS]
    EO.fit(*matrices(g), *want, 6, **hyper(g))
    for f, w in zip(FACTORS, want):
        assert getattr(model, f) is init[f] and np.array_equal(init[f], w), f
    assert model.num_aspects == int(g["num_aspects"])
    one = model.score(2, 5)
    assert one == model.U2[5].dot(model.U1[2]) + model.H2[5].dot(model.H1[2])
    with pytest.raises(ScoreException):
        model.score(ts.num_users + 3)
    users = np.arange(12)
    ids, sc = model.rank_batch(users, 6)
    for q, u in enumerate(users):
        ranked, scores = model.rank(int(u), k=6)
        assert np.array_equal(ranked[:6], ids[q]) and np.array_equal(scores[ids[q]], sc[q])
    recs = model.recommend_batch([ts.user_ids[u] for u in users], k=6)
    assert [[ts.iid_map[i] for i in r] for r in recs] == ids.tolist()
    # the transform() cache serves the same rank rows and does not change score(u)
    plain = model.score(3)
    ranked, scores = model.rank(3)
    model.transform(ts)
    assert model._b200_eval_cache is not None
    r2, s2 = model.rank(3)
    assert np.array_equal(r2, ranked) and np.array_equal(s2, scores) and np.array_equal(model.score(3), plain)
    # save / load
    loaded = EFM.load(model.save(str(tmp_path)))
    assert np.array_equal(loaded.rank(3)[1], scores) and np.array_equal(loaded.score(3), plain)
    # trainable=False keeps the given factors
    frozen = EFM(trainable=False, init_params={f: getattr(model, f).copy() for f in FACTORS}, **kw).fit(ts)
    assert np.array_equal(frozen.rank(3)[1], scores)
    # dtype / shape errors and a missing modality
    with pytest.raises(ValueError, match="Buffer dtype mismatch"):
        EFM(init_params={"U1": g["U10"].astype(np.float64)}, **kw).fit(ts)
    with pytest.raises(ValueError, match="must have shape"):
        EFM(init_params={"V": g["V0"][:, :3].copy()}, **kw).fit(ts)
    from cornac.data import Dataset
    bare = Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])], seed=1)
    with pytest.raises(ValueError, match="sentiment"):
        EFM(**kw).fit(bare)


@needs_cornac
def test_batched_ranking_eval_equals_per_user():
    from cornac.data import SentimentModality
    from cornac.eval_methods import RatioSplit
    from cornac.eval_methods.base_method import ranking_eval as ref_ranking_eval
    from cornac.metrics import AUC, MAP, NDCG, Recall
    from cornac_b200 import EFM
    from cornac_b200.evaluation import ranking_eval
    unpack_reviews = fixture_helpers().unpack_reviews
    g = golden("efm_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123,
                    sentiment=SentimentModality(data=unpack_reviews(g)))
    model = EFM(num_explicit_factors=8, num_latent_factors=12, num_most_cared_aspects=5, max_iter=20, seed=123)
    model.fit(rs.train_set)
    metrics = [NDCG(k=50), AUC(), Recall(k=10), MAP()]
    mine, _ = ranking_eval(model, metrics, rs.train_set, rs.test_set, rating_threshold=1.0, exclude_unknowns=True)
    ref, _ = ref_ranking_eval(model, metrics, rs.train_set, rs.test_set, rating_threshold=1.0, exclude_unknowns=True)
    assert np.allclose(mine, ref, rtol=1e-12, atol=1e-12)


@needs_cornac
def test_experiment_metrics_match_the_reference(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    import cornac
    from cornac.data import SentimentModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, NDCG, RMSE, Recall
    from cornac_b200 import EFM
    unpack_reviews = fixture_helpers().unpack_reviews
    g = golden("efm_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123,
                    sentiment=SentimentModality(data=unpack_reviews(g)))
    metrics = [RMSE(), NDCG(k=50), AUC(), Recall(k=10)]
    assert [m.name for m in metrics] == list(g["metric_names"])
    with contextlib.redirect_stdout(io.StringIO()):
        exp = cornac.Experiment(eval_method=rs, models=[EFM(num_explicit_factors=8, num_latent_factors=12,
                                                            num_most_cared_aspects=5, max_iter=20, seed=123)],
                                metrics=metrics, user_based=True, verbose=False)
        exp.run()
    got = np.array([exp.result[0].metric_avg_results[m.name] for m in metrics])
    # the fit agrees with the reference to f32 rounding (its sdot order is unspecified), so the metrics agree closely
    assert np.all(np.abs(got - g["metrics"]) <= 2e-3), (got, g["metrics"])
