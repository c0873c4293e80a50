"""PMF on the GPU: b200_pmf_fit bit-identical to the compiled reference's fixtures and to the serial oracle, the f64 scores
and top-k, the exhaustive sigmoid check, and the plug-in through save / load and an unchanged Experiment."""
import io
import tempfile
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from conftest import golden, needs_cornac, synth_csr
from oracle import pmf_oracle as PO

pytestmark = pytest.mark.gpu

FIT_CASES = ["pmf_linear_k5", "pmf_linear_k10_mid", "pmf_nonlinear_k10", "pmf_nonlinear_unit", "pmf_linear_init_u_k7",
             "pmf_nonlinear_k1", "pmf_linear_k1"]


def device_fit(uid, iid, rat, n_users, n_items, variant, U0, V0, n_epochs, lam, lr, gamma, loss=False, split=None):
    from cornac_b200 import engine
    data = engine.PmfData(uid, iid, rat, n_users, n_items)
    U, V = engine.to_device(U0, torch.float64), engine.to_device(V0, torch.float64)
    cu, cv = torch.zeros_like(U), torch.zeros_like(V)
    terms = torch.empty((n_epochs, len(uid)), dtype=torch.float64, device="cuda") if loss else None
    if split is None:
        engine.pmf_fit(data, variant, U, V, cu, cv, n_epochs, lam, lr, gamma, loss=terms)
    else:                                                     # two calls of a and b epochs == one call of a + b
        engine.pmf_fit(data, variant, U, V, cu, cv, split, lam, lr, gamma)
        engine.pmf_fit(data, variant, U, V, cu, cv, n_epochs - split, lam, lr, gamma)
    out = (U.cpu().numpy(), V.cpu().numpy())
    return out + (terms.cpu().numpy(),) if loss else out


def _hyper(g):
    return float(g["lambda_reg"]), float(g["learning_rate"]), float(g["gamma"])


def _dataset(u, i, r):
    from cornac.data import Dataset
    return Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)], seed=None)


@pytest.mark.parametrize("name", FIT_CASES)
def test_fit_is_bit_identical_to_the_reference(name):
    g = golden(name)
    U, V = device_fit(g["uid"], g["iid"], g["rat"], int(g["num_users"]), int(g["num_items"]), str(g["variant"]),
                      g["U0"], g["V0"], int(g["max_iter"]), *_hyper(g))
    assert np.array_equal(U, g["U"]) and np.array_equal(V, g["V"])


def test_split_calls_and_loss_terms_equal_the_reference():
    g = golden("pmf_nonlinear_k10")
    args = (g["uid"], g["iid"], g["rat"], int(g["num_users"]), int(g["num_items"]), "non_linear", g["U0"], g["V0"],
            int(g["max_iter"])) + _hyper(g)
    U, V = device_fit(*args, split=7)
    assert np.array_equal(U, g["U"]) and np.array_equal(V, g["V"])
    U, V, terms = device_fit(*args, loss=True)
    assert np.array_equal(np.add.accumulate(terms, axis=1)[:, -1], g["loss"])
    _, want = PO.pmf_fit("non_linear", g["uid"], g["iid"], g["rat"], g["U0"].copy(), g["V0"].copy(), int(g["max_iter"]),
                         *_hyper(g), terms=True)
    assert np.array_equal(terms, want)


@pytest.mark.parametrize("variant", ["linear", "non_linear"])
@pytest.mark.parametrize("order", ["shuffled", "csr"])
def test_ml1m_shape_is_bit_identical_to_the_oracle(variant, order):
    indptr, indices = synth_csr(6040, 3706, 1000000, seed=3)
    rng = np.random.RandomState(4)
    uid = np.repeat(np.arange(6040), np.diff(indptr)).astype(np.int32)
    iid = indices.astype(np.int32)
    if order == "shuffled":
        p = rng.permutation(len(uid))
        uid, iid = uid[p], iid[p]
    rat = rng.randint(1, 6, size=len(uid)).astype(np.float32)
    if variant == "non_linear":
        rat = (rat - np.float32(1)) / np.float32(4)
    U0, V0 = rng.normal(0, 0.001, (6040, 10)), rng.normal(0, 0.001, (3706, 10))
    U, V = device_fit(uid, iid, rat, 6040, 3706, variant, U0, V0, 3, 0.001, 0.001, 0.9)
    Uo, Vo = U0.copy(), V0.copy()
    PO.pmf_fit(variant, uid, iid, rat, Uo, Vo, 3, 0.001, 0.001, 0.9)
    assert np.array_equal(U, Uo) and np.array_equal(V, Vo)


def test_sigmoid_is_exact_for_every_float_in_range():
    """Every f32 z in [-6, 6] (both signs of zero included): the device sigmoid equals the oracle's libm expf one."""
    from cornac_b200 import engine
    six, msix = int(np.float32(6).view(np.uint32)), int(np.float32(-6).view(np.uint32))
    chunk = 1 << 27
    host = np.empty(chunk, dtype=np.float32)
    n_checked = 0
    for lo, hi in ((0, six + 1), (0x80000000, msix + 1)):
        for first in range(lo, hi, chunk):
            n = min(chunk, hi - first)
            start = first - (1 << 32) if first >= (1 << 31) else first
            z = (torch.arange(n, dtype=torch.int32, device="cuda") + start).view(torch.float32)
            got = engine.pmf_sigmoid(z)
            PO.sigmoid_bits(first, n, host)
            want = torch.from_numpy(host[:n]).cuda()
            bad = int((got.view(torch.int32) != want.view(torch.int32)).sum())
            assert bad == 0, "%d mismatches among bit patterns [%#x, %#x)" % (bad, first, first + n)
            n_checked += n
    assert n_checked == (six + 1) + (msix + 1 - 0x80000000)


def test_score_batch_f64_is_the_index_order_dot():
    from cornac_b200 import engine
    rng = np.random.RandomState(5)
    for k in (1, 7, 16, 33):
        U, V = rng.normal(0, 1, (50, k)), rng.normal(0, 1, (1000, k))
        users = rng.randint(50, size=37)
        got = engine.score_batch_f64(engine.to_device(U, torch.float64), engine.to_device(V, torch.float64),
                                     user_idx=engine.to_device(users, torch.int64)).cpu().numpy()
        want = np.zeros((len(users), len(V)))
        for f in range(k):
            want = want + U[users, f][:, None] * V[:, f][None, :]
        assert np.array_equal(got, want)
        blas = np.stack([V.dot(U[u]) for u in users])
        assert np.all(np.abs(got - blas) <= 1e-14 * np.maximum(np.abs(blas), np.abs(V).dot(np.abs(U[users]).T).T))


@pytest.mark.parametrize("topk", [1, 2, 3, 4, 17, 1000, 4096])
def test_topk_rows_f64_equals_lexsort_with_exclusions_and_ties(topk):
    from cornac_b200 import engine
    rng = np.random.RandomState(topk)
    n_q, n = 9, 5000
    S = rng.normal(0, 1, (n_q, n))
    S[1] = np.round(S[1], 1)                                   # many ties
    S[2] = 0.0
    S[2, ::7] = -0.0                                           # -0.0 ties with +0.0
    S[3, :10] = [np.inf, -np.inf, 1e300, -1e300, 5e-324, -5e-324, 1.0, 1.0, 1.0 + 2 ** -52, 1.0]
    S[4] = np.arange(n) // 3                                   # ties of three
    excl = [np.sort(rng.choice(n, size=rng.randint(0, 300), replace=False)) for _ in range(n_q)]
    excl[5] = np.arange(n - 10)                                # fewer candidates than topk
    excl[6] = np.arange(n)                                     # no candidate
    ptr = np.concatenate([[0], np.cumsum([len(e) for e in excl])]).astype(np.int64)
    idx = np.concatenate(excl).astype(np.int32)
    ids, sc = engine.topk_rows_f64(engine.to_device(S, torch.float64), topk, engine.to_device(ptr, torch.int64),
                                   engine.to_device(idx, torch.int32))
    ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
    for q in range(n_q):
        cand = np.setdiff1d(np.arange(n), excl[q])
        order = cand[np.lexsort((cand, -(S[q, cand] + 0.0)))][:topk]
        m = len(order)
        assert np.array_equal(ids[q, :m], order), q
        assert np.array_equal(sc[q, :m], S[q, order])
        assert np.all(ids[q, m:] == -1)
    # no exclusions
    ids2, _ = engine.topk_rows_f64(engine.to_device(S, torch.float64), topk)
    for q in range(n_q):
        assert np.array_equal(ids2[q].cpu().numpy()[: min(topk, n)], np.lexsort((np.arange(n), -(S[q] + 0.0)))[:topk])


@needs_cornac
@pytest.mark.parametrize("name", ["pmf_linear_k5", "pmf_nonlinear_k10", "pmf_nonlinear_unit"])
def test_plugin_fit_and_scores_match_the_reference(name):
    from cornac_b200 import PMF
    g = golden(name)
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    m = PMF(k=int(g["k"]), max_iter=int(g["max_iter"]), variant=str(g["variant"]), seed=int(g["seed"]),
            learning_rate=float(g["learning_rate"]), gamma=float(g["gamma"]), lambda_reg=float(g["lambda_reg"])).fit(ds)
    assert np.array_equal(m.U, g["U"]) and np.array_equal(m.V, g["V"])
    single = np.array([m.score(int(u), int(i)) for u, i in g["single_pairs"]])
    assert np.array_equal(single, g["single_scores"])


@needs_cornac
def test_init_params_are_trained_in_place():
    from cornac_b200 import PMF
    g = golden("pmf_linear_init_u_k7")
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    U = g["U0"].copy()
    m = PMF(k=7, max_iter=int(g["max_iter"]), variant="linear", seed=int(g["seed"]), learning_rate=float(g["learning_rate"]),
            init_params={"U": U}).fit(ds)
    assert m.U is U and np.array_equal(U, g["U"]) and np.array_equal(m.V, g["V"])


@needs_cornac
def test_verbose_prints_the_reference_losses():
    from cornac_b200 import PMF
    g = golden("pmf_nonlinear_k10")
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    buf = io.StringIO()
    m = PMF(k=10, max_iter=int(g["max_iter"]), seed=int(g["seed"]), learning_rate=float(g["learning_rate"]),
            gamma=float(g["gamma"]), lambda_reg=float(g["lambda_reg"]), verbose=True)
    m._B200_LOSS_BYTES = 8 * len(g["uid"]) * 3                # several epoch chunks
    with redirect_stdout(buf):
        m.fit(ds)
    lines = [x for x in buf.getvalue().splitlines() if x.startswith("epoch")]
    assert lines == ["epoch %i, loss: %f" % (e, x) for e, x in enumerate(g["loss"])]
    assert np.array_equal(m.U, g["U"])


@needs_cornac
def test_plugin_matches_reference_edge_behaviour():
    from cornac.exception import ScoreException
    from cornac.models import PMF as RefPMF
    from cornac_b200 import PMF
    g = golden("pmf_nonlinear_k10")
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    kw = dict(k=10, max_iter=5, seed=3, learning_rate=0.05)
    ref, ours = RefPMF(**kw).fit(ds), PMF(**kw).fit(ds)
    assert np.array_equal(ref.U, ours.U) and np.array_equal(ref.V, ours.V)
    for m in (ref, ours):
        with pytest.raises(ScoreException):
            m.score(ds.num_users)
        with pytest.raises(ScoreException):
            m.score(0, ds.num_items)
    for u in (0, 5, ds.num_users - 1):
        raw = ours.score(u)                                    # the raw dot, not the sigmoid
        assert np.all(np.abs(raw - ref.score(u)) <= 1e-14 * np.abs(ref.V).dot(np.abs(ref.U[u])))
        assert ours.score(u, 3) == ref.score(u, 3)
    ours.transform(ds)                                         # a cached row never answers the single-item case
    assert ours.score(1, 4) == ref.score(1, 4) and ours.score(1, 4) != ours.score(1)[4]


@needs_cornac
def test_rank_and_rank_batch_follow_recommender_rank():
    from cornac_b200 import PMF
    g = golden("pmf_linear_k10_mid")
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    m = PMF(k=10, max_iter=5, variant="linear", seed=1, learning_rate=0.01).fit(ds)
    rng = np.random.RandomState(0)
    n = ds.num_items
    for cached in (False, True):
        if cached:
            m.transform(ds)
        for u in (0, 17, ds.num_users - 1):
            row = m.score(u)
            full = np.lexsort((np.arange(n), -row))
            ranked, sc = m.rank(u)
            assert np.array_equal(ranked, full) and np.array_equal(sc, row)
            ranked, _ = m.rank(u, k=10)
            assert np.array_equal(ranked[:10], full[:10]) and np.array_equal(np.sort(ranked), np.arange(n))
            cand = np.sort(rng.choice(n, size=50, replace=False))
            ranked, sc = m.rank(u, cand, k=5)
            want = cand[np.lexsort((cand, -row[cand]))]
            assert np.array_equal(ranked[:5], want[:5]) and np.array_equal(sc, row[cand])
            assert np.array_equal(np.sort(ranked), cand)
    # unknown user: every item scores default_score()
    ranked, sc = m.rank(ds.num_users + 3, k=5)
    assert np.all(sc == m.default_score()) and np.array_equal(ranked, np.arange(n))
    # rank_batch with the training items excluded
    users = np.arange(0, ds.num_users, 7)
    ids, top = m.rank_batch(users, 20, exclude=ds.csr_matrix)
    for q, u in enumerate(users):
        row = m.score(int(u))
        cand = np.setdiff1d(np.arange(n), ds.csr_matrix[u].indices)
        want = cand[np.lexsort((cand, -row[cand]))][:20]
        assert np.array_equal(ids[q], want) and np.array_equal(top[q], row[want])
    recs = m.recommend_batch([ds.user_ids[0], ds.user_ids[3]], k=5, remove_seen=True, train_set=ds)
    assert recs == [m.recommend(ds.user_ids[0], k=5, remove_seen=True, train_set=ds)[:5],
                    m.recommend(ds.user_ids[3], k=5, remove_seen=True, train_set=ds)[:5]]


@needs_cornac
def test_save_load_round_trip():
    from cornac_b200 import PMF
    g = golden("pmf_linear_k5")
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    m = PMF(k=5, max_iter=10, variant="linear", seed=2).fit(ds)
    with tempfile.TemporaryDirectory() as d:
        path = m.save(d)
        m2 = PMF.load(path)
    assert np.array_equal(m2.U, m.U) and np.array_equal(m2.V, m.V)
    assert np.array_equal(m2.score(3), m.score(3))
    assert np.array_equal(m2.rank(3, k=10)[0][:10], m.rank(3, k=10)[0][:10])
    c = m.clone()
    assert c.k == 5 and c.variant == "linear" and c.seed == 2


@needs_cornac
def test_experiment_metrics_equal_the_reference():
    import cornac
    import cornac_b200
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, MAE, NDCG, RMSE, Recall
    g = golden("pmf_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, seed=123, verbose=False)
    models = [cornac_b200.PMF(k=10, max_iter=60, learning_rate=0.01, lambda_reg=0.01, variant="linear", seed=123,
                              name="PMF-linear"),
              cornac_b200.PMF(k=10, max_iter=60, learning_rate=0.01, lambda_reg=0.01, seed=123, name="PMF-non_linear")]
    exp = cornac.Experiment(eval_method=rs, models=models, metrics=[RMSE(), MAE(), Recall(k=10), NDCG(k=10), AUC()],
                            verbose=False)
    exp.run()
    res = {r.model_name: r.metric_avg_results for r in exp.result}
    names = [str(x) for x in g["metric_names"]]
    for model, key in (("PMF-linear", "linear"), ("PMF-non_linear", "non_linear")):
        got = np.array([res[model][n] for n in names])
        assert np.all(np.abs(got - g[key]) <= 1e-12), (model, dict(zip(names, got)), dict(zip(names, g[key])))


@needs_cornac
def test_quick_start_comparison_runs_on_the_gpu():
    """The reference README's quick start (MF, PMF, BPR in one Experiment) with the drop-ins on synthetic ratings."""
    import cornac
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import MAE, RMSE, Precision, Recall, NDCG, AUC, MAP
    from cornac_b200 import MF, PMF, BPR
    indptr, indices = synth_csr(943, 1682, 100000, seed=100)
    rng = np.random.RandomState(100)
    users = np.repeat(np.arange(943), np.diff(indptr))
    data = [(str(u), str(i), float(r)) for u, i, r in zip(users, indices, rng.randint(1, 6, size=len(indices)))]
    rs = RatioSplit(data=data, test_size=0.2, rating_threshold=4.0, seed=123, verbose=False)
    models = [MF(k=10, max_iter=25, learning_rate=0.01, lambda_reg=0.02, use_bias=True, seed=123),
              PMF(k=10, max_iter=100, learning_rate=0.001, lambda_reg=0.001, seed=123),
              BPR(k=10, max_iter=200, learning_rate=0.001, lambda_reg=0.01, seed=123)]
    exp = cornac.Experiment(eval_method=rs, models=models,
                            metrics=[MAE(), RMSE(), Precision(k=10), Recall(k=10), NDCG(k=10), AUC(), MAP()],
                            user_based=True, verbose=False)
    exp.run()
    assert [r.model_name for r in exp.result] == ["MF", "PMF", "BPR"]
    for r in exp.result:
        assert all(np.isfinite(v) for v in r.metric_avg_results.values())
