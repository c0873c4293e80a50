"""LRPPM on the GPU: the seeded fit against the serial oracle and the compiled reference (tests/golden/lrppm_*.npz), the
convergence stop, split calls, the unseeded fit, the rank rows and every rank path, and an unchanged Experiment."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_lrppm_cpu import CASES, GOLDEN, PARAMS, case_data, draws, load  # noqa: E402

from oracle import lrppm_oracle as LO  # noqa: E402

pytestmark = pytest.mark.gpu


def device_fit(g, d, n_iter, calls=(None,)):
    """The device fit from the fixture's initial parameters over its draws, in calls of the given sizes."""
    from cornac_b200 import engine
    dd = engine.LrppmDeviceData(d)
    n_s, n_r = int(g["n_samples"]), int(g["n_ranking_samples"])
    pos, pu, nu = draws(g, n_iter)
    per = np.concatenate([pos.reshape(n_iter, n_s), pu.reshape(n_iter, n_r), nu.reshape(n_iter, n_r)], axis=1)
    params = [torch.from_numpy(g[p + "0"].copy()).cuda() for p in PARAMS]
    work = torch.zeros(engine.lrppm_workspace_bytes(dd, params[0].shape[1], n_s, n_r), dtype=torch.uint8, device="cuda")
    counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    sizes = [n_iter] if calls == (None,) else list(calls)
    lo = 0
    for n in sizes:
        engine.lrppm_fit(dd, params, torch.from_numpy(per[lo:lo + n].astype(np.int32)).cuda(), n, n_s, n_r,
                         lr=float(g["lr"]), reg=float(g["reg"]), ld=float(g["ld"]), counts=counts, workspace=work,
                         iter0=lo)
        lo += n
        if counts[3].item():
            break
    return [p.cpu().numpy() for p in params], counts.cpu().numpy()


@pytest.mark.parametrize("name", CASES)
def test_device_fit_equals_oracle_and_reference(name):
    g = load(name)
    d = case_data(g)
    for mi in g["max_iters"]:
        mi = int(mi)
        want = {p: g[p + "0"].copy() for p in PARAMS}
        ran, conv, correct, skipped, *_ = LO.fit(d, want, draws(g, mi), mi, int(g["n_samples"]),
                                                 int(g["n_ranking_samples"]), lr=float(g["lr"]), reg=float(g["reg"]),
                                                 ld=float(g["ld"]))
        got, counts = device_fit(g, d, mi)
        for p, x in zip(PARAMS, got):
            assert np.array_equal(x.view(np.uint32), want[p].view(np.uint32)), (name, mi, p)
            assert np.array_equal(x.view(np.uint32), g["%s_%d" % (p, mi)].view(np.uint32)), (name, mi, p)
        assert counts.tolist() == [int(correct.sum()), int(skipped.sum()), ran, int(conv)], (name, mi)


@pytest.mark.parametrize("name", ["lrppm_default", "lrppm_k3", "lrppm_nan", "lrppm_converge"])
def test_split_calls_equal_one_call(name):
    g = load(name)
    d = case_data(g)
    mi = int(g["max_iters"][-1])
    one, c1 = device_fit(g, d, mi)
    two, c2 = device_fit(g, d, mi, calls=(1, mi - 1))
    for a, b in zip(one, two):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert c1[2:].tolist() == c2[2:].tolist()


def fixture_train_set(g):
    from make_golden_efm import train_set
    sys.path.insert(0, GOLDEN)
    ts = train_set(g)
    ts.uir_tuple = (g["ts_u"], g["ts_i"], g["ts_r"])
    return ts


@pytest.mark.parametrize("name", ["lrppm_default", "lrppm_converge"])
def test_plugin_seeded_fit_equals_reference(name, capsys):
    from cornac_b200 import LRPPM
    g = load(name)
    ts = fixture_train_set(g)
    hyper = {k: g[k].item() for k in ("rating_scale", "n_factors", "ld", "reg", "alpha", "num_top_aspects",
                                      "n_ranking_samples", "n_samples", "lr")}
    mi = int(g["max_iters"][-1])
    m = LRPPM(max_iter=mi, seed=int(g["seed"]), init_params={p: g[p + "0"].copy() for p in PARAMS}, **hyper).fit(ts)
    for p in PARAMS:
        assert np.array_equal(np.asarray(getattr(m, p)).view(np.uint32), g["%s_%d" % (p, mi)].view(np.uint32)), p
    assert m.n_iter_run == int(g["calls_%d" % mi])
    assert ("Stop training because model converged!" in capsys.readouterr().out) == bool(g["converged_%d" % mi])


def test_unseeded_fit_lowers_the_loss():
    from cornac_b200 import LRPPM
    g = load("lrppm_default")
    ts = fixture_train_set(g)

    def mse(m):
        u, i, r = ts.uir_tuple
        return float(np.mean((np.sum(m.U[u] * m.I[i], axis=1) - r) ** 2))
    m0 = LRPPM(max_iter=0, init_params={p: g[p + "0"].copy() for p in PARAMS}).fit(ts)
    before = mse(m0)
    # lr = 0.1 drives some aspect rows of this fixture to inf (the reference's seeded fit does too): a smaller step
    m = LRPPM(max_iter=300, lr=0.005, init_params={p: g[p + "0"].copy() for p in PARAMS}).fit(ts)
    for p in PARAMS:
        x = np.asarray(getattr(m, p))
        assert np.all(np.isfinite(x)) and np.all(x >= 0)
    assert 1 <= m.n_iter_run <= 300
    assert mse(m) < before


def rank_restatement(U, I, UA, IA, Q, u, n_top, alpha, scale):
    """The device's rank row of user u in f64: each dot an f64 sum rounded to f32."""
    dot = lambda a, b: (a.astype(np.float64) * b.astype(np.float64)).sum(axis=-1).astype(np.float32)  # noqa: E731
    uau = dot(UA, U[u][None, :])
    iia = dot(I[:, None, :], IA[None, :, :])
    du = dot(I, U[u][None, :])
    s = ((uau[None, :] + iia).astype(np.float32) + du[:, None]).astype(np.float32)
    return LO.rank_rows(s, Q.toarray(), n_top, alpha, scale, du)


@pytest.mark.parametrize("name,n_top", [("lrppm_default", 99999), ("lrppm_default", 10), ("lrppm_k5", 4)])
def test_rank_rows_equal_restatement(name, n_top):
    from cornac_b200 import engine
    g = load(name)
    mi = int(g["max_iters"][-1])
    U, I, UA, IA = (g["%s_%d" % (p, mi)] for p in PARAMS)
    Q = sp.csr_matrix((g["Q_data"], g["Q_indices"], g["Q_indptr"]), shape=(int(g["num_items"]), int(g["num_aspects"])))
    n_top = min(n_top, UA.shape[0])
    alpha, scale = float(g["alpha"]), float(g["rating_scale"])
    dv = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()                  # noqa: E731
    users = np.arange(U.shape[0])
    rows = engine.lrppm_rank_rows(dv(U), dv(I), dv(UA), dv(IA), engine.LrppmQuality(Q), dv(users.astype(np.int64)),
                                  n_top, alpha, scale).cpu().numpy()
    for u in users:
        want = rank_restatement(U, I, UA, IA, Q, u, n_top, alpha, scale)
        assert np.allclose(rows[u], want, rtol=1e-13, atol=1e-13), (name, u)


def test_rank_rows_ties_take_the_smaller_aspect():
    from cornac_b200 import engine
    k, n_items, n_aspects = 4, 3, 40
    U = np.ones((1, k), np.float32)
    I = np.zeros((n_items, k), np.float32)
    UA = np.zeros((n_aspects, k), np.float32)
    UA[::3] = 0.25                                    # ties among aspects 0, 3, 6, ...
    IA = np.zeros((n_aspects, k), np.float32)
    Q = sp.csr_matrix(np.random.RandomState(0).uniform(0.1, 1, (n_items, n_aspects)))
    dv = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()                  # noqa: E731
    for n_top in (5, 14, 20):
        rows = engine.lrppm_rank_rows(dv(U), dv(I), dv(UA), dv(IA), engine.LrppmQuality(Q),
                                      dv(np.zeros(1, np.int64)), n_top, 1.0, 5.0).cpu().numpy()[0]
        want = rank_restatement(U, I, UA, IA, Q, 0, n_top, 1.0, 5.0)
        assert np.allclose(rows, want, rtol=1e-13, atol=0), n_top


@pytest.mark.parametrize("alpha,n_top", [(1, 99999), (0.6, 5), (0, 99999)])
def test_rank_paths_agree(alpha, n_top):
    from cornac_b200 import LRPPM
    g = load("lrppm_default")
    ts = fixture_train_set(g)
    mi = int(g["max_iters"][-1])
    m = LRPPM(max_iter=0, alpha=alpha, num_top_aspects=n_top,
              init_params={p: g["%s_%d" % (p, mi)].copy() for p in PARAMS}).fit(ts)
    users = np.arange(ts.num_users)
    if alpha == 0:
        row = m._scores_dev([3])[0].cpu().numpy()
        assert np.allclose(row, m.score(3), rtol=1e-6, atol=1e-6)
    ids_b, sc_b = m.rank_batch(users, 10)
    for u in users[:10]:
        ranked, scores = m.rank(int(u))
        assert np.array_equal(ranked[:10], ids_b[u])
        top, _ = m.rank(int(u), k=10)
        assert np.array_equal(top[:10], ids_b[u])
    rec = m.recommend_batch([ts.user_ids[u] for u in users[:5]], k=10)
    assert [[ts.iid_map[i] for i in r] for r in rec] == ids_b[:5].tolist()
    m.transform(ts)
    for u in users[:10]:
        ranked, scores = m.rank(int(u))
        assert np.array_equal(ranked[:10], ids_b[u])


def test_experiment_metrics():
    import cornac
    from cornac.data import SentimentModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, NDCG, RMSE
    from cornac_b200 import LRPPM
    from make_golden_efm import unpack_reviews
    g = load("lrppm_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123,
                    sentiment=SentimentModality(data=unpack_reviews(g)))
    model = LRPPM(max_iter=int(g["max_iter"]), num_top_aspects=99999, seed=123)
    exp = cornac.Experiment(eval_method=rs, models=[model], metrics=[RMSE(), AUC(), NDCG(k=50)], user_based=True,
                            verbose=False)
    exp.run()
    res = exp.result[0].metric_avg_results
    for p in PARAMS:
        assert np.array_equal(np.asarray(getattr(model, p)), g["fit_" + p]), p
    got = [res[n] for n in g["metric_names"]]
    # the parameters are the reference's; RMSE is the host dot; AUC / NDCG from rows that differ from numpy's only in
    # how each dot is rounded to f32
    assert abs(got[0] - g["metrics"][0]) <= 1e-9
    assert abs(got[1] - g["metrics"][1]) <= 2e-3 and abs(got[2] - g["metrics"][2]) <= 2e-3, (got, g["metrics"])
