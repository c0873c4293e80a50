"""ComparERSub on the GPU: the seeded fit bit-identical to the serial oracle (every fixture, split calls, a pair with
earlier == later, no pair samples equal to mter_fit), the unseeded fit, the aspect-mixed rank rows against an f64
restatement, every rank path against each other, score(u) as MTER's rating row, and an unchanged cornac.Experiment
against the reference's metrics."""
import contextlib
import io

import numpy as np
import pytest
import torch

from conftest import golden, needs_cornac
from oracle import comparer_oracle as CO
from test_comparer_cpu import CASES, draws, fixture_data, helpers, hyper, model_kwargs

pytestmark = pytest.mark.gpu
PARAMS = CO.PARAMS


def device_fit(data, init, draw_list, n_iter, n_el, n_bpr, n_pair, hy, split=None):
    """The device fit from `init` over the given draws; returns params, sgrad and counts on the host."""
    from cornac_b200 import engine
    dd = engine.ComparerDeviceData(data)
    params = [torch.from_numpy(init[p].copy()).cuda() for p in PARAMS]
    sgrad = [torch.zeros_like(x) for x in params]
    uia, uao, iao, pair, pos, neg = (np.asarray(d, np.int64).reshape(n_iter, -1) for d in draw_list)
    per = np.concatenate([uia, uao, iao, pos, neg, pair], axis=1).astype(np.int32)
    dims = tuple(int(x) for x in init["G1"].shape) + (int(init["G2"].shape[2]),)
    work = torch.zeros(engine.comparer_sub_workspace_bytes(dd, dims, n_el, n_bpr, n_pair), dtype=torch.uint8,
                       device="cuda")
    counts = torch.zeros(3, dtype=torch.int64, device="cuda")
    done = 0
    for n in ([n_iter] if split is None else [split, n_iter - split]):
        dr = torch.from_numpy(np.ascontiguousarray(per[done:done + n])).cuda()
        engine.comparer_sub_fit(dd, params, sgrad, dr, n, n_el, n_bpr, n_pair, counts=counts, workspace=work, **hy)
        done += n
    torch.cuda.synchronize()
    assert not work[: 4 * sum(x.numel() for x in params)].any()          # the del buffer is left zero
    return ({p: x.cpu().numpy() for p, x in zip(PARAMS, params)}, {p: x.cpu().numpy() for p, x in zip(PARAMS, sgrad)},
            counts.cpu().numpy())


def oracle_fit(g, data, n_iter, draw_list=None):
    want = {p: g[p + "0"].copy() for p in PARAMS}
    ws = {p: np.zeros_like(x) for p, x in want.items()}
    out = CO.fit(data, want, ws, draws(g, n_iter) if draw_list is None else draw_list, n_iter, **hyper(g))
    return want, ws, out


def sizes(g):
    return int(g["n_element_samples"]), int(g["n_bpr_samples"]), int(g["n_pair_samples"])


@pytest.mark.parametrize("case", CASES)
def test_fit_equals_oracle(case):
    g = golden(case)
    data = fixture_data(g)
    n_iter = int(max(g["max_iters"]))
    want, ws, (c, s, _, _, ac) = oracle_fit(g, data, n_iter)
    init = {p: g[p + "0"] for p in PARAMS}
    for split in (None, 1):
        got, gs, counts = device_fit(data, init, draws(g, n_iter), n_iter, *sizes(g), hyper(g), split=split)
        for p in PARAMS:
            assert np.array_equal(got[p], want[p]), (case, split, p)
            assert np.array_equal(gs[p], ws[p]), (case, split, "sgrad_" + p)
        assert counts.tolist() == [int(c.sum()), int(s.sum()), int(ac.sum())]


def test_earlier_equals_later_pairs_equal_oracle():
    """Pairs whose earlier and later items are the same (the reference's build never makes one, but the fit takes any
    list): the I row takes -v then +v for every term."""
    g = golden("comparer_sub_window")
    data = fixture_data(g)
    rng = np.random.RandomState(3)
    n = len(data.p_user_indices)
    same = rng.rand(n) < 0.3
    data.later_indices = np.where(same, data.earlier_indices, data.later_indices).astype(np.int32)
    n_iter = 4
    want, ws, _ = oracle_fit(g, data, n_iter)
    got, gs, _ = device_fit(data, {p: g[p + "0"] for p in PARAMS}, draws(g, n_iter), n_iter, *sizes(g), hyper(g))
    for p in PARAMS:
        assert np.array_equal(got[p], want[p]) and np.array_equal(gs[p], ws[p]), p


def test_no_pair_samples_equals_mter_fit():
    from cornac_b200 import engine
    g = golden("comparer_sub_nopair")
    data = fixture_data(g)
    n_el, n_bpr, _ = sizes(g)
    n_iter = 3
    got, gs, _ = device_fit(data, {p: g[p + "0"] for p in PARAMS}, draws(g, n_iter), n_iter, n_el, n_bpr, 0, hyper(g))
    dd = engine.MterDeviceData(data)
    params = [torch.from_numpy(g[p + "0"].copy()).cuda() for p in PARAMS]
    sgrad = [torch.zeros_like(x) for x in params]
    d = draws(g, n_iter)
    per = np.concatenate([np.asarray(x, np.int64).reshape(n_iter, -1) for k, x in enumerate(d) if k != 3], axis=1)
    hy = hyper(g)
    hy.pop("lambda_d")
    engine.mter_fit(dd, params, sgrad, torch.from_numpy(per.astype(np.int32)).cuda(), n_iter, n_el, n_bpr, **hy)
    for p, x, sx in zip(PARAMS, params, sgrad):
        assert np.array_equal(got[p], x.cpu().numpy()) and np.array_equal(gs[p], sx.cpu().numpy()), p


@needs_cornac
def test_seeded_plugin_equals_oracle():
    from cornac_b200 import ComparERSub
    g = golden("comparer_sub_window")
    mk = helpers()
    m = ComparERSub(max_iter=10, seed=int(g["seed"]), init_params={p: g[p + "0"].copy() for p in PARAMS},
                    **model_kwargs(g)).fit(mk.train_set(g))
    want, _, _ = oracle_fit(g, fixture_data(g), 10)
    for p in PARAMS:
        assert np.array_equal(getattr(m, p), want[p]), p


@needs_cornac
def test_unseeded_fit_learns_pairs_and_bpr():
    from cornac_b200 import engine
    from cornac_b200.recom_comparer import build_data
    g = golden("comparer_sub_default")
    ts = helpers().train_set(g)
    data = build_data(ts, int(g["num_users"]), int(g["num_items"]), 5.0)
    dd = engine.ComparerDeviceData(data)
    params = [torch.from_numpy(g[p + "0"].copy()).cuda() for p in PARAMS]
    sgrad = [torch.zeros_like(x) for x in params]
    work = torch.zeros(engine.comparer_sub_workspace_bytes(dd, (8, 8, 8, 8), 50, 1000, 1000), dtype=torch.uint8,
                       device="cuda")
    acc = []
    for it in range(300):
        counts = torch.zeros(3, dtype=torch.int64, device="cuda")
        engine.comparer_sub_fit(dd, params, sgrad, None, 1, 50, 1000, 1000, counts=counts, workspace=work,
                                unordered=True, philox_seed=777, iter0=it, lambda_d=1.0)
        c, s, a = counts.tolist()
        acc.append((c / max(1000 - s, 1), a / 1000))
    acc = np.array(acc)
    assert acc[-30:, 0].mean() > acc[:30, 0].mean() and acc[-30:, 1].mean() > acc[:30, 1].mean(), acc[[0, -1]]
    for p, x in zip(PARAMS, params):
        assert bool(torch.isfinite(x).all()) and bool((x >= 0).all()), p


def _rank_f64(m, u):
    """The reference's rank formula in f64 (recom_comparer_sub.pyx:765-776)."""
    G1, U, I, A = (np.asarray(getattr(m, p), np.float64) for p in ("G1", "U", "I", "A"))
    ts3 = np.einsum("Mb,Nb->MN", I[: m.num_items], np.einsum("bc,Nc->Nb", np.einsum("abc,a->bc", G1, U[u]), A))
    n = min(m.n_top_aspects, m.num_aspects)
    top = -np.sort(-ts3[:, :-1], axis=1)[:, :n]
    return m.alpha * top.mean(axis=1) + (1 - m.alpha) * ts3[:, -1]


def _fitted(case, **over):
    from cornac_b200 import ComparERSub
    g = golden(case)
    kw = model_kwargs(g)
    kw.update(over)
    return ComparERSub(max_iter=5, seed=int(g["seed"]), **kw).fit(helpers().train_set(g)), g


@needs_cornac
@pytest.mark.parametrize("case,n_top", [("comparer_sub_window", 5), ("comparer_sub_default", 100),
                                        ("comparer_sub_default", 7), ("comparer_sub_nonpos", 3)])
def test_rank_rows_equal_f64_restatement(case, n_top):
    m, _ = _fitted(case, n_top_aspects=n_top)
    rows = m._scores_dev(np.arange(m.num_users)).cpu().numpy()
    for u in range(m.num_users):
        want = _rank_f64(m, u)
        assert np.allclose(rows[u], want, rtol=2 ** -23, atol=1e-30 + 2 ** -23 * np.abs(want).max()), (case, u)
    half = m._scores_dev(np.arange(3), n_items=m.num_items // 2).cpu().numpy()
    assert np.array_equal(half, rows[:3, : m.num_items // 2])


@needs_cornac
def test_rank_paths_agree_and_score_stays_mters_row():
    from cornac_b200 import MTER
    m, g = _fitted("comparer_sub_window")
    users = np.arange(m.num_users)
    ids, sc = m.rank_batch(users, 10)
    rows = m._scores_dev(users).cpu().numpy()
    for u in users:
        r_ids, r_sc = m.rank(int(u))
        assert np.array_equal(ids[u], r_ids[:10]) and np.array_equal(r_sc, rows[u])
        assert np.array_equal(r_ids, np.lexsort((np.arange(m.num_items), -rows[u].astype(np.float64))))
    dids, _ = m.rank_batch_device(users, 10)
    assert np.array_equal(dids.cpu().numpy(), ids)
    m.transform(SimpleTest(users))
    for u in users[::3]:
        assert np.array_equal(m.rank(int(u))[0], np.lexsort((np.arange(m.num_items), -rows[u].astype(np.float64))))
    rec = m.recommend_batch([m.user_ids[u] for u in users[:5]], k=5)
    assert [[m.iid_map[i] for i in r] for r in rec] == ids[:5, :5].tolist()
    # score(u) is MTER's rating row (the reference inherits MTER.score)
    mt = MTER(**{k: getattr(m, k) for k in ("n_user_factors", "n_item_factors", "n_aspect_factors",
                                             "n_opinion_factors")},
              init_params={p: getattr(m, p) for p in PARAMS}, trainable=False, seed=1).fit(helpers().train_set(g))
    for u in (0, 5):
        assert np.array_equal(m.score(u), mt.score(u))
        assert m.score(u, 2) == mt.score(u, 2)


class SimpleTest:
    def __init__(self, users):
        self.uir_tuple = (np.asarray(users), np.zeros(len(users), np.int64), np.ones(len(users)))


@needs_cornac
def test_alpha_zero_ranks_as_mter():
    from cornac_b200 import MTER
    m, g = _fitted("comparer_sub_exact")
    assert m.alpha == 0
    mt = MTER(**{k: getattr(m, k) for k in ("n_user_factors", "n_item_factors", "n_aspect_factors",
                                             "n_opinion_factors")},
              init_params={p: getattr(m, p) for p in PARAMS}, trainable=False, seed=1).fit(helpers().train_set(g))
    users = np.arange(m.num_users)
    assert np.array_equal(m.rank_batch(users, 10)[0], mt.rank_batch(users, 10)[0])


def _split(g):
    from cornac.data import SentimentModality
    from cornac.eval_methods import RatioSplit
    import make_golden_efm
    data = [(str(a), str(b), float(c), int(d)) for a, b, c, d in zip(g["uir_u"], g["uir_i"], g["uir_r"], g["uir_t"])]
    return RatioSplit(data=data, fmt="UIRT", test_size=0.1, exclude_unknowns=True, verbose=False, seed=123,
                      sentiment=SentimentModality(data=make_golden_efm.unpack_reviews(g)))


@needs_cornac
def test_experiment_metrics_match_the_reference(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    import cornac
    from cornac.metrics import NDCG, RMSE
    from cornac_b200 import ComparERSub
    helpers()
    g = golden("comparer_sub_experiment")
    rs = _split(g)
    metrics = [RMSE(), NDCG(k=10), NDCG(k=20), NDCG(k=50)]
    assert [m.name for m in metrics] == list(g["metric_names"])
    model = ComparERSub(n_top_aspects=10, max_iter=int(g["max_iter"]), seed=123)
    with contextlib.redirect_stdout(io.StringIO()):
        exp = cornac.Experiment(eval_method=rs, models=[model], metrics=metrics, user_based=True, verbose=False)
        exp.run()
    got = np.array([exp.result[0].metric_avg_results[m.name] for m in metrics])
    # The fit equals the oracle bit for bit (test_fit_equals_oracle); over these 200 iterations at lr = 0.5 the
    # parameters end 4.7e-5 from the reference's (largest |delta| / max|value| per array, U, measured on an H100), past
    # the 4e-5 MTER's Experiment test pins for its 9.3e-6: MTER's unexplained per-iteration drift (test_comparer_cpu)
    # compounds over more updates per iteration here.  Pinned with a 4x margin; RMSE within 1e-4 and NDCG within 2e-3,
    # MTER's bounds (items whose scores are closer than the parameters' difference can swap places).
    for p in PARAMS:
        ref = g["fit_" + p]
        err = np.max(np.abs(getattr(model, p) - ref)) / np.max(np.abs(ref))
        assert err <= 2e-4, (p, err)
    assert abs(got[0] - g["metrics"][0]) <= 1e-4, (got, g["metrics"])
    assert np.all(np.abs(got[1:] - g["metrics"][1:]) <= 2e-3), (got, g["metrics"])


@needs_cornac
def test_batched_ranking_eval_equals_per_user():
    from cornac.eval_methods.base_method import ranking_eval as ref_ranking_eval
    from cornac.metrics import AUC, MAP, NDCG, Recall
    from cornac_b200 import ComparERSub
    from cornac_b200.evaluation import ranking_eval
    helpers()
    g = golden("comparer_sub_experiment")
    rs = _split(g)
    model = ComparERSub(n_top_aspects=10, max_iter=50, seed=123).fit(rs.train_set)
    assert model._b200_scores_nan_free()
    metrics = [NDCG(k=20), AUC(), Recall(k=10), MAP()]
    mine, _ = ranking_eval(model, metrics, rs.train_set, rs.test_set, rating_threshold=1.0, exclude_unknowns=True)
    ref, _ = ref_ranking_eval(model, metrics, rs.train_set, rs.test_set, rating_threshold=1.0, exclude_unknowns=True)
    assert np.allclose(mine, ref, rtol=1e-12, atol=1e-12)
