"""HPF / PF on the GPU: b200_hpf_update bit-identical to the serial oracle given the same expectations, b200_hpf_expect
against scipy, the whole fit against the compiled reference's fixtures (whole and split), and the plug-in through
ranking, an unchanged Experiment, save / load and trainable=False."""
import tempfile

import numpy as np
import pytest
import scipy.special
import torch

from conftest import golden, needs_cornac, synth_csr
from oracle import hpf_oracle as HO

pytestmark = pytest.mark.gpu

FIT_CASES = ["hpf_k5", "pf_k5", "hpf_k1", "pf_k1", "hpf_k10", "pf_k10", "hpf_k37", "pf_k37", "hpf_warm_k6", "pf_warm_k6",
             "hpf_nonpos_k4", "pf_nonpos_k4"]
KEYS = ("Gs", "Gr", "Ls", "Lr")


def dev(a):
    from cornac_b200 import engine
    return engine.to_device(np.ascontiguousarray(a, dtype=np.float64), torch.float64)


def rel_max(got, want):
    return float(np.max(np.abs(got - want)) / np.max(np.abs(want)))


def _data(rid, cid, val, n, d):
    from cornac_b200 import engine
    return engine.HpfData(rid, cid, np.asarray(val, np.float64), n, d)


def _golden_data(g):
    n, d = int(g["num_users"]), int(g["num_items"])
    X = HO.csc(g["rid"], g["cid"], g["val"], n, d)
    return _data(g["rid"], g["cid"], g["val"], n, d), X, n, d


def _start(g, hierarchical, X, n, d, key="0"):
    """A golden state plus the K_r, T_r hpf_cpp sets before its loop (ones for PF)."""
    st = [g[x + key].copy() for x in KEYS] + [np.ones(n), np.ones(d)]
    HO.fit(hierarchical, X, *st, 0)
    return st


def _check_update(data, X, hierarchical, st):
    from cornac_b200 import engine
    Lt, Lb = HO.expect(st[0], st[1]), HO.expect(st[2], st[3])
    d_st = [dev(x) for x in st]
    engine.hpf_update(data, hierarchical, dev(Lt), dev(Lb), *d_st)
    want = [x.copy() for x in st]
    HO.update(hierarchical, X, Lt, Lb, *want)
    for a, b, key in zip(d_st, want, KEYS + ("Kr", "Tr")):
        assert np.array_equal(a.cpu().numpy(), b), key


@pytest.mark.parametrize("name", FIT_CASES)
def test_update_is_bit_identical_to_the_oracle(name):
    g = golden(name)
    h = bool(g["hierarchical"])
    data, X, n, d = _golden_data(g)
    _check_update(data, X, h, _start(g, h, X, n, d))
    m = int(g["iters"][-1])
    _check_update(data, X, h, _start(g, h, X, n, d, "_%d" % m))


@pytest.mark.parametrize("hierarchical", [True, False])
def test_update_at_the_ml1m_shape_is_bit_identical_to_the_oracle(hierarchical):
    indptr, indices = synth_csr(6040, 3706, 1000000, seed=5)
    rid = np.repeat(np.arange(6040), np.diff(indptr))
    rng = np.random.RandomState(5)
    val = rng.randint(1, 6, size=len(indices)).astype(np.float64)
    data = _data(rid, indices, val, 6040, 3706)
    X = HO.csc(rid, indices, val, 6040, 3706)
    k = 10
    st = [rng.gamma(100.0, 0.003, (6040, k)), rng.gamma(100.0, 0.003, (6040, k)), rng.gamma(100.0, 0.003, (3706, k)),
          rng.gamma(100.0, 0.003, (3706, k)), np.ones(6040), np.ones(3706)]
    HO.fit(hierarchical, X, *st, 0)
    _check_update(data, X, hierarchical, st)


def _expect_tolerance(s, r, got, want):
    """exp turns the rounding of its argument e = digamma(s) - log(r) into relative error, so the bound scales with |e|."""
    with np.errstate(all="ignore"):
        e = np.abs(scipy.special.digamma(s) - np.log(r))
    ok = (s > 0) & (r > 0) & (want > np.finfo(float).tiny)
    assert np.all(np.abs(got - want)[ok] <= 1e-14 * np.maximum(1.0, e[ok]) * want[ok])


@pytest.mark.parametrize("name", FIT_CASES)
def test_expect_matches_scipy(name):
    from cornac_b200 import engine
    g = golden(name)
    for key in ["0"] + ["_%d" % m for m in g["iters"]]:
        for s, r in ((g["Gs" + key], g["Gr" + key]), (g["Ls" + key], g["Lr" + key])):
            got = engine.hpf_expect(dev(s), dev(r)).cpu().numpy()
            with np.errstate(all="ignore"):
                want = np.exp(scipy.special.digamma(s) - np.log(r))
            _expect_tolerance(s, r, got, want)
            # the stored-entry rules: a dropped term is left out, both dropped is exactly 0
            both = (s <= 0) & (r <= 0)
            assert np.all(got[both] == 0.0)
            only_r = (s <= 0) & (r > 0)
            e = np.abs(np.log(r[only_r]))
            assert np.all(np.abs(got[only_r] - 1.0 / r[only_r]) <= 1e-14 * np.maximum(1.0, e) * got[only_r])
            only_s = (s > 0) & (r <= 0)
            e = scipy.special.digamma(s[only_s])
            assert np.all(np.abs(got[only_s] - np.exp(e)) <= 1e-14 * np.maximum(1.0, np.abs(e)) * np.exp(e))


def test_expect_rules_on_special_values():
    from cornac_b200 import engine
    s = np.array([0.7, 0.0, -1.0, 0.7, 0.0, -2.0, np.nan, 2.5, 1e-300, 1e300])
    r = np.array([1.3, 1.3, 0.4, 0.0, -1.0, 0.0, 1.3, np.nan, 1.0, 1.0])
    got = engine.hpf_expect(dev(s), dev(r)).cpu().numpy()
    want = HO.expect(s, r)
    assert got[4] == 0.0 and got[5] == 0.0 and got[8] == 0.0
    assert np.all(np.abs(got - want) <= 1e-14 * np.abs(want))


@pytest.mark.parametrize("split", [None, 1])
@pytest.mark.parametrize("name", FIT_CASES)
def test_fit_matches_the_reference(name, split):
    from cornac_b200 import engine
    g = golden(name)
    h = bool(g["hierarchical"])
    data, X, n, d = _golden_data(g)
    for m in g["iters"]:
        m = int(m)
        st = [dev(g[x + "0"]) for x in KEYS] + [dev(np.ones(n)), dev(np.ones(d))]
        if split is None or m <= split:
            engine.hpf_fit(data, h, *st, m)
        else:                                                     # two calls of a and b iterations == one of a + b
            engine.hpf_fit(data, h, *st, split)
            engine.hpf_fit(data, h, *st, m - split)
        got = [t.cpu().numpy() for t in st[:4]]
        got += [got[0] / got[1], got[2] / got[3]]
        for a, key in zip(got, KEYS + ("Theta", "Beta")):
            assert rel_max(a, g["%s_%d" % (key, m)]) <= 1e-10, (m, key)


def test_split_fit_is_bit_identical_to_one_fit():
    from cornac_b200 import engine
    g = golden("hpf_k10")
    data, X, n, d = _golden_data(g)
    one = [dev(g[x + "0"]) for x in KEYS] + [dev(np.ones(n)), dev(np.ones(d))]
    two = [t.clone() for t in one]
    engine.hpf_fit(data, True, *one, 9)
    for m in (2, 0, 7):
        engine.hpf_fit(data, True, *two, m)
    for a, b in zip(one, two):
        assert torch.equal(a, b)


def test_bad_arguments():
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    g = golden("hpf_k1")
    data, X, n, d = _golden_data(g)
    st = [dev(g[x + "0"]) for x in KEYS] + [dev(np.ones(n)), dev(np.ones(d))]
    with pytest.raises(B200Error, match="shape"):
        engine.hpf_fit(data, True, st[2], st[3], st[0], st[1], st[4], st[5], 1)
    with pytest.raises(B200Error, match="Kr"):
        engine.hpf_fit(data, True, *st[:4], st[5], st[5], 1)
    with pytest.raises(B200Error, match="outside"):
        _data([0, 3], [0, 1], [1.0, 1.0], 2, 2)
    with pytest.raises(B200Error, match="twice"):
        _data([0, 0], [1, 1], [1.0, 1.0], 2, 2)


def _dataset(g):
    from cornac.data import Dataset
    return Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])], seed=None)


@needs_cornac
@pytest.mark.parametrize("name", ["hpf_k5", "pf_k5"])
def test_plugin_fit_matches_the_reference(name, capsys):
    from cornac_b200 import HPF
    g = golden(name)
    m = HPF(k=int(g["k"]), max_iter=100, hierarchical=bool(g["hierarchical"]), seed=int(g["seed"])).fit(_dataset(g))
    assert capsys.readouterr().out == "Learning...\nLearning completed!\n"
    for key in KEYS + ("Theta", "Beta"):
        assert rel_max(getattr(m, key), g["%s_100" % key]) <= 1e-10, key
    # a second fit() warm-starts from the stored state
    warm = HPF(k=int(g["k"]), max_iter=1, hierarchical=bool(g["hierarchical"]),
               init_params={"G_s": m.Gs, "G_r": m.Gr, "L_s": m.Ls, "L_r": m.Lr}).fit(_dataset(g))
    m.max_iter = 1
    m.fit(_dataset(g))
    assert not np.array_equal(m.Gs, g["Gs_100"])
    for key in KEYS + ("Theta", "Beta"):
        assert np.array_equal(getattr(m, key), getattr(warm, key)), key


@needs_cornac
def test_rank_top10_is_the_host_ranking_of_theta_and_beta():
    from cornac_b200 import HPF
    g = golden("hpf_k10")
    ds = _dataset(g)
    m = HPF(k=10, max_iter=20, seed=4).fit(ds)
    n = ds.num_items
    for u in (0, 5, ds.num_users - 1):
        row = np.zeros(n)
        for f in range(10):                                   # the device dot: f ascending, no FMA
            row = row + m.Theta[u, f] * m.Beta[:, f]
        want = np.lexsort((np.arange(n), -row))[:10]
        ranked, scores = m.rank(u, k=10)
        assert np.array_equal(ranked[:10], want) and np.array_equal(scores, row)
        assert np.array_equal(m.score(u), row)
        assert np.all(np.abs(row - m.Beta.dot(m.Theta[u])) <= 1e-14 * np.max(np.abs(row)))
    ids, top = m.rank_batch(np.arange(ds.num_users), 10, exclude=ds.csr_matrix)
    for u in (0, 7):
        cand = np.setdiff1d(np.arange(n), ds.csr_matrix[u].indices)
        row = m.score(u)
        assert np.array_equal(ids[u], cand[np.lexsort((cand, -row[cand]))][:10])
    recs = m.recommend_batch([ds.user_ids[0], ds.user_ids[3]], k=5, remove_seen=True, train_set=ds)
    assert recs == [m.recommend(ds.user_ids[0], k=5, remove_seen=True, train_set=ds)[:5],
                    m.recommend(ds.user_ids[3], k=5, remove_seen=True, train_set=ds)[:5]]


@needs_cornac
def test_experiment_metrics_equal_the_reference():
    import cornac
    import cornac_b200
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, NDCG, Recall
    g = golden("hpf_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123, rating_threshold=0.5)
    models = [cornac_b200.HPF(k=5, seed=123, hierarchical=False, name="PF"), cornac_b200.HPF(k=5, seed=123)]
    exp = cornac.Experiment(eval_method=rs, models=models, metrics=[Recall(k=20), NDCG(k=20), AUC()], user_based=True,
                            verbose=False)
    exp.run()
    res = {r.model_name: r.metric_avg_results for r in exp.result}
    names = [str(n) for n in g["metric_names"]]
    for model, key in (("PF", "pf"), ("HPF", "hpf")):
        got = np.array([res[model][n] for n in names])
        assert np.all(np.abs(got - g[key]) <= 1e-9), (model, dict(zip(names, got)))


@needs_cornac
def test_save_load_and_untrained_scoring():
    from cornac_b200 import HPF
    g = golden("pf_k10")
    ds = _dataset(g)
    m = HPF(k=10, max_iter=10, hierarchical=False, seed=2).fit(ds)
    with tempfile.TemporaryDirectory() as d:
        m2 = HPF.load(m.save(d))
    for attr in ("Theta", "Beta", "Gs", "Gr", "Ls", "Lr"):
        assert np.array_equal(getattr(m2, attr), getattr(m, attr))
    assert np.array_equal(m2.score(3), m.score(3)) and m2.score(3, 4) == m.score(3, 4)
    assert np.array_equal(m2.rank(3, k=10)[0][:10], m.rank(3, k=10)[0][:10])
    m3 = HPF(k=10, trainable=False, init_params={"Theta": m.Theta, "Beta": m.Beta}).fit(ds)
    assert m3.Gs is None and np.array_equal(m3.score(3), m.score(3))
    assert np.array_equal(m3.rank(5, k=10)[0][:10], m.rank(5, k=10)[0][:10])
