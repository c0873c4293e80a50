"""SoRec and MCF on the GPU: b200_cofactor_fit bit-identical to the compiled reference's fixtures and to the serial oracle
at FilmTrust and Epinions scale, the loss terms, and the plug-ins through ranking, save / load and an unchanged
Experiment."""
import io
import os
import sys
import tempfile
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from conftest import ROOT, golden, needs_cornac
from oracle import cofactor_oracle as CO

sys.path.insert(0, os.path.join(ROOT, "tools"))
from cofactor_bench import SHAPES, synth  # noqa: E402

pytestmark = pytest.mark.gpu

FIT_CASES = ["sorec_k5", "sorec_nolink_k10", "sorec_k1", "sorec_k37", "sorec_step_product", "sorec_minmax",
             "sorec_loops_dups", "sorec_empty_graph", "sorec_warm_k6", "mcf_k5", "mcf_unit_k10", "mcf_const_k1",
             "mcf_warm_k37"]


def device_fit(variant, net_a, net_b, net_val, uid, iid, rat, n_users, n_items, U0, V0, Z0, n_epochs, lambda_c,
               lambda_reg, lr, gamma, loss=False, split=None):
    from cornac_b200 import engine
    data = engine.CofactorData(variant, net_a, net_b, net_val, uid, iid, rat, n_users, n_items)
    dev = [engine.to_device(x, torch.float64) for x in (U0, V0, Z0)]
    caches = [torch.zeros_like(x) for x in dev]
    hyper = (lambda_c, lambda_reg, lr, gamma)
    terms = torch.empty((n_epochs, len(net_a) + len(uid)), dtype=torch.float64, device="cuda") if loss else None
    if split is None:
        engine.cofactor_fit(data, *dev, *caches, n_epochs, *hyper, loss=terms)
    else:                                                     # two calls of a and b epochs == one call of a + b
        engine.cofactor_fit(data, *dev, *caches, split, *hyper)
        engine.cofactor_fit(data, *dev, *caches, n_epochs - split, *hyper)
    out = tuple(x.cpu().numpy() for x in dev)
    return out + (terms.cpu().numpy(),) if loss else out


def _fixture_args(g):
    return (str(g["model"]), g["net_a"], g["net_b"], g["net_val"], g["uid"], g["iid"], g["rat"], int(g["num_users"]),
            int(g["num_items"]), g["U0"], g["V0"], g["Z0"], int(g["max_iter"]), float(g["lambda_c"]),
            float(g["lambda_reg"]), float(g["learning_rate"]), float(g["gamma"]))


def _same(got, g):
    return all(np.array_equal(x, g[n]) for x, n in zip(got, "UVZ"))


@pytest.mark.parametrize("split", [None, 4])
@pytest.mark.parametrize("name", FIT_CASES)
def test_fit_is_bit_identical_to_the_reference(name, split):
    g = golden(name)
    assert _same(device_fit(*_fixture_args(g), split=split), g)


@pytest.mark.parametrize("name", ["sorec_k5", "sorec_step_product", "mcf_unit_k10"])
def test_loss_terms_equal_the_reference(name):
    g = golden(name)
    *factors, terms = device_fit(*_fixture_args(g), loss=True)
    assert _same(factors, g)
    assert np.array_equal(np.add.accumulate(terms, axis=1)[:, -1], g["loss"])
    U, V, Z = g["U0"].copy(), g["V0"].copy(), g["Z0"].copy()
    _, want = CO.fit(str(g["model"]), g["net_a"], g["net_b"], g["net_val"], g["uid"], g["iid"], g["rat"], U, V, Z,
                     int(g["max_iter"]), float(g["lambda_c"]), float(g["lambda_reg"]), float(g["learning_rate"]),
                     float(g["gamma"]), terms=True)
    assert np.array_equal(terms, want)


@pytest.mark.parametrize("order", ["shuffled", "csr"])
@pytest.mark.parametrize("shape", [s[0] for s in SHAPES])
def test_bench_shapes_are_bit_identical_to_the_oracle(shape, order):
    name, variant, nu, ni, nr, ne = next(s for s in SHAPES if s[0] == shape)
    net_a, net_b, net_val, uid, iid, rat = synth(variant, nu, ni, nr, ne, seed=3, order=order)
    rng = np.random.RandomState(4)
    n_z = nu if variant == "sorec" else ni
    init = [rng.normal(0, 0.01, (n, 10)) for n in (nu, ni, n_z)]
    got = device_fit(variant, net_a, net_b, net_val, uid, iid, rat, nu, ni, *init, 2, 10.0, 0.001, 0.01, 0.9)
    want = [x.copy() for x in init]
    CO.fit(variant, net_a, net_b, net_val, uid, iid, rat, *want, 2, 10.0, 0.001, 0.01, 0.9)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_smoke_step():
    import __graft_entry__
    __graft_entry__.smoke_cofactor(np.random.RandomState(0))


# ---- plug-ins --------------------------------------------------------------------------------------------------------
def _dataset(g):
    from cornac.data import Dataset, GraphModality
    ds = Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])], seed=None)
    sorec = str(g["model"]) == "sorec"
    gm = GraphModality(data=[(str(a), str(b), float(v)) for a, b, v in zip(g["graph_a"], g["graph_b"], g["graph_val"])])
    gm.build(id_map=ds.uid_map if sorec else ds.iid_map)
    ds.add_modalities(**{("user_graph" if sorec else "item_graph"): gm})
    return ds


def _model(g, **kw):
    import cornac_b200
    hyper = {str(n): float(v) for n, v in zip(g["hyper_names"], g["hyper_values"])}
    if "weight_link" in hyper:
        hyper["weight_link"] = bool(hyper["weight_link"])
    cls = cornac_b200.SoRec if str(g["model"]) == "sorec" else cornac_b200.MCF
    return cls(**dict(dict(hyper, k=int(g["k"]), max_iter=int(g["max_iter"]), seed=int(g["seed"])), **kw))


@needs_cornac
@pytest.mark.parametrize("name", [n for n in FIT_CASES if "warm" not in n])
def test_plugin_fit_and_scores_match_the_reference(name):
    g = golden(name)
    m = _model(g).fit(_dataset(g))
    assert np.array_equal(m.U, g["U"]) and np.array_equal(m.V, g["V"]) and np.array_equal(m.Z, g["Z"])
    single = np.array([m.score(int(u), int(i)) for u, i in g["single_pairs"]])
    assert np.array_equal(single, g["single_scores"])


@needs_cornac
@pytest.mark.parametrize("name", ["sorec_warm_k6", "mcf_warm_k37"])
def test_init_params_are_trained_in_place(name):
    g = golden(name)
    given = {str(key): g[str(key) + "0"].copy() for key in g["init_given"]}
    m = _model(g, init_params=dict(given)).fit(_dataset(g))
    for key, x in given.items():
        assert getattr(m, key) is x
    assert np.array_equal(m.U, g["U"]) and np.array_equal(m.V, g["V"]) and np.array_equal(m.Z, g["Z"])


@needs_cornac
@pytest.mark.parametrize("name", ["sorec_nolink_k10", "mcf_k5", "sorec_empty_graph"])
def test_verbose_prints_the_reference_losses(name):
    g = golden(name)
    m = _model(g, verbose=True)
    m._B200_LOSS_BYTES = 8 * (len(g["net_a"]) + len(g["uid"])) * 3      # several epoch chunks
    buf = io.StringIO()
    with redirect_stdout(buf):
        m.fit(_dataset(g))
    lines = [x for x in buf.getvalue().splitlines() if x.startswith("epoch")]
    assert lines == ["epoch %i, loss: %f" % (e, x) for e, x in enumerate(g["loss"])]
    assert np.array_equal(m.U, g["U"])


@needs_cornac
@pytest.mark.parametrize("name", ["sorec_k5", "mcf_k5"])
def test_plugin_matches_reference_edge_behaviour(name):
    from cornac.exception import ScoreException
    from cornac.models import MCF as RefMCF, SoRec as RefSoRec
    import cornac_b200
    g = golden(name)
    ds = _dataset(g)
    ref_cls, cls = (RefSoRec, cornac_b200.SoRec) if str(g["model"]) == "sorec" else (RefMCF, cornac_b200.MCF)
    kw = dict(k=5, max_iter=5, seed=3, learning_rate=0.05)
    ref, ours = ref_cls(**kw).fit(ds), cls(**kw).fit(ds)
    assert np.array_equal(ref.U, ours.U) and np.array_equal(ref.V, ours.V) and np.array_equal(ref.Z, ours.Z)
    for call in (lambda m: m.score(ds.num_users), lambda m: m.score(0, ds.num_items)):
        msgs = []
        for m in (ref, ours):
            with pytest.raises(ScoreException) as e:
                call(m)
            msgs.append(str(e.value))
        assert msgs[0] == msgs[1]
    for u in (0, 5, ds.num_users - 1):
        raw = ours.score(u)                                    # the raw dot, not the sigmoid
        assert np.all(np.abs(raw - ref.score(u)) <= 1e-14 * np.abs(ref.V).dot(np.abs(ref.U[u])))
        assert ours.score(u, 3) == ref.score(u, 3)
    ours.transform(ds)                                         # a cached row never answers the single-item case
    assert ours.score(1, 4) == ref.score(1, 4)


@needs_cornac
@pytest.mark.parametrize("name", ["sorec_nolink_k10", "mcf_unit_k10"])
def test_rank_and_rank_batch_follow_recommender_rank(name):
    from cornac.models import Recommender
    g = golden(name)
    ds = _dataset(g)
    m = _model(g, max_iter=5).fit(ds)
    n = ds.num_items
    rng = np.random.RandomState(0)
    for cached in (False, True):
        if cached:
            m.transform(ds)
        for u in (0, 17, ds.num_users - 1):
            want_ids, want_sc = Recommender.rank(m, u)         # the reference's rank over score(u)
            ranked, sc = m.rank(u)
            assert np.array_equal(ranked, want_ids) and np.array_equal(sc, want_sc)
            cand = np.sort(rng.choice(n, size=50, replace=False))
            want_ids, want_sc = Recommender.rank(m, u, cand, k=5)
            ranked, sc = m.rank(u, cand, k=5)
            assert np.array_equal(ranked[:5], want_ids[:5]) and np.array_equal(sc, want_sc)
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
@pytest.mark.parametrize("name", ["sorec_k5", "mcf_k5"])
def test_save_load_and_trainable_false(name):
    g = golden(name)
    ds = _dataset(g)
    m = _model(g, max_iter=10).fit(ds)
    with tempfile.TemporaryDirectory() as d:
        path = m.save(d)
        m2 = type(m).load(path)
    for key in "UVZ":
        assert np.array_equal(getattr(m2, key), getattr(m, key))
    assert np.array_equal(m2.score(3), m.score(3))
    assert np.array_equal(m2.rank(3, k=10)[0][:10], m.rank(3, k=10)[0][:10])
    c = m.clone()
    assert c.k == m.k and c.seed == m.seed
    frozen = type(m)(k=m.k, trainable=False, init_params={"U": m.U.copy(), "V": m.V.copy(), "Z": m.Z.copy()}).fit(ds)
    assert np.array_equal(frozen.U, m.U) and np.array_equal(frozen.score(2), m.score(2))


@needs_cornac
@pytest.mark.parametrize("model", ["sorec", "mcf"])
def test_experiment_metrics_equal_the_reference(model):
    import cornac
    import cornac_b200
    from cornac.data import GraphModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import NDCG, RMSE, Precision, Recall
    g = golden(model + "_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    gm = GraphModality(data=[(str(a), str(b), float(v)) for a, b, v in zip(g["graph_a"], g["graph_b"], g["graph_val"])])
    if model == "sorec":
        rs = RatioSplit(data=data, test_size=0.2, rating_threshold=2.5, exclude_unknowns=True, verbose=False,
                        user_graph=gm, seed=123)
        m = cornac_b200.SoRec(k=10, max_iter=50, learning_rate=0.001, verbose=False, seed=123)
        metrics = [RMSE(), NDCG(k=-1), Precision(k=20), Recall(k=20)]
    else:
        rs = RatioSplit(data=data, test_size=0.2, rating_threshold=3.5, exclude_unknowns=True, verbose=False,
                        item_graph=gm, seed=123)
        m = cornac_b200.MCF(k=10, max_iter=40, learning_rate=0.001, verbose=False, seed=123)
        metrics = [RMSE(), NDCG(k=-1), Recall(k=20), Precision(k=20)]
    exp = cornac.Experiment(eval_method=rs, models=[m], metrics=metrics, verbose=False)
    exp.run()
    res = exp.result[0].metric_avg_results
    got = np.array([res[str(n)] for n in g["metric_names"]])
    assert np.all(np.abs(got - g["metrics"]) <= 1e-12), (dict(zip(g["metric_names"], got)), g["metrics"])
