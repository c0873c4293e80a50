"""C2PF on the GPU: one iteration bit-identical to the C oracle given the same expectations, split fits, the two-phase
fit against the compiled reference's fixtures, and the plug-in's scoring, ranking, persistence and Experiment contract."""
import contextlib
import io

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import golden, have_cornac, needs_cornac
from oracle import c2pf_oracle as CO

pytestmark = pytest.mark.gpu

VARIANTS = ("c2pf", "tc2pf", "rc2pf")
CASES = ["%s_%s" % (v, c) for v in VARIANTS for c in ("k1", "k5", "k37", "warm_k4", "nonpos_k4", "dup_k3")]
KEYS = ("G_s", "G_r", "L_s", "L_r", "L2_s", "L2_r", "L3_s", "L3_r")


def rel_max(got, want):
    return float(np.max(np.abs(got - want)) / np.max(np.abs(want)))


def problem(g):
    """(X, G, state with kappa on the pattern and T3_r) of a fixture."""
    n, d = int(g["num_users"]), int(g["num_items"])
    tX, C = g["tX"], g["C"]
    X = CO.csc(tX[:, 0].astype(int), tX[:, 1].astype(int), tX[:, 2], n, d)
    G = CO.Graph(C[:, 0], C[:, 1], C[:, 2], d)
    st = [g[key + "0"].copy() if key + "0" in g else None for key in KEYS]
    st[6], st[7] = G.values(st[6]), G.values(st[7])
    return tX, X, G, st + [np.ones(d)]


def office_problem(k, seed=5):
    """A seeded problem of the Amazon Office shape: 3 703 users x 6 523 items x 53 282 ratings, ~100 000 context edges."""
    rng = np.random.RandomState(seed)
    n, d, nnz = 3703, 6523, 53282
    key = rng.choice(n * d, size=nnz, replace=False)
    tX = np.column_stack([key // d, key % d, rng.randint(1, 6, size=nnz)]).astype(np.float64)
    pairs = np.unique(rng.choice(d * d, size=50500, replace=False))
    a, b = pairs // d, pairs % d
    a, b = a[a != b], b[a != b]
    G = CO.Graph(np.concatenate([a, b]), np.concatenate([b, a]), np.ones(2 * len(a)), d)
    X = CO.csc(tX[:, 0].astype(int), tX[:, 1].astype(int), tX[:, 2], n, d)
    st = [rng.gamma(100, 0.003, (rows, k)) for rows in (n, n, d, d, d, d)]
    st += [rng.gamma(100, 0.005, G.nnz), rng.gamma(100, 0.005, G.nnz), np.ones(d)]
    return tX, X, G, st


def for_variant(variant, st):
    st = [None if x is None else x.copy() for x in st]
    if variant == "tc2pf":
        st[4] = st[5] = None
    if variant == "rc2pf":
        st[2] = st[3] = None
    return st


def device_graph(tX, G, n):
    from cornac_b200 import engine
    data = engine.HpfData(tX[:, 0].astype(int), tX[:, 1].astype(int), tX[:, 2], n, G.d)
    return engine.C2pfGraph(data, G.ptr, G.row, G.mirrors(), G.util)


def dev(x):
    import torch
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x).copy()).cuda()


def check_update(variant, tX, X, G, st, at, bt):
    from cornac_b200 import engine
    E = CO.expectations(variant, G, st)
    dgraph = device_graph(tX, G, len(st[0]))
    dst, dE = [dev(x) for x in st], [dev(x) for x in E]
    CO.update(variant, X, G, at, bt, st, E)
    engine.c2pf_update(dgraph, variant, at, bt, dst, dE, given=[dev(x) for x in E[:4]])
    for j, (got, want) in enumerate(zip(dst + [dE[4]], st + [E[4]])):
        if want is not None and not (variant == "tc2pf" and j in (4, 5)):
            assert np.array_equal(got.cpu().numpy(), want), (variant, at, j)
    return dgraph, dst, dE


@pytest.mark.parametrize("name", CASES)
def test_update_is_bit_identical_to_the_oracle(name):
    g = golden(name)
    variant = str(g["variant"])
    for at, bt in (CO.PHASE_ONE, CO.PHASE_TWO[variant]):
        tX, X, G, st = problem(g)
        check_update(variant, tX, X, G, st, at, bt)


@pytest.mark.parametrize("variant", VARIANTS)
def test_update_is_bit_identical_at_the_office_shape(variant):
    tX, X, G, st = office_problem(100)
    check_update(variant, tX, X, G, for_variant(variant, st), *CO.PHASE_TWO[variant])


@pytest.mark.parametrize("variant", VARIANTS)
def test_split_fit_equals_one_fit(variant):
    from cornac_b200 import engine
    g = golden(variant + "_k5")
    tX, X, G, st = problem(g)
    dgraph = device_graph(tX, G, len(st[0]))
    for at, bt in (CO.PHASE_ONE, CO.PHASE_TWO[variant]):
        one, two = [dev(x) for x in st], [dev(x) for x in st]
        engine.c2pf_fit(dgraph, variant, at, bt, one, 7)
        engine.c2pf_fit(dgraph, variant, at, bt, two, 3)
        engine.c2pf_fit(dgraph, variant, at, bt, two, 4)
        for a, b in zip(one, two):
            assert a is None or np.array_equal(a.cpu().numpy(), b.cpu().numpy())


def _dataset(g, C=None):
    """A cornac Dataset whose user / item indices are the fixture's, with the context triplets as its item graph."""
    from cornac.data import Dataset, GraphModality
    tX = g["tX"]
    n, d = int(g["num_users"]), int(g["num_items"])
    C = g["C"] if C is None else C
    uid = {str(u): u for u in range(n)}
    iid = {str(i): i for i in range(d)}
    ds = Dataset.build(data=[(str(int(u)), str(int(i)), float(r)) for u, i, r in tX], fmt="UIR", global_uid_map=uid,
                       global_iid_map=iid, seed=None)
    gm = GraphModality(data=[(str(int(a)), str(int(b)), float(v)) for a, b, v in C])
    gm.build(id_map=ds.iid_map)
    ds.add_modalities(item_graph=gm)
    return ds


def _fit(g, m):
    """The plug-in's fit on a fixture's triplets as the reference's extension received them (a Dataset would drop the
    context of the fixture's unrated item before the fit sees it)."""
    from cornac_b200 import C2PF
    from cornac_b200.recom_c2pf import ContextGraph
    init = {key: g[key + "0"].copy() for key in KEYS if key + "0" in g}
    model = C2PF(k=int(g["k"]), max_iter=int(m), variant=str(g["variant"]), init_params=init)
    n, d, tX, C = int(g["num_users"]), int(g["num_items"]), g["tX"], g["C"]
    graph = ContextGraph(C, d)
    model._fit_b200(tX[:, 0].astype(int), tX[:, 1].astype(int), tX[:, 2], (n, d), graph, model._init_state(n, d, C, graph))
    return model


@needs_cornac
@pytest.mark.parametrize("name", CASES)
def test_two_phase_fit_matches_the_reference(name):
    g = golden(name)
    for m in g["iters"]:
        model = _fit(g, m)
        for key, attr in zip(KEYS + ("Z", "W", "Q"), ("Gs", "Gr", "Ls", "Lr", "L2s", "L2r", "L3s", "L3r", "Theta", "Beta", "Xi")):
            want = g["%s_%d" % (key, m)] if "%s_%d" % (key, m) in g else None
            got = getattr(model, attr)
            assert (got is None) == (want is None), (m, key)
            if want is not None:
                assert np.all(np.isfinite(got)) and rel_max(np.asarray(got), want) <= 1e-10, (m, key)


@needs_cornac
@pytest.mark.parametrize("variant", VARIANTS)
def test_scores_ranks_and_persistence(variant, tmp_path):
    from cornac_b200 import C2PF
    g = golden(variant + "_k5")
    np.random.seed(3)
    with contextlib.redirect_stdout(io.StringIO()) as out:
        model = C2PF(k=5, max_iter=6, variant=variant).fit(_dataset(g))
    assert out.getvalue() == "Learning...\nLearning completed!\n"
    assert model.name == variant.upper() and (model.L2s is None) == (variant == "tc2pf") and (model.Ls is None) == (variant == "rc2pf")
    Theta, Beta, Xi = (np.asarray(x) for x in (model.Theta, model.Beta, model.Xi))
    items = Xi if variant == "rc2pf" else Beta + Xi
    d = items.shape[0]
    for u in (0, 7, Theta.shape[0] - 1):
        want = (Xi.dot(Theta[u]) if variant == "rc2pf" else Beta.dot(Theta[u]) + Xi.dot(Theta[u]))
        got = model.score(u)
        assert got.dtype == np.float64 and np.max(np.abs(got - want)) <= 1e-12 * np.max(np.abs(want))
        ranked, scores = model.rank(u)
        assert np.array_equal(scores, got) and np.array_equal(ranked, got.argsort()[::-1])     # Recommender.rank's order
        ranked5, _ = model.rank(u, k=5)
        assert np.array_equal(got[ranked5[:5]], got[ranked[:5]]) and sorted(ranked5) == list(range(d))
        one = model.score(u, 3)
        ref = (Xi[3] * Theta[u]).sum() if variant == "rc2pf" else Beta[3].dot(Theta[u]) + Xi.dot(Theta[u])
        assert np.allclose(one, np.ravel(ref), rtol=1e-12, atol=0)
    users = np.arange(10)
    ids, sc = model.rank_batch(users, 6)
    for q, u in enumerate(users):
        row = model.score(int(u))
        assert np.array_equal(ids[q], np.lexsort((np.arange(d), -row))[:6]) and np.array_equal(sc[q], row[ids[q]])
    recs = model.recommend_batch([str(u) for u in users], k=6)
    assert [[int(i) for i in r] for r in recs] == ids.tolist()
    path = model.save(str(tmp_path))
    loaded = C2PF.load(path)
    assert np.array_equal(loaded.score(2), model.score(2))
    frozen = C2PF(k=5, variant=variant, trainable=False, init_params=dict(Theta=model.Theta, Beta=model.Beta, Xi=model.Xi))
    frozen.fit(_dataset(g))
    assert np.array_equal(frozen.score(2), model.score(2))
    # a warm start: a second fit() continues from the stored state
    before = model.Gs.copy()
    with contextlib.redirect_stdout(io.StringIO()):
        model.fit(_dataset(g))
    assert not np.array_equal(before, model.Gs) and np.all(np.isfinite(model.Theta))


@needs_cornac
def test_no_item_graph_and_asymmetric_graph_raise():
    from cornac.data import Dataset
    from cornac_b200 import C2PF
    g = golden("c2pf_k1")
    ds = Dataset.from_uir([(str(int(u)), str(int(i)), float(r)) for u, i, r in g["tX"]], seed=None)
    with pytest.raises(ValueError, match="item_graph"):
        C2PF(k=1, max_iter=1).fit(ds)
    a = golden("c2pf_asym")
    with pytest.raises(ValueError, match="symmetric=True"):
        C2PF(k=1, max_iter=1).fit(_dataset(g, C=a["C"]))


@pytest.mark.skipif(not have_cornac(), reason="reference cornac install (oracle/_ref) not importable")
def test_experiment_metrics_equal_the_reference(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)                             # Experiment writes its log to the working directory
    import cornac
    from cornac.data import GraphModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import MRR, NDCG, Precision, Recall
    from cornac_b200 import C2PF
    g = golden("c2pf_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    graph = [(str(int(a)), str(int(b)), float(v)) for a, b, v in g["C"]]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123, rating_threshold=0.5,
                    item_graph=GraphModality(data=graph))
    metrics = [NDCG(k=-1), MRR(), Recall(k=20), Precision(k=20)]
    assert [m.name for m in metrics] == list(g["metric_names"])
    for variant in ("c2pf", "tc2pf"):
        np.random.seed(5)
        with contextlib.redirect_stdout(io.StringIO()):
            exp = cornac.Experiment(eval_method=rs, models=[C2PF(k=6, max_iter=10, variant=variant)], metrics=metrics,
                                    user_based=True, verbose=False)
            exp.run()
        got = np.array([exp.result[0].metric_avg_results[m.name] for m in metrics])
        assert np.max(np.abs(got - g[variant])) <= 1e-12, (variant, got, g[variant])
