"""EASE on the GPU: the Gram matrix bit for bit, the FP64 tensor-core SPD inverse against numpy, the weights and score rows
bit for bit given the same inputs, the plug-in against the reference's fixtures and an unchanged Experiment."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import golden, needs_cornac, synth_csr

pytestmark = pytest.mark.gpu

CASES = ["ease_l500_pos", "ease_l500_all", "ease_l1_pos", "ease_l001_all", "ease_n1", "ease_n130", "ease_tie"]


def torch_():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


def fixture_matrix(g):
    return sp.csr_matrix((g["X_data"], g["X_indices"], g["X_indptr"]), shape=(int(g["num_users"]), int(g["num_items"])))


def host_gram(X, lamb):
    G = X.T.dot(X).toarray()
    G[np.diag_indices(G.shape[0])] = G.diagonal() + lamb
    return np.ascontiguousarray(G)


def device_gram(X, lamb):
    torch = torch_()
    from cornac_b200 import engine
    n = X.shape[1]
    G = torch.empty((n, n), dtype=torch.float64, device="cuda")
    return engine.ease_gram(engine.EaseGramInput(X), lamb, G)


def synth_X(n_users, n_items, nnz, seed, dyadic=True):
    indptr, indices = synth_csr(n_users, n_items, nnz, seed)
    rng = np.random.RandomState(seed + 1)
    data = rng.randint(1, 6, size=len(indices)).astype(np.float64)
    if not dyadic:
        data = data * 0.7 + rng.uniform(0, 0.1, size=len(data))
    return sp.csr_matrix((data, indices, indptr), shape=(n_users, n_items))


def host_weights(P, posB):
    B = P / (-np.diag(P))
    B[np.diag_indices(B.shape[0])] = 0.0
    if posB:
        B[B < 0] = 0
    return B


def lexsort_top(rows, k, excl=None):
    out = []
    for q, r in enumerate(rows):
        ids = np.arange(len(r))
        if excl is not None:
            keep = np.ones(len(r), bool)
            keep[excl[q]] = False
            ids = ids[keep]
        out.append(ids[np.lexsort((ids, -r[ids]))][:k])
    return np.stack(out)


# ---- 1. Gram ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_gram_is_scipy_on_the_fixtures(name):
    g = golden(name)
    X = fixture_matrix(g)
    assert np.array_equal(device_gram(X, float(g["lamb"])).cpu().numpy(), host_gram(X, float(g["lamb"])))


def test_gram_is_scipy_on_an_ml1m_shape_with_non_dyadic_ratings():
    X = synth_X(6040, 3706, 1_000_000, 11, dyadic=False)
    assert np.array_equal(device_gram(X, 500.0).cpu().numpy(), host_gram(X, 500.0))


def test_gram_is_scipy_on_the_workspace_accumulator_path():
    """Above 28 160 items one f64 accumulator row no longer fits shared memory: the rows accumulate in the workspace."""
    torch = torch_()
    from cornac_b200 import _lib
    n = 28_300
    assert _lib.load().b200_ease_gram_workspace_bytes(n) > 0
    X = synth_X(3000, n, 60_000, 12, dyadic=False)
    got = device_gram(X, 3.0)
    Gs = X.T.dot(X).tocoo()
    want = torch.zeros((n, n), dtype=torch.float64, device="cuda")
    want.view(-1)[torch.from_numpy(Gs.row.astype(np.int64) * n + Gs.col).cuda()] = torch.from_numpy(Gs.data).cuda()
    diag = X.T.dot(X).diagonal() + 3.0
    want.view(-1)[torch.arange(n, device="cuda") * (n + 1)] = torch.from_numpy(diag).cuda()
    assert torch.equal(got.view(torch.int64), want.view(torch.int64))


# ---- 2. inverse ------------------------------------------------------------------------------------------------------
def spd(n, lamb, seed):
    X = synth_X(max(2 * n, 20), n, max(6 * n, 10), seed)
    return host_gram(X, lamb)


@pytest.mark.parametrize("n", [1, 2, 3, 63, 64, 65, 127, 128, 129, 1000, 3706])
def test_inverse_against_numpy(n):
    torch = torch_()
    from cornac_b200 import engine
    for lamb in (500.0, 1.0, 0.01):
        G = spd(n, lamb, n)
        A = torch.from_numpy(G).cuda()
        P = engine.spd_inverse(A.clone()).cpu().numpy()
        assert np.array_equal(P, P.T)
        back = np.linalg.norm(G @ P - np.eye(n)) / (np.linalg.norm(G) * np.linalg.norm(P))
        assert back <= 1e-14, (lamb, back)
        if lamb == 500.0:
            want = np.linalg.inv(G)
            assert np.linalg.norm(P - want) <= 1e-12 * np.linalg.norm(want)
        again = engine.spd_inverse(A.clone()).cpu().numpy()
        assert np.array_equal(P, again)


# ---- 3. singular input -----------------------------------------------------------------------------------------------
def test_singular_input_raises_linalg_error_naming_the_column():
    torch_()
    from cornac_b200 import engine
    X = synth_X(200, 90, 1500, 3)
    X = X.tolil()
    X[:, 37] = 0
    X = X.tocsr()
    X.eliminate_zeros()
    with pytest.raises(np.linalg.LinAlgError, match="column 37"):
        engine.ease_fit(X, 0.0, True)
    d = host_gram(X, 0.0).diagonal()
    with pytest.raises(np.linalg.LinAlgError, match="column 0 "):
        engine.ease_fit(X, -(d.max() + 1.0), True)
    B = engine.ease_fit(X, 500.0, True).cpu().numpy()
    assert np.isfinite(B).all()


# ---- 4. weights and scores -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("posB", [True, False])
def test_weights_are_numpy_given_p(posB):
    torch = torch_()
    from cornac_b200 import engine
    P = np.linalg.inv(spd(300, 5.0, 8))
    got = engine.ease_weights(torch.from_numpy(np.ascontiguousarray(P)).cuda(), posB).cpu().numpy()
    assert np.array_equal(got, host_weights(P, posB))
    assert np.array_equal(np.signbit(got), np.signbit(host_weights(P, posB)))


@pytest.mark.parametrize("name", CASES)
def test_scores_are_scipy_given_b(name):
    torch = torch_()
    from cornac_b200 import engine
    g = golden(name)
    X = fixture_matrix(g)
    B = torch.from_numpy(np.ascontiguousarray(g["B"])).cuda()
    got = engine.ease_score(B, g["query_users"], engine.EaseRatings(X)).cpu().numpy()
    assert np.array_equal(got.view(np.int64), g["query_scores"].view(np.int64))
    users = np.arange(X.shape[0])
    rows = engine.ease_score(B, users, engine.EaseRatings(X))
    want = X.dot(g["B"])
    assert np.array_equal(rows.cpu().numpy().view(np.int64), want.view(np.int64))
    excl = [X[u].indices for u in users]
    ep = torch.from_numpy(X.indptr.astype(np.int64)).cuda()
    ei = torch.from_numpy(X.indices.astype(np.int32) if X.nnz else np.zeros(1, np.int32)).cuda()
    k = min(10, X.shape[1])
    ids, _ = engine.topk_rows_f64(rows, k, ep, ei)
    ids = ids.cpu().numpy()
    for q in users:
        n_left = X.shape[1] - len(excl[q])
        want_q = lexsort_top(want[q:q + 1], k, [excl[q]])[0][:n_left]
        assert np.array_equal(ids[q][:len(want_q)], want_q)


def test_score_rows_whose_products_are_all_negative_zero():
    """scipy starts every output at +0.0: a row whose only products are -0.0 scores +0.0, where an accumulator seeded with
    the first product would give -0.0."""
    torch = torch_()
    from cornac_b200 import engine
    X = sp.csr_matrix((np.array([1.0, -1.0, -1.0, 2.0]), np.array([0, 1, 0, 1]), np.array([0, 1, 2, 4])), shape=(3, 2))
    B = np.array([[-0.0, 1.0], [0.0, -0.0]])
    got = engine.ease_score(torch.from_numpy(B).cuda(), [0, 1, 2], engine.EaseRatings(X)).cpu().numpy()
    want = X.dot(B)
    assert not np.signbit(want[0, 0]) and not np.signbit(want[1, 0])
    assert np.array_equal(got.view(np.int64), want.view(np.int64))


def test_score_refuses_mismatched_inputs():
    torch = torch_()
    from cornac_b200 import B200Error, engine
    X = synth_X(30, 20, 100, 6)
    r = engine.EaseRatings(X)
    with pytest.raises(B200Error):
        engine.ease_score(torch.zeros((19, 19), dtype=torch.float64, device="cuda"), [0], r)
    with pytest.raises(B200Error):
        engine.ease_score(torch.zeros((20, 19), dtype=torch.float64, device="cuda"), [0], r)
    B = torch.zeros((20, 20), dtype=torch.float64, device="cuda")
    for bad in ([30], [-1], torch.tensor([30], device="cuda")):
        with pytest.raises(B200Error):
            engine.ease_score(B, bad, r)


# ---- 5. plug-in against the fixtures ---------------------------------------------------------------------------------
def fitted(g):
    from cornac.data import Dataset
    from cornac_b200 import EASE
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    ds = Dataset.from_uir(data, seed=None)
    return EASE(lamb=float(g["lamb"]), posB=bool(g["posB"]), verbose=False).fit(ds), ds


@needs_cornac
@pytest.mark.parametrize("name", CASES)
def test_plugin_against_the_fixtures(name, tmp_path):
    torch_()
    g = golden(name)
    m, ds = fitted(g)
    Bref = g["B"]
    assert np.max(np.abs(m.B - Bref)) <= 1e-12 * max(np.max(np.abs(Bref)), 1e-300)
    assert (m.U != fixture_matrix(g)).nnz == 0
    u0 = int(g["query_users"][0])
    assert m.score(u0).shape == (1, m.num_items)
    assert np.asarray(m.score(u0, 0)).shape == (1,)
    assert np.array_equal(m.score(u0, 0), m.U[u0, :].dot(m.B[:, 0]))
    # score rows from the plug-in's own B are scipy's bit for bit; against the reference's within rounding
    for q, u in enumerate(g["query_users"]):
        row = m.score(int(u))[0]
        assert np.array_equal(row, m.U[int(u), :].dot(m.B)[0])
        ref = g["query_scores"][q]
        assert np.max(np.abs(row - ref)) <= 1e-11 * max(np.max(np.abs(ref)), 1.0)
    # rank top-10 of the unrated items, in (score desc, id asc)
    for u in g["query_users"]:
        cand = np.setdiff1d(np.arange(m.num_items), m.U[int(u)].indices)
        if len(cand) == 0:
            continue
        k = min(10, len(cand))
        ranked, _ = m.rank(int(u), item_indices=cand, k=k)
        row = m.score(int(u))[0]
        assert np.array_equal(ranked[:k], cand[np.lexsort((cand, -row[cand]))][:k])
        # the reference's top-k of the same candidates: the same items up to ties, judged by the reference's own scores
        ref_top = g["rank_top10"][list(g["query_users"]).index(u)][:k]
        ref_row = g["query_scores"][list(g["query_users"]).index(u)]
        scale = max(np.max(np.abs(ref_row)), 1.0)
        assert np.allclose(ref_row[ranked[:k]], ref_row[ref_top], rtol=0, atol=1e-11 * scale)
    users = np.arange(m.num_users)
    ids, sc = m.rank_batch(users, min(5, m.num_items), exclude=ds.csr_matrix)
    for q in users[:20]:
        excl = ds.csr_matrix[q].indices
        want = lexsort_top(m.score(int(q)), min(5, m.num_items), [excl])[0]
        assert np.array_equal(ids[q][:len(want)], want)
    some = list(m.user_ids[:25])
    kr = min(3, m.num_items)
    recs = m.recommend_batch(some, k=kr, remove_seen=True, train_set=ds)
    assert recs == [m.recommend(uid, k=kr, remove_seen=True, train_set=ds) for uid in some]
    u_idx = np.array([m.uid_map[uid] for uid in some])
    top, _ = m.rank_batch(u_idx, kr, exclude=ds.csr_matrix)
    assert recs == [[m.item_ids[i] for i in row if i >= 0] for row in top]
    from cornac_b200 import EASE
    m2 = EASE.load(m.save(str(tmp_path)))
    assert np.array_equal(m2.B, m.B)
    assert np.array_equal(m2.score(u0), m.score(u0))


def test_tie_fixture_orders_exact_zeros_by_id():
    torch_()
    g = golden("ease_tie")
    m, _ = fitted(g)
    row = m.score(0)[0]
    zeros = np.flatnonzero(row == 0.0)
    assert np.all(row[20:] == 0.0) and len(zeros) >= 20
    ranked, _ = m.rank(0)
    pos = ranked[np.isin(ranked, zeros)]
    assert np.array_equal(pos, np.sort(pos))


# ---- 6. unchanged Experiment -----------------------------------------------------------------------------------------
@needs_cornac
def test_experiment_metrics_equal_the_reference():
    torch_()
    import cornac
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import NDCG, Recall
    from cornac_b200 import EASE
    g = golden("ease_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, seed=123, rating_threshold=0.8, verbose=False)
    models = [EASE(lamb=500, name="pos", posB=True, verbose=False), EASE(lamb=500, name="all", posB=False, verbose=False)]
    exp = cornac.Experiment(eval_method=rs, models=models, metrics=[Recall(k=20), Recall(k=50), NDCG(k=100)],
                            user_based=True, save_dir=None, verbose=False)
    exp.run()
    res = {r.model_name: r.metric_avg_results for r in exp.result}
    for key in ("pos", "all"):
        got = np.array([res[key][str(n)] for n in g["metric_names"]])
        np.testing.assert_allclose(got, g[key], rtol=0, atol=1e-12)


# ---- 7. memory refusal -----------------------------------------------------------------------------------------------
def test_refuses_before_allocating_when_the_matrix_does_not_fit(monkeypatch):
    torch = torch_()
    from cornac_b200 import B200Error, engine
    X = synth_X(100, 5000, 2000, 4)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (5000 * 5000 * 8 - 1, 80 << 30))
    monkeypatch.setattr(torch.cuda, "memory_reserved", lambda *a: 0)
    monkeypatch.setattr(torch.cuda, "memory_allocated", lambda *a: 0)
    before = torch.cuda.memory_stats().get("allocated_bytes.all.allocated", 0)
    with pytest.raises(B200Error, match="5000 x 5000"):
        engine.ease_fit(X, 500.0, True)
    assert torch.cuda.memory_stats().get("allocated_bytes.all.allocated", 0) == before


# ---- 8. full size ----------------------------------------------------------------------------------------------------
def test_full_size_ml20m_shape():
    torch = torch_()
    from cornac_b200 import engine
    n_users, n = 138_493, 26_744
    X = synth_X(n_users, n, 20_000_000, 20)
    A = device_gram(X, 500.0)
    engine.spd_inverse(A)
    P = A.cpu().numpy()
    rng = np.random.RandomState(0)
    for _ in range(3):
        x = rng.normal(size=n)
        y = P @ x
        r = X.T.dot(X.dot(y)) + 500.0 * y - x
        assert np.linalg.norm(r) <= 1e-10 * np.linalg.norm(x)
    del P
    engine.ease_weights(A, True)
    users = rng.choice(n_users, 1000, replace=False)
    rows = engine.ease_score(A, users, engine.EaseRatings(X))
    sub = X[users]
    ep = torch.from_numpy(sub.indptr.astype(np.int64)).cuda()
    ei = torch.from_numpy(sub.indices.astype(np.int32)).cuda()
    ids, _ = engine.topk_rows_f64(rows, 100, ep, ei)
    Bh = A.cpu().numpy()
    want = sub.dot(Bh)
    assert np.array_equal(rows.cpu().numpy(), want)
    assert np.array_equal(ids.cpu().numpy(), lexsort_top(want, 100, [sub[q].indices for q in range(1000)]))
