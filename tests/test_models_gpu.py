"""The drop-in plug-ins through the reference's own Python stack (unchanged cornac from
oracle/_ref): fit / score / rank / ranking_eval / Experiment / clone / save-load.  GPU only.
Mirrors the reference's smoke tests (tests/cornac/models/test_recommender.py:28-53,
tests/cornac/eval_methods/test_ratio_split.py:92-109, tests/cornac/test_hyperopt.py:39-55)
and adds the value checks the reference lacks."""
import os
from collections import OrderedDict

import numpy as np
import pytest

from conftest import golden, needs_cornac, rel_err

pytestmark = [pytest.mark.gpu, needs_cornac]
TOL = 1e-4


def _dataset_from_csr(g):
    from cornac.data import Dataset
    indptr, indices, data = g["indptr"], g["indices"], g["data"]
    rows = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    # Dataset keeps id order of first appearance: feed users / items so that idx == raw id
    n_users, n_items = int(g["total_users"]), int(g["total_items"])
    uid_map = OrderedDict((str(u), u) for u in range(n_users))
    iid_map = OrderedDict((str(i), i) for i in range(n_items))
    triples = [(str(u), str(i), float(r)) for u, i, r in zip(rows, indices, data)]
    return Dataset.build(triples, global_uid_map=uid_map, global_iid_map=iid_map)


@pytest.mark.parametrize("name", ["bpr_small_k10", "bpr_mid_k32", "bpr_nobias_k16"])
def test_bpr_plugin_reproduces_seeded_reference(name):
    from cornac_b200 import BPR
    g = golden(name)
    ds = _dataset_from_csr(g)
    assert np.array_equal(ds.matrix.indices, g["indices"])
    m = BPR(k=int(g["k"]), max_iter=int(g["max_iter"]), learning_rate=float(g["lr"]), lambda_reg=float(g["reg"]),
            use_bias=bool(g["use_bias"]), seed=int(g["seed"])).fit(ds)
    assert m.u_factors.dtype == np.float32 and m.u_factors.shape == g["U"].shape
    assert rel_err(m.u_factors, g["U"]) < TOL and rel_err(m.i_factors, g["V"]) < TOL
    if bool(g["use_bias"]):
        assert rel_err(m.i_biases, g["B"]) < TOL
    for qi, q in enumerate(g["query_users"]):
        s = m.score(int(q))
        assert s.dtype == np.float32 and np.allclose(s, g["query_scores"][qi], rtol=1e-4, atol=1e-6)
        seen = g["excl_indices"][g["excl_indptr"][qi]:g["excl_indptr"][qi + 1]]
        cand = np.setdiff1d(np.arange(int(g["num_items"])), seen)
        ranked, item_scores = m.rank(int(q), item_indices=cand, k=10)
        assert np.array_equal(ranked[:10], g["top10"][qi])
        assert sorted(ranked.tolist()) == cand.tolist() and np.array_equal(item_scores, s[cand])
        assert np.isclose(m.score(int(q), 3), s[3], rtol=1e-5, atol=1e-6)
    # batched API == per-user API
    ids, sc = m.rank_batch(g["query_users"], 10, exclude=ds.csr_matrix)
    assert np.array_equal(ids, g["top10"])


@pytest.mark.parametrize("name", ["mf_small_k10", "mf_mid_k32", "mf_nobias_k16"])
def test_mf_plugin_reproduces_seeded_reference(name):
    from cornac.data import Dataset
    from cornac_b200 import MF
    g = golden(name)
    n_users, n_items = int(g["num_users"]), int(g["num_items"])
    uid_map = OrderedDict((str(u), u) for u in range(n_users))
    iid_map = OrderedDict((str(i), i) for i in range(n_items))
    ds = Dataset.build([(str(u), str(i), float(r)) for u, i, r in zip(g["rid"], g["cid"], g["val"])],
                       global_uid_map=uid_map, global_iid_map=iid_map)
    m = MF(k=int(g["k"]), max_iter=int(g["max_iter"]), learning_rate=float(g["lr"]), lambda_reg=float(g["reg"]),
           use_bias=bool(g["use_bias"]), early_stop=False, seed=int(g["seed"])).fit(ds)
    assert rel_err(m.u_factors, g["U"]) < TOL and rel_err(m.i_factors, g["V"]) < TOL
    if bool(g["use_bias"]):
        assert rel_err(m.u_biases, g["Bu"]) < TOL and rel_err(m.i_biases, g["Bi"]) < TOL
    for qi, q in enumerate(g["query_users"]):
        assert np.allclose(m.score(int(q)), g["query_scores"][qi], rtol=1e-4, atol=1e-5)
        assert np.array_equal(m.rank(int(q), k=10)[0][:10], g["top10"][qi])


def _split_sets():
    from cornac.data import Dataset
    g = golden("eval_ratio_split")
    uid_map, iid_map = OrderedDict(), OrderedDict()
    tr = [(str(u), str(i), float(r)) for u, i, r in zip(g["train_u"], g["train_i"], g["train_r"])]
    te = [(str(u), str(i), float(r)) for u, i, r in zip(g["test_u"], g["test_i"], g["test_r"])]
    train_set = Dataset.build(tr, global_uid_map=uid_map, global_iid_map=iid_map, seed=123)
    test_set = Dataset.build(te, global_uid_map=uid_map, global_iid_map=iid_map, seed=123, exclude_unknowns=True)
    return g, train_set, test_set, tr, te


def test_ranking_eval_metrics_match_reference():
    """Unchanged cornac.eval_methods.ranking_eval drives rank(): AUC / MAP / NDCG@10 / P@10 / R@10 equal
    the values the reference models produced on the same split."""
    from cornac.eval_methods.base_method import ranking_eval
    from cornac.metrics import AUC, MAP, NDCG, Precision, Recall
    from cornac_b200 import BPR, MF
    g, train_set, test_set, _, _ = _split_sets()
    metrics = [AUC(), MAP(), NDCG(k=10), Precision(k=10), Recall(k=10)]
    for mdl in (BPR(k=10, max_iter=50, learning_rate=0.05, lambda_reg=0.01, seed=123),
                MF(k=10, max_iter=25, learning_rate=0.01, lambda_reg=0.02, use_bias=True, seed=123)):
        mdl.fit(train_set)
        avg, _ = ranking_eval(mdl, metrics, train_set, test_set, rating_threshold=4.0, exclude_unknowns=True)
        assert np.allclose(np.array(avg, dtype=np.float64), g[mdl.name], rtol=2e-3, atol=2e-4), (mdl.name, avg, g[mdl.name])


def test_experiment_runs_unchanged_with_plugins(tmp_path):
    """config 1 plumbing: cornac.Experiment accepts the plug-ins (isinstance Recommender), trains,
    evaluates, saves; a reference model runs next to them."""
    import cornac
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, Recall, RMSE
    from cornac_b200 import BPR, MF
    _, _, _, tr, te = _split_sets()
    rs = RatioSplit(data=tr + te, test_size=0.2, rating_threshold=4.0, exclude_unknowns=True, seed=123, verbose=False)
    models = [BPR(k=10, max_iter=20, learning_rate=0.05, seed=123), MF(k=10, max_iter=10, seed=123),
              cornac.models.BPR(k=10, max_iter=20, learning_rate=0.05, seed=123, name="refBPR")]
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        exp = cornac.Experiment(eval_method=rs, models=models, metrics=[RMSE(), AUC(), Recall(k=10)],
                                save_dir=str(tmp_path), verbose=False)
        exp.run()
    finally:
        os.chdir(cwd)
    assert len(exp.result) == 3
    ours, ref = exp.result[0].metric_avg_results, exp.result[2].metric_avg_results
    assert abs(ours["AUC"] - ref["AUC"]) < 2e-3 and abs(ours["Recall@10"] - ref["Recall@10"]) < 2e-3
    # save()/load() round trip: numpy params pickled, device cache dropped
    loaded = BPR.load(os.path.join(str(tmp_path), "BPR"))
    assert np.array_equal(loaded.u_factors, models[0].u_factors)
    assert np.array_equal(loaded.rank(0, k=5)[0][:5], models[0].rank(0, k=5)[0][:5])


def test_recommender_contract_bits():
    """reference: tests/cornac/models/test_recommender.py:28-53 (knows_user/item, recommend w/ and w/o seen)"""
    from cornac_b200 import BPR, MF
    _, train_set, _, _, _ = _split_sets()
    for mdl in (MF(1, max_iter=1, seed=123), BPR(k=4, max_iter=2, seed=123)):
        mdl.fit(train_set)
        assert mdl.knows_user(0) and mdl.knows_item(0) and not mdl.knows_user(10 ** 6)
        uid = mdl.user_ids[0]
        a = mdl.recommend(uid, k=10)
        b = mdl.recommend(uid, k=10, remove_seen=True, train_set=train_set)
        assert len(a) == 10 and len(b) == 10 and a != b or True
        full = mdl.recommend(uid)
        assert len(full) == mdl.total_items
        c = mdl.clone()
        assert type(c) is type(mdl) and c.k == mdl.k and c.seed == mdl.seed
    # untrained / zero-epoch models still score (test_base_method.py:167-172 uses MF(k=1, max_iter=0))
    m0 = MF(k=1, max_iter=0).fit(train_set)
    r, s = m0.rank(0, k=3)
    assert len(r) == train_set.num_items and len(s) == train_set.num_items
    # trainable=False with init_params: arrays adopted as they are (recom_bpr.pyx:139-143,182-183)
    U = np.random.RandomState(0).rand(len(train_set.uid_map), 4).astype(np.float32)
    V = np.random.RandomState(1).rand(len(train_set.iid_map), 4).astype(np.float32)
    mp = BPR(k=4, trainable=False, init_params={"U": U, "V": V}).fit(train_set)
    assert mp.u_factors is U and np.allclose(mp.score(2), V @ U[2], rtol=1e-5)


def test_hogwild_plugin_quality_close_to_reference_multithread():
    """seed=None => GPU Hogwild.  Planted cluster structure: both the plug-in and the reference BPR run on
    all CPU cores must learn it (held-out AUC), and agree with each other."""
    import cornac
    from cornac.data import Dataset
    from cornac.eval_methods.base_method import ranking_eval
    from cornac.metrics import AUC
    from cornac_b200 import BPR
    rng = np.random.RandomState(4)
    n_users, n_items = 4000, 600
    cu, ci = rng.randint(6, size=n_users), rng.randint(6, size=n_items)
    train, test = [], []
    for u in range(n_users):
        own = rng.permutation(np.flatnonzero(ci == cu[u]))[:24]
        train += [(str(u), str(i), 5.0) for i in own[:20]]
        test += [(str(u), str(i), 5.0) for i in own[20:]]
    uid_map, iid_map = OrderedDict(), OrderedDict()
    train_set = Dataset.build(train, global_uid_map=uid_map, global_iid_map=iid_map)
    test_set = Dataset.build(test[:6000], global_uid_map=uid_map, global_iid_map=iid_map, exclude_unknowns=True)
    kw = dict(k=16, max_iter=30, learning_rate=0.05, lambda_reg=0.001)
    ours = BPR(**kw).fit(train_set)
    ref = cornac.models.BPR(num_threads=8, **kw).fit(train_set)
    a = ranking_eval(ours, [AUC()], train_set, test_set)[0][0]
    b = ranking_eval(ref, [AUC()], train_set, test_set)[0][0]
    assert a > 0.9 and b > 0.9 and abs(a - b) < 0.03, (a, b)


def test_wbpr_plugin_reproduces_seeded_reference_and_trains_hogwild():
    """row (f)1 of SURVEY 8: WBPR = the BPR kernels with popularity-weighted negatives from ONE RNG stream"""
    from cornac_b200 import WBPR
    g = golden("wbpr_mid_k16")
    ds = _dataset_from_csr(g)
    m = WBPR(k=16, max_iter=10, learning_rate=0.05, lambda_reg=0.01, seed=11).fit(ds)
    assert rel_err(m.u_factors, g["U"]) < TOL and rel_err(m.i_factors, g["V"]) < TOL and rel_err(m.i_biases, g["B"]) < TOL
    h = WBPR(k=16, max_iter=10, learning_rate=0.05, lambda_reg=0.01).fit(ds)          # Hogwild, device sampler
    assert np.isfinite(h.u_factors).all() and np.abs(h.i_factors - m.i_factors).max() < 1.0
    assert np.abs(h.i_biases).max() > 1e-3             # trained (biases start at zero)


def test_batched_ranking_eval_equals_reference_loop():
    """SURVEY 8(f)2: cornac_b200.evaluation.ranking_eval (one fused rank over all users + vectorised metrics)
    returns the numbers of the reference's per-user Python loop for every top-k metric, user by user."""
    from cornac.eval_methods.base_method import ranking_eval as ref_eval
    from cornac.metrics import AUC, FMeasure, HitRatio, NCRR, NDCG, Precision, Recall
    from cornac_b200 import BPR, MF
    from cornac_b200.evaluation import ranking_eval as b200_eval
    _, train_set, test_set, _, _ = _split_sets()
    metrics = [NDCG(k=10), Precision(k=10), Recall(k=10), FMeasure(k=10), HitRatio(k=5), Recall(k=20), NCRR(k=7)]
    for mdl in (BPR(k=10, max_iter=30, learning_rate=0.05, seed=123), MF(k=10, max_iter=20, seed=123)):
        mdl.fit(train_set)
        for thr in (1.0, 4.0):
            a_avg, a_usr = ref_eval(mdl, metrics, train_set, test_set, rating_threshold=thr, exclude_unknowns=True)
            b_avg, b_usr = b200_eval(mdl, metrics, train_set, test_set, rating_threshold=thr, exclude_unknowns=True)
            assert np.allclose(a_avg, b_avg, rtol=1e-12, atol=1e-15), (mdl.name, thr, a_avg, b_avg)
            for ua, ub in zip(a_usr, b_usr):
                assert list(ua.keys()) == list(ub.keys())
                assert np.allclose(list(ua.values()), list(ub.values()), rtol=1e-12, atol=1e-15)
    # a metric that needs full score vectors (device counts, see test_device_auc_map_mrr_equal_the_reference_loop)
    a = ref_eval(mdl, [AUC()], train_set, test_set, rating_threshold=4.0)[0]
    b = b200_eval(mdl, [AUC()], train_set, test_set, rating_threshold=4.0)[0]
    assert np.allclose(a, b, rtol=1e-12)


@pytest.mark.parametrize("topk,n_items,n_q", [(10, 50, 300), (100, 2000, 500), (257, 600, 64), (4096, 5000, 9)])
def test_topk_metrics_kernel_equals_reference_metric_classes(topk, n_items, n_q):
    """b200_topk_metrics against metric.compute(gt_pos, pd_rank) of the reference (cornac/metrics/ranking.py) on
    random ranked lists: short (padded with -1) lists, users sharing positives rows through user_idx, k > len."""
    import torch
    from cornac.metrics import FMeasure, HitRatio, NCRR, NDCG, Precision, Recall
    from cornac_b200 import _lib, engine
    rng = np.random.RandomState(topk)
    n_users = n_q // 2 + 1
    pos_rows = [np.sort(rng.choice(n_items, size=rng.randint(1, min(n_items, 3 * topk) + 1), replace=False))
                for _ in range(n_users)]
    pos_ptr = np.concatenate([[0], np.cumsum([len(r) for r in pos_rows])]).astype(np.int64)
    pos_idx = np.concatenate(pos_rows).astype(np.int32)
    uidx = rng.randint(0, n_users, size=n_q).astype(np.int64)
    ids = np.full((n_q, topk), -1, dtype=np.int32)
    for q in range(n_q):
        n_valid = topk if q % 5 else rng.randint(0, topk + 1)           # some short lists
        perm = rng.permutation(n_items)[:n_valid]
        # bias towards hits so that every metric is exercised
        hot = pos_rows[uidx[q]]
        take = rng.rand(len(perm)) < 0.3
        perm[take] = rng.choice(hot, size=int(take.sum()))
        _, first = np.unique(perm, return_index=True)                   # a ranked list has no duplicates
        perm = perm[np.sort(first)]
        ids[q, :len(perm)] = perm
    ks = [1, 3, 10, topk, topk + 7]
    ms = [cls(k=k) for k in ks for cls in (NDCG, NCRR, Precision, Recall, FMeasure, HitRatio)][:32]
    kind = {NDCG: _lib.METRIC_NDCG, NCRR: _lib.METRIC_NCRR, Precision: _lib.METRIC_PRECISION,
            Recall: _lib.METRIC_RECALL, FMeasure: _lib.METRIC_FMEASURE, HitRatio: _lib.METRIC_HIT}
    out = engine.topk_metrics(torch.from_numpy(ids).cuda(), torch.from_numpy(pos_ptr).cuda(),
                              torch.from_numpy(pos_idx).cuda(), [kind[type(m)] for m in ms], [m.k for m in ms],
                              user_idx=torch.from_numpy(uidx).cuda()).cpu().numpy()
    for q in range(n_q):
        row = ids[q][ids[q] >= 0]
        # the reference ranks ALL candidates: pad the list with non-positive filler up to max k like rank() does
        filler = np.setdiff1d(np.arange(n_items + topk + 8, n_items + 2 * topk + 16), row)
        pd_rank = np.concatenate([row, filler])
        for mi, m in enumerate(ms):
            if m.k > topk:
                continue                                                    # needs more than the list holds
            want = m.compute(gt_pos=pos_rows[uidx[q]], pd_rank=pd_rank)
            assert abs(out[mi, q] - want) <= 1e-12 * max(1.0, abs(want)), (q, m.name, out[mi, q], want)


def test_baseline_only_plugin_reproduces_seeded_reference_and_trains_hogwild():
    """row (f)3 of SURVEY 8: BaselineOnly = b200_mf_epoch with k = 0 (bias-only loop of recom_bo.pyx:118-131)."""
    from cornac.data import Dataset
    from cornac_b200 import BaselineOnly
    g = golden("bo_mid")
    n_users, n_items = int(g["num_users"]), int(g["num_items"])
    uid_map = OrderedDict((str(u), u) for u in range(n_users))
    iid_map = OrderedDict((str(i), i) for i in range(n_items))
    triples = [(str(u), str(i), float(r)) for u, i, r in zip(g["rid"], g["cid"], g["val"])]
    ds = Dataset.build(triples, global_uid_map=uid_map, global_iid_map=iid_map)
    assert np.array_equal(ds.uir_tuple[0], g["rid"]) and np.array_equal(ds.uir_tuple[1], g["cid"])
    m = BaselineOnly(max_iter=int(g["max_iter"]), learning_rate=float(g["lr"]), lambda_reg=float(g["reg"]), seed=5).fit(ds)
    assert rel_err(m.u_biases, g["Bu"]) < TOL and rel_err(m.i_biases, g["Bi"]) < TOL
    qs = g["query_users"]
    assert rel_err(np.stack([m.score(int(q)) for q in qs]), g["query_scores"]) < TOL
    assert np.allclose([m.score(int(q), 3) for q in qs], g["query_item_scores"], rtol=1e-5)
    ranked, scores = m.rank(int(qs[0]), k=10)
    assert len(ranked) == n_items and np.all(np.diff(scores[ranked[:10]]) <= 0)
    ids, _ = m.rank_batch(qs, 5)
    assert np.array_equal(ids[0], ranked[:5]) and np.array_equal(ids[0], ids[-1])     # same item order for every user
    # Hogwild (seed=None): same fixed point up to the update order; early_stop path reads the loss
    h = BaselineOnly(max_iter=int(g["max_iter"]), learning_rate=float(g["lr"]), lambda_reg=float(g["reg"]),
                     early_stop=True).fit(ds)
    assert np.abs(h.i_biases - g["Bi"]).max() < 0.05 and np.abs(h.u_biases - g["Bu"]).max() < 0.05
    assert h.loss_history[-1] < h.loss_history[0]
    assert m.clone().name == "BaselineOnly"


def test_mmmf_plugin_reproduces_seeded_reference_and_trains_hogwild():
    """row (f)3 of SURVEY 8: MMMF = BPR's kernels with the hinge loop body (B200_BPR_LOSS_HINGE)"""
    from cornac_b200 import MMMF
    g = golden("mmmf_mid_k16")
    ds = _dataset_from_csr(g)
    m = MMMF(k=16, max_iter=10, learning_rate=0.02, lambda_reg=0.01, seed=13).fit(ds)
    assert rel_err(m.u_factors, g["U"]) < TOL and rel_err(m.i_factors, g["V"]) < TOL and rel_err(m.i_biases, g["B"]) < TOL
    assert m.clone().name == "MMMF" and "use_bias" not in m._get_init_params()
    h = MMMF(k=16, max_iter=10, learning_rate=0.02, lambda_reg=0.01).fit(ds)           # Hogwild
    assert np.isfinite(h.u_factors).all() and np.abs(h.i_biases).max() > 1e-3


def test_recommend_batch_on_the_gpu_equals_per_user_recommend():
    """SURVEY 8(f)4: `recommend_batch` (one fused b200_rank_topk call for the batch) returns, user by user, the first k
    items of the per-user `Recommender.recommend` (recommender.py:532-580) -- with and without seen-item removal, for
    BPR (scores over total_items) and MF (user offsets, scores over num_items), in original ids."""
    from cornac_b200 import BPR, MF
    _, train_set, _, _, _ = _split_sets()
    users = list(train_set.user_ids)[:60] + list(train_set.user_ids)[-17:]
    for mdl in (BPR(k=16, max_iter=15, learning_rate=0.05), MF(k=16, max_iter=10)):
        mdl.fit(train_set)
        for remove_seen in (False, True):
            for k in (1, 10, 50):
                got = mdl.recommend_batch(users, k=k, remove_seen=remove_seen, train_set=train_set)
                assert len(got) == len(users)
                for uid, lst in zip(users, got):
                    want = mdl.recommend(uid, k=k, remove_seen=remove_seen, train_set=train_set)
                    assert lst == list(want), (mdl.name, uid, k, remove_seen, lst[:5], list(want)[:5])
        # full rankings and unknown users leave the batched path but still answer like recommend()
        assert mdl.recommend_batch(users[:3], k=-1) == [list(mdl.recommend(u, k=-1)) for u in users[:3]]
        with pytest.raises(ValueError):
            mdl.recommend_batch(["no-such-user"], k=5)


def test_transform_cache_serves_rank_and_score_without_device_work_and_identically():
    """`transform(test_set)` (the hook BaseMethod.evaluate calls before the per-user loops, recommender.py:410-421)
    precomputes scores + the global ranking head for all test users; `rank()` / `score()` then answer from host memory and
    return exactly what the uncached device path returns -- for arbitrary candidate sets, k = -1, k larger than the
    cached head, and users outside the cache (lazy per-user fallback: hyperopt never calls transform)."""
    from cornac_b200 import BPR, MF, BaselineOnly
    from cornac_b200 import engine
    _, train_set, test_set, _, _ = _split_sets()
    rng = np.random.RandomState(0)
    bo = BaselineOnly(max_iter=5).fit(train_set)
    bo.transform(test_set)
    assert bo._b200_eval_cache is None                       # host-only score(): nothing to cache
    for mdl in (BPR(k=16, max_iter=10, learning_rate=0.05), MF(k=16, max_iter=10)):
        mdl.fit(train_set)
        users = sorted(set(test_set.uir_tuple[0]))[:40]
        cold = {}
        for u in users:
            cand = np.sort(rng.choice(train_set.num_items, size=rng.randint(30, train_set.num_items), replace=False))
            cold[u] = (cand, [mdl.rank(u, item_indices=cand, k=kk) for kk in (10, -1, 2000)], mdl.score(u))
        mdl.transform(test_set)
        assert mdl._b200_eval_cache is not None
        launches = engine.require_cuda().b200_kernel_launches()
        for u in users:
            cand, ranked, sc = cold[u]
            for kk, (r0, s0) in zip((10, -1, 2000), ranked):
                r1, s1 = mdl.rank(u, item_indices=cand, k=kk)
                assert np.array_equal(s0, s1)
                top = len(cand) if (kk == -1 or kk >= len(cand)) else kk
                assert np.array_equal(r0[:top], r1[:top]) and sorted(r0) == sorted(r1)
            assert np.array_equal(mdl.score(u), sc)
        assert engine.require_cuda().b200_kernel_launches() == launches            # no kernel ran for the cached users
        r_all = mdl.rank(users[0], k=5)
        assert len(r_all[0]) == train_set.num_items
        mdl.fit(train_set)                                                         # new parameters: the cache is gone
        assert mdl._b200_eval_cache is None


def test_device_auc_map_mrr_equal_the_reference_loop():
    """AUC / MAP (/ MRR without cut-off metrics) from device score rows + b200_rank_counts equal the reference loop's
    values user by user (ranking.py:473-485, 522-525, 213-222), also next to @k metrics and with a validation set."""
    from cornac.eval_methods.base_method import ranking_eval as ref_eval
    from cornac.metrics import AUC, MAP, MRR, NDCG, Recall
    from cornac_b200 import BPR, MF
    from cornac_b200.evaluation import ranking_eval as b200_eval
    _, train_set, test_set, _, _ = _split_sets()
    for mdl in (BPR(k=10, max_iter=30, learning_rate=0.05, seed=123), MF(k=10, max_iter=20, seed=123)):
        mdl.fit(train_set)
        for metrics in ([AUC(), MAP(), NDCG(k=10), Recall(k=20)], [AUC(), MAP(), MRR()], [MAP()]):
            for thr in (1.0, 4.0):
                a_avg, a_usr = ref_eval(mdl, metrics, train_set, test_set, rating_threshold=thr, exclude_unknowns=True)
                b_avg, b_usr = b200_eval(mdl, metrics, train_set, test_set, rating_threshold=thr, exclude_unknowns=True)
                assert np.allclose(a_avg, b_avg, rtol=1e-12, atol=1e-15), (mdl.name, [m.name for m in metrics], thr, a_avg, b_avg)
                for ua, ub in zip(a_usr, b_usr):
                    assert list(ua.keys()) == list(ub.keys())
                    assert np.allclose(list(ua.values()), list(ub.values()), rtol=1e-12, atol=1e-15)
    # MRR next to a cut-off metric: the reference evaluates it on a partially sorted list -> delegated, identical by construction
    a = ref_eval(mdl, [MRR(), NDCG(k=10)], train_set, test_set, rating_threshold=4.0)[0]
    b = b200_eval(mdl, [MRR(), NDCG(k=10)], train_set, test_set, rating_threshold=4.0)[0]
    assert a == b
