"""Generate the committed golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Run in the build container (needs oracle/_ref, i.e.
`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden.py

The reference's own tests hold no golden values for trained BPR/MF parameters or
ranked lists (SURVEY.md 8c), so these fixtures are produced by running the reference
itself: cornac.models.BPR / MF with a seed (=> single thread => deterministic,
cornac/models/bpr/recom_bpr.pyx:132-133, cornac/models/mf/recom_mf.py:124-125),
their score()/rank(), and cornac.eval_methods.ranking_eval.  Inputs are synthetic
(numpy, seeded here) so no reference file is copied.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

import cornac  # noqa: E402
from cornac.data import Dataset  # noqa: E402
from cornac.eval_methods import RatioSplit  # noqa: E402
from cornac.eval_methods.base_method import ranking_eval  # noqa: E402
from cornac.metrics import AUC, MAP, NDCG, Precision, Recall  # noqa: E402
from cornac.models import BPR, MF, MMMF, WBPR  # noqa: E402


def synth_uir(n_users, n_items, nnz, seed):
    """Unique (u, i) pairs with Zipf-ish item popularity, ratings in {1..5}."""
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** 0.8
    p /= p.sum()
    pairs = set()
    while len(pairs) < nnz:
        u = rng.randint(n_users, size=nnz)
        i = rng.choice(n_items, size=nnz, p=p)
        for a, b in zip(u, i):
            if len(pairs) < nnz:
                pairs.add((int(a), int(b)))
    pairs = sorted(pairs)
    rng.shuffle(pairs)
    u = np.array([a for a, _ in pairs], dtype=np.int64)
    i = np.array([b for _, b in pairs], dtype=np.int64)
    r = rng.randint(1, 6, size=nnz).astype(np.float64)
    return u, i, r


def dataset_from(u, i, r):
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    return Dataset.from_uir(data, seed=None)


def bpr_case(name, n_users, n_items, nnz, k, max_iter, lr, reg, use_bias, seed, dseed):
    u, i, r = synth_uir(n_users, n_items, nnz, dseed)
    ds = dataset_from(u, i, r)
    m = BPR(k=k, max_iter=max_iter, learning_rate=lr, lambda_reg=reg, use_bias=use_bias, seed=seed).fit(ds)
    X = ds.matrix
    qs = np.arange(0, ds.num_users, max(1, ds.num_users // 8))[:8]
    scores = np.stack([m.score(int(q)) for q in qs])
    excl_ptr, excl_idx, top_ids = [0], [], []
    for q in qs:
        seen = np.sort(X.indices[X.indptr[q]:X.indptr[q + 1]])
        cand = np.setdiff1d(np.arange(ds.num_items), seen)
        ranked, _ = m.rank(int(q), item_indices=cand, k=10)
        top_ids.append(ranked[:10])
        excl_idx.extend(seen.tolist())
        excl_ptr.append(len(excl_idx))
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        indptr=X.indptr.astype(np.int32), indices=X.indices.astype(np.int32), data=X.data.astype(np.float32),
        num_users=ds.num_users, num_items=ds.num_items, total_users=m.total_users, total_items=m.total_items,
        k=k, max_iter=max_iter, lr=lr, reg=reg, use_bias=use_bias, seed=seed,
        U=m.u_factors, V=m.i_factors, B=m.i_biases,
        query_users=qs.astype(np.int64), query_scores=scores.astype(np.float32),
        excl_indptr=np.array(excl_ptr, np.int32), excl_indices=np.array(excl_idx, np.int32),
        top10=np.stack(top_ids).astype(np.int64),
    )
    print(name, "ok", m.u_factors.shape, m.i_factors.shape)


def wbpr_case(name, n_users, n_items, nnz, k, max_iter, lr, reg, seed, dseed):
    u, i, r = synth_uir(n_users, n_items, nnz, dseed)
    ds = dataset_from(u, i, r)
    m = WBPR(k=k, max_iter=max_iter, learning_rate=lr, lambda_reg=reg, use_bias=True, seed=seed).fit(ds)
    X = ds.matrix
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        indptr=X.indptr.astype(np.int32), indices=X.indices.astype(np.int32), data=X.data.astype(np.float32),
        num_users=ds.num_users, num_items=ds.num_items, total_users=m.total_users, total_items=m.total_items,
        k=k, max_iter=max_iter, lr=lr, reg=reg, use_bias=True, seed=seed,
        U=m.u_factors, V=m.i_factors, B=m.i_biases)
    print(name, "ok")


def mmmf_case(name, n_users, n_items, nnz, k, max_iter, lr, reg, seed, dseed):
    u, i, r = synth_uir(n_users, n_items, nnz, dseed)
    ds = dataset_from(u, i, r)
    m = MMMF(k=k, max_iter=max_iter, learning_rate=lr, lambda_reg=reg, seed=seed).fit(ds)
    X = ds.matrix
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        indptr=X.indptr.astype(np.int32), indices=X.indices.astype(np.int32), data=X.data.astype(np.float32),
        num_users=ds.num_users, num_items=ds.num_items, total_users=m.total_users, total_items=m.total_items,
        k=k, max_iter=max_iter, lr=lr, reg=reg, use_bias=True, seed=seed,
        U=m.u_factors, V=m.i_factors, B=m.i_biases)
    print(name, "ok")


def mf_case(name, n_users, n_items, nnz, k, max_iter, lr, reg, use_bias, early_stop, seed, dseed):
    u, i, r = synth_uir(n_users, n_items, nnz, dseed)
    ds = dataset_from(u, i, r)
    m = MF(k=k, max_iter=max_iter, learning_rate=lr, lambda_reg=reg, use_bias=use_bias,
           early_stop=early_stop, seed=seed).fit(ds)
    rid, cid, val = ds.uir_tuple
    qs = np.arange(0, ds.num_users, max(1, ds.num_users // 8))[:8]
    scores = np.stack([m.score(int(q)) for q in qs])
    top = np.stack([m.rank(int(q), k=10)[0][:10] for q in qs])
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        rid=rid.astype(np.int64), cid=cid.astype(np.int64), val=val.astype(np.float32),
        num_users=ds.num_users, num_items=ds.num_items, global_mean=ds.global_mean,
        k=k, max_iter=max_iter, lr=lr, reg=reg, use_bias=use_bias, early_stop=early_stop, seed=seed,
        U=m.u_factors, V=m.i_factors, Bu=m.u_biases, Bi=m.i_biases, mu=np.float32(m.global_mean),
        query_users=qs.astype(np.int64), query_scores=scores.astype(np.float32), top10=top.astype(np.int64),
    )
    print(name, "ok")


def bo_case(name, n_users, n_items, nnz, max_iter, lr, reg, seed, dseed):
    """BaselineOnly (baseline_only/recom_bo.pyx): biases after a seeded (single-thread) fit + scores."""
    from cornac.models import BaselineOnly
    u, i, r = synth_uir(n_users, n_items, nnz, dseed)
    ds = dataset_from(u, i, r)
    m = BaselineOnly(max_iter=max_iter, learning_rate=lr, lambda_reg=reg, seed=seed).fit(ds)
    rid, cid, val = ds.uir_tuple
    qs = np.arange(0, ds.num_users, max(1, ds.num_users // 8))[:8]
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        rid=rid.astype(np.int64), cid=cid.astype(np.int64), val=val.astype(np.float32),
        num_users=ds.num_users, num_items=ds.num_items, global_mean=ds.global_mean,
        max_iter=max_iter, lr=lr, reg=reg, seed=seed, Bu=m.u_biases, Bi=m.i_biases,
        query_users=qs.astype(np.int64), query_scores=np.stack([m.score(int(q)) for q in qs]).astype(np.float32),
        query_item_scores=np.array([m.score(int(q), 3) for q in qs], dtype=np.float64),
    )
    print(name, "ok")


def eval_case(name, n_users, n_items, nnz, dseed):
    """BPR + MF through RatioSplit + ranking_eval: golden metric values and the
    split itself (so the GPU box can rebuild identical train/test sets without
    depending on RatioSplit's RNG)."""
    u, i, r = synth_uir(n_users, n_items, nnz, dseed)
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    rs = RatioSplit(data=data, test_size=0.2, rating_threshold=4.0, exclude_unknowns=True, seed=123, verbose=False)
    metrics = [AUC(), MAP(), NDCG(k=10), Precision(k=10), Recall(k=10)]
    out = {}
    for mdl in (BPR(k=10, max_iter=50, learning_rate=0.05, lambda_reg=0.01, seed=123),
                MF(k=10, max_iter=25, learning_rate=0.01, lambda_reg=0.02, use_bias=True, seed=123)):
        mdl.fit(rs.train_set)
        avg, _ = ranking_eval(mdl, metrics, rs.train_set, rs.test_set, rating_threshold=4.0,
                              exclude_unknowns=True)
        out[mdl.name] = np.array(avg, dtype=np.float64)
        print(name, mdl.name, dict(zip([m.name for m in metrics], avg)))
    tr, te = rs.train_set, rs.test_set
    inv_u = {v: k for k, v in tr.uid_map.items()}
    inv_i = {v: k for k, v in tr.iid_map.items()}
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        train_u=np.array([int(inv_u[x]) for x in tr.uir_tuple[0]]), train_i=np.array([int(inv_i[x]) for x in tr.uir_tuple[1]]),
        train_r=tr.uir_tuple[2],
        test_u=np.array([int(inv_u[x]) for x in te.uir_tuple[0]]), test_i=np.array([int(inv_i[x]) for x in te.uir_tuple[1]]),
        test_r=te.uir_tuple[2],
        metric_names=np.array([m.name for m in metrics]), BPR=out["BPR"], MF=out["MF"],
    )


def vebpr_case(name, n_users, n_items, nnz, n_view, k, max_iter, lr, reg, alpha, seed, dseed):
    """VEBPR (cornac/models/bpr/recom_vebpr.pyx) on a PurchaseViewDataset: ~30 % of the users have no viewed item
    (the BPR fall-back branch of the loop, :246-275)."""
    from cornac.data import PurchaseViewDataset
    from cornac.models.bpr.recom_vebpr import VEBPR
    u, i, r = synth_uir(n_users, n_items, nnz, dseed)
    ds = dataset_from(u, i, r)
    rng = np.random.RandomState(dseed + 100)
    viewers = rng.permutation(n_users)[: int(0.7 * n_users)]
    views = sorted(set(zip(rng.choice(viewers, size=n_view).tolist(), rng.randint(n_items, size=n_view).tolist())))
    pv = PurchaseViewDataset.attach_view(ds, [(str(a), str(b), 1.0) for a, b in views])
    m = VEBPR(k=k, max_iter=max_iter, learning_rate=lr, lambda_reg=reg, alpha=alpha, seed=seed).fit(pv)
    X, W = pv.matrix, pv.view_matrix
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        indptr=X.indptr.astype(np.int32), indices=X.indices.astype(np.int32), data=X.data.astype(np.float32),
        view_indptr=W.indptr.astype(np.int32), view_indices=W.indices.astype(np.int32),
        num_users=pv.num_users, num_items=pv.num_items, total_users=m.total_users, total_items=m.total_items,
        k=k, max_iter=max_iter, lr=lr, reg=reg, alpha=alpha, seed=seed, U=m.u_factor, V=m.i_factor)
    print(name, "ok")


def sbpr_case(name, n_users, n_items, nnz, k, max_iter, lr, lbd_u, lbd_v, lbd_b, use_bias, seed, dseed):
    """SBPR (cornac/models/sbpr/recom_sbpr.pyx).  The reference's SBPR.fit cannot run as written (it calls
    self._prepare_data() / self._prepare_social_data() without the train_set argument, :168-169 -> TypeError), so the
    fixture drives the pieces fit() names, in its order: Recommender.fit, _init, _prepare_data, _prepare_social_data,
    the two RNGVectors (:173-174) and max_iter calls of the compiled _fit_sgd (:193-300)."""
    from cornac.data import GraphModality
    from cornac.models import Recommender
    from cornac.models.bpr.recom_bpr import RNGVector
    from cornac.models.sbpr.recom_sbpr import SBPR
    from scipy.sparse import csr_matrix
    u, i, r = synth_uir(n_users, n_items, nnz, dseed)
    ds = dataset_from(u, i, r)
    rng = np.random.RandomState(dseed + 200)
    edges = set()
    for a in range(n_users):
        if rng.rand() < 0.7:                      # ~30 % of the users have no friend: the plain-BPR branch (:247-265)
            for b in rng.randint(n_users, size=rng.randint(1, 5)):
                if a != int(b):
                    edges.add((a, int(b)))
    # k_id = social_item_ids[social_indptr[u] + ...] is read even for users WITHOUT social items (:231-233); for such users
    # at the END of the user range that index is one past the array (undefined behaviour in the reference).  The LAST train
    # user therefore gets friends, so that every index the kernel reads exists and the fixture is reproducible.
    last = max(ds.uid_map.values())
    inv = {v: int(k_) for k_, v in ds.uid_map.items()}
    edges.update((inv[last], inv[b]) for b in range(3))
    gm = GraphModality(data=[(str(a), str(b), 1.0) for a, b in sorted(edges)])
    gm.build(id_map=ds.uid_map)
    ds.add_modalities(user_graph=gm)
    m = SBPR(k=k, max_iter=max_iter, learning_rate=lr, lambda_u=lbd_u, lambda_v=lbd_v, lambda_b=lbd_b, use_bias=use_bias, seed=seed)
    try:
        m.fit(ds)
        raise SystemExit("the reference's SBPR.fit ran: regenerate this fixture through fit()")
    except TypeError:
        pass
    m = SBPR(k=k, max_iter=max_iter, learning_rate=lr, lambda_u=lbd_u, lambda_v=lbd_v, lambda_b=lbd_b, use_bias=use_bias, seed=seed)
    Recommender.fit(m, ds)
    m._init()
    X, _, user_ids = m._prepare_data(ds)
    s_ids, s_cnts, s_ptr = m._prepare_social_data(ds)
    assert s_ptr[-1] > s_ptr[-2], "the last user must have social items (see above)"
    rp = RNGVector(1, len(user_ids) - 1, m.rng.randint(2 ** 31))
    rn = RNGVector(1, ds.num_items - 1, m.rng.randint(2 ** 31))
    skipped = [m._fit_sgd(rp, rn, 1, user_ids, X.indices, X.indptr, s_ids, s_cnts, s_ptr, m.u_factors, m.i_factors, m.i_biases)
               for _ in range(max_iter)]
    train_users = set(ds.uir_tuple[0])
    rid, cid, val = ds.user_graph.get_train_triplet(train_users, train_users)
    Y = csr_matrix((val, (rid, cid)), shape=(ds.num_users, ds.num_users))
    Y.sort_indices()
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        indptr=X.indptr.astype(np.int32), indices=X.indices.astype(np.int32), data=X.data.astype(np.float32),
        graph_indptr=Y.indptr.astype(np.int32), graph_indices=Y.indices.astype(np.int32),
        social_item_ids=s_ids.astype(np.int32), social_item_counts=s_cnts.astype(np.int32), social_indptr=s_ptr.astype(np.int32),
        num_users=ds.num_users, num_items=ds.num_items, total_users=m.total_users, total_items=m.total_items,
        k=k, max_iter=max_iter, lr=lr, lbd_u=lbd_u, lbd_v=lbd_v, lbd_b=lbd_b, use_bias=use_bias, seed=seed,
        skipped=np.array(skipped, np.int64), U=m.u_factors, V=m.i_factors, B=m.i_biases)
    print(name, "ok")


if __name__ == "__main__":
    print("cornac", cornac.__version__)
    if len(sys.argv) > 1 and sys.argv[1] == "sbpr":          # regenerate one fixture
        sbpr_case("sbpr_mid_k16", 150, 100, 2000, k=16, max_iter=8, lr=0.05, lbd_u=0.02, lbd_v=0.03, lbd_b=0.04, use_bias=True, seed=19, dseed=10)
        sys.exit(0)
    bpr_case("bpr_small_k10", 60, 40, 600, k=10, max_iter=30, lr=0.05, reg=0.01, use_bias=True, seed=123, dseed=1)
    bpr_case("bpr_mid_k32", 300, 200, 5700, k=32, max_iter=5, lr=0.05, reg=0.01, use_bias=True, seed=7, dseed=2)
    bpr_case("bpr_nobias_k16", 120, 90, 1500, k=16, max_iter=8, lr=0.02, reg=0.001, use_bias=False, seed=42, dseed=3)
    mf_case("mf_small_k10", 60, 40, 600, k=10, max_iter=25, lr=0.01, reg=0.02, use_bias=True, early_stop=False, seed=123, dseed=1)
    mf_case("mf_mid_k32", 300, 200, 5700, k=32, max_iter=5, lr=0.01, reg=0.02, use_bias=True, early_stop=False, seed=7, dseed=2)
    mf_case("mf_nobias_k16", 120, 90, 1500, k=16, max_iter=8, lr=0.02, reg=0.01, use_bias=False, early_stop=False, seed=42, dseed=3)
    eval_case("eval_ratio_split", 200, 150, 6000, dseed=5)
    wbpr_case("wbpr_mid_k16", 150, 100, 2000, k=16, max_iter=10, lr=0.05, reg=0.01, seed=11, dseed=6)
    bo_case("bo_mid", 150, 100, 2000, max_iter=15, lr=0.01, reg=0.02, seed=5, dseed=8)
    mmmf_case("mmmf_mid_k16", 150, 100, 2000, k=16, max_iter=10, lr=0.02, reg=0.01, seed=13, dseed=7)
    vebpr_case("vebpr_mid_k16", 150, 100, 2000, n_view=1500, k=16, max_iter=8, lr=0.05, reg=0.01, alpha=0.3, seed=17, dseed=9)
    sbpr_case("sbpr_mid_k16", 150, 100, 2000, k=16, max_iter=8, lr=0.05, lbd_u=0.02, lbd_v=0.03, lbd_b=0.04, use_bias=True, seed=19, dseed=10)
