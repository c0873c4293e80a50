"""Generate the UserKNN / ItemKNN golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_knn.py

Each case fits cornac.models.UserKNN / ItemKNN (cornac/models/knn/recom_knn.py) on synthetic, seeded ratings and stores
the inputs, the weight matrix fit() passes to compute_similarity, the similarity before and after the amplify map,
mean_arr, score rows, score(u, i) values and rank() top-10 lists.  No reference file is copied.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import dataset_from, synth_uir  # noqa: E402  (puts oracle/_ref on sys.path and imports cornac)


def tie_uir(n_users, n_bases, n_base_ratings, seed):
    """Every base item appears as four item columns: two copies of its ratings (in {1, 2}) and two copies doubled.
    Cosine on the raw ratings is scale-free and the doubling is exact, so the four columns have bitwise equal
    similarities to every item while their mean-centred values differ: tie groups of four with two distinct values."""
    rng = np.random.RandomState(seed)
    pairs = sorted(set(zip(rng.randint(n_users, size=n_base_ratings).tolist(), rng.randint(n_bases, size=n_base_ratings).tolist())))
    u, i, r = [], [], []
    for a, b in pairs:
        x = float(rng.randint(1, 3))
        for copy, f in enumerate((1.0, 1.0, 2.0, 2.0)):
            u.append(a)
            i.append(4 * b + copy)
            r.append(x * f)
    return np.array(u), np.array(i), np.array(r)


def knn_case(name, cls, uir, k, n_query=24, **kw):
    """UserKNN / ItemKNN (cornac/models/knn/recom_knn.py) on the compiled reference.  compute_similarity is wrapped to
    record the weight matrix fit() passes it and the similarity it returns (before the amplify map)."""
    from cornac.models.knn import recom_knn
    seen = {}
    real = recom_knn.compute_similarity

    def spy(data_mat, **a):
        seen["weight"] = data_mat.tocsr().copy()
        seen["raw"] = real(data_mat, **a)
        return seen["raw"].copy()

    recom_knn.compute_similarity = spy
    try:
        ds = dataset_from(*uir)
        m = cls(k=k, seed=1, verbose=False, **kw).fit(ds)
    finally:
        recom_knn.compute_similarity = real
    X, W, R, S = ds.matrix, seen["weight"], seen["raw"], m.sim_mat
    # with amplify == 1 the returned similarity is sim_mat itself; it is stored once
    raw = {} if kw.get("amplify", 1.0) == 1.0 else dict(
        raw_indptr=R.indptr.astype(np.int32), raw_indices=R.indices.astype(np.int32), raw_data=R.data)
    qs = np.linspace(0, ds.num_users - 1, n_query).astype(np.int64)
    rows = np.stack([m.score(int(q)) for q in qs])
    rng = np.random.RandomState(0)
    pairs = np.stack([rng.choice(qs, 12), rng.randint(ds.num_items, size=12)], axis=1)
    single = np.array([m.score(int(a), int(b)) for a, b in pairs])
    top_ids, top_scores = [], []
    for q in qs:
        ranked, sc = m.rank(int(q), k=10)
        top_ids.append(ranked[:10])
        top_scores.append(sc[ranked[:10]])
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        uir_u=np.asarray(uir[0], np.int64), uir_i=np.asarray(uir[1], np.int64), uir_r=np.asarray(uir[2], np.float64),
        indptr=X.indptr.astype(np.int32), indices=X.indices.astype(np.int32), data=X.data.astype(np.float64),
        num_users=ds.num_users, num_items=ds.num_items, model=cls.__name__, k=k,
        similarity=kw.get("similarity", "cosine"), mean_centered=kw.get("mean_centered", False),
        weighting=str(kw.get("weighting", None)), amplify=kw.get("amplify", 1.0),
        w_indptr=W.indptr.astype(np.int32), w_indices=W.indices.astype(np.int32), w_data=W.data, w_cols=W.shape[1],
        sim_indptr=S.indptr.astype(np.int32), sim_indices=S.indices.astype(np.int32), sim_data=S.data,
        mean_arr=m.mean_arr, query_users=qs, query_scores=rows,
        single_pairs=pairs.astype(np.int64), single_scores=single,
        top10=np.stack(top_ids).astype(np.int64), top10_scores=np.stack(top_scores),
        **raw)
    print(name, "ok", S.shape, S.nnz)


def knn_cases():
    from cornac.models import ItemKNN, UserKNN
    exp = synth_uir(220, 200, 4000, 21)
    knn_case("knn_user_cosine_k20", UserKNN, exp, k=20)
    knn_case("knn_user_pearson_idf_k10", UserKNN, synth_uir(150, 200, 2500, 23), k=10, similarity="pearson", weighting="idf",
             amplify=2.0)
    knn_case("knn_item_cosine_bm25_k20", ItemKNN, exp, k=20, mean_centered=True, weighting="bm25")
    knn_case("knn_item_pearson_k5", ItemKNN, exp, k=5, similarity="pearson", amplify=0.5)
    u, i, _ = exp
    imp = (u, i, np.ones(len(u)))
    knn_case("knn_item_implicit_k20", ItemKNN, imp, k=20)
    knn_case("knn_user_implicit_k20", UserKNN, imp, k=20)
    tie = tie_uir(120, 40, 700, 22)
    knn_case("knn_item_tie_k3", ItemKNN, tie, k=3)
    knn_case("knn_user_tie_k3", UserKNN, tie, k=3)


if __name__ == "__main__":
    knn_cases()
