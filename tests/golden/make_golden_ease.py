"""Generate the EASE golden vectors from the UNMODIFIED reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_ease.py

Each fit case runs cornac.models.EASE (cornac/models/ease/recom_ease.py) on synthetic, seeded ratings and stores the rating
matrix exactly as fit() sees it (train_set.matrix), the weight matrix B, a few score(u) rows and the reference's rank()
top-10 of the items each user has not rated.  The experiment case stores the metrics of an unchanged Experiment with the
settings of the reference's EASE example.  No reference file is copied.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import dataset_from, synth_uir  # noqa: E402  (puts oracle/_ref on sys.path and imports cornac)


def ease_case(name, uir, lamb, posB):
    from cornac.models import EASE
    ds = dataset_from(*uir)
    m = EASE(lamb=lamb, posB=posB, verbose=False).fit(ds)
    X = m.U.tocsr()
    users = np.unique(np.linspace(0, ds.num_users - 1, 8).astype(np.int64))
    rows = np.stack([np.asarray(m.score(int(u))).ravel() for u in users])
    top = np.full((len(users), 10), -1, dtype=np.int64)
    for q, u in enumerate(users):
        cand = np.setdiff1d(np.arange(ds.num_items), X[int(u)].indices)
        k = min(10, len(cand))
        if k:
            top[q, :k] = m.rank(int(u), item_indices=cand, k=k)[0][:k]
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        uir_u=np.asarray(uir[0], np.int64), uir_i=np.asarray(uir[1], np.int64), uir_r=np.asarray(uir[2], np.float64),
        X_indptr=X.indptr, X_indices=X.indices, X_data=X.data, num_users=ds.num_users, num_items=ds.num_items,
        lamb=float(lamb), posB=bool(posB), B=m.B, query_users=users, query_scores=rows, rank_top10=top)
    print(name, "ok", ds.num_users, ds.num_items, X.nnz, "max|B| = %r" % float(np.abs(m.B).max()))


def tie_uir():
    """Two disconnected groups: users 0-39 rate only items 0-19, users 40-79 only items 20-39.  P is block diagonal, so B
    and the scores of a user on the other group's items are exact zeros."""
    rng = np.random.RandomState(61)
    u, i = [], []
    for g in range(2):
        for a in range(40 * g, 40 * g + 40):
            items = rng.choice(20, size=6, replace=False) + 20 * g
            u += [a] * 6
            i += items.tolist()
    return np.array(u), np.array(i), rng.randint(1, 6, size=len(u)).astype(np.float64)


def experiment_case(name):
    """Both posB settings through RatioSplit + an unchanged Experiment (examples/ease_movielens.py's settings)."""
    import cornac
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import NDCG, Recall
    u, i, r = synth_uir(400, 300, 12000, 71)
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, seed=123, rating_threshold=0.8, verbose=False)
    metrics = [Recall(k=20), Recall(k=50), NDCG(k=100)]
    models = [cornac.models.EASE(lamb=500, name="pos", posB=True, verbose=False),
              cornac.models.EASE(lamb=500, name="all", posB=False, verbose=False)]
    exp = cornac.Experiment(eval_method=rs, models=models, metrics=metrics, user_based=True, save_dir=None, verbose=False)
    exp.run()
    res = {r.model_name: r.metric_avg_results for r in exp.result}
    names = [m.name for m in metrics]
    np.savez_compressed(os.path.join(HERE, name + ".npz"), uir_u=u, uir_i=i, uir_r=r, metric_names=np.array(names),
                        pos=np.array([res["pos"][n] for n in names]), all=np.array([res["all"][n] for n in names]))
    print(name, res)


def ease_cases():
    base = synth_uir(300, 200, 6000, 51)
    ease_case("ease_l500_pos", base, 500, True)
    ease_case("ease_l500_all", base, 500, False)
    ease_case("ease_l1_pos", base, 1, True)
    u, i, r = synth_uir(250, 150, 4000, 52)
    ease_case("ease_l001_all", (u, i, r * 0.7), 0.01, False)             # non-dyadic ratings, weakest regularisation
    one = np.random.RandomState(53).randint(1, 6, 40).astype(np.float64)
    ease_case("ease_n1", (np.arange(40), np.zeros(40, np.int64), one), 500, True)           # a single item
    ease_case("ease_n130", synth_uir(220, 130, 3000, 54), 20, False)   # not a multiple of the block size
    ease_case("ease_tie", tie_uir(), 500, False)
    experiment_case("ease_experiment")


if __name__ == "__main__":
    ease_cases()
