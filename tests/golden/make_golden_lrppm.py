"""Generate the LRPPM golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_lrppm.py

Each fit case builds a train set from seeded synthetic ratings and sentiment reviews through a real SentimentModality
and stores: the inputs; the arrays `fit` hands to `_fit` and the dicts `_build_data` returns (as key / value arrays);
the item x aspect quality CSR; the parameters the reference's `_init` draws (a fit with max_iter=0); the three stream
seeds and the draws of every iteration (mt19937 + boost's uniform_int_distribution, written in make_golden_mter); and
the parameters after a few values of max_iter, each fit from the initial parameters through init_params with the
case's seed, with the number of `_fit` calls the fit made (a counting wrapper on the class).  The reference's `rank`
reads `csr_matrix.A`, which scipy >= 1.14 no longer has: this script installs the read the reference meant,
`.toarray()`, as a property for its own run.  The experiment case stores a RatioSplit with sentiment and the metrics an
unchanged Experiment reports.  No reference file is copied.
"""
import contextlib
import io
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import synth_uir  # noqa: E402  (puts oracle/_ref on sys.path and imports cornac)
from make_golden_efm import pack_reviews, synth_reviews, train_set, unpack_reviews  # noqa: E402
from make_golden_mter import MT19937  # noqa: E402

import scipy.sparse as sp  # noqa: E402

if not hasattr(sp.csr_matrix, "A"):
    sp.csr_matrix.A = property(lambda self: self.toarray())

PARAMS = ("U", "I", "UA", "IA")
HYPER = ("rating_scale", "n_factors", "ld", "reg", "alpha", "num_top_aspects", "n_ranking_samples", "n_samples", "lr")


def stream_seeds(seed):
    rng = np.random.RandomState(seed)
    return [int(np.random.RandomState(int(rng.randint(2 ** 31))).randint(2 ** 31)) for _ in range(3)]


def fit_calls(model, ts):
    """Fit with a counting wrapper on the class's `_fit`; returns (model, number of _fit calls, stdout)."""
    cls = type(model)
    orig = cls._fit
    calls = [0]

    def counted(self, *a, **kw):
        calls[0] += 1
        return orig(self, *a, **kw)
    cls._fit = counted
    buf = io.StringIO()
    try:
        with contextlib.redirect_stdout(buf):
            model.fit(ts)
    finally:
        cls._fit = orig
    return model, calls[0], buf.getvalue()


def fit_case(name, n_users, n_items, nnz, n_aspects, seed, max_iters=(1, 3), init=None, drop_ratings=0,
             review_kw=None, rank_users=6, **hyper):
    import cornac
    u, i, r = synth_uir(n_users, n_items, nnz, seed)
    out = dict(uir_u=u, uir_i=i, uir_r=r.astype(np.float64),
               **pack_reviews(synth_reviews(u, i, n_aspects, seed + 1, **(review_kw or {}))))
    ts = train_set(out)
    if drop_ratings:               # review pairs without a training rating: their rating reads 0 in the loop
        uu, ii, rr = (np.asarray(x) for x in ts.uir_tuple)
        ts.uir_tuple = (uu[drop_ratings:], ii[drop_ratings:], rr[drop_ratings:])
        out["drop_ratings"] = np.array(drop_ratings)
    out["ts_u"], out["ts_i"], out["ts_r"] = (np.asarray(x) for x in ts.uir_tuple)
    base = dict(rating_scale=5, n_factors=8, ld=1, reg=0.01, alpha=1, num_top_aspects=99999, n_ranking_samples=1000,
                n_samples=200, lr=0.1)
    base.update(hyper)
    for key in HYPER:
        out[key] = np.array(base[key])
    m0, _, _ = fit_calls(cornac.models.LRPPM(max_iter=0, seed=seed, **base), ts)
    params0 = {p: np.asarray(getattr(m0, p), dtype=np.float32).copy() for p in PARAMS}
    for p in PARAMS:
        out["draw0_" + p] = params0[p]
    if init is not None:
        init(params0, np.random.RandomState(seed + 2))
    out["num_users"], out["num_items"], out["num_aspects"] = ts.num_users, ts.num_items, m0.num_aspects
    rating_dict, uia, uia_dict, quality, counts = m0._build_data(ts)
    keys = list(uia.keys())
    out["ref_X_uids"], out["ref_X_iids"], out["ref_X_aids"] = (np.array([t[c] for t in keys], np.int64) for c in range(3))
    out["ref_X_values"] = np.array([uia[t] for t in keys], np.float64)
    out["ref_X_l_ui"] = np.array([1.0 / (counts[(t[0], t[1])] * (m0.num_aspects - counts[(t[0], t[1])])) for t in keys],
                                 dtype=np.float32)
    out["ref_rating_keys"], out["ref_rating_values"] = rating_dict.to_arrays()
    out["ref_aspect_keys"], out["ref_aspect_values"] = uia_dict.to_arrays()
    Q = quality.tocsr()
    out["Q_indptr"], out["Q_indices"], out["Q_data"] = Q.indptr.astype(np.int64), Q.indices.astype(np.int64), Q.data
    for p in PARAMS:
        out[p + "0"] = params0[p]
    out["seed"] = np.array(seed)
    seeds = stream_seeds(seed)
    out["stream_seeds"] = np.array(seeds, dtype=np.int64)
    out["max_iters"] = np.array(max_iters)
    runs = []
    for mi in max_iters:
        m, calls, text = fit_calls(cornac.models.LRPPM(max_iter=mi, seed=seed,
                                                       init_params={p: params0[p].copy() for p in PARAMS}, **base), ts)
        runs.append(calls)
        for p in PARAMS:
            out["%s_%d" % (p, mi)] = np.asarray(getattr(m, p))
        out["calls_%d" % mi] = np.array(calls)
        out["converged_%d" % mi] = np.array("Stop training because model converged!" in text)
    n_it = max(runs)
    n_trip = len(keys)
    his = [len(out["ts_r"]) - 1, n_trip - 1, m0.num_aspects - 1]
    ns = [base["n_samples"], base["n_ranking_samples"], base["n_ranking_samples"]]
    for tag, s, hi, n in zip(("pos", "pos_uia", "neg_uia"), seeds, his, ns):
        g = MT19937(s)
        out["draws_" + tag] = np.array([g.draw(hi) for _ in range(n_it * n)], dtype=np.int64)
    # the reference's rank of some users after the last fit
    m.num_top_aspects = base["num_top_aspects"]
    users = np.arange(min(rank_users, ts.num_users))
    out["rank_users"] = users
    out["rank_scores"] = np.stack([m.rank(int(uu))[1] for uu in users])
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, dict(triples=n_trip, ratings=len(out["ts_r"]), calls=runs))


def experiment_case(name):
    """LRPPM with examples/lrppm_example.py's model settings (fewer iterations) through a RatioSplit with sentiment and
    an unchanged Experiment."""
    import cornac
    from cornac.data import SentimentModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, NDCG, RMSE
    u, i, r = synth_uir(150, 120, 3000, 181)
    out = dict(uir_u=u, uir_i=i, uir_r=r.astype(np.float64), **pack_reviews(synth_reviews(u, i, 25, 182)))
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123,
                    sentiment=SentimentModality(data=unpack_reviews(out)))
    metrics = [RMSE(), AUC(), NDCG(k=50)]
    names = [mm.name for mm in metrics]
    out["metric_names"] = np.array(names)
    out["max_iter"] = np.array(100)
    model = cornac.models.LRPPM(max_iter=100, num_top_aspects=99999, seed=123)
    with contextlib.redirect_stdout(io.StringIO()):
        exp = cornac.Experiment(eval_method=rs, models=[model], metrics=metrics, user_based=True, verbose=False,
                                save_dir=tempfile.mkdtemp())
        exp.run()
    res = exp.result[0].metric_avg_results
    out["metrics"] = np.array([res[mm] for mm in names])
    for p in PARAMS:
        out["fit_" + p] = np.asarray(getattr(model, p))
    print(name, res)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)


def _nan_neg(params, rng):
    params["U"][1, 2] = np.nan
    params["I"][0, 1] = -0.5
    params["UA"][3, 0] = -0.0
    params["IA"][2, 4] = np.nan


CASES = dict(
    lrppm_default=dict(n_users=60, n_items=40, nnz=900, n_aspects=20, seed=11, max_iters=(1, 3)),
    lrppm_k1=dict(n_users=40, n_items=30, nnz=500, n_aspects=12, seed=21, n_factors=1, n_samples=57,
                  n_ranking_samples=301, lr=0.05, reg=0.03, ld=0.7, max_iters=(1, 4)),
    lrppm_k3=dict(n_users=40, n_items=30, nnz=500, n_aspects=12, seed=22, n_factors=3, n_samples=57,
                  n_ranking_samples=301, lr=0.05, reg=0.03, ld=0.7, max_iters=(1, 4)),
    lrppm_k5=dict(n_users=50, n_items=30, nnz=600, n_aspects=9, seed=23, n_factors=5, n_samples=80,
                  n_ranking_samples=400, lr=0.07, max_iters=(1, 4), num_top_aspects=4, alpha=0.6),
    lrppm_collide=dict(n_users=300, n_items=67, nnz=6000, n_aspects=20, seed=31, max_iters=(1, 2),
                       review_kw=dict(frac=1.0, max_tuples=8)),
    lrppm_norating=dict(n_users=40, n_items=30, nnz=500, n_aspects=10, seed=41, drop_ratings=60, max_iters=(1, 3)),
    lrppm_nan=dict(n_users=40, n_items=30, nnz=500, n_aspects=10, seed=51, init=_nan_neg, max_iters=(1, 3)),
    lrppm_converge=dict(n_users=30, n_items=20, nnz=300, n_aspects=8, seed=61, lr=3.0, max_iters=(1, 60)),
)

if __name__ == "__main__":
    only = sys.argv[1:]
    for case, kw in CASES.items():
        if not only or case in only:
            fit_case(case, **kw)
    if not only or "lrppm_experiment" in only:
        experiment_case("lrppm_experiment")
