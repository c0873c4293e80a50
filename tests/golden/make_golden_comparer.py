"""Generate the ComparERSub golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_comparer.py

Each fit case builds a train set with timestamps from seeded synthetic ratings and sentiment reviews through a real
SentimentModality and stores: the inputs; the arrays `fit` hands to `_fit_mter` (the reference's `_build_data` output
flattened as `fit` flattens it, the f64 quality values of its user-item-aspect dict, its item quality matrix Y and the
pair list); the parameters the reference's `_init` draws (a fit with max_iter=0); the six stream seeds and the draws of
every iteration; and the parameters after a few values of max_iter, each fit from the initial parameters through
init_params with the case's seed.  The experiment case stores a RatioSplit with sentiment and timestamps and the
metrics an unchanged Experiment reports.  No reference file is copied.
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
from make_golden_efm import pack_reviews, synth_reviews, unpack_reviews  # noqa: E402
from make_golden_mter import MT19937, PARAMS  # noqa: E402

HYPER = ("rating_scale", "n_user_factors", "n_item_factors", "n_aspect_factors", "n_opinion_factors", "n_pair_samples",
         "n_bpr_samples", "n_element_samples", "n_top_aspects", "alpha", "min_user_freq", "min_pair_freq",
         "min_common_freq", "use_item_aspect_popularity", "lambda_reg", "lambda_bpr", "lambda_d", "lr")
PAIRS = ("p_user_indices", "earlier_indices", "later_indices", "aspect_indices", "pair_freq")
BASE = dict(rating_scale=5.0, n_user_factors=8, n_item_factors=8, n_aspect_factors=8, n_opinion_factors=8,
            n_pair_samples=1000, n_bpr_samples=1000, n_element_samples=50, n_top_aspects=100, alpha=0.5,
            min_user_freq=2, min_pair_freq=1, min_common_freq=1, use_item_aspect_popularity=True, enum_window=None,
            lambda_reg=0.1, lambda_bpr=10, lambda_d=0.01, lr=0.5)


def stream_seeds(seed):
    """The six RNGVector engine seeds of a fit whose _init draws nothing (every parameter given)."""
    rng = np.random.RandomState(seed)
    return [int(np.random.RandomState(int(rng.randint(2 ** 31))).randint(2 ** 31)) for _ in range(6)]


def train_set(g):
    """A train set of a fixture's ratings and timestamps with its SentimentModality built on it, as BaseMethod builds
    it; then the stored train tuple and timestamps (which may repeat an item in a history) replace the built ones."""
    from cornac.data import Dataset, SentimentModality
    data = [(str(a), str(b), float(c), int(t)) for a, b, c, t in zip(g["uir_u"], g["uir_i"], g["uir_r"], g["uir_t"])]
    ts = Dataset.from_uirt(data, seed=1)
    md = SentimentModality(data=unpack_reviews(g))
    md.build(uid_map=ts.uid_map, iid_map=ts.iid_map, dok_matrix=ts.dok_matrix)
    ts.add_modalities(sentiment=md)
    if "ts_t" in g:
        ts.uir_tuple = (np.asarray(g["ts_u"]), np.asarray(g["ts_i"]), np.asarray(g["ts_r"]))
        ts.timestamps = np.asarray(g["ts_t"])
    return ts


def flatten(model, ts):
    """The arrays `fit` builds from `_build_data` (recom_comparer_sub.pyx:376-422), with the f64 values of X."""
    rating_matrix, rating_dict, uia, uao, iao, pu, pe, pl, pa, pf = model._build_data(ts)
    out = {}
    for prefix, d, names in (("X", uia, ("uids", "iids", "aids")), ("YU", uao, ("uids", "aids", "oids")),
                             ("YI", iao, ("iids", "aids", "oids"))):
        keys = list(d.keys())
        out[prefix] = np.array([d[k] for k in keys], dtype=np.float32)
        for c, n in enumerate(names):
            out["%s_%s" % (prefix, n)] = np.array([k[c] for k in keys], dtype=np.int32)
    out["X64"] = np.array([uia[k] for k in uia.keys()], dtype=np.float64)
    out["indptr"] = rating_matrix.indptr.astype(np.int32)
    out["indices"] = rating_matrix.indices.astype(np.int32)
    for name, x in zip(PAIRS, (pu, pe, pl, pa, pf)):
        out[name] = np.asarray(x)
    out["Y"] = model._build_item_quality_matrix(ts, ts.sentiment).toarray().astype(np.float32)
    return out


def fit_case(name, n_users, n_items, nnz, n_aspects, seed, max_iters=(1, 3), dyadic=False, repeat_items=0,
             tie_times=False, same_pair=False, **hyper):
    import cornac
    u, i, r = synth_uir(n_users, n_items, nnz, seed)
    r = r.astype(np.float64)
    rng = np.random.RandomState(seed + 3)
    t = rng.randint(0, 40 if tie_times else 10 ** 6, size=len(u)).astype(np.int64)
    out = dict(uir_u=u, uir_i=i, uir_r=r, uir_t=t, **pack_reviews(synth_reviews(u, i, n_aspects, seed + 1)))
    ts = train_set(out)
    if repeat_items:               # histories that hold some items twice, at other times, with another rating
        uu, ii, rr = (np.asarray(x) for x in ts.uir_tuple)
        tt = np.asarray(ts.timestamps)
        ts.uir_tuple = (np.concatenate([uu, uu[:repeat_items]]), np.concatenate([ii, ii[:repeat_items]]),
                        np.concatenate([rr, rr[:repeat_items] % 5 + 1]))
        ts.timestamps = np.concatenate([tt, tt[:repeat_items] + rng.randint(-5, 6, size=repeat_items)])
    out["ts_u"], out["ts_i"], out["ts_r"] = (np.asarray(x) for x in ts.uir_tuple)
    out["ts_t"] = np.asarray(ts.timestamps)
    base = dict(BASE)
    base.update(hyper)
    for k in HYPER:
        out[k] = np.array(base[k])
    out["enum_window"] = np.array(-1 if base["enum_window"] is None else base["enum_window"])
    m0 = cornac.models.ComparERSub(max_iter=0, seed=seed, **base).fit(ts)
    init = {p: np.asarray(getattr(m0, p), dtype=np.float32).copy() for p in PARAMS}
    for p in PARAMS:
        out["draw0_" + p] = init[p]
    if dyadic:
        rng2 = np.random.RandomState(seed + 2)
        init = {p: (rng2.randint(1, 5, size=x.shape) / 4.0).astype(np.float32) for p, x in init.items()}
    out.update(flatten(m0, ts))
    out["num_users"], out["num_items"] = ts.num_users, ts.num_items
    out["num_aspects"], out["num_opinions"] = m0.num_aspects, m0.num_opinions
    for p in PARAMS:
        out[p + "0"] = init[p]
    out["seed"] = np.array(seed)
    seeds = stream_seeds(seed)
    out["stream_seeds"] = np.array(seeds, dtype=np.int64)
    n_it = max(max_iters)
    his = [len(out["X"]) - 1, len(out["YU"]) - 1, len(out["YI"]) - 1, len(out["p_user_indices"]) - 1,
           len(out["indices"]) - 1, ts.num_items - 1]
    ns = [base["n_element_samples"]] * 3 + [base["n_pair_samples"]] + [base["n_bpr_samples"]] * 2
    for tag, s, hi, n in zip(("uia", "uao", "iao", "pair", "pos", "neg"), seeds, his, ns):
        g = MT19937(s)
        out["draws_" + tag] = np.array([g.draw(hi) for _ in range(n_it * n)], dtype=np.int64)
    out["max_iters"] = np.array(max_iters)
    for mi in max_iters:
        m = cornac.models.ComparERSub(max_iter=mi, seed=seed, init_params={p: init[p].copy() for p in PARAMS},
                                      **base).fit(ts)
        for p in PARAMS:
            out["%s_%d" % (p, mi)] = np.asarray(getattr(m, p))
    # the reference's rank of a few users after the last fit (its f32 einsums)
    users = np.arange(min(6, ts.num_users))
    out["rank_users"] = users
    out["rank_scores"] = np.stack([np.asarray(m.rank(int(x))[1], dtype=np.float64) for x in users])
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, {k: len(out[k]) for k in ("X", "YU", "YI", "indices", "p_user_indices")})


def experiment_case(name):
    """ComparERSub through a RatioSplit with sentiment and timestamps and an unchanged Experiment."""
    import cornac
    from cornac.data import SentimentModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import NDCG, RMSE
    u, i, r = synth_uir(150, 120, 3000, 181)
    t = np.random.RandomState(183).randint(0, 10 ** 6, size=len(u)).astype(np.int64)
    out = dict(uir_u=u, uir_i=i, uir_r=r.astype(np.float64), uir_t=t, **pack_reviews(synth_reviews(u, i, 25, 182)))
    data = [(str(a), str(b), float(c), int(d)) for a, b, c, d in zip(u, i, r, t)]
    rs = RatioSplit(data=data, fmt="UIRT", test_size=0.1, exclude_unknowns=True, verbose=False, seed=123,
                    sentiment=SentimentModality(data=unpack_reviews(out)))
    metrics = [RMSE(), NDCG(k=10), NDCG(k=20), NDCG(k=50)]
    names = [m.name for m in metrics]
    out["metric_names"] = np.array(names)
    out["max_iter"] = np.array(200)
    model = cornac.models.ComparERSub(n_top_aspects=10, max_iter=200, seed=123)
    with contextlib.redirect_stdout(io.StringIO()):
        exp = cornac.Experiment(eval_method=rs, models=[model], metrics=metrics, user_based=True, verbose=False,
                                save_dir=tempfile.mkdtemp())
        exp.run()
    res = exp.result[0].metric_avg_results
    out["metrics"] = np.array([res[m] for m in names])
    for p in PARAMS:
        out["fit_" + p] = np.asarray(getattr(model, p))
    print(name, res)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)


CASES = dict(
    comparer_sub_default=dict(n_users=40, n_items=30, nnz=600, n_aspects=20, seed=51),
    comparer_sub_window=dict(n_users=40, n_items=30, nnz=700, n_aspects=12, seed=61, enum_window=4, min_user_freq=5,
                             min_common_freq=3, n_pair_samples=300, n_top_aspects=5, n_user_factors=3,
                             n_item_factors=5, n_aspect_factors=2, n_opinion_factors=4, n_element_samples=37,
                             n_bpr_samples=211, lambda_d=0.3, lr=0.23, max_iters=(1, 4, 10)),
    comparer_sub_ties=dict(n_users=25, n_items=14, nnz=250, n_aspects=7, seed=71, repeat_items=30, tie_times=True,
                           n_user_factors=4, n_item_factors=6, n_aspect_factors=3, n_opinion_factors=5,
                           n_pair_samples=400, use_item_aspect_popularity=False, lambda_d=1.5, max_iters=(1, 5)),
    comparer_sub_nonpos=dict(n_users=30, n_items=20, nnz=400, n_aspects=9, seed=81, rating_scale=-0.5,
                             n_top_aspects=3, n_pair_samples=200, lambda_d=0.7, max_iters=(1, 3)),
    comparer_sub_exact=dict(n_users=30, n_items=25, nnz=400, n_aspects=10, seed=91, n_user_factors=6,
                            n_item_factors=7, n_aspect_factors=5, n_opinion_factors=3, alpha=0.0, lambda_d=0.5,
                            max_iters=(1,), dyadic=True),
    comparer_sub_nopair=dict(n_users=30, n_items=20, nnz=350, n_aspects=8, seed=101, n_pair_samples=0,
                             n_top_aspects=50, max_iters=(1, 3)),
)

if __name__ == "__main__":
    only = sys.argv[1:]
    for name, kw in CASES.items():
        if not only or name in only:
            fit_case(name, **kw)
    if not only or "comparer_sub_experiment" in only:
        experiment_case("comparer_sub_experiment")
