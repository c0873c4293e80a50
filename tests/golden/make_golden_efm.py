"""Generate the EFM golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_efm.py

Each fit case builds a train set from seeded synthetic ratings and sentiment reviews (aspect, opinion, polarity tuples)
through a real SentimentModality, and stores: the inputs; A, X and Y as the reference's _build_matrices builds them; the
initial factors the reference draws (a fit with max_iter=0); the factors after a few values of max_iter, each fit from
those initial factors; and EFM.rank of some users after the last fit.  The exact-dot case starts from dyadic factors
(multiples of 1/16 in (0, 1]) so that every prediction is exact in any summation order, with non-dyadic ratings and
non-unit lambdas, and max_iter=1.  The experiment case stores a RatioSplit with sentiment and the metrics an unchanged
Experiment reports.  No reference file is copied.
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

FACTORS = ("U1", "U2", "V", "H1", "H2")
HYPER = ("num_explicit_factors", "num_latent_factors", "num_most_cared_aspects", "rating_scale", "alpha", "lambda_x",
         "lambda_y", "lambda_u", "lambda_h", "lambda_v", "use_item_aspect_popularity")


def synth_reviews(u, i, n_aspects, seed, frac=0.8, max_tuples=4, skip_users=(), skip_items=(), repeat=0, ghost=False):
    """Reviews (user, item, tuples) for a seeded fraction of the rated pairs: 1..max_tuples tuples over aspects [0,
    n_aspects) with polarities in {-1, 1} and some non-integer ones.  `repeat` pairs get a second, different review (the
    modality keeps the last); with `ghost` the first review of a repeated pair names aspect n_aspects, which no kept
    review mentions."""
    rng = np.random.RandomState(seed)
    reviews = []
    for a, b in zip(u, i):
        if a in skip_users or b in skip_items or rng.rand() > frac:
            continue
        n = rng.randint(1, max_tuples + 1)
        tups = [(int(rng.randint(n_aspects)), int(rng.randint(20)), float(rng.choice([-1.0, 1.0, 0.5, -0.25, 2.0])))
                for _ in range(n)]
        reviews.append((int(a), int(b), tups))
    for t in range(min(repeat, len(reviews))):
        a, b, tups = reviews[t]
        first = [(n_aspects, 0, 1.0)] if ghost else tups
        reviews[t] = (a, b, first)
        reviews.append((a, b, [(int(rng.randint(n_aspects)), 1, -1.0), (int(rng.randint(n_aspects)), 2, 1.0)]))
    return reviews


def pack_reviews(reviews):
    return dict(rev_u=np.array([r[0] for r in reviews], np.int64), rev_i=np.array([r[1] for r in reviews], np.int64),
                rev_n=np.array([len(r[2]) for r in reviews], np.int64),
                tup_a=np.array([t[0] for r in reviews for t in r[2]], np.int64),
                tup_o=np.array([t[1] for r in reviews for t in r[2]], np.int64),
                tup_p=np.array([t[2] for r in reviews for t in r[2]], np.float64))


def unpack_reviews(g):
    """The SentimentModality data of a fixture: [(user id, item id, [(aspect, opinion, polarity), ...]), ...]."""
    out, t = [], 0
    for a, b, n in zip(g["rev_u"], g["rev_i"], g["rev_n"]):
        tups = [("a%d" % g["tup_a"][t + s], "o%d" % g["tup_o"][t + s], float(g["tup_p"][t + s])) for s in range(n)]
        out.append((str(a), str(b), tups))
        t += n
    return out


def train_set(g):
    """A train set of a fixture's ratings with its SentimentModality built on it, as BaseMethod builds it."""
    from cornac.data import Dataset, SentimentModality
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    ts = Dataset.from_uir(data, seed=1)
    md = SentimentModality(data=unpack_reviews(g))
    md.build(uid_map=ts.uid_map, iid_map=ts.iid_map, dok_matrix=ts.dok_matrix)
    ts.add_modalities(sentiment=md)
    return ts


def csr_fields(prefix, M):
    return {prefix + "_indptr": M.indptr.astype(np.int64), prefix + "_indices": M.indices.astype(np.int64),
            prefix + "_data": M.data.astype(np.float32)}


def fit_case(name, n_users, n_items, nnz, n_aspects, seed, max_iters=(1, 3, 10), dyadic=False, rank_users=8,
             zero_rating=False, tie=False, review_kw=None, **hyper):
    import cornac
    u, i, r = synth_uir(n_users, n_items, nnz, seed)
    r = r.astype(np.float64)
    if dyadic:                                              # non-dyadic ratings: the chains still round
        r = r * 0.7 + 0.13
    if zero_rating:
        r[3] = 0.0
    out = dict(uir_u=u, uir_i=i, uir_r=r, **pack_reviews(synth_reviews(u, i, n_aspects, seed + 1, **(review_kw or {}))))
    ts = train_set(out)
    base = dict(num_explicit_factors=40, num_latent_factors=60, num_most_cared_aspects=15, rating_scale=5.0,
                alpha=0.85, lambda_x=1, lambda_y=1, lambda_u=0.01, lambda_h=0.01, lambda_v=0.01,
                use_item_aspect_popularity=True)
    base.update(hyper)
    for k in HYPER:
        out[k] = np.array(base[k])
    m0 = cornac.models.EFM(max_iter=0, seed=seed, **base).fit(ts)
    init = {f: np.asarray(getattr(m0, f), dtype=np.float32).copy() for f in FACTORS}
    if dyadic:
        rng = np.random.RandomState(seed + 2)
        init = {f: (rng.randint(1, 17, size=x.shape) / 16.0).astype(np.float32) for f, x in init.items()}
    if tie:                                 # two equal V rows above the others: an exact tie in X_ at the N-th place
        init["V"][0] = init["V"][1] = 1.0
    A, X, Y = m0._build_matrices(ts)
    out.update(**csr_fields("A", A), **csr_fields("X", X), **csr_fields("Y", Y))
    out["num_users"], out["num_items"], out["num_aspects"] = ts.num_users, ts.num_items, m0.num_aspects
    for f in FACTORS:
        out[f + "0"] = init[f]
    out["max_iters"] = np.array(max_iters)
    for mi in max_iters:
        m = cornac.models.EFM(max_iter=mi, init_params={f: init[f].copy() for f in FACTORS}, **base).fit(ts)
        for f in FACTORS:
            out["%s_%d" % (f, mi)] = np.asarray(getattr(m, f))
    users = np.unique(np.linspace(0, ts.num_users - 1, rank_users).astype(np.int64))
    out["rank_users"] = users
    out["rank_scores"] = np.stack([m.rank(int(q))[1] for q in users]).astype(np.float64)
    out["score_rows"] = np.stack([m.score(int(q)) for q in users]).astype(np.float64)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, {k: np.shape(v) for k, v in out.items() if k in ("A_data", "X_data", "Y_data")}, "aspects",
          m0.num_aspects)


def experiment_case(name):
    """EFM with examples/efm_example.py's metrics through a RatioSplit with sentiment + an unchanged Experiment."""
    import cornac
    from cornac.data import SentimentModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, NDCG, RMSE, Recall
    u, i, r = synth_uir(150, 120, 3000, 71)
    out = dict(uir_u=u, uir_i=i, uir_r=r.astype(np.float64), **pack_reviews(synth_reviews(u, i, 25, 72)))
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123,
                    sentiment=SentimentModality(data=unpack_reviews(out)))
    metrics = [RMSE(), NDCG(k=50), AUC(), Recall(k=10)]
    names = [m.name for m in metrics]
    out["metric_names"] = np.array(names)
    model = cornac.models.EFM(num_explicit_factors=8, num_latent_factors=12, num_most_cared_aspects=5, max_iter=20,
                              seed=123)
    with contextlib.redirect_stdout(io.StringIO()):
        exp = cornac.Experiment(eval_method=rs, models=[model], metrics=metrics, user_based=True, verbose=False,
                                save_dir=tempfile.mkdtemp())
        exp.run()
    res = exp.result[0].metric_avg_results
    out["metrics"] = np.array([res[m] for m in names])
    print(name, res)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)


CASES = dict(
    efm_default=dict(n_users=120, n_items=90, nnz=1500, n_aspects=30, seed=11),
    efm_odd=dict(n_users=70, n_items=60, nnz=800, n_aspects=23, seed=21, num_explicit_factors=7,
                 num_latent_factors=37, num_most_cared_aspects=4),
    efm_nopop=dict(n_users=70, n_items=60, nnz=800, n_aspects=18, seed=31, num_explicit_factors=12,
                   num_latent_factors=9, use_item_aspect_popularity=False),
    efm_lambdas=dict(n_users=70, n_items=60, nnz=800, n_aspects=18, seed=41, num_explicit_factors=9,
                     num_latent_factors=33, lambda_x=0.7, lambda_y=1.9, lambda_u=0.3, lambda_h=0.07, lambda_v=0.45,
                     rating_scale=4.0, alpha=0.6),
    efm_sparse=dict(n_users=60, n_items=50, nnz=500, n_aspects=15, seed=51, num_explicit_factors=6,
                    num_latent_factors=5, zero_rating=True,
                    review_kw=dict(frac=0.6, skip_users=(0, 1, 2, 3), skip_items=(0, 1, 2), repeat=3, ghost=True)),
    efm_bign=dict(n_users=50, n_items=40, nnz=400, n_aspects=10, seed=61, num_explicit_factors=5,
                  num_latent_factors=4, num_most_cared_aspects=25),
    efm_tie=dict(n_users=50, n_items=40, nnz=400, n_aspects=10, seed=81, num_explicit_factors=5, num_latent_factors=4,
                 num_most_cared_aspects=1, max_iters=(0,), tie=True),
    efm_exact=dict(n_users=80, n_items=70, nnz=1200, n_aspects=20, seed=91, max_iters=(1,), dyadic=True,
                   num_explicit_factors=33, num_latent_factors=40, lambda_x=0.7, lambda_y=1.3, lambda_u=0.03,
                   lambda_h=0.02, lambda_v=0.05),
)

if __name__ == "__main__":
    for name, kw in CASES.items():
        fit_case(name, **kw)
    experiment_case("efm_experiment")
