"""Generate the MTER golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_mter.py

Each fit case builds a train set from seeded synthetic ratings and sentiment reviews through a real SentimentModality
and stores: the inputs; the arrays `fit` hands to `_fit_mter` (the reference's `_build_data` dicts flattened as `fit`
flattens them); the parameters the reference's `_init` draws (a fit with max_iter=0); the five stream seeds and the
draws of every iteration, from a plain-Python mt19937 + boost uniform_int_distribution written here; and the parameters
after a few values of max_iter, each fit from the initial parameters through init_params with the case's seed.  The
experiment case stores a RatioSplit with sentiment and the metrics an unchanged Experiment reports.  No reference file
is copied.
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

PARAMS = ("U", "I", "A", "O", "G1", "G2", "G3")
HYPER = ("rating_scale", "n_user_factors", "n_item_factors", "n_aspect_factors", "n_opinion_factors", "n_bpr_samples",
         "n_element_samples", "lambda_reg", "lambda_bpr", "lr")
DATA = ("X", "X_uids", "X_iids", "X_aids", "YU", "YU_uids", "YU_aids", "YU_oids", "YI", "YI_iids", "YI_aids", "YI_oids")


class MT19937:
    """std::mt19937 (boost::random::mt19937) in plain Python, with boost's uniform_int_distribution(0, hi)."""

    def __init__(self, seed):
        self.mt = [0] * 624
        self.mt[0] = seed & 0xFFFFFFFF
        for i in range(1, 624):
            self.mt[i] = (1812433253 * (self.mt[i - 1] ^ (self.mt[i - 1] >> 30)) + i) & 0xFFFFFFFF
        self.idx = 624

    def next(self):
        if self.idx >= 624:
            mt = self.mt
            for i in range(624):
                y = (mt[i] & 0x80000000) | (mt[(i + 1) % 624] & 0x7FFFFFFF)
                mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ (0x9908B0DF if y & 1 else 0)
            self.idx = 0
        y = self.mt[self.idx]
        self.idx += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        y ^= y >> 18
        return y

    def draw(self, hi):
        if hi == 0:
            return 0
        bucket = 0xFFFFFFFF // (hi + 1)
        if 0xFFFFFFFF % (hi + 1) == hi:
            bucket += 1
        while True:
            v = self.next() // bucket
            if v <= hi:
                return v


def stream_seeds(seed):
    """The five RNGVector engine seeds of a fit whose _init draws nothing (every parameter given)."""
    rng = np.random.RandomState(seed)
    return [int(np.random.RandomState(int(rng.randint(2 ** 31))).randint(2 ** 31)) for _ in range(5)]


def flatten(model, ts):
    """The arrays `fit` builds from `_build_data` (recom_mter.pyx:326-371)."""
    rating_matrix, rating_dict, uia, uao, iao = model._build_data(ts)
    out = {}
    for prefix, d, names in (("X", uia, ("uids", "iids", "aids")), ("YU", uao, ("uids", "aids", "oids")),
                             ("YI", iao, ("iids", "aids", "oids"))):
        keys = list(d.keys())
        out[prefix] = np.array([d[k] for k in keys], dtype=np.float32)
        for c, n in enumerate(names):
            out["%s_%s" % (prefix, n)] = np.array([k[c] for k in keys], dtype=np.int32)
    out["indptr"] = rating_matrix.indptr.astype(np.int32)
    out["indices"] = rating_matrix.indices.astype(np.int32)
    return out


def fit_case(name, n_users, n_items, nnz, n_aspects, seed, max_iters=(1, 3), dyadic=False, repeat_pairs=0, **hyper):
    import cornac
    u, i, r = synth_uir(n_users, n_items, nnz, seed)
    r = r.astype(np.float64)
    out = dict(uir_u=u, uir_i=i, uir_r=r, **pack_reviews(synth_reviews(u, i, n_aspects, seed + 1)))
    ts = train_set(out)
    if repeat_pairs:               # a train set holding some (user, item) pairs twice, with another rating
        uu, ii, rr = (np.asarray(x) for x in ts.uir_tuple)
        rr2 = rr[:repeat_pairs] % 5 + 1
        ts.uir_tuple = (np.concatenate([uu, uu[:repeat_pairs]]), np.concatenate([ii, ii[:repeat_pairs]]),
                        np.concatenate([rr, rr2]))
        out["repeat_pairs"] = np.array(repeat_pairs)
    out["ts_u"], out["ts_i"], out["ts_r"] = (np.asarray(x) for x in ts.uir_tuple)
    base = dict(rating_scale=5.0, n_user_factors=15, n_item_factors=15, n_aspect_factors=12, n_opinion_factors=12,
                n_bpr_samples=1000, n_element_samples=50, lambda_reg=0.1, lambda_bpr=10, lr=0.1)
    base.update(hyper)
    for k in HYPER:
        out[k] = np.array(base[k])
    m0 = cornac.models.MTER(max_iter=0, seed=seed, **base).fit(ts)
    init = {p: np.asarray(getattr(m0, p), dtype=np.float32).copy() for p in PARAMS}
    for p in PARAMS:
        out["draw0_" + p] = init[p]                # what the reference's _init draws with this seed
    if dyadic:                                     # quarters: every prediction of the first iteration is exact
        rng = np.random.RandomState(seed + 2)
        init = {p: (rng.randint(1, 5, size=x.shape) / 4.0).astype(np.float32) for p, x in init.items()}
    out.update(flatten(m0, ts))
    out["num_users"], out["num_items"] = ts.num_users, ts.num_items
    out["num_aspects"], out["num_opinions"] = m0.num_aspects, m0.num_opinions
    for p in PARAMS:
        out[p + "0"] = init[p]
    out["seed"] = np.array(seed)
    seeds = stream_seeds(seed)
    out["stream_seeds"] = np.array(seeds, dtype=np.int64)
    n_it = max(max_iters)
    his = [len(out["X"]) - 1, len(out["YU"]) - 1, len(out["YI"]) - 1, len(out["indices"]) - 1, ts.num_items - 1]
    ns = [base["n_element_samples"]] * 3 + [base["n_bpr_samples"]] * 2
    for tag, s, hi, n in zip(("uia", "uao", "iao", "pos", "neg"), seeds, his, ns):
        g = MT19937(s)
        out["draws_" + tag] = np.array([g.draw(hi) for _ in range(n_it * n)], dtype=np.int64)
    out["max_iters"] = np.array(max_iters)
    for mi in max_iters:
        m = cornac.models.MTER(max_iter=mi, seed=seed, init_params={p: init[p].copy() for p in PARAMS}, **base).fit(ts)
        for p in PARAMS:
            out["%s_%d" % (p, mi)] = np.asarray(getattr(m, p))
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, {k: len(out[k]) for k in ("X", "YU", "YI", "indices")})


def experiment_case(name):
    """MTER with examples/mter_example.py's model settings (fewer iterations) through a RatioSplit with sentiment and
    an unchanged Experiment."""
    import cornac
    from cornac.data import SentimentModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import NDCG, RMSE
    u, i, r = synth_uir(150, 120, 3000, 171)
    out = dict(uir_u=u, uir_i=i, uir_r=r.astype(np.float64), **pack_reviews(synth_reviews(u, i, 25, 172)))
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    rs = RatioSplit(data=data, test_size=0.1, exclude_unknowns=True, verbose=False, seed=123,
                    sentiment=SentimentModality(data=unpack_reviews(out)))
    metrics = [RMSE(), NDCG(k=10), NDCG(k=20), NDCG(k=50)]
    names = [m.name for m in metrics]
    out["metric_names"] = np.array(names)
    out["max_iter"] = np.array(200)
    model = cornac.models.MTER(n_user_factors=8, n_item_factors=8, n_aspect_factors=8, n_opinion_factors=8,
                               n_bpr_samples=1000, n_element_samples=50, lambda_reg=0.1, lambda_bpr=5, max_iter=200,
                               lr=0.5, seed=123)
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
    mter_default=dict(n_users=60, n_items=40, nnz=900, n_aspects=20, seed=11),
    mter_odd=dict(n_users=50, n_items=30, nnz=600, n_aspects=9, seed=21, n_user_factors=3, n_item_factors=5,
                  n_aspect_factors=2, n_opinion_factors=4, n_element_samples=37, n_bpr_samples=211,
                  lambda_reg=0.07, lambda_bpr=3.5, lr=0.23, rating_scale=4.0, max_iters=(1, 4, 10)),
    mter_ties=dict(n_users=30, n_items=12, nnz=250, n_aspects=7, seed=31, n_user_factors=4, n_item_factors=6,
                   n_aspect_factors=3, n_opinion_factors=5, n_element_samples=20, n_bpr_samples=300,
                   repeat_pairs=25, max_iters=(1, 5)),
    mter_exact=dict(n_users=40, n_items=30, nnz=500, n_aspects=10, seed=41, n_user_factors=6, n_item_factors=7,
                    n_aspect_factors=5, n_opinion_factors=3, max_iters=(1,), dyadic=True),
)

if __name__ == "__main__":
    only = sys.argv[1:]
    for name, kw in CASES.items():
        if not only or name in only:
            fit_case(name, **kw)
    if not only or "mter_experiment" in only:
        experiment_case("mter_experiment")
