"""Generate the NMF golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_nmf.py

Each fit case runs cornac.models.NMF (cornac/models/nmf/recom_nmf.pyx) on synthetic, seeded ratings and stores the CSR
ratings fit() hands to _fit_sgd, the initial and trained factors and biases, the hyperparameters and a few single-item
scores.  The experiment case stores the metrics an unchanged Experiment on a RatioSplit gives, with the example's
settings (use_bias=False, rating and ranking metrics) and with use_bias=True (rating metrics only: the reference's
score(u) cannot rank a biased model).  No reference file is copied.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import dataset_from, synth_uir  # noqa: E402  (puts oracle/_ref on sys.path and imports cornac)


def nmf_case(name, uir, init=None, **kw):
    from cornac.models import NMF
    seen = {}

    class Spy(NMF):
        def _fit_sgd(self, rid, cid, val, user_counts, item_counts, U, V, Bu, Bi):
            seen.update(U0=np.array(U, copy=True), V0=np.array(V, copy=True), Bu0=np.array(Bu, copy=True),
                        Bi0=np.array(Bi, copy=True), mu=np.float32(self.global_mean))
            return NMF._fit_sgd(self, rid, cid, val, user_counts, item_counts, U, V, Bu, Bi)

    ds = dataset_from(*uir)
    params = None if init is None else init(ds.num_users, ds.num_items, kw.get("k", 15))
    m = Spy(init_params=params, **kw).fit(ds)
    X = ds.matrix
    rng = np.random.RandomState(0)
    pairs = np.stack([rng.randint(ds.num_users, size=16), rng.randint(ds.num_items, size=16)], axis=1)
    single = np.array([m.score(int(u), int(i)) for u, i in pairs])
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        uir_u=np.asarray(uir[0], np.int64), uir_i=np.asarray(uir[1], np.int64), uir_r=np.asarray(uir[2], np.float64),
        indptr=X.indptr.astype(np.int32), indices=X.indices.astype(np.int32), data=X.data.astype(np.float32),
        num_users=ds.num_users, num_items=ds.num_items, global_mean=ds.global_mean, mu=seen["mu"],
        k=m.k, max_iter=m.max_iter, learning_rate=m.learning_rate, lambda_reg=m.lambda_reg, lambda_u=m.lambda_u,
        lambda_v=m.lambda_v, lambda_bu=m.lambda_bu, lambda_bi=m.lambda_bi, use_bias=m.use_bias, seed=m.seed,
        init_given=np.array(sorted(params) if params else [], dtype="U2"),
        U0=seen["U0"], V0=seen["V0"], Bu0=seen["Bu0"], Bi0=seen["Bi0"],
        U=m.u_factors, V=m.i_factors, Bu=m.u_biases, Bi=m.i_biases,
        single_pairs=pairs.astype(np.int64), single_scores=single, single_dtype=str(np.asarray(single).dtype))
    print(name, "ok", ds.num_users, ds.num_items, X.nnz, single.dtype)


def experiment_case(name):
    import cornac
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, MAE, NDCG, RMSE, Precision, Recall
    u, i, r = synth_uir(300, 250, 7000, 51)
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    rs = RatioSplit(data=data, test_size=0.2, rating_threshold=4.0, exclude_unknowns=True, seed=123, verbose=False)
    hyper = dict(k=15, max_iter=50, learning_rate=0.005, lambda_u=0.06, lambda_v=0.06, lambda_bu=0.02, lambda_bi=0.02,
                 seed=123)
    metrics = [MAE(), RMSE(), Recall(k=20), Precision(k=20), NDCG(), AUC()]
    exp = cornac.Experiment(eval_method=rs, models=[cornac.models.NMF(use_bias=False, **hyper)], metrics=metrics,
                            user_based=True, verbose=False)
    exp.run()
    plain = exp.result[0].metric_avg_results
    rating_metrics = [MAE(), RMSE()]
    exp = cornac.Experiment(eval_method=rs, models=[cornac.models.NMF(use_bias=True, **hyper)], metrics=rating_metrics,
                            user_based=True, verbose=False)
    exp.run()
    biased = exp.result[0].metric_avg_results
    names = [m.name for m in metrics]
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"), uir_u=u, uir_i=i, uir_r=r,
        metric_names=np.array(names), plain=np.array([plain[n] for n in names]),
        bias_metric_names=np.array([m.name for m in rating_metrics]),
        bias=np.array([biased[m.name] for m in rating_metrics]))
    print(name, plain, biased)


def nmf_cases():
    small = synth_uir(120, 100, 1500, 61)
    mid = synth_uir(500, 400, 12000, 62)
    nmf_case("nmf_default_k15", small, seed=7)
    nmf_case("nmf_bias_k10", synth_uir(200, 160, 4000, 63), k=10, max_iter=30, learning_rate=0.01, use_bias=True, seed=8)
    nmf_case("nmf_lambda_reg_k8", small, k=8, max_iter=20, lambda_reg=0.03, use_bias=True, seed=9)

    def init_u_bi(n_users, n_items, k):
        g = np.random.RandomState(5)
        return {"U": g.uniform(0, 1, (n_users, k)).astype(np.float32),
                "Bi": g.normal(0, 0.3, n_items).astype(np.float32)}

    nmf_case("nmf_init_u_bi_k6", small, init=init_u_bi, k=6, max_iter=25, use_bias=False, seed=10)
    nmf_case("nmf_k1", small, k=1, max_iter=40, seed=11)
    nmf_case("nmf_bias_k1", small, k=1, max_iter=40, use_bias=True, seed=12)
    nmf_case("nmf_mid_k12", mid, k=12, max_iter=10, use_bias=True, learning_rate=0.01, seed=13)
    experiment_case("nmf_experiment")


if __name__ == "__main__":
    nmf_cases()
