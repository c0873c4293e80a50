"""Generate the PMF golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_pmf.py

Each fit case runs cornac.models.PMF (cornac/models/pmf/recom_pmf.py) on synthetic, seeded ratings and stores the ratings
exactly as fit() passes them to pmf_linear / pmf_non_linear (after the `scale` call), the initial factors, the trained
factors, the per-epoch loss (from a direct call of the same Cython function with the same arguments, since fit() drops
it) and a few scores.  The experiment case stores a RatioSplit and the metrics an unchanged Experiment gives.
No reference file is copied.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import dataset_from, synth_uir  # noqa: E402  (puts oracle/_ref on sys.path and imports cornac)


def pmf_case(name, uir, k, max_iter, variant, seed=7, init_u=None, **hyper):
    from cornac.models import PMF
    from cornac.models.pmf import pmf as cy
    ds = dataset_from(*uir)
    kw = dict(k=k, max_iter=max_iter, variant=variant, seed=seed, **hyper)
    init = None
    if init_u is not None:
        init = {"U": init_u(ds.num_users, k)}
    U_given = None if init is None else init["U"].copy()
    # the inputs fit() hands the Cython function (recom_pmf.py:129-135)
    seen = {}
    fn_name = "pmf_linear" if variant == "linear" else "pmf_non_linear"
    real = getattr(cy, fn_name)

    def spy(uid, iid, rat, **a):
        seen.update(uid=np.array(uid), iid=np.array(iid), rat=np.array(rat), args=dict(a))
        U0, V0 = cy._init_factors(a["n_users"], a["n_items"], a["k"], a["init_params"], a["seed"])
        seen.update(U0=np.array(U0, copy=True), V0=np.array(V0, copy=True))
        return real(uid, iid, rat, **a)

    setattr(cy, fn_name, spy)
    try:
        m = PMF(init_params=init, **kw).fit(ds)
    finally:
        setattr(cy, fn_name, real)
    a = dict(seen["args"])
    a["init_params"] = {"U": seen["U0"].copy(), "V": seen["V0"].copy()}
    res = real(seen["uid"], seen["iid"], seen["rat"], **a)
    assert np.array_equal(np.asarray(res["U"]), m.U) and np.array_equal(np.asarray(res["V"]), m.V)
    rng = np.random.RandomState(0)
    pairs = np.stack([rng.randint(ds.num_users, size=16), rng.randint(ds.num_items, size=16)], axis=1)
    single = np.array([m.score(int(u), int(i)) for u, i in pairs])
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        uir_u=np.asarray(uir[0], np.int64), uir_i=np.asarray(uir[1], np.int64), uir_r=np.asarray(uir[2], np.float64),
        uid=seen["uid"].astype(np.int32), iid=seen["iid"].astype(np.int32), rat=seen["rat"].astype(np.float32),
        num_users=ds.num_users, num_items=ds.num_items, min_rating=ds.min_rating, max_rating=ds.max_rating,
        k=k, max_iter=max_iter, variant=variant, seed=seed, init_u_given=U_given is not None,
        learning_rate=m.learning_rate, gamma=m.gamma, lambda_reg=m.lambda_reg,
        U0=seen["U0"], V0=seen["V0"], U=m.U, V=m.V, loss=np.asarray(res["loss"]),
        single_pairs=pairs.astype(np.int64), single_scores=single)
    print(name, "ok", ds.num_users, ds.num_items, len(seen["uid"]), "loss[-1]=%r" % float(res["loss"][-1]))


def experiment_case(name):
    """PMF (both variants) through RatioSplit + an unchanged Experiment: the split and the metric values."""
    import cornac
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, MAE, NDCG, RMSE, Recall
    u, i, r = synth_uir(300, 250, 7000, 31)
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, seed=123, verbose=False)
    metrics = [RMSE(), MAE(), Recall(k=10), NDCG(k=10), AUC()]
    models = [cornac.models.PMF(k=10, max_iter=60, learning_rate=0.01, lambda_reg=0.01, variant="linear", seed=123,
                                name="PMF-linear"),
              cornac.models.PMF(k=10, max_iter=60, learning_rate=0.01, lambda_reg=0.01, seed=123, name="PMF-non_linear")]
    exp = cornac.Experiment(eval_method=rs, models=models, metrics=metrics, verbose=False)
    exp.run()
    res = {r.model_name: r.metric_avg_results for r in exp.result}
    names = [m.name for m in metrics]
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"), uir_u=u, uir_i=i, uir_r=r, metric_names=np.array(names),
        linear=np.array([res["PMF-linear"][n] for n in names]), non_linear=np.array([res["PMF-non_linear"][n] for n in names]))
    print(name, res)


def pmf_cases():
    small = synth_uir(120, 100, 1500, 41)
    mid = synth_uir(500, 400, 12000, 42)
    pmf_case("pmf_linear_k5", small, k=5, max_iter=100, variant="linear")
    pmf_case("pmf_linear_k10_mid", mid, k=10, max_iter=20, variant="linear", learning_rate=0.01, lambda_reg=0.01)
    pmf_case("pmf_nonlinear_k10", synth_uir(200, 160, 4000, 43), k=10, max_iter=40, variant="non_linear",
             learning_rate=0.05, lambda_reg=0.01, gamma=0.8)
    u, i, r = synth_uir(150, 120, 2500, 44)
    unit = (u, i, (r - 1.0) / 4.0)                     # already in [0, 1]: fit() skips the scale call
    pmf_case("pmf_nonlinear_unit", unit, k=6, max_iter=40, variant="non_linear", learning_rate=0.05)
    pmf_case("pmf_linear_init_u_k7", small, k=7, max_iter=30, variant="linear", learning_rate=0.01,
             init_u=lambda n, k: np.random.RandomState(5).normal(0, 0.1, (n, k)))
    pmf_case("pmf_nonlinear_k1", small, k=1, max_iter=50, variant="non_linear", learning_rate=0.05)
    pmf_case("pmf_linear_k1", small, k=1, max_iter=50, variant="linear", learning_rate=0.01)
    experiment_case("pmf_experiment")


if __name__ == "__main__":
    pmf_cases()
