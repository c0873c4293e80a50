"""Generate the HPF / PF golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_hpf.py

Each fit case runs cornac.models.HPF (cornac/models/hpf/recom_hpf.py) on synthetic, seeded ratings and stores the
ratings exactly as fit() hands them to hpf_cpp / pf_cpp (sp.find of the CSC matrix, values through float32), the initial
state, and the state, Theta and Beta after each of a few iteration counts, each from the same initial state.  The initial
state is drawn as hpf.pyx draws it (get_rng(seed), then `gamma` for G_s, G_r, L_s, L_r in that order), and the generator
checks that a fit from those arrays equals the seeded fit.  The experiment case stores a RatioSplit and the metrics an
unchanged Experiment gives with the settings of the reference's examples/hpf_movielens.py.  No reference file is copied.
"""
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import dataset_from, synth_uir  # noqa: E402  (puts oracle/_ref on sys.path and imports cornac)


def draw_state(n, d, k, hierarchical, seed):
    """hpf.pyx:35-82 / 100-149: the four gamma draws in order."""
    from cornac.utils import get_rng
    from cornac.utils.init_utils import gamma
    rng = get_rng(seed)
    shape, scale = (100.0, 0.3 / 100.0) if hierarchical else (0.3, 1 / 0.3)
    Gs = gamma(shape, scale=scale, size=n * k, random_state=rng).reshape(n, k)
    Gr = gamma(shape, scale=scale, size=n * k, random_state=rng).reshape(n, k)
    Ls = gamma(shape, scale=scale, size=d * k, random_state=rng).reshape(d, k)
    Lr = gamma(shape, scale=scale, size=d * k, random_state=rng).reshape(d, k)
    return [np.ascontiguousarray(x, dtype=np.float64) for x in (Gs, Gr, Ls, Lr)]


def _fit(ds, k, hierarchical, max_iter, init=None, seed=None):
    from cornac.models import HPF
    params = None if init is None else dict(zip(("G_s", "G_r", "L_s", "L_r"), [x.copy() for x in init]))
    return HPF(k=k, max_iter=max_iter, hierarchical=hierarchical, seed=seed, init_params=params).fit(ds)


def hpf_case(name, uir, k, hierarchical, iters, seed=7, init=None):
    """init: None (the seeded draw) or a function (n, d, k) -> [G_s, G_r, L_s, L_r]."""
    ds = dataset_from(*uir)
    n, d = ds.num_users, ds.num_items
    rid, cid, val = sp.find(ds.csc_matrix)
    val = np.array(val, dtype="float32")
    if init is None:
        state0 = draw_state(n, d, k, hierarchical, seed)
        seeded = _fit(ds, k, hierarchical, iters[0], seed=seed)
        given = _fit(ds, k, hierarchical, iters[0], init=state0)
        for a in ("Gs", "Gr", "Ls", "Lr", "Theta", "Beta"):
            assert np.array_equal(getattr(seeded, a), getattr(given, a)), a
    else:
        state0 = init(n, d, k)
    out = dict(uir_u=np.asarray(uir[0], np.int64), uir_i=np.asarray(uir[1], np.int64),
               uir_r=np.asarray(uir[2], np.float64), rid=rid.astype(np.int32), cid=cid.astype(np.int32), val=val,
               num_users=n, num_items=d, k=k, hierarchical=hierarchical, seed=seed, seeded=init is None,
               iters=np.array(iters), Gs0=state0[0], Gr0=state0[1], Ls0=state0[2], Lr0=state0[3])
    for m in iters:
        r = _fit(ds, k, hierarchical, m, init=state0)
        for a in ("Gs", "Gr", "Ls", "Lr", "Theta", "Beta"):
            out["%s_%d" % (a, m)] = np.asarray(getattr(r, a), np.float64)
        assert np.all(np.isfinite(r.Theta)) and np.all(np.isfinite(r.Beta)), (name, m)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "ok", n, d, len(val), "k=%d" % k, "iters", iters)


def experiment_case(name):
    """PF and HPF with examples/hpf_movielens.py's settings through RatioSplit + an unchanged Experiment."""
    import cornac
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import AUC, NDCG, Recall
    u, i, r = synth_uir(300, 250, 7000, 61)
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123, rating_threshold=0.5)
    models = [cornac.models.HPF(k=5, seed=123, hierarchical=False, name="PF"), cornac.models.HPF(k=5, seed=123)]
    metrics = [Recall(k=20), NDCG(k=20), AUC()]
    exp = cornac.Experiment(eval_method=rs, models=models, metrics=metrics, user_based=True, verbose=False)
    exp.run()
    res = {r.model_name: r.metric_avg_results for r in exp.result}
    names = [m.name for m in metrics]
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"), uir_u=u, uir_i=i, uir_r=r, metric_names=np.array(names),
        pf=np.array([res["PF"][n] for n in names]), hpf=np.array([res["HPF"][n] for n in names]))
    print(name, res)


def _nonpositive(hierarchical):
    """A drawn state with some entries set to 0 or negative values: shape only, rate only, and both at once."""
    def init(n, d, k):
        st = draw_state(n, d, k, hierarchical, 11)
        rng = np.random.RandomState(12)
        for x in st:
            m = x.shape[0]
            rows = rng.choice(m, size=max(1, m // 20), replace=False)
            cols = rng.randint(k, size=len(rows))
            x[rows, cols] = np.where(rng.rand(len(rows)) < 0.5, 0.0, -0.05 * x[rows, cols])
        # entries where both the shape and the rate are dropped
        for s, r in ((st[0], st[1]), (st[2], st[3])):
            s[1, 0], r[1, 0] = 0.0, -0.1
            s[2, k - 1], r[2, k - 1] = -0.2, 0.0
        return st
    return init


def _warm(hierarchical):
    """A warm start: the state a 10-iteration fit from the seeded draw leaves (what a second fit() starts from)."""
    def init(n, d, k):
        ds = dataset_from(*WARM_UIR)
        m = _fit(ds, k, hierarchical, 10, seed=3)
        return [np.ascontiguousarray(x) for x in (m.Gs, m.Gr, m.Ls, m.Lr)]
    return init


WARM_UIR = None


def hpf_cases():
    global WARM_UIR
    mid = synth_uir(500, 400, 12000, 71)
    small = synth_uir(200, 160, 4000, 72)
    WARM_UIR = small
    hpf_case("hpf_k5", mid, k=5, hierarchical=True, iters=[1, 10, 100])
    hpf_case("pf_k5", mid, k=5, hierarchical=False, iters=[1, 10, 100])
    hpf_case("hpf_k1", small, k=1, hierarchical=True, iters=[1, 10, 100])
    hpf_case("pf_k1", small, k=1, hierarchical=False, iters=[1, 100])
    hpf_case("hpf_k10", small, k=10, hierarchical=True, iters=[10, 100])
    hpf_case("pf_k10", small, k=10, hierarchical=False, iters=[10, 100])
    hpf_case("hpf_k37", small, k=37, hierarchical=True, iters=[1, 100])
    hpf_case("pf_k37", small, k=37, hierarchical=False, iters=[1, 100])
    hpf_case("hpf_warm_k6", small, k=6, hierarchical=True, iters=[10], init=_warm(True))
    hpf_case("pf_warm_k6", small, k=6, hierarchical=False, iters=[10], init=_warm(False))
    hpf_case("hpf_nonpos_k4", small, k=4, hierarchical=True, iters=[1, 10], init=_nonpositive(True))
    hpf_case("pf_nonpos_k4", small, k=4, hierarchical=False, iters=[1, 10], init=_nonpositive(False))
    experiment_case("hpf_experiment")


if __name__ == "__main__":
    hpf_cases()
