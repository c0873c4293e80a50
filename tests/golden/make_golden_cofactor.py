"""Generate the SoRec and MCF golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_cofactor.py

Each fit case runs cornac.models.SoRec / MCF (cornac/models/sorec/recom_sorec.py, cornac/models/mcf/recom_mcf.py) on
synthetic, seeded ratings and a synthetic graph modality, and stores the graph and rating triplets exactly as fit() hands
them to the Cython sorec / mcf function (after weight_link and the scale calls), the initial factors, the trained factors,
the per-epoch loss (from a direct call of the same Cython function with the same arguments, since fit() drops it) and a
few single-pair scores.  The experiment cases store the metrics an unchanged Experiment gives with the settings of the
reference's examples/sorec_filmtrust.py and examples/mcf_office.py.  No reference file is copied.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import dataset_from, synth_uir  # noqa: E402  (puts oracle/_ref on sys.path and imports cornac)


def synth_graph(n_nodes, n_edges, seed, self_loops=False, duplicates=False, values=None):
    """Raw (a, b, value) edges over node ids [0, n_nodes); distinct pairs without self-loops unless asked."""
    rng = np.random.RandomState(seed)
    edges = []
    seen = set()
    while len(edges) < n_edges:
        a, b = int(rng.randint(n_nodes)), int(rng.randint(n_nodes))
        if (a == b and not self_loops) or ((a, b) in seen and not duplicates):
            continue
        seen.add((a, b))
        edges.append((a, b))
    if self_loops:
        edges += [(a, a) for a in rng.randint(n_nodes, size=5).tolist()]
    if duplicates:
        edges += [edges[j] for j in rng.randint(len(edges), size=8).tolist()]
    vals = np.ones(len(edges)) if values is None else values(rng, len(edges))
    return np.array(edges, dtype=np.int64).reshape(-1, 2), np.asarray(vals, dtype=np.float64)


def _with_graph(ds, kind, edges, vals):
    from cornac.data import GraphModality
    gm = GraphModality(data=[(str(a), str(b), float(v)) for (a, b), v in zip(edges, vals)])
    gm.build(id_map=ds.uid_map if kind == "user" else ds.iid_map)
    ds.add_modalities(**{kind + "_graph": gm})
    return ds


def cofactor_case(name, model, uir, edges, vals, k, max_iter, seed=7, init=None, **hyper):
    """model: "sorec" or "mcf".  init: None or a function (num_users, num_items, k) -> init_params dict (f64 arrays)."""
    from cornac.utils import get_rng
    from cornac.utils.init_utils import normal
    if model == "sorec":
        from cornac.models import SoRec as Model
        from cornac.models.sorec import sorec as cy
    else:
        from cornac.models import MCF as Model
        from cornac.models.mcf import mcf as cy
    ds = _with_graph(dataset_from(*uir), "user" if model == "sorec" else "item", edges, vals)
    n_nodes = ds.num_users if model == "sorec" else ds.num_items
    ip = None if init is None else init(ds.num_users, ds.num_items, k)
    given = {} if ip is None else {key: x.copy() for key, x in ip.items()}
    seen = {}
    real = getattr(cy, model)

    def spy(rat_uid, rat_iid, rat_val, net_a, net_b, net_val, **a):
        seen.update(uid=np.array(rat_uid), iid=np.array(rat_iid), rat=np.array(rat_val), net_a=np.array(net_a),
                    net_b=np.array(net_b), net_val=np.array(net_val), args=dict(a))
        rng = get_rng(a["seed"])                           # sorec.pyx:63-75 / mcf.pyx:66-78: U, V, Z from one generator
        f0 = {}
        for key, n in (("U", a["n_users"]), ("V", a["n_items"]), ("Z", n_nodes)):
            x = a["init_params"].get(key, None)
            f0[key] = normal((n, a["k"]), mean=0.0, std=0.001, random_state=rng, dtype=np.double) if x is None else x
        seen.update({key + "0": np.array(x, copy=True) for key, x in f0.items()})
        return real(rat_uid, rat_iid, rat_val, net_a, net_b, net_val, **a)

    setattr(cy, model, spy)
    try:
        m = Model(k=k, max_iter=max_iter, seed=seed, init_params=ip, **hyper).fit(ds)
    finally:
        setattr(cy, model, real)
    a = dict(seen["args"])
    a["init_params"] = {key: seen[key + "0"].copy() for key in "UVZ"}
    res = real(seen["uid"], seen["iid"], seen["rat"], seen["net_a"], seen["net_b"], seen["net_val"], **a)
    for key in "UVZ":
        assert np.array_equal(np.asarray(res[key]), getattr(m, key)), key
    rng = np.random.RandomState(0)
    pairs = np.stack([rng.randint(ds.num_users, size=16), rng.randint(ds.num_items, size=16)], axis=1)
    single = np.array([m.score(int(u), int(i)) for u, i in pairs])
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        model=model, uir_u=np.asarray(uir[0], np.int64), uir_i=np.asarray(uir[1], np.int64),
        uir_r=np.asarray(uir[2], np.float64), graph_a=edges[:, 0], graph_b=edges[:, 1], graph_val=vals,
        uid=seen["uid"].astype(np.int32), iid=seen["iid"].astype(np.int32), rat=seen["rat"].astype(np.float32),
        net_a=seen["net_a"].astype(np.int32), net_b=seen["net_b"].astype(np.int32), net_val=seen["net_val"].astype(np.float32),
        num_users=ds.num_users, num_items=ds.num_items, min_rating=ds.min_rating, max_rating=ds.max_rating,
        k=k, max_iter=max_iter, seed=seed, init_given=np.array(sorted(given)),
        hyper_names=np.array(sorted(hyper)), hyper_values=np.array([float(hyper[h]) for h in sorted(hyper)]),
        learning_rate=float(m.learning_rate), gamma=float(m.gamma),
        lambda_reg=float(m.lambda_reg if model == "sorec" else m.lamda),
        lambda_c=float(m.lambda_c) if model == "sorec" else 0.0, weight_link=bool(getattr(m, "weight_link", False)),
        U0=seen["U0"], V0=seen["V0"], Z0=seen["Z0"], U=m.U, V=m.V, Z=m.Z, loss=np.asarray(res["loss"]),
        single_pairs=pairs.astype(np.int64), single_scores=single)
    print(name, "ok", ds.num_users, ds.num_items, len(seen["uid"]), "edges", len(seen["net_a"]),
          "loss[-1]=%r" % float(res["loss"][-1]))


def experiment_case(name, model):
    """The settings of examples/sorec_filmtrust.py / examples/mcf_office.py on synthetic ratings and a synthetic graph."""
    import cornac
    from cornac.data import GraphModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import NDCG, RMSE, Precision, Recall
    u, i, r = synth_uir(300, 250, 7000, 61 if model == "sorec" else 62)
    edges, vals = synth_graph(300 if model == "sorec" else 250, 1200, 63)
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    gm = GraphModality(data=[(str(a), str(b), float(v)) for (a, b), v in zip(edges, vals)])
    if model == "sorec":
        rs = RatioSplit(data=data, test_size=0.2, rating_threshold=2.5, exclude_unknowns=True, verbose=False,
                        user_graph=gm, seed=123)
        m = cornac.models.SoRec(k=10, max_iter=50, learning_rate=0.001, verbose=False, seed=123)
        metrics = [RMSE(), NDCG(k=-1), Precision(k=20), Recall(k=20)]
    else:
        rs = RatioSplit(data=data, test_size=0.2, rating_threshold=3.5, exclude_unknowns=True, verbose=False,
                        item_graph=gm, seed=123)
        m = cornac.models.MCF(k=10, max_iter=40, learning_rate=0.001, verbose=False, seed=123)
        metrics = [RMSE(), NDCG(k=-1), Recall(k=20), Precision(k=20)]
    exp = cornac.Experiment(eval_method=rs, models=[m], metrics=metrics, verbose=False)
    exp.run()
    res = exp.result[0].metric_avg_results
    names = [x.name for x in metrics]
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"), model=model, uir_u=u, uir_i=i, uir_r=r, graph_a=edges[:, 0],
        graph_b=edges[:, 1], graph_val=vals, metric_names=np.array(names), metrics=np.array([res[n] for n in names]))
    print(name, res)


def cofactor_cases():
    small = synth_uir(120, 100, 1500, 71)
    mid = synth_uir(300, 220, 5000, 72)
    g_small = synth_graph(120, 400, 73)
    g_item = synth_graph(100, 350, 74, values=lambda rng, n: rng.randint(1, 9, size=n) * 0.5)
    # SoRec
    cofactor_case("sorec_k5", "sorec", small, *g_small, k=5, max_iter=30, learning_rate=0.01)
    cofactor_case("sorec_nolink_k10", "sorec", mid, *synth_graph(300, 900, 75), k=10, max_iter=20, learning_rate=0.01,
                  weight_link=False, lambda_reg=0.01)
    cofactor_case("sorec_k1", "sorec", small, *g_small, k=1, max_iter=25, learning_rate=0.02, lambda_c=2.0)
    cofactor_case("sorec_k37", "sorec", small, *g_small, k=37, max_iter=10, learning_rate=0.01, gamma=0.8)
    lc, lr = 3.3, 0.0123                                   # f32(lc) * f32(lr) rounds away from the f64 product
    assert float(np.float32(lc) * np.float32(lr)) != float(np.float32(lc)) * float(np.float32(lr))
    cofactor_case("sorec_step_product", "sorec", small, *g_small, k=6, max_iter=20, learning_rate=lr, lambda_c=lc)
    u, i, _ = small
    cofactor_case("sorec_minmax", "sorec", (u, i, np.full(len(u), 4.0)), *g_small, k=4, max_iter=15, learning_rate=0.01)
    cofactor_case("sorec_loops_dups", "sorec", small, *synth_graph(120, 300, 76, self_loops=True, duplicates=True), k=5,
                  max_iter=15, learning_rate=0.01)
    # an empty graph: every edge names a user outside the ratings
    cofactor_case("sorec_empty_graph", "sorec", small, np.array([[1000, 1001], [1002, 1000]]), np.ones(2), k=5,
                  max_iter=10, learning_rate=0.01)
    cofactor_case("sorec_warm_k6", "sorec", small, *g_small, k=6, max_iter=15, learning_rate=0.01,
                  init=lambda nu, ni, k: {"U": np.random.RandomState(5).normal(0, 0.1, (nu, k)),
                                          "Z": np.random.RandomState(6).normal(0, 0.1, (nu, k))})
    # MCF: the three edge-scaling branches (values spanning [0, 1], a constant, anything else)
    cofactor_case("mcf_k5", "mcf", small, *g_item, k=5, max_iter=30, learning_rate=0.01)
    cofactor_case("mcf_unit_k10", "mcf", mid, *synth_graph(220, 700, 77, values=lambda rng, n: np.r_[0.0, 1.0, rng.rand(n - 2)]),
                  k=10, max_iter=20, learning_rate=0.01, lamda=0.01)
    cofactor_case("mcf_const_k1", "mcf", small, *synth_graph(100, 300, 78, values=lambda rng, n: np.full(n, 2.0)), k=1,
                  max_iter=25, learning_rate=0.02)
    cofactor_case("mcf_warm_k37", "mcf", small, *g_item, k=37, max_iter=10, learning_rate=0.01, gamma=0.8,
                  init=lambda nu, ni, k: {"V": np.random.RandomState(8).normal(0, 0.1, (ni, k))})
    experiment_case("sorec_experiment", "sorec")
    experiment_case("mcf_experiment", "mcf")


if __name__ == "__main__":
    cofactor_cases()
