"""Generate the C2PF golden vectors from the UNMODIFIED compiled reference.

TEST INFRASTRUCTURE.  Needs oracle/_ref (`bash oracle/build_ref.sh` first):

    python tests/golden/make_golden_c2pf.py

Each fit case calls the compiled cornac.models.c2pf.c2pf functions (c2pf / t_c2pf / r_c2pf of c2pf.pyx) the way
recom_c2pf.py's fit() does, on synthetic seeded ratings and context triplets, and stores the inputs, the initial state
and everything the call returns for a few values of max_iter, each from the same initial state.  max_iter < 5 has no
second phase (int(0.2 * max_iter) == 0), so those results are the state after phase one.  The initial state is drawn as
c2pf.pyx draws it (the global numpy generator, G_s, G_r, L_s, L_r, L2_s, L2_r, L3_s, L3_r in that order, the variant's
matrices only), and the generator checks that a fit from those arrays equals the fit after np.random.seed.  The
asymmetric case stores how the reference's process ends when an edge's mirror is missing.  The experiment case stores a
RatioSplit, a graph and the metrics an unchanged Experiment gives with examples/c2pf_example.py's metrics.  No reference
file is copied.
"""
import contextlib
import io
import os
import subprocess
import sys
import tempfile

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import synth_uir  # noqa: E402  (puts oracle/_ref on sys.path and imports cornac)

STATE = ("G_s", "G_r", "L_s", "L_r", "L2_s", "L2_r", "L3_s", "L3_r")
HAS = {"c2pf": STATE, "tc2pf": ("G_s", "G_r", "L_s", "L_r", "L3_s", "L3_r"),
       "rc2pf": ("G_s", "G_r", "L2_s", "L2_r", "L3_s", "L3_r")}


def ratings_triplets(u, i, r, n, d):
    """recom_c2pf.py:149-159: sp.find of the CSR matrix, values through float32, as one f64 array."""
    X = sp.csr_matrix((np.asarray(r, np.float32), (u, i)), shape=(n, d))
    rid, cid, val = sp.find(X)
    val = np.array(val, dtype="float32")
    rid, cid = np.array(rid, dtype="int32"), np.array(cid, dtype="int32")
    return np.concatenate((np.concatenate(([rid], [cid]), axis=0).T, val.reshape((len(val), 1))), axis=1)


def synth_context(d, n_pairs, seed, isolated=(), symmetric=True):
    """[m, 3] (row, col, value) context triplets over items [0, d) without self-loops; both directions of each pair when
    symmetric; no edge touches an item of `isolated`."""
    rng = np.random.RandomState(seed)
    ok = np.setdiff1d(np.arange(d), isolated)
    pairs = set()
    while len(pairs) < n_pairs:
        a, b = rng.choice(ok, size=2, replace=False)
        pairs.add((min(a, b), max(a, b)))
    pairs = np.array(sorted(pairs))
    pairs = pairs[rng.permutation(len(pairs))]
    if symmetric:
        pairs = np.concatenate([pairs, pairs[:, ::-1]])
        pairs = pairs[rng.permutation(len(pairs))]
    return np.column_stack([pairs.astype(np.float64), rng.randint(1, 4, size=len(pairs)).astype(np.float64)])


def draw_state(variant, n, d, k, C, seed):
    """c2pf.pyx:62-119 (and its t_ / r_ twins): the draws from the global generator, in order."""
    np.random.seed(seed)
    st = {}
    for key in HAS[variant]:
        if key.startswith("L3"):
            t = np.copy(C)
            t[:, 2] = np.random.gamma(100, scale=0.5 / 100, size=C.shape[0])
            st[key] = t
        else:
            rows = n if key.startswith("G") else d
            st[key] = np.random.gamma(100, scale=0.3 / 100, size=rows * k).reshape(rows, k)
    return st


def run_ref(variant, tX, n, d, C, k, max_iter, init=None):
    from cornac.models.c2pf import c2pf as ext
    fn = {"c2pf": ext.c2pf, "tc2pf": ext.t_c2pf, "rc2pf": ext.r_c2pf}[variant]
    params = {key: None for key in STATE}
    if init is not None:
        params.update({key: np.copy(v) for key, v in init.items()})
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(tX, n, d, C, d, d, k, max_iter, params)


def c2pf_case(name, variant, uir, n, d, C, k, iters, seed=7, init=None):
    """init: None (the seeded draw) or a function (variant, n, d, k, C) -> {key: array}."""
    tX = ratings_triplets(*uir, n, d)
    if init is None:
        state0 = draw_state(variant, n, d, k, C, seed)
        np.random.seed(seed)
        # r_c2pf cannot draw the kappa triplets itself (c2pf.pyx:316-317 assigns a column of a C++ vector: TypeError)
        l3 = {key: state0[key] for key in ("L3_s", "L3_r")} if variant == "rc2pf" else None
        seeded = run_ref(variant, tX, n, d, C, k, iters[0], init=l3)
        given = run_ref(variant, tX, n, d, C, k, iters[0], init=state0)
        for key in ("Z", "W", "Q") + HAS[variant]:
            assert np.array_equal(np.asarray(seeded[key]), np.asarray(given[key])), key
    else:
        state0 = init(variant, n, d, k, C)
    out = dict(tX=tX, C=C, num_users=n, num_items=d, k=k, variant=variant, seed=seed, seeded=init is None,
               iters=np.array(iters))
    out.update({key + "0": v for key, v in state0.items()})
    finite = True
    for m in iters:
        res = run_ref(variant, tX, n, d, C, k, m, init=state0)
        for key in ("Z", "W", "Q") + STATE:
            if res[key] is None:
                assert key not in HAS[variant]
                continue
            out["%s_%d" % (key, m)] = np.asarray(res[key], np.float64)
            finite = finite and bool(np.all(np.isfinite(out["%s_%d" % (key, m)])))
        finite = finite and bool(np.all(np.isfinite(res["Z"])) and np.all(np.isfinite(res["Q"])))
    out["finite"] = finite
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    assert finite or "asym" in name, name
    print(name, "ok", n, d, len(tX), len(C), "k=%d" % k, "iters", iters, "finite", finite)


def _nonpositive(variant, n, d, k, C):
    """A drawn state with some dense entries set to 0 or negative values: shape only, rate only, and both at once.  Only
    c2pf's L_r, whose quotients the reference guards, gets exact zeros among the rates: G_r sums L2_s / L2_r unguarded
    (and tc2pf's L2 is its L)."""
    st = draw_state(variant, n, d, k, C, 11)
    rng = np.random.RandomState(12)
    dense = [key for key in HAS[variant] if not key.startswith("L3")]
    for key in dense:
        x = st[key]
        rows = rng.choice(x.shape[0], size=max(1, x.shape[0] // 20), replace=False)
        cols = rng.randint(k, size=len(rows))
        zero = (rng.rand(len(rows)) < 0.5) & (key.endswith("_s") or (key == "L_r" and variant == "c2pf"))
        x[rows, cols] = np.where(zero, 0.0, -0.05 * x[rows, cols])
    for s, r in zip(dense[0::2], dense[1::2]):
        st[s][1, 0], st[r][1, 0] = 0.0, -0.1
        st[s][2, k - 1], st[r][2, k - 1] = -0.2, -0.3
    return st


def _warm(uir, n, d, iters):
    """A warm start: what a fit from the seeded draw returns (what a second fit() starts from)."""
    def init(variant, n_, d_, k, C):
        l3 = draw_state(variant, n, d, k, C, 3)
        np.random.seed(3)
        res = run_ref(variant, ratings_triplets(*uir, n, d), n, d, C, k, iters,
                      init={key: l3[key] for key in ("L3_s", "L3_r")} if variant == "rc2pf" else None)
        return {key: np.ascontiguousarray(res[key]) for key in HAS[variant]}
    return init


def experiment_case(name):
    """The three variants with examples/c2pf_example.py's metrics through RatioSplit + an unchanged Experiment."""
    import cornac
    from cornac.data import GraphModality
    from cornac.eval_methods import RatioSplit
    from cornac.metrics import MRR, NDCG, Precision, Recall
    u, i, r = synth_uir(150, 120, 3000, 61)
    C = synth_context(120, 400, 62)
    data = [(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)]
    graph = [(str(int(a)), str(int(b)), float(v)) for a, b, v in C]
    rs = RatioSplit(data=data, test_size=0.2, exclude_unknowns=True, verbose=False, seed=123, rating_threshold=0.5,
                    item_graph=GraphModality(data=graph))
    metrics = [NDCG(k=-1), MRR(), Recall(k=20), Precision(k=20)]
    names = [m.name for m in metrics]
    out = dict(uir_u=u, uir_i=i, uir_r=r, C=C, metric_names=np.array(names))
    for variant in ("c2pf", "tc2pf"):          # the reference's rc2pf cannot start without given kappa triplets
        np.random.seed(5)
        model = cornac.models.C2PF(k=6, max_iter=10, variant=variant)
        with contextlib.redirect_stdout(io.StringIO()):
            exp = cornac.Experiment(eval_method=rs, models=[model], metrics=metrics, user_based=True, verbose=False,
                                    save_dir=tempfile.mkdtemp())
            exp.run()
        res = exp.result[0].metric_avg_results
        out[variant] = np.array([res[m] for m in names])
        print(name, variant, res)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)


def c2pf_cases():
    n, d = 70, 56
    u, i, r = synth_uir(n, d - 1, 700, 71)                       # item d - 1 has no rating (and has context)
    uir = (u, i, r)
    rated = np.unique(i)
    lonely = int(rated[len(rated) // 2])                         # an item with ratings and no context
    C = synth_context(d, 90, 72, isolated=[lonely])
    assert d - 1 in C[:, 0] and d - 1 not in i
    for v in HAS:
        c2pf_case("%s_k1" % v, v, uir, n, d, C, 1, [4, 10])
        c2pf_case("%s_k5" % v, v, uir, n, d, C, 5, [1, 4, 10])
        c2pf_case("%s_k37" % v, v, uir, n, d, C, 37, [5])
        c2pf_case("%s_warm_k4" % v, v, uir, n, d, C, 4, [5], init=_warm(uir, n, d, 5))
        c2pf_case("%s_nonpos_k4" % v, v, uir, n, d, C, 4, [1, 5], init=_nonpositive)
        # every fifth triplet repeated later with another value: the pattern is unchanged, the LAST value of a pair is
        # the one the fit uses and util_sum adds both
        rep = C[::5].copy()
        rep[:, 2] += 2.0
        c2pf_case("%s_dup_k3" % v, v, uir, n, d, np.concatenate([C, rep]), 3, [5])
    experiment_case("c2pf_experiment")
    # an edge whose mirror is missing: what does the reference do?  Each variant runs in a process of its own, because the
    # answer is that the process dies: the walk of the column inserts a zero shape at the missing mirror, L3_s then has
    # one entry more than the triplet list it is written back to, and csc_sparse_to_triplet writes past its end.
    Ca = np.concatenate([C, [[3.0, float(lonely), 1.0]]])
    np.savez_compressed(os.path.join(HERE, "c2pf_asym_in.npz"), u=u, i=i, r=r, C=Ca, num_users=n, num_items=d)
    codes = [subprocess.run([sys.executable, os.path.abspath(__file__), "--asym", v]).returncode for v in HAS]
    if os.path.exists(os.path.join(HERE, "c2pf_asym_k3.npz")):
        os.remove(os.path.join(HERE, "c2pf_asym_k3.npz"))
    print("asymmetric pattern: return codes", dict(zip(HAS, codes)))
    np.savez_compressed(os.path.join(HERE, "c2pf_asym.npz"), u=u, i=i, r=r, C=Ca, num_users=n, num_items=d,
                        variants=np.array(list(HAS)), returncodes=np.array(codes))
    os.remove(os.path.join(HERE, "c2pf_asym_in.npz"))


def asym_run(variant):
    g = np.load(os.path.join(HERE, "c2pf_asym_in.npz"))
    c2pf_case("c2pf_asym_k3", variant, (g["u"], g["i"], g["r"]), int(g["num_users"]), int(g["num_items"]), g["C"], 3, [1])


if __name__ == "__main__":
    if sys.argv[1:2] == ["--asym"]:
        asym_run(sys.argv[2])
    else:
        c2pf_cases()
