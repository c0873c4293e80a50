"""C2PF without a GPU: the C oracle against the compiled reference's fixtures (both phases, the kappa triplet lists, the
rc2pf by-value rule, repeated edges), what the reference does on an asymmetric graph, and the plug-in's host logic."""
import contextlib
import io

import numpy as np
import pytest

from conftest import golden, needs_cornac
from oracle import c2pf_oracle as CO

VARIANTS = ("c2pf", "tc2pf", "rc2pf")
CASES = ["%s_%s" % (v, c) for v in VARIANTS for c in ("k1", "k5", "k37", "warm_k4", "nonpos_k4", "dup_k3")]
KEYS = ("G_s", "G_r", "L_s", "L_r", "L2_s", "L2_r", "L3_s", "L3_r")


def rel_max(got, want):
    return float(np.max(np.abs(got - want)) / np.max(np.abs(want)))


def problem(g):
    n, d = int(g["num_users"]), int(g["num_items"])
    tX, C = g["tX"], g["C"]
    X = CO.csc(tX[:, 0].astype(int), tX[:, 1].astype(int), tX[:, 2], n, d)
    G = CO.Graph(C[:, 0], C[:, 1], C[:, 2], d)
    st = [g[key + "0"].copy() if key + "0" in g else None for key in KEYS] + [np.ones(d)]
    return X, G, st


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_the_reference(name):
    """max_iter < 5 has no second phase, so those fixtures pin phase one alone."""
    g = golden(name)
    variant = str(g["variant"])
    for m in g["iters"]:
        X, G, st = problem(g)
        Z, W, Q = CO.fit_two_phase(variant, X, G, st, int(m))
        for key, got in zip(KEYS + ("Z", "W", "Q"), st[:8] + [Z, W, Q]):
            name_m = "%s_%d" % (key, m)
            assert (got is None) == (name_m not in g), (m, key)          # tc2pf: no L2; rc2pf: no L
            if got is None:
                continue
            want = g[name_m]
            assert np.all(np.isfinite(want)) and np.all(np.isfinite(got))
            if key.startswith("L3"):
                assert np.array_equal(got[:, :2], want[:, :2]), (m, key)
                got, want = got[:, 2], want[:, 2]
            assert rel_max(got, want) <= 1e-13, (m, key)


def test_fixtures_cover_the_cases():
    assert {int(golden(n)["k"]) for n in CASES} >= {1, 5, 37}
    for v in VARIANTS:
        g = golden(v + "_k5")
        assert bool(g["seeded"]) and {1, 4, 10} <= {int(m) for m in g["iters"]}
        assert int(0.2 * 4) == 0 and int(0.2 * 10) == 2
        d = int(g["num_items"])
        rated, ctx = np.unique(g["tX"][:, 1]), np.unique(g["C"][:, 0])
        assert len(np.setdiff1d(np.arange(d), rated)) and len(np.setdiff1d(rated, ctx))
        n = golden(v + "_nonpos_k4")
        dense = [k for k in KEYS[:6] if k + "0" in n]
        for s, r in zip(dense[0::2], dense[1::2]):
            s, r = n[s + "0"], n[r + "0"]
            assert np.any((s <= 0) & (r > 0)) and np.any((s > 0) & (r <= 0)) and np.any((s <= 0) & (r <= 0))


@pytest.mark.parametrize("variant", VARIANTS)
def test_kappa_triplets_come_back_in_csc_order_and_rc2pf_keeps_the_draw(variant):
    g = golden(variant + "_k5")
    C, got0, got = g["C"], g["L3_s0"], g["L3_s_10"]
    if variant == "rc2pf":
        assert np.array_equal(got, got0) and np.array_equal(g["L3_r_10"], g["L3_r0"])
        return
    order = np.lexsort((C[:, 0], C[:, 1]))
    assert np.array_equal(got[:, :2], C[order, :2]) and not np.array_equal(got[:, :2], C[:, :2])
    assert not np.array_equal(got[:, 2], got0[order, 2])


@pytest.mark.parametrize("variant", VARIANTS)
def test_repeated_edges_keep_the_last_value_and_the_tail_of_the_list(variant):
    g = golden(variant + "_dup_k3")
    C = g["C"]
    G = CO.Graph(C[:, 0], C[:, 1], C[:, 2], int(g["num_items"]))
    assert G.nnz < len(C)
    pairs = {}
    for r, c, v in C:
        pairs[(r, c)] = v
    assert np.array_equal(G.values(C), [pairs[(r, c)] for r, c in zip(G.row, G.col)])
    assert G.util.sum() == C[:, 2].sum() > G.values(C).sum()
    if variant != "rc2pf":                                  # rows past nnz are never written back
        assert np.array_equal(g["L3_s_5"][G.nnz:], g["L3_s0"][G.nnz:])


def test_the_reference_dies_on_an_asymmetric_graph_and_the_oracle_reports_it():
    """Evidence for the ValueError of the plug-in: on a graph with one unmirrored edge, each variant of the compiled
    reference ended its process with SIGSEGV (return code -11) when the fixture was generated."""
    g = golden("c2pf_asym")
    assert list(g["variants"]) == list(VARIANTS) and np.all(g["returncodes"] == -11)
    C = g["C"]
    G = CO.Graph(C[:, 0], C[:, 1], C[:, 2], int(g["num_items"]))
    with pytest.raises(ValueError):
        G.mirrors()


def test_oracle_split_fit_equals_one_fit():
    for variant in VARIANTS:
        X, G, st = problem(golden(variant + "_k5"))
        st[6], st[7] = G.values(st[6]), G.values(st[7])
        for at, bt in (CO.PHASE_ONE, CO.PHASE_TWO[variant]):
            one = [None if x is None else x.copy() for x in st]
            two = [None if x is None else x.copy() for x in st]
            CO.fit(variant, X, G, at, bt, one, 7)
            CO.fit(variant, X, G, at, bt, two, 3)
            CO.fit(variant, X, G, at, bt, two, 4)
            for a, b in zip(one, two):
                assert a is None or np.array_equal(a, b)


def test_oracle_update_equals_one_fit_iteration():
    for variant in VARIANTS:
        X, G, st = problem(golden(variant + "_k5"))
        st[6], st[7] = G.values(st[6]), G.values(st[7])
        at, bt = CO.PHASE_TWO[variant]
        a = [None if x is None else x.copy() for x in st]
        CO.fit(variant, X, G, at, bt, a, 0)                # c2pf: T3_r from the state
        E = CO.expectations(variant, G, a)
        CO.update(variant, X, G, at, bt, a, E)
        CO.fit(variant, X, G, at, bt, st, 1)
        for x, y in zip(a, st):
            assert x is None or np.array_equal(x, y)


@needs_cornac
def test_constructor_contract_matches_the_reference():
    from cornac.models import C2PF as RefC2PF
    from cornac_b200 import C2PF
    attrs = ("name", "k", "max_iter", "trainable", "verbose", "variant", "init_params", "eps", "Theta", "Beta", "Xi", "Gs",
             "Gr", "Ls", "Lr", "L2s", "L2r", "L3s", "L3r")
    for kw in ({}, dict(k=3, max_iter=7), dict(variant="tc2pf"), dict(variant="rc2pf", name="R"), dict(variant="other"),
               dict(trainable=False, verbose=True)):
        a, b = RefC2PF(**kw), C2PF(**kw)
        for attr in attrs:
            assert getattr(a, attr) == getattr(b, attr), (kw, attr)
        assert np.array_equal(a.ll, b.ll) and a.ll.dtype == b.ll.dtype
    assert C2PF(variant="tc2pf").name == "TC2PF" and C2PF(variant="other")._variant() == "c2pf"
    c = C2PF(k=4, variant="rc2pf").clone()
    assert isinstance(c, C2PF) and c.k == 4 and c.variant == "rc2pf"
    c = C2PF(k=4).clone(dict(k=6, max_iter=3))
    assert c.k == 6 and c.max_iter == 3 and len(c.ll) == 3


@needs_cornac
@pytest.mark.parametrize("variant", VARIANTS)
def test_initial_state_is_the_reference_draw(variant):
    from cornac_b200 import C2PF
    from cornac_b200.recom_c2pf import ContextGraph
    g = golden(variant + "_k5")
    n, d, C = int(g["num_users"]), int(g["num_items"]), g["C"]
    np.random.seed(int(g["seed"]))
    st = C2PF(k=5, variant=variant)._init_state(n, d, C, ContextGraph(C, d))
    assert list(st) == [key for key in KEYS if key + "0" in g]
    for key, x in st.items():
        assert np.array_equal(x, g[key + "0"]), key


@needs_cornac
def test_graph_preparation_and_validation():
    from cornac_b200 import C2PF
    from cornac_b200.recom_c2pf import ContextGraph
    g = golden("c2pf_dup_k3")
    d, C = int(g["num_items"]), g["C"]
    G, H = CO.Graph(C[:, 0], C[:, 1], C[:, 2], d), ContextGraph(C, d)
    assert np.array_equal(H.ptr, G.ptr) and np.array_equal(H.row, G.row) and np.array_equal(H.mir, G.mirrors())
    assert np.array_equal(H.util, G.util) and np.array_equal(H.values(C, "L3_s"), G.values(C))
    assert np.array_equal(H.row[H.mir], H.col) and np.array_equal(H.col[H.mir], H.row)
    trip = g["L3_s0"].copy()
    H.write_back(trip, np.arange(H.nnz, dtype=np.float64))
    assert np.array_equal(trip[: H.nnz], G.triplets(np.arange(H.nnz))) and np.array_equal(trip[H.nnz:], g["L3_s0"][H.nnz:])
    a = golden("c2pf_asym")["C"]
    with pytest.raises(ValueError, match=r"edge \(3, %d\).*symmetric=True" % int(a[-1, 1])):
        ContextGraph(a, d)
    n = int(g["num_users"])
    m = C2PF(k=3)
    for bad, match in (({"G_s": np.ones((n, 3), np.float32)}, "float64"), ({"L_r": np.ones((d + 1, 3))}, "shape"),
                       ({"L2_s": np.ones(d)}, "shape"), ({"L3_s": C[:, :2]}, "triplets"), ({"L3_r": C[:-50]}, "each context edge"),
                       ({"L3_s": C.astype(np.float32)}, "float64"), ({"L3_r": C * [1, 1, 0]}, "positive")):
        m = C2PF(k=3, init_params=bad)
        with pytest.raises(ValueError, match=match):
            m._init_state(n, d, C, H)


@needs_cornac
def test_single_scores_are_the_reference_expression_without_a_gpu():
    from cornac.models import C2PF as RefC2PF
    from cornac_b200 import C2PF
    for variant in VARIANTS:
        g = golden(variant + "_k5")
        params = dict(Theta=np.asmatrix(g["Z_10"]), Beta=np.asmatrix(g["W_10"]), Xi=np.asmatrix(g["Q_10"]))
        a = RefC2PF(k=5, variant=variant, trainable=False, init_params=params)
        b = C2PF(k=5, variant=variant, trainable=False, init_params=params)
        for u, i in ((0, 0), (3, 17)):
            assert np.array_equal(a.score(u, i), b.score(u, i))
        assert len(b.score(0, 0)) == (1 if variant == "rc2pf" else int(g["num_items"]))
        assert np.array_equal(a.get_user_vectors(), b.get_user_vectors())
        assert np.array_equal(a.get_item_vectors(), b.get_item_vectors())


@needs_cornac
def test_fit_without_a_gpu_raises():
    import torch
    from cornac_b200 import B200Error, C2PF
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from test_c2pf_gpu import _dataset
    with contextlib.redirect_stdout(io.StringIO()), pytest.raises(B200Error):
        C2PF(k=1, max_iter=1).fit(_dataset(golden("c2pf_k1")))
