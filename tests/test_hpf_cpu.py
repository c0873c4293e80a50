"""HPF / PF without a GPU: the C oracle against the compiled reference's fixtures, the oracle's stored-entry rules and
digamma, and the plug-in's constructor, init_params and score contracts."""
import numpy as np
import pytest
import scipy.special

from conftest import golden, needs_cornac
from oracle import hpf_oracle as HO

FIT_CASES = ["hpf_k5", "pf_k5", "hpf_k1", "pf_k1", "hpf_k10", "pf_k10", "hpf_k37", "pf_k37", "hpf_warm_k6", "pf_warm_k6",
             "hpf_nonpos_k4", "pf_nonpos_k4"]
KEYS = ("Gs", "Gr", "Ls", "Lr", "Theta", "Beta")


def rel_max(got, want):
    return float(np.max(np.abs(got - want)) / np.max(np.abs(want)))


def oracle_fit(g, m):
    X = HO.csc(g["rid"], g["cid"], g["val"], int(g["num_users"]), int(g["num_items"]))
    st = [g[x + "0"].copy() for x in ("Gs", "Gr", "Ls", "Lr")]
    Kr, Tr = np.ones(len(st[0])), np.ones(len(st[2]))
    HO.fit(bool(g["hierarchical"]), X, *st, Kr, Tr, m)
    return dict(zip(KEYS, st + [st[0] / st[1], st[2] / st[3]]))


@pytest.mark.parametrize("name", FIT_CASES)
def test_oracle_matches_the_reference(name):
    g = golden(name)
    for m in g["iters"]:
        got = oracle_fit(g, int(m))
        for key in KEYS:
            assert rel_max(got[key], g["%s_%d" % (key, m)]) <= 1e-12, (m, key)


def test_fixtures_cover_the_cases():
    ks = {int(golden(n)["k"]) for n in FIT_CASES}
    assert {1, 5, 10, 37} <= ks
    assert {bool(golden(n)["hierarchical"]) for n in FIT_CASES} == {True, False}
    assert {1, 10, 100} <= {int(m) for n in FIT_CASES for m in golden(n)["iters"]}
    for name in ("hpf_nonpos_k4", "pf_nonpos_k4"):
        g = golden(name)
        for s, r in ((g["Gs0"], g["Gr0"]), (g["Ls0"], g["Lr0"])):
            assert np.any((s <= 0) & (r > 0)) and np.any((s > 0) & (r <= 0)) and np.any((s <= 0) & (r <= 0))
    g = golden("hpf_k5")
    assert bool(g["seeded"]) and int(g["seed"]) == 7


def test_oracle_split_fit_equals_one_fit():
    g = golden("hpf_k10")
    X = HO.csc(g["rid"], g["cid"], g["val"], int(g["num_users"]), int(g["num_items"]))
    one = [g[x + "0"].copy() for x in ("Gs", "Gr", "Ls", "Lr")] + [np.ones(int(g["num_users"])), np.ones(int(g["num_items"]))]
    two = [x.copy() for x in one]
    HO.fit(True, X, *one, 7)
    HO.fit(True, X, *two, 3)
    HO.fit(True, X, *two, 4)
    for a, b in zip(one, two):
        assert np.array_equal(a, b)


def test_oracle_stored_entry_rules():
    s = np.array([0.7, 0.0, -1.0, 0.7, 0.0, -2.0, np.nan, 2.5])
    r = np.array([1.3, 1.3, 0.4, 0.0, -1.0, 0.0, 1.3, np.nan])
    e = HO.expect(s, r)
    dg, lg = scipy.special.digamma, np.log
    want = [np.exp(dg(0.7) - lg(1.3)), np.exp(-lg(1.3)), np.exp(-lg(0.4)), np.exp(dg(0.7)), 0.0, 0.0, np.exp(-lg(1.3)),
            np.exp(dg(2.5))]
    assert np.all(np.abs(e - want) <= 1e-14 * np.abs(want))
    assert e[4] == 0.0 and e[5] == 0.0


def test_oracle_digamma_is_accurate():
    x = np.concatenate([np.geomspace(1e-3, 1e6, 400), [0.3, 1.0, 1.4616321449683622, 10.0, 100.0]])
    got = HO.digamma(x)
    want = scipy.special.digamma(x)
    # a few ulps: absolute where |psi| < 1 (around the root at 1.46, where the recurrence's sum cancels), relative elsewhere
    assert np.all(np.abs(got - want) <= 8 * np.finfo(float).eps * np.maximum(np.abs(want), 1.0))


@needs_cornac
def test_constructor_contract_matches_the_reference():
    from cornac.models import HPF as RefHPF
    from cornac_b200 import HPF
    attrs = ("name", "k", "max_iter", "trainable", "verbose", "hierarchical", "seed", "init_params", "eps", "Theta",
             "Beta", "Gs", "Gr", "Ls", "Lr")
    for kw in ({}, dict(k=3, max_iter=7), dict(hierarchical=False, name="PF", seed=3), dict(trainable=False, verbose=True)):
        a, b = RefHPF(**kw), HPF(**kw)
        for attr in attrs:
            assert getattr(a, attr) == getattr(b, attr), (kw, attr)
        for attr in ("ll", "etp_r", "etp_c"):
            assert np.array_equal(getattr(a, attr), getattr(b, attr)) and getattr(a, attr).dtype == getattr(b, attr).dtype
    c = HPF(k=4, seed=5, hierarchical=False).clone()
    assert isinstance(c, HPF) and c.k == 4 and c.seed == 5 and not c.hierarchical
    c = HPF(k=4).clone(dict(k=6, max_iter=3))
    assert c.k == 6 and c.max_iter == 3 and len(c.ll) == 3


def _dataset(g):
    from cornac.data import Dataset
    return Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])], seed=None)


@needs_cornac
def test_initial_state_is_the_reference_draw():
    from cornac_b200 import HPF
    for name in ("hpf_k5", "pf_k5"):
        g = golden(name)
        m = HPF(k=int(g["k"]), hierarchical=bool(g["hierarchical"]), seed=int(g["seed"]))
        st = m._init_state(int(g["num_users"]), int(g["num_items"]))
        for a, key in zip(st, ("Gs0", "Gr0", "Ls0", "Lr0")):
            assert np.array_equal(a, g[key]), (name, key)


@needs_cornac
def test_init_params_are_validated():
    from cornac_b200 import HPF
    g = golden("hpf_k1")
    ds = _dataset(g)
    n, d = ds.num_users, ds.num_items
    for bad, match in (({"G_s": np.ones((n, 1), np.float32)}, "float64"), ({"L_r": np.ones((d + 1, 1))}, "shape"),
                       ({"G_r": np.ones((n, 2))}, "shape"), ({"L_s": np.ones(d)}, "shape")):
        with pytest.raises(ValueError, match=match):
            HPF(k=1, max_iter=1, init_params=bad).fit(ds)


@needs_cornac
def test_score_exceptions_and_single_scores_without_a_gpu():
    from cornac.exception import ScoreException
    from cornac_b200 import HPF
    g = golden("hpf_k5")
    ds = _dataset(g)
    Theta, Beta = g["Theta_100"], g["Beta_100"]
    m = HPF(k=5, trainable=False, init_params={"Theta": Theta, "Beta": Beta}).fit(ds)
    with pytest.raises(ScoreException, match="Can't make score prediction for user %d" % ds.num_users):
        m.score(ds.num_users)
    with pytest.raises(ScoreException, match="Can't make score prediction for item %d" % ds.num_items):
        m.score(0, ds.num_items)
    for u, i in ((0, 0), (3, 17), (ds.num_users - 1, ds.num_items - 1)):
        s = m.score(u, i)
        assert type(s) is np.float64 and s == np.array(Beta[i, :].dot(Theta[u, :]), dtype="float64").flatten()[0]
    assert m.get_user_vectors() is Theta and m.get_item_vectors() is Beta
