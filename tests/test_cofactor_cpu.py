"""SoRec and MCF without a GPU: the C oracle against the compiled reference's fixtures, the mixed edge + rating level
schedule, PMF's schedule through the shared routine, the link weights, and the plug-ins' argument checks (which run
before any device work)."""
import math

import numpy as np
import pytest

from conftest import golden, needs_cornac
from oracle import cofactor_oracle as CO

SOREC_CASES = ["sorec_k5", "sorec_nolink_k10", "sorec_k1", "sorec_k37", "sorec_step_product", "sorec_minmax",
               "sorec_loops_dups", "sorec_empty_graph", "sorec_warm_k6"]
MCF_CASES = ["mcf_k5", "mcf_unit_k10", "mcf_const_k1", "mcf_warm_k37"]
FIT_CASES = SOREC_CASES + MCF_CASES


def oracle_fit(g, terms=False):
    U, V, Z = g["U0"].copy(), g["V0"].copy(), g["Z0"].copy()
    out = CO.fit(str(g["model"]), g["net_a"], g["net_b"], g["net_val"], g["uid"], g["iid"], g["rat"], U, V, Z,
                 int(g["max_iter"]), float(g["lambda_c"]), float(g["lambda_reg"]), float(g["learning_rate"]),
                 float(g["gamma"]), terms=terms)
    return U, V, Z, out


@pytest.mark.parametrize("name", FIT_CASES)
def test_oracle_is_bit_identical_to_the_reference(name):
    g = golden(name)
    U, V, Z, loss = oracle_fit(g)
    assert np.array_equal(U, g["U"]) and np.array_equal(V, g["V"]) and np.array_equal(Z, g["Z"])
    assert np.array_equal(loss, g["loss"])


def test_oracle_loss_terms_sum_to_the_epoch_loss():
    g = golden("sorec_k5")
    _, _, _, (loss, terms) = oracle_fit(g, terms=True)
    assert terms.shape == (int(g["max_iter"]), len(g["net_a"]) + len(g["uid"]))
    assert np.array_equal(np.add.accumulate(terms, axis=1)[:, -1], g["loss"])


def test_fixtures_cover_the_reference_branches():
    g = golden("sorec_step_product")                          # the f32 step product differs from the f64 one
    lc, lr = np.float32(g["lambda_c"]), np.float32(g["learning_rate"])
    assert float(lc * lr) != float(lc) * float(lr)
    assert CO.lib().cofactor_sorec_step(float(lc), float(lr)) == float(lc * lr)
    assert not golden("sorec_nolink_k10")["weight_link"] and golden("sorec_k5")["weight_link"]
    assert np.all(golden("sorec_nolink_k10")["net_val"] == 1.0) and np.any(golden("sorec_k5")["net_val"] < 1.0)
    g = golden("sorec_minmax")                                # min == max: every rating scales to 1
    assert float(g["min_rating"]) == float(g["max_rating"]) and np.all(g["rat"] == 1.0)
    g = golden("sorec_loops_dups")
    pairs = list(zip(g["net_a"].tolist(), g["net_b"].tolist()))
    assert any(a == b for a, b in pairs) and len(set(pairs)) < len(pairs)
    assert len(golden("sorec_empty_graph")["net_a"]) == 0
    assert list(golden("sorec_warm_k6")["init_given"]) == ["U", "Z"]
    assert list(golden("mcf_warm_k37")["init_given"]) == ["V"]
    # MCF's edge values: [0, 1] passed through, a constant scaled onto 1, anything else min/max-scaled
    g = golden("mcf_unit_k10")
    assert np.array_equal(np.sort(g["net_val"]), np.sort(g["graph_val"].astype(np.float32)))
    assert np.all(golden("mcf_const_k1")["net_val"] == 1.0)
    g = golden("mcf_k5")
    assert g["graph_val"].min() > 0 and g["net_val"].min() == 0.0 and g["net_val"].max() == 1.0


# ---- schedules ------------------------------------------------------------------------------------------------------
def _python_levels(rows):
    """rows: list of (row_a, row_b) in one id space; the level rule, in plain Python."""
    last, lv = {}, []
    for a, b in rows:
        x = max(last.get(a, 0), last.get(b, 0)) + 1
        last[a] = last[b] = x
        lv.append(x)
    return np.array(lv, dtype=np.int64)


def _mixed_rows(variant, net_a, net_b, uid, iid):
    a_kind = "U" if variant == "sorec" else "V"
    return ([((a_kind, int(a)), ("Z", int(b))) for a, b in zip(net_a, net_b)]
            + [(("U", int(u)), ("V", int(i))) for u, i in zip(uid, iid)])


def check_cofactor_schedule(variant, net_a, net_b, uid, iid, n_users, n_items):
    from cornac_b200 import engine
    order, level_ptr = engine.cofactor_schedule(variant, net_a, net_b, uid, iid, n_users, n_items)
    rows = _mixed_rows(variant, net_a, net_b, uid, iid)
    n = len(rows)
    assert np.array_equal(np.sort(order), np.arange(n))                       # a permutation
    assert level_ptr[0] == 0 and level_ptr[-1] == n and np.all(np.diff(level_ptr) > 0)
    level_of = np.empty(n, dtype=np.int64)
    for l in range(len(level_ptr) - 1):
        s = order[level_ptr[l]:level_ptr[l + 1]]
        assert np.all(np.diff(s) > 0)                                          # stored order inside a level
        touched = [r for j in s for r in rows[j]]
        assert len(set(touched)) == len(touched)                               # disjoint rows
        level_of[s] = l + 1
    assert np.array_equal(level_of, _python_levels(rows))
    return order, level_ptr


def _random_stream(rng, variant, n_users, n_items, n_edges, n_ratings):
    n_nodes = n_users if variant == "sorec" else n_items
    net_a, net_b = rng.randint(n_nodes, size=n_edges), rng.randint(n_nodes, size=n_edges)   # loops and duplicates too
    key = rng.choice(n_users * n_items, size=n_ratings, replace=False)
    return net_a, net_b, key // n_items, key % n_items


@pytest.mark.parametrize("variant", ["sorec", "mcf"])
@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (5, 4, 0, 12), (5, 4, 9, 0), (30, 20, 200, 300), (200, 150, 1500, 4000)])
def test_mixed_schedule_is_a_row_disjoint_permutation_in_stored_order(variant, shape):
    n_users, n_items, n_edges, n_ratings = shape
    rng = np.random.RandomState(n_edges + 7 * n_ratings)
    check_cofactor_schedule(variant, *_random_stream(rng, variant, n_users, n_items, n_edges, n_ratings), n_users,
                            n_items)


@pytest.mark.parametrize("name", FIT_CASES)
def test_mixed_schedule_of_the_fixtures(name):
    g = golden(name)
    order, level_ptr = check_cofactor_schedule(str(g["model"]), g["net_a"], g["net_b"], g["uid"], g["iid"],
                                               int(g["num_users"]), int(g["num_items"]))
    # edges and ratings may share a level: never deeper than one level sequence per pass
    depth_edges = max(_python_levels(_mixed_rows(str(g["model"]), g["net_a"], g["net_b"], [], [])), default=0)
    depth_ratings = max(_python_levels(_mixed_rows(str(g["model"]), [], [], g["uid"], g["iid"])), default=0)
    assert len(level_ptr) - 1 <= depth_edges + depth_ratings


def test_mixed_schedule_rejects_bad_ids():
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    ok = dict(uid=np.array([0, 1]), iid=np.array([0, 0]), n_users=2, n_items=1)
    with pytest.raises(B200Error, match="outside"):                           # SoRec's edges join users
        engine.cofactor_schedule("sorec", np.array([0]), np.array([2]), **ok)
    with pytest.raises(B200Error, match="outside"):                           # MCF's edges join items
        engine.cofactor_schedule("mcf", np.array([1]), np.array([0]), **ok)
    with pytest.raises(B200Error, match="outside"):
        engine.cofactor_schedule("mcf", np.array([0]), np.array([0]), np.array([0, 2]), np.array([0, 0]), 2, 1)
    with pytest.raises(B200Error, match="variant"):
        engine.cofactor_schedule("pmf", np.array([0]), np.array([0]), **ok)
    engine.cofactor_schedule("sorec", np.array([0]), np.array([1]), **ok)
    engine.cofactor_schedule("mcf", np.array([0]), np.array([0]), **ok)
    o, lp = engine.cofactor_schedule("sorec", np.zeros(0), np.zeros(0), np.zeros(0), np.zeros(0), 0, 0)
    assert len(o) == 0 and list(lp) == [0]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_pmf_schedule_output_is_unchanged(seed):
    """b200_pmf_schedule through the shared level routine: the stable counting sort of the PMF level of each rating."""
    from cornac_b200 import engine
    rng = np.random.RandomState(seed)
    n_users, n_items = rng.randint(1, 60), rng.randint(1, 60)
    nnz = rng.randint(1, n_users * n_items + 1)
    key = rng.choice(n_users * n_items, size=nnz, replace=False)
    uid, iid = key // n_items, key % n_items
    order, level_ptr = engine.pmf_schedule(uid, iid, n_users, n_items)
    lv = _python_levels([(("U", int(u)), ("V", int(i))) for u, i in zip(uid, iid)])
    assert np.array_equal(order, np.argsort(lv, kind="stable"))
    assert np.array_equal(level_ptr, np.concatenate([[0], np.cumsum(np.bincount(lv)[1:])]))


# ---- plug-ins --------------------------------------------------------------------------------------------------------
def _dataset(g, with_graph=True):
    from cornac.data import Dataset, GraphModality
    ds = Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])], seed=None)
    if with_graph:
        sorec = str(g["model"]) == "sorec"
        gm = GraphModality(data=[(str(a), str(b), float(v)) for a, b, v in zip(g["graph_a"], g["graph_b"], g["graph_val"])])
        gm.build(id_map=ds.uid_map if sorec else ds.iid_map)
        ds.add_modalities(**{("user_graph" if sorec else "item_graph"): gm})
    return ds


@needs_cornac
@pytest.mark.parametrize("name", ["sorec_k5", "sorec_loops_dups", "sorec_warm_k6"])
def test_link_weights_equal_the_reference_loop_bit_for_bit(name):
    from cornac_b200.recom_sorec import link_weights
    g = golden(name)
    ds = _dataset(g)
    train = set(ds.uir_tuple[0])
    a, b, val = ds.user_graph.get_train_triplet(train, train)
    degree = ds.user_graph.get_node_degree(train, train)          # {node: [in, out]}
    want = np.array([math.sqrt(degree[int(j)][0] / (degree[int(j)][0] + degree[int(u)][1])) * v
                     for u, j, v in zip(a, b, val)])
    got = link_weights(a, b, val)
    assert got.dtype == np.float64 and np.array_equal(got.view(np.int64), want.view(np.int64))
    assert np.array_equal(got.astype(np.float32), g["net_val"])


@needs_cornac
def test_plugins_validate_like_the_reference_before_touching_the_device():
    from cornac.models import MCF as RefMCF, SoRec as RefSoRec
    from cornac_b200 import MCF, SoRec
    gs, gm = golden("sorec_k5"), golden("mcf_k5")
    ds_s, ds_m = _dataset(gs), _dataset(gm)
    # SoRec checks k in its constructor, with the reference's text
    for cls in (RefSoRec, SoRec):
        for key in ("U", "V", "Z"):
            with pytest.raises(ValueError, match="initial parameters %s dimension error" % key):
                cls(k=3, init_params={key: np.zeros((4, 2))})
    # a wrong dtype or shape is a ValueError before any device work (no device on this machine)
    for cls, ds, n_z in ((SoRec, ds_s, ds_s.num_users), (MCF, ds_m, ds_m.num_items)):
        with pytest.raises(ValueError, match="dtype"):
            cls(k=3, max_iter=1, init_params={"U": np.zeros((ds.num_users, 3), np.float32)}).fit(ds)
        with pytest.raises(ValueError, match="shape"):
            cls(k=3, max_iter=1, init_params={"Z": np.zeros((n_z - 1, 3))}).fit(ds)
    # the reference's memoryview refuses f32 init_params with a ValueError too
    for cls, ds in ((RefSoRec, ds_s), (RefMCF, ds_m)):
        with pytest.raises(ValueError):
            cls(k=3, max_iter=1, init_params={"U": np.zeros((ds.num_users, 3), np.float32)}).fit(ds)
    # a missing graph modality is a ValueError naming it (the reference raises AttributeError)
    with pytest.raises(ValueError, match="user_graph"):
        SoRec(k=3, max_iter=1).fit(_dataset(gs, with_graph=False))
    with pytest.raises(ValueError, match="item_graph"):
        MCF(k=3, max_iter=1).fit(_dataset(gm, with_graph=False))
    with pytest.raises(AttributeError):
        RefSoRec(k=3, max_iter=1).fit(_dataset(gs, with_graph=False))
    # trainable=False never touches the graph or the device
    SoRec(k=3, trainable=False).fit(_dataset(gs, with_graph=False))
    MCF(k=3, trainable=False).fit(_dataset(gm, with_graph=False))


@needs_cornac
def test_plugin_defaults_and_attributes_match_the_reference():
    from cornac.models import MCF as RefMCF, SoRec as RefSoRec
    from cornac_b200 import MCF, SoRec
    common = ("k", "max_iter", "learning_rate", "gamma", "name", "trainable", "verbose", "seed", "eps", "init_params", "U",
              "V", "Z")
    for (a, b), extra in (((RefSoRec(), SoRec()), ("lambda_c", "lambda_reg", "weight_link")),
                          ((RefMCF(), MCF()), ("lamda",))):
        for attr in common + extra:
            assert getattr(a, attr) == getattr(b, attr), attr
        assert np.array_equal(a.ll, b.ll)
