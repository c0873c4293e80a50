"""PMF without a GPU: the C oracle against the compiled reference's fixtures, the level schedule, and the plug-in's
argument checks (which run before any device work)."""
import numpy as np
import pytest

from conftest import golden, needs_cornac
from oracle import pmf_oracle as PO

FIT_CASES = ["pmf_linear_k5", "pmf_linear_k10_mid", "pmf_nonlinear_k10", "pmf_nonlinear_unit", "pmf_linear_init_u_k7",
             "pmf_nonlinear_k1", "pmf_linear_k1"]


def oracle_fit(g, terms=False):
    U, V = g["U0"].copy(), g["V0"].copy()
    out = PO.pmf_fit(str(g["variant"]), g["uid"], g["iid"], g["rat"], U, V, int(g["max_iter"]), float(g["lambda_reg"]),
                     float(g["learning_rate"]), float(g["gamma"]), terms=terms)
    return U, V, out


@pytest.mark.parametrize("name", FIT_CASES)
def test_oracle_is_bit_identical_to_the_reference(name):
    g = golden(name)
    U, V, loss = oracle_fit(g)
    assert np.array_equal(U, g["U"]) and np.array_equal(V, g["V"])
    assert np.array_equal(loss, g["loss"])


def test_oracle_loss_terms_sum_to_the_epoch_loss():
    g = golden("pmf_nonlinear_k10")
    _, _, (loss, terms) = oracle_fit(g, terms=True)
    assert np.array_equal(np.add.accumulate(terms, axis=1)[:, -1], loss)
    assert np.array_equal(loss, g["loss"])


def test_fixtures_cover_the_scale_branch():
    g = golden("pmf_nonlinear_unit")
    assert [float(g["min_rating"]), float(g["max_rating"])] == [0.0, 1.0]
    assert np.array_equal(np.sort(g["rat"]), np.sort(g["uir_r"].astype(np.float32)))    # passed through unscaled
    g = golden("pmf_nonlinear_k10")
    assert float(g["rat"].min()) == 0.0 and float(g["rat"].max()) == 1.0      # 1..5 mapped onto [0, 1]


def _levels_python(uid, iid):
    last_u, last_i, lv = {}, {}, []
    for u, i in zip(uid.tolist(), iid.tolist()):
        x = max(last_u.get(u, 0), last_i.get(i, 0)) + 1
        last_u[u] = last_i[i] = x
        lv.append(x)
    return np.array(lv, dtype=np.int64)


def _random_ratings(rng, n_users, n_items, nnz):
    key = rng.choice(n_users * n_items, size=nnz, replace=False)
    return (key // n_items).astype(np.int32), (key % n_items).astype(np.int32)


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 50, 40), (50, 1, 40), (30, 20, 300), (200, 150, 5000)])
def test_schedule_is_a_row_disjoint_permutation_in_stored_order(shape):
    from cornac_b200 import engine
    n_users, n_items, nnz = shape
    uid, iid = _random_ratings(np.random.RandomState(nnz), n_users, n_items, nnz)
    order, level_ptr = engine.pmf_schedule(uid, iid, n_users, n_items)
    assert np.array_equal(np.sort(order), np.arange(nnz))
    assert level_ptr[0] == 0 and level_ptr[-1] == nnz and np.all(np.diff(level_ptr) > 0)
    level_of = np.empty(nnz, dtype=np.int64)
    for l in range(len(level_ptr) - 1):
        s = order[level_ptr[l]:level_ptr[l + 1]]
        assert np.all(np.diff(s) > 0)                                  # stored order inside a level
        assert len(np.unique(uid[s])) == len(s) and len(np.unique(iid[s])) == len(s)   # row-disjoint
        level_of[s] = l + 1
    # every pair sharing a row keeps its stored order: consecutive ratings of one row sit on increasing levels
    for ids in (uid, iid):
        by_row = np.lexsort((np.arange(nnz), ids))
        same = ids[by_row][1:] == ids[by_row][:-1]
        assert np.all(level_of[by_row][1:][same] > level_of[by_row][:-1][same])
    assert np.array_equal(level_of, _levels_python(uid, iid))


def test_schedule_of_a_fixture_and_bad_ids():
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    g = golden("pmf_linear_k10_mid")
    order, level_ptr = engine.pmf_schedule(g["uid"], g["iid"], int(g["num_users"]), int(g["num_items"]))
    lv = _levels_python(g["uid"], g["iid"])
    assert len(level_ptr) - 1 == lv.max()
    assert np.array_equal(np.diff(level_ptr), np.bincount(lv)[1:])
    with pytest.raises(B200Error, match="outside"):
        engine.pmf_schedule(np.array([0, 3]), np.array([0, 0]), 3, 1)
    o, lp = engine.pmf_schedule(np.zeros(0), np.zeros(0), 0, 0)
    assert len(o) == 0 and list(lp) == [0]


@needs_cornac
def test_plugin_validates_like_the_reference_before_touching_the_device():
    from cornac.models import PMF as RefPMF
    from cornac_b200 import PMF
    g = golden("pmf_linear_k5")
    ds = _dataset(g)
    # an unknown variant raises only when the model is trained
    for cls in (RefPMF, PMF):
        with pytest.raises(ValueError, match="variant must be one of"):
            cls(k=3, max_iter=1, variant="nope").fit(ds)
        m = cls(k=3, max_iter=1, variant="nope", trainable=False,
                init_params={"U": np.zeros((ds.num_users, 3)), "V": np.zeros((ds.num_items, 3))}).fit(ds)
        assert m.variant == "nope"
    # f32 init_params: the reference's memoryview refuses them with a ValueError
    for cls in (RefPMF, PMF):
        with pytest.raises(ValueError):
            cls(k=3, max_iter=1, variant="linear", init_params={"U": np.zeros((ds.num_users, 3), np.float32)}).fit(ds)
    # defaults and attributes
    a, b = RefPMF(), PMF()
    for attr in ("k", "max_iter", "learning_rate", "gamma", "lambda_reg", "name", "variant", "trainable", "verbose", "seed",
                 "eps", "init_params", "U", "V"):
        assert getattr(a, attr) == getattr(b, attr), attr
    assert np.array_equal(a.ll, b.ll)


def _dataset(g):
    from cornac.data import Dataset
    return Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])], seed=None)
