"""NMF without a GPU: the C oracle against the compiled reference's fixtures, the CSC position map, the bias schedule, and
the plug-in's constructor contract."""
import numpy as np
import pytest

from conftest import golden, needs_cornac, synth_csr
from oracle import nmf_oracle as NO

FIT_CASES = ["nmf_default_k15", "nmf_bias_k10", "nmf_lambda_reg_k8", "nmf_init_u_bi_k6", "nmf_k1", "nmf_bias_k1",
             "nmf_mid_k12"]


def hyper(g):
    return dict(mu=float(g["mu"]), lr=float(g["learning_rate"]), lambda_u=float(g["lambda_u"]),
                lambda_v=float(g["lambda_v"]), lambda_bu=float(g["lambda_bu"]), lambda_bi=float(g["lambda_bi"]),
                use_bias=bool(g["use_bias"]))


@pytest.mark.parametrize("name", FIT_CASES)
def test_oracle_is_bit_identical_to_the_reference(name):
    g = golden(name)
    U, V, Bu, Bi = (g[x].copy() for x in ("U0", "V0", "Bu0", "Bi0"))
    NO.nmf_fit(g["indptr"], g["indices"], g["data"], U, V, Bu, Bi, int(g["max_iter"]), **hyper(g))
    for got, key in ((U, "U"), (V, "V"), (Bu, "Bu"), (Bi, "Bi")):
        assert np.array_equal(got, g[key]), key


def test_fixtures_cover_the_cases():
    assert int(golden("nmf_default_k15")["k"]) == 15 and int(golden("nmf_default_k15")["max_iter"]) == 50
    g = golden("nmf_init_u_bi_k6")                 # Bi given and non-zero, not trained: it enters the prediction only
    assert not bool(g["use_bias"]) and np.any(g["Bi0"] != 0) and np.array_equal(g["Bi"], g["Bi0"])
    g = golden("nmf_lambda_reg_k8")
    assert float(g["lambda_u"]) == float(g["lambda_bi"]) == float(g["lambda_reg"]) == 0.03
    assert bool(golden("nmf_bias_k10")["use_bias"]) and float(golden("nmf_bias_k10")["mu"]) != 0.0
    assert int(golden("nmf_k1")["k"]) == 1


@pytest.mark.parametrize("shape", [(1, 1, 1), (30, 20, 300), (943, 1682, 20000)])
def test_b200_csc_map_is_a_stable_permutation(shape):
    from cornac_b200 import engine
    n_users, n_items, nnz = shape
    indptr, indices = synth_csr(n_users, n_items, nnz, seed=nnz)
    csc_ptr, csc_pos = engine.csc_map(indptr, indices, n_items)
    n = len(indices)
    assert np.array_equal(np.sort(csc_pos), np.arange(n))
    assert np.array_equal(np.diff(csc_ptr), np.bincount(indices, minlength=n_items))
    for i in range(n_items):
        col = csc_pos[csc_ptr[i]:csc_ptr[i + 1]]
        assert np.all(indices[col] == i) and np.all(np.diff(col) > 0)
    assert np.array_equal(csc_pos, np.argsort(indices, kind="stable"))
    deg = np.diff(csc_ptr)
    item_order = engine.longest_first(deg)
    assert item_order.dtype == np.int32 and np.array_equal(item_order, np.lexsort((np.arange(n_items), -deg)))


def test_csc_map_rejects_bad_input():
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    with pytest.raises(B200Error, match="outside"):
        engine.csc_map(np.array([0, 2]), np.array([0, 3]), 3)
    with pytest.raises(B200Error, match="indptr"):
        engine.csc_map(np.array([0, 3]), np.array([0, 1]), 3)
    with pytest.raises(B200Error, match="decreases"):
        engine.csc_map(np.array([0, 2, 1, 2]), np.array([0, 1]), 3)
    ptr_, pos = engine.csc_map(np.zeros(1), np.zeros(0), 0)
    order = engine.longest_first(np.diff(ptr_))
    assert list(ptr_) == [0] and len(pos) == 0 and len(order) == 0


def test_bias_pass_uses_the_pmf_schedule_of_the_csr_order():
    """The biased rating pass runs over b200_pmf_schedule of (user, item) in stored order: on the ML-100K shape it has
    the level count of the Python recurrence."""
    from cornac_b200 import engine
    indptr, indices = synth_csr(943, 1682, 100000, seed=3)
    uid = np.repeat(np.arange(943), np.diff(indptr)).astype(np.int32)
    order, level_ptr = engine.pmf_schedule(uid, indices, 943, 1682)
    last_u, last_i, top = np.zeros(943, np.int64), np.zeros(1682, np.int64), 0
    for u, i in zip(uid.tolist(), indices.tolist()):
        lv = max(last_u[u], last_i[i]) + 1
        last_u[u] = last_i[i] = lv
        top = max(top, lv)
    assert len(level_ptr) - 1 == top
    assert np.array_equal(np.sort(order), np.arange(len(uid)))


@needs_cornac
def test_constructor_contract_matches_the_reference():
    from cornac.models import NMF as RefNMF
    from cornac_b200 import NMF
    attrs = ("name", "k", "max_iter", "learning_rate", "lambda_reg", "lambda_u", "lambda_v", "lambda_bu", "lambda_bi",
             "use_bias", "num_threads", "trainable", "verbose", "seed", "init_params", "u_factors", "i_factors",
             "u_biases", "i_biases", "global_mean")
    for kw in ({}, dict(lambda_reg=0.1), dict(lambda_reg=0.1, lambda_u=0.5), dict(seed=3), dict(num_threads=1),
               dict(num_threads=10 ** 6), dict(k=4, use_bias=True, init_params={"mu": 2.0})):
        a, b = RefNMF(**kw), NMF(**kw)
        for attr in attrs:
            assert getattr(a, attr) == getattr(b, attr), (kw, attr)
    c = NMF(k=4, lambda_reg=0.2, seed=5, use_bias=True).clone()
    assert isinstance(c, NMF) and c.k == 4 and c.lambda_u == 0.2 and c.num_threads == 1 and c.use_bias
    c = NMF(k=4).clone(dict(k=6))
    assert c.k == 6
