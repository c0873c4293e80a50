"""MTER without a GPU: the host data against the compiled reference's _build_data, the seeded streams against the
fixtures' draws, the C oracle of the fit against the reference's fixtures, the error cases, and glibc's expf formula
(the device's, restated here) against libm."""
import ctypes
import ctypes.util
import sys

import numpy as np
import pytest

from conftest import GOLDEN, golden, needs_cornac
from oracle import mter_oracle as MO

PARAMS = MO.PARAMS
CASES = ("mter_default", "mter_odd", "mter_ties", "mter_exact")
DATA = ("X", "X_uids", "X_iids", "X_aids", "YU", "YU_uids", "YU_aids", "YU_oids", "YI", "YI_iids", "YI_aids", "YI_oids",
        "indptr", "indices")
# After one iteration the oracle equals the compiled reference bit for bit on every fixture.  Over more iterations it
# does not: the largest |oracle - reference| / max|reference| per parameter array over every fixture and max_iter (up
# to 10) is 3.3e-7 (mter_default, I after 3 iterations), measured on x86-64.  Pinned with a 6x margin.
ORACLE_BOUND = 2e-6


def fixture_helpers():
    sys.path.insert(0, GOLDEN)
    try:
        import make_golden_efm
        import make_golden_mter
    finally:
        sys.path.remove(GOLDEN)
    return make_golden_efm, make_golden_mter


def fixture_data(g):
    """MterData of a fixture, from the reference's own arrays (the pair ratings from the train set's triples)."""
    from types import SimpleNamespace
    n_items = int(g["num_items"])
    pair = g["ts_u"].astype(np.int64) * n_items + g["ts_i"]
    _, last_rev = np.unique(pair[::-1], return_index=True)
    pr = g["ts_r"][len(pair) - 1 - last_rev].astype(np.float32)
    uid = np.repeat(np.arange(int(g["num_users"])), np.diff(g["indptr"])).astype(np.int32)
    return SimpleNamespace(n_users=int(g["num_users"]), n_items=n_items, n_aspects=int(g["num_aspects"]),
                           n_opinions=int(g["num_opinions"]), user_ids=uid, pair_rating=pr,
                           **{k: g[k] for k in DATA})


def draws(g, n_iter):
    ne, nb = int(g["n_element_samples"]), int(g["n_bpr_samples"])
    return [g["draws_" + t][: n_iter * n] for t, n in (("uia", ne), ("uao", ne), ("iao", ne), ("pos", nb), ("neg", nb))]


def hyper(g):
    return dict(lr=float(g["lr"]), lambda_reg=float(g["lambda_reg"]), lambda_bpr=float(g["lambda_bpr"]))


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference(case):
    g = golden(case)
    data = fixture_data(g)
    for mi in g["max_iters"]:
        params = {p: g[p + "0"].copy() for p in PARAMS}
        sgrad = {p: np.zeros_like(x) for p, x in params.items()}
        MO.fit(data, params, sgrad, draws(g, int(mi)), int(mi), **hyper(g))
        for p in PARAMS:
            want = g["%s_%d" % (p, mi)]
            if mi == 1:
                assert np.array_equal(params[p], want), (case, mi, p)
            else:
                err = np.max(np.abs(params[p] - want)) / np.max(np.abs(want))
                assert err <= ORACLE_BOUND, (case, mi, p, err)


def test_oracle_split_calls_equal_one_call():
    g = golden("mter_odd")
    data = fixture_data(g)
    one = {p: g[p + "0"].copy() for p in PARAMS}
    s_one = {p: np.zeros_like(x) for p, x in one.items()}
    MO.fit(data, one, s_one, draws(g, 4), 4, **hyper(g))
    two = {p: g[p + "0"].copy() for p in PARAMS}
    s_two = {p: np.zeros_like(x) for p, x in two.items()}
    d4 = draws(g, 4)
    ne, nb = int(g["n_element_samples"]), int(g["n_bpr_samples"])
    MO.fit(data, two, s_two, [d[: 3 * (ne if k < 3 else nb)] for k, d in enumerate(d4)], 3, **hyper(g))
    MO.fit(data, two, s_two, [d[3 * (ne if k < 3 else nb):] for k, d in enumerate(d4)], 1, **hyper(g))
    for p in PARAMS:
        assert np.array_equal(one[p], two[p]) and np.array_equal(s_one[p], s_two[p]), p


@needs_cornac
@pytest.mark.parametrize("case", CASES)
def test_host_data_equals_reference(case):
    from cornac_b200.recom_mter import build_data
    efm, _ = fixture_helpers()
    g = golden(case)
    ts = efm.train_set(g)
    if "repeat_pairs" in g:
        ts.uir_tuple = (g["ts_u"], g["ts_i"], g["ts_r"])
    d = build_data(ts, int(g["num_users"]), int(g["num_items"]), float(g["rating_scale"]))
    for k in DATA:
        got = getattr(d, k)
        assert got.dtype == g[k].dtype and np.array_equal(got, g[k]), k
    ref = fixture_data(g)
    assert np.array_equal(d.pair_rating, ref.pair_rating) and np.array_equal(d.user_ids, ref.user_ids)


def test_repeated_pair_keeps_the_last_rating():
    g = golden("mter_ties")
    n = int(g["repeat_pairs"])
    data = fixture_data(g)
    # the first n pairs appear again at the end with another rating: the pair rating is the later one
    u, i, r = g["ts_u"], g["ts_i"], g["ts_r"]
    for t in range(n):
        pos = data.indptr[u[t]] + np.searchsorted(data.indices[data.indptr[u[t]]:data.indptr[u[t] + 1]], i[t])
        assert data.pair_rating[pos] == np.float32(r[len(r) - n + t]) != np.float32(r[t])


@needs_cornac
@pytest.mark.parametrize("case", CASES)
def test_streams_equal_the_fixture_draws(case):
    from cornac.utils import get_rng
    from cornac_b200 import engine
    from cornac_b200.recom_mter import stream_seeds
    g = golden(case)
    seeds = stream_seeds(get_rng(int(g["seed"])))
    assert seeds == g["stream_seeds"].tolist()
    n_iter = int(max(g["max_iters"]))
    his = [len(g["X"]) - 1, len(g["YU"]) - 1, len(g["YI"]) - 1, len(g["indices"]) - 1, int(g["num_items"]) - 1]
    for s, hi, want in zip(seeds, his, draws(g, n_iter)):
        assert np.array_equal(engine.MTSampler(s).fill(hi, len(want)), want)


@needs_cornac
def test_init_draws_and_untrainable_fit():
    from cornac_b200 import MTER
    efm, _ = fixture_helpers()
    g = golden("mter_default")
    hy = {k: g[k].item() for k in ("rating_scale", "n_user_factors", "n_item_factors", "n_aspect_factors",
                                    "n_opinion_factors", "n_bpr_samples", "n_element_samples")}
    m = MTER(max_iter=5, seed=int(g["seed"]), trainable=False, **hy).fit(efm.train_set(g))
    for p in PARAMS:
        assert np.array_equal(getattr(m, p), g["draw0_" + p]), p
    assert m.n_threads == 1 and m.num_aspects == int(g["num_aspects"]) and m.num_opinions == int(g["num_opinions"])


@needs_cornac
def test_empty_tensor_and_missing_modality_raise():
    from cornac.data import Dataset
    from cornac_b200 import MTER
    efm, _ = fixture_helpers()
    g = dict(golden("mter_odd"))
    g["tup_p"] = -np.abs(g["tup_p"])                       # no positive opinion: YU and YI are empty
    with pytest.raises(ValueError, match="user-aspect-opinion tensor YU"):
        MTER(max_iter=1, seed=1).fit(efm.train_set(g))
    ts = Dataset.from_uir([("a", "x", 1.0), ("b", "y", 2.0)], seed=1)
    with pytest.raises(ValueError, match="sentiment modality"):
        MTER(max_iter=1, seed=1).fit(ts)


def _expf_header():
    """The table and the constants of csrc/expf.cuh, read from the header itself."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(GOLDEN), "..", "cornac_b200", "csrc", "expf.cuh")).read()
    tab = re.search(r"EXPF_TAB\[32\] = \{(.*?)\};", src, re.S).group(1)
    tab = np.array([int(h, 16) for h in re.findall(r"0x([0-9a-f]+)ull", tab)], dtype=np.uint64)
    body = src[src.index("pmf_expf(float x)"):src.index("glibc_expf(float x)")]
    hexf = lambda name: float.fromhex(re.search(name + r" = (0x[0-9a-fp.+-]+)", body).group(1))    # noqa: E731
    c0 = float.fromhex(re.search(r"C0 = (0x[0-9a-fp.+-]+) / 32 / 32 / 32", body).group(1)) / 32 / 32 / 32
    c1 = float.fromhex(re.search(r"C1 = (0x[0-9a-fp.+-]+) / 32 / 32", body).group(1)) / 32 / 32
    c2 = float.fromhex(re.search(r"C2 = (0x[0-9a-fp.+-]+) / 32", body).group(1)) / 32
    inv = float.fromhex(re.search(r"INV_LN2_N = (0x[0-9a-fp.+-]+) \* 32", body).group(1)) * 32
    glibc = src[src.index("glibc_expf(float x)"):]
    hi = float.fromhex(re.search(r"x > (0x[0-9a-fp.+-]+)f", glibc).group(1))
    lo = -float.fromhex(re.search(r"x < -(0x[0-9a-fp.+-]+)f", glibc).group(1))
    return tab, inv, hexf("SHIFT"), c0, c1, c2, hi, lo


def _expf_formula(x):
    """expf.cuh's glibc_expf in numpy f64 with the header's own table and constants (IEEE f64 steps, no FMA)."""
    tab_bits, inv, shift, c0, c1, c2, hi, lo = _expf_header()
    x = np.asarray(x, dtype=np.float32)
    z = np.float64(inv) * x.astype(np.float64)
    kd = z + np.float64(shift)
    ki = kd.view(np.uint64)
    kd = kd - np.float64(shift)
    r = z - kd
    s = (tab_bits[ki % np.uint64(32)] + (ki << np.uint64(47))).view(np.float64)
    p = c0 * r + c1
    r2 = r * r
    y = c2 * r + 1.0
    y = p * r2 + y
    with np.errstate(over="ignore"):
        out = (y * s).astype(np.float32)
    out[x > np.float32(hi)] = np.inf
    out[x < np.float32(lo)] = 0
    return out


def test_device_expf_formula_matches_libm():
    """The arguments MTER's BPR weight reaches are differences of two scores; every f32 in [-110, 90] of a dense
    sample, and the range edges, must give libm's expf bit for bit through the header's table and constants."""
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.expf.restype, libm.expf.argtypes = ctypes.c_float, [ctypes.c_float]
    rng = np.random.RandomState(0)
    xs = np.concatenate([rng.uniform(-110, 90, 200000), np.linspace(-1, 1, 20001),
                         [float.fromhex("0x1.62e42ep6"), np.nextafter(np.float32(float.fromhex("0x1.62e42ep6")), np.float32(100)), -float.fromhex("0x1.9fe368p6"),
                          np.nextafter(np.float32(-float.fromhex("0x1.9fe368p6")), np.float32(-200)), -87.5, -100.0, 0.0]]
                        ).astype(np.float32)
    want = np.array([libm.expf(float(v)) for v in xs], dtype=np.float32)
    got = _expf_formula(xs)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
