"""LRPPM host checks: build_data against the compiled reference's arrays, the serial oracle against the reference's
fits (tests/golden/lrppm_*.npz, from tests/golden/make_golden_lrppm.py), the key, isclose and rank restatements."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(GOLDEN))

from oracle import lrppm_oracle as LO  # noqa: E402

CASES = ["lrppm_default", "lrppm_k1", "lrppm_k3", "lrppm_k5", "lrppm_collide", "lrppm_norating", "lrppm_nan",
         "lrppm_converge"]
PARAMS = ("U", "I", "UA", "IA")


def load(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))


def case_data(g):
    """The plug-in's build_data of a fixture's train set."""
    from make_golden_efm import train_set
    from cornac_b200.recom_lrppm import build_data
    ts = train_set(g)
    ts.uir_tuple = (g["ts_u"], g["ts_i"], g["ts_r"])
    return build_data(ts, int(g["num_users"]), int(g["num_items"]))


def draws(g, n):
    """The stored draws of n iterations; past the ones stored (the reference stopped there) zeros, never read."""
    n_s, n_r = int(g["n_samples"]), int(g["n_ranking_samples"])
    pad = lambda x, m: np.concatenate([x[:m], np.zeros(max(0, m - len(x)), np.int64)])      # noqa: E731
    return pad(g["draws_pos"], n * n_s), pad(g["draws_pos_uia"], n * n_r), pad(g["draws_neg_uia"], n * n_r)


@pytest.mark.parametrize("name", CASES)
def test_build_data_equals_reference(name):
    g = load(name)
    d = case_data(g)
    for f in ("X_uids", "X_iids", "X_aids"):
        assert np.array_equal(getattr(d, f), g["ref_" + f]), f
    assert np.array_equal(d.X_values, g["ref_X_values"])
    assert np.array_equal(d.X_l_ui, g["ref_X_l_ui"])
    assert np.array_equal(d.rating_keys, g["ref_rating_keys"])
    assert np.array_equal(d.rating_values, g["ref_rating_values"].astype(np.float32))
    assert np.array_equal(d.aspect_keys, g["ref_aspect_keys"])
    Q = d.item_aspect_quality
    assert np.array_equal(Q.indptr, g["Q_indptr"]) and np.array_equal(Q.indices, g["Q_indices"])
    assert np.array_equal(Q.data, g["Q_data"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_reference(name):
    """Bit for bit at every stored max_iter, including the iteration at which the reference stops."""
    g = load(name)
    d = case_data(g)
    hyper = dict(lr=float(g["lr"]), reg=float(g["reg"]), ld=float(g["ld"]))
    for mi in g["max_iters"]:
        params = {p: g[p + "0"].copy() for p in PARAMS}
        ran, conv, *_ = LO.fit(d, params, draws(g, int(mi)), int(mi), int(g["n_samples"]), int(g["n_ranking_samples"]),
                               **hyper)
        assert ran == int(g["calls_%d" % mi]) and conv == bool(g["converged_%d" % mi]), (mi, ran, conv)
        for p in PARAMS:
            want = g["%s_%d" % (p, mi)]
            assert np.array_equal(params[p].view(np.uint32), want.view(np.uint32)), (mi, p)


def test_converge_fixture_stops_after_the_first_iteration():
    g = load("lrppm_converge")
    assert bool(g["converged_60"]) and 1 < int(g["calls_60"]) < 60


def test_keys_equal_the_reference_on_the_collision_fixture():
    """The wrapped keys of the triples (the fixture's keys pass 2^31 and wrap) are the reference's dict keys."""
    g = load("lrppm_collide")
    d = case_data(g)
    k1 = LO.get_key(d.X_uids, d.X_iids)
    k3 = LO.get_key(k1, d.X_aids)
    assert np.array_equal(np.unique(k3), g["ref_aspect_keys"])
    from cornac_b200.recom_lrppm import get_key3
    assert np.array_equal(get_key3(d.X_uids, d.X_iids, d.X_aids), k3)
    assert np.any(k3 < 0)


def test_norating_fixture_has_review_pairs_without_rating():
    g = load("lrppm_norating")
    d = case_data(g)
    k = LO.get_key(d.X_uids, d.X_iids)
    assert not np.all(np.isin(k, d.rating_keys))


def test_isclose_equals_numpy():
    rng = np.random.RandomState(0)
    y = np.concatenate([rng.uniform(-3, 3, 200), [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-8, 1.0, 1e30, 1e-40]])
    y = y.astype(np.float32)
    tol = (np.float32(1e-8) + np.float32(1e-5) * np.abs(y)).astype(np.float32)
    xs = [y, y + tol, y - tol, np.nextafter(y + tol, np.float32(np.inf)), np.nextafter(y - tol, np.float32(-np.inf)),
          -y, np.zeros_like(y), np.full_like(y, np.nan), np.full_like(y, np.inf), np.full_like(y, -0.0)]
    for x in xs:
        x = x.astype(np.float32)
        with np.errstate(all="ignore"):
            assert np.array_equal(LO.isclose(x, y), np.isclose(x, y))
            assert np.array_equal(LO.isclose(y, x), np.isclose(y, x))


@pytest.mark.parametrize("name", ["lrppm_default", "lrppm_k5", "lrppm_norating"])
def test_rank_restatement_equals_reference(name):
    """The reference's rank rows (with `.A` read as `.toarray()`) from the fixture's last fit."""
    g = load(name)
    mi = int(g["max_iters"][-1])
    U, I, UA, IA = (g["%s_%d" % (p, mi)] for p in PARAMS)
    Q = sp.csr_matrix((g["Q_data"], g["Q_indices"], g["Q_indptr"]), shape=(int(g["num_items"]), int(g["num_aspects"])))
    n_top = min(int(g["num_top_aspects"]), int(g["num_aspects"]))
    alpha, scale = float(g["alpha"]), float(g["rating_scale"])
    for row, u in enumerate(g["rank_users"]):
        s = UA.dot(U[u]) + I.dot(IA.T) + np.expand_dims(I.dot(U[u]), axis=1)
        srt = -np.sort(-s, axis=1)
        no_tie = np.ones(len(s), bool) if n_top >= s.shape[1] else srt[:, n_top - 1] != srt[:, n_top]
        assert no_tie.mean() > 0.5
        want = LO.rank_rows(s, Q.toarray(), n_top, alpha, scale, I.dot(U[u]))[no_tie]
        got = g["rank_scores"][row][: len(no_tie)][no_tie]
        assert np.all(np.abs(want - got) <= 1e-12 * np.maximum(1.0, np.abs(got))), name


def test_plugin_refuses_a_pair_that_mentions_every_aspect():
    """The reference divides by zero there: the plug-in raises the same error before any device work."""
    from cornac.data import Dataset, SentimentModality
    from cornac_b200 import LRPPM
    data = [("u0", "i0", 4.0), ("u0", "i1", 3.0), ("u1", "i0", 5.0)]
    ts = Dataset.from_uir(data, seed=1)
    md = SentimentModality(data=[("u0", "i0", [("a0", "o", 1.0), ("a1", "o", -1.0)]), ("u1", "i0", [("a0", "o", 1.0)])])
    md.build(uid_map=ts.uid_map, iid_map=ts.iid_map, dok_matrix=ts.dok_matrix)
    ts.add_modalities(sentiment=md)
    with pytest.raises(ZeroDivisionError):
        LRPPM(max_iter=1, seed=1).fit(ts)


def test_plugin_refuses_f64_params():
    from cornac_b200.recom_lrppm import LRPPM
    m = LRPPM(init_params={"U": np.zeros((2, 8))})
    m.num_users, m.num_items, m.num_aspects = 2, 1, 1
    m.I, m.UA, m.IA = (np.zeros(s, np.float32) for s in ((1, 8), (1, 8), (1, 8)))
    with pytest.raises(ValueError, match="Buffer dtype mismatch"):
        m._check_params()
