"""Host-side product logic and the C-ABI surface.  CPU only: no kernel is launched."""
import ctypes
import os
import re

import numpy as np
import pytest

from conftest import ROOT, golden
from oracle import oracle as O


def _product():
    from cornac_b200 import _lib
    return _lib


def test_library_loads_and_exports_every_declared_symbol_of_abi_3():
    _lib = _product()
    L = _lib.load()
    header = open(os.path.join(ROOT, "include", "b200cornac.h")).read()
    declared = set(re.findall(r"B200_API\s+[\w\s\*]+?\b(b200_\w+)\s*\(", header))
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(L, name), "include/b200cornac.h declares %s but the library does not export it" % name
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert L.b200_abi_version() == 3 and L.b200_kernel_launches() >= 0


def test_sampler_matches_oracle_streams():
    from cornac_b200.engine import MTSampler
    for seed in (0, 1, 123, 2 ** 31 - 1):
        for hi in (0, 1, 9, 5699, 10 ** 9 - 1, 2 ** 32 - 2, 2 ** 32 - 1, 2 ** 32, 2 ** 45 + 3):
            a = MTSampler(seed).fill(hi, 3000)
            b = O.MT19937(seed).fill(hi, 3000)
            assert np.array_equal(a, b), (seed, hi)
    a = MTSampler(5).fill(999, 1000, dtype=np.int32)
    b = O.MT19937(5).fill(999, 1000)
    assert a.dtype == np.int32 and np.array_equal(a, b)
    # state carries across calls (the reference keeps one RNGVector for all epochs, recom_bpr.pyx:190-197)
    s = MTSampler(9)
    a = np.concatenate([s.fill(77, 10), s.fill(77, 15)])
    assert np.array_equal(a, O.MT19937(9).fill(77, 25))


def test_sampler_rejects_bad_arguments():
    _lib = _product()
    L = _lib.load()
    h = L.b200_mt_sampler_create(1)
    out = np.empty(4, dtype=np.int64)
    assert L.b200_mt_sampler_fill_i64(h, -1, 4, out.ctypes.data) != 0
    assert b"bad argument" in L.b200_last_error()
    assert L.b200_mt_sampler_fill_i32(h, 2 ** 31, 4, out.ctypes.data) != 0
    L.b200_mt_sampler_destroy(h)


def test_device_draw_law_is_uniform_and_in_range():
    from cornac_b200 import engine
    ii, jj = engine.bpr_draw_host(seed=42, epoch=3, n=200000, nnz=1000, n_neg=50)
    assert ii.min() >= 0 and ii.max() < 1000 and jj.min() >= 0 and jj.max() < 50
    assert np.all(np.abs(np.bincount(jj, minlength=50) / 4000.0 - 1) < 0.1)
    assert np.all(np.abs(np.bincount(ii // 100, minlength=10) / 20000.0 - 1) < 0.05)
    # stream is a pure function of (seed, epoch, sample): sub-ranges agree, epochs differ
    ii2, jj2 = engine.bpr_draw_host(seed=42, epoch=3, n=1000, nnz=1000, n_neg=50, sample_base=500)
    assert np.array_equal(ii2, ii[500:1500]) and np.array_equal(jj2, jj[500:1500])
    ii3, _ = engine.bpr_draw_host(seed=42, epoch=4, n=1000, nnz=1000, n_neg=50)
    assert not np.array_equal(ii3, ii[:1000])


def test_product_never_touches_the_oracle():
    # neither the oracle nor the reference install may be named on the product path (imports, paths, dlopen)
    pat = re.compile(r"oracle|baseline[/\\.]|_ref\b", re.I)
    for base, _, files in os.walk(os.path.join(ROOT, "cornac_b200")):
        if os.path.basename(base) in ("build", "lib", "__pycache__"):
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(base, f)).read()
                hits = [l for l in txt.splitlines() if pat.search(l) and "summation order shared with the oracle" not in l]
                assert not hits, (f, hits[:3])


def test_kernels_fail_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    with pytest.raises(B200Error):
        engine.require_cuda()


def test_recommend_batch_host_logic_with_a_stubbed_device():
    """id mapping, argument errors and seen-item plumbing of DeviceScoringMixin.recommend_batch (the kernel call itself is
    stubbed: rank_batch is covered on the GPU)."""
    import scipy.sparse as sp
    from conftest import have_cornac
    if not have_cornac():
        pytest.skip("needs the cornac package")
    from cornac.models.recommender import Recommender
    from cornac_b200._scoring import DeviceScoringMixin

    class Stub(DeviceScoringMixin, Recommender):
        def __init__(self):
            Recommender.__init__(self, name="stub")
            self.calls = []

        def rank_batch(self, user_indices, k, exclude=None):
            self.calls.append((np.asarray(user_indices).tolist(), k, None if exclude is None else exclude.shape))
            n = len(user_indices)
            ids = np.tile(np.arange(k, dtype=np.int32), (n, 1))
            ids[:, -1] = -1                                   # a padded (short) list
            return ids, np.zeros((n, k), np.float32)

    m = Stub()
    m.uid_map = {"a": 0, "b": 1, "c": 2}
    m.iid_map = {"i%d" % j: j for j in range(6)}
    m.num_users, m.num_items = 3, 6
    out = m.recommend_batch(["c", "a"], k=3)
    assert out == [["i0", "i1"], ["i0", "i1"]] and m.calls[-1] == ([2, 0], 3, None)
    train = type("T", (), {"csr_matrix": sp.csr_matrix(np.eye(2, 6, dtype=np.float32))})()
    m.recommend_batch(["c"], k=2, remove_seen=True, train_set=train)
    assert m.calls[-1] == ([2], 2, (3, 6))                   # exclusion matrix padded to cover user 2
    with pytest.raises(ValueError):
        m.recommend_batch(["zz"], k=2)
    with pytest.raises(ValueError):
        m.recommend_batch(["a"], k=7)
    with pytest.raises(ValueError):
        m.recommend_batch(["a"], k=2, remove_seen=True)


def test_cache_blocked_sample_order_keeps_the_per_epoch_law():
    """b200_bpr_draw_host2 (the host twin of the B200_BPR_BLOCKED kernels): over one epoch every interaction is drawn once
    in expectation, negatives are uniform over all items, every window of the interaction list meets every item block,
    windows / blocks receive exactly their share; plan 1 x 1 is the unblocked stream bit for bit."""
    from cornac_b200 import engine
    nnz, n_neg = 120_007, 9_001
    for epoch, plan in ((0, (5, 3)), (4, (7, 4)), (1, (1, 6)), (2, (9, 1))):
        ii, jj = engine.bpr_draw_host(11, epoch, nnz, nnz, n_neg, plan=plan)
        assert ii.min() >= 0 and ii.max() < nnz and jj.min() >= 0 and jj.max() < n_neg
        wn, bn = plan
        wb = np.array([w * (nnz // wn) + min(w, nnz % wn) for w in range(wn + 1)])
        bb = np.array([b * (n_neg // bn) + min(b, n_neg % bn) for b in range(bn + 1)])
        w_of, b_of = np.searchsorted(wb, ii, side="right") - 1, np.searchsorted(bb, jj, side="right") - 1
        assert np.unique(w_of * bn + b_of).size == wn * bn                          # all (window, block) runs occur
        share_w = np.bincount(w_of, minlength=wn) / nnz
        assert np.allclose(share_w, np.diff(wb) / nnz, atol=2.0 / (wn * bn) * 0.51 + 1e-9)     # whole runs per window
        # negatives: uniform over the items (chi-square-ish bound on the block shares, Poisson noise per item)
        assert np.allclose(np.bincount(b_of, minlength=bn) / nnz, np.diff(bb) / n_neg, atol=0.02)
        cnt = np.bincount(jj, minlength=n_neg)
        assert abs(cnt.mean() - nnz / n_neg) < 1e-9 and cnt.std() < 1.5 * np.sqrt(nnz / n_neg)
        # interactions: mean 1 draw each, Poisson-like spread
        ci = np.bincount(ii, minlength=nnz)
        assert abs(ci.mean() - 1.0) < 1e-9 and 0.9 < ci.var() < 1.1
    a = engine.bpr_draw_host(5, 2, 5000, nnz, n_neg, sample_base=123)
    b = engine.bpr_draw_host(5, 2, 5000, nnz, n_neg, sample_base=123, plan=(1, 1))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert engine.bpr_block_plan(1000, 2000, 64) == (1, 1) and engine.bpr_block_plan(10_000_000, 1_000_000, 128) == (123, 13)


def test_host_samplers_reproduce_the_oracle_streams():
    """b200_vebpr_draw_host / b200_sbpr_draw_host == the streams the oracle traces (RNG order of the reference)."""
    from cornac_b200 import _lib, engine
    from oracle import oracle as O
    L = _lib.load()
    g = golden("vebpr_mid_k16")
    r = O.vebpr_fit(g["indptr"], g["indices"], g["view_indptr"], g["view_indices"], int(g["num_items"]), int(g["total_users"]),
                    int(g["total_items"]), int(g["k"]), 2, float(g["lr"]), float(g["reg"]), float(g["alpha"]), int(g["seed"]), trace=True)
    rng, _, _, _ = O.bpr_init(int(g["seed"]), int(g["total_users"]), int(g["total_items"]), int(g["k"]))
    gens = [engine.MTSampler(O.rngvector_seed(rng.randint(2 ** 31))) for _ in range(3)]
    nnz = len(g["indices"])
    coo = O.coo_rows(g["indptr"])
    vp, vi = np.ascontiguousarray(g["view_indptr"]), np.ascontiguousarray(g["view_indices"])
    for e in range(2):
        oi, ov, oj = np.empty(nnz, np.int64), np.empty(nnz, np.int32), np.empty(nnz, np.int32)
        assert L.b200_vebpr_draw_host(gens[0]._h, gens[1]._h, gens[2]._h, nnz, int(g["num_items"]), coo.ctypes.data, vp.ctypes.data,
                                      vi.ctypes.data, nnz, oi.ctypes.data, ov.ctypes.data, oj.ctypes.data) == 0
        assert np.array_equal(oi, r["i_index"][e]) and np.array_equal(ov, r["v_id"][e]) and np.array_equal(oj, r["j_id"][e])
    g = golden("sbpr_mid_k16")
    r = O.sbpr_fit(g["indptr"], g["indices"], g["social_item_ids"], g["social_item_counts"], g["social_indptr"], int(g["num_items"]),
                   int(g["total_users"]), int(g["total_items"]), int(g["k"]), 2, float(g["lr"]), float(g["lbd_u"]), float(g["lbd_v"]),
                   float(g["lbd_b"]), True, int(g["seed"]), trace=True)
    rng, _, _, _ = O.bpr_init(int(g["seed"]), int(g["total_users"]), int(g["total_items"]), int(g["k"]))
    gens = [engine.MTSampler(O.rngvector_seed(rng.randint(2 ** 31))) for _ in range(2)]
    nnz = len(g["indices"])
    coo = O.coo_rows(g["indptr"])
    sp_ = np.ascontiguousarray(g["social_indptr"])
    for e in range(2):
        oi, oj, ok = np.empty(nnz, np.int64), np.empty(nnz, np.int32), np.empty(nnz, np.int64)
        assert L.b200_sbpr_draw_host(gens[0]._h, gens[1]._h, nnz, int(g["num_items"]), coo.ctypes.data, sp_.ctypes.data, nnz,
                                     oi.ctypes.data, oj.ctypes.data, ok.ctypes.data) == 0
        assert np.array_equal(oi, r["i_index"][e]) and np.array_equal(oj, r["j_id"][e]) and np.array_equal(ok, r["k_index"][e])


def test_sbpr_social_item_lists_match_the_reference_fixture():
    """cornac_b200.recom_bprx.prepare_social_data (vectorised) == SBPR._prepare_social_data of the compiled reference
    (recom_sbpr.pyx:119-145; arrays stored in the fixture) == the oracle's per-user restatement.  Host code only."""
    pytest.importorskip("cornac")
    import scipy.sparse as sp
    from cornac_b200.recom_bprx import check_tri_factor_width, prepare_social_data
    g = golden("sbpr_mid_k16")
    n_users, n_items = int(g["num_users"]), int(g["num_items"])
    X = sp.csr_matrix((g["data"], g["indices"], g["indptr"]), shape=(n_users, n_items))
    Y = sp.csr_matrix((np.ones(len(g["graph_indices"])), g["graph_indices"], g["graph_indptr"]), shape=(n_users, n_users))
    ids, cnts, ptr_ = prepare_social_data(X, Y)
    assert ids.dtype == X.indices.dtype
    assert np.array_equal(ids, g["social_item_ids"]) and np.array_equal(cnts, g["social_item_counts"])
    assert np.array_equal(ptr_, g["social_indptr"])
    o_ids, o_cnts, o_ptr = O.sbpr_social_items(g["indptr"], g["indices"], g["graph_indptr"], g["graph_indices"])
    assert np.array_equal(ids, o_ids) and np.array_equal(cnts, o_cnts) and np.array_equal(ptr_, o_ptr)
    # a user who is her own friend, and friends listed twice, change nothing / count twice like the reference's row selection
    Y2 = sp.csr_matrix((np.ones(3), ([0, 0, 1], [0, 1, 0])), shape=(n_users, n_users))
    ids2, cnts2, ptr2 = prepare_social_data(X, Y2)
    own0 = set(X[0].indices.tolist())
    want0 = sorted(set(X[1].indices.tolist()) - own0)
    assert ids2[ptr2[0]:ptr2[1]].tolist() == want0 and set(cnts2[ptr2[0]:ptr2[1]].tolist()) <= {1}
    for k in (1, 126, 128, 512):
        assert check_tri_factor_width(k) == k
    for k in (0, 130, 516, 1024):
        with pytest.raises(ValueError):
            check_tri_factor_width(k)


def test_block_plan_of_the_cache_blocked_order_is_host_arithmetic():
    """b200_bpr_block_plan (no CUDA): 1 x 1 while the rows fit two 40 MB parts, else ceil(bytes / 40 MB) windows / item blocks --
    the configs[2] whole-model plan the bench reports (123 x 13) -- and the dev knob B200_BPR_PART_MB rescales it."""
    from cornac_b200 import _lib
    L = _lib.load()
    wn, bn = ctypes.c_uint32(), ctypes.c_uint32()

    def plan(n_users, n_items, k):
        assert L.b200_bpr_block_plan(n_users, n_items, k, ctypes.byref(wn), ctypes.byref(bn)) == 0
        return wn.value, bn.value

    os.environ.pop("B200_BPR_PART_MB", None)
    assert plan(943, 1682, 10) == (1, 1)
    assert plan(10_000_000, 1_000_000, 128) == (123, 13)
    assert plan(1_250_000, 1_000_000, 128) == (16, 13)
    os.environ["B200_BPR_PART_MB"] = "80"
    try:
        assert plan(10_000_000, 1_000_000, 128) == (62, 7)
    finally:
        os.environ.pop("B200_BPR_PART_MB", None)
    assert L.b200_bpr_block_plan(0, 10, 8, ctypes.byref(wn), ctypes.byref(bn)) != 0      # bad argument -> error code, no crash
