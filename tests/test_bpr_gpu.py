"""BPR kernels (through the C ABI) against the oracle and the golden vectors.  GPU only."""
import numpy as np
import pytest

from conftest import golden, rel_err, synth_csr
from oracle import oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-4    # north_star: trained embeddings within 1e-4 relative (norm-wise) under the same update order


def _dev(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).cuda()


def _data(indptr, indices):
    from cornac_b200 import engine
    return engine.BprData.from_host(indptr, indices)


@pytest.mark.parametrize("name", ["bpr_small_k10", "bpr_mid_k32", "bpr_nobias_k16"])
def test_seeded_fit_matches_reference_golden(name):
    """host mt19937 sampler + serial-equivalent replay kernel == seeded compiled reference."""
    import torch
    from cornac_b200 import engine
    g = golden(name)
    k, nnz, num_items = int(g["k"]), len(g["indices"]), int(g["num_items"])
    rng, U0, V0, B0 = O.bpr_init(int(g["seed"]), int(g["total_users"]), int(g["total_items"]), k)
    s_pos, s_neg = rng.randint(2 ** 31), rng.randint(2 ** 31)
    g_pos = engine.MTSampler(O.rngvector_seed(s_pos))
    g_neg = engine.MTSampler(O.rngvector_seed(s_neg))
    data = _data(g["indptr"], g["indices"])
    assert np.array_equal(data.coo_row.cpu().numpy(), O.coo_rows(g["indptr"]))
    # b200_bpr_prepare: pairs == (coo_row, indices) interleaved; every stored key is in the table
    data.prepare()
    pairs = data.pairs.cpu().numpy()
    assert np.array_equal(pairs[:, 0], O.coo_rows(g["indptr"])) and np.array_equal(pairs[:, 1], g["indices"])
    tbl = data.table.cpu().numpy().view(np.uint64)
    keys = (pairs[:, 0].astype(np.uint64) << np.uint64(32)) | pairs[:, 1].astype(np.uint64)
    stored = tbl[tbl != np.uint64(2 ** 64 - 1)]
    assert len(stored) == len(keys) and np.array_equal(np.sort(stored), np.sort(keys))
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    ref = O.bpr_fit(g["indptr"], g["indices"], num_items, int(g["total_users"]), int(g["total_items"]), k,
                    int(g["max_iter"]), float(g["lr"]), float(g["reg"]), bool(g["use_bias"]), int(g["seed"]))
    for ep in range(int(g["max_iter"])):
        ii = _dev(g_pos.fill(nnz - 1, nnz))
        jj = _dev(g_neg.fill(num_items - 1, nnz, dtype=np.int32))
        stats.zero_()
        engine.bpr_epoch_replay(data, ii, jj, U, V, B, float(g["lr"]), float(g["reg"]), bool(g["use_bias"]), stats)
        c, s = stats.cpu().tolist()
        assert s == ref["stats"][ep][1]
        assert abs(c - ref["stats"][ep][0]) <= 2
    for got, want in ((U, g["U"]), (V, g["V"])):
        got = got.cpu().numpy()
        assert rel_err(got, want) < TOL
        assert np.allclose(got, want, rtol=1e-4, atol=1e-6)
    if bool(g["use_bias"]):
        assert rel_err(B.cpu().numpy(), g["B"]) < TOL
    else:
        assert np.all(B.cpu().numpy() == 0)


@pytest.mark.parametrize("k", [1, 7, 10, 33, 64, 128, 200])
def test_replay_matches_oracle_on_arbitrary_stream(k):
    import torch
    from cornac_b200 import engine
    n_users, n_items, nnz = 700, 300, 9000
    indptr, indices = synth_csr(n_users, n_items, nnz, seed=k)
    nnz = len(indices)
    rng = np.random.RandomState(100 + k)
    U0 = rng.normal(0, 0.1, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.1, (n_items, k)).astype(np.float32)
    B0 = rng.normal(0, 0.1, n_items).astype(np.float32)
    n = 20001                                       # not a multiple of 32
    ii = rng.randint(nnz, size=n).astype(np.int64)
    jj = rng.randint(n_items, size=n).astype(np.int32)
    Ur, Vr, Br = U0.copy(), V0.copy(), B0.copy()
    c_ref, s_ref = O.bpr_replay(ii, jj, indptr, indices, Ur, Vr, Br, 0.05, 0.01, True)
    data = _data(indptr, indices)
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    engine.bpr_epoch_replay(data, _dev(ii), _dev(jj), U, V, B, 0.05, 0.01, True, stats)
    c, s = stats.cpu().tolist()
    assert s == s_ref and s > 0 and abs(c - c_ref) <= 2
    assert rel_err(U.cpu().numpy(), Ur) < 1e-5 and rel_err(V.cpu().numpy(), Vr) < 1e-5
    assert rel_err(B.cpu().numpy(), Br) < 1e-5


def _conflict_free_prefix(ii, jj, coo, indices):
    """longest prefix of the stream whose samples touch pairwise-disjoint user and item rows"""
    seen_u, seen_i = set(), set()
    for t in range(len(ii)):
        u, i, j = int(coo[ii[t]]), int(indices[ii[t]]), int(jj[t])
        if u in seen_u or i in seen_i or j in seen_i or i == j:
            return t
        seen_u.add(u)
        seen_i.update((i, j))
    return len(ii)


def conflict_free_window(seed, epoch, nnz, n_items, coo, indices, want=48, tries=200):
    """(sample_base, n): a window of the Philox stream with >= `want` pairwise-disjoint samples"""
    from cornac_b200 import engine
    best = (0, 0)
    for w in range(tries):
        base = w * 1000
        ii, jj = engine.bpr_draw_host(seed, epoch, 200, nnz, n_items, sample_base=base)
        n = _conflict_free_prefix(ii, jj, coo, indices)
        if n > best[1]:
            best = (base, n)
        if n >= want:
            break
    return best


@pytest.mark.parametrize("atomic", [False, True])
@pytest.mark.parametrize("k", [4, 10, 16, 32, 33, 64, 100, 128, 256, 512])
def test_hogwild_equals_sequential_when_conflict_free(k, atomic):
    """With pairwise-disjoint rows Hogwild has no races: the throughput kernel must then equal the
    oracle's sequential application of the SAME Philox stream (b200_bpr_draw_host)."""
    import torch
    from cornac_b200 import engine
    n_users, n_items = 40000, 30000
    indptr, indices = synth_csr(n_users, n_items, 120000, seed=3, zipf=0.0)
    nnz = len(indices)
    coo = O.coo_rows(indptr)
    seed, epoch = 1234 + k, 7
    base, n = conflict_free_window(seed, epoch, nnz, n_items, coo, indices)
    assert n >= 48, n
    ii, jj = engine.bpr_draw_host(seed, epoch, n, nnz, n_items, sample_base=base)
    rng = np.random.RandomState(k)
    U0 = rng.normal(0, 0.3, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    B0 = rng.normal(0, 0.3, n_items).astype(np.float32)
    Ur, Vr, Br = U0.copy(), V0.copy(), B0.copy()
    c_ref, s_ref = O.bpr_replay(ii[:n], jj[:n], indptr, indices, Ur, Vr, Br, 0.05, 0.02, True)
    data = _data(indptr, indices)
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    engine.bpr_epoch(data, n_items, U, V, B, 0.05, 0.02, True, seed, epoch, stats, n_samples=n, sample_base=base,
                     atomic=atomic, exact_exp=True)
    c, s = stats.cpu().tolist()
    assert (c, s) == (c_ref, s_ref)
    for got, want in ((U, Ur), (V, Vr), (B, Br)):
        got = got.cpu().numpy()
        assert rel_err(got, want) < 1e-6
        assert np.allclose(got, want, rtol=2e-5, atol=1e-6)
    # untouched rows are bit-identical
    touched = np.zeros(n_users, bool)
    touched[coo[ii[:n]]] = True
    assert np.array_equal(U.cpu().numpy()[~touched], U0[~touched])


def test_hogwild_fast_exp_close_to_exact():
    import torch
    from cornac_b200 import engine
    indptr, indices = synth_csr(5000, 3000, 60000, seed=9)
    k = 64
    rng = np.random.RandomState(0)
    U0 = rng.normal(0, 0.3, (5000, k)).astype(np.float32)
    V0 = rng.normal(0, 0.3, (3000, k)).astype(np.float32)
    outs = []
    for exact in (False, True):
        data = _data(indptr, indices)
        U, V, B = _dev(U0), _dev(V0), _dev(np.zeros(3000, np.float32))
        stats = torch.zeros(2, dtype=torch.int64, device="cuda")
        engine.bpr_epoch(data, 3000, U, V, B, 0.01, 0.01, True, 5, 0, stats, n_samples=64, exact_exp=exact)
        outs.append(U.cpu().numpy())
    assert rel_err(outs[0], outs[1]) < 1e-6


@pytest.mark.parametrize("k", [10, 64, 128])
def test_hogwild_lr0_is_identity_and_counts_match_stream(k):
    """lr = 0: factors must come back bit-identical and (correct, skipped) must equal what the
    oracle counts on the same stream -- a size-independent property, here at 2M samples."""
    import torch
    from cornac_b200 import engine
    n_users, n_items = 20000, 2000
    indptr, indices = synth_csr(n_users, n_items, 400000, seed=5)
    nnz = len(indices)
    rng = np.random.RandomState(1)
    U0 = rng.normal(0, 0.3, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    B0 = rng.normal(0, 0.3, n_items).astype(np.float32)
    n = 2_000_003
    data = _data(indptr, indices)
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    engine.bpr_epoch(data, n_items, U, V, B, 0.0, 0.01, True, 77, 2, stats, n_samples=n, exact_exp=True)
    c, s = stats.cpu().tolist()
    assert np.array_equal(U.cpu().numpy(), U0) and np.array_equal(V.cpu().numpy(), V0)
    assert np.array_equal(B.cpu().numpy(), B0)
    ii, jj = engine.bpr_draw_host(77, 2, n, nnz, n_items)
    Ur, Vr, Br = U0.copy(), V0.copy(), B0.copy()
    c_ref, s_ref = O.bpr_replay(ii, jj, indptr, indices, Ur, Vr, Br, 0.0, 0.01, True)
    assert s == s_ref and s > 1000
    assert abs(c - c_ref) <= max(3, int(2e-5 * n))      # only |score| ~ 1e-7 borderline samples may flip


def test_hogwild_atomic_conserves_item_mass():
    """reg = 0: every update adds +d to row i and -d to row j, so the column sums of V and the
    sum of B are invariants when no update is lost (B200_SGD_ATOMIC)."""
    import torch
    from cornac_b200 import engine
    n_users, n_items, k = 30000, 500, 64           # few items => heavy contention on V rows
    indptr, indices = synth_csr(n_users, n_items, 300000, seed=8, zipf=1.0)
    rng = np.random.RandomState(2)
    U0 = rng.normal(0, 0.3, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    data = _data(indptr, indices)
    U, V, B = _dev(U0), _dev(V0), _dev(np.zeros(n_items, np.float32))
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    engine.bpr_epoch(data, n_items, U, V, B, 0.05, 0.0, True, 3, 0, stats, n_samples=1_000_000, atomic=True)
    Vn, Bn = V.cpu().numpy().astype(np.float64), B.cpu().numpy().astype(np.float64)
    moved = np.abs(Vn - V0).sum()
    assert moved > 100.0
    assert np.abs(Vn.sum(0) - V0.astype(np.float64).sum(0)).max() < 1e-4 * moved / k
    assert abs(Bn.sum()) < 1e-4 * np.abs(Bn).sum()


def test_hogwild_training_tracks_cpu_hogwild():
    """Throughput mode is not order-identical to anything (neither is the multi-thread reference,
    recom_bpr.pyx:86-88): compare learning progress with the oracle's OpenMP Hogwild port."""
    import torch
    from cornac_b200 import engine
    n_users, n_items, k = 3000, 800, 32
    # planted structure: users like items of their own cluster
    rng = np.random.RandomState(4)
    cu, ci = rng.randint(8, size=n_users), rng.randint(8, size=n_items)
    rows = []
    for u in range(n_users):
        own = np.flatnonzero(ci == cu[u])
        rows.append(np.sort(rng.choice(own, size=min(20, len(own)), replace=False)))
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    indices = np.concatenate(rows).astype(np.int32)
    nnz = len(indices)
    _, U0, V0, B0 = O.bpr_init(1, n_users, n_items, k)
    Uc, Vc, Bc = U0.copy(), V0.copy(), B0.copy()
    cpu = [O.bpr_epoch_omp(indptr, indices, n_items, Uc, Vc, Bc, 0.05, 0.001, True, O.n_threads(), seed=e) for e in range(15)]
    data = _data(indptr, indices)
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    gpu = []
    for e in range(15):
        stats = torch.zeros(2, dtype=torch.int64, device="cuda")
        engine.bpr_epoch(data, n_items, U, V, B, 0.05, 0.001, True, 99, e, stats)
        gpu.append(tuple(stats.cpu().tolist()))
    acc_cpu = cpu[-1][0] / (nnz - cpu[-1][1])
    acc_gpu = gpu[-1][0] / (nnz - gpu[-1][1])
    assert acc_cpu > 0.9 and acc_gpu > 0.9 and abs(acc_cpu - acc_gpu) < 0.03
    assert abs(gpu[0][1] / nnz - cpu[0][1] / nnz) < 0.01          # same skip rate


def test_bad_arguments_are_reported():
    import torch
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    indptr, indices = synth_csr(10, 10, 30, seed=1)
    data = _data(indptr, indices)
    U = torch.zeros((10, 2000), dtype=torch.float32, device="cuda")
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    with pytest.raises(B200Error, match="out of range"):
        engine.bpr_epoch(data, 10, U, U, U[:, 0].contiguous(), 0.1, 0.1, True, 1, 0, stats)
    with pytest.raises(B200Error, match="contiguous CUDA tensor"):
        engine.bpr_epoch(data, 10, U.cpu(), U, U[:, 0].contiguous(), 0.1, 0.1, True, 1, 0, stats)


def test_hogwild_weighted_negatives_follow_item_popularity():
    """B200_BPR_NEG_WEIGHTED: with lr=0 the skip count must equal the oracle's count on the stream whose
    negatives are items of uniformly drawn interactions (b200_bpr_draw_host with n_neg = nnz)."""
    import torch
    from cornac_b200 import engine
    indptr, indices = synth_csr(5000, 400, 60000, seed=12, zipf=1.0)
    nnz, k = len(indices), 16
    rng = np.random.RandomState(0)
    U0 = rng.normal(0, 0.3, (5000, k)).astype(np.float32)
    V0 = rng.normal(0, 0.3, (400, k)).astype(np.float32)
    B0 = np.zeros(400, np.float32)
    data = _data(indptr, indices)
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    n = 300001
    engine.bpr_epoch(data, 400, U, V, B, 0.0, 0.01, True, 21, 0, stats, n_samples=n, neg_weighted=True, exact_exp=True)
    ii, jidx = engine.bpr_draw_host(21, 0, n, nnz, nnz)
    c_ref, s_ref = O.bpr_replay(ii, indices[jidx], indptr, indices, U0.copy(), V0.copy(), B0.copy(), 0.0, 0.01, True)
    c, s = stats.cpu().tolist()
    assert s == s_ref and s > 0.02 * n and abs(c - c_ref) <= 5        # popular negatives are skipped far more often


def test_sharded_fit_entry_single_process_and_host_rank_entry():
    """parallel.bpr_fit_sharded with one process == engine.bpr_train_host on the whole matrix (same Philox key
    layout), and engine.rank_topk_host == oracle on the trained factors."""
    from cornac_b200 import engine, parallel
    indptr, indices = synth_csr(3000, 1200, 40000, seed=21)
    k = 32
    _, U0, V0, B0 = O.bpr_init(3, 3000, 1200, k)
    Ua, Va, Ba = U0.copy(), V0.copy(), B0.copy()
    bounds, hist = parallel.bpr_fit_sharded(indptr, indices, 1200, Ua, Va, Ba, 0.05, 0.01, True, max_iter=3, key=5)
    assert bounds.tolist() == [0, 3000] and len(hist) == 3
    assert np.abs(Ua - U0).max() > 1e-4 and np.isfinite(Va).all()
    dU, dV, dB = _dev(Ua), _dev(Va), _dev(Ba)
    users = np.arange(0, 3000, 7, dtype=np.int64)
    ex_ptr = np.concatenate([[0], np.cumsum(np.diff(indptr)[users])]).astype(np.int64)
    ex_idx = np.concatenate([indices[indptr[u]:indptr[u + 1]] for u in users]).astype(np.int32)
    ids, sc = engine.rank_topk_host(dU, dV, 10, users, item_base=dB, excl_indptr=ex_ptr, excl_indices=ex_idx)
    want = O.score_batch(Ua[users], Va, Ba)
    for q, u in enumerate(users):
        wi, ws, _ = O.topk(want[q], 10, indices[indptr[u]:indptr[u + 1]])
        assert np.array_equal(ids[q], wi) and np.array_equal(sc[q], ws)


@pytest.mark.parametrize("k", [10, 64])
def test_hinge_loss_kernels_match_oracle(k):
    """MMMF loop body in both kernels: replay == oracle on an arbitrary stream; Hogwild == oracle when conflict-free."""
    import torch
    from cornac_b200 import engine
    n_users, n_items = 40000, 30000
    indptr, indices = synth_csr(n_users, n_items, 120000, seed=3, zipf=0.0)
    nnz = len(indices)
    coo = O.coo_rows(indptr)
    rng = np.random.RandomState(k)
    U0 = rng.normal(0, 0.3, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    B0 = rng.normal(0, 0.3, n_items).astype(np.float32)
    data = _data(indptr, indices)
    # replay, 20k samples with conflicts
    ii = rng.randint(nnz, size=20000).astype(np.int64)
    jj = rng.randint(n_items, size=20000).astype(np.int32)
    Ur, Vr, Br = U0.copy(), V0.copy(), B0.copy()
    c_ref, s_ref = O.bpr_replay(ii, jj, indptr, indices, Ur, Vr, Br, 0.05, 0.02, True, mmmf=True)
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    engine.bpr_epoch_replay(data, _dev(ii), _dev(jj), U, V, B, 0.05, 0.02, True, stats, hinge=True)
    c, s = stats.cpu().tolist()
    assert s == s_ref and abs(c - c_ref) <= 2 and 0.2 * 20000 < c < 0.8 * 20000
    assert rel_err(U.cpu().numpy(), Ur) < 1e-5 and rel_err(V.cpu().numpy(), Vr) < 1e-5 and rel_err(B.cpu().numpy(), Br) < 1e-5
    # Hogwild on a conflict-free window
    seed, epoch = 777 + k, 1
    base, n = conflict_free_window(seed, epoch, nnz, n_items, coo, indices)
    ii, jj = engine.bpr_draw_host(seed, epoch, n, nnz, n_items, sample_base=base)
    Ur, Vr, Br = U0.copy(), V0.copy(), B0.copy()
    c_ref, s_ref = O.bpr_replay(ii, jj, indptr, indices, Ur, Vr, Br, 0.05, 0.02, True, mmmf=True)
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats.zero_()
    engine.bpr_epoch(data, n_items, U, V, B, 0.05, 0.02, True, seed, epoch, stats, n_samples=n, sample_base=base, hinge=True)
    assert tuple(stats.cpu().tolist()) == (c_ref, s_ref)
    for got, want in ((U, Ur), (V, Vr), (B, Br)):
        assert np.allclose(got.cpu().numpy(), want, rtol=2e-5, atol=1e-6)


def test_edge_cases_empty_rows_tiny_shapes_zero_samples():
    """ragged / empty inputs: users without interactions, a single interaction, k = 1, zero samples"""
    import torch
    from cornac_b200 import engine
    # 6 users, rows 0, 2, 5 empty; 4 items
    indptr = np.array([0, 0, 2, 2, 3, 5, 5], dtype=np.int32)
    indices = np.array([1, 3, 0, 0, 2], dtype=np.int32)
    for k in (1, 3, 8):
        rng = np.random.RandomState(k)
        U0 = rng.normal(0, 0.3, (6, k)).astype(np.float32)
        V0 = rng.normal(0, 0.3, (4, k)).astype(np.float32)
        B0 = rng.normal(0, 0.3, 4).astype(np.float32)
        data = _data(indptr, indices)
        U, V, B = _dev(U0), _dev(V0), _dev(B0)
        stats = torch.zeros(2, dtype=torch.int64, device="cuda")
        engine.bpr_epoch(data, 4, U, V, B, 0.05, 0.01, True, 9, 0, stats, n_samples=0)          # nothing to do
        assert stats.cpu().tolist() == [0, 0] and np.array_equal(U.cpu().numpy(), U0)
        # sequential semantics on the tiny matrix: replay == oracle, empty rows untouched
        ii = rng.randint(5, size=200).astype(np.int64)
        jj = rng.randint(4, size=200).astype(np.int32)
        Ur, Vr, Br = U0.copy(), V0.copy(), B0.copy()
        c_ref, s_ref = O.bpr_replay(ii, jj, indptr, indices, Ur, Vr, Br, 0.05, 0.01, True)
        engine.bpr_epoch_replay(data, _dev(ii), _dev(jj), U, V, B, 0.05, 0.01, True, stats)
        assert stats.cpu().tolist() == [c_ref, s_ref]
        assert rel_err(U.cpu().numpy(), Ur) < 1e-5 and rel_err(V.cpu().numpy(), Vr) < 1e-5
        assert np.array_equal(U.cpu().numpy()[[0, 2, 5]], U0[[0, 2, 5]])
        # Hogwild on the same matrix only ever touches users that have interactions
        U, V, B = _dev(U0), _dev(V0), _dev(B0)
        stats.zero_()
        engine.bpr_epoch(data, 4, U, V, B, 0.05, 0.01, True, 9, 1, stats, n_samples=500)
        c, s = stats.cpu().tolist()
        assert 0 <= c and 0 < s < 500 and np.array_equal(U.cpu().numpy()[[0, 2, 5]], U0[[0, 2, 5]])
        assert np.isfinite(V.cpu().numpy()).all()
    # a matrix with a single interaction: every sample has u=0, i=0; j=0 is always skipped
    data = _data(np.array([0, 1], np.int32), np.array([0], np.int32))
    U, V, B = _dev(np.ones((1, 4), np.float32)), _dev(np.ones((2, 4), np.float32)), _dev(np.zeros(2, np.float32))
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    engine.bpr_epoch(data, 2, U, V, B, 0.01, 0.0, True, 1, 0, stats, n_samples=64)
    c, s = stats.cpu().tolist()
    assert c + s <= 64 and s > 0 and B.cpu().numpy()[0] > 0 > B.cpu().numpy()[1]


@pytest.mark.parametrize("hot", [False, True])
def test_scheduled_replay_is_bit_identical_to_serial_replay(hot, monkeypatch):
    """the phase-scheduled replay kernel == bpr_replay_kernel (one warp, strictly serial), bit for bit, including on a
    matrix so small that almost every phase is one long conflict chain.  The `hot` matrix fits shared memory, so the
    scheduled kernel runs on an on-chip copy of the factors; the other one (5000 x 3000, k = 24: about 780 KB of factors)
    does not, so the same kernel runs on the global factors."""
    import torch
    from cornac_b200 import engine
    n_users, n_items, nnz = (40, 12, 300) if hot else (5000, 3000, 60000)
    indptr, indices = synth_csr(n_users, n_items, nnz, seed=17)
    nnz = len(indices)
    k = 24
    rng = np.random.RandomState(5)
    U0 = rng.normal(0, 0.3, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    B0 = rng.normal(0, 0.3, n_items).astype(np.float32)
    ii = rng.randint(nnz, size=30011).astype(np.int64)
    jj = rng.randint(n_items, size=30011).astype(np.int32)
    outs = []
    for serial in ("1", "0"):
        monkeypatch.setenv("B200_REPLAY_SERIAL", serial)
        data = _data(indptr, indices)
        U, V, B = _dev(U0), _dev(V0), _dev(B0)
        stats = torch.zeros(2, dtype=torch.int64, device="cuda")
        engine.bpr_epoch_replay(data, _dev(ii), _dev(jj), U, V, B, 0.05, 0.01, True, stats)
        outs.append((U.cpu().numpy(), V.cpu().numpy(), B.cpu().numpy(), stats.cpu().tolist()))
    for other in outs[1:]:
        for a, b in zip(outs[0][:3], other[:3]):
            assert np.array_equal(a, b)
        assert outs[0][3] == other[3]
    Ur, Vr, Br = U0.copy(), V0.copy(), B0.copy()
    c_ref, s_ref = O.bpr_replay(ii, jj, indptr, indices, Ur, Vr, Br, 0.05, 0.01, True)
    assert outs[1][3][1] == s_ref and rel_err(outs[1][0], Ur) < 1e-5 and rel_err(outs[1][1], Vr) < 1e-5


@pytest.mark.parametrize("k", [10, 128])
def test_deterministic_epoch_repeats_bit_for_bit_and_trains(k):
    """deterministic=True (what fit() and the bench run): two runs of the same blocked epochs give identical factors and
    counts; the skip count equals the oracle's on the same stream; with lr = 0 the factors are untouched; the model
    learns (more correctly ranked samples in the last epoch than in the first)."""
    import torch
    from cornac_b200 import engine
    n_users, n_items = 30000, 3000
    indptr, indices = synth_csr(n_users, n_items, 600000, seed=8)
    nnz = len(indices)
    rng = np.random.RandomState(2)
    U0 = rng.normal(0, 0.1, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.1, (n_items, k)).astype(np.float32)
    B0 = np.zeros(n_items, np.float32)
    data = _data(indptr, indices)
    runs = []
    for _ in range(2):
        U, V, B = _dev(U0), _dev(V0), _dev(B0)
        counts = []
        for e in range(4):
            stats = torch.zeros(2, dtype=torch.int64, device="cuda")
            engine.bpr_epoch(data, n_items, U, V, B, 0.05, 0.01, True, 31, e, stats, blocked=True, deterministic=True)
            counts.append(tuple(stats.cpu().tolist()))
        runs.append((U.cpu().numpy(), V.cpu().numpy(), B.cpu().numpy(), counts))
    for a, b in zip(runs[0][:3], runs[1][:3]):
        assert np.array_equal(a, b)
    assert runs[0][3] == runs[1][3]
    assert runs[0][3][-1][0] > runs[0][3][0][0]
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    engine.bpr_epoch(data, n_items, U, V, B, 0.0, 0.01, True, 31, 0, stats, deterministic=True, exact_exp=True)
    assert np.array_equal(U.cpu().numpy(), U0) and np.array_equal(V.cpu().numpy(), V0)
    ii, jj = engine.bpr_draw_host(31, 0, nnz, nnz, n_items)
    c_ref, s_ref = O.bpr_replay(ii, jj, indptr, indices, U0.copy(), V0.copy(), B0.copy(), 0.0, 0.01, True)
    c, s = stats.cpu().tolist()
    assert s == s_ref and abs(c - c_ref) <= 3


@pytest.mark.parametrize("k", [10, 64])
def test_deterministic_round_equals_numpy_restatement(k):
    """ONE round of the deterministic mode (16384 samples, unbounded): every live sample's update is computed from the
    factors as they were at the start of the round and the updates are summed -- restated here in float64 with numpy,
    sample by sample from the host copy of the Philox stream; the changes of U, V and B and the counts must agree."""
    import torch
    from cornac_b200 import engine
    n_users, n_items, n = 30000, 3000, 16384
    indptr, indices = synth_csr(n_users, n_items, 600000, seed=9)
    nnz = len(indices)
    rng = np.random.RandomState(3)
    U0 = rng.normal(0, 0.1, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.1, (n_items, k)).astype(np.float32)
    B0 = rng.normal(0, 0.1, n_items).astype(np.float32)
    lr, reg = 0.05, 0.01
    data = _data(indptr, indices)
    U, V, B = _dev(U0), _dev(V0), _dev(B0)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    engine.bpr_epoch(data, n_items, U, V, B, lr, reg, True, 5, 3, stats, n_samples=n, exact_exp=True, unbounded=True,
                     deterministic=True)
    ii, jj = engine.bpr_draw_host(5, 3, n, nnz, n_items)
    users = np.repeat(np.arange(n_users), np.diff(indptr))[ii]
    pos = indices[ii]
    dU, dV, dB = np.zeros(U0.shape), np.zeros(V0.shape), np.zeros(B0.shape)
    correct = skipped = 0
    U64, V64, B64 = U0.astype(np.float64), V0.astype(np.float64), B0.astype(np.float64)
    for u, i, j in zip(users, pos, jj):
        if j in indices[indptr[u]:indptr[u + 1]]:
            skipped += 1
            continue
        score = B64[i] - B64[j] + U64[u] @ (V64[i] - V64[j])
        z = 1.0 / (1.0 + np.exp(score))
        correct += z < 0.5
        dU[u] += lr * (z * (V64[i] - V64[j]) - reg * U64[u])
        dV[i] += lr * (z * U64[u] - reg * V64[i])
        dV[j] += lr * (-z * U64[u] - reg * V64[j])
        dB[i] += lr * (z - reg * B64[i])
        dB[j] += lr * (-z - reg * B64[j])
    c, s = stats.cpu().tolist()
    assert s == skipped and abs(c - correct) <= 3
    assert rel_err(U.cpu().numpy().astype(np.float64) - U64, dU) < 1e-4
    assert rel_err(V.cpu().numpy().astype(np.float64) - V64, dV) < 1e-4
    assert rel_err(B.cpu().numpy().astype(np.float64) - B64, dB) < 1e-4
