"""Tensor-core (wgmma) rank path: the approximate pass against an fp16 matmul, and the fused
b200_rank_topk against the oracle -- ids and scores bit-exact.  GPU only."""
import os

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu


def _dev(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).cuda()


def _rank_topk(U, V, base, uidx, uoff, excl, topk):
    import torch
    from cornac_b200._lib import check, current_stream, load, ptr
    L = load()
    n_q = len(uidx) if uidx is not None else U.shape[0]
    n_items, k = V.shape
    ids = torch.empty((n_q, topk), dtype=torch.int32, device="cuda")
    sc = torch.empty((n_q, topk), dtype=torch.float32, device="cuda")
    nbytes = int(L.b200_rank_topk_workspace_bytes(n_q, n_items, k, topk))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device="cuda")
    dp = dx = None
    if excl is not None:
        ex_ptr = np.concatenate([[0], np.cumsum([len(e) for e in excl])]).astype(np.int64)
        ex_idx = np.concatenate([np.sort(e) for e in excl]).astype(np.int32) if ex_ptr[-1] else np.zeros(1, np.int32)
        dp, dx = _dev(ex_ptr), _dev(ex_idx)
    keep = [_dev(U), _dev(V), None if base is None else _dev(base), None if uidx is None else _dev(uidx),
            None if uoff is None else _dev(uoff)]
    check(L.b200_rank_topk(ptr(keep[0]), ptr(keep[3]), n_q, ptr(keep[1]), n_items, k, ptr(keep[2]), ptr(keep[4]),
                           ptr(dp), ptr(dx), topk, ptr(ids), ptr(sc), ptr(ws), nbytes, current_stream()), "b200_rank_topk")
    torch.cuda.synchronize()
    return ids.cpu().numpy(), sc.cpu().numpy()


@pytest.mark.parametrize("k,n_items,n_q", [(16, 1024, 128), (64, 1500, 100), (128, 3000, 260), (100, 2048, 37), (8, 1100, 5)])
def test_tensor_pass_matches_fp16_matmul(k, n_items, n_q):
    """GMMA descriptors / packing / power-of-two scaling / accumulator hand-off: dense approximate scores ==
    fp16 x fp16 -> f32 of the scaled operands, unscaled."""
    import torch
    from cornac_b200._lib import check, current_stream, load, ptr
    L = load()
    assert L.b200_rank_topk_workspace_bytes(n_q, n_items, k, 10) > 0
    rng = np.random.RandomState(k + n_items)
    U = rng.normal(0, 0.5, (n_q, k)).astype(np.float32)
    V = rng.normal(0, 0.5, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.5, n_items).astype(np.float32)
    dU, dV, db = _dev(U), _dev(V), _dev(base)
    rows, cols = (n_q + 127) // 128 * 128, (n_items + 255) // 256 * 256
    out = torch.full((rows, cols), float("nan"), dtype=torch.float32, device="cuda")
    nbytes = int(L.b200_rank_topk_workspace_bytes(n_q, n_items, k, 10))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    check(L.b200_rank_tc_debug_scores(ptr(dU), n_q, ptr(dV), n_items, k, ptr(db), ptr(out), out.numel(), ptr(ws), nbytes,
                                      current_stream()), "b200_rank_tc_debug_scores")
    torch.cuda.synchronize()
    got = out.cpu().numpy()[:n_q]
    def p2(m):                                              # the kernel's scales: m * s in [2^13, 2^14)
        return 2.0 ** (14 - np.frexp(np.asarray(m, dtype=np.float32))[1])
    sU, sV = p2(np.abs(U).max(axis=1, keepdims=True)), float(p2(np.abs(V).max()))     # one scale per user row
    Ub = (dU * _dev(sU.astype(np.float32))).half().double().cpu().numpy() / sU
    Vb = (dV * float(sV)).half().double().cpu().numpy() / sV
    want = Ub @ Vb.T + base[None, :].astype(np.float64)
    scale = np.abs(Ub) @ np.abs(Vb).T + np.abs(base)[None, :]
    err = np.abs(got[:, :n_items] - want)
    # f32 accumulation of exact fp16 products + the item base carried as two fp16 (2^-22 relative)
    assert np.all(err <= 2e-6 * scale + 1e-6 * np.abs(base)[None, :] + 1e-7), float((err / (scale + 1e-9)).max())
    assert np.all(got[:, n_items:] < -1e38)                 # padding items score -inf
    # the rigorous bound the candidate filter relies on (row_eps in rank_tc.cu), against the exact f64 scores
    exact = U.astype(np.float64) @ V.astype(np.float64).T + base[None, :].astype(np.float64)
    un = np.linalg.norm(U.astype(np.float64), axis=1)[:, None]
    vmax, bmax = np.linalg.norm(V.astype(np.float64), axis=1).max(), np.abs(base).max()
    eps = 0.00098 * un * vmax + 2e-6 * (un * vmax + bmax) + 4.8e-7 * bmax
    assert np.all(np.abs(got[:, :n_items] - exact) <= eps)


@pytest.mark.parametrize("k,n_items,n_q,topk", [(64, 20000, 300, 100), (128, 5000, 64, 100), (128, 100003, 130, 100),
                                                (10, 1682, 40, 10), (100, 1024, 129, 256), (32, 4096, 1, 1),
                                                (64, 30000, 200, 256), (30, 5000, 70, 20)])
def test_fused_rank_is_bit_exact(k, n_items, n_q, topk):
    rng = np.random.RandomState(k + n_q)
    U = rng.normal(0, 0.3, (1000, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    uidx = rng.randint(1000, size=n_q).astype(np.int64)
    uoff = rng.normal(0, 0.3, n_q).astype(np.float32)
    excl = [np.unique(rng.randint(n_items, size=rng.randint(0, 300))) for _ in range(n_q)]
    ids, sc = _rank_topk(U, V, base, uidx, uoff, excl, topk)
    want = O.score_batch(U[uidx], V, base, uoff)
    for q in range(n_q):
        wi, ws, w = O.topk(want[q], topk, excl[q])
        assert np.array_equal(ids[q], wi), (q, ids[q][:8], wi[:8])
        assert np.array_equal(sc[q][:w], ws[:w])


def test_fused_rank_plain_rows_no_exclusion_no_bias():
    rng = np.random.RandomState(3)
    U = rng.normal(0, 1, (200, 64)).astype(np.float32)
    V = rng.normal(0, 1, (7000, 64)).astype(np.float32)
    ids, sc = _rank_topk(U, V, None, None, None, None, 50)
    want = O.score_batch(U, V)
    for q in range(200):
        wi, ws, _ = O.topk(want[q], 50)
        assert np.array_equal(ids[q], wi) and np.array_equal(sc[q], ws)


def test_fused_rank_degenerate_rows_fall_back_to_exact():
    """zero / tied rows overflow the candidate lists: those users are redone by the exact path"""
    rng = np.random.RandomState(5)
    U = rng.normal(0, 0.3, (140, 64)).astype(np.float32)
    U[3] = 0.0                                              # every score == base
    U[77] = 0.0
    V = rng.normal(0, 0.3, (3000, 64)).astype(np.float32)
    base = np.zeros(3000, np.float32)                       # => rows 3, 77: 3000-way tie
    V[100:1200] = V[100]                                    # 1100 identical items: ties inside every row
    ids, sc = _rank_topk(U, V, base, None, None, None, 100)
    want = O.score_batch(U, V, base)
    for q in range(140):
        wi, ws, _ = O.topk(want[q], 100)
        assert np.array_equal(ids[q], wi), q
        assert np.array_equal(sc[q], ws)


@pytest.mark.parametrize("case", ["tiny", "huge", "mixed_rows", "base_dominates", "base_negligible", "wide_elements",
                                  "subnormal"])
def test_fused_rank_dynamic_range(case):
    """the fp16 tensor pass rescales both operands by powers of two: magnitudes far outside the fp16 range, rows of
    very different size, a base that dwarfs (or vanishes next to) the dot products -- ids and scores stay exact"""
    rng = np.random.RandomState(len(case))
    n_q, n_items, k, topk = 150, 6000, 64, 50
    U = rng.normal(0, 0.3, (n_q, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    if case == "tiny":
        U *= np.float32(1e-9); V *= np.float32(1e-7); base *= np.float32(1e-16)
    elif case == "huge":
        U *= np.float32(3e6); V *= np.float32(1e7); base *= np.float32(1e13)
    elif case == "mixed_rows":
        U *= (10.0 ** rng.uniform(-6, 3, (n_q, 1))).astype(np.float32)
        V *= (10.0 ** rng.uniform(-3, 2, (n_items, 1))).astype(np.float32)
    elif case == "base_dominates":
        base *= np.float32(1e9)
    elif case == "base_negligible":
        base *= np.float32(1e-12)
    elif case == "wide_elements":
        U *= (10.0 ** rng.uniform(-8, 0, (n_q, k))).astype(np.float32)
        V *= (10.0 ** rng.uniform(-8, 0, (n_items, k))).astype(np.float32)
    elif case == "subnormal":
        U *= np.float32(1e-30); V *= np.float32(1e-12); base *= np.float32(1e-42)
    excl = [np.unique(rng.randint(n_items, size=rng.randint(0, 80))) for _ in range(n_q)]
    ids, sc = _rank_topk(U, V, base, None, None, excl, topk)
    want = O.score_batch(U, V, base)
    for q in range(n_q):
        wi, ws, w = O.topk(want[q], topk, excl[q])
        assert np.array_equal(ids[q], wi), (case, q, ids[q][:8], wi[:8])
        assert np.array_equal(sc[q][:w], ws[:w])


def test_tensor_path_and_exact_path_agree(monkeypatch):
    rng = np.random.RandomState(9)
    U = rng.normal(0, 0.3, (300, 128)).astype(np.float32)
    V = rng.normal(0, 0.3, (9000, 128)).astype(np.float32)
    base = rng.normal(0, 0.3, 9000).astype(np.float32)
    a = _rank_topk(U, V, base, None, None, None, 100)
    monkeypatch.setenv("B200_RANK_TC", "0")
    b = _rank_topk(U, V, base, None, None, None, 100)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("k,n_items,n_q,topk", [(129, 3000, 70, 50), (144, 2500, 40, 20), (64, 3000, 50, 257),
                                                (64, 3000, 33, 300), (64, 1023, 20, 10), (4, 2000, 10, 5)])
def test_limits_of_the_fused_kernel_take_the_exact_path(k, n_items, n_q, topk):
    """outside k <= 128 / topk <= 256 / n_items >= 1024 / k >= 8 the tensor-core pass is not used (rank_tc_supported):
    b200_rank_topk answers through the exact kernels and the results are the oracle's all the same"""
    rng = np.random.RandomState(k * 7 + topk)
    U = rng.normal(0, 0.3, (n_q, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    excl = [np.unique(rng.randint(n_items, size=rng.randint(0, 60))) for _ in range(n_q)]
    ids, sc = _rank_topk(U, V, base, None, None, excl, topk)
    want = O.score_batch(U, V, base)
    for q in range(n_q):
        wi, ws, w = O.topk(want[q], topk, excl[q])
        assert np.array_equal(ids[q], wi) and np.array_equal(sc[q][:w], ws[:w])


def test_packed_item_side_built_once_gives_the_same_answer_and_is_really_used():
    """b200_rank_pack_items + b200_rank_topk_packed: the fp16 item tiles and norms built once give exactly the result of
    b200_rank_topk (which packs per call); that the packed buffer is what the kernel reads is shown by changing V in
    place: the stale buffer then yields the OLD model's candidates' exact scores order (not the oracle's), a rebuilt one
    the oracle's again."""
    import torch
    from cornac_b200 import engine
    rng = np.random.RandomState(4)
    U = torch.from_numpy(rng.normal(0, 0.3, (200, 64)).astype(np.float32)).cuda()
    Vh = rng.normal(0, 0.3, (5000, 64)).astype(np.float32)
    V = torch.from_numpy(Vh.copy()).cuda()
    B = torch.from_numpy(rng.normal(0, 0.3, 5000).astype(np.float32)).cuda()
    packed = engine.rank_pack_items(V, B)
    assert packed is not None and packed.dtype == torch.uint8
    a = engine.rank_topk(U, V, 20, item_base=B)
    b = engine.rank_topk(U, V, 20, item_base=B, packed_items=packed)
    b2 = engine.rank_topk(U, V, 20, item_base=B, packed_items=packed)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(b[0], b2[0])
    V.copy_(torch.from_numpy(Vh[::-1].copy()).cuda())              # same storage, new content
    want = O.score_batch(U.cpu().numpy(), Vh[::-1].copy(), B.cpu().numpy())
    stale = engine.rank_topk(U, V, 20, item_base=B, packed_items=packed)
    fresh = engine.rank_topk(U, V, 20, item_base=B, packed_items=engine.rank_pack_items(V, B))
    n_same = 0
    for q in range(200):
        wi, wsc, _ = O.topk(want[q], 20)
        assert np.array_equal(fresh[0][q].cpu().numpy(), wi) and np.array_equal(fresh[1][q].cpu().numpy(), wsc)
        n_same += int(np.array_equal(stale[0][q].cpu().numpy(), wi))
    assert n_same < 100                                             # the stale tiles nominated the wrong candidates
    assert engine.rank_pack_items(torch.zeros((500, 64), device="cuda")) is None      # tiny catalogue: exact path, nothing to pack
    with pytest.raises(Exception):
        engine.rank_topk(U, V[:4000].contiguous(), 20, packed_items=packed)
