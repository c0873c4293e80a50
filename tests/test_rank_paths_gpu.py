"""The fused rank path (b200_rank_topk) along the branches of its host loop that small inputs never take: more than one
user chunk, the exact repairs of overflowed rows in a later chunk (row by row, and the whole chunk in slabs), finish
rows with more survivors than the warp kernel holds, factor rows off a 16-byte boundary, the exact path over several
slabs and the score grid once it wraps.  Ids and scores are checked bit for bit against the oracle on chosen rows and
against the exact device path on every row; the kernel launch count of each call shows which branches ran.  GPU only."""
import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

# Kernel launches of one b200_rank_topk call on the tensor-core path, following rank_tc() in csrc/rank_tc.cu:
#   item side: norm_kernel, scale_items_kernel, pack_kernel                       3 (none when packed_items is given)
#   each user chunk: norm_kernel + pack_kernel of its users, rank_tc_kernel, then
#     staged finish (k % 4 == 0, k <= 128, V 16-byte aligned): warp kernel + block kernel for its big rows   5
#     otherwise: rank_tc_finish_kernel<false>                                                              4
#   each overflowed row repaired on its own (n_over <= 256, or a slab would hold < 8 rows): score + top-k     2
#   each slab of a chunk redone whole on the exact path (n_over > 256):                      score + top-k     2
# The exact path (rank_tc_supported() says no) launches score + top-k per slab of queries: 2 each.
LIST_BYTES_PER_TILE = 8 * 1024 * 32 * 8     # candidate lists of one user tile: EPI_WARPS x CAP x 32 lanes x 8 bytes
FW_KEYS = 512                               # survivors the warp finish kernel holds; more go to big_rows
MIN_SLAB_ROWS = 8                           # fewer score rows per slab than this: per-row repair instead
EVAL_BATCH = 75776                          # ranking_eval's default batch_users (cornac_b200/evaluation.py)


def _tc_launches(n_chunks, staged=True, packed=False, rows_repaired=0, slabs=0):
    return (0 if packed else 3) + n_chunks * (5 if staged else 4) + 2 * rows_repaired + 2 * slabs


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ceil(a, b):
    return -(-a // b)


def _ws(L, n_q, n_items, k, topk):
    return int(L.b200_rank_topk_workspace_bytes(n_q, n_items, k, topk))


def _first(pred, hi=1 << 40):
    """smallest n in [1, hi] with pred(n), pred monotone"""
    lo = 1
    while lo < hi:
        mid = (lo + hi) // 2
        if pred(mid):
            hi = mid
        else:
            lo = mid + 1
    return lo


def _tc_chunk(L, n_items, k, topk):
    """(rows per user chunk, rows per user tile) of the tensor-core pass: its workspace grows by one step per tile of
    users and stops growing at one chunk"""
    full = _ws(L, 1 << 40, n_items, k, topk)
    last = _first(lambda n: _ws(L, n, n_items, k, topk) >= full)           # first row of a chunk's last tile
    prev = _ws(L, last - 1, n_items, k, topk)
    tile = last - _first(lambda n: _ws(L, n, n_items, k, topk) >= prev)
    return last - 1 + tile, tile


def _slab_rows(n_q, n_items, chunk, tile):
    """score rows per slab of the whole-chunk repair: the candidate-list area of one chunk over one score row"""
    return min(_ceil(n_q, tile), chunk // tile) * LIST_BYTES_PER_TILE // (4 * n_items)


def _exclusions(rng, n_q, n_items, max_len=60, lead=1000, tail=500):
    """Sorted exclusion lists of 0..max_len ids per query as a CSR whose indptr starts `lead` entries into a larger
    indices array; the entries outside every row's span are valid ids too, so a misplaced read excludes wrong items."""
    n = rng.randint(0, max_len + 1, n_q)
    row = np.repeat(np.arange(n_q, dtype=np.int64), n)
    key = np.unique(row * n_items + rng.randint(n_items, size=len(row)))
    cnt = np.bincount(key // n_items, minlength=n_q)
    indptr = lead + np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    indices = rng.randint(n_items, size=lead + len(key) + tail).astype(np.int32)
    indices[lead:lead + len(key)] = key % n_items
    return indptr, indices


def _rows(rng, n_q, chunk, extra=()):
    """rows checked against the oracle: +-130 around each chunk boundary, the first and the last, `extra` and ~300
    random ones"""
    sel = [np.array([0, n_q - 1]), np.asarray(extra, np.int64), rng.choice(n_q, min(300, n_q), replace=False)]
    sel += [np.arange(max(b - 130, 0), min(b + 131, n_q)) for b in range(chunk, n_q, chunk)]
    return np.unique(np.concatenate(sel))


def _check_oracle(ids, sc, rows, U, uidx, V, base, uoff, indptr, indices, topk):
    """rows `rows` of the device result == the oracle's top-k of the same query: ids and scores bit for bit"""
    import torch
    sel = torch.from_numpy(rows).to(ids.device)
    ids, sc = ids[sel].cpu().numpy(), sc[sel].cpu().numpy()
    for b in range(0, len(rows), 64):
        r = rows[b:b + 64]
        want = O.score_batch(U[r if uidx is None else uidx[r]], V, base, None if uoff is None else uoff[r])
        for j, q in enumerate(r):
            wi, wsc, _ = O.topk(want[j], topk, indices[indptr[q]:indptr[q + 1]])
            assert np.array_equal(ids[b + j], wi), (q, ids[b + j][:8], wi[:8])
            assert np.array_equal(sc[b + j], wsc), q


def _launched(L, call):
    """(call's result, kernel launches it made)"""
    import torch
    before = int(L.b200_kernel_launches())
    out = call()
    torch.cuda.synchronize()
    return out, int(L.b200_kernel_launches()) - before


def _check_exact_path(monkeypatch, L, call, got, n_q, n_items, k, topk):
    """the same call on the exact device path gives the same ids and scores on every row"""
    import torch
    with monkeypatch.context() as m:
        m.setenv("B200_RANK_TC", "0")
        slab = _ws(L, 1 << 40, n_items, k, topk) // (4 * n_items)
        (ids, sc), n = _launched(L, call)
    assert n == 2 * _ceil(n_q, slab)
    assert torch.equal(ids, got[0]) and torch.equal(sc, got[1])


CHUNK_CASES = [("eval_batch", "rows", "rank_topk"), ("eval_batch", "idx", "packed"), ("two_chunks", "rows", "packed"),
               ("two_chunks", "idx", "rank_topk"), ("two_chunks", "idx", "host")]


@pytest.mark.parametrize("size,users,entry", CHUNK_CASES)
def test_every_user_chunk_ranks_its_own_queries(monkeypatch, size, users, entry):
    """n_q = ranking_eval's default batch (two chunks) or 2 chunks + 1000: the q0 offsets of every later chunk into U or
    user_idx, user_off, the un-rebased exclusion CSR and the outputs; through rank_topk, with packed_items and through
    rank_topk_host (what rank_batch calls)"""
    import torch
    from cornac_b200 import engine
    L = engine.require_cuda()
    k, n_items, topk = 64, 2000, 100
    chunk, _ = _tc_chunk(L, n_items, k, topk)
    n_q = EVAL_BATCH if size == "eval_batch" else 2 * chunk + 1000
    assert n_q > chunk
    rng = np.random.RandomState(CHUNK_CASES.index((size, users, entry)))
    U = rng.normal(0, 0.3, (n_q if users == "rows" else 5000, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    uidx = None if users == "rows" else rng.randint(5000, size=n_q).astype(np.int64)
    uoff = None if entry == "host" else rng.normal(0, 0.3, n_q).astype(np.float32)
    indptr, indices = _exclusions(rng, n_q, n_items)
    dU, dV, dB = _dev(U), _dev(V), _dev(base)
    d_uidx, d_uoff = (None if a is None else _dev(a) for a in (uidx, uoff))
    dp, dx = _dev(indptr), _dev(indices)
    packed = None
    if entry == "packed":
        packed, n = _launched(L, lambda: engine.rank_pack_items(dV, dB))
        assert n == 3

    def call(packed_items=None):
        if entry == "host":
            return tuple(map(torch.from_numpy, engine.rank_topk_host(dU, dV, topk, uidx, item_base=dB, excl_indptr=indptr,
                                                                     excl_indices=indices)))
        return engine.rank_topk(dU, dV, topk, user_idx=d_uidx, item_base=dB, user_off=d_uoff, excl_indptr=dp,
                                excl_indices=dx, packed_items=packed_items)

    got, n = _launched(L, lambda: call(packed))
    assert n == _tc_launches(_ceil(n_q, chunk), packed=packed is not None)
    _check_oracle(*got, _rows(rng, n_q, chunk), U, uidx, V, base, uoff, indptr, indices, topk)
    _check_exact_path(monkeypatch, L, call, got, n_q, n_items, k, topk)


def test_overflowed_rows_of_later_chunks_are_repaired_row_by_row_and_whole_chunk(monkeypatch):
    """~100 degenerate rows in chunk 2 (per-row repair, global query index), 300 in chunk 3 (> 256: the chunk is redone
    in slabs from g0 = q0 + r0).  A degenerate row -- zero U row, no item base, a user offset -- scores every item the
    same, so its candidate lists overflow."""
    from cornac_b200 import engine
    L = engine.require_cuda()
    k, n_items, topk = 64, 2000, 100
    chunk, tile = _tc_chunk(L, n_items, k, topk)
    n_q = 2 * chunk + 1000
    rng = np.random.RandomState(17)
    U = rng.normal(0, 0.3, (n_q, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    uoff = rng.normal(0, 0.3, n_q).astype(np.float32)
    second = np.unique(np.concatenate([chunk + np.arange(20), 2 * chunk - 1 - np.arange(20),
                                       rng.choice(np.arange(chunk + 20, 2 * chunk - 20), 60, replace=False)]))
    third = 2 * chunk + np.unique(np.concatenate([np.arange(10), [999], rng.choice(1000, 290, replace=False)]))
    assert len(second) == 100 and len(third) > 256
    U[second] = 0.0
    U[third] = 0.0
    indptr, indices = _exclusions(rng, n_q, n_items)
    dU, dV, d_uoff, dp, dx = map(_dev, (U, V, uoff, indptr, indices))

    def call():
        return engine.rank_topk(dU, dV, topk, user_off=d_uoff, excl_indptr=dp, excl_indices=dx)

    slab = _slab_rows(n_q, n_items, chunk, tile)
    assert slab >= MIN_SLAB_ROWS
    got, n = _launched(L, call)
    assert n == _tc_launches(3, rows_repaired=len(second), slabs=_ceil(1000, slab))
    rows = _rows(rng, n_q, chunk, np.concatenate([second, third]))
    _check_oracle(*got, rows, U, None, V, None, uoff, indptr, indices, topk)
    _check_exact_path(monkeypatch, L, call, got, n_q, n_items, k, topk)


@pytest.mark.parametrize("n_items", [100000, 300000])
def test_whole_chunk_repair_slab_loop_and_its_per_row_fallback(monkeypatch, n_items):
    """280 of 300 rows degenerate (> 256 overflowed): with 100,000 items the chunk's candidate-list area holds 15 score
    rows, so the chunk is redone in 20 slabs; with 300,000 it holds 5 (< 8) and every overflowed row is repaired alone"""
    from cornac_b200 import engine
    L = engine.require_cuda()
    n_q, k, topk = 300, 32, 100
    chunk, tile = _tc_chunk(L, n_items, k, topk)
    rng = np.random.RandomState(n_items % 1000 + 3)
    U = rng.normal(0, 0.3, (n_q, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    uoff = rng.normal(0, 0.3, n_q).astype(np.float32)
    degenerate = np.concatenate([[0, n_q - 1], 1 + rng.choice(n_q - 2, 278, replace=False)])
    U[degenerate] = 0.0
    indptr, indices = _exclusions(rng, n_q, n_items)
    dU, dV, d_uoff, dp, dx = map(_dev, (U, V, uoff, indptr, indices))

    def call():
        return engine.rank_topk(dU, dV, topk, user_off=d_uoff, excl_indptr=dp, excl_indices=dx)

    slab = _slab_rows(n_q, n_items, chunk, tile)
    got, n = _launched(L, call)
    if n_items == 100000:
        assert slab >= MIN_SLAB_ROWS and _ceil(n_q, slab) > 1
        assert n == _tc_launches(1, slabs=_ceil(n_q, slab))
    else:
        assert slab < MIN_SLAB_ROWS
        assert n == _tc_launches(1, rows_repaired=len(degenerate))
    _check_oracle(*got, np.arange(n_q), U, None, V, None, uoff, indptr, indices, topk)
    _check_exact_path(monkeypatch, L, call, got, n_q, n_items, k, topk)


def test_rows_with_more_survivors_than_the_warp_finish_holds(monkeypatch):
    """800 items d + 1e-6 noise are the top items of users close to 0.5 d, in both chunks: their fp16 images are equal
    (d is a multiple of 1/8, so d times any power-of-two scale is an fp16 number the noise does not leave), so all 800
    tie in the approximate pass and survive the filter, while their f32 scores differ.  Such a row has more than FW_KEYS
    survivors and is redone by the block finish kernel from big_rows (chunk-local indices)."""
    import torch
    from cornac_b200 import engine
    from cornac_b200._lib import check, current_stream, ptr
    L = engine.require_cuda()
    k, n_items, topk, n_cl = 64, 4096, 100, 800
    chunk, tile = _tc_chunk(L, n_items, k, topk)
    n_q = chunk + 3000
    rng = np.random.RandomState(41)
    d = (rng.randint(1, 9, k) * rng.choice([-1, 1], k)).astype(np.float32) / np.float32(8)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    V[rng.choice(n_items, n_cl, replace=False)] = d + np.float32(1e-6) * rng.normal(size=(n_cl, k)).astype(np.float32)
    U = rng.normal(0, 0.3, (n_q, k)).astype(np.float32)
    big = np.unique(np.concatenate([np.arange(chunk - 40, chunk + 40), rng.choice(n_q, 120, replace=False)]))
    assert (big < chunk).any() and (big >= chunk).any()
    U[big] = np.float32(0.5) * d + np.float32(0.01) * rng.normal(size=(len(big), k)).astype(np.float32)
    uoff = rng.normal(0, 0.3, n_q).astype(np.float32)
    dU, dV, d_uoff = map(_dev, (U, V, uoff))

    # the approximate scores of the big rows (they depend on the row alone): more than FW_KEYS items reach the row's
    # K-th best, and the filter never rises above it
    dUb = _dev(U[big])
    nbytes = _ws(L, len(big), n_items, k, topk)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = torch.empty((_ceil(len(big), tile) * tile, n_items), dtype=torch.float32, device="cuda")
    assert n_items % 256 == 0                                  # no padding columns in the dump
    check(L.b200_rank_tc_debug_scores(ptr(dUb), len(big), ptr(dV), n_items, k, None, ptr(out), out.numel(), ptr(ws),
                                      nbytes, current_stream()), "b200_rank_tc_debug_scores")
    approx = out[:len(big)]
    kth = approx.topk(topk, dim=1).values[:, -1:]
    assert int((approx >= kth).sum(dim=1).min()) > FW_KEYS
    del ws, out

    def call():
        return engine.rank_topk(dU, dV, topk, user_off=d_uoff)

    got, n = _launched(L, call)
    assert n == _tc_launches(2)                                # no row overflowed
    rows = _rows(rng, n_q, chunk, big)
    _check_oracle(*got, rows, U, None, V, None, uoff, np.zeros(n_q + 1, np.int64), np.zeros(0, np.int32), topk)
    _check_exact_path(monkeypatch, L, call, got, n_q, n_items, k, topk)


@pytest.mark.parametrize("k", [64, 128])
def test_factor_rows_four_bytes_off_a_16_byte_boundary(monkeypatch, k):
    """V and U contiguous views 4 bytes into a flat buffer: the norm kernel drops its float4 loads and the finish runs
    unstaged (rank_tc_finish_kernel<false>, scalar gathers) with k a multiple of 4"""
    import torch
    from cornac_b200 import engine
    L = engine.require_cuda()
    n_q, n_items, topk = 3000, 5000, 100
    rng = np.random.RandomState(k)
    U = rng.normal(0, 0.3, (n_q, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    uoff = rng.normal(0, 0.3, n_q).astype(np.float32)
    indptr, indices = _exclusions(rng, n_q, n_items)

    def misaligned(a):
        flat = torch.empty(a.size + 1, dtype=torch.float32, device="cuda")
        t = flat[1:].view(a.shape)
        t.copy_(torch.from_numpy(a))
        assert t.is_contiguous() and t.data_ptr() % 16 == 4
        return t

    dU, dV = misaligned(U), misaligned(V)
    dB, d_uoff, dp, dx = map(_dev, (base, uoff, indptr, indices))

    def call():
        return engine.rank_topk(dU, dV, topk, item_base=dB, user_off=d_uoff, excl_indptr=dp, excl_indices=dx)

    got, n = _launched(L, call)
    assert n == _tc_launches(1, staged=False)
    _check_oracle(*got, _rows(rng, n_q, n_q), U, None, V, base, uoff, indptr, indices, topk)
    _check_exact_path(monkeypatch, L, call, got, n_q, n_items, k, topk)


def test_exact_path_over_several_slabs():
    """1000 items (below the tensor-core pass's minimum): 140,000 queries in slabs of 256 MiB of scores, with the
    query-row offsets of U, user_off, the exclusions and the outputs in every slab after the first"""
    from cornac_b200 import engine
    L = engine.require_cuda()
    n_q, k, n_items, topk = 140000, 64, 1000, 100
    assert int(L.b200_rank_items_bytes(n_items, k)) == 0       # the exact path
    slab = _ws(L, 1 << 40, n_items, k, topk) // (4 * n_items)
    assert _ceil(n_q, slab) == 3
    rng = np.random.RandomState(23)
    U = rng.normal(0, 0.3, (n_q, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    uoff = rng.normal(0, 0.3, n_q).astype(np.float32)
    indptr, indices = _exclusions(rng, n_q, n_items)
    dU, dV, dB, d_uoff, dp, dx = map(_dev, (U, V, base, uoff, indptr, indices))
    got, n = _launched(L, lambda: engine.rank_topk(dU, dV, topk, item_base=dB, user_off=d_uoff, excl_indptr=dp,
                                                   excl_indices=dx))
    assert n == 2 * 3
    _check_oracle(*got, _rows(rng, n_q, slab), U, None, V, base, uoff, indptr, indices, topk)


def test_score_batch_f64_past_the_grid_height():
    """600,000 queries against 7 items: 75,000 query groups of 8, more than the grid's 65,535 rows, so every block
    loops over gridDim.y; every row == the index-order f64 sum"""
    import torch
    from cornac_b200 import engine
    L = engine.require_cuda()
    n_q, n_items, k = 600000, 7, 5
    rng = np.random.RandomState(29)
    U, V = rng.normal(0, 1, (1000, k)), rng.normal(0, 1, (n_items, k))
    users = rng.randint(1000, size=n_q)
    dU, dV, d_users = (engine.to_device(a, t) for a, t in ((U, torch.float64), (V, torch.float64),
                                                           (users, torch.int64)))
    got, n = _launched(L, lambda: engine.score_batch_f64(dU, dV, user_idx=d_users))
    assert n == 1
    want = np.zeros((n_q, n_items))
    for f in range(k):
        want = want + U[users, f][:, None] * V[:, f][None, :]
    assert np.array_equal(got.cpu().numpy(), want)
