"""Score / top-k / rank (through the C ABI) against the oracle: bit-exact.  GPU only."""
import numpy as np
import pytest

from conftest import golden
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def _dev(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).cuda()


@pytest.mark.parametrize("k,n_items,n_q", [(1, 5, 3), (2, 2, 1), (10, 1682, 9), (32, 257, 17), (64, 1000, 8),
                                           (100, 4099, 5), (128, 2048, 33), (200, 300, 2),
                                           (16, 7, 600000)])        # 75,000 query groups: the grid's y loop wraps
def test_score_batch_bit_exact(k, n_items, n_q):
    from cornac_b200 import engine
    rng = np.random.RandomState(k * 7 + n_items)
    U = rng.normal(0, 0.3, (50, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    uidx = rng.randint(50, size=n_q).astype(np.int64)
    uoff = rng.normal(0, 0.3, n_q).astype(np.float32)
    want = O.score_batch(U[uidx], V, base, uoff)
    got = engine.score_batch(_dev(U), _dev(V), user_idx=_dev(uidx), item_base=_dev(base), user_off=_dev(uoff))
    assert np.array_equal(got.cpu().numpy(), want)
    want = O.score_batch(U[:n_q], V)
    got = engine.score_batch(_dev(U[:n_q]), _dev(V))
    assert np.array_equal(got.cpu().numpy(), want)


def test_single_user_score_entry_equals_the_batched_one():
    """b200_score (one user, scalar offset: the fast_dot call of BPR.score / MF.score) == row of b200_score_batch, bit for bit."""
    import torch
    from cornac_b200 import _lib, engine
    from cornac_b200._lib import check, current_stream, ptr
    L = _lib.load()
    rng = np.random.RandomState(3)
    k, n_items = 48, 3001
    U = rng.normal(0, 0.3, (20, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    dU, dV, dB = _dev(U), _dev(V), _dev(base)
    out = torch.empty(n_items, dtype=torch.float32, device="cuda")
    for u, off in ((0, 0.0), (7, 0.25), (19, -1.5)):
        check(L.b200_score(ptr(dU), u, ptr(dV), n_items, k, ptr(dB), off, ptr(out), current_stream()), "b200_score")
        want = O.score_batch(U[u:u + 1], V, base, np.array([off], np.float32))[0]
        assert np.array_equal(out.cpu().numpy(), want)
    check(L.b200_score(ptr(dU), 3, ptr(dV), n_items, k, None, 0.0, ptr(out), current_stream()), "b200_score")
    assert np.array_equal(out.cpu().numpy(), O.score_batch(U[3:4], V)[0])


def test_fast_dot_known_answers_on_device():
    # reference: tests/cornac/utils/test_fastdot.py:26-37
    from cornac_b200 import engine
    got = engine.score_batch(_dev(np.ones((1, 2), np.float32)), _dev(np.ones((2, 2), np.float32)))
    assert got.cpu().numpy().tolist() == [[2.0, 2.0]]
    got = engine.score_batch(_dev(np.array([[1, 2]], np.float32)), _dev(np.array([[1, 2], [3, 4]], np.float32)))
    assert got.cpu().numpy().tolist() == [[5.0, 11.0]]


@pytest.mark.parametrize("name", ["bpr_small_k10", "bpr_mid_k32", "mf_mid_k32"])
def test_scores_and_top10_match_reference_golden(name):
    from cornac_b200 import engine
    g = golden(name)
    if name.startswith("bpr"):
        base, uoff = g["B"], None
    else:
        base, uoff = (np.float32(g["mu"]) + g["Bi"]).astype(np.float32), g["Bu"][g["query_users"]]
    sc = engine.score_batch(_dev(g["U"]), _dev(g["V"]), user_idx=_dev(g["query_users"]), item_base=_dev(base),
                            user_off=None if uoff is None else _dev(uoff), n_items=int(g["num_items"]))
    # the reference sums in BLAS order: agreement to f32 rounding, ids identical
    assert np.allclose(sc.cpu().numpy(), g["query_scores"][:, : int(g["num_items"])], rtol=1e-5, atol=1e-6)
    if "excl_indptr" in g.files:
        ids, _ = engine.topk_rows(sc, 10, _dev(g["excl_indptr"].astype(np.int64)), _dev(g["excl_indices"]))
    else:
        ids, _ = engine.topk_rows(sc, 10)
    assert np.array_equal(ids.cpu().numpy(), g["top10"])


def _check_topk(scores, k, excl_lists=None):
    from cornac_b200 import engine
    n_q = scores.shape[0]
    ex_ptr = ex_idx = None
    if excl_lists is not None:
        ptr = np.concatenate([[0], np.cumsum([len(e) for e in excl_lists])]).astype(np.int64)
        flat = np.concatenate([np.sort(e) for e in excl_lists]).astype(np.int32) if ptr[-1] else np.zeros(1, np.int32)
        ex_ptr, ex_idx = _dev(ptr), _dev(flat)
    ids, sc = engine.topk_rows(_dev(scores), k, ex_ptr, ex_idx)
    ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
    for q in range(n_q):
        wi, ws, w = O.topk(scores[q], k, None if excl_lists is None else excl_lists[q])
        assert np.array_equal(ids[q], wi), (q, ids[q][:10], wi[:10])
        assert np.array_equal(sc[q][:w], ws[:w])
        assert np.all(np.isneginf(sc[q][w:]))


@pytest.mark.parametrize("n_items,k", [(1, 1), (5, 3), (31, 31), (33, 10), (1000, 100), (16384, 100), (50001, 1000),
                                        (300000, 100), (1000, 4096)])
def test_topk_rows_bit_exact(n_items, k):
    rng = np.random.RandomState(n_items + k)
    scores = rng.normal(0, 1, (5, n_items)).astype(np.float32)
    _check_topk(scores, k)
    excl = [np.unique(rng.randint(n_items, size=rng.randint(0, min(n_items, 200)))) for _ in range(5)]
    _check_topk(scores, k, excl)


def test_topk_rows_ties_and_degenerate_rows():
    rng = np.random.RandomState(0)
    quant = np.round(rng.normal(0, 1, (4, 5000)) * 4).astype(np.float32) / 4     # massive ties
    quant[0, :100] = -0.0
    quant[0, 100:200] = 0.0
    _check_topk(quant, 100)
    _check_topk(quant, 100, [np.arange(0, 5000, 3)] * 4)
    _check_topk(np.zeros((2, 3000), np.float32), 50)                               # untrained model: all equal
    _check_topk(np.full((1, 700), -np.inf, dtype=np.float32), 10)
    allx = [np.arange(64)]                                                         # everything excluded
    _check_topk(rng.normal(0, 1, (1, 64)).astype(np.float32), 5, allx)
    neg = -np.abs(rng.normal(0, 1, (3, 999))).astype(np.float32)                   # all negative keys
    _check_topk(neg, 17)


@pytest.mark.parametrize("k,n_items,n_q,topk", [(10, 1682, 40, 10), (64, 20000, 300, 100), (128, 5000, 64, 100)])
def test_rank_topk_equals_score_then_topk(k, n_items, n_q, topk):
    import torch
    from cornac_b200._lib import load, check, ptr, current_stream
    rng = np.random.RandomState(k)
    U = rng.normal(0, 0.3, (1000, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    base = rng.normal(0, 0.3, n_items).astype(np.float32)
    uidx = rng.randint(1000, size=n_q).astype(np.int64)
    excl = [np.unique(rng.randint(n_items, size=rng.randint(0, 150))) for _ in range(n_q)]
    ex_ptr = np.concatenate([[0], np.cumsum([len(e) for e in excl])]).astype(np.int64)
    ex_idx = np.concatenate(excl).astype(np.int32)
    L = load()
    ids = torch.empty((n_q, topk), dtype=torch.int32, device="cuda")
    sc = torch.empty((n_q, topk), dtype=torch.float32, device="cuda")
    nbytes = L.b200_rank_topk_workspace_bytes(n_q, n_items, k, topk)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dU, dV, db, du, dp, dx = _dev(U), _dev(V), _dev(base), _dev(uidx), _dev(ex_ptr), _dev(ex_idx)
    check(L.b200_rank_topk(ptr(dU), ptr(du), n_q, ptr(dV), n_items, k, ptr(db), None, ptr(dp), ptr(dx), topk,
                           ptr(ids), ptr(sc), ptr(ws), nbytes, current_stream()), "b200_rank_topk")
    want_scores = O.score_batch(U[uidx], V, base)
    ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
    for q in range(n_q):
        wi, wsc, w = O.topk(want_scores[q], topk, excl[q])
        assert np.array_equal(ids[q], wi) and np.array_equal(sc[q][:w], wsc[:w])
