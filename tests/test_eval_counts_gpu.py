"""The device evaluation kernels (csrc/eval.cu) at the inputs where counts go wrong, and the batched ranking_eval
(cornac_b200/evaluation.py) against the reference's per-user loop, user by user.

  * b200_rank_counts against an exact numpy restatement: ties between positives and candidates, -0.0 next to +0.0, +-inf,
    all-equal rows, up to ~3000 positives per user (several 1024-wide passes of the kernel), more score rows than one grid
    wave, rows sharing a positives row, out-of-range exclusions, 1 to 300 000 items;
  * b200_topk_metrics against the reference metric classes: several grid waves of lists, ids_stride > topk, 1 and 32
    metrics, positive rows longer than the list (and than 4096), all -1 lists;
  * ranking_eval on exactly tied f32 scores and a trained MF, users with more than 1024 / 2048 test positives, several
    score slabs, @k chunks and the vectorised MAP, with the reference loop forbidden during the batched call; NaN scores
    and a test set without a positive at the threshold give what the reference loop gives."""
import functools
from collections import OrderedDict

import numpy as np
import pytest

from conftest import needs_cornac

pytestmark = pytest.mark.gpu


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _csr(rows):
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    idx = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows]) if rows else np.zeros(0, np.int32)
    return ptr, idx.astype(np.int32)


# ---------------------------------------------------------------------------------------------------- b200_rank_counts
_OUT_OF_RANGE = (-2 ** 31, -1)                        # plus n_items, n_items + 7 and 2**31 - 1 per case


def _scores(rng, kind, shape):
    if kind == "continuous":
        return rng.standard_normal(shape).astype(np.float32)
    if kind == "quantised":                           # few levels: positives tie with each other and with candidates
        return rng.choice(np.array([-1.0, -0.0, 0.0, 0.5, 1.0], np.float32), size=shape)
    assert kind == "infinities"
    return rng.choice(np.array([-np.inf, -1.0, 0.0, 2.0, np.inf], np.float32), size=shape)


def _rank_counts_case(name, sms):
    """(scores [n_q, n_items] f32, positives rows per user, user_idx or None, exclusion rows per score row)"""
    rng = np.random.RandomState(sum(map(ord, name)))
    waves = 8 * sms + 61                               # more rows than the kernel's grid (8 blocks per SM)
    if name in ("continuous", "quantised", "infinities"):
        n_items, n_users = 1500, waves
        pos = [np.sort(rng.choice(n_items, size=(1, 2, 3, 5, 7, int(rng.randint(8, 60)))[u % 6], replace=False))
               for u in range(n_users)]
        uidx = None
        scores = _scores(rng, name, (waves, n_items))
        if name == "quantised":
            scores[::17] = 0.5                         # all-equal rows
            scores[5] = rng.choice(np.array([-0.0, 0.0], np.float32), size=n_items)
        if name == "infinities":                       # every positive at +inf, every positive at -inf
            scores[3, pos[3]] = np.inf
            scores[4, pos[4]] = -np.inf
            scores[10, :] = np.inf
    elif name == "shared_rows":                        # a permuted user_idx with repeats: rows share a positives row
        n_items, n_users = 700, 500
        pos = [np.sort(rng.choice(n_items, size=int(rng.randint(1, 40)), replace=False)) for _ in range(n_users)]
        uidx = np.concatenate([rng.permutation(n_users), rng.randint(0, n_users, size=waves - n_users)]).astype(np.int64)
        scores = _scores(rng, "quantised", (waves, n_items))
    elif name == "long_rows":                          # 1024-wide passes; quantised rows tie across pass boundaries
        n_items = 4000
        counts = [1023, 1024, 1025, 2048, 3001]
        kinds = ["continuous", "quantised", "infinities"]
        pos = [np.sort(rng.choice(n_items, size=c, replace=False)) for c in counts for _ in kinds]
        uidx = None
        scores = np.stack([_scores(rng, k, n_items) for _ in counts for k in kinds])
    elif name == "one_item":
        n_items = 1
        pos = [np.array([0])] * 5
        uidx = None
        scores = np.array([[0.0], [-0.0], [np.inf], [-np.inf], [3.0]], np.float32)
    elif name == "all_excluded_but_positives":
        n_items = 31
        pos = [np.sort(rng.choice(n_items, size=int(rng.randint(1, n_items + 1)), replace=False)) for _ in range(40)]
        uidx = None
        scores = _scores(rng, "quantised", (40, n_items))
    else:
        assert name == "wide"
        n_items = 300_000
        pos = [np.sort(rng.choice(n_items, size=c, replace=False)) for c in (1, 1025, 7, 3)]
        uidx = None
        scores = np.stack([_scores(rng, k, n_items) for k in ("continuous", "quantised", "infinities", "continuous")])
    n_q = len(scores)
    bad = list(_OUT_OF_RANGE) + [n_items, n_items + 7, 2 ** 31 - 1]
    excl, first_row = [], {}
    for q in range(n_q):
        u = q if uidx is None else int(uidx[q])
        if u in first_row:                             # rows of one user: same scores and exclusions, so that the
            scores[q] = scores[first_row[u]]           # positives' counts they write agree
            excl.append(excl[first_row[u]])
            continue
        first_row[u] = q
        others = np.setdiff1d(np.arange(n_items), pos[u])
        if name == "all_excluded_but_positives":
            e = others
        elif q % 5 == 0 or len(others) == 0:
            e = np.zeros(0, np.int64)                  # nothing excluded
        else:
            e = rng.choice(others, size=min(len(others), int(rng.randint(1, 200))), replace=False)
        if q % 3 == 0:
            e = np.concatenate([e, rng.choice(bad, size=2, replace=False)])
        excl.append(np.sort(e.astype(np.int64)).astype(np.int32))
    return scores, pos, uidx, excl


def _restate_rank_counts(scores, pos_ptr, pos_idx, uidx, excl):
    """less_p = #{c in C : s_c < s_p}, n_cand = |C|, before = #{c in C : s_c > s_b or (s_c == s_b and c < b)} with b the
    positive of largest score, smallest id among equals; C = all items minus the in-range exclusions."""
    n_q, n_items = scores.shape
    less = np.full(len(pos_idx), -7, np.int64)
    pscore = np.full(len(pos_idx), -7.0, np.float32)
    n_cand, before = np.empty(n_q, np.int64), np.empty(n_q, np.int64)
    for q in range(n_q):
        u = q if uidx is None else int(uidx[q])
        row = scores[q]
        cand = np.ones(n_items, dtype=bool)
        e = excl[q].astype(np.int64)
        cand[e[(e >= 0) & (e < n_items)]] = False
        cs = np.sort(row[cand])
        lo, hi = pos_ptr[u], pos_ptr[u + 1]
        p = pos_idx[lo:hi].astype(np.int64)
        less[lo:hi] = np.searchsorted(cs, row[p], side="left")
        pscore[lo:hi] = row[p]
        n_cand[q] = len(cs)
        b = p[np.lexsort((p, -row[p].astype(np.float64)))[0]]
        cid = np.flatnonzero(cand)
        cv = row[cid]
        before[q] = int(np.sum(cv > row[b]) + np.sum((cv == row[b]) & (cid < b)))
    return less, pscore, n_cand, before


@pytest.mark.parametrize("name", ["continuous", "quantised", "infinities", "shared_rows", "long_rows", "one_item",
                                  "all_excluded_but_positives", "wide"])
def test_rank_counts_equal_an_exact_restatement(name):
    import torch
    from cornac_b200 import engine
    scores, pos, uidx, excl = _rank_counts_case(name, _sms())
    n_q, n_items = scores.shape
    pos_ptr, pos_idx = _csr(pos)
    ex_ptr, ex_idx = _csr(excl)
    want_less, want_ps, want_nc, want_bf = _restate_rank_counts(scores, pos_ptr, pos_idx, uidx, excl)

    dev = torch.from_numpy(scores.copy()).cuda()
    less = torch.full((len(pos_idx),), -7, dtype=torch.int64, device="cuda")
    ps = torch.full((len(pos_idx),), -7.0, dtype=torch.float32, device="cuda")
    ei = torch.from_numpy(ex_idx).cuda() if len(ex_idx) else torch.zeros(1, dtype=torch.int32, device="cuda")
    got_less, got_ps, nc, bf = engine.rank_counts(
        dev, torch.from_numpy(pos_ptr).cuda(), torch.from_numpy(pos_idx).cuda(),
        user_idx=None if uidx is None else torch.from_numpy(uidx).cuda(), excl_indptr=torch.from_numpy(ex_ptr).cuda(),
        excl_indices=ei, less=less, pos_score=ps)
    got_less, got_ps = got_less.cpu().numpy(), got_ps.cpu().numpy()
    # every listed positive written, nothing else (the sentinel -7 stays), integers equal, scores bit-equal
    assert np.array_equal(got_less, want_less), np.flatnonzero(got_less != want_less)[:10]
    assert np.array_equal(got_ps.view(np.uint32), want_ps.view(np.uint32))
    assert np.array_equal(nc.cpu().numpy(), want_nc)
    assert np.array_equal(bf.cpu().numpy(), want_bf), np.flatnonzero(bf.cpu().numpy() != want_bf)[:10]
    if name == "all_excluded_but_positives":
        assert np.array_equal(want_nc, np.diff(pos_ptr))
    # the documented side effect: NaN exactly at the in-range exclusions, every other score untouched
    blanked = scores.copy()
    for q in range(n_q):
        e = excl[q].astype(np.int64)
        blanked[q, e[(e >= 0) & (e < n_items)]] = np.nan
    after = dev.cpu().numpy()
    assert np.array_equal(np.isnan(after), np.isnan(blanked))
    keep = ~np.isnan(blanked)
    assert np.array_equal(after[keep].view(np.uint32), scores[keep].view(np.uint32))


def test_rank_counts_with_nan_positive_scores_write_exactly_the_listed_positives():
    """A NaN score reads as an excluded item, so a NaN positive has no defined count; still every listed positive gets
    its own less / pos_score slot (NaN and +inf positives sort inside the pass, never the padding), and no other slot
    is written."""
    import torch
    from cornac_b200 import engine
    rng = np.random.RandomState(3)
    n_items, n_users = 3000, 40
    pos = [np.sort(rng.choice(n_items, size=s, replace=False)) for s in rng.choice([1, 3, 6, 700, 1025, 2100], n_users)]
    pos_ptr, pos_idx = _csr(pos)
    uidx = np.array([0, 1, 2, 5, 8, 13, 21, 34, 3, 7], dtype=np.int64)              # not every user is listed
    scores = _scores(rng, "infinities", (len(uidx), n_items))
    for q, u in enumerate(uidx):
        p = pos[u]
        scores[q, rng.choice(p, size=max(1, len(p) // 3), replace=False)] = np.nan     # NaN positives
        scores[q, rng.choice(n_items, size=50, replace=False)] = np.nan                 # NaN candidates
    less = torch.full((len(pos_idx),), -7, dtype=torch.int64, device="cuda")
    ps = torch.full((len(pos_idx),), -7.0, dtype=torch.float32, device="cuda")
    got_less, got_ps, nc, _ = engine.rank_counts(torch.from_numpy(scores.copy()).cuda(), torch.from_numpy(pos_ptr).cuda(),
                                                 torch.from_numpy(pos_idx).cuda(), user_idx=torch.from_numpy(uidx).cuda(),
                                                 less=less, pos_score=ps)
    got_less, got_ps = got_less.cpu().numpy(), got_ps.cpu().numpy()
    listed = np.zeros(len(pos_idx), dtype=bool)
    want_ps = np.full(len(pos_idx), -7.0, np.float32)
    for q, u in enumerate(uidx):
        lo, hi = pos_ptr[u], pos_ptr[u + 1]
        listed[lo:hi] = True
        want_ps[lo:hi] = scores[q, pos_idx[lo:hi]]
        assert np.all((got_less[lo:hi] >= 0) & (got_less[lo:hi] <= nc[q].item()))
    assert np.all(got_less[~listed] == -7)
    assert np.array_equal(got_ps.view(np.uint32), want_ps.view(np.uint32))
    assert np.array_equal(nc.cpu().numpy(), (~np.isnan(scores)).sum(axis=1))


# --------------------------------------------------------------------------------------------------- b200_topk_metrics
def _topk_case(name, rng):
    """(ids [n_q, stride] int32, topk, positives rows per user, user_idx, metrics)"""
    from cornac.metrics import FMeasure, HitRatio, NCRR, NDCG, Precision, Recall
    kinds = (NDCG, NCRR, Precision, Recall, FMeasure, HitRatio)
    n_items, topk, stride, n_q, npos_hi = 200, 10, 10, 64, 30
    if name == "grid_waves":
        n_q = 20000
        metrics = [NDCG(k=10), Recall(k=7), HitRatio(k=1), FMeasure(k=10)]
    elif name == "ids_stride":
        stride = 24
        metrics = [NDCG(k=10), NCRR(k=10), Precision(k=3), Recall(k=10)]
    elif name == "one_metric":
        topk = stride = 16
        metrics = [NCRR(k=7)]
    elif name == "thirty_two_metrics":
        topk = stride = 64
        metrics = [cls(k=k) for k in (1, 5, 17, 40, 64) for cls in kinds] + [NDCG(k=2), HitRatio(k=63)]
    elif name == "long_positive_rows":
        n_items, topk, stride, npos_hi = 12000, 50, 50, 6000
        metrics = [cls(k=k) for k in (10, 50) for cls in kinds]
    else:
        assert name == "all_minus_one"
        metrics = [cls(k=10) for cls in kinds]
    n_users = n_q // 2 + 1
    sizes = rng.randint(1, npos_hi + 1, size=n_users)
    if name == "long_positive_rows":
        sizes[:3] = (topk + 1, 4097, npos_hi)
    pos = [np.sort(rng.choice(n_items, size=int(s), replace=False)) for s in sizes]
    uidx = rng.randint(0, n_users, size=n_q).astype(np.int64)
    ids = np.full((n_q, stride), -1, dtype=np.int32)
    for q in range(n_q):
        if name == "all_minus_one":
            break
        n_valid = topk if q % 5 else int(rng.randint(0, topk + 1))
        lst = rng.choice(n_items, size=n_valid, replace=False)
        hot = pos[uidx[q]]
        take = rng.rand(n_valid) < 0.4
        lst[take] = rng.choice(hot, size=int(take.sum()))
        _, first = np.unique(lst, return_index=True)
        lst = lst[np.sort(first)]
        ids[q, :len(lst)] = lst
        if stride > topk:                             # beyond topk: positives that would count if read
            ids[q, topk:] = rng.choice(hot, size=stride - topk)
    return ids, topk, pos, uidx, metrics


@needs_cornac
@pytest.mark.parametrize("name", ["grid_waves", "ids_stride", "one_metric", "thirty_two_metrics", "long_positive_rows",
                                  "all_minus_one"])
def test_topk_metrics_equal_the_reference_metric_classes_at_the_edges(name):
    import torch
    from cornac.metrics import FMeasure, HitRatio, NCRR, NDCG, Precision, Recall
    from cornac_b200 import _lib, engine
    ids, topk, pos, uidx, metrics = _topk_case(name, np.random.RandomState(len(name)))
    assert len(metrics) <= 32
    kind = {NDCG: _lib.METRIC_NDCG, NCRR: _lib.METRIC_NCRR, Precision: _lib.METRIC_PRECISION,
            Recall: _lib.METRIC_RECALL, FMeasure: _lib.METRIC_FMEASURE, HitRatio: _lib.METRIC_HIT}
    pos_ptr, pos_idx = _csr(pos)
    out = engine.topk_metrics(torch.from_numpy(ids).cuda(), torch.from_numpy(pos_ptr).cuda(),
                              torch.from_numpy(pos_idx).cuda(), [kind[type(m)] for m in metrics], [m.k for m in metrics],
                              user_idx=torch.from_numpy(uidx).cuda(), topk=topk).cpu().numpy()
    assert out.shape == (len(metrics), len(ids))
    n_items = int(pos_idx.max()) + 1
    for q in range(len(ids)):
        row = ids[q, :topk][ids[q, :topk] >= 0]
        # the reference ranks every candidate: fill the list up with items that are nobody's positive
        pd_rank = np.concatenate([row, np.arange(n_items + 8, n_items + 8 + topk)])
        for mi, m in enumerate(metrics):
            want = m.compute(gt_pos=pos[uidx[q]], pd_rank=pd_rank)
            assert abs(out[mi, q] - want) <= 1e-12 * max(1.0, abs(want)), (q, m.name, out[mi, q], want)


# ------------------------------------------------------------------------------------------------ batched ranking_eval
@functools.lru_cache(maxsize=1)
def _eval_sets():
    """~3000 test users over 4000 items: users 0 and 1 with 1500 and 2600 test positives, train ratings on both sides of
    the 4.0 threshold, test items that are also train items, and a validation set."""
    from cornac.data import Dataset
    rng = np.random.RandomState(2024)
    n_users, n_items = 3000, 4000
    rating = lambda: float(rng.randint(1, 6))
    train = OrderedDict()
    for i in range(n_items):                           # every item and user is known to the train set
        train[(i % n_users, i)] = rating()
    for u in range(n_users):
        for i in rng.choice(n_items, size=int(rng.randint(3, 25)), replace=False):
            train[(u, int(i))] = rating()
    test = OrderedDict()
    for u in range(n_users):
        if u % 11 == 10:
            continue                                   # not a test user
        for i in rng.choice(n_items, size=int(rng.randint(1, 8)), replace=False):
            test[(u, int(i))] = rating()
    for u, n in ((0, 1500), (1, 2600)):
        for i in rng.choice(n_items, size=n, replace=False):
            test[(u, int(i))] = float(rng.randint(4, 6))
    val = OrderedDict(((int(u), int(i)), rating()) for u, i in zip(rng.randint(0, n_users, 4000),
                                                                   rng.randint(0, n_items, 4000)))
    triples = lambda d: [(str(u), str(i), r) for (u, i), r in d.items()]
    uid_map, iid_map = OrderedDict(), OrderedDict()
    train_set = Dataset.build(triples(train), global_uid_map=uid_map, global_iid_map=iid_map, seed=1)
    test_set = Dataset.build(triples(test), global_uid_map=uid_map, global_iid_map=iid_map, seed=1, exclude_unknowns=True)
    val_set = Dataset.build(triples(val), global_uid_map=uid_map, global_iid_map=iid_map, seed=1, exclude_unknowns=True)
    return train_set, test_set, val_set


def _tied_bpr(train_set, nan_user=None):
    """BPR scores from small integer factors and biases in {0, 0.5}: every f32 score exact, and heavily tied."""
    from cornac_b200 import BPR
    rng = np.random.RandomState(5)
    U = rng.randint(-1, 3, size=(len(train_set.uid_map), 4)).astype(np.float32)
    V = rng.randint(-1, 2, size=(len(train_set.iid_map), 4)).astype(np.float32)
    Bi = rng.choice(np.array([0.0, 0.5], np.float32), size=len(train_set.iid_map))
    if nan_user is not None:                          # a diverged fit: one user's factors, one item's bias
        U[nan_user, 1] = np.nan
        Bi[7] = np.nan
    return BPR(k=4, trainable=False, init_params={"U": U, "V": V, "Bi": Bi}).fit(train_set)


def _metric_sets():
    from cornac.metrics import AUC, MAP, MRR, FMeasure, HitRatio, NCRR, NDCG, Recall
    return ([AUC(), MAP(), MRR()],
            [AUC(), MAP(), NDCG(k=10), Recall(k=50), NCRR(k=7), HitRatio(k=1), FMeasure(k=100)])


def _assert_same(want, got, rtol):
    (wa, wu), (ga, gu) = want, got
    assert np.allclose(wa, ga, rtol=rtol, atol=1e-15, equal_nan=True), (wa, ga)
    for a, b in zip(wu, gu):
        assert list(a.keys()) == list(b.keys())
        x, y = np.array(list(a.values()), np.float64), np.array(list(b.values()), np.float64)
        bad = ~np.isclose(x, y, rtol=rtol, atol=1e-15, equal_nan=True)
        assert not bad.any(), (np.array(list(a.keys()))[bad][:5], x[bad][:5], y[bad][:5])


def _forbid_reference(*args, **kwargs):
    raise AssertionError("the batched ranking_eval delegated to the reference loop")


@needs_cornac
@pytest.mark.parametrize("model_name", ["tied_bpr", "mf"])
def test_batched_ranking_eval_equals_the_reference_loop_at_ties_long_rows_and_many_batches(model_name, monkeypatch):
    from cornac.eval_methods.base_method import ranking_eval as ref_eval
    from cornac.metrics import MAP
    from cornac_b200 import MF, evaluation
    train_set, test_set, val_set = _eval_sets()
    mdl = _tied_bpr(train_set) if model_name == "tied_bpr" else \
        MF(k=8, max_iter=5, learning_rate=0.01, use_bias=True, seed=3).fit(train_set)
    n_items = train_set.num_items
    slab_rows = 600
    monkeypatch.setattr(evaluation, "_SCORE_SLAB_BYTES", 4 * n_items * slab_rows)
    test_pos = evaluation._positives(test_set.csr_matrix, 4.0, test_set.csr_matrix.shape[0], n_items)
    npos = np.diff(test_pos.indptr)
    assert npos.max() > 2048 and np.sum(npos > 1024) >= 2
    assert np.sum(npos > 0) > 3 * slab_rows and np.sum(npos > 0) > 3 * 700          # >= 4 slabs, >= 4 @k chunks
    kw = dict(val_set=val_set, exclude_unknowns=True)
    for metrics in _metric_sets():
        for thr in (1.0, 4.0):
            want = ref_eval(mdl, metrics, train_set, test_set, rating_threshold=thr, **kw)
            with monkeypatch.context() as m:
                m.setattr(evaluation, "_reference_ranking_eval", _forbid_reference)
                got = evaluation.ranking_eval(mdl, metrics, train_set, test_set, rating_threshold=thr, batch_users=700, **kw)
                _assert_same(want, got, rtol=1e-12)
                if thr == 4.0 and len(metrics) == 3:
                    # the vectorised MAP reduction (f64 instead of the loop's own dtype): rounding differences only
                    m.setattr(evaluation, "_MAP_EXACT_USERS", 0)
                    got = evaluation.ranking_eval(mdl, [MAP()], train_set, test_set, rating_threshold=thr, **kw)
                    _assert_same(ref_eval(mdl, [MAP()], train_set, test_set, rating_threshold=thr, **kw), got, rtol=1e-6)


@needs_cornac
def test_nan_scores_give_the_reference_loop_results():
    """A diverged fit scores NaN; b200_rank_counts would read NaN as an excluded item, the reference loop keeps it as a
    candidate (a negative in AUC, NaN for MAP): the batched call returns the reference loop's numbers."""
    from cornac.eval_methods.base_method import ranking_eval as ref_eval
    from cornac_b200 import evaluation
    train_set, test_set, val_set = _eval_sets()
    mdl = _tied_bpr(train_set, nan_user=0)
    assert not mdl._b200_scores_nan_free()
    for metrics in _metric_sets():
        want = ref_eval(mdl, metrics, train_set, test_set, rating_threshold=4.0, val_set=val_set)
        got = evaluation.ranking_eval(mdl, metrics, train_set, test_set, rating_threshold=4.0, val_set=val_set)
        _assert_same(want, got, rtol=1e-12)
        assert np.isnan(got[1][1][0])                  # MAP of the NaN user, as scipy's rankdata gives it


@needs_cornac
def test_scores_nan_free_follows_the_parameters():
    """NaN needs a non-finite parameter or item_base + user_off overflowing next to an opposite infinite dot product."""
    from cornac_b200 import MF
    train_set, _, _ = _eval_sets()
    n_u, n_i = len(train_set.uid_map), len(train_set.iid_map)

    def mf(**changes):
        p = dict(U=np.ones((n_u, 2), np.float32), V=np.ones((n_i, 2), np.float32), Bu=np.zeros(n_u, np.float32),
                 Bi=np.zeros(n_i, np.float32))
        for key, (pos, val) in changes.items():
            p[key][pos] = val
        return MF(k=2, trainable=False, use_bias=True, init_params=p).fit(train_set)

    big = np.float32(3e38)
    assert mf()._b200_scores_nan_free()
    assert mf(Bi=(0, big), V=((0, 0), big))._b200_scores_nan_free()       # an inf score, no NaN
    assert not mf(U=((0, 1), np.nan))._b200_scores_nan_free()
    assert not mf(V=((5, 0), -np.inf))._b200_scores_nan_free()
    assert not mf(Bi=(0, big), Bu=(1, big))._b200_scores_nan_free()        # the f32 bias sum can overflow


@needs_cornac
def test_no_test_positive_at_the_threshold_raises_what_the_reference_raises():
    from cornac.eval_methods.base_method import ranking_eval as ref_eval
    from cornac_b200 import evaluation
    train_set, test_set, _ = _eval_sets()
    mdl = _tied_bpr(train_set)
    for metrics in _metric_sets():
        with pytest.raises(ZeroDivisionError):
            ref_eval(mdl, metrics, train_set, test_set, rating_threshold=6.0)
        with pytest.raises(ZeroDivisionError):
            evaluation.ranking_eval(mdl, metrics, train_set, test_set, rating_threshold=6.0)
