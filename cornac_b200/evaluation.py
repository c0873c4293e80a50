"""Batched, device-side replacement of the per-user loop of cornac's `ranking_eval`.

Reference: `cornac/eval_methods/base_method.py:108-226` iterates over the test users in Python and, for each, builds two
dense item masks, calls `model.rank(user, item_indices, k)` and feeds the ranked list to every metric
(`cornac/metrics/ranking.py`).  Here the candidate sets are expressed as per-user exclusion lists (train / validation
positives that are not test positives) and ALL users are handled in batches on the GPU:

  * the @k metrics (NDCG, NCRR, Precision, Recall, FMeasure, HitRatio with k > 0) only look at `pd_rank[:k]`:
    `rank_batch_device` (one fused tensor-core kernel per chunk of users) + `b200_topk_metrics` (csrc/eval.cu);
  * the full-vector metrics AUC, MAP (and MRR when no metric carries a cut-off) need, per test positive, the number of
    candidates scoring below it: `b200_score_batch` rows + `b200_rank_counts` (csrc/eval.cu) -- the score matrix of a batch
    of users never leaves the device, only the integer counts of the positives do, and the ratios are formed in f64 with
    the reference's own formulas (ranking.py:473-485 AUC, :522-525 MAP, :213-222 MRR).

Anything else (custom metrics, MRR next to @k metrics -- the reference then evaluates it on a partially sorted list --
`exclude_unknowns=False`, models without the batched entry points, models whose scores could be NaN (a diverged fit), a
test set without a positive at the threshold) is delegated to the reference implementation unchanged.
Results are the numbers the reference loop produces with the same model (same order: score desc, item id asc).
SURVEY.md section 8, row (f)2.
"""
import numpy as np
import scipy.sparse as sp
import torch

from cornac.eval_methods.base_method import ranking_eval as _reference_ranking_eval
from cornac.metrics import AUC, MAP, MRR, FMeasure, HitRatio, NCRR, NDCG, Precision, Recall

from . import _lib, engine

# most-derived classes first is not needed: none of these derives from another one in the list
_KIND = ((NDCG, _lib.METRIC_NDCG), (NCRR, _lib.METRIC_NCRR), (Precision, _lib.METRIC_PRECISION),
         (Recall, _lib.METRIC_RECALL), (FMeasure, _lib.METRIC_FMEASURE), (HitRatio, _lib.METRIC_HIT))
_TOPK_ONLY = tuple(c for c, _ in _KIND)
_FULL = (AUC, MAP, MRR)
_SCORE_SLAB_BYTES = 1 << 30                     # score rows kept on the device at a time by the full-vector path
# MAP of the reference is (L / rank).mean() with L, rank = scipy.stats.rankdata(..., "max") of float32 scores
# (ranking.py:522-525): the arithmetic runs in whatever dtype this scipy returns for float32 input -- reproduced exactly
try:
    from scipy.stats import rankdata as _rankdata
    _MAP_DTYPE = _rankdata(np.zeros(2, dtype=np.float32), "max").dtype
except Exception:                               # pragma: no cover
    _MAP_DTYPE = np.dtype(np.float64)
_MAP_EXACT_USERS = 500_000                      # above this many users MAP is reduced vectorised (f64; differs from the f32 loop by rounding only)


def _kind(metric):
    for cls, kind in _KIND:
        if type(metric) is cls:
            return kind
    raise TypeError(type(metric).__name__)


def _positives(mat, threshold, n_rows, n_cols):
    """CSR 0/1 matrix of the entries with rating >= threshold, reshaped to [n_rows, n_cols]."""
    m = mat.tocsr()
    keep = m.data >= threshold
    rows = np.repeat(np.arange(m.shape[0]), np.diff(m.indptr))[keep]
    cols = m.indices[keep]
    ok = (rows < n_rows) & (cols < n_cols)
    return sp.csr_matrix((np.ones(int(ok.sum()), dtype=np.int8), (rows[ok], cols[ok])), shape=(n_rows, n_cols))


def _supported(model, metrics, exclude_unknowns, train_set):
    if not (hasattr(model, "rank_batch_device") and exclude_unknowns):
        return False
    max_k = max(m.k for m in metrics)
    for m in metrics:
        if type(m) in _TOPK_ONLY:
            if not (0 < m.k <= 4096):                       # b200_topk_rows / b200_topk_metrics: topk <= 4096
                return False
        elif type(m) in (AUC, MAP):
            continue
        elif type(m) is MRR:
            if max_k != -1:                                 # the reference scans a list that is only sorted up to max_k
                return False
        else:
            return False
    try:
        n_score = model._b200_shape()[1]
    except Exception:
        return False
    # every train item has a score row; and no score is NaN: b200_rank_counts reads NaN as an excluded item, while the
    # reference loop keeps it as a candidate (a negative in AUC, a NaN MAP, a place in the ranked list)
    return n_score >= train_set.num_items and model._b200_scores_nan_free()


def _rank_within_segments(seg, score):
    """for entries grouped in segments: number of entries of the same segment with a strictly smaller score"""
    n = len(seg)
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    order = np.lexsort((score, seg))
    s_sorted, g_sorted = score[order], seg[order]
    seg_start = np.zeros(n, dtype=np.int64)
    new_seg = np.concatenate([[True], g_sorted[1:] != g_sorted[:-1]])
    seg_start = np.maximum.accumulate(np.where(new_seg, np.arange(n), 0))
    new_grp = new_seg | np.concatenate([[True], s_sorted[1:] != s_sorted[:-1]])
    grp_start = np.maximum.accumulate(np.where(new_grp, np.arange(n), 0))
    less_sorted = grp_start - seg_start
    out = np.empty(n, dtype=np.int64)
    out[order] = less_sorted
    return out


def ranking_eval(model, metrics, train_set, test_set, val_set=None, rating_threshold=1.0, exclude_unknowns=True,
                 verbose=False, batch_users=75776):
    """Same signature and return value as cornac.eval_methods.base_method.ranking_eval."""
    if len(metrics) == 0:
        return [], []
    if not _supported(model, metrics, exclude_unknowns, train_set):
        return _reference_ranking_eval(model, metrics, train_set, test_set, val_set=val_set,
                                       rating_threshold=rating_threshold, exclude_unknowns=exclude_unknowns,
                                       verbose=verbose)
    n_items = train_set.num_items                               # exclude_unknowns: candidates are the train items
    n_rows = max(test_set.csr_matrix.shape[0], train_set.csr_matrix.shape[0])
    test_pos = _positives(test_set.csr_matrix, rating_threshold, n_rows, n_items)
    seen = _positives(train_set.csr_matrix, rating_threshold, n_rows, n_items)
    if val_set is not None:
        seen = seen + _positives(val_set.csr_matrix, rating_threshold, n_rows, n_items)
    excl = (seen - seen.multiply(test_pos)).tocsr()             # train/val positives that are not test positives
    excl.eliminate_zeros()
    excl.sort_indices()
    test_pos.sort_indices()

    # same user order as the reference loop (`for user_idx in set(test_set.uir_tuple[0])`), same skip rule
    full_test = _positives(test_set.csr_matrix, rating_threshold, n_rows, test_set.csr_matrix.shape[1])
    users = np.fromiter((u for u in set(test_set.uir_tuple[0]) if full_test.indptr[u + 1] > full_test.indptr[u]),
                        dtype=np.int64)
    n_model_users = model._b200_shape()[0]
    if (len(users) == 0 or users.max() >= n_model_users or users.min() < 0
            or np.any(test_pos.indptr[users + 1] == test_pos.indptr[users])):
        # no user with a test positive (the reference's average then divides by zero), users the model has no row for
        # (the reference scores them through its unknown-user branch), or users whose test positives are all unknown
        # items (the reference then divides by zero per metric): not batched, so the caller sees the reference's result
        return _reference_ranking_eval(model, metrics, train_set, test_set, val_set=val_set,
                                       rating_threshold=rating_threshold, exclude_unknowns=exclude_unknowns,
                                       verbose=verbose)
    per_metric = np.empty((len(metrics), len(users)), dtype=np.float64)
    topk_idx = [i for i, m in enumerate(metrics) if type(m) in _TOPK_ONLY]
    full_idx = [i for i, m in enumerate(metrics) if type(m) in _FULL]
    pos_ptr = engine.to_device(test_pos.indptr.astype(np.int64), torch.int64)
    pos_idx = engine.to_device(test_pos.indices.astype(np.int32) if test_pos.nnz else np.zeros(1, np.int32),
                               torch.int32)

    if topk_idx:
        kinds = [_kind(metrics[i]) for i in topk_idx]
        ks = [int(metrics[i].k) for i in topk_idx]
        max_k = max(ks)
        for b0 in range(0, len(users), batch_users):
            ub = users[b0:b0 + batch_users]
            ids, _ = model.rank_batch_device(ub, max_k, exclude=excl, n_items=n_items)    # [n, max_k] int32 CUDA, -1 padded
            vals = engine.topk_metrics(ids, pos_ptr, pos_idx, kinds, ks, user_idx=engine.to_device(ub, torch.int64))
            per_metric[topk_idx, b0:b0 + len(ub)] = vals.cpu().numpy()

    if full_idx:
        _full_vector_metrics(model, [metrics[i] for i in full_idx], users, test_pos, excl, n_items, pos_ptr, pos_idx,
                             per_metric, full_idx)

    # per-user values carry the dtype the reference's metric returns (MAP: the dtype of scipy's rankdata, float32 here),
    # so that the reference's own averaging expression `sum(values) / len(values)` rounds the same way
    user_results = []
    for m, vals in zip(metrics, per_metric):
        if type(m) is MAP and _MAP_DTYPE != np.float64:
            user_results.append(dict(zip(users.tolist(), list(vals.astype(_MAP_DTYPE)))))
        else:
            user_results.append(dict(zip(users.tolist(), vals.tolist())))
    avg_results = [sum(r.values()) / len(r) for r in user_results]
    return avg_results, user_results


def _full_vector_metrics(model, metrics, users, test_pos, excl, n_items, pos_ptr, pos_idx, per_metric, rows_out):
    """AUC / MAP / MRR of `users` from device score rows: per positive p of a user with candidate set C (|C| = n_cand) and
    positives P,  less_p = #{c in C : s_c < s_p}  (b200_rank_counts),  lessP_p = #{p' in P : s_p' < s_p}:
        AUC = sum_p (less_p - lessP_p) / (|P| (|C| - |P|))                         ranking.py:473-485
        AP  = mean_p ((|P| - lessP_p) / (|C| - less_p))      rankdata(.., "max")   ranking.py:522-525
        MRR = 1 / (1 + #{c ranked ahead of the best positive})                     ranking.py:213-222"""
    n_users = len(users)
    batch = max(1, min(n_users, _SCORE_SLAB_BYTES // (4 * n_items)))
    less = torch.zeros(max(test_pos.nnz, 1), dtype=torch.int64, device="cuda")
    pscore = torch.zeros(max(test_pos.nnz, 1), dtype=torch.float32, device="cuda")
    n_cand = np.empty(n_users, dtype=np.int64)
    before = np.empty(n_users, dtype=np.int64)
    slab = torch.empty((batch, n_items), dtype=torch.float32, device="cuda")
    for b0 in range(0, n_users, batch):
        ub = users[b0:b0 + batch]
        sc = model._scores_dev(ub, n_items=n_items, out=slab[: len(ub)])
        uidx = engine.to_device(ub, torch.int64)
        ex = excl[ub]
        ex.sort_indices()
        ep = engine.to_device(ex.indptr.astype(np.int64), torch.int64)
        ei = engine.to_device(ex.indices.astype(np.int32) if ex.nnz else np.zeros(1, np.int32), torch.int32)
        _, _, nc, bf = engine.rank_counts(sc, pos_ptr, pos_idx, user_idx=uidx, excl_indptr=ep, excl_indices=ei, less=less,
                                          pos_score=pscore)
        n_cand[b0:b0 + len(ub)] = nc.cpu().numpy()
        before[b0:b0 + len(ub)] = bf.cpu().numpy()
    less_h, ps_h = less.cpu().numpy(), pscore.cpu().numpy()
    # gather the positives of the evaluated users (in `users` order) into flat segment arrays
    lo, hi = test_pos.indptr[users], test_pos.indptr[users + 1]
    cnt = (hi - lo).astype(np.int64)
    seg = np.repeat(np.arange(n_users), cnt)
    flat = np.concatenate([np.arange(a, b) for a, b in zip(lo, hi)]) if n_users else np.zeros(0, np.int64)
    l_p, s_p = less_h[flat].astype(np.int64), ps_h[flat]
    less_pp = _rank_within_segments(seg, s_p)                  # positives of the same user scoring strictly below
    P = cnt.astype(np.float64)
    starts = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
    for m, row in zip(metrics, rows_out):
        if type(m) is AUC:
            num = np.add.reduceat((l_p - less_pp).astype(np.float64), starts)
            with np.errstate(divide="ignore", invalid="ignore"):
                per_metric[row] = num / (P * (n_cand - cnt).astype(np.float64))
        elif type(m) is MAP:
            L_p = (cnt[seg] - less_pp).astype(_MAP_DTYPE)       # rankdata(-scores[relevant], "max")
            r_p = (n_cand[seg] - l_p).astype(_MAP_DTYPE)        # rankdata(-scores, "max")[relevant]
            if n_users <= _MAP_EXACT_USERS:                     # the reference's own expression, user by user
                ends = starts + cnt
                per_metric[row] = [(L_p[a:b] / r_p[a:b]).mean() for a, b in zip(starts, ends)]
            else:
                per_metric[row] = np.add.reduceat((L_p / r_p).astype(np.float64), starts) / P
        else:                                                   # MRR
            per_metric[row] = 1.0 / (1.0 + before.astype(np.float64))
