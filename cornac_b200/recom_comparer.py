"""ComparERSub on an H100: drop-in for cornac.models.ComparERSub (MTER with comparative aspect constraints).

Same constructor arguments, defaults, attributes and fit()/score()/rank() behaviour as the reference class
(cornac/models/comparer/recom_comparer_sub.pyx:47-806), which subclasses MTER; this class subclasses cornac_b200.MTER
and reuses its parameter draws, data, checks and verbose report.  On top of MTER's data, the fit needs the
chronological order of each user's items (the train set's timestamps) to build the list of comparative pairs (user,
earlier item, later item, aspect); `build_pairs` builds it in vectorised numpy, element for element and in the
reference's order.  The fit is b200_comparer_sub_fit: MTER's device fit with a third sample phase over the pairs,
bit-identical to the reference's serial float loop given the six seeded streams (uia, uao, iao, pair, pos, neg).

rank() is not a dot product: for user u every item scores alpha * mean(top n_top_aspects of ts3[i, :n_aspects]) +
(1 - alpha) * ts3[i, n_aspects], ts3[i, a] = sum G1[p, q, r] U[u, p] I[i, q] A[a, r] (b200_comparer_rank_rows, f64
throughout, one f32 rounding).  rank, rank_batch, rank_batch_device, recommend_batch, the transform() cache and the
batched ranking_eval take those rows.  score(u) and score(u, i) stay MTER's rating row and host einsum, as in the
reference, which inherits MTER.score.  With alpha <= 0 or n_top_aspects <= 0 the reference ranks by score(), and so
does this class: it then ranks exactly as cornac_b200.MTER.
"""
import numpy as np
import scipy.sparse as sp
import torch

from . import engine
from ._scoring import ScoringMixin
from .engine import MterData
from .recom_mter import MTER, build_data as mter_build_data, check_data, stream_seeds

_PAIR_CHUNK = 1 << 21        # position pairs of one user handled at once (bounds the host memory of build_pairs)


def _quality(total, rating_scale):
    return 1 + (rating_scale - 1) / (1 + np.exp(-total))


def item_quality(sentiment, num_items, rating_scale, use_item_aspect_popularity):
    """The item aspect quality matrix Y, an f32 CSR [num_items, num_aspects], as the reference's
    _build_item_quality_matrix (recom_comparer_sub.pyx:178-211): per item, the f64 sum of an aspect's polarities over
    its reviews in the modality's order (or that sum over the aspect's tuple count), through the quality score, then
    f32."""
    n_aspects = int(sentiment.num_aspects)
    ev_i, ev_a, ev_p = [], [], []
    for i, by_user in sentiment.item_sentiment.items():
        if i is None or not (0 <= i < num_items):                 # the reference's knows_item
            continue
        for tup_idx in by_user.values():
            tups = sentiment.sentiment[tup_idx]
            ev_i.append(np.full(len(tups), i, dtype=np.int64))
            ev_a.append(np.fromiter((t[0] for t in tups), dtype=np.int64, count=len(tups)))
            ev_p.append(np.fromiter((t[2] for t in tups), dtype=np.float64, count=len(tups)))
    if not ev_i:
        return sp.csr_matrix((num_items, n_aspects), dtype=np.float32)
    ev_i, ev_a, ev_p = np.concatenate(ev_i), np.concatenate(ev_a), np.concatenate(ev_p)
    keys, pos = np.unique(ev_i * n_aspects + ev_a, return_inverse=True)
    pos = pos.ravel()
    total = np.zeros(len(keys), dtype=np.float64)
    np.add.at(total, pos, ev_p)                                   # in event order: the reference's running sums
    if not use_item_aspect_popularity:
        total = total / np.bincount(pos, minlength=len(keys))
    return sp.csr_matrix((_quality(total, rating_scale).astype(np.float32), (keys // n_aspects, keys % n_aspects)),
                         shape=(num_items, n_aspects))


def _position_pairs(n, window):
    """The (earlier, later) positions of the reference's windowed enumeration of a history of n items, each position
    pair once, in the order of its first appearance, with the number of windows it appears in."""
    gaps = np.arange(1, window, dtype=np.int64)                  # later - earlier, below the window
    a = np.concatenate([np.arange(n - d, dtype=np.int64) for d in gaps]) if len(gaps) else np.zeros(0, np.int64)
    b = a + np.repeat(gaps, n - gaps)
    first = np.maximum(0, b - window + 1)                         # the first window holding both positions
    count = np.minimum(a, n - window) - first + 1
    order = np.lexsort((b, a, first))                             # windows in turn, combinations() order inside one
    return a[order], b[order], count[order]


def build_pairs(train_set, data, num_items, Y, min_user_freq=2, min_common_freq=1, enum_window=None):
    """(p_user_indices, earlier_indices, later_indices, aspect_indices, pair_freq) as the reference's
    _build_chrono_purchased_pairs builds them (recom_comparer_sub.pyx:293-351), element for element and in order.

    For each user of train_set.chrono_user_data with at least min_user_freq items, the (earlier, later) item pairs of
    every window of enum_window consecutive items (the whole history without a window), counted per (user, earlier,
    later) triple over windows and repeated items; the triples sorted stably by count, descending, over their first
    appearance (Counter.most_common); inside a triple the aspects k < num_aspects - 1 (the reference never compares the
    last one) where the later item's f64 quality beats the earlier's (0 where the user gave the item no tuple of that
    aspect); and only item pairs with at least min_common_freq aspects k < num_aspects - 1 of positive quality Y on
    both items.  Works user by user, in chunks of position pairs.  data: the MterData of the train set (X64 and the
    X index arrays give each (user, item, aspect) quality)."""
    n_aspects = int(data.n_aspects)
    n_cmp = max(n_aspects - 1, 0)
    # quality rows: the aspect entries k < n_aspects - 1 of each reviewed (user, item), sorted by (user, item, k)
    sel = data.X_aids < n_cmp
    qkey = data.X_uids[sel].astype(np.int64) * num_items + data.X_iids[sel]
    qa, qv = data.X_aids[sel].astype(np.int64), data.X64[sel]
    order = np.lexsort((qa, qkey))
    qkey, qa, qv = qkey[order], qa[order], qv[order]
    rows, row_start = np.unique(qkey, return_index=True)
    row_ptr = np.append(row_start, len(qkey)).astype(np.int64)
    Ypos = Y[:, :n_cmp] > 0
    ybits = np.zeros((num_items, (n_cmp + 7) // 8), dtype=np.uint8)     # a bit per (item, aspect): Y > 0
    for r0 in range(0, num_items, 1 << 16):
        ybits[r0:r0 + (1 << 16)] = np.packbits(Ypos[r0:r0 + (1 << 16)].toarray(), axis=1)
    popcount = np.array([bin(x).count("1") for x in range(256)], dtype=np.int64)

    def row_of(keys):
        """The quality row of each (user, item) key, -1 where the user gave the item no compared aspect."""
        if len(rows) == 0:
            return np.full(len(keys), -1, dtype=np.int64)
        r = np.minimum(np.searchsorted(rows, keys), len(rows) - 1)
        return np.where(rows[r] == keys, r, -1)

    def entries(t_rows):
        """(triple index, aspect, quality) of every entry of the given quality rows (-1: none)."""
        ok = t_rows >= 0
        t = np.flatnonzero(ok)
        lo, hi = row_ptr[t_rows[ok]], row_ptr[t_rows[ok] + 1]
        n = hi - lo
        tt = np.repeat(t, n)
        idx = np.repeat(lo - np.cumsum(n) + n, n) + np.arange(n.sum())
        return tt, qa[idx], qv[idx]

    out_u, out_e, out_l, out_k, out_c = [], [], [], [], []
    for u, (items, *_) in train_set.chrono_user_data.items():
        n = len(items)
        if n < min_user_freq or n < 2:
            continue
        items = np.asarray(items, dtype=np.int64)
        window = n if enum_window is None else min(enum_window, n)
        pa, pb, pc = _position_pairs(n, window)
        # triples (u, earlier item, later item) in order of first appearance, with their total counts
        tk = items[pa] * num_items + items[pb]
        uk, first, inv = np.unique(tk, return_index=True, return_inverse=True)
        cnt = np.bincount(inv.ravel(), weights=pc, minlength=len(uk)).astype(np.int64)
        o = np.argsort(first, kind="stable")
        te, tl, tc = uk[o] // num_items, uk[o] % num_items, cnt[o]
        step = max(1, _PAIR_CHUNK // max(n_cmp, 1))
        for c0 in range(0, len(te), step):
            e, l, c = te[c0:c0 + step], tl[c0:c0 + step], tc[c0:c0 + step]
            common = popcount[np.bitwise_and(ybits[e], ybits[l])].sum(axis=1)
            live = common >= min_common_freq
            if not live.any():
                continue
            e, l, c = e[live], l[live], c[live]
            lt, lk, lv = entries(row_of(u * num_items + l))
            et, ek, ev = entries(row_of(u * num_items + e))
            keys = np.concatenate([lt * n_cmp + lk, et * n_cmp + ek])
            if len(keys) == 0:
                continue
            uniq, pos = np.unique(keys, return_inverse=True)
            pos = pos.ravel()
            ql = np.bincount(pos[:len(lt)], weights=lv, minlength=len(uniq))   # one entry per key: exact
            qe = np.bincount(pos[len(lt):], weights=ev, minlength=len(uniq))
            win = uniq[ql > qe]                                   # (triple, aspect) ascending
            t = win // n_cmp
            out_u.append(np.full(len(win), u, dtype=np.int64))
            out_e.append(e[t])
            out_l.append(l[t])
            out_k.append(win % n_cmp)
            out_c.append(c[t])
    cat = lambda parts: np.concatenate(parts) if parts else np.zeros(0, np.int64)     # noqa: E731
    pu, pe, pl, pk, pc = (cat(x) for x in (out_u, out_e, out_l, out_k, out_c))
    o = np.argsort(-pc, kind="stable")                            # most_common(): count descending, stable
    return tuple(x[o].astype(np.int32) for x in (pu, pe, pl, pk, pc))


def build_data(train_set, num_users, num_items, rating_scale, min_user_freq=2, min_common_freq=1, enum_window=None,
               use_item_aspect_popularity=True):
    """MTER's MterData of the train set plus the pair list (p_user_indices, earlier_indices, later_indices,
    aspect_indices, pair_freq) of the reference's _build_data (recom_comparer_sub.pyx:213-291).  Raises the
    reference's ValueError (from Dataset.chrono_user_data) when the train set has no timestamps."""
    data = mter_build_data(train_set, num_users, num_items, rating_scale)
    Y = item_quality(train_set.sentiment, num_items, rating_scale, use_item_aspect_popularity)
    pairs = build_pairs(train_set, data, num_items, Y, min_user_freq, min_common_freq, enum_window)
    kw = dict(data.__dict__)
    kw.update(zip(("p_user_indices", "earlier_indices", "later_indices", "aspect_indices", "pair_freq"), pairs))
    return MterData(**kw)


class ComparERSub(MTER):
    """Explainable Recommendation with Comparative Constraints on Subjective Aspect-Level Quality (Le and Lauw, WSDM
    2021), trained on the GPU.

    Parameters are the reference's: name="ComparERSub", rating_scale=5.0, n_user_factors=8, n_item_factors=8,
    n_aspect_factors=8, n_opinion_factors=8, n_pair_samples=1000, n_bpr_samples=1000, n_element_samples=50,
    n_top_aspects=100, alpha=0.5, min_user_freq=2, min_pair_freq=1 (reported only), min_common_freq=1,
    use_item_aspect_popularity=True, enum_window=None, lambda_reg=0.1, lambda_bpr=10, lambda_d=0.01, max_iter=200000,
    lr=0.5, n_threads=0, trainable=True, verbose=False, init_params=None, seed=None.

    The train set needs a SentimentModality and timestamps.  With verbose=True each iteration reports MTER's four
    figures, as the reference does.
    """

    def __init__(self, name="ComparERSub", rating_scale=5.0, n_user_factors=8, n_item_factors=8, n_aspect_factors=8,
                 n_opinion_factors=8, n_pair_samples=1000, n_bpr_samples=1000, n_element_samples=50, n_top_aspects=100,
                 alpha=0.5, min_user_freq=2, min_pair_freq=1, min_common_freq=1, use_item_aspect_popularity=True,
                 enum_window=None, lambda_reg=0.1, lambda_bpr=10, lambda_d=0.01, max_iter=200000, lr=0.5, n_threads=0,
                 trainable=True, verbose=False, init_params=None, seed=None):
        super().__init__(name=name, rating_scale=rating_scale, n_user_factors=n_user_factors,
                         n_item_factors=n_item_factors, n_aspect_factors=n_aspect_factors,
                         n_opinion_factors=n_opinion_factors, n_bpr_samples=n_bpr_samples,
                         n_element_samples=n_element_samples, lambda_reg=lambda_reg, lambda_bpr=lambda_bpr,
                         max_iter=max_iter, lr=lr, n_threads=n_threads, seed=seed, trainable=trainable,
                         init_params=init_params, verbose=verbose)
        self.lambda_d = lambda_d
        self.n_pair_samples = n_pair_samples
        self.n_top_aspects = n_top_aspects
        self.alpha = alpha
        self.min_user_freq = min_user_freq
        self.min_pair_freq = min_pair_freq
        self.min_common_freq = min_common_freq
        self.use_item_aspect_popularity = use_item_aspect_popularity
        self.enum_window = enum_window

    # reference: recom_comparer_sub.pyx:354-482
    def fit(self, train_set, val_set=None):
        from cornac.models.recommender import Recommender
        Recommender.fit(self, train_set, val_set)
        if getattr(train_set, "sentiment", None) is None:
            raise ValueError("ComparERSub needs the sentiment modality: build the train set with a SentimentModality "
                             "(e.g. RatioSplit(..., sentiment=SentimentModality(data=...)))")
        self._init(train_set)
        self._b200_invalidate()
        if not self.trainable:
            return self
        data = build_data(train_set, self.num_users, self.num_items, self.rating_scale, self.min_user_freq,
                          self.min_common_freq, self.enum_window, self.use_item_aspect_popularity)
        check_data(data)
        if int(self.n_pair_samples) > 0 and len(data.p_user_indices) == 0:
            raise ValueError("ComparERSub cannot sample from an empty comparative pair list (no user has a later item "
                             "of better aspect quality than an earlier one): set n_pair_samples=0 or relax "
                             "min_user_freq / min_common_freq / enum_window")
        if int(self.n_pair_samples) < 0:
            raise ValueError("n_pair_samples must not be negative")
        seeds = stream_seeds(self.rng, 6)          # uia, uao, iao, pair, pos, neg (recom_comparer_sub.pyx:426-431)
        self._fit_b200(data, seeds)
        return self

    def _b200_fit_parts(self, data, seeds, dims, n_el, n_bpr, max_chunk, seeded):
        n_pair = int(self.n_pair_samples)
        ddata = engine.ComparerDeviceData(data)
        work = torch.zeros(engine.comparer_sub_workspace_bytes(ddata, dims, n_el, n_bpr, n_pair), dtype=torch.uint8,
                           device="cuda")
        hyper = dict(lr=self.lr, lambda_reg=self.lambda_reg, lambda_bpr=self.lambda_bpr, lambda_d=self.lambda_d)

        def fit(params, sgrad, draws, n, **kw):
            engine.comparer_sub_fit(ddata, params, sgrad, draws, n, n_el, n_bpr, n_pair, workspace=work, **hyper, **kw)
        return fit, (engine.comparer_draws(seeds, data, n_el, n_bpr, n_pair, max_chunk) if seeded else None)

    # ---- rank rows: the aspect-mixed score of recom_comparer_sub.pyx:762-806 -----------------------------------------
    def _b200_mixed(self):
        return self.alpha > 0 and self.n_top_aspects > 0

    def _b200_aspect_device(self):
        dev = self._b200_device()
        if "aspect" not in dev:
            f32 = lambda x: engine.to_device(np.ascontiguousarray(x, dtype=np.float32), torch.float32)    # noqa: E731
            dev["aspect"] = dict(U=f32(self.U), I=f32(np.asarray(self.I)[: self.num_items]), A=f32(self.A),
                                 G1=f32(self.G1))
        return dev["aspect"]

    def _aspect_rows(self, user_indices, n_items=None, out=None):
        """[n_q, n_items] f32 device rank rows of the given users (b200_comparer_rank_rows)."""
        d = self._b200_aspect_device()
        user_indices = self._b200_check_users(user_indices, self.num_users)
        n_top = min(int(self.n_top_aspects), int(self.num_aspects))
        return engine.comparer_rank_rows(d["U"], d["I"], d["A"], d["G1"], engine.to_device(user_indices, torch.int64),
                                         n_top, float(self.alpha), n_items=n_items, out=out)

    def _scores_dev(self, user_indices, n_items=None, out=None):
        """The rows every rank path orders (rank, rank_batch, the transform() cache, the batched ranking_eval): the
        aspect-mixed rows, or MTER's rating rows when the reference falls back to score()."""
        if not self._b200_mixed():
            return super()._scores_dev(user_indices, n_items=n_items, out=out)
        return self._aspect_rows(user_indices, n_items=n_items, out=out)

    def _b200_scores_nan_free(self):
        """The aspect-mixed rows are f64 sums of products of finite f32 values (no overflow) rounded once, so finite
        parameters give finite rows."""
        if not self._b200_mixed():
            return super()._b200_scores_nan_free()
        return all(bool(np.isfinite(np.asarray(getattr(self, p))).all()) for p in ("U", "I", "A", "G1"))

    def rank_batch(self, user_indices, k, exclude=None):
        if not self._b200_mixed():
            return super().rank_batch(user_indices, k, exclude=exclude)
        return ScoringMixin.rank_batch(self, user_indices, k, exclude=exclude)

    def rank_batch_device(self, user_indices, k, exclude=None, _rows=None, n_items=None):
        if not self._b200_mixed():
            return super().rank_batch_device(user_indices, k, exclude=exclude, _rows=_rows, n_items=n_items)
        user_indices = self._b200_check_users(user_indices, self.num_users)
        ex_ptr, ex_idx = _rows if _rows is not None else self._b200_exclusion_rows(user_indices, exclude)
        n_rank = self.num_items if n_items is None else min(int(n_items), self.num_items)
        sc = self._aspect_rows(user_indices, n_items=n_rank)
        ep = None if ex_ptr is None else engine.to_device(ex_ptr, torch.int64)
        ei = None if ex_ptr is None else (engine.to_device(ex_idx, torch.int32) if len(ex_idx) else
                                          torch.zeros(1, dtype=torch.int32, device="cuda"))
        return self._b200_topk(sc, k, ep, ei)

    # reference: MTER.score (recom_mter.pyx:677-714), inherited by the reference class: the rating row
    def score(self, u_idx, i_idx=None):
        if i_idx is None and not self.is_unknown_user(u_idx):
            return super()._scores_dev([u_idx])[0].cpu().numpy()
        return super().score(u_idx, i_idx)
