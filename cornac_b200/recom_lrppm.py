"""Learning to Rank user Preferences on Phrase-level sentiment across Multiple categories on an H100: drop-in for
cornac.models.LRPPM.

Same constructor arguments, defaults, attributes and fit()/score()/rank() behaviour as the reference class
(cornac/models/lrppm/recom_lrppm.pyx:56-560).  The parameters are drawn on the host as the reference's `_init` draws
them; the data of `_build_data` and of the flattening in `fit` -- the review triples (user, item, aspect) and their
weights, the item x aspect quality matrix, and the two hash dicts the loop looks up -- are built here in vectorised
numpy, in the reference's order (the seeded samplers pick entries by position).  The dict keys are the reference's
Cantor keys in C int, with its two's-complement wrap: a wrapped key that collides with another skips a ranking sample
the triples alone would not skip, and the fit reproduces that.

The three sample streams are the reference's RNGVector streams, drawn on the host in bulk; the compiled loop of `_fit`
runs as b200_lrppm_fit, bit-identical to the reference's compiled float loop given those draws, and stops after the
first iteration that leaves every parameter isclose to its value before it, as the reference does.  Without a seed the
reference runs its loop on several threads that race on shared arrays and repeat the dense step per thread; here the
samples are drawn on the device (Philox4x32-10, the same uniform law) and the same ordered kernel applies one step per
iteration.

rank() (and rank_batch, recommend_batch, the transform() cache and the batched ranking_eval) orders the aspect-mixed
rows of the reference when alpha > 0 and num_top_aspects > 0 (b200_lrppm_rank_rows, f64): the quality-weighted mean of
each item's top aspect scores, mixed with the rating score.  At a tie at the N-th aspect the smaller aspect ids are
taken; the reference's argsort there is not stable, so it may take others.  Otherwise the rows are score(u) = I . U[u].
score(u, i) and score(u) are the reference's host dots, so rating metrics are the reference's.
"""
import multiprocessing

import numpy as np
import scipy.sparse as sp
import torch

from cornac.exception import ScoreException
from cornac.models.recommender import Recommender
from cornac.utils import get_rng
from cornac.utils.init_utils import uniform

from . import engine
from ._scoring import DeviceScoringMixin, ScoringMixin
from .engine import LrppmData
from .recom_bpr import _copy_back
from .recom_mter import stream_seeds

DTYPE = np.float32
PARAMS = ("U", "I", "UA", "IA")


def get_key(i, j):
    """recom_mter.get_key in C int: (i + j) (i + j + 1) // 2 + j with two's-complement wrap (int64 arrays in, int64
    holding int32 values out)."""
    i, j = np.asarray(i, dtype=np.int64), np.asarray(j, dtype=np.int64)
    s = (i + j) & 0xFFFFFFFF
    p = (s * ((s + 1) & 0xFFFFFFFF)) & 0xFFFFFFFF
    p = np.where(p >= 2 ** 31, p - 2 ** 32, p)                     # the int32 product, then an exact floor halving
    k = ((p >> 1) + j) & 0xFFFFFFFF
    return np.where(k >= 2 ** 31, k - 2 ** 32, k)


def get_key3(i, j, k):
    return get_key(get_key(i, j), k)


def build_data(train_set, num_users, num_items):
    """LrppmData of a train set with a SentimentModality, equal array for array to the reference's `_build_data` and
    the flattening in `fit` (recom_lrppm.pyx:207-303).

    The triples (u, i, a) of known users, in order of first appearance, hold the sum of their polarities; X_l_ui is
    f32(1 / (cnt (n_aspects - cnt))) with cnt the number of distinct aspects of (u, i) (None where cnt == n_aspects:
    the reference divides by zero there).  The quality of (i, a) sums, per review, the polarity of the review's last
    tuple under that tuple's aspect -- the reference's statement sits after the tuple loop."""
    sentiment = train_set.sentiment
    n_aspects = int(sentiment.num_aspects)
    ev_u, ev_i, ev_a, ev_p, q_i, q_a, q_p = [], [], [], [], [], [], []
    aid = pol = None
    for u, by_item in sentiment.user_sentiment.items():
        if u is None or not (0 <= u < num_users):                   # the reference's knows_user
            continue
        for i, tup_idx in by_item.items():
            tups = sentiment.sentiment[tup_idx]
            for aid, _, pol in tups:
                ev_u.append(u)
                ev_i.append(i)
                ev_a.append(aid)
                ev_p.append(pol)
            if aid is None:
                raise NameError("free variable 'aid' referenced before assignment")
            q_i.append(i)
            q_a.append(aid)
            q_p.append(pol)
    ev_u, ev_i, ev_a = (np.asarray(x, dtype=np.int64) for x in (ev_u, ev_i, ev_a))
    ev_p = np.asarray(ev_p, dtype=np.float64)

    def first_order(keys):
        """(distinct keys in order of first appearance, index of each event's key in that order)."""
        uniq, first, inv = np.unique(keys, return_index=True, return_inverse=True)
        order = np.argsort(first, kind="stable")
        rank = np.empty(len(uniq), dtype=np.int64)
        rank[order] = np.arange(len(uniq))
        return first[order], rank[inv.ravel()]

    first, pos = first_order((ev_u * num_items + ev_i) * max(n_aspects, 1) + ev_a)
    total = np.zeros(len(first), dtype=np.float64)
    np.add.at(total, pos, ev_p)                                      # in tuple order, as the reference's loop
    X_uids, X_iids, X_aids = ev_u[first], ev_i[first], ev_a[first]
    pair = X_uids * num_items + X_iids
    _, pinv, pcnt = np.unique(pair, return_inverse=True, return_counts=True)
    cnt = pcnt[pinv.ravel()]
    neg = n_aspects - cnt
    X_l_ui = None if np.any(neg == 0) else (1.0 / (cnt * neg)).astype(np.float32)
    # the item x aspect quality
    q_i, q_a = np.asarray(q_i, dtype=np.int64), np.asarray(q_a, dtype=np.int64)
    qf, qpos = first_order(q_i * max(n_aspects, 1) + q_a)
    qtot = np.zeros(len(qf), dtype=np.float64)
    np.add.at(qtot, qpos, np.asarray(q_p, dtype=np.float64))
    quality = sp.csr_matrix((1.0 / (1.0 + np.exp(-qtot)), (q_i[qf], q_a[qf])), shape=(num_items, n_aspects))
    # the two dicts: sorted distinct keys; the rating dict keeps the last value of a key
    u_idx, i_idx, r_val = train_set.uir_tuple
    rkeys = get_key(u_idx, i_idx)
    rrev = rkeys[::-1]
    rk, rlast = np.unique(rrev, return_index=True)
    rvals = np.asarray(r_val, dtype=np.float64)[::-1][rlast].astype(np.float32)
    return LrppmData(n_users=int(num_users), n_items=int(num_items), n_aspects=n_aspects,
                     u_indices=np.asarray(u_idx).astype(np.int32), i_indices=np.asarray(i_idx).astype(np.int32),
                     r_values=np.asarray(r_val).astype(np.float32),
                     X_uids=X_uids.astype(np.int32), X_iids=X_iids.astype(np.int32), X_aids=X_aids.astype(np.int32),
                     X_values=total, X_l_ui=X_l_ui, aspect_keys=np.unique(get_key3(X_uids, X_iids, X_aids)).astype(np.int32),
                     rating_keys=rk.astype(np.int32), rating_values=rvals, item_aspect_quality=quality)


def check_data(data):
    """The reference divides by zero where a review pair mentions every aspect, and draws from
    uniform_int_distribution(0, len - 1) over the triples and the ratings: both are errors here, before any device
    work."""
    if data.X_l_ui is None:
        raise ZeroDivisionError("float division by zero")
    for name, n in (("user-item-aspect triples (no sentiment reviews)", len(data.X_uids)),
                    ("rating matrix (no ratings)", len(data.r_values))):
        if n == 0:
            raise ValueError("LRPPM cannot sample from an empty %s" % name)


class LRPPM(DeviceScoringMixin, Recommender):
    """LRPPM (Chen et al., SIGIR 2016), trained on the GPU.

    Parameters are the reference's: name="LRPPM", rating_scale=5, n_factors=8, ld=1, reg=0.01, alpha=1,
    num_top_aspects=99999, n_ranking_samples=1000, n_samples=200, max_iter=200000, lr=0.1, n_threads=0 (kept for
    compatibility: the fit runs on the GPU), trainable=True, verbose=False, init_params=None ({'U', 'I', 'UA', 'IA'};
    f32 arrays are trained in place), seed=None.

    The train set needs a SentimentModality.  With verbose=True each iteration reports the reference's five figures;
    the losses are summed in f64 on the device, so their last digits may differ from the reference's f32 sums.
    """

    def __init__(self, name="LRPPM", rating_scale=5, n_factors=8, ld=1, reg=0.01, alpha=1, num_top_aspects=99999,
                 n_ranking_samples=1000, n_samples=200, max_iter=200000, lr=0.1, n_threads=0, trainable=True,
                 verbose=False, init_params=None, seed=None):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.n_factors = n_factors
        self.rating_scale = rating_scale
        self.ld = ld
        self.reg = reg
        self.alpha = alpha
        self.num_top_aspects = num_top_aspects
        self.n_samples = n_samples
        self.n_ranking_samples = n_ranking_samples
        self.max_iter = max_iter
        self.lr = lr
        self.seed = seed
        if seed is not None:                                   # recom_lrppm.pyx:171-176
            self.n_threads = 1
        elif n_threads > 0 and n_threads < multiprocessing.cpu_count():
            self.n_threads = n_threads
        else:
            self.n_threads = multiprocessing.cpu_count()
        self.rng = get_rng(seed)
        self.init_params = {} if init_params is None else init_params
        for p in PARAMS:
            setattr(self, p, self.init_params.get(p, None))
        self._b200_register_ignored()

    # reference: recom_lrppm.pyx:186-202 (IA is drawn with UA's shape)
    def _init(self, train_set):
        n_users, n_items = train_set.num_users, train_set.num_items
        self.num_aspects = train_set.sentiment.num_aspects
        for name, shape in (("U", (n_users, self.n_factors)), ("I", (n_items, self.n_factors)),
                            ("UA", (self.num_aspects, self.n_factors)), ("IA", (self.num_aspects, self.n_factors))):
            if getattr(self, name) is None:
                setattr(self, name, uniform(shape, random_state=self.rng))

    # reference: recom_lrppm.pyx:259-351
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        if getattr(train_set, "sentiment", None) is None:
            raise ValueError("LRPPM needs the sentiment modality: build the train set with a SentimentModality "
                             "(e.g. RatioSplit(..., sentiment=SentimentModality(data=...)))")
        self._init(train_set)
        self._b200_invalidate()
        data = build_data(train_set, self.num_users, self.num_items)
        self.item_aspect_quality = data.item_aspect_quality
        if not self.trainable:
            return self
        check_data(data)
        seeds = stream_seeds(self.rng, 3)                     # pos, pos_uia, neg_uia (recom_lrppm.pyx:307-309)
        self._fit_b200(data, seeds)
        return self

    def _check_params(self):
        """The reference's `floating` buffers take only f32 here (its r_values and X_l_ui are float32)."""
        k = self.n_factors
        for name, shape in (("U", (self.num_users, k)), ("I", (self.num_items, k)), ("UA", (self.num_aspects, k)),
                            ("IA", (self.num_aspects, k))):
            x = np.asarray(getattr(self, name))
            if x.dtype != DTYPE:
                got = "double" if x.dtype == np.float64 else str(x.dtype)
                raise ValueError("Buffer dtype mismatch, expected 'float' but got '%s'" % got)
            if x.shape != shape:
                raise ValueError("%s must have shape %s, got %s" % (name, shape, x.shape))

    def _fit_b200(self, data, seeds):
        self._check_params()
        engine.require_cuda()
        n_s, n_rk = int(self.n_samples), int(self.n_ranking_samples)
        if n_s < 0 or n_rk < 0:
            raise ValueError("n_samples and n_ranking_samples must not be negative")
        params = [engine.to_device(np.ascontiguousarray(getattr(self, n)), torch.float32) for n in PARAMS]
        ddata = engine.LrppmDeviceData(data)
        work = torch.zeros(engine.lrppm_workspace_bytes(ddata, self.n_factors, n_s, n_rk), dtype=torch.uint8,
                           device="cuda")
        counts = torch.zeros(4, dtype=torch.int64, device="cuda")
        losses = torch.zeros(3, dtype=torch.float64, device="cuda") if self.verbose else None
        seeded = self.seed is not None
        draws = engine.lrppm_draws(seeds, data, n_s, n_rk, 1 if self.verbose else self.max_iter) if seeded else None
        chunk = 1 if self.verbose else (draws.chunk if seeded else max(int(self.max_iter), 1))
        done, converged = 0, False
        while done < self.max_iter and not converged:
            n = min(chunk, self.max_iter - done)
            counts.zero_()
            engine.lrppm_fit(ddata, params, draws.next(n) if seeded else None, n, n_s, n_rk, lr=self.lr, reg=self.reg,
                             ld=self.ld, counts=counts, losses=losses, workspace=work,
                             philox_seed=None if seeded else seeds[0], iter0=done)
            correct, skipped, ran, conv = counts.tolist()
            done += ran
            converged = bool(conv)
            if self.verbose:
                loss, ranking_loss, r_loss = losses.tolist()
                live = n_rk - skipped
                print("iter %d: loss %.2f, ranking_loss %.2f, r_loss %.2f, correct %.2f%%, skipped %.2f%%"
                      % (done, loss / max(n_s, 1), ranking_loss / max(live, 1), r_loss / max(live, 1),
                         100.0 * correct / (live + 1e-8), 100.0 * skipped / max(n_rk, 1)))
                losses.zero_()
        self.n_iter_run = done
        if converged:
            print("Stop training because model converged!")
        if self.verbose:
            print("Optimization finished!")
        for name, d in zip(PARAMS, params):
            setattr(self, name, _copy_back(getattr(self, name), d))

    # ---- device scoring ---------------------------------------------------------------------------------------------
    def _b200_host_params(self):
        return (np.ascontiguousarray(self.U, dtype=DTYPE), np.ascontiguousarray(np.asarray(self.I)[: self.num_items],
                                                                                 dtype=DTYPE),
                None, None, self.num_items)

    def _b200_mixed(self):
        return self.alpha > 0 and self.num_top_aspects > 0

    @property
    def _B200_SCORE_DTYPE(self):
        return np.float64 if self._b200_mixed() else np.float32

    def _b200_aspect_device(self):
        dev = self._b200_device()
        if "aspect" not in dev:
            f32 = lambda x: engine.to_device(np.ascontiguousarray(x, dtype=DTYPE), torch.float32)    # noqa: E731
            dev["aspect"] = dict(UA=f32(self.UA), IA=f32(self.IA),
                                 Q=engine.LrppmQuality(self.item_aspect_quality))
        return dev["aspect"]

    def _aspect_rows(self, user_indices, n_items=None):
        """[n_q, n_items] f64 device rank rows of the given users (b200_lrppm_rank_rows)."""
        dev, d = self._b200_device(), self._b200_aspect_device()
        user_indices = self._b200_check_users(user_indices, self.num_users)
        n_top = min(int(self.num_top_aspects), int(self.num_aspects))
        return engine.lrppm_rank_rows(dev["U"], dev["V"], d["UA"], d["IA"], d["Q"],
                                      engine.to_device(user_indices, torch.int64), n_top, float(self.alpha),
                                      float(self.rating_scale), n_items=n_items)

    def _scores_dev(self, user_indices, n_items=None, out=None):
        """The rows every rank path orders: the aspect-mixed f64 rows, or score(u) when the reference falls back to
        it.  An f32 `out` (the batched ranking_eval's slab) receives the f64 rows rounded once."""
        if not self._b200_mixed():
            return super()._scores_dev(user_indices, n_items=n_items, out=out)
        rows = self._aspect_rows(user_indices, n_items=n_items)
        if out is None:
            return rows
        out.copy_(rows)
        return out

    def _b200_scores_nan_free(self):
        if not self._b200_mixed():
            return super()._b200_scores_nan_free()
        return all(bool(np.isfinite(np.asarray(getattr(self, p))).all()) for p in PARAMS)

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

    # reference: recom_lrppm.pyx:484-517
    def score(self, u_idx, i_idx=None):
        if i_idx is None:
            if not self.knows_user(u_idx):
                raise ScoreException("Can't make score prediction for (user_id=%d)" % u_idx)
            return self.I.dot(self.U[u_idx])
        if not (self.knows_user(u_idx) and self.knows_item(i_idx)):
            raise ScoreException("Can't make score prediction for (user_id=%d, item_id=%d)" % (u_idx, i_idx))
        return self.I[i_idx].dot(self.U[u_idx])
