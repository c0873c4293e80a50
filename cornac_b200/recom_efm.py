"""Explicit Factor Models on an H100: drop-in for cornac.models.EFM.

Same constructor arguments, defaults, attributes and fit()/score() behaviour as the reference class
(cornac/models/efm/recom_efm.pyx:46-528).  The initial factors are drawn on the host as the reference's `_init` draws
them; the three matrices of `_build_matrices` -- ratings A, user aspect attentions X, item aspect qualities Y -- are
built here in vectorised numpy, equal element for element to the reference's; the compiled loop of `_fit_efm` runs as
b200_efm_fit in the reference's f32 arithmetic and summation order.

Arithmetic contract.  The reference's predictions are BLAS sdot calls, whose summation order is unspecified.  Here a
dot is the f64 sum in index order of the exact f32 products, rounded once to f32 (the project's defined dot), so the fit
is bit-identical to a serial C restatement of the reference loop with that dot, and equals the reference exactly wherever every
prediction is exact (a dyadic start); elsewhere it agrees with the reference to f32 rounding.

rank(u) is the reference's aspect-weighted row  alpha * explicit + (1 - alpha) * score  with
explicit[i] = sum_t X_[a_t] (U2[i] . V[a_t]) / (N * rating_scale) over the user's N most cared aspects a_t.  That row is
one dot product: with W = [U2 | H2], row[i] = W[i] . q_u where
    q_u = [ alpha / (N * rating_scale) * sum_t X_[a_t] V[a_t] + (1 - alpha) U1[u],  (1 - alpha) H1[u] ].
b200_efm_queries computes q_u per user (X_ with the defined dot, the top aspects in the order (X_ desc, id asc), the
weighted sum in f64, q_u rounded once to f32), and the rows, rank_batch, recommend_batch, the transform() cache and the
batched ranking_eval take the shared f32 scoring path (DeviceScoringMixin) with U := Q and V := W.  This replaces the
reference's staged f32 BLAS arithmetic by the f32 rounding of an f64 dot: scores differ from the reference's by f32
rounding, and an aspect within one rounding of the N-th place can be chosen differently.  score(u) is the plain row
W . [U1[u], H1[u]] on the device; score(u, i) is the reference's host expression.
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
from ._scoring import DeviceScoringMixin
from .recom_bpr import _copy_back

DTYPE = np.float32


def build_matrices(train_set, num_users, num_items, num_aspects, rating_scale, use_item_aspect_popularity):
    """(A, X, Y) of EFM._build_matrices (recom_efm.pyx:361-432) as scipy CSR matrices, element for element.

    A: the f32 ratings (repeated pairs summed, as scipy builds it).  X[u, a] = f32(1 + (s - 1)(2 / (1 + e^-count) - 1))
    with count the number of the user's sentiment tuples on aspect a.  Y[i, a] = f32(1 + (s - 1) / (1 + e^-total)),
    total the f64 sum of the polarities of the item's tuples on aspect a in the reference's order (the item's reviews in
    insertion order, each review's tuples in order); without aspect popularity total / count replaces total."""
    uid, iid, rat = train_set.uir_tuple
    keep = (np.asarray(uid) < num_users) & (np.asarray(iid) < num_items)
    A = sp.csr_matrix((np.asarray(rat, dtype=np.float32)[keep], (np.asarray(uid, dtype=np.int32)[keep],
                                                                  np.asarray(iid, dtype=np.int32)[keep])),
                      shape=(num_users, num_items))
    sentiment = train_set.sentiment
    # every sentiment tuple of every review the modality kept, item by item in the reference's order
    t_user, t_item, t_aspect, t_pol = [], [], [], []
    for i, by_user in sentiment.item_sentiment.items():
        if i >= num_items:
            continue
        for u, idx in by_user.items():
            tups = sentiment.sentiment[idx]
            if not tups:
                continue
            t_user.append(np.full(len(tups), u, dtype=np.int64))
            t_item.append(np.full(len(tups), i, dtype=np.int64))
            t_aspect.append(np.fromiter((t[0] for t in tups), dtype=np.int64, count=len(tups)))
            t_pol.append(np.fromiter((t[2] for t in tups), dtype=np.float64, count=len(tups)))
    cat = lambda parts, dt: np.concatenate(parts) if parts else np.zeros(0, dt)     # noqa: E731
    t_user, t_item, t_aspect, t_pol = (cat(t_user, np.int64), cat(t_item, np.int64), cat(t_aspect, np.int64),
                                       cat(t_pol, np.float64))
    s = rating_scale
    ku = t_user < num_users
    ua, count = np.unique(t_user[ku] * num_aspects + t_aspect[ku], return_counts=True)
    att = (1 + (s - 1) * (2 / (1 + np.exp(-count.astype(np.float64))) - 1)).astype(np.float32)
    X = sp.csr_matrix((att, (ua // num_aspects, ua % num_aspects)), shape=(num_users, num_aspects))
    ia, inv, icount = np.unique(t_item * num_aspects + t_aspect, return_inverse=True, return_counts=True)
    total = np.zeros(len(ia), dtype=np.float64)
    np.add.at(total, inv, t_pol)                                         # in tuple order, as the reference's loop
    if not use_item_aspect_popularity:
        total = total / icount
    qual = (1 + (s - 1) / (1 + np.exp(-total))).astype(np.float32)
    Y = sp.csr_matrix((qual, (ia // num_aspects, ia % num_aspects)), shape=(num_items, num_aspects))
    return A, X, Y


class EFM(DeviceScoringMixin, Recommender):
    """Explicit Factor Models (Zhang et al., SIGIR 2014), trained on the GPU.

    Parameters are the reference's: name="EFM", num_explicit_factors=40, num_latent_factors=60,
    num_most_cared_aspects=15, rating_scale=5.0, alpha=0.85, lambda_x=1, lambda_y=1, lambda_u=0.01, lambda_h=0.01,
    lambda_v=0.01, use_item_aspect_popularity=True, max_iter=100, num_threads=0 (kept for compatibility: the fit runs on
    the GPU), trainable=True, verbose=False, init_params=None ({'U1', 'U2', 'V', 'H1', 'H2'}; f32 arrays are trained in
    place), seed=None (initial factors only; the fit itself is deterministic).

    The train set needs a SentimentModality (`sentiment=` of the eval method).  With verbose=True each iteration's loss
    is printed; it is summed in f64 on the device, so its last digits may differ from the reference's f32 figure; the
    trained parameters do not.
    """

    def __init__(self, name="EFM", num_explicit_factors=40, num_latent_factors=60, num_most_cared_aspects=15,
                 rating_scale=5.0, alpha=0.85, lambda_x=1, lambda_y=1, lambda_u=0.01, lambda_h=0.01, lambda_v=0.01,
                 use_item_aspect_popularity=True, max_iter=100, num_threads=0, trainable=True, verbose=False,
                 init_params=None, seed=None):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.num_explicit_factors = num_explicit_factors
        self.num_latent_factors = num_latent_factors
        self.num_most_cared_aspects = num_most_cared_aspects
        self.rating_scale = rating_scale
        self.alpha = alpha
        self.lambda_x = lambda_x
        self.lambda_y = lambda_y
        self.lambda_u = lambda_u
        self.lambda_h = lambda_h
        self.lambda_v = lambda_v
        self.use_item_aspect_popularity = use_item_aspect_popularity
        self.max_iter = max_iter
        self.seed = seed

        if seed is not None:                                    # recom_efm.pyx:151-156
            self.num_threads = 1
        elif num_threads > 0 and num_threads < multiprocessing.cpu_count():
            self.num_threads = num_threads
        else:
            self.num_threads = multiprocessing.cpu_count()

        self.init_params = {} if init_params is None else init_params
        self.U1 = self.init_params.get("U1", None)
        self.U2 = self.init_params.get("U2", None)
        self.V = self.init_params.get("V", None)
        self.H1 = self.init_params.get("H1", None)
        self.H2 = self.init_params.get("H2", None)
        self._b200_register_ignored()

    # reference: recom_efm.pyx:166-185
    def _init(self, train_set):
        rng = get_rng(self.seed)
        self.num_aspects = train_set.sentiment.num_aspects
        n_aspects = self.num_aspects
        n_users, n_items = self.num_users, self.num_items
        n_efactors = self.num_explicit_factors
        n_lfactors = self.num_latent_factors
        high = np.sqrt(self.rating_scale / (n_efactors + n_lfactors))
        if self.U1 is None:
            self.U1 = uniform((n_users, n_efactors), high=high, random_state=rng)
        if self.U2 is None:
            self.U2 = uniform((n_items, n_efactors), high=high, random_state=rng)
        if self.V is None:
            self.V = uniform((n_aspects, n_efactors), high=high, random_state=rng)
        if self.H1 is None:
            self.H1 = uniform((n_users, n_lfactors), high=high, random_state=rng)
        if self.H2 is None:
            self.H2 = uniform((n_items, n_lfactors), high=high, random_state=rng)

    # reference: recom_efm.pyx:187-226
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        if getattr(train_set, "sentiment", None) is None:
            raise ValueError("EFM needs the sentiment modality: build the train set with a SentimentModality "
                             "(e.g. RatioSplit(..., sentiment=SentimentModality(data=...)))")
        self._init(train_set)
        self._b200_invalidate()
        if self.trainable:
            A, X, Y = build_matrices(train_set, self.num_users, self.num_items, self.num_aspects, self.rating_scale,
                                     self.use_item_aspect_popularity)
            if self.verbose:
                print("Building matrices completed!")
            self._fit_b200(A, X, Y)
        return self

    def _factor_shapes(self):
        E, L = self.num_explicit_factors, self.num_latent_factors
        return (("U1", (self.num_users, E)), ("U2", (self.num_items, E)), ("V", (self.num_aspects, E)),
                ("H1", (self.num_users, L)), ("H2", (self.num_items, L)))

    def _check_params(self):
        """The reference's `floating[:, :]` buffers take only f32 here (the ratings fix the type)."""
        for name, shape in self._factor_shapes():
            x = np.asarray(getattr(self, name))
            if x.dtype != DTYPE:
                got = "double" if x.dtype == np.float64 else str(x.dtype)
                raise ValueError("Buffer dtype mismatch, expected 'float' but got '%s'" % got)
            if x.ndim != 2 or x.shape[0] < shape[0] or x.shape[1] != shape[1]:
                raise ValueError("%s must have shape %s, got %s" % (name, shape, x.shape))

    def _fit_b200(self, A, X, Y):
        self._check_params()
        engine.require_cuda()
        data = engine.EfmData(A, X, Y)
        # rows beyond the model's users / items (a larger init_params array) are not touched, as in the reference
        dev = [engine.to_device(np.ascontiguousarray(np.asarray(getattr(self, name))[: shape[0]]), torch.float32)
               for name, shape in self._factor_shapes()]
        hyper = dict(lambda_x=self.lambda_x, lambda_y=self.lambda_y, lambda_u=self.lambda_u, lambda_h=self.lambda_h,
                     lambda_v=self.lambda_v)
        if self.verbose:
            work = torch.empty(max(engine.efm_workspace_floats(data.n_users, data.n_items, data.n_aspects,
                                                               self.num_explicit_factors, self.num_latent_factors), 1),
                               dtype=torch.float32, device="cuda")
            loss = torch.zeros(1, dtype=torch.float64, device="cuda")
            for t in range(1, self.max_iter + 1):
                loss.zero_()
                engine.efm_fit(data, *dev, 1, loss=loss, workspace=work, **hyper)
                print("iter: %d, loss: %f" % (t, loss.item()))
            print("Optimization finished!")
        else:
            engine.efm_fit(data, *dev, self.max_iter, **hyper)
        for (name, _), d in zip(self._factor_shapes(), dev):
            setattr(self, name, self._copy_rows_back(getattr(self, name), d))

    @staticmethod
    def _copy_rows_back(host, dev):
        """The trained rows into the caller's array (an init_params array is trained in place)."""
        n = int(dev.shape[0])
        if isinstance(host, np.ndarray) and host.shape[0] > n and host.dtype == DTYPE and host.flags.writeable:
            host[:n] = dev.cpu().numpy()
            return host
        return _copy_back(host, dev)

    # ---- device scoring: U := Q (the rank queries of every U1 row), V := W = [U2 | H2] -------------------------------
    def _b200_device(self):
        dev = getattr(self, "_b200_dev", None)
        if dev is None:
            engine.require_cuda()
            f32 = lambda x: engine.to_device(np.ascontiguousarray(x, dtype=DTYPE), torch.float32)    # noqa: E731
            U1, H1, V = f32(self.U1), f32(self.H1), f32(self.V)
            n_items = self.num_items
            W = f32(np.concatenate([np.asarray(self.U2)[:n_items], np.asarray(self.H2)[:n_items]], axis=1))
            Q = engine.efm_queries(U1, H1, V, self.num_most_cared_aspects, self.alpha, self.rating_scale)
            dev = dict(U=Q, V=W, item_base=None, user_off=None, n_items=n_items, UH=torch.cat([U1, H1], dim=1))
            self._b200_dev = dev
        return dev

    def _b200_rank_row(self, user_idx):
        # the reference's rank() indexes U1 directly: any U1 row ranks, a row beyond it raises IndexError
        return self._scores_dev([user_idx])[0]

    # reference: recom_efm.pyx:440-469
    def score(self, user_idx, item_idx=None):
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            d = self._b200_device()
            uidx = torch.as_tensor(self._b200_check_users([user_idx], d["UH"].shape[0])).cuda()
            return engine.score_batch(d["UH"], d["V"], user_idx=uidx)[0].cpu().numpy()
        return self.U2[item_idx, :].dot(self.U1[user_idx, :]) + self.H2[item_idx, :].dot(self.H1[user_idx, :])
