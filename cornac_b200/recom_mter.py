"""Multi-Task Explainable Recommendation on an H100: drop-in for cornac.models.MTER.

Same constructor arguments, defaults, attributes and fit()/score() behaviour as the reference class
(cornac/models/mter/recom_mter.pyx:59-714).  The parameters are drawn on the host as the reference's `_init` draws
them; the data of `_build_data` and of the array flattening in `fit` -- the user-item-aspect tensor X, the
user-aspect-opinion tensor YU, the item-aspect-opinion tensor YI, the rating CSR and the pair ratings -- are built here
in vectorised numpy, element for element and in the reference's order (the seeded samplers pick entries by position).
The five sample streams are the reference's RNGVector streams, drawn on the host in bulk; the compiled loop of
`_fit_mter` runs as b200_mter_fit, bit-identical to the reference's serial float loop given those draws.

Without a seed the reference runs its loop on several threads that add into shared arrays without synchronisation, so
no order is defined; here the samples are drawn on the device (Philox4x32-10, the same uniform law) and each sample
adds its rows' gradients with f32 atomics (b200_mter_fit's unordered mode), so an unseeded fit can differ from run to
run by rounding.

score(u) and the rank are one dot product: score(u)[i] = sum_abc G1[a, b, c] U[u, a] I[i, b] A[-1, c] = I[i] . q_u with
q_u = U[u] . M and M[a, b] = sum_c G1[a, b, c] A[-1, c].  b200_mter_queries computes M and every q_u (f64 sums in index
order, each rounded once to f32), and score rows, rank, rank_batch, recommend_batch, the transform() cache and the
batched ranking_eval take the shared f32 scoring path (DeviceScoringMixin) with U := Q and V := I.  These differ from
the reference's numpy f32 einsum by f32 rounding (ties are broken by item id).  score(u, i) is the reference's host
einsum, so rating metrics are the reference's.
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
from .engine import MterData, MterDraws  # noqa: F401  (MterData: build_data's result)
from .recom_bpr import _copy_back

DTYPE = np.float32
PARAMS = ("U", "I", "A", "O", "G1", "G2", "G3")


def build_data(train_set, num_users, num_items, rating_scale):
    """MterData of a train set with a SentimentModality, equal element for element to the reference's _build_data plus
    the flattening of its dicts (recom_mter.pyx:225-296, 334-371).

    X holds, for every review (user, item) in `sentiment.user_sentiment` order, the key (u, i, n_aspects) with the
    rating, then the key (u, i, a) of each tuple, in order of first appearance; a tuple key's value is
    1 + (s - 1) / (1 + e^-total), total the f64 sum of its polarities in tuple order.  YU (YI) holds the keys (u, a, o)
    ((i, a, o)) of the positive tuples in order of first appearance, valued 1 + (s - 1)(2 / (1 + e^-count) - 1).
    X64 holds X's f64 values, before the f32 cast (ComparERSub compares them)."""
    sentiment = train_set.sentiment
    n_aspects, n_opinions = int(sentiment.num_aspects), int(sentiment.num_opinions)
    u_idx, i_idx, r_val = train_set.uir_tuple
    u_idx, i_idx = np.asarray(u_idx, dtype=np.int64), np.asarray(i_idx, dtype=np.int64)
    rating_matrix = sp.csr_matrix((r_val, (u_idx, i_idx)), shape=(num_users, num_items))
    # every review and its tuples, in the reference's loop order
    ev_u, ev_i, ev_a, ev_o, ev_p, ev_t = [], [], [], [], [], []
    for u, by_item in sentiment.user_sentiment.items():
        if u is None or not (0 <= u < num_users):                 # the reference's knows_user
            continue
        for i, tup_idx in by_item.items():
            tups = sentiment.sentiment[tup_idx]
            n = len(tups)
            ev_u.append(np.full(n + 1, u, dtype=np.int64))
            ev_i.append(np.full(n + 1, i, dtype=np.int64))
            ev_a.append(np.fromiter([n_aspects] + [t[0] for t in tups], dtype=np.int64, count=n + 1))
            ev_o.append(np.fromiter([-1] + [t[1] for t in tups], dtype=np.int64, count=n + 1))
            ev_p.append(np.fromiter([0.0] + [t[2] for t in tups], dtype=np.float64, count=n + 1))
            ev_t.append(np.arange(n + 1) > 0)
    cat = lambda parts, dt: np.concatenate(parts) if parts else np.zeros(0, dt)        # noqa: E731
    ev_u, ev_i, ev_a, ev_o = (cat(x, np.int64) for x in (ev_u, ev_i, ev_a, ev_o))
    ev_p, ev_t = cat(ev_p, np.float64), cat(ev_t, bool)
    s = rating_scale

    def first_order(keys):
        """(distinct keys in order of first appearance, index of each event's key in that order)."""
        uniq, first, inv = np.unique(keys, return_index=True, return_inverse=True)
        order = np.argsort(first, kind="stable")
        rank = np.empty(len(uniq), dtype=np.int64)
        rank[order] = np.arange(len(uniq))
        return first[order], rank[inv.ravel()]

    # X: user item aspect
    first, pos = first_order((ev_u * num_items + ev_i) * (n_aspects + 1) + ev_a)
    total = np.zeros(len(first), dtype=np.float64)
    np.add.at(total, pos[ev_t], ev_p[ev_t])                      # in tuple order, as the reference's loop
    xa = ev_a[first]
    X = (1 + (s - 1) / (1 + np.exp(-total))).astype(np.float64)
    rev = xa == n_aspects
    if rev.any():
        X[rev] = np.asarray(rating_matrix[ev_u[first][rev], ev_i[first][rev]], dtype=np.float64).ravel()
    X_uids, X_iids, X_aids = ev_u[first], ev_i[first], xa
    # YU / YI: positive opinions, counted
    positive = ev_t & (ev_p > 0)
    pu, pi, pa, po = ev_u[positive], ev_i[positive], ev_a[positive], ev_o[positive]

    def counted(keys):
        first, pos = first_order(keys)
        count = np.bincount(pos, minlength=len(first)).astype(np.int64)
        att = 1 + (s - 1) * (2 / (1 + np.exp(-count)) - 1)
        return first, att

    fu, YU = counted((pu * n_aspects + pa) * max(n_opinions, 1) + po)
    fi, YI = counted((pi * n_aspects + pa) * max(n_opinions, 1) + po)
    # ratings: the CSR (sorted, duplicates summed) and the last rating of each exact pair
    indptr = rating_matrix.indptr.astype(np.int32)
    indices = rating_matrix.indices.astype(np.int32)
    user_ids = np.repeat(np.arange(num_users), np.diff(rating_matrix.indptr)).astype(np.int32)
    pair = u_idx * num_items + i_idx
    rev_pair = pair[::-1]
    upair, last_rev = np.unique(rev_pair, return_index=True)
    last = len(pair) - 1 - last_rev
    pair_rating = np.asarray(r_val, dtype=np.float64)[last].astype(np.float32)
    assert len(upair) == len(indices)
    return MterData(n_users=int(num_users), n_items=int(num_items), n_aspects=n_aspects, n_opinions=n_opinions,
                    X64=X, X=X.astype(np.float32), X_uids=X_uids.astype(np.int32), X_iids=X_iids.astype(np.int32),
                    X_aids=X_aids.astype(np.int32),
                    YU=YU.astype(np.float32), YU_uids=pu[fu].astype(np.int32), YU_aids=pa[fu].astype(np.int32),
                    YU_oids=po[fu].astype(np.int32),
                    YI=YI.astype(np.float32), YI_iids=pi[fi].astype(np.int32), YI_aids=pa[fi].astype(np.int32),
                    YI_oids=po[fi].astype(np.int32),
                    indptr=indptr, indices=indices, user_ids=user_ids, pair_rating=pair_rating)


def check_data(data):
    """The reference draws from uniform_int_distribution(0, len - 1) over each tensor and the ratings; an empty one is
    undefined behaviour there and an error here, before any device work."""
    for name, n in (("user-item-aspect tensor X (no sentiment reviews)", len(data.X)),
                    ("user-aspect-opinion tensor YU (no positive opinion)", len(data.YU)),
                    ("item-aspect-opinion tensor YI (no positive opinion)", len(data.YI)),
                    ("rating matrix (no ratings)", len(data.indices))):
        if n == 0:
            raise ValueError("MTER cannot sample from an empty %s" % name)


def stream_seeds(rng, n=5):
    """The mt19937 seeds of the five RNGVector streams (uia, uao, iao, pos, neg), in the reference's order: each stream
    takes self.rng.randint(2**31) and seeds its engine with get_rng(that).randint(2**31) (recom_bpr.pyx:54-59).  n:
    the number of streams (ComparERSub has six)."""
    return [int(get_rng(int(rng.randint(2 ** 31))).randint(2 ** 31)) for _ in range(n)]


class MTER(DeviceScoringMixin, Recommender):
    """Multi-Task Explainable Recommendation (Wang et al., SIGIR 2018), trained on the GPU.

    Parameters are the reference's: name="MTER", rating_scale=5.0, n_user_factors=15, n_item_factors=15,
    n_aspect_factors=12, n_opinion_factors=12, n_bpr_samples=1000, n_element_samples=50, lambda_reg=0.1,
    lambda_bpr=10, max_iter=200000, lr=0.1, n_threads=0 (kept for compatibility: the fit runs on the GPU),
    trainable=True, verbose=False, init_params=None ({'U', 'I', 'A', 'O', 'G1', 'G2', 'G3'}; f32 arrays are trained in
    place), seed=None.

    The train set needs a SentimentModality.  With verbose=True each iteration reports the reference's four figures;
    the losses are summed in f64 on the device, so their last digits may differ from the reference's f32 sums; the
    trained parameters do not.
    """

    def __init__(self, name="MTER", rating_scale=5.0, n_user_factors=15, n_item_factors=15, n_aspect_factors=12,
                 n_opinion_factors=12, n_bpr_samples=1000, n_element_samples=50, lambda_reg=0.1, lambda_bpr=10,
                 max_iter=200000, lr=0.1, n_threads=0, trainable=True, verbose=False, init_params=None, seed=None):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.rating_scale = rating_scale
        self.n_user_factors = n_user_factors
        self.n_item_factors = n_item_factors
        self.n_aspect_factors = n_aspect_factors
        self.n_opinion_factors = n_opinion_factors
        self.n_bpr_samples = n_bpr_samples
        self.n_element_samples = n_element_samples
        self.lambda_reg = lambda_reg
        self.lambda_bpr = lambda_bpr
        self.max_iter = max_iter
        self.lr = lr
        self.seed = seed
        if seed is not None:                                   # recom_mter.pyx:180-185
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

    # reference: recom_mter.pyx:198-223
    def _init(self, train_set):
        n_users, n_items = train_set.num_users, train_set.num_items
        n_aspects, n_opinions = train_set.sentiment.num_aspects, train_set.sentiment.num_opinions
        self.num_aspects, self.num_opinions = n_aspects, n_opinions
        d1, d2, d3, d4 = self.n_user_factors, self.n_item_factors, self.n_aspect_factors, self.n_opinion_factors
        for name, shape in (("G1", (d1, d2, d3)), ("G2", (d1, d3, d4)), ("G3", (d2, d3, d4)), ("U", (n_users, d1)),
                            ("I", (n_items, d2)), ("A", (n_aspects + 1, d3)), ("O", (n_opinions, d4))):
            if getattr(self, name) is None:
                setattr(self, name, uniform(shape, random_state=self.rng))

    # reference: recom_mter.pyx:304-429
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        if getattr(train_set, "sentiment", None) is None:
            raise ValueError("MTER needs the sentiment modality: build the train set with a SentimentModality "
                             "(e.g. RatioSplit(..., sentiment=SentimentModality(data=...)))")
        self._init(train_set)
        self._b200_invalidate()
        if not self.trainable:
            return self
        data = build_data(train_set, self.num_users, self.num_items, self.rating_scale)
        check_data(data)
        seeds = stream_seeds(self.rng)
        self._fit_b200(data, seeds)
        return self

    def _shapes(self):
        d1, d2, d3, d4 = self.n_user_factors, self.n_item_factors, self.n_aspect_factors, self.n_opinion_factors
        return (("U", (self.num_users, d1)), ("I", (self.num_items, d2)), ("A", (self.num_aspects + 1, d3)),
                ("O", (self.num_opinions, d4)), ("G1", (d1, d2, d3)), ("G2", (d1, d3, d4)), ("G3", (d2, d3, d4)))

    def _check_params(self):
        """The reference's `floating` buffers take only f32 here (its del_* arrays are float32)."""
        for name, shape in self._shapes():
            x = np.asarray(getattr(self, name))
            if x.dtype != DTYPE:
                got = "double" if x.dtype == np.float64 else str(x.dtype)
                raise ValueError("Buffer dtype mismatch, expected 'float' but got '%s'" % got)
            if x.shape != shape:
                raise ValueError("%s must have shape %s, got %s" % (name, shape, x.shape))

    def _fit_b200(self, data, seeds):
        self._check_params()
        engine.require_cuda()
        n_el, n_bpr = int(self.n_element_samples), int(self.n_bpr_samples)
        if n_el < 1 or n_bpr < 1:
            raise ValueError("n_element_samples and n_bpr_samples must be positive")
        params = [engine.to_device(np.ascontiguousarray(getattr(self, n)), torch.float32) for n, _ in self._shapes()]
        sgrad = [torch.zeros_like(p) for p in params]
        dims = (self.n_user_factors, self.n_item_factors, self.n_aspect_factors, self.n_opinion_factors)
        counts = torch.zeros(3, dtype=torch.int64, device="cuda")
        losses = torch.zeros(3, dtype=torch.float64, device="cuda") if self.verbose else None
        seeded = self.seed is not None
        # seeded: the reference's streams, drawn on the host; unseeded: Philox on the device, keyed by the first
        # stream seed, and the rows' gradients summed without a fixed order (the reference's threads define none)
        fit, draws = self._b200_fit_parts(data, seeds, dims, n_el, n_bpr, 1 if self.verbose else self.max_iter, seeded)
        chunk = 1 if self.verbose else (draws.chunk if seeded else self.max_iter)
        done = 0
        while done < self.max_iter:
            n = min(chunk, self.max_iter - done)
            fit(params, sgrad, draws.next(n) if seeded else None, n, counts=counts, losses=losses,
                unordered=not seeded, philox_seed=None if seeded else seeds[0], iter0=done)
            done += n
            if self.verbose:
                correct, skipped = counts.tolist()[:2]
                loss, bpr_loss = losses.tolist()[:2]
                print("iter %d: loss %.2f, bpr_loss %.2f, correct %.2f%%, skipped %.2f%%"
                      % (done, loss / 3 / n_el, bpr_loss / n_bpr,
                         100.0 * correct / max(n_bpr - skipped, 1), 100.0 * skipped / n_bpr))
                counts.zero_()
                losses.zero_()
        if self.verbose:
            print("Optimization finished!")
        for (name, _), d in zip(self._shapes(), params):
            setattr(self, name, _copy_back(getattr(self, name), d))

    def _b200_fit_parts(self, data, seeds, dims, n_el, n_bpr, max_chunk, seeded):
        """(fit, draws) of _fit_b200: fit(params, sgrad, draws, n_iter, **kw) runs n_iter iterations of the device fit
        over this fit's device data and workspace; draws is the MterDraws of the seeded streams, or None."""
        ddata = engine.MterDeviceData(data)
        work = torch.zeros(engine.mter_workspace_bytes(ddata, dims, n_el, n_bpr), dtype=torch.uint8, device="cuda")
        hyper = dict(lr=self.lr, lambda_reg=self.lambda_reg, lambda_bpr=self.lambda_bpr)

        def fit(params, sgrad, draws, n, **kw):
            engine.mter_fit(ddata, params, sgrad, draws, n, n_el, n_bpr, workspace=work, **hyper, **kw)
        return fit, (MterDraws(seeds, data, n_el, n_bpr, max_chunk) if seeded else None)

    # ---- device scoring: U := Q (the rank queries of every user), V := I --------------------------------------------
    def _b200_device(self):
        dev = getattr(self, "_b200_dev", None)
        if dev is None:
            engine.require_cuda()
            f32 = lambda x: engine.to_device(np.ascontiguousarray(x, dtype=DTYPE), torch.float32)    # noqa: E731
            U, G1, A = f32(self.U), f32(self.G1), f32(self.A)
            Q = engine.mter_queries(U, G1, A)
            dev = dict(U=Q, V=f32(np.asarray(self.I)[: self.num_items]), item_base=None, user_off=None,
                       n_items=self.num_items)
            self._b200_dev = dev
        return dev

    # reference: recom_mter.pyx:677-714
    def score(self, u_idx, i_idx=None):
        if self.is_unknown_user(u_idx):
            raise ScoreException("Can't make score prediction for user %d" % u_idx)
        if i_idx is not None and self.is_unknown_item(i_idx):
            raise ScoreException("Can't make score prediction for item %d" % i_idx)
        if i_idx is None:
            return self._scores_dev([u_idx])[0].cpu().numpy()
        tensor_value1 = np.einsum("abc,a->bc", self.G1, self.U[u_idx])
        tensor_value2 = np.einsum("bc,b->c", tensor_value1, self.I[i_idx])
        return np.einsum("c,c-> ", tensor_value2, self.A[-1])
