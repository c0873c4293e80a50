"""Probabilistic matrix factorisation on an H100: drop-in for cornac.models.PMF.

Same constructor arguments, defaults, attributes, errors and fit()/score()/rank() behaviour as the reference class
(cornac/models/pmf/recom_pmf.py:25-252).  Data preparation and the initial factors are the reference's host numpy; the
serial RMSProp loops of pmf_linear / pmf_non_linear (cornac/models/pmf/cython/pmf.pyx:55-173) run as b200_pmf_fit over a
level schedule of the ratings, with the reference's f64 arithmetic, so U and V are bit-identical to the reference's.
The full score rows of score(u) / rank() are f64 device dots (b200_score_batch_f64) ranked on the device
(b200_topk_rows_f64).
"""
import numpy as np
import torch

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils import get_rng
from cornac.utils.common import scale, sigmoid
from cornac.utils.init_utils import normal

from . import engine

VARIANTS = ("linear", "non_linear")


class PMF(Recommender, ANNMixin):
    """Probabilistic Matrix Factorization (Mnih and Salakhutdinov, NIPS 2008), trained on the GPU.

    Parameters are the reference's: k=5, max_iter=100, learning_rate=0.001, gamma=0.9, lambda_reg=0.001, name="PMF",
    variant="non_linear" ("linear" or "non_linear"), trainable=True, verbose=False, init_params=None ({'U': ..., 'V': ...},
    f64 arrays, trained in place), seed=None (initial factors only; the fit itself is deterministic).
    """

    _B200_IGNORED = ("_b200_dev", "_b200_eval_cache")
    _B200_EVAL_CACHE_BYTES = 1 << 30            # host budget of the transform() cache (f64 score rows of the test users)
    _B200_EVAL_TOP = 1024                       # length of the cached per-user global ranking
    _B200_LOSS_BYTES = 256 << 20                # device budget of the per-rating loss terms when verbose

    def __init__(self, k=5, max_iter=100, learning_rate=0.001, gamma=0.9, lambda_reg=0.001, name="PMF",
                 variant="non_linear", trainable=True, verbose=False, init_params=None, seed=None):
        Recommender.__init__(self, name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.gamma = gamma
        self.lambda_reg = lambda_reg
        self.variant = variant
        self.seed = seed

        self.ll = np.full(max_iter, 0)
        self.eps = 0.000000001

        self.init_params = {} if init_params is None else init_params
        self.U = self.init_params.get("U", None)
        self.V = self.init_params.get("V", None)
        for a in self._B200_IGNORED:
            if a not in self.ignored_attrs:
                self.ignored_attrs.append(a)
        self._b200_dev = None
        self._b200_eval_cache = None

    # reference: recom_pmf.py:108-189
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set)
        self._b200_dev = None
        self._b200_eval_cache = None
        if self.trainable:
            uid, iid, rat = train_set.uir_tuple
            rat = np.array(rat, dtype="float32")
            if self.variant == "non_linear":
                if [self.min_rating, self.max_rating] != [0, 1]:
                    rat = scale(rat, 0.0, 1.0, self.min_rating, self.max_rating)
            uid = np.array(uid, dtype="int32")
            iid = np.array(iid, dtype="int32")
            if self.verbose:
                print("Learning...")
            if self.variant not in VARIANTS:
                raise ValueError('variant must be one of {"linear","non_linear"}')
            self._fit_b200(uid, iid, rat.astype(np.float32))
            if self.verbose:
                print("Learning completed")
        elif self.verbose:
            print("%s is trained already (trainable = False)" % (self.name))
        return self

    def _init_factors(self):
        """pmf.pyx:40-51: U drawn before V from one generator, each only when init_params does not supply it."""
        rng = get_rng(self.seed)
        U = self.U
        if U is None:
            U = normal((self.num_users, self.k), mean=0.0, std=0.001, random_state=rng, dtype=np.double)
        V = self.V
        if V is None:
            V = normal((self.num_items, self.k), mean=0.0, std=0.001, random_state=rng, dtype=np.double)
        for name, x, n in (("U", U, self.num_users), ("V", V, self.num_items)):
            x = np.asarray(x)
            if x.dtype != np.float64:                         # what the reference's double[:, :] memoryview raises
                raise ValueError("Buffer dtype mismatch, expected 'double' but got '%s'" % x.dtype)
            if x.ndim != 2 or x.shape[0] < n or x.shape[1] != self.k:
                raise ValueError("%s must have shape (%d, %d), got %s" % (name, n, self.k, x.shape))
        return U, V

    def _fit_b200(self, uid, iid, rat):
        U, V = self._init_factors()
        engine.require_cuda()
        data = engine.PmfData(uid, iid, rat, self.num_users, self.num_items)
        Ud = engine.to_device(np.ascontiguousarray(U), torch.float64)
        Vd = engine.to_device(np.ascontiguousarray(V), torch.float64)
        cu, cv = torch.zeros_like(Ud), torch.zeros_like(Vd)
        hyper = (float(np.float32(self.lambda_reg)), float(np.float32(self.learning_rate)), float(np.float32(self.gamma)))
        if self.verbose and data.nnz > 0:
            # each rating's loss term lands at its stored index; summing a row in stored order is the reference's sum
            chunk = max(1, self._B200_LOSS_BYTES // (8 * data.nnz))
            for e0 in range(0, self.max_iter, chunk):
                n = min(chunk, self.max_iter - e0)
                terms = torch.empty((n, data.nnz), dtype=torch.float64, device="cuda")
                engine.pmf_fit(data, self.variant, Ud, Vd, cu, cv, n, *hyper, loss=terms)
                loss = np.add.accumulate(terms.cpu().numpy(), axis=1)[:, -1]
                for j in range(n):
                    print("epoch %i, loss: %f" % (e0 + j, loss[j]))
        elif self.verbose:
            for e in range(self.max_iter):
                print("epoch %i, loss: %f" % (e, 0.0))
        else:
            engine.pmf_fit(data, self.variant, Ud, Vd, cu, cv, self.max_iter, *hyper)
        # an f64 init_params array is trained in place, as through the reference's memoryview
        U[...] = Ud.cpu().numpy()
        V[...] = Vd.cpu().numpy()
        self.U, self.V = U, V
        self._b200_dev = dict(U=Ud, V=Vd) if U.shape == (self.num_users, self.k) and V.shape == (self.num_items, self.k) else None

    # ---- device scores ---------------------------------------------------------------------------------------------
    def _b200_device(self):
        if getattr(self, "_b200_dev", None) is None:          # None after fit(); absent after load()
            engine.require_cuda()
            self._b200_dev = dict(U=engine.to_device(np.ascontiguousarray(self.U[: self.num_users]), torch.float64),
                                  V=engine.to_device(np.ascontiguousarray(self.V[: self.num_items]), torch.float64))
        return self._b200_dev

    def _scores_dev(self, user_indices):
        """[n_q, num_items] f64 device scores V.dot(U[u]) of known users."""
        d = self._b200_device()
        user_indices = np.asarray(user_indices, dtype=np.int64)
        if user_indices.size and (int(user_indices.min()) < 0 or int(user_indices.max()) >= self.num_users):
            raise IndexError("user index out of bounds for the %d users of the model" % self.num_users)
        return engine.score_batch_f64(d["U"], d["V"], user_idx=engine.to_device(user_indices, torch.int64))

    # ---- Recommender.transform: the score rows and ranking heads of every test user --------------------------------
    def transform(self, test_set):
        """`Recommender.transform` hook (cornac/models/recommender.py:410-421), called once by BaseMethod.evaluate before
        the per-user loops: the f64 score rows of all users of `test_set` and, per user, the head of the global ranking
        (score desc, id asc, b200_topk_rows_f64) are computed in a few kernel calls and kept in host memory, so that
        score(u), rank() and rate() of those users are host work.  Skipped when the rows do not fit the host budget."""
        self._b200_eval_cache = None
        if self._B200_EVAL_CACHE_BYTES <= 0:
            return
        try:
            users = np.unique(np.asarray(test_set.uir_tuple[0], dtype=np.int64))
        except Exception:
            return
        users = users[(users >= 0) & (users < self.num_users)]
        n = self.num_items
        if len(users) == 0 or n == 0 or len(users) * n * 8 > self._B200_EVAL_CACHE_BYTES:
            return
        m_top = min(n, self._B200_EVAL_TOP)
        rows = np.empty((len(users), n), dtype=np.float64)
        top = np.empty((len(users), m_top), dtype=np.int32)
        batch = max(1, (256 << 20) // (8 * n))
        for b0 in range(0, len(users), batch):
            ub = users[b0:b0 + batch]
            sc = self._scores_dev(ub)
            ids, _ = engine.topk_rows_f64(sc, m_top)
            rows[b0:b0 + len(ub)] = sc.cpu().numpy()
            top[b0:b0 + len(ub)] = ids.cpu().numpy()
        pos_of = np.full(self.num_users, -1, dtype=np.int64)
        pos_of[users] = np.arange(len(users))
        self._b200_eval_cache = dict(pos_of=pos_of, scores=rows, top=top)

    def _cached_row(self, user_idx):
        c = getattr(self, "_b200_eval_cache", None)
        if c is None or not (0 <= user_idx < len(c["pos_of"])) or c["pos_of"][user_idx] < 0:
            return None
        return c["scores"][c["pos_of"][user_idx]]

    # reference: recom_pmf.py:191-222
    def score(self, user_idx, item_idx=None):
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            row = self._cached_row(user_idx)
            return row.copy() if row is not None else self._scores_dev([user_idx])[0].cpu().numpy()
        # one item: the reference's host expression (a cached row is never used here: it holds the raw dot)
        user_pred = self.V[item_idx, :].dot(self.U[user_idx, :])
        if self.variant == "non_linear":
            user_pred = sigmoid(user_pred)
            user_pred = scale(user_pred, self.min_rating, self.max_rating, 0.0, 1.0)
        return user_pred

    # reference: recommender.py:476-530, with the total order (score desc, item id asc)
    def rank(self, user_idx, item_indices=None, k=-1, **kwargs):
        total = self.total_items
        item_indices = np.arange(self.num_items) if item_indices is None else np.asarray(item_indices)
        if not self.knows_user(user_idx):                      # score() raises ScoreException: every item gets default_score
            item_scores = (np.ones(total) * self.default_score())[item_indices]
            return item_indices[np.lexsort((item_indices, -item_scores))], item_scores
        row = self._cached_row(user_idx)
        c = self._b200_eval_cache if row is not None else None
        if row is None:
            row_dev = self._scores_dev([user_idx])
            row = row_dev[0].cpu().numpy()
        if len(row) == total:
            all_scores = row
        else:                                                  # unknown items get the MIN score (:507-511)
            all_scores = np.ones(total) * np.min(row)
            all_scores[: len(row)] = row
        item_scores = all_scores[item_indices]
        n_cand = len(item_indices)
        if k == -1 or k >= n_cand or k > 4096:
            return item_indices[np.lexsort((item_indices, -item_scores))], item_scores
        topk = None
        if c is not None:                                      # the first k candidates of the cached global ranking
            head = c["top"][c["pos_of"][user_idx]]
            member = np.zeros(total, dtype=bool)
            member[item_indices] = True
            surv = head[member[head]]
            if len(surv) >= k:
                topk = surv[:k].astype(item_indices.dtype)
            else:
                topk = item_indices[np.lexsort((item_indices, -item_scores))[:k]]
        else:
            all_dev = torch.from_numpy(np.ascontiguousarray(all_scores)).cuda()[None, :]
            ex_ptr = ex_idx = None
            if not (n_cand == total and np.array_equal(item_indices, np.arange(total))):
                mask = np.ones(total, dtype=bool)
                mask[item_indices] = False
                excl = np.flatnonzero(mask).astype(np.int32)
                ex_ptr = engine.to_device(np.array([0, len(excl)], dtype=np.int64), torch.int64, pinned=False)
                ex_idx = engine.to_device(excl if len(excl) else np.zeros(1, np.int32), torch.int32, pinned=False)
            ids, _ = engine.topk_rows_f64(all_dev, int(k), ex_ptr, ex_idx)
            topk = ids[0].cpu().numpy().astype(item_indices.dtype)
        in_top = np.zeros(total, dtype=bool)
        in_top[topk] = True
        return np.concatenate([topk, item_indices[~in_top[item_indices]]]), item_scores

    # ---- batched rank ------------------------------------------------------------------------------------------------
    def rank_batch(self, user_indices, k, exclude=None):
        """Top-k item ids and scores for many users at once: (ids int32 [n_q, k] (-1 padded), scores f64 [n_q, k]) as numpy
        arrays in the order (score desc, item id asc).  exclude: optional scipy CSR matrix (rows = user index) whose
        stored columns are removed from each user's candidates (e.g. train_set.csr_matrix)."""
        user_indices = np.asarray(user_indices, dtype=np.int64)
        n_q, n = len(user_indices), self.num_items
        ids_h = np.empty((n_q, int(k)), dtype=np.int32)
        sc_h = np.empty((n_q, int(k)), dtype=np.float64)
        batch = max(1, (256 << 20) // (8 * max(n, 1)))
        for b0 in range(0, n_q, batch):
            ub = user_indices[b0:b0 + batch]
            sc = self._scores_dev(ub)
            ep = ei = None
            if exclude is not None:
                sub = exclude[ub].tocsr()
                sub.sort_indices()
                ep = engine.to_device(sub.indptr.astype(np.int64), torch.int64)
                ei = engine.to_device(sub.indices.astype(np.int32) if sub.nnz else np.zeros(1, np.int32), torch.int32)
            ids, top = engine.topk_rows_f64(sc, int(k), ep, ei)
            ids_h[b0:b0 + len(ub)] = ids.cpu().numpy()
            sc_h[b0:b0 + len(ub)] = top.cpu().numpy()
        return ids_h, sc_h

    def recommend_batch(self, batch_users, k=-1, remove_seen=False, train_set=None):
        """The batched form of `Recommender.recommend` (cornac/models/recommender.py:532-580): top-k recommendations of
        many users, in ORIGINAL ids.  Seen items are removed before the top-k.  Returns a list of lists of item ids."""
        user_idx = [self.uid_map.get(uid, -1) for uid in batch_users]
        if any(i == -1 for i in user_idx):
            raise ValueError(f"{batch_users} is unknown to the model.")
        if k < -1 or k > self.total_items:
            raise ValueError(f"k={k} is invalid, there are {self.total_users} users in total.")
        if remove_seen and train_set is None:
            raise ValueError("train_set must be provided to remove seen items.")
        if k == -1 or k > 4096 or any(not self.knows_user(u) for u in user_idx):
            return [self.recommend(uid, k=k, remove_seen=remove_seen, train_set=train_set) for uid in batch_users]
        exclude = None
        if remove_seen:
            exclude = train_set.csr_matrix
            n_rows = max(user_idx) + 1
            if exclude.shape[0] < n_rows:                     # users without a training row have nothing to remove
                import scipy.sparse as sp
                exclude = sp.vstack([exclude, sp.csr_matrix((n_rows - exclude.shape[0], exclude.shape[1]),
                                                            dtype=exclude.dtype)]).tocsr()
        ids, _ = self.rank_batch(np.asarray(user_idx, dtype=np.int64), int(k), exclude=exclude)
        item_ids = self.item_ids
        return [[item_ids[i] for i in row if i >= 0] for row in ids]

    # ---- ANNMixin (recom_pmf.py:224-252) -----------------------------------------------------------------------------
    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return self.U

    def get_item_vectors(self):
        return self.V
