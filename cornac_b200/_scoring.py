"""The scoring half of the cornac.models.Recommender contract, shared by every plug-in.

`score()` rows, `rank()`, `rank_batch()`, `recommend_batch()` and the `transform()` cache (reference:
cornac/models/recommender.py:410-441, 476-580) are implemented once here, over the score rows a model computes on the
device; ranking runs on the device in the order (score desc, item id asc).  A model family supplies only
`_scores_dev(users)`: the f32 factor models through `DeviceScoringMixin` (which adds the fused tensor-core
`rank_batch`), the models scored by two f64 factor matrices through `F64DotScoringMixin`; EASE and the KNN models
define their own.
"""
import numpy as np
import torch

from cornac.exception import ScoreException

from . import engine


class EvalCacheMixin:
    """The transform() cache and the score rows it serves.  The subclass provides `_scores_dev(user_indices)`: the
    [n_q, n] device score rows, in `_B200_SCORE_DTYPE`, of user rows of the model (IndexError outside them)."""

    _B200_IGNORED = ("_b200_dev", "_b200_eval_cache")
    _B200_SCORE_DTYPE = np.float64
    _B200_EVAL_CACHE_BYTES = 1 << 30            # host budget of the transform() cache (score rows of the test users)
    _B200_EVAL_TOP = 1024                       # length of the cached per-user global ranking (0: none)

    def _b200_register_ignored(self):
        for a in self._B200_IGNORED:
            if a not in self.ignored_attrs:
                self.ignored_attrs.append(a)
        self._b200_invalidate()

    def _b200_invalidate(self):
        """Drop the device state and the transform() cache: the parameters changed.  A model restored by load() has
        neither attribute; both are rebuilt lazily."""
        self._b200_dev = None
        self._b200_eval_cache = None

    def _b200_shape(self):
        """(number of user rows, width of a score row) of `_scores_dev`."""
        return self.num_users, self.num_items

    @staticmethod
    def _b200_check_users(user_indices, n_rows):
        """The kernels gather user rows without a bounds check: an index outside [0, n_rows) raises here, like the
        reference's numpy indexing does (IndexError), instead of reading foreign device memory."""
        user_indices = np.asarray(user_indices, dtype=np.int64)
        if user_indices.size and (int(user_indices.min()) < 0 or int(user_indices.max()) >= int(n_rows)):
            bad = user_indices[(user_indices < 0) | (user_indices >= n_rows)]
            raise IndexError("user index %d is out of bounds for the %d user rows of the model" % (int(bad[0]), int(n_rows)))
        return user_indices

    @staticmethod
    def _b200_topk(scores, k, excl_indptr=None, excl_indices=None):
        """Exact top-k (score desc, id asc) of each device row, by the kernel of the rows' dtype."""
        topk = engine.topk_rows if scores.dtype == torch.float32 else engine.topk_rows_f64
        return topk(scores, int(k), excl_indptr, excl_indices)

    # ---- Recommender.transform: batch-precompute what the per-user eval loop will ask for -------------------------
    def transform(self, test_set):
        """`Recommender.transform` hook (cornac/models/recommender.py:410-421), called once by `BaseMethod.evaluate`
        (cornac/eval_methods/base_method.py:746, 766) before the per-user loops of rating_eval / ranking_eval.

        All users of `test_set` are scored in a few batched kernel calls and, per user, the head of the global ranking
        (score desc, id asc) is selected on the device; both are kept in host memory.  `rank()` / `score()` of a cached
        user are then pure host work -- no kernel launch, no device copy per user -- and return exactly what the
        uncached path returns: the top-k of ANY candidate set is the first k members of the global ranking that belong
        to it.  The cache is skipped when it would not fit the host budget (then, and for callers that never call
        transform -- hyperopt, cornac/hyperopt.py:162 -- rank() falls back to the per-user device path); it is dropped
        whenever the parameters change (fit)."""
        self._b200_eval_cache = None
        if self._B200_EVAL_CACHE_BYTES <= 0:
            return
        try:
            users = np.unique(np.asarray(test_set.uir_tuple[0], dtype=np.int64))
        except Exception:
            return
        n_rows, n = self._b200_shape()
        users = users[(users >= 0) & (users < n_rows)]
        size = np.dtype(self._B200_SCORE_DTYPE).itemsize
        if len(users) == 0 or n == 0 or len(users) * n * size > self._B200_EVAL_CACHE_BYTES:
            return
        m_top = min(n, self._B200_EVAL_TOP)
        rows = np.empty((len(users), n), dtype=self._B200_SCORE_DTYPE)
        top = np.empty((len(users), m_top), dtype=np.int32) if m_top else None
        batch = max(1, (256 << 20) // (size * n))
        for b0 in range(0, len(users), batch):
            ub = users[b0:b0 + batch]
            sc = self._scores_dev(ub)
            if m_top:
                top[b0:b0 + len(ub)] = self._b200_topk(sc, m_top)[0].cpu().numpy()
            rows[b0:b0 + len(ub)] = sc.cpu().numpy()
        pos_of = np.full(n_rows, -1, dtype=np.int64)
        pos_of[users] = np.arange(len(users))
        self._b200_eval_cache = dict(pos_of=pos_of, scores=rows, top=top)

    def _b200_cache_pos(self, user_idx):
        """The user's row in the transform() cache, or -1."""
        c = getattr(self, "_b200_eval_cache", None)
        if c is None or not 0 <= user_idx < len(c["pos_of"]):
            return -1
        return c["pos_of"][user_idx]

    def _b200_row(self, user_idx, item_idx=None):
        """The score row of a user row of the model (a copy), or its entries at item_idx: from the transform() cache,
        else from the device."""
        pos = self._b200_cache_pos(user_idx)
        if pos < 0:
            row = self._scores_dev([user_idx])[0].cpu().numpy()
        else:
            row = self._b200_eval_cache["scores"][pos]
            if item_idx is None:
                row = row.copy()
        return row if item_idx is None else row[item_idx]


class ScoringMixin(EvalCacheMixin):
    """`rank()`, `rank_batch()` and `recommend_batch()` over the rows of `_scores_dev`."""

    def _b200_rank_row(self, user_idx):
        """The score row rank() orders for a user outside the transform() cache: a device row of `_scores_dev`, or a
        host row.  A ScoreException scores every item default_score(), as Recommender.rank does (recommender.py:499-503);
        a model whose score(u) serves unknown users overrides this."""
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        return self._scores_dev([user_idx])[0]

    # ---- Recommender.rank ------------------------------------------------------------------------------------------
    def rank(self, user_idx, item_indices=None, k=-1, **kwargs):
        """`Recommender.rank` (recommender.py:476-530) with the total order (score desc, item id asc): for k == -1,
        k >= len(candidates) or k > 4096 every candidate sorted, else the top k sorted and then the other candidates in
        candidate order.  Returns (ranked_items, item_scores)."""
        total = self.total_items
        item_indices = np.arange(self.num_items) if item_indices is None else np.asarray(item_indices)
        pos, row_dev, head = self._b200_cache_pos(user_idx), None, None
        if pos >= 0:
            row, head = self._b200_eval_cache["scores"][pos], self._b200_eval_cache["top"]
            head = None if head is None else head[pos]
        else:
            try:
                row = self._b200_rank_row(user_idx)
            except ScoreException:
                row = np.full(total, self.default_score(), dtype=self._B200_SCORE_DTYPE)
            if isinstance(row, torch.Tensor):
                if len(row) < total:                    # unknown items get the MIN score (:507-511)
                    row = torch.cat((row, row.min().expand(total - len(row))))
                row_dev, row = row, row.cpu().numpy()
            row = np.asarray(row, dtype=self._B200_SCORE_DTYPE)
        if len(row) < total:                            # unknown items get the MIN score (:507-511)
            row = np.concatenate((row, np.full(total - len(row), row.min(), dtype=row.dtype)))
        item_scores = row[item_indices]
        n_cand = len(item_indices)
        if k == -1 or k >= n_cand or k > 4096:          # full ordering: host sort in the same total order
            return item_indices[np.lexsort((item_indices, -item_scores.astype(np.float64)))], item_scores
        topk = None
        if head is not None:                            # the first k candidates of the cached global ranking
            member = np.zeros(len(row), dtype=bool)
            member[item_indices] = True
            surv = head[member[head]]
            topk = surv[:k] if len(surv) >= k else None
        elif row_dev is not None:
            ex_ptr = ex_idx = None
            if not (n_cand == len(row) and np.array_equal(item_indices, np.arange(n_cand))):
                mask = np.ones(len(row), dtype=bool)
                mask[item_indices] = False
                excl = np.flatnonzero(mask).astype(np.int32)
                ex_ptr = engine.to_device(np.array([0, len(excl)], dtype=np.int64), torch.int64, pinned=False)
                ex_idx = engine.to_device(excl if len(excl) else np.zeros(1, np.int32), torch.int32, pinned=False)
            topk = self._b200_topk(row_dev[None, :], k, ex_ptr, ex_idx)[0][0].cpu().numpy()
        if topk is None:                                # a host row, or a cached head with fewer than k candidates
            topk = item_indices[np.lexsort((item_indices, -item_scores.astype(np.float64)))[:k]]
        in_top = np.zeros(len(row), dtype=bool)
        in_top[topk] = True
        return np.concatenate([topk.astype(item_indices.dtype), item_indices[~in_top[item_indices]]]), item_scores

    # ---- batched rank ----------------------------------------------------------------------------------------------
    def rank_batch(self, user_indices, k, exclude=None):
        """Top-k item ids and scores for many users at once.

        user_indices : int array [n_q]
        exclude      : optional scipy CSR matrix (rows = user index) whose stored columns
                       are removed from each user's candidates (e.g. train_set.csr_matrix)
        Returns (ids int32 [n_q, k] (-1 padded), scores [n_q, k] in the dtype of the score rows) as numpy arrays,
        ordered by (score desc, item id asc).
        """
        user_indices = np.asarray(user_indices, dtype=np.int64)
        size = np.dtype(self._B200_SCORE_DTYPE).itemsize
        ids_h = np.empty((len(user_indices), int(k)), dtype=np.int32)
        sc_h = np.empty((len(user_indices), int(k)), dtype=self._B200_SCORE_DTYPE)
        batch = max(1, (256 << 20) // (size * max(self._b200_shape()[1], 1)))
        for b0 in range(0, len(user_indices), batch):
            ub = user_indices[b0:b0 + batch]
            sc = self._scores_dev(ub)
            ep = ei = None
            if exclude is not None:
                ex_ptr, ex_idx = self._b200_exclusion_rows(ub, exclude)
                ep = engine.to_device(ex_ptr, torch.int64)
                ei = engine.to_device(ex_idx if len(ex_idx) else np.zeros(1, np.int32), torch.int32)
            ids, top = self._b200_topk(sc, k, ep, ei)
            ids_h[b0:b0 + len(ub)] = ids.cpu().numpy()
            sc_h[b0:b0 + len(ub)] = top.cpu().numpy()
        return ids_h, sc_h

    @staticmethod
    def _b200_exclusion_rows(user_indices, exclude):
        """The rows of `exclude` of the given users as a CSR with sorted rows: (indptr int64, indices int32)."""
        if exclude is None:
            return None, None
        n_q = len(user_indices)
        sub = exclude[user_indices] if n_q != exclude.shape[0] or not np.array_equal(
            user_indices, np.arange(exclude.shape[0])) else exclude
        sub = sub.tocsr()
        sub.sort_indices()
        return sub.indptr.astype(np.int64), sub.indices.astype(np.int32)

    # ---- batched Recommender.recommend -----------------------------------------------------------------------------
    def recommend_batch(self, batch_users, k=-1, remove_seen=False, train_set=None):
        """Top-k recommendations for many users in one batched ranking, in ORIGINAL ids: the batched form of
        `Recommender.recommend` (cornac/models/recommender.py:532-580), with the signature of the reference's only batched
        precedent (`ANNMixin.recommend_batch`, cornac/models/ann/recom_ann_base.py:182-235).  Seen items are removed
        BEFORE the top-k (every list has k items, unlike the ANN post-filter).  Returns a list of lists of item ids."""
        user_idx = [self.uid_map.get(uid, -1) for uid in batch_users]
        if any(i == -1 for i in user_idx):
            raise ValueError(f"{batch_users} is unknown to the model.")
        if k < -1 or k > self.total_items:
            raise ValueError(f"k={k} is invalid, there are {self.total_users} users in total.")
        if remove_seen and train_set is None:
            raise ValueError("train_set must be provided to remove seen items.")
        if k == -1 or k > 4096 or any(not self.knows_user(u) for u in user_idx):
            # full rankings / unknown users: not the batched path
            return [self.recommend(uid, k=k, remove_seen=remove_seen, train_set=train_set) for uid in batch_users]
        exclude = None
        if remove_seen:
            exclude = train_set.csr_matrix
            n_rows = max(user_idx) + 1
            if exclude.shape[0] < n_rows:                 # users without a training row have nothing to remove
                import scipy.sparse as sp
                exclude = sp.vstack([exclude, sp.csr_matrix((n_rows - exclude.shape[0], exclude.shape[1]), dtype=exclude.dtype)]).tocsr()
        ids, _ = self.rank_batch(np.asarray(user_idx, dtype=np.int64), int(k), exclude=exclude)
        item_ids = self.item_ids
        return [[item_ids[i] for i in row if i >= 0] for row in ids]


class F64DotScoringMixin(ScoringMixin):
    """f64 score rows U[u] . V (b200_score_batch_f64) of the models scored by two f64 factor matrices, named by
    `_B200_FACTORS` (user side, item side)."""

    _B200_FACTORS = ("U", "V")

    def _b200_device(self):
        if getattr(self, "_b200_dev", None) is None:      # None after fit(); absent after load()
            engine.require_cuda()
            u, v = self._B200_FACTORS
            self._b200_dev = dict(U=engine.to_device(np.ascontiguousarray(getattr(self, u)[: self.num_users]), torch.float64),
                                  V=engine.to_device(np.ascontiguousarray(getattr(self, v)[: self.num_items]), torch.float64))
        return self._b200_dev

    def _scores_dev(self, user_indices):
        """[n_q, num_items] f64 device scores V.dot(U[u]) of known users."""
        d = self._b200_device()
        user_indices = self._b200_check_users(user_indices, self.num_users)
        return engine.score_batch_f64(d["U"], d["V"], user_idx=engine.to_device(user_indices, torch.int64))


class DeviceScoringMixin(ScoringMixin):
    """The f32 factor models (BPR, MF and their kin): scores (item_base[i] + user_off[u]) + U[u] . V[i] on the device,
    ranked for many users at once by the fused tensor-core kernel.  Expects the subclass to provide
    `_b200_host_params()` returning (U, V, item_base, user_off_vector_or_None, n_score_items) as numpy arrays."""

    _B200_SCORE_DTYPE = np.float32

    def _b200_device(self):
        dev = getattr(self, "_b200_dev", None)
        if dev is None:
            engine.require_cuda()
            U, V, item_base, user_off, n_items = self._b200_host_params()
            dev = dict(
                U=engine.to_device(U, torch.float32),
                V=engine.to_device(V, torch.float32),
                item_base=None if item_base is None else engine.to_device(item_base, torch.float32),
                user_off=None if user_off is None else engine.to_device(user_off, torch.float32),
                n_items=int(n_items),
            )
            self._b200_dev = dev
        return dev

    def _b200_adopt_device(self, U, V, item_base, user_off, n_items):
        """Keep the freshly trained device tensors as the scoring cache (no re-upload)."""
        self._b200_dev = dict(U=U, V=V, item_base=item_base, user_off=user_off, n_items=int(n_items))

    def _b200_shape(self):
        d = self._b200_device()
        return int(d["U"].shape[0]), d["n_items"]

    def _b200_scores_nan_free(self):
        """True when no score row can hold NaN.  score_batch sums U[u] . V[i] in f64, where products and sums of finite
        f32 values cannot overflow, and rounds it to f32 once; so a NaN needs a non-finite parameter, or an f32 sum
        item_base[i] + user_off[u] that overflows to inf next to a dot product that rounds to the opposite inf."""
        d = self._b200_device()
        bound = 0.0
        for name in ("U", "V", "item_base", "user_off"):
            t = d[name]
            if t is None or t.numel() == 0:
                continue
            if not bool(torch.isfinite(t).all()):
                return False
            if name in ("item_base", "user_off"):
                bound += float(t.abs().max())
        return bound <= float(np.finfo(np.float32).max)

    def _b200_packed_items(self, n_rank):
        """fp16 tile images of the item side for the fused rank, built once per (trained model, candidate count) and kept
        with the device cache: V and the item base are constant until the next fit() / parameter change, which drops
        the whole cache (_b200_invalidate)."""
        d = self._b200_device()
        cache = d.setdefault("packed", {})
        if n_rank not in cache:
            cache.clear()                                   # one candidate count at a time (288 MB at 1 M items)
            cache[n_rank] = engine.rank_pack_items(d["V"], d["item_base"], n_rank)
        return cache[n_rank]

    def _scores_dev(self, user_indices, n_items=None, out=None):
        """[n_q, n_items] f32 device scores of user rows of the model (n_items: the first n_items items, default all
        scored items; out: an optional [n_q, n_items] f32 device buffer to write)."""
        d = self._b200_device()
        user_indices = self._b200_check_users(user_indices, d["U"].shape[0])
        uidx = torch.as_tensor(user_indices).cuda()
        uoff = None if d["user_off"] is None else d["user_off"][uidx].contiguous()
        return engine.score_batch(d["U"], d["V"], user_idx=uidx, item_base=d["item_base"], user_off=uoff,
                                  n_items=d["n_items"] if n_items is None else n_items, out=out)

    # ---- batched rank (the throughput path) ----------------------------------------
    def rank_batch(self, user_indices, k, exclude=None):
        """Top-k item ids and scores for many users at once.

        user_indices : int array [n_q]
        exclude      : optional scipy CSR matrix (rows = user index) whose stored columns
                       are removed from each user's candidates (e.g. train_set.csr_matrix)
        Returns (ids int32 [n_q, k] (-1 padded), scores float32 [n_q, k]) as numpy arrays,
        ordered by (score desc, item id asc).
        """
        d = self._b200_device()
        user_indices = self._b200_check_users(user_indices, d["U"].shape[0])
        ex_ptr, ex_idx = self._b200_exclusion_rows(user_indices, exclude)
        if d["user_off"] is None and d["n_items"] == d["V"].shape[0]:
            return engine.rank_topk_host(d["U"], d["V"], int(k), user_indices, item_base=d["item_base"],
                                         excl_indptr=ex_ptr, excl_indices=ex_idx, packed_items=self._b200_packed_items(d["n_items"]))
        ids, sc = self.rank_batch_device(user_indices, k, exclude=exclude, _rows=(ex_ptr, ex_idx))
        return ids.cpu().numpy(), sc.cpu().numpy()

    def rank_batch_device(self, user_indices, k, exclude=None, _rows=None, n_items=None):
        """`rank_batch` leaving the result on the GPU: (ids int32 [n_q, k], scores f32 [n_q, k]) CUDA tensors
        (what the device-side metric reduction of cornac_b200.evaluation consumes).  `n_items` restricts the candidates
        to the first n_items item rows (ranking_eval with exclude_unknowns: only the train items, base_method.py:200-202)."""
        d = self._b200_device()
        user_indices = self._b200_check_users(user_indices, d["U"].shape[0])
        ex_ptr, ex_idx = _rows if _rows is not None else self._b200_exclusion_rows(user_indices, exclude)
        uidx = engine.to_device(user_indices, torch.int64)
        uoff = None if d["user_off"] is None else d["user_off"][uidx].contiguous()
        ep = None if ex_ptr is None else engine.to_device(ex_ptr, torch.int64)
        ei = None if ex_ptr is None else (engine.to_device(ex_idx, torch.int32) if len(ex_idx) else
                                          torch.zeros(1, dtype=torch.int32, device="cuda"))
        n_rank = d["n_items"] if n_items is None else min(int(n_items), d["n_items"])
        return engine.rank_topk(d["U"], d["V"], int(k), user_idx=uidx, item_base=d["item_base"], user_off=uoff,
                                excl_indptr=ep, excl_indices=ei, n_items=n_rank, packed_items=self._b200_packed_items(n_rank))
