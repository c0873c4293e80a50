"""Device-resident scoring/ranking shared by the BPR and MF plug-ins.

Implements the `score()` / `rank()` half of the cornac.models.Recommender contract
(reference: cornac/models/recommender.py:423-441, 476-530) on the GPU, plus the batched
`rank_batch()` that the reference lacks (it ranks one user per Python call).
"""
import numpy as np
import torch

from . import engine
from ._lib import B200Error


class DeviceScoringMixin:
    """Expects the subclass to provide `_b200_host_params()` returning
    (U, V, item_base, user_off_vector_or_None, n_score_items) as numpy arrays."""

    _B200_IGNORED = ("_b200_dev", "_b200_eval_cache")
    _B200_EVAL_CACHE_BYTES = 1 << 30            # host budget of the transform() cache (score rows of the test users)
    _B200_EVAL_TOP = 1024                       # length of the cached per-user global ranking

    def _b200_register_ignored(self):
        for a in self._B200_IGNORED:
            if a not in self.ignored_attrs:
                self.ignored_attrs.append(a)
        self._b200_dev = None
        self._b200_eval_cache = None

    # ---- device cache --------------------------------------------------------------
    def _b200_invalidate(self):
        self._b200_dev = None
        self._b200_eval_cache = None

    # ---- Recommender.transform: batch-precompute what the per-user eval loop will ask for -------------------------
    def transform(self, test_set):
        """`Recommender.transform` hook (cornac/models/recommender.py:410-421), called once by `BaseMethod.evaluate`
        (cornac/eval_methods/base_method.py:746, 766) before the per-user loops of rating_eval / ranking_eval.

        All users of `test_set` are scored in a few batched kernel calls (b200_score_batch, exact scores) and, per user,
        the head of the global ranking (score desc, id asc) is selected on the device (b200_topk_rows); both are kept in
        host memory.  `rank()` / `score()` of a cached user are then pure host work -- no kernel launch, no device copy
        per user -- and return exactly what the uncached path returns: the top-k of ANY candidate set is the first k
        members of the global ranking that belong to it.  The cache is skipped when it would not fit the host budget
        (then, and for callers that never call transform -- hyperopt, cornac/hyperopt.py:162 -- rank() falls back to the
        per-user device path); it is dropped whenever the parameters change (fit)."""
        self._b200_eval_cache = None
        if self._B200_EVAL_CACHE_BYTES <= 0:
            return
        try:
            users = np.unique(np.asarray(test_set.uir_tuple[0], dtype=np.int64))
        except Exception:
            return
        self._b200_precompute_users(users)

    def _b200_precompute_users(self, users):
        d = self._b200_device()
        n_rows, n_score = int(d["U"].shape[0]), int(d["n_items"])
        users = users[(users >= 0) & (users < n_rows)]
        if len(users) == 0 or len(users) * n_score * 4 > self._B200_EVAL_CACHE_BYTES:
            return
        m_top = min(n_score, self._B200_EVAL_TOP)
        scores_h = np.empty((len(users), n_score), dtype=np.float32)
        top_h = np.empty((len(users), m_top), dtype=np.int32)
        batch = max(1, min(len(users), (256 << 20) // (4 * n_score)))
        for b0 in range(0, len(users), batch):
            ub = users[b0:b0 + batch]
            uidx = engine.to_device(ub, torch.int64)
            uoff = None if d["user_off"] is None else d["user_off"][uidx].contiguous()
            sc = engine.score_batch(d["U"], d["V"], user_idx=uidx, item_base=d["item_base"], user_off=uoff, n_items=n_score)
            ids, _ = engine.topk_rows(sc, m_top)
            scores_h[b0:b0 + len(ub)] = sc.cpu().numpy()
            top_h[b0:b0 + len(ub)] = ids.cpu().numpy()
        pos_of = np.full(n_rows, -1, dtype=np.int64)
        pos_of[users] = np.arange(len(users))
        self._b200_eval_cache = dict(pos_of=pos_of, scores=scores_h, top=top_h)

    def _b200_cached_scores(self, user_idx):
        """The cached full score vector of a user (read-only view) or None."""
        c = getattr(self, "_b200_eval_cache", None)
        if c is None or not (0 <= user_idx < len(c["pos_of"])) or c["pos_of"][user_idx] < 0:
            return None
        return c["scores"][c["pos_of"][user_idx]]

    def _b200_cached_rank(self, user_idx, item_indices, k):
        """`Recommender.rank` (recommender.py:476-530) from the transform() cache, or None on a miss: same
        (ranked_items, item_scores) as `_b200_rank` on the device scores."""
        row = self._b200_cached_scores(user_idx)
        if row is None:
            return None
        c = self._b200_eval_cache
        total = self.total_items
        if len(row) == total:
            all_scores = row
        else:                                               # unknown items get the MIN score (recommender.py:507-511)
            all_scores = np.full(total, row.min(), dtype=np.float32)
            all_scores[: len(row)] = row
        item_indices = np.arange(self.num_items) if item_indices is None else np.asarray(item_indices)
        item_scores = all_scores[item_indices]
        n_cand = len(item_indices)
        if k == -1 or k >= n_cand:
            order = np.lexsort((item_indices, -item_scores.astype(np.float64)))
            return item_indices[order], item_scores
        top = c["top"][c["pos_of"][user_idx]]
        member = np.zeros(total, dtype=bool)
        member[item_indices] = True
        surv = top[member[top]]
        if len(surv) >= k:
            topk = surv[:k].astype(item_indices.dtype)
        else:                                               # the cached head holds fewer than k candidates: exact host selection
            order = np.lexsort((item_indices, -item_scores.astype(np.float64)))
            topk = item_indices[order[:k]]
        in_top = np.zeros(total, dtype=bool)
        in_top[topk] = True
        return np.concatenate([topk, item_indices[~in_top[item_indices]]]), item_scores

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

    # ---- scores --------------------------------------------------------------------
    @staticmethod
    def _b200_check_users(user_indices, n_rows):
        """The kernels gather U rows without a bounds check: an index outside [0, n_rows) raises here, like the
        reference's numpy indexing does (IndexError), instead of reading foreign device memory."""
        user_indices = np.asarray(user_indices, dtype=np.int64)
        if user_indices.size and (int(user_indices.min()) < 0 or int(user_indices.max()) >= int(n_rows)):
            bad = user_indices[(user_indices < 0) | (user_indices >= n_rows)]
            raise IndexError("user index %d is out of bounds for the %d user rows of the model" % (int(bad[0]), int(n_rows)))
        return user_indices

    def _b200_scores_dev(self, user_indices):
        """[n_q, n_items] device scores for known users."""
        d = self._b200_device()
        user_indices = self._b200_check_users(user_indices, d["U"].shape[0])
        uidx = torch.as_tensor(user_indices).cuda()
        uoff = None if d["user_off"] is None else d["user_off"][uidx].contiguous()
        return engine.score_batch(d["U"], d["V"], user_idx=uidx, item_base=d["item_base"], user_off=uoff,
                                  n_items=d["n_items"])

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

    @staticmethod
    def _b200_exclusion_rows(user_indices, exclude):
        if exclude is None:
            return None, None
        n_q = len(user_indices)
        sub = exclude[user_indices] if n_q != exclude.shape[0] or not np.array_equal(
            user_indices, np.arange(exclude.shape[0])) else exclude
        sub = sub.tocsr()
        sub.sort_indices()
        return sub.indptr.astype(np.int64), sub.indices.astype(np.int32)

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

    # ---- batched Recommender.recommend ---------------------------------------------
    def recommend_batch(self, batch_users, k=-1, remove_seen=False, train_set=None):
        """Top-k recommendations for many users in one fused kernel call, in ORIGINAL ids: the batched form of
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

    # ---- Recommender.rank ------------------------------------------------------------
    def _b200_rank(self, all_scores_dev, item_indices, k):
        """Reference semantics of Recommender.rank (recommender.py:513-530) given the
        device score vector [1, total]: returns (ranked_items, item_scores)."""
        total = all_scores_dev.shape[1]
        all_item_scores = all_scores_dev[0].cpu().numpy()
        if item_indices is None:
            item_indices = np.arange(self.num_items)
            n_cand_all = self.num_items == total
        else:
            item_indices = np.asarray(item_indices)
            n_cand_all = False
        item_scores = all_item_scores[item_indices]
        n_cand = len(item_indices)
        if k == -1 or k >= n_cand or k > 4096:
            # full ordering requested: not the hot path (MRR-style metrics); host sort with the
            # same total order (score desc, id asc)
            order = np.lexsort((item_indices, -item_scores.astype(np.float64)))
            return item_indices[order], item_scores
        if n_cand_all:
            ex_ptr = ex_idx = None
        else:
            mask = np.ones(total, dtype=bool)
            mask[item_indices] = False
            excl = np.flatnonzero(mask).astype(np.int32)
            ex_ptr = engine.to_device(np.array([0, len(excl)], dtype=np.int64), torch.int64, pinned=False)
            ex_idx = engine.to_device(excl if len(excl) else np.zeros(1, np.int32), torch.int32, pinned=False)
        ids, _ = engine.topk_rows(all_scores_dev, int(k), ex_ptr, ex_idx)
        top = ids[0].cpu().numpy().astype(item_indices.dtype)
        in_top = np.zeros(total, dtype=bool)
        in_top[top] = True
        rest = item_indices[~in_top[item_indices]]
        return np.concatenate([top, rest]), item_scores


class F64RankingMixin:
    """`score()` rows, `rank()`, `rank_batch()`, `recommend_batch()` and the `transform()` cache of the models whose score
    rows are f64 (PMF, EASE), ranked on the device by b200_topk_rows_f64 in the order (score desc, item id asc).  The
    subclass provides `_scores_dev(user_indices)`: the [n_q, num_items] f64 device score rows of known users."""

    _B200_IGNORED = ("_b200_dev", "_b200_eval_cache")
    _B200_EVAL_CACHE_BYTES = 1 << 30            # host budget of the transform() cache (f64 score rows of the test users)
    _B200_EVAL_TOP = 1024                       # length of the cached per-user global ranking

    def _b200_register_f64(self):
        for a in self._B200_IGNORED:
            if a not in self.ignored_attrs:
                self.ignored_attrs.append(a)
        self._b200_dev = None
        self._b200_eval_cache = None

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

    def _b200_row(self, user_idx):
        """A copy of the f64 score row of a known user, from the transform() cache or the device."""
        row = self._cached_row(user_idx)
        return row.copy() if row is not None else self._scores_dev([user_idx])[0].cpu().numpy()

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
