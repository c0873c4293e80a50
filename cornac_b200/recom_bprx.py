"""VEBPR and SBPR on an H100: drop-ins for cornac.models.VEBPR / cornac.models.SBPR (SURVEY.md 8(f)-3).

Both are BPR with a THIRD item per sample -- a viewed-but-not-purchased item (VEBPR,
cornac/models/bpr/recom_vebpr.pyx:50-392) or an item a friend has (SBPR, cornac/models/sbpr/recom_sbpr.pyx:38-300) --
and run on the kernels of csrc/bprx.cu behind b200_vebpr_* / b200_sbpr_* (include/b200cornac.h).  Constructor arguments,
attribute names and fit()/score()/rank() behaviour are the reference classes'; `mode` ("auto" | "replay" | "hogwild") is the
one extra argument and means what it means for cornac_b200.BPR: a seed selects the deterministic replay of the reference's
seeded single-thread sample stream (trained factors within 1e-4 of the reference), no seed the Hogwild epoch over the GPU.
"""
import numpy as np

from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils import get_rng
from cornac.utils.init_utils import uniform, zeros

from . import engine
from ._scoring import DeviceScoringMixin
from .recom_bpr import BPR, DTYPE, _writable_f32, replay_hint


def check_tri_factor_width(k):
    """The four-row kernels keep a sample's rows in registers: k <= 512 when k % 4 == 0, else k <= 128 (csrc/bprx.cu)."""
    k = int(k)
    if k < 1 or k > 512 or (k % 4 != 0 and k > 128):
        raise ValueError("k=%d is not supported: the VEBPR / SBPR kernels take 1 <= k <= 512 with k %% 4 == 0, or k <= 128 "
                         "otherwise (pad k to a multiple of 4)" % k)
    return k


class VEBPR(DeviceScoringMixin, Recommender, ANNMixin):
    """View-Enhanced BPR trained and served on an H100.  Parameters are those of cornac.models.VEBPR (k, max_iter,
    learning_rate, lambda_reg, num_threads, trainable, verbose, init_params, seed, alpha) plus `mode`; the train set must be a
    cornac.data.PurchaseViewDataset (its `view_matrix` = viewed-but-not-purchased CSR with sorted rows)."""

    def __init__(self, name="VEBPR", k=10, max_iter=100, learning_rate=0.01, lambda_reg=0.1, num_threads=0, trainable=True,
                 verbose=False, init_params=None, seed=None, alpha=0.5, mode="auto"):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.k = check_tri_factor_width(k)
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.lambda_reg = lambda_reg
        self.alpha = float(alpha)
        self.seed = seed
        self.rng = get_rng(seed)
        self.num_threads = num_threads
        if mode not in ("auto", "replay", "hogwild"):
            raise ValueError("mode must be 'auto', 'replay' or 'hogwild'")
        self.mode = mode
        self.init_params = {} if init_params is None else init_params
        self.u_factor = self.init_params.get("U", None)
        self.i_factor = self.init_params.get("V", None)
        self._b200_register_ignored()

    # reference: recom_vebpr.pyx:133-139
    def _init(self):
        n_users, n_items = self.total_users, self.total_items
        if self.u_factor is None:
            self.u_factor = (uniform((n_users, self.k), random_state=self.rng, dtype=DTYPE) - 0.5) / self.k
        if self.i_factor is None:
            self.i_factor = (uniform((n_items, self.k), random_state=self.rng, dtype=DTYPE) - 0.5) / self.k

    # reference: recom_vebpr.pyx:151-210
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        from cornac.data import PurchaseViewDataset
        if not isinstance(train_set, PurchaseViewDataset):
            raise ValueError(
                "VEBPR requires a PurchaseViewDataset. Build one with "
                "PurchaseViewDataset.build(purchase_data, view_data) or "
                "PurchaseViewDataset.attach_view(dataset, view_data)."
            )
        self.view_matrix = train_set.view_matrix
        self._init()
        self._b200_invalidate()
        if not self.trainable:
            return self
        engine.require_cuda()
        X, W = train_set.matrix, train_set.view_matrix
        if X.nnz == 0 or self.max_iter <= 0:
            return self
        replay = (self.seed is not None) if self.mode == "auto" else (self.mode == "replay")
        if replay and self.mode == "auto":
            replay_hint(X.nnz, self.name)
        # the three RNGVector seeds are always drawn, in this order (recom_vebpr.pyx:198-200)
        seeds = [self.rng.randint(2 ** 31) for _ in range(3)]
        replay_seeds = tuple(get_rng(s).randint(2 ** 31) for s in seeds) if replay else None
        self.u_factor = _writable_f32(self.u_factor)
        self.i_factor = _writable_f32(self.i_factor)
        nnz = X.nnz

        def on_epoch(epoch, correct, skipped):
            print("epoch %d: correct %.2f%% skipped %.2f%%" % (epoch, 100.0 * correct / (nnz - skipped + 1e-8), 100.0 * skipped / nnz))

        self.epoch_stats, dev = engine.tri_train_host(
            "vebpr", X.indptr, X.indices, (W.indptr, W.indices), train_set.num_items, self.u_factor, self.i_factor, None,
            dict(lr=self.learning_rate, reg=self.lambda_reg, alpha=self.alpha), self.max_iter,
            key=(int(seeds[0]) << 31) ^ (int(seeds[1]) << 15) ^ int(seeds[2]), replay_seeds=replay_seeds,
            on_epoch=on_epoch if self.verbose else None, keep_device=True)
        self._b200_adopt_device(dev[0], dev[1], None, None, self.total_items)
        if self.verbose:
            print("Optimization finished!")
        return self

    def _b200_host_params(self):
        return self.u_factor, self.i_factor, None, None, self.i_factor.shape[0]

    # reference: recom_vebpr.pyx:339-363
    def score(self, user_idx, item_idx=None):
        if item_idx is None:
            cached = self._b200_cached_scores(user_idx)
            return cached.copy() if cached is not None else self._b200_scores_dev([user_idx])[0].cpu().numpy()
        return np.dot(self.u_factor[user_idx], self.i_factor[item_idx])

    # reference: recommender.py:476-530
    def rank(self, user_idx, item_indices=None, k=-1, **kwargs):
        hit = self._b200_cached_rank(user_idx, item_indices, k)
        if hit is not None:
            return hit
        return self._b200_rank(self._b200_scores_dev([user_idx]), item_indices, k)

    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return self.u_factor

    def get_item_vectors(self):
        return self.i_factor


def prepare_social_data(X, Y):
    """SBPR._prepare_social_data (recom_sbpr.pyx:119-145) without the per-user Python loop: X = train CSR [n_users, n_items],
    Y = social CSR [n_users, n_users] (Y[u] = the friends of u among the train users).  Per user: the items her friends
    have and she has not, ascending, with the number of friends having each.  Returns (social_item_ids,
    social_item_counts, social_indptr) with X.indices' dtype, like the reference."""
    import scipy.sparse as sp
    Xb = sp.csr_matrix((np.ones(X.nnz, dtype=np.int64), X.indices, X.indptr), shape=X.shape)
    Xb.sum_duplicates()
    Xb.data[:] = 1                                          # np.unique(X[uid].indices): an item counts once per friend row
    # the reference concatenates the rows X[f] for every stored entry f of Y[uid] (duplicated friends count twice)
    Yc = sp.csr_matrix((np.ones(len(Y.indices), dtype=np.int64), Y.indices, Y.indptr), shape=Y.shape)
    Yc.sum_duplicates()
    Xc = sp.csr_matrix((np.ones(X.nnz, dtype=np.int64), X.indices, X.indptr), shape=X.shape)
    Xc.sum_duplicates()                                      # X[f].indices may repeat an item: each repeat counts (np.unique counts)
    S = (Yc @ Xc).tocsr()                                    # S[u, i] = number of (friend, occurrence) pairs having i
    S = S - S.multiply(Xb)                                   # drop the user's own items
    S.eliminate_zeros()
    S.sort_indices()
    dt = X.indices.dtype
    return S.indices.astype(dt), S.data.astype(dt), S.indptr.astype(dt)


class SBPR(BPR):
    """Social BPR trained and served on an H100.  Parameters are those of cornac.models.SBPR (k, max_iter, learning_rate,
    lambda_u, lambda_v, lambda_b, use_bias, num_threads, trainable, verbose, init_params, seed) plus `mode`; the train set
    must carry a `user_graph` modality.

    NOTE: the reference's SBPR.fit cannot run as written -- it calls self._prepare_data() and self._prepare_social_data()
    without the train_set argument (recom_sbpr.pyx:168-169, a TypeError).  This fit() does what that method names, in its
    order: Recommender.fit, _init, the social-item lists, the two RNGVector seeds, max_iter epochs of _fit_sgd (:193-300);
    the parity fixture (tests/golden/sbpr_mid_k16.npz) drives the reference's compiled _fit_sgd the same way."""

    def __init__(self, name="SBPR", k=10, max_iter=100, learning_rate=0.001, lambda_u=0.01, lambda_v=0.01, lambda_b=0.01,
                 use_bias=True, num_threads=0, trainable=True, verbose=False, init_params=None, seed=None, mode="auto"):
        super().__init__(name=name, k=k, max_iter=max_iter, learning_rate=learning_rate, use_bias=use_bias,
                         num_threads=num_threads, trainable=trainable, verbose=verbose, init_params=init_params, seed=seed,
                         mode=mode)
        check_tri_factor_width(k)
        self.lambda_u = lambda_u
        self.lambda_v = lambda_v
        self.lambda_b = lambda_b

    def _prepare_social_data(self, train_set):
        from scipy.sparse import csr_matrix
        X = train_set.matrix
        n_users = train_set.num_users
        train_user_indices = set(train_set.uir_tuple[0])
        rid, cid, val = train_set.user_graph.get_train_triplet(train_user_indices, train_user_indices)
        Y = csr_matrix((val, (rid, cid)), shape=(n_users, n_users))
        return prepare_social_data(X, Y)

    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._init()
        self._b200_invalidate()
        if not self.trainable:
            return self
        engine.require_cuda()
        X = train_set.matrix
        if X.nnz == 0 or self.max_iter <= 0:
            return self
        if getattr(train_set, "user_graph", None) is None:
            raise ValueError("SBPR requires a train set with a user_graph modality (cornac.data.GraphModality)")
        s_ids, s_cnts, s_indptr = self._prepare_social_data(train_set)
        replay = (self.seed is not None) if self.mode == "auto" else (self.mode == "replay")
        if replay and self.mode == "auto":
            replay_hint(X.nnz, self.name)
        s_pos = self.rng.randint(2 ** 31)                                  # recom_sbpr.pyx:173-174
        s_neg = self.rng.randint(2 ** 31)
        replay_seeds = (get_rng(s_pos).randint(2 ** 31), get_rng(s_neg).randint(2 ** 31)) if replay else None
        self.u_factors = _writable_f32(self.u_factors)
        self.i_factors = _writable_f32(self.i_factors)
        self.i_biases = _writable_f32(self.i_biases)
        nnz = X.nnz

        def on_epoch(epoch, correct, skipped):
            print("epoch %d: skipped %.2f%%" % (epoch, 100.0 * skipped / nnz))

        self.epoch_stats, dev = engine.tri_train_host(
            "sbpr", X.indptr, X.indices, (s_indptr, s_ids, s_cnts), train_set.num_items, self.u_factors, self.i_factors,
            self.i_biases, dict(lr=self.learning_rate, lambda_u=self.lambda_u, lambda_v=self.lambda_v, lambda_b=self.lambda_b,
                                use_bias=self.use_bias), self.max_iter,
            key=(int(s_pos) << 31) | int(s_neg), replay_seeds=replay_seeds, on_epoch=on_epoch if self.verbose else None,
            keep_device=True)
        self._b200_adopt_device(dev[0], dev[1], dev[2], None, self.total_items)
        if self.verbose:
            print("Optimization finished!")
        return self
