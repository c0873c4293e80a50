"""BPR on an H100: drop-in for cornac.models.BPR.

Same constructor arguments, attributes and fit()/score()/rank() behaviour as the
reference class (cornac/models/bpr/recom_bpr.pyx:65-333); the Cython/OpenMP `_fit_sgd`
(:208-269) is replaced by the sm_90a kernels behind include/b200cornac.h.

Modes (chosen like the reference chooses its thread count, recom_bpr.pyx:132-137):
  * seed given  -> deterministic: the mt19937 sample streams of RNGVector are reproduced on
    the host (b200_mt_sampler_*) and applied by the serial-equivalent replay kernel, so the
    trained factors match the seeded single-thread reference within 1e-4;
  * seed=None   -> Hogwild over the whole GPU with on-device Philox sampling (the analogue
    of the reference's all-cores run, which is not reproducible either).
`mode` ("auto" | "replay" | "hogwild") overrides the choice; it is the only extra argument.
"""
import numpy as np
import torch

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils import get_rng
from cornac.utils.init_utils import uniform, zeros

from . import engine
from ._lib import B200Error
from ._scoring import DeviceScoringMixin

DTYPE = np.float32

# interactions above which a seeded ("auto" -> replay) fit prints a one-time hint: the serial-equivalent replay
# reproduces the seeded reference but runs at ~1e7 samples/s, like one CPU thread; mode="hogwild" keeps the seed
# for initialisation and the sampler key and trains at ~1e9 samples/s
_REPLAY_HINT_NNZ = 5_000_000
_replay_hint_given = False


def check_factor_width(k):
    """The Hogwild kernels keep a factor row in registers, 4 floats (k % 4 == 0) or 1 float per lane and slot, at most
    8 slots of 32 lanes: k <= 1024 when k % 4 == 0, else k <= 256 (b200_bpr_epoch / b200_mf_epoch)."""
    k = int(k)
    if k < 1 or k > 1024 or (k % 4 != 0 and k > 256):
        raise ValueError("k=%d is not supported: the GPU kernels take 1 <= k <= 1024 with k %% 4 == 0, or k <= 256 otherwise "
                         "(pad k to a multiple of 4)" % k)
    return k


def replay_hint(nnz, name):
    global _replay_hint_given
    if nnz > _REPLAY_HINT_NNZ and not _replay_hint_given:
        _replay_hint_given = True
        import warnings
        warnings.warn("%s: seed given -> deterministic replay mode (reference-identical, serial-equivalent, ~1e7 samples/s); "
                      "%d interactions per epoch will take a while.  Pass mode='hogwild' to train on the whole GPU "
                      "(the seed then fixes the initialisation and the sampler key only)." % (name, nnz), stacklevel=3)


class BPR(DeviceScoringMixin, Recommender, ANNMixin):
    """Bayesian Personalized Ranking trained and served on an H100.

    NOTE on `seed`: like the reference (which drops to ONE thread when a seed is given, recom_bpr.pyx:132-133), a seeded
    model trains in the deterministic replay mode -- reference-identical but serial-equivalent (~1e7 samples/s).  For
    large data pass mode="hogwild": the seed still fixes the initial factors and the sampler key, and the epoch runs on
    the whole GPU (~1e9 samples/s).

    Parameters are those of cornac.models.BPR (k, max_iter, learning_rate, lambda_reg,
    use_bias, num_threads, trainable, verbose, init_params, seed) plus `mode` and
    `atomic_updates` (default True: scatter with red.global.add -- no lost updates;
    False = the reference's racy plain stores) in Hogwild mode.
    `num_threads` is accepted for API compatibility and ignored (the GPU is the pool).
    """
    _b200_hinge = False          # MMMF switches the loop body to the hinge variant

    def __init__(self, name="BPR", k=10, max_iter=100, learning_rate=0.001, lambda_reg=0.01, use_bias=True,
                 num_threads=0, trainable=True, verbose=False, init_params=None, seed=None, mode="auto",
                 atomic_updates=True):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.k = check_factor_width(k)
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.lambda_reg = lambda_reg
        self.use_bias = use_bias
        self.seed = seed
        self.rng = get_rng(seed)
        self.num_threads = num_threads
        if mode not in ("auto", "replay", "hogwild"):
            raise ValueError("mode must be 'auto', 'replay' or 'hogwild'")
        self.mode = mode
        self.atomic_updates = atomic_updates

        self.init_params = {} if init_params is None else init_params
        self.u_factors = self.init_params.get("U", None)
        self.i_factors = self.init_params.get("V", None)
        self.i_biases = self.init_params.get("Bi", None)
        self._b200_register_ignored()

    # reference: recom_bpr.pyx:145-152
    def _init(self):
        n_users, n_items = self.total_users, self.total_items
        if self.u_factors is None:
            self.u_factors = (uniform((n_users, self.k), random_state=self.rng, dtype=DTYPE) - 0.5) / self.k
        if self.i_factors is None:
            self.i_factors = (uniform((n_items, self.k), random_state=self.rng, dtype=DTYPE) - 0.5) / self.k
        self.i_biases = zeros(n_items, dtype=DTYPE) if self.i_biases is None or self.use_bias is False else self.i_biases

    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._init()
        self._b200_invalidate()
        if not self.trainable:
            return self

        engine.require_cuda()
        X = train_set.matrix                                   # CSR, sorted indices
        if X.nnz == 0 or self.max_iter <= 0:
            return self
        replay = (self.seed is not None) if self.mode == "auto" else (self.mode == "replay")
        if replay and self.mode == "auto":
            replay_hint(X.nnz, self.name)
        # the two RNGVector seeds are always drawn, in this order (recom_bpr.pyx:190-191)
        s_pos = self.rng.randint(2 ** 31)
        s_neg = self.rng.randint(2 ** 31)
        # thread 0 of each RNGVector is mt19937(get_rng(seed).randint(2**31))  (recom_bpr.pyx:55-58)
        replay_seeds = (get_rng(s_pos).randint(2 ** 31), get_rng(s_neg).randint(2 ** 31)) if replay else None
        # factors are trained in the SAME numpy arrays (init_params arrays are updated in place,
        # recom_bpr.pyx:141-143,197)
        self.u_factors = _writable_f32(self.u_factors)
        self.i_factors = _writable_f32(self.i_factors)
        self.i_biases = _writable_f32(self.i_biases)
        nnz = X.nnz

        def on_epoch(epoch, correct, skipped):
            if self.verbose:
                print("epoch %d: correct %.2f%% skipped %.2f%%" % (
                    epoch, 100.0 * correct / (nnz - skipped + 1e-8), 100.0 * skipped / nnz))

        self.epoch_stats, dev = engine.bpr_train_host(
            X.indptr, X.indices, train_set.num_items, self.u_factors, self.i_factors, self.i_biases,
            self.learning_rate, self.lambda_reg, self.use_bias, self.max_iter,
            key=(int(s_pos) << 31) | int(s_neg), replay_seeds=replay_seeds, atomic=self.atomic_updates,
            hinge=self._b200_hinge,
            on_epoch=on_epoch if self.verbose else None, keep_device=True)
        self._b200_adopt_device(dev[0], dev[1], dev[2], None, self.total_items)
        if self.verbose:
            print("Optimization finished!")
        return self

    def _b200_host_params(self):
        return self.u_factors, self.i_factors, self.i_biases, None, len(self.i_biases)

    # reference: recom_bpr.pyx:272-297
    def score(self, user_idx, item_idx=None):
        if item_idx is None:
            cached = self._b200_cached_scores(user_idx)
            return cached.copy() if cached is not None else self._b200_scores_dev([user_idx])[0].cpu().numpy()
        item_score = self.i_biases[item_idx]
        item_score += np.dot(self.u_factors[user_idx], self.i_factors[item_idx])
        return item_score

    # reference: recommender.py:476-530
    def rank(self, user_idx, item_indices=None, k=-1, **kwargs):
        hit = self._b200_cached_rank(user_idx, item_indices, k)          # filled by transform() before an evaluation
        if hit is not None:
            return hit
        scores = self._b200_scores_dev([user_idx])          # [1, total_items]
        return self._b200_rank(scores, item_indices, k)

    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return np.concatenate((self.u_factors, np.ones([self.u_factors.shape[0], 1])), axis=1)

    def get_item_vectors(self):
        return np.concatenate((self.i_factors, self.i_biases.reshape((-1, 1))), axis=1)


def _writable_f32(a):
    """The array itself when it can be trained in place, else a float32 C-contiguous copy."""
    if isinstance(a, np.ndarray) and a.dtype == DTYPE and a.flags["C_CONTIGUOUS"] and a.flags.writeable:
        return a
    return np.ascontiguousarray(a, dtype=DTYPE).copy()


def _copy_back(host, dev):
    out = dev.cpu().numpy()
    if isinstance(host, np.ndarray) and host.shape == out.shape and host.dtype == out.dtype and host.flags.writeable:
        np.copyto(host, out)
        return host
    return out


class WBPR(BPR):
    """Weighted BPR (negatives sampled in proportion to item popularity): drop-in for
    cornac.models.WBPR (cornac/models/bpr/recom_wbpr.pyx:30-142).  Same kernels as BPR with the
    sampler switched: j = item of a uniformly drawn interaction, one shared RNG stream."""

    def __init__(self, name="WBPR", k=10, max_iter=100, learning_rate=0.001, lambda_reg=0.01, use_bias=True,
                 num_threads=0, trainable=True, verbose=False, init_params=None, seed=None, mode="auto",
                 atomic_updates=True):
        super().__init__(name=name, k=k, max_iter=max_iter, learning_rate=learning_rate, lambda_reg=lambda_reg,
                         use_bias=use_bias, num_threads=num_threads, trainable=trainable, verbose=verbose,
                         init_params=init_params, seed=seed, mode=mode, atomic_updates=atomic_updates)

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
        replay = (self.seed is not None) if self.mode == "auto" else (self.mode == "replay")
        s_vec = self.rng.randint(2 ** 31)                                   # recom_wbpr.pyx:128
        self.u_factors = _writable_f32(self.u_factors)
        self.i_factors = _writable_f32(self.i_factors)
        self.i_biases = _writable_f32(self.i_biases)
        self.epoch_stats, dev = engine.bpr_train_host(
            X.indptr, X.indices, train_set.num_items, self.u_factors, self.i_factors, self.i_biases,
            self.learning_rate, self.lambda_reg, self.use_bias, self.max_iter, key=int(s_vec),
            weighted_seed=get_rng(s_vec).randint(2 ** 31) if replay else None, neg_weighted=True,
            atomic=self.atomic_updates, keep_device=True)
        self._b200_adopt_device(dev[0], dev[1], dev[2], None, self.total_items)
        return self


class MMMF(BPR):
    """Maximum Margin Matrix Factorization: drop-in for cornac.models.MMMF
    (cornac/models/mmmf/recom_mmmf.pyx:33-156) -- BPR's sampler and kernels with the hinge loop body
    (pairs already ranked correctly are left alone, otherwise the BPR update with z = 1; item biases are
    always trained)."""
    _b200_hinge = True

    def __init__(self, name="MMMF", k=10, max_iter=100, learning_rate=0.001, lambda_reg=0.01, num_threads=0,
                 trainable=True, verbose=False, init_params=None, seed=None, mode="auto", atomic_updates=True):
        super().__init__(name=name, k=k, max_iter=max_iter, learning_rate=learning_rate, lambda_reg=lambda_reg,
                         use_bias=True, num_threads=num_threads, trainable=trainable, verbose=verbose,
                         init_params=init_params, seed=seed, mode=mode, atomic_updates=atomic_updates)
