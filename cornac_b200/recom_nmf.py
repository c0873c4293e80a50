"""Non-negative matrix factorisation on an H100: drop-in for cornac.models.NMF.

Same constructor arguments, defaults, attributes and fit()/score() behaviour as the reference class
(cornac/models/nmf/recom_nmf.pyx:37-350).  Initialisation and data preparation are the reference's host numpy; the
compiled loop of `_fit_sgd` (:182-267) runs as b200_nmf_fit, in the reference's f32 arithmetic and summation order, so
the trained factors and biases are bit-identical to the reference's.  score(u) / rank() / rank_batch() are the shared
device scoring path (DeviceScoringMixin, as MF).
"""
import multiprocessing

import numpy as np
import torch

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils import get_rng
from cornac.utils.init_utils import uniform, zeros

from . import engine
from ._scoring import DeviceScoringMixin
from .recom_bpr import _copy_back

DTYPE = np.float32


class NMF(DeviceScoringMixin, Recommender, ANNMixin):
    """Non-negative Matrix Factorization (Lee and Seung, NIPS 2001), trained on the GPU.

    Parameters are the reference's: name="NMF", k=15, max_iter=50, learning_rate=0.005, lambda_reg=0.0 (when > 0 it
    replaces lambda_u, lambda_v, lambda_bu and lambda_bi), lambda_u=0.06, lambda_v=0.06, lambda_bu=0.02, lambda_bi=0.02,
    use_bias=False, num_threads=0 (kept for compatibility: the fit runs on the GPU), trainable=True, verbose=False,
    init_params=None ({'U', 'V', 'Bu', 'Bi', 'mu'}; f32 arrays are trained in place), seed=None (initial factors only;
    the fit itself is deterministic).

    With verbose=True a progress bar shows each epoch's loss.  That loss is summed in f64 on the device, so its last
    digits may differ from the reference's f32 figure; the trained parameters do not.

    With use_bias=True the reference's score(u) and rank() raise a ValueError (an f64 score row meets its f32 dot
    routine).  Here they rank by the f32 row (global_mean + i_biases) + u_biases[u] + U[u].V, as MF does.
    """

    def __init__(self, name="NMF", k=15, max_iter=50, learning_rate=0.005, lambda_reg=0.0, lambda_u=0.06, lambda_v=0.06,
                 lambda_bu=0.02, lambda_bi=0.02, use_bias=False, num_threads=0, trainable=True, verbose=False,
                 init_params=None, seed=None):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.lambda_reg = lambda_reg
        self.lambda_u = lambda_u
        self.lambda_v = lambda_v
        self.lambda_bu = lambda_bu
        self.lambda_bi = lambda_bi
        self.use_bias = use_bias
        self.seed = seed

        if self.lambda_reg > 0:                                 # recom_nmf.pyx:113-117
            self.lambda_u = self.lambda_reg
            self.lambda_v = self.lambda_reg
            self.lambda_bu = self.lambda_reg
            self.lambda_bi = self.lambda_reg

        if seed is not None:                                    # :119-124
            self.num_threads = 1
        elif num_threads > 0 and num_threads < multiprocessing.cpu_count():
            self.num_threads = num_threads
        else:
            self.num_threads = multiprocessing.cpu_count()

        self.init_params = {} if init_params is None else init_params
        self.u_factors = self.init_params.get("U", None)
        self.i_factors = self.init_params.get("V", None)
        self.u_biases = self.init_params.get("Bu", None)
        self.i_biases = self.init_params.get("Bi", None)
        self.global_mean = self.init_params.get("mu", None)
        self._b200_register_ignored()

    # reference: recom_nmf.pyx:134-145
    def _init(self):
        rng = get_rng(self.seed)
        n_users, n_items = self.num_users, self.num_items
        if self.u_factors is None:
            self.u_factors = uniform((n_users, self.k), random_state=rng)
        if self.i_factors is None:
            self.i_factors = uniform((n_items, self.k), random_state=rng)
        self.u_biases = zeros(n_users) if self.u_biases is None else self.u_biases
        self.i_biases = zeros(n_items) if self.i_biases is None else self.i_biases
        self.global_mean = self.global_mean if self.use_bias else 0.0

    # reference: recom_nmf.pyx:147-180
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._init()
        self._b200_invalidate()
        if self.trainable:
            X = train_set.matrix
            self._fit_b200(X.indptr, X.indices, X.data.astype(np.float32))
        return self

    def _check_params(self):
        """The reference's `floating[:, :]` / `floating[:]` buffers take only f32 here (the ratings fix the type)."""
        shapes = (("U", self.u_factors, (self.num_users, self.k)), ("V", self.i_factors, (self.num_items, self.k)),
                  ("Bu", self.u_biases, (self.num_users,)), ("Bi", self.i_biases, (self.num_items,)))
        for name, x, shape in shapes:
            x = np.asarray(x)
            if x.dtype != DTYPE:
                got = "double" if x.dtype == np.float64 else str(x.dtype)
                raise ValueError("Buffer dtype mismatch, expected 'float' but got '%s'" % got)
            if x.shape[0] < shape[0] or x.shape[1:] != shape[1:]:
                raise ValueError("%s must have shape %s, got %s" % (name, shape, x.shape))

    def _fit_b200(self, indptr, indices, data):
        from tqdm.auto import trange
        self._check_params()
        engine.require_cuda()
        n_users, n_items, k = self.num_users, self.num_items, self.k
        nd = engine.NmfData(indptr, indices, data, n_items, self.use_bias)
        # rows beyond the model's users / items (a larger init_params array) are not touched, as in the reference
        dev = [engine.to_device(np.ascontiguousarray(np.asarray(x)[:n]), torch.float32)
               for x, n in ((self.u_factors, n_users), (self.i_factors, n_items), (self.u_biases, n_users),
                            (self.i_biases, n_items))]
        U, V, Bu, Bi = dev
        hyper = dict(mu=float(self.global_mean), learning_rate=self.learning_rate, lambda_u=self.lambda_u,
                     lambda_v=self.lambda_v, lambda_bu=self.lambda_bu, lambda_bi=self.lambda_bi)
        work = torch.empty_like(U)
        if self.verbose:
            progress = trange(self.max_iter, disable=False)
            loss = torch.zeros(1, dtype=torch.float64, device="cuda")
            for _ in progress:
                loss.zero_()
                engine.nmf_fit(nd, U, V, Bu, Bi, 1, loss=loss, workspace=work, **hyper)
                progress.set_postfix({"loss": "%.2f" % loss.item()})
            progress.close()
        else:
            engine.nmf_fit(nd, U, V, Bu, Bi, self.max_iter, workspace=work, **hyper)
        self.u_factors = self._copy_rows_back(self.u_factors, U)
        self.i_factors = self._copy_rows_back(self.i_factors, V)
        self.u_biases = self._copy_rows_back(self.u_biases, Bu)
        self.i_biases = self._copy_rows_back(self.i_biases, Bi)
        if self.verbose:
            print("Optimization finished!")

    @staticmethod
    def _copy_rows_back(host, dev):
        """The trained rows into the caller's array (an init_params array is trained in place)."""
        n = int(dev.shape[0])
        if isinstance(host, np.ndarray) and host.shape[0] > n and host.dtype == DTYPE and host.flags.writeable:
            host[:n] = dev.cpu().numpy()
            return host
        return _copy_back(host, dev)

    def _b200_host_params(self):
        item_base = (self.global_mean + self.i_biases).astype(DTYPE)        # recom_nmf.pyx:288
        return (self.u_factors[: self.num_users], self.i_factors[: self.num_items], item_base[: self.num_items],
                np.asarray(self.u_biases[: self.num_users], dtype=DTYPE), self.num_items)

    # reference: recom_nmf.pyx:270-303
    def score(self, user_idx, item_idx=None):
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            return self._b200_row(user_idx) if self.knows_user(user_idx) else self.global_mean + self.i_biases
        item_score = self.global_mean + self.i_biases[item_idx]
        if self.knows_user(user_idx):
            item_score += self.u_biases[user_idx]
            item_score += self.u_factors[user_idx].dot(self.i_factors[item_idx])
        return item_score

    def _b200_rank_row(self, user_idx):
        return self._scores_dev([user_idx])[0] if self.knows_user(user_idx) else self.global_mean + self.i_biases

    # ---- ANNMixin (recom_nmf.pyx:305-350) ------------------------------------------------------------------------------
    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        user_vectors = self.u_factors
        if self.use_bias:
            user_vectors = np.concatenate((user_vectors, np.ones([user_vectors.shape[0], 1])), axis=1)
        return user_vectors

    def get_item_vectors(self):
        item_vectors = self.i_factors
        if self.use_bias:
            item_vectors = np.concatenate((item_vectors, self.i_biases.reshape((-1, 1))), axis=1)
        return item_vectors
