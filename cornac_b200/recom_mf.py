"""Biased matrix factorisation on an H100: drop-in for cornac.models.MF (backend "cpu").

Same constructor arguments and behaviour as the reference class
(cornac/models/mf/recom_mf.py:31-326); `backend_cpu.fit_sgd`
(cornac/models/mf/backend_cpu.pyx:35-97) is replaced by b200_mf_epoch.

  * seed given -> the ratings are applied in stored order with the same result as the
    reference's single-thread loop (ordered replay kernel);
  * seed=None  -> Hogwild over the whole GPU.
`backend` accepts "cpu" (the reference's default name, kept so existing scripts work) and
"b200"; both run on the GPU -- there is no CPU path here.
"""
import numpy as np
import torch

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils import get_rng
from cornac.utils.init_utils import normal, zeros

from . import engine
from ._scoring import DeviceScoringMixin
from .recom_bpr import _copy_back, check_factor_width, replay_hint

DTYPE = np.float32


class MF(DeviceScoringMixin, Recommender, ANNMixin):
    def __init__(self, name="MF", k=10, backend="cpu", optimizer="sgd", max_iter=20, learning_rate=0.01,
                 batch_size=256, lambda_reg=0.02, dropout=0.0, use_bias=True, early_stop=False, num_threads=0,
                 trainable=True, verbose=False, init_params=None, seed=None, mode="auto", atomic_updates=True):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.k = check_factor_width(k)
        self.backend = backend
        self.optimizer = optimizer
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.batch_size = batch_size
        self.lambda_reg = lambda_reg
        self.dropout = dropout
        self.use_bias = use_bias
        self.early_stop = early_stop
        self.seed = seed
        self.num_threads = num_threads
        if mode not in ("auto", "replay", "hogwild"):
            raise ValueError("mode must be 'auto', 'replay' or 'hogwild'")
        self.mode = mode
        self.atomic_updates = atomic_updates

        self.init_params = {} if init_params is None else init_params
        self.u_factors = self.init_params.get("U", None)
        self.i_factors = self.init_params.get("V", None)
        self.u_biases = self.init_params.get("Bu", None)
        self.i_biases = self.init_params.get("Bi", None)
        self._b200_register_ignored()

    # reference: recom_mf.py:138-156
    def _init(self):
        rng = get_rng(self.seed)
        if self.u_factors is None:
            self.u_factors = normal([self.num_users, self.k], std=0.01, random_state=rng, dtype=DTYPE)
        if self.i_factors is None:
            self.i_factors = normal([self.num_items, self.k], std=0.01, random_state=rng, dtype=DTYPE)
        self.u_biases = zeros(self.num_users, dtype=DTYPE) if self.u_biases is None else self.u_biases
        self.i_biases = zeros(self.num_items, dtype=DTYPE) if self.i_biases is None else self.i_biases
        self.global_mean = np.dtype(DTYPE).type(self.global_mean if self.use_bias else 0.0)

    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._init()
        self._b200_invalidate()
        if self.trainable:
            if self.backend not in ("cpu", "b200"):
                raise ValueError(f"{self.backend} is not supported")
            self._fit_b200(train_set)
        return self

    def _fit_b200(self, train_set):
        engine.require_cuda()
        rid, cid, val = train_set.uir_tuple
        n = len(val)
        if n == 0 or self.max_iter <= 0:
            return
        d_rid = engine.to_device(np.asarray(rid), torch.int32)     # ids narrowed to int32 on the device
        d_cid = engine.to_device(np.asarray(cid), torch.int32)
        d_val = engine.to_device(np.asarray(val).astype(DTYPE), torch.float32)
        U = engine.to_device(np.ascontiguousarray(self.u_factors, dtype=DTYPE))
        V = engine.to_device(np.ascontiguousarray(self.i_factors, dtype=DTYPE))
        Bu = engine.to_device(np.ascontiguousarray(self.u_biases, dtype=DTYPE))
        Bi = engine.to_device(np.ascontiguousarray(self.i_biases, dtype=DTYPE))
        loss_dev = torch.zeros(1, dtype=torch.float32, device="cuda")
        ordered = (self.seed is not None) if self.mode == "auto" else (self.mode == "replay")
        if ordered and self.mode == "auto":
            replay_hint(n, self.name)
        lr, reg = float(np.float32(self.learning_rate)), float(np.float32(self.lambda_reg))
        loss = np.float32(0)
        self.loss_history = []
        for epoch in range(self.max_iter):                     # backend_cpu.pyx:58-93
            last_loss = loss
            engine.mf_epoch(d_rid, d_cid, d_val, U, V, Bu, Bi, lr, reg, float(self.global_mean), self.use_bias,
                            loss_dev, ordered=ordered, atomic=self.atomic_updates)
            if self.early_stop or self.verbose:
                loss = np.float32(0.5) * np.float32(loss_dev.item())
                self.loss_history.append(float(loss))
                if self.verbose:
                    print("epoch %d: loss %.2f" % (epoch, loss))
                if self.early_stop and abs(np.float32(loss - last_loss)) < 1e-5:
                    if self.verbose:
                        print("Early stopping, delta_loss = %.4f" % (loss - last_loss))
                    break
        self.u_factors = _copy_back(self.u_factors, U)
        self.i_factors = _copy_back(self.i_factors, V)
        if self.use_bias:
            self.u_biases = _copy_back(self.u_biases, Bu)
            self.i_biases = _copy_back(self.i_biases, Bi)
        if self.verbose:
            print("Optimization finished!")

    def _b200_host_params(self):
        item_base = (self.global_mean + self.i_biases).astype(DTYPE)       # recom_mf.py:273
        return self.u_factors, self.i_factors, item_base, self.u_biases, self.num_items

    # reference: recom_mf.py:254-286
    def score(self, user_idx, item_idx=None):
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            if self.knows_user(user_idx):
                cached = self._b200_cached_scores(user_idx)
                return cached.copy() if cached is not None else self._b200_scores_dev([user_idx])[0].cpu().numpy()
            return self.global_mean + self.i_biases
        item_score = self.global_mean + self.i_biases[item_idx]
        if self.knows_user(user_idx):
            item_score += self.u_biases[user_idx]
            item_score += self.u_factors[user_idx].dot(self.i_factors[item_idx])
        return item_score

    # reference: recommender.py:476-530
    def rank(self, user_idx, item_indices=None, k=-1, **kwargs):
        hit = self._b200_cached_rank(user_idx, item_indices, k) if self.knows_user(user_idx) else None
        if hit is not None:
            return hit
        if not self.knows_user(user_idx):
            known = torch.from_numpy(np.asarray(self.global_mean + self.i_biases, dtype=DTYPE)).cuda()[None, :]
        else:
            known = self._b200_scores_dev([user_idx])       # [1, num_items]
        if known.shape[1] != self.total_items:               # unknown items get the MIN score (:507-511)
            allsc = torch.full((1, self.total_items), float(known.min().item()), dtype=torch.float32, device="cuda")
            allsc[:, : self.num_items] = known
            known = allsc
        return self._b200_rank(known, item_indices, k)

    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return np.concatenate((self.u_factors, np.ones([self.u_factors.shape[0], 1])), axis=1)

    def get_item_vectors(self):
        return np.concatenate((self.i_factors, self.i_biases.reshape((-1, 1))), axis=1)
