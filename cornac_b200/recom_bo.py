"""Bias-only rating model on an H100: drop-in for cornac.models.BaselineOnly.

Same constructor arguments and behaviour as the reference class
(cornac/models/baseline_only/recom_bo.pyx:34-214).  Its `_fit_sgd` (:101-140) is the MF loop of
backend_cpu.fit_sgd without the factor rows, so one epoch is b200_mf_epoch with k = 0:
  * seed given -> ratings applied in stored order (ordered replay kernel) = the single-thread reference;
  * seed=None  -> Hogwild over the whole GPU.
SURVEY.md section 8, row (f)3.
"""
import numpy as np
import torch

from cornac.models.recommender import Recommender
from cornac.utils.init_utils import zeros

from . import engine
from ._scoring import DeviceScoringMixin
from .recom_bpr import _copy_back

DTYPE = np.float32


class BaselineOnly(DeviceScoringMixin, Recommender):
    # score() is three host additions (recom_bo.pyx:183-197, in the arrays' own precision): nothing to precompute in
    # transform(); a cache of device-computed float32 rows would differ from it in the last bit
    _B200_EVAL_CACHE_BYTES = 0

    def __init__(self, name="BaselineOnly", max_iter=20, learning_rate=0.01, lambda_reg=0.02, early_stop=False,
                 num_threads=0, trainable=True, verbose=False, init_params=None, seed=None, mode="auto",
                 atomic_updates=True):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.lambda_reg = lambda_reg
        self.early_stop = early_stop
        self.seed = seed
        self.num_threads = num_threads
        if mode not in ("auto", "replay", "hogwild"):
            raise ValueError("mode must be 'auto', 'replay' or 'hogwild'")
        self.mode = mode
        self.atomic_updates = atomic_updates
        self.init_params = {} if init_params is None else init_params
        self.u_biases = self.init_params.get("Bu", None)
        self.i_biases = self.init_params.get("Bi", None)
        self.global_mean = 0.0
        self._b200_register_ignored()

    # reference: recom_bo.pyx:75-80
    def _init(self):
        self.u_biases = zeros(self.num_users) if self.u_biases is None else self.u_biases
        self.i_biases = zeros(self.num_items) if self.i_biases is None else self.i_biases

    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._b200_invalidate()
        if self.trainable:
            self._init()
            self._fit_b200(train_set)
        return self

    def _fit_b200(self, train_set):
        engine.require_cuda()
        rid, cid, val = train_set.uir_tuple
        if len(val) == 0 or self.max_iter <= 0:
            return
        d_rid = engine.to_device(np.asarray(rid), torch.int32)
        d_cid = engine.to_device(np.asarray(cid), torch.int32)
        d_val = engine.to_device(np.asarray(val).astype(DTYPE), torch.float32)
        Bu = engine.to_device(np.ascontiguousarray(self.u_biases, dtype=DTYPE))
        Bi = engine.to_device(np.ascontiguousarray(self.i_biases, dtype=DTYPE))
        loss_dev = torch.zeros(1, dtype=torch.float32, device="cuda")
        ordered = (self.seed is not None) if self.mode == "auto" else (self.mode == "replay")
        lr, reg = float(np.float32(self.learning_rate)), float(np.float32(self.lambda_reg))
        mu = float(np.float32(self.global_mean))                # `floating mu = self.global_mean`, recom_bo.pyx:113
        loss = np.float32(0)
        self.loss_history = []
        for epoch in range(self.max_iter):                     # recom_bo.pyx:118-138
            last_loss = loss
            engine.mf_epoch(d_rid, d_cid, d_val, None, None, Bu, Bi, lr, reg, mu, True, loss_dev, ordered=ordered,
                            atomic=self.atomic_updates)
            if self.early_stop or self.verbose:
                loss = np.float32(0.5) * np.float32(loss_dev.item())
                self.loss_history.append(float(loss))
                if self.early_stop and abs(np.float32(loss - last_loss)) < 1e-5:
                    if self.verbose:
                        print("Early stopping, delta_loss = %.4f" % (loss - last_loss))
                    break
        self.u_biases = _copy_back(self.u_biases, Bu)
        self.i_biases = _copy_back(self.i_biases, Bi)
        if self.verbose:
            print("Optimization finished!")

    # reference: recom_bo.pyx:183-211 (including its single-item branch, which adds the user bias when the
    # ITEM is known -- kept as is)
    def score(self, user_idx, item_idx=None):
        if item_idx is None:
            known_item_scores = np.add(self.i_biases, self.global_mean)
            if self.knows_user(user_idx):
                known_item_scores = np.add(known_item_scores, self.u_biases[user_idx])
            return known_item_scores
        item_score = self.global_mean
        if self.knows_item(item_idx):
            item_score += self.u_biases[user_idx]
        if self.knows_item(item_idx):
            item_score += self.i_biases[item_idx]
        return item_score

    # Every user's ranking is the ranking of (global_mean + Bi): rank through the shared device path with a
    # zero-width factor pair replaced by one zero column (the dot contributes exactly +0).
    def _b200_host_params(self):
        item_base = np.add(self.i_biases, self.global_mean).astype(DTYPE)
        zu = np.zeros((self.num_users, 1), dtype=DTYPE)
        zv = np.zeros((self.num_items, 1), dtype=DTYPE)
        return zu, zv, item_base, np.asarray(self.u_biases, dtype=DTYPE), self.num_items

    # rank() orders the host score(u) row: the device row's __fadd_rn sums round differently from the host's f64 sum
    def _b200_rank_row(self, user_idx):
        return self.score(user_idx)
