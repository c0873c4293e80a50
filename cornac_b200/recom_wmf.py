"""Weighted matrix factorisation on an H100: drop-in for cornac.models.WMF.

Same constructor arguments, attributes (`U`, `V`) and fit()/score()/rank() behaviour as the reference class
(cornac/models/wmf/recom_wmf.py:28-251).  The reference trains through a TensorFlow-1 graph
(cornac/models/wmf/wmf.py:34-55); here each `sess.run([opt, loss])` over one item mini-batch is one b200_wmf_step
(csrc/wmf.cu): weighted residual, clipped gradients, dense Adam on U, TF-1 (non-lazy) sparse Adam on V.
The mini-batch schedule is the reference's own: `train_set.item_iter(batch_size, shuffle=True)`
(recom_wmf.py:184-185), so the same Dataset seed visits the items in the same order.
TensorFlow is not installed in this environment, so the reference's WMF cannot be run here: the tests compare against
a CPU restatement of the graph only ("parity unpinned" against a real TF run) -- see DESIGN.md.
"""
import numpy as np

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils import get_rng
from cornac.utils.init_utils import xavier_uniform

from . import engine
from ._scoring import DeviceScoringMixin

DTYPE = np.float32


class WMF(DeviceScoringMixin, Recommender, ANNMixin):
    def __init__(self, name="WMF", k=200, lambda_u=0.01, lambda_v=0.01, a=1, b=0.01, learning_rate=0.001, batch_size=128,
                 max_iter=100, trainable=True, verbose=True, init_params=None, seed=None):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.lambda_u = lambda_u
        self.lambda_v = lambda_v
        self.a = a
        self.b = b
        self.learning_rate = learning_rate
        self.name = name
        self.init_params = init_params
        self.max_iter = max_iter
        self.batch_size = batch_size
        self.verbose = verbose
        self.seed = seed
        self.init_params = {} if init_params is None else init_params
        self.U = self.init_params.get("U", None)
        self.V = self.init_params.get("V", None)
        self._b200_register_ignored()

    # reference: recom_wmf.py:121-126
    def _init(self):
        rng = get_rng(self.seed)
        if self.U is None:
            self.U = xavier_uniform((self.num_users, self.k), rng)
        if self.V is None:
            self.V = xavier_uniform((self.num_items, self.k), rng)

    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._init()
        self._b200_invalidate()
        if self.trainable:
            self._fit_cf(train_set)
        return self

    # reference: recom_wmf.py:152-212
    def _fit_cf(self, train_set):
        np.random.seed(self.seed)
        trainer = engine.WmfTrainer(train_set.csc_matrix, np.asarray(self.U, dtype=DTYPE), np.asarray(self.V, dtype=DTYPE),
                                    self.a, self.b, self.lambda_u, self.lambda_v, self.learning_rate)
        self.loss_history = []
        for epoch in range(self.max_iter):
            sum_loss, count = 0.0, 0
            for i, batch_ids in enumerate(train_set.item_iter(self.batch_size, shuffle=True)):
                want = self.verbose and (i % 10 == 0)          # the reference reads the loss of every step (a sync each);
                loss = trainer.step(batch_ids, want_loss=want)  # here only where it is displayed
                if want:
                    sum_loss += loss
                    count += len(batch_ids)
            if self.verbose and count:
                self.loss_history.append(sum_loss / count)
                print("epoch %d: loss per item (sampled) %.4f" % (epoch, sum_loss / count))
        self.U, self.V = trainer.download()
        self._b200_adopt_device(trainer.U, trainer.V, None, None, self.num_items)
        if self.verbose:
            print("Learning completed!")

    def _b200_host_params(self):
        return np.asarray(self.U, dtype=DTYPE), np.asarray(self.V, dtype=DTYPE), None, None, self.num_items

    # reference: recom_wmf.py:214-240
    def score(self, user_idx, item_idx=None):
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            return self._b200_row(user_idx)
        return self.V[item_idx, :].dot(self.U[user_idx, :])

    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return self.U

    def get_item_vectors(self):
        return self.V
