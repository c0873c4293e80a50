"""MCF (matrix co-factorisation of ratings and an item-affinity graph) on an H100: drop-in for cornac.models.MCF.

Same constructor arguments, defaults, attributes, errors and fit()/score()/rank() behaviour as the reference class
(cornac/models/mcf/recom_mcf.py), except that a train set without an `item_graph` modality raises a ValueError naming it
(the reference fails with an AttributeError), and so does a graph with no edge between training items (the reference's
min() of an empty sequence).  The graph triplets and the rating and edge scaling are prepared on the host as the
reference prepares them; the serial RMSProp loop of mcf.pyx runs as b200_cofactor_fit (see _cofactor.py), so U, V and Z
are bit-identical to the reference's.  The full score rows of score(u) / rank() are f64 device dots; rank() orders them
as the reference's Recommender.rank does, and rank_batch / recommend_batch rank them on the device.
"""
import numpy as np

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils.common import scale, sigmoid

from ._cofactor import CofactorMixin
from ._scoring import F64DotScoringMixin


class MCF(CofactorMixin, F64DotScoringMixin, Recommender, ANNMixin):
    """Matrix co-factorisation (Park et al., WWW 2017), trained on the GPU.

    Parameters are the reference's: k=5, max_iter=100, learning_rate=0.001, gamma=0.9, lamda=0.001, name="MCF",
    trainable=True, verbose=False, init_params=None ({'U', 'V', 'Z'}: f64 arrays, trained in place), seed=None (initial
    factors only; the fit itself is deterministic).  The train set needs an `item_graph`.
    """

    _COFACTOR = "mcf"

    def __init__(self, k=5, max_iter=100, learning_rate=0.001, gamma=0.9, lamda=0.001, name="MCF", trainable=True,
                 verbose=False, init_params=None, seed=None):
        Recommender.__init__(self, name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.gamma = gamma
        self.lamda = lamda
        self.seed = seed

        self.ll = np.full(max_iter, 0)
        self.eps = 0.000000001

        self.init_params = {} if init_params is None else init_params
        self.U = self.init_params.get("U", None)
        self.V = self.init_params.get("V", None)
        self.Z = self.init_params.get("Z", None)
        self._b200_register_ignored()

    # reference: recom_mcf.py:110-191
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._b200_invalidate()
        if self.trainable:
            if getattr(train_set, "item_graph", None) is None:
                raise ValueError("MCF requires a train set with an item_graph modality (cornac.data.GraphModality)")
            rat_uid, rat_iid, rat_val = train_set.uir_tuple
            train_items = set(rat_iid)
            net_iid, net_jid, net_val = train_set.item_graph.get_train_triplet(train_items, train_items)
            if len(net_val) == 0:
                raise ValueError("MCF requires at least one item_graph edge between training items")
            if [self.min_rating, self.max_rating] != [0, 1]:
                if self.min_rating == self.max_rating:
                    rat_val = scale(rat_val, 0.0, 1.0, 0.0, self.max_rating)
                else:
                    rat_val = scale(rat_val, 0.0, 1.0, self.min_rating, self.max_rating)
            lo, hi = np.min(net_val), np.max(net_val)
            if [lo, hi] != [0, 1]:
                if lo == hi:
                    net_val = scale(net_val, 0.0, 1.0, 0.0, hi)
                else:
                    net_val = scale(net_val, 0.0, 1.0, lo, hi)
            if self.verbose:
                print("Learning...")
            self._fit_cofactor(np.array(net_iid, dtype="int32"), np.array(net_jid, dtype="int32"),
                               np.array(net_val, dtype="float32"), np.array(rat_uid, dtype="int32"),
                               np.array(rat_iid, dtype="int32"), np.array(rat_val, dtype="float32"), 0.0, self.lamda)
            if self.verbose:
                print("Learning completed")
        elif self.verbose:
            print("%s is trained already (trainable = False)" % self.name)
        return self

    # reference: recom_mcf.py:193-229
    def score(self, user_idx, item_idx=None):
        if item_idx is None:
            if not self.knows_user(user_idx):
                raise ScoreException("Can't make score prediction for (user_id=%d)" % user_idx)
            return self._b200_row(user_idx)
        if not (self.knows_user(user_idx) and self.knows_item(item_idx)):
            raise ScoreException("Can't make score prediction for (user_id=%d, item_id=%d)" % (user_idx, item_idx))
        # one item: the reference's host expression (a cached row is never used here: it holds the raw dot)
        user_pred = self.V[item_idx, :].dot(self.U[user_idx, :])
        user_pred = sigmoid(user_pred)
        if self.min_rating == self.max_rating:
            user_pred = scale(user_pred, 0.0, self.max_rating, 0.0, 1.0)
        else:
            user_pred = scale(user_pred, self.min_rating, self.max_rating, 0.0, 1.0)
        return user_pred

    # ---- ANNMixin (recom_mcf.py:231-259) -----------------------------------------------------------------------------
    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return self.U

    def get_item_vectors(self):
        return self.V
