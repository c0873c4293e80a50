"""SoRec (social recommendation by co-factorising ratings and a trust graph) on an H100: drop-in for cornac.models.SoRec.

Same constructor arguments, defaults, attributes, errors and fit()/score()/rank() behaviour as the reference class
(cornac/models/sorec/recom_sorec.py), except that a train set without a `user_graph` modality raises a ValueError naming
it (the reference fails with an AttributeError).  The graph triplets, the link weights and the rating scaling are
prepared on the host as the reference prepares them; the serial RMSProp loop of sorec.pyx runs as b200_cofactor_fit
(see _cofactor.py), so U, V and Z are bit-identical to the reference's.  The full score rows of score(u) / rank() are
f64 device dots (b200_score_batch_f64); rank() orders them as the reference's Recommender.rank does, and rank_batch /
recommend_batch rank them on the device (b200_topk_rows_f64).
"""
import numpy as np

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils.common import scale, sigmoid

from ._cofactor import CofactorMixin
from ._scoring import F64DotScoringMixin


def link_weights(net_uid, net_jid, net_val):
    """recom_sorec.py:157-167, vectorised: sqrt(j_in / (j_in + u_out)) * val per edge (u, j), with the in- and
    out-degrees counted over the same training edges.  The same f64 operations per edge, so the same bits."""
    net_uid, net_jid = np.asarray(net_uid, dtype=np.int64), np.asarray(net_jid, dtype=np.int64)
    n = int(max(net_uid.max(initial=-1), net_jid.max(initial=-1))) + 1
    u_out = np.bincount(net_uid, minlength=n)[net_uid]
    j_in = np.bincount(net_jid, minlength=n)[net_jid]
    return np.sqrt(j_in / (j_in + u_out)) * np.asarray(net_val, dtype=np.float64)


class SoRec(CofactorMixin, F64DotScoringMixin, Recommender, ANNMixin):
    """Social recommendation using probabilistic matrix factorisation (Ma et al., CIKM 2008), trained on the GPU.

    Parameters are the reference's: name="SoRec", k=5, max_iter=100, learning_rate=0.001, lambda_c=10, lambda_reg=0.001,
    gamma=0.9, weight_link=True, trainable=True, verbose=False, init_params=None ({'U', 'V', 'Z'}: f64 arrays, trained in
    place), seed=None (initial factors only; the fit itself is deterministic).  The train set needs a `user_graph`.
    """

    _COFACTOR = "sorec"

    def __init__(self, name="SoRec", k=5, max_iter=100, learning_rate=0.001, lambda_c=10, lambda_reg=0.001, gamma=0.9,
                 weight_link=True, trainable=True, verbose=False, init_params=None, seed=None):
        Recommender.__init__(self, name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.lambda_c = lambda_c
        self.lambda_reg = lambda_reg
        self.gamma = gamma
        self.weight_link = weight_link

        self.ll = np.full(max_iter, 0)
        self.eps = 0.000000001
        self.seed = seed

        self.init_params = {} if init_params is None else init_params
        self.U = self.init_params.get("U", None)
        self.V = self.init_params.get("V", None)
        self.Z = self.init_params.get("Z", None)
        for key in ("U", "V", "Z"):                        # recom_sorec.py:118-125
            x = getattr(self, key)
            if x is not None and x.shape[1] != self.k:
                raise ValueError("initial parameters %s dimension error" % key)
        self._b200_register_ignored()

    # reference: recom_sorec.py:127-218
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._b200_invalidate()
        if self.trainable:
            if getattr(train_set, "user_graph", None) is None:
                raise ValueError("SoRec requires a train set with a user_graph modality (cornac.data.GraphModality)")
            rat_uid, rat_iid, rat_val = train_set.uir_tuple
            train_users = set(rat_uid)
            net_uid, net_jid, net_val = train_set.user_graph.get_train_triplet(train_users, train_users)
            if self.weight_link:
                net_val = link_weights(net_uid, net_jid, net_val)
            if [self.min_rating, self.max_rating] != [0, 1]:
                if self.min_rating == self.max_rating:
                    rat_val = scale(rat_val, 0.0, 1.0, 0.0, self.max_rating)
                else:
                    rat_val = scale(rat_val, 0.0, 1.0, self.min_rating, self.max_rating)
            if self.verbose:
                print("Learning...")
            self._fit_cofactor(np.array(net_uid, dtype="int32"), np.array(net_jid, dtype="int32"),
                               np.array(net_val, dtype="float32"), np.array(rat_uid, dtype="int32"),
                               np.array(rat_iid, dtype="int32"), np.array(rat_val, dtype="float32"), self.lambda_c,
                               self.lambda_reg)
            if self.verbose:
                print("Learning completed")
        elif self.verbose:
            print("%s is trained already (trainable = False)" % self.name)
        return self

    # reference: recom_sorec.py:220-249
    def score(self, user_idx, item_idx=None):
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            return self._b200_row(user_idx)
        # one item: the reference's host expression (a cached row is never used here: it holds the raw dot)
        user_pred = self.V[item_idx, :].dot(self.U[user_idx, :])
        user_pred = sigmoid(user_pred)
        if self.min_rating == self.max_rating:
            user_pred = scale(user_pred, 0.0, self.max_rating, 0.0, 1.0)
        else:
            user_pred = scale(user_pred, self.min_rating, self.max_rating, 0.0, 1.0)
        return user_pred

    # ---- ANNMixin (recom_sorec.py:251-279) ---------------------------------------------------------------------------
    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return self.U

    def get_item_vectors(self):
        return self.V
