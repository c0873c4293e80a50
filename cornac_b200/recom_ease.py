"""EASE^R on an H100: drop-in for cornac.models.EASE.

Same constructor arguments, defaults, attributes and fit()/score()/rank() behaviour as the reference class
(cornac/models/ease/recom_ease.py:8-156).  fit() computes the Gram matrix (b200_ease_gram, bit-identical to scipy's), its
inverse on the FP64 tensor cores (b200_spd_inverse, Cholesky instead of the reference's LU: equal to it within rounding)
and the weights (b200_ease_weights) on the device; `B` is then copied to the host.  The full score rows of score(u) /
rank() are f64 device rows in scipy's order (b200_ease_score) ranked on the device (b200_topk_rows_f64).
"""
import numpy as np

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender

from . import engine
from ._scoring import F64RankingMixin


class EASE(F64RankingMixin, Recommender, ANNMixin):
    """Embarrassingly Shallow Autoencoders for Sparse Data (Steck, WWW 2019), fitted on the GPU.

    Parameters are the reference's: name="EASEᴿ", lamb=500 (L2 regularisation added to the Gram matrix's diagonal),
    posB=True (negative weights set to 0), trainable=True, verbose=True, seed=None, B=None, U=None.  Like the reference,
    fit() always refits, whatever `trainable` and a given `B` say.  When the Gram matrix is not positive definite (possible
    only for lamb <= 0) fit() raises numpy.linalg.LinAlgError, where the reference's LU inverse may still return a result.
    """

    def __init__(self, name="EASEᴿ", lamb=500, posB=True, trainable=True, verbose=True, seed=None, B=None, U=None):
        Recommender.__init__(self, name=name, trainable=trainable, verbose=verbose)
        self.lamb = lamb
        self.posB = posB
        self.verbose = verbose
        self.seed = seed
        self.B = B
        self.U = U
        self._b200_register_f64()

    # reference: recom_ease.py:57-97
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._b200_dev = None
        self._b200_eval_cache = None
        self.U = train_set.matrix
        B = engine.ease_fit(self.U, self.lamb, self.posB)
        self.B = B.cpu().numpy()
        self._b200_dev = dict(B=B, X=engine.EaseRatings(self.U))
        return self

    # ---- device scores ---------------------------------------------------------------------------------------------
    def _b200_device(self):
        if getattr(self, "_b200_dev", None) is None:          # None after fit(); absent after load()
            engine.require_cuda()
            self._b200_dev = dict(B=engine.to_device(np.ascontiguousarray(self.B, dtype=np.float64)),
                                  X=engine.EaseRatings(self.U))
        return self._b200_dev

    def _scores_dev(self, user_indices):
        """[n_q, num_items] f64 device scores X[u, :] . B of known users."""
        d = self._b200_device()
        user_indices = np.asarray(user_indices, dtype=np.int64)
        if user_indices.size and (int(user_indices.min()) < 0 or int(user_indices.max()) >= d["X"].n_rows):
            raise IndexError("user index out of bounds for the %d users of the model" % d["X"].n_rows)
        return engine.ease_score(d["B"], user_indices, d["X"])

    # reference: recom_ease.py:99-126
    def score(self, user_idx, item_idx=None):
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            return self._b200_row(user_idx)[None, :]          # the reference's sparse row . dense: shape (1, n_items)
        return self.U[user_idx, :].dot(self.B[:, item_idx])

    # ---- ANNMixin (recom_ease.py:128-156) ----------------------------------------------------------------------------
    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return self.U

    def get_item_vectors(self):
        return self.B
