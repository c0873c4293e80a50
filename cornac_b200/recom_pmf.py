"""Probabilistic matrix factorisation on an H100: drop-in for cornac.models.PMF.

Same constructor arguments, defaults, attributes, errors and fit()/score()/rank() behaviour as the reference class
(cornac/models/pmf/recom_pmf.py:25-252).  Data preparation and the initial factors are the reference's host numpy; the
serial RMSProp loops of pmf_linear / pmf_non_linear (cornac/models/pmf/cython/pmf.pyx:55-173) run as b200_pmf_fit over a
level schedule of the ratings, with the reference's f64 arithmetic, so U and V are bit-identical to the reference's.
The full score rows of score(u) / rank() are f64 device dots (b200_score_batch_f64) ranked on the device
(b200_topk_rows_f64).
"""
import numpy as np
import torch

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils import get_rng
from cornac.utils.common import scale, sigmoid
from cornac.utils.init_utils import normal

from . import engine
from ._scoring import F64RankingMixin

VARIANTS = ("linear", "non_linear")


class PMF(F64RankingMixin, Recommender, ANNMixin):
    """Probabilistic Matrix Factorization (Mnih and Salakhutdinov, NIPS 2008), trained on the GPU.

    Parameters are the reference's: k=5, max_iter=100, learning_rate=0.001, gamma=0.9, lambda_reg=0.001, name="PMF",
    variant="non_linear" ("linear" or "non_linear"), trainable=True, verbose=False, init_params=None ({'U': ..., 'V': ...},
    f64 arrays, trained in place), seed=None (initial factors only; the fit itself is deterministic).
    """

    _B200_LOSS_BYTES = 256 << 20                # device budget of the per-rating loss terms when verbose

    def __init__(self, k=5, max_iter=100, learning_rate=0.001, gamma=0.9, lambda_reg=0.001, name="PMF",
                 variant="non_linear", trainable=True, verbose=False, init_params=None, seed=None):
        Recommender.__init__(self, name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.max_iter = max_iter
        self.learning_rate = learning_rate
        self.gamma = gamma
        self.lambda_reg = lambda_reg
        self.variant = variant
        self.seed = seed

        self.ll = np.full(max_iter, 0)
        self.eps = 0.000000001

        self.init_params = {} if init_params is None else init_params
        self.U = self.init_params.get("U", None)
        self.V = self.init_params.get("V", None)
        self._b200_register_f64()

    # reference: recom_pmf.py:108-189
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set)
        self._b200_dev = None
        self._b200_eval_cache = None
        if self.trainable:
            uid, iid, rat = train_set.uir_tuple
            rat = np.array(rat, dtype="float32")
            if self.variant == "non_linear":
                if [self.min_rating, self.max_rating] != [0, 1]:
                    rat = scale(rat, 0.0, 1.0, self.min_rating, self.max_rating)
            uid = np.array(uid, dtype="int32")
            iid = np.array(iid, dtype="int32")
            if self.verbose:
                print("Learning...")
            if self.variant not in VARIANTS:
                raise ValueError('variant must be one of {"linear","non_linear"}')
            self._fit_b200(uid, iid, rat.astype(np.float32))
            if self.verbose:
                print("Learning completed")
        elif self.verbose:
            print("%s is trained already (trainable = False)" % (self.name))
        return self

    def _init_factors(self):
        """pmf.pyx:40-51: U drawn before V from one generator, each only when init_params does not supply it."""
        rng = get_rng(self.seed)
        U = self.U
        if U is None:
            U = normal((self.num_users, self.k), mean=0.0, std=0.001, random_state=rng, dtype=np.double)
        V = self.V
        if V is None:
            V = normal((self.num_items, self.k), mean=0.0, std=0.001, random_state=rng, dtype=np.double)
        for name, x, n in (("U", U, self.num_users), ("V", V, self.num_items)):
            x = np.asarray(x)
            if x.dtype != np.float64:                         # what the reference's double[:, :] memoryview raises
                raise ValueError("Buffer dtype mismatch, expected 'double' but got '%s'" % x.dtype)
            if x.ndim != 2 or x.shape[0] < n or x.shape[1] != self.k:
                raise ValueError("%s must have shape (%d, %d), got %s" % (name, n, self.k, x.shape))
        return U, V

    def _fit_b200(self, uid, iid, rat):
        U, V = self._init_factors()
        engine.require_cuda()
        data = engine.PmfData(uid, iid, rat, self.num_users, self.num_items)
        Ud = engine.to_device(np.ascontiguousarray(U), torch.float64)
        Vd = engine.to_device(np.ascontiguousarray(V), torch.float64)
        cu, cv = torch.zeros_like(Ud), torch.zeros_like(Vd)
        hyper = (float(np.float32(self.lambda_reg)), float(np.float32(self.learning_rate)), float(np.float32(self.gamma)))
        if self.verbose and data.nnz > 0:
            # each rating's loss term lands at its stored index; summing a row in stored order is the reference's sum
            chunk = max(1, self._B200_LOSS_BYTES // (8 * data.nnz))
            for e0 in range(0, self.max_iter, chunk):
                n = min(chunk, self.max_iter - e0)
                terms = torch.empty((n, data.nnz), dtype=torch.float64, device="cuda")
                engine.pmf_fit(data, self.variant, Ud, Vd, cu, cv, n, *hyper, loss=terms)
                loss = np.add.accumulate(terms.cpu().numpy(), axis=1)[:, -1]
                for j in range(n):
                    print("epoch %i, loss: %f" % (e0 + j, loss[j]))
        elif self.verbose:
            for e in range(self.max_iter):
                print("epoch %i, loss: %f" % (e, 0.0))
        else:
            engine.pmf_fit(data, self.variant, Ud, Vd, cu, cv, self.max_iter, *hyper)
        # an f64 init_params array is trained in place, as through the reference's memoryview
        U[...] = Ud.cpu().numpy()
        V[...] = Vd.cpu().numpy()
        self.U, self.V = U, V
        self._b200_dev = dict(U=Ud, V=Vd) if U.shape == (self.num_users, self.k) and V.shape == (self.num_items, self.k) else None

    # ---- device scores ---------------------------------------------------------------------------------------------
    def _b200_device(self):
        if getattr(self, "_b200_dev", None) is None:          # None after fit(); absent after load()
            engine.require_cuda()
            self._b200_dev = dict(U=engine.to_device(np.ascontiguousarray(self.U[: self.num_users]), torch.float64),
                                  V=engine.to_device(np.ascontiguousarray(self.V[: self.num_items]), torch.float64))
        return self._b200_dev

    def _scores_dev(self, user_indices):
        """[n_q, num_items] f64 device scores V.dot(U[u]) of known users."""
        d = self._b200_device()
        user_indices = np.asarray(user_indices, dtype=np.int64)
        if user_indices.size and (int(user_indices.min()) < 0 or int(user_indices.max()) >= self.num_users):
            raise IndexError("user index out of bounds for the %d users of the model" % self.num_users)
        return engine.score_batch_f64(d["U"], d["V"], user_idx=engine.to_device(user_indices, torch.int64))

    # reference: recom_pmf.py:191-222
    def score(self, user_idx, item_idx=None):
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            return self._b200_row(user_idx)
        # one item: the reference's host expression (a cached row is never used here: it holds the raw dot)
        user_pred = self.V[item_idx, :].dot(self.U[user_idx, :])
        if self.variant == "non_linear":
            user_pred = sigmoid(user_pred)
            user_pred = scale(user_pred, self.min_rating, self.max_rating, 0.0, 1.0)
        return user_pred

    # ---- ANNMixin (recom_pmf.py:224-252) -----------------------------------------------------------------------------
    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return self.U

    def get_item_vectors(self):
        return self.V
