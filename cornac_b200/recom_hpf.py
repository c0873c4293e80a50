"""(Hierarchical) Poisson factorisation on an H100: drop-in for cornac.models.HPF.

Same constructor arguments, defaults, attributes, printed lines, errors and fit()/score()/rank() behaviour as the
reference class (cornac/models/hpf/recom_hpf.py:25-243).  The initial state is the reference's host draw
(cornac/models/hpf/cython/hpf.pyx:35-164); the serial f64 iterations of hpf_cpp / pf_cpp
(cornac/models/hpf/cpp/cpp_hpf.cpp:139-275) run as b200_hpf_fit in the reference's update order.  The update arithmetic
is the reference's to the bit; exp, log and digamma are the GPU's own, so the fit agrees with the reference to rounding.
The full score rows of score(u) / rank() are f64 device dots (b200_score_batch_f64) ranked on the device
(b200_topk_rows_f64).
"""
import numpy as np
import scipy.sparse as sp
import torch

from cornac.exception import ScoreException
from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender
from cornac.utils import get_rng
from cornac.utils.init_utils import gamma

from . import engine
from ._scoring import F64DotScoringMixin

_STATE = (("G_s", "Gs"), ("G_r", "Gr"), ("L_s", "Ls"), ("L_r", "Lr"))


class HPF(F64DotScoringMixin, Recommender, ANNMixin):
    """Hierarchical Poisson Factorization (Gopalan, Hofman and Blei, UAI 2015), trained on the GPU.

    Parameters are the reference's: k=5, max_iter=100, name="HPF", trainable=True, verbose=False, hierarchical=True
    (False: plain Poisson factorisation), seed=None (initial state only; the fit itself is deterministic),
    init_params=None (a dict of f64 arrays: "G_s", "G_r" of shape (n_users, k), "L_s", "L_r" of shape (n_items, k) to
    start from, and "Theta", "Beta" to score with when trainable=False).
    """

    _B200_FACTORS = ("Theta", "Beta")

    def __init__(self, k=5, max_iter=100, name="HPF", trainable=True, verbose=False, hierarchical=True, seed=None,
                 init_params=None):
        Recommender.__init__(self, name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.max_iter = max_iter

        self.ll = np.full(max_iter, 0)
        self.etp_r = np.full(max_iter, 0)
        self.etp_c = np.full(max_iter, 0)
        self.eps = 0.000000001
        self.hierarchical = hierarchical
        self.seed = seed

        self.init_params = {} if init_params is None else init_params
        self.Theta = self.init_params.get("Theta", None)
        self.Beta = self.init_params.get("Beta", None)
        self.Gs = self.init_params.get("G_s", None)
        self.Gr = self.init_params.get("G_r", None)
        self.Ls = self.init_params.get("L_s", None)
        self.Lr = self.init_params.get("L_r", None)
        self._b200_register_ignored()

    # reference: recom_hpf.py:110-180
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._b200_invalidate()
        if self.trainable:
            X = train_set.csc_matrix
            rid, cid, val = sp.find(X)
            val = np.array(val, dtype="float32")
            Gs, Gr, Ls, Lr = self._init_state(X.shape[0], X.shape[1])
            print("Learning...")
            self._fit_b200(rid, cid, val.astype(np.float64), X.shape, Gs, Gr, Ls, Lr)
            print("Learning completed!")
        elif self.verbose:
            print("%s is trained already (trainable = False)" % (self.name))
        return self

    def _init_state(self, n, d):
        """hpf.pyx:51-79 (PF) and 118-146 (HPF): G_s, G_r, L_s, L_r drawn in that order from one generator, each only
        when it is not given.  A given array must be f64 of the fit's shape (the reference would crash instead)."""
        rng = get_rng(self.seed)
        shape, scale = (100.0, 0.3 / 100.0) if self.hierarchical else (0.3, 1 / 0.3)
        out = []
        for (key, attr), rows in zip(_STATE, (n, n, d, d)):
            x = getattr(self, attr)
            if x is None:
                x = gamma(shape, scale=scale, size=rows * self.k, random_state=rng).reshape(rows, self.k)
            else:
                x = np.asarray(x)
                if x.dtype != np.float64:
                    raise ValueError("init_params['%s'] must be a float64 array, got dtype %s" % (key, x.dtype))
                if x.shape != (rows, self.k):
                    raise ValueError("init_params['%s'] must have shape (%d, %d), got %s" % (key, rows, self.k, x.shape))
            out.append(np.ascontiguousarray(x, dtype=np.float64))
        return out

    def _fit_b200(self, rid, cid, val, shape, Gs, Gr, Ls, Lr):
        engine.require_cuda()
        n, d = shape
        data = engine.HpfData(rid, cid, val, n, d)
        st = [engine.to_device(x, torch.float64) for x in (Gs, Gr, Ls, Lr)]
        Kr = torch.ones(n, dtype=torch.float64, device="cuda")
        Tr = torch.ones(d, dtype=torch.float64, device="cuda")
        engine.hpf_fit(data, self.hierarchical, *st, Kr, Tr, self.max_iter)
        Gs, Gr, Ls, Lr = (t.cpu().numpy() for t in st)
        # hpf.pyx:88-95 / 155-162: Theta and Beta are the host quotients of the returned state
        self.Theta = Gs / Gr
        self.Beta = Ls / Lr
        self.Gs, self.Gr, self.Ls, self.Lr = Gs, Gr, Ls, Lr

    # reference: recom_hpf.py:182-213
    def score(self, user_idx, item_idx=None):
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        if item_idx is None:
            return self._b200_row(user_idx)
        user_pred = self.Beta[item_idx, :].dot(self.Theta[user_idx, :])
        user_pred = np.array(user_pred, dtype="float64").flatten()[0]
        return user_pred

    # ---- ANNMixin (recom_hpf.py:215-243) -----------------------------------------------------------------------------
    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        return self.Theta

    def get_item_vectors(self):
        return self.Beta
