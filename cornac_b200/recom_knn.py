"""Neighbourhood models on an H100: drop-ins for cornac.models.UserKNN / ItemKNN.

Same constructor arguments, validation, attributes (`mean_arr`, `sim_mat`, and `iu_mat` / `ui_mat`) and
fit()/score()/rank() behaviour as the reference classes (cornac/models/knn/recom_knn.py:91-435).  The host preprocessing
(mean centring, idf / bm25 weighting) is the reference's, vectorised; the similarity (b200_knn_similarity), its
compaction into `sim_mat` and the neighbour scores (b200_knn_score_users / b200_knn_score_items) run on the GPU.
The dense f64 similarity stays on the device for scoring; it is rebuilt from `sim_mat` after load().
"""
import multiprocessing

import numpy as np
from scipy.sparse import coo_matrix

from cornac.exception import ScoreException
from cornac.models.recommender import Recommender
from cornac.utils import get_rng

from . import engine
from ._scoring import EvalCacheMixin

EPS = 1e-8
SIMILARITIES = ["cosine", "pearson"]
WEIGHTING_OPTIONS = ["idf", "bm25"]


def _mean_centered(m):
    """recom_knn.py:34-45 without the per-row loop: every stored value minus its row's mean, exact zeros replaced by EPS.
    The rows of one length are averaged together as a 2-D np.mean, which sums each row exactly as np.mean of the row
    does, so the means are bitwise the reference's.  Modifies and returns `m` (CSR) and the row means."""
    counts = np.diff(m.indptr)
    mean = np.zeros(m.shape[0])
    for n in np.unique(counts[counts > 0]):
        rows = np.flatnonzero(counts == n)
        mean[rows] = m.data[m.indptr[rows][:, None] + np.arange(n)].mean(axis=1)
    data = m.data - np.repeat(mean, counts)
    data[data == 0] = EPS
    m.data = data
    return m, mean


def _idf_weight(ui):
    X = coo_matrix(ui)
    idf = np.log(float(X.shape[0]) / np.bincount(X.col))
    return idf[ui.indices] + EPS


def _bm25_weight(ui):
    K1, B = 1.2, 0.8
    X = coo_matrix(ui)
    X.data = np.ones_like(X.data)
    idf = np.log(float(X.shape[0]) / np.bincount(X.col))
    row_sums = np.ravel(X.sum(axis=1))
    length_norm = (1.0 - B) + B * row_sums / row_sums.mean()
    return (K1 + 1.0) / (K1 * length_norm[X.row] + X.data) * idf[X.col] + EPS


class _KNNBase(EvalCacheMixin, Recommender):
    _B200_EVAL_TOP = 0                          # rank() sorts every candidate: the transform() cache keeps rows only
    _USER_MODE = None

    def __init__(self, name, k, similarity, mean_centered, weighting, amplify, num_threads, trainable, verbose, seed):
        super().__init__(name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.similarity = similarity
        self.mean_centered = mean_centered
        self.weighting = weighting
        self.amplify = amplify
        self.seed = seed
        self.rng = get_rng(seed)
        if self.similarity not in SIMILARITIES:
            raise ValueError("Invalid similarity choice, supported {}".format(SIMILARITIES))
        if self.weighting is not None and self.weighting not in WEIGHTING_OPTIONS:
            raise ValueError("Invalid weighting choice, supported {}".format(WEIGHTING_OPTIONS))
        if not k >= 1:                           # the reference indexes an empty heap for k < 1
            raise ValueError("k must be >= 1, got {}".format(k))
        if seed is not None:
            self.num_threads = 1
        elif 0 < num_threads < multiprocessing.cpu_count():
            self.num_threads = num_threads
        else:
            self.num_threads = multiprocessing.cpu_count()
        self._b200_register_ignored()

    def _weighted(self, weight_mat, train_set):
        if self.weighting == "idf":
            weight_mat.data *= np.sqrt(_idf_weight(train_set.matrix))
        elif self.weighting == "bm25":
            weight_mat.data *= np.sqrt(_bm25_weight(train_set.matrix))
        return weight_mat

    def _centred_ratings(self, train_set):
        ui = train_set.matrix.copy()
        mean = np.zeros(ui.shape[0])
        if self.min_rating != self.max_rating:  # explicit feedback
            ui, mean = _mean_centered(ui)
        return ui, mean

    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._b200_invalidate()
        weight_mat, ui, self.mean_arr = self._host_prepare(train_set)
        self._keep_ratings(ui)
        S, self.sim_mat = engine.knn_similarity(weight_mat, self.amplify)
        self._b200_dev = dict(S=S, ratings=engine.KnnRatings(self._score_ratings(), self.mean_arr))
        return self

    def _b200_device(self):
        if getattr(self, "_b200_dev", None) is None:         # None after fit(); absent after load()
            self._b200_dev = dict(S=engine.knn_dense(self.sim_mat),
                                  ratings=engine.KnnRatings(self._score_ratings(), self.mean_arr))
        return self._b200_dev

    def _scores_dev(self, user_indices):
        d = self._b200_device()
        return engine.knn_score(self._USER_MODE, d["S"], np.asarray(user_indices, dtype=np.int64), d["ratings"], int(self.k))

    def rank(self, user_idx, item_indices=None, k=-1, **kwargs):
        """`Recommender.rank` (cornac/models/recommender.py:476-530) with the total order (score desc, item id asc)."""
        try:
            known = self.score(user_idx, **kwargs)
        except ScoreException:
            known = np.ones(self.total_items) * self.default_score()
        if len(known) == self.total_items:
            all_scores = known
        else:                                           # unknown items get the MIN score
            all_scores = np.ones(self.total_items) * np.min(known)
            all_scores[: self.num_items] = known
        item_indices = np.arange(self.num_items) if item_indices is None else np.asarray(item_indices)
        item_scores = all_scores[item_indices]
        order = np.lexsort((item_indices, -item_scores))
        return item_indices[order], item_scores


class UserKNN(_KNNBase):
    """User-based nearest neighbours (cornac.models.UserKNN, recom_knn.py:91-264) with the similarity and the scores on
    the GPU."""

    _USER_MODE = True

    def __init__(self, name="UserKNN", k=20, similarity="cosine", mean_centered=False, weighting=None, amplify=1.0,
                 num_threads=0, trainable=True, verbose=True, seed=None):
        super().__init__(name, k, similarity, mean_centered, weighting, amplify, num_threads, trainable, verbose, seed)

    # reference: recom_knn.py:183-203
    def _host_prepare(self, train_set):
        ui, mean = self._centred_ratings(train_set)
        weight_mat = ui.copy() if (self.mean_centered or self.similarity == "pearson") else train_set.matrix.copy()
        return self._weighted(weight_mat, train_set), ui, mean

    def _keep_ratings(self, ui):
        self.iu_mat = ui.T.tocsr()

    def _score_ratings(self):
        return self.iu_mat

    # reference: recom_knn.py:212-264
    def score(self, user_idx, item_idx=None):
        if not self.knows_user(user_idx):
            raise ScoreException("Can't make score prediction for (user_id=%d)" % user_idx)
        if item_idx is not None and not self.knows_item(item_idx):
            raise ScoreException("Can't make score prediction for (item_id=%d)" % item_idx)
        return self._b200_row(user_idx, item_idx)


class ItemKNN(_KNNBase):
    """Item-based nearest neighbours (cornac.models.ItemKNN, recom_knn.py:267-435) with the similarity and the scores on
    the GPU."""

    _USER_MODE = False

    def __init__(self, name="ItemKNN", k=20, similarity="cosine", mean_centered=False, weighting=None, amplify=1.0,
                 num_threads=0, trainable=True, verbose=True, seed=None):
        super().__init__(name, k, similarity, mean_centered, weighting, amplify, num_threads, trainable, verbose, seed)

    # reference: recom_knn.py:359-381
    def _host_prepare(self, train_set):
        ui, mean = self._centred_ratings(train_set)
        weight_mat = ui.copy() if self.mean_centered else train_set.matrix.copy()
        if self.similarity == "pearson":                 # centred by columns
            weight_mat, _ = _mean_centered(weight_mat.T.tocsr())
            weight_mat = weight_mat.T.tocsr()
        return self._weighted(weight_mat, train_set).T.tocsr(), ui, mean

    def _keep_ratings(self, ui):
        self.ui_mat = ui

    def _score_ratings(self):
        return self.ui_mat

    # reference: recom_knn.py:389-435
    def score(self, user_idx, item_idx=None):
        if self.is_unknown_user(user_idx):
            raise ScoreException("Can't make score prediction for user %d" % user_idx)
        if item_idx is not None and self.is_unknown_item(item_idx):
            raise ScoreException("Can't make score prediction for item %d" % item_idx)
        return self._b200_row(user_idx, item_idx)
