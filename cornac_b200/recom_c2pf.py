"""Collaborative Context Poisson Factorization on an H100: drop-in for cornac.models.C2PF.

Same constructor arguments, defaults, name rule, attributes, printed lines and fit()/score()/rank() behaviour as the
reference class (cornac/models/c2pf/recom_c2pf.py), with these differences, each where the reference cannot run:
  * a train set without an `item_graph` modality raises a ValueError naming it (the reference: AttributeError);
  * a context edge (r, i) whose mirror (i, r) is not among the training edges raises a ValueError naming the edge and
    GraphModality(symmetric=True): on such a graph the reference writes past the end of its kappa triplets and the
    process dies (see DESIGN.md K13);
  * variant="rc2pf" draws its kappa triplets like the other two variants, where the reference raises a TypeError unless
    both are given (c2pf.pyx:316-317 assigns a column of a C++ vector).
The initial state is the reference's host draw from the global numpy generator (c2pf.pyx); the two calls of the serial f64
fit that c2pf.pyx makes (kappa pinned, then its prior) run as b200_c2pf_fit in the reference's update order, with the
reference's handling of the kappa triplet lists in between; Theta, Beta and Xi are the reference's host expressions.
The update arithmetic is the reference's to the bit; exp, log and digamma are the GPU's own, so the fit agrees with the
reference to rounding.  The full score rows of score(u) / rank() are f64 device dots of Theta with Beta + Xi
(b200_score_batch_f64) ranked on the device (b200_topk_rows_f64); score(u, i) is the reference's host expression.
"""
import numpy as np
import scipy.sparse as sp
import torch

from cornac.models.recommender import ANNMixin, MEASURE_DOT, Recommender

from . import engine
from ._scoring import F64DotScoringMixin

_STATE = (("G_s", "Gs"), ("G_r", "Gr"), ("L_s", "Ls"), ("L_r", "Lr"), ("L2_s", "L2s"), ("L2_r", "L2r"), ("L3_s", "L3s"),
          ("L3_r", "L3r"))
_ABSENT = {"c2pf": (), "tc2pf": ("L2_s", "L2_r"), "rc2pf": ("L_s", "L_r")}
PHASE_ONE = (1e15, 1e15)                                    # c2pf.pyx: kappa pinned during the first max_iter iterations
PHASE_TWO = {"c2pf": (2.0, 5.0), "tc2pf": (2.0, 4.0), "rc2pf": (2.0, 4.0)}


class ContextGraph:
    """The context triplets [m, 3] (row, col, value) as the reference's fit holds them: the CSC pattern of
    triplet_to_csc_sparse, util_sum (scipy's column sums, which ADD the values of a repeated pair) and, for each stored
    (r, i), the position of (i, r).  ValueError when a mirror is missing."""

    def __init__(self, C, d):
        self.d = int(d)
        rid, cid = C[:, 0].astype(np.int64), C[:, 1].astype(np.int64)
        self.keys = np.unique(cid * self.d + rid)                               # sorted: column, then row = CSC order
        self.nnz = len(self.keys)
        self.row, self.col = self.keys % self.d, self.keys // self.d
        self.ptr = np.zeros(self.d + 1, dtype=np.int64)
        np.cumsum(np.bincount(self.col, minlength=self.d), out=self.ptr[1:])
        self.util = sp.csc_matrix((C[:, 2], (rid, cid)), shape=(self.d, self.d)).sum(axis=0).A1     # c2pf.pyx:123-124
        mkeys = self.row * self.d + self.col
        self.mir = np.minimum(np.searchsorted(self.keys, mkeys), max(self.nnz - 1, 0))
        bad = np.flatnonzero(self.keys[self.mir] != mkeys) if self.nnz else []
        if len(bad):
            order = {k: j for j, k in reversed(list(enumerate(cid * self.d + rid)))}
            first = min(bad, key=lambda p: order[self.keys[p]])
            raise ValueError(
                "C2PF needs a symmetric item context: the edge (%d, %d) (item indices) has no mirror (%d, %d) among the "
                "training edges; build the item graph with GraphModality(symmetric=True)"
                % (self.row[first], self.col[first], self.col[first], self.row[first]))

    def values(self, trip, key):
        """triplet_to_csc_sparse of a kappa triplet list: a value per stored entry, the LAST of a repeated pair."""
        trip = np.asarray(trip)
        if trip.dtype != np.float64:
            raise ValueError("init_params['%s'] must be a float64 array, got dtype %s" % (key, trip.dtype))
        if trip.ndim != 2 or trip.shape[1] != 3:
            raise ValueError("init_params['%s'] must have shape (m, 3): (row, col, value) triplets, got %s" % (key, trip.shape))
        k = trip[:, 1].astype(np.int64) * self.d + trip[:, 0].astype(np.int64)
        slot = np.minimum(np.searchsorted(self.keys, k), max(self.nnz - 1, 0))
        if (self.nnz == 0 and len(k)) or not np.array_equal(self.keys[slot], k) or len(np.unique(slot)) != self.nnz:
            raise ValueError("init_params['%s'] must have one triplet for each context edge of the train set" % key)
        if not np.all(trip[:, 2] > 0):
            raise ValueError("init_params['%s'] must hold positive values" % key)
        out = np.empty(self.nnz, dtype=np.float64)
        out[slot] = trip[:, 2]                          # repeated indices: numpy assigns the last
        return out

    def write_back(self, trip, values):
        """csc_sparse_to_triplet: the first nnz rows of the list become the entries in CSC order; rows beyond (the list
        had repeated pairs) keep what they held."""
        trip[: self.nnz, 0], trip[: self.nnz, 1], trip[: self.nnz, 2] = self.row, self.col, values


class C2PF(F64DotScoringMixin, Recommender, ANNMixin):
    """Collaborative Context Poisson Factorization (Salah and Lauw, IJCAI 2018), trained on the GPU.

    Parameters are the reference's: k=100, max_iter=100, variant="c2pf" ("tc2pf": tied, "rc2pf": reduced; anything else
    runs as "c2pf"), name=None (variant.upper()), trainable=True, verbose=False, init_params=None (a dict of f64 arrays:
    "G_s", "G_r" of shape (n_users, k), "L_s", "L_r", "L2_s", "L2_r" of shape (n_items, k), "L3_s", "L3_r" (row, col,
    value) triplets over the context edges, to start from; "Theta", "Beta", "Xi" to score with when trainable=False).
    The initial state comes from the global numpy generator (np.random.seed).  The train set needs an `item_graph`.
    """

    def __init__(self, k=100, max_iter=100, variant="c2pf", name=None, trainable=True, verbose=False, init_params=None):
        if name is None:
            Recommender.__init__(self, name=variant.upper(), trainable=trainable, verbose=verbose)
        else:
            Recommender.__init__(self, name=name, trainable=trainable, verbose=verbose)
        self.k = k
        self.max_iter = max_iter

        self.ll = np.full(max_iter, 0)
        self.eps = 0.000000001
        self.variant = variant

        self.init_params = {} if init_params is None else init_params
        self.Theta = self.init_params.get("Theta", None)
        self.Beta = self.init_params.get("Beta", None)
        self.Xi = self.init_params.get("Xi", None)
        for key, attr in _STATE:
            setattr(self, attr, self.init_params.get(key, None))
        self._b200_register_ignored()

    def _variant(self):
        return self.variant if self.variant in PHASE_TWO else "c2pf"            # recom_c2pf.py:219-230

    # reference: recom_c2pf.py:132-249
    def fit(self, train_set, val_set=None):
        Recommender.fit(self, train_set, val_set)
        self._b200_invalidate()
        if self.trainable:
            if getattr(train_set, "item_graph", None) is None:
                raise ValueError("C2PF requires a train set with an item_graph modality (cornac.data.GraphModality)")
            X = train_set.csr_matrix
            rid, cid, val = sp.find(X)
            val = np.array(val, dtype="float32")
            train_item_indices = set(train_set.uir_tuple[1])
            c_rid, c_cid, c_val = train_set.item_graph.get_train_triplet(train_item_indices, train_item_indices)
            C = np.hstack((c_rid.reshape(-1, 1), c_cid.reshape(-1, 1), c_val.reshape(-1, 1))).astype(np.float64)
            graph = ContextGraph(C, X.shape[1])
            state = self._init_state(X.shape[0], X.shape[1], C, graph)
            print("Learning...")
            self._fit_b200(rid, cid, val.astype(np.float64), X.shape, graph, state)
            print("Learning completed!")
        elif self.verbose:
            print("%s is trained already (trainable = False)" % (self.name))
        return self

    def _init_state(self, n, d, C, graph):
        """c2pf.pyx:62-119 and its t_ / r_ twins: G_s, G_r, L_s, L_r, L2_s, L2_r, L3_s, L3_r drawn in that order from the
        global numpy generator, the variant's matrices only and each only when it is not given.  A given array must be
        f64 of the fit's shape (the reference would crash instead).  Returns {key: array}; kappa as triplet lists."""
        out = {}
        for key, attr in _STATE:
            if key in _ABSENT[self._variant()]:
                continue
            x = getattr(self, attr)
            if key.startswith("L3"):
                if x is None:
                    x = np.copy(C)
                    x[:, 2] = np.random.gamma(100, scale=0.5 / 100, size=C.shape[0])
                graph.values(x, key)
                out[key] = np.array(x, dtype=np.float64)
                continue
            rows = n if key.startswith("G") else d
            if x is None:
                x = np.random.gamma(100, scale=0.3 / 100, size=rows * self.k).reshape(rows, self.k)
            else:
                x = np.asarray(x)
                if x.dtype != np.float64:
                    raise ValueError("init_params['%s'] must be a float64 array, got dtype %s" % (key, x.dtype))
                if x.shape != (rows, self.k):
                    raise ValueError("init_params['%s'] must have shape (%d, %d), got %s" % (key, rows, self.k, x.shape))
            out[key] = np.ascontiguousarray(x, dtype=np.float64)
        return out

    def _fit_b200(self, rid, cid, val, shape, graph, state):
        engine.require_cuda()
        n, d = shape
        variant = self._variant()
        dgraph = engine.C2pfGraph(engine.HpfData(rid, cid, val, n, d), graph.ptr, graph.row, graph.mir, graph.util)
        L3s, L3r = state["L3_s"], state["L3_r"]
        edge = lambda x: engine.to_device(x if len(x) else np.zeros(1), torch.float64)          # noqa: E731
        dev = [None if key in _ABSENT[variant] else engine.to_device(state[key], torch.float64) for key, _ in _STATE[:6]]
        dev += [edge(graph.values(L3s, "L3_s")), edge(graph.values(L3r, "L3_r")),
                torch.ones(d, dtype=torch.float64, device="cuda")]
        for (at, bt), n_iter in ((PHASE_ONE, self.max_iter), (PHASE_TWO[variant], int(0.2 * self.max_iter))):
            engine.c2pf_fit(dgraph, variant, at, bt, dev, n_iter)
            if variant != "rc2pf":                      # rc2pf_cpp takes the triplets by value: what it learns is dropped
                graph.write_back(L3s, dev[6].cpu().numpy()[: graph.nnz])
                graph.write_back(L3r, dev[7].cpu().numpy()[: graph.nnz])
            if variant == "rc2pf" or len(L3s) > graph.nnz or len(L3r) > graph.nnz:
                dev[6], dev[7] = edge(graph.values(L3s, "L3_s")), edge(graph.values(L3r, "L3_r"))
        host = {key: None if t is None else t.cpu().numpy() for (key, _), t in zip(_STATE[:6], dev)}
        host["L3_s"], host["L3_r"] = L3s, L3r
        # c2pf.pyx:133-149 and its twins, recom_c2pf.py:232-244
        M3 = sp.csc_matrix((L3s[:, 2] / L3r[:, 2], (L3s[:, 0], L3s[:, 1])), shape=(d, d))
        ctx = "L" if variant == "tc2pf" else "L2"
        Q = M3 * (host[ctx + "_s"] / host[ctx + "_r"])
        W = Q if variant == "rc2pf" else host["L_s"] / host["L_r"]
        self.Theta = sp.csc_matrix(host["G_s"] / host["G_r"]).todense()
        self.Beta = sp.csc_matrix(W).todense()
        self.Xi = sp.csc_matrix(Q).todense()
        for key, attr in _STATE:
            setattr(self, attr, host[key])

    def _b200_device(self):
        """Theta and the item matrix the score row multiplies it with: Beta + Xi (rc2pf: Xi), formed once on the host."""
        if getattr(self, "_b200_dev", None) is None:      # None after fit(); absent after load()
            engine.require_cuda()
            items = np.asarray(self.Xi) if self.variant == "rc2pf" else np.asarray(self.Beta) + np.asarray(self.Xi)
            self._b200_dev = dict(
                U=engine.to_device(np.ascontiguousarray(np.asarray(self.Theta)[: self.num_users], dtype=np.float64), torch.float64),
                V=engine.to_device(np.ascontiguousarray(items[: self.num_items], dtype=np.float64), torch.float64))
        return self._b200_dev

    # reference: recom_c2pf.py:251-298
    def score(self, user_idx, item_idx=None):
        if item_idx is None:
            return self._b200_row(user_idx)
        # one item: the reference's host expression as it stands.  For c2pf / tc2pf it does not index Xi, so it returns
        # the vector Beta[i] . Theta[u] + Xi Theta[u] over all items
        if self.variant == "rc2pf":
            user_pred = self.Xi[item_idx,] * self.Theta[user_idx, :].T
        else:
            user_pred = self.Beta[item_idx, :] * self.Theta[user_idx, :].T + self.Xi * self.Theta[user_idx, :].T
        user_pred = np.array(user_pred, dtype="float64").flatten()
        return user_pred

    def rank(self, user_idx, item_indices=None, k=-1, **kwargs):
        """Recommender.rank as written, over the f64 row of score(u), for SoRec's reason (_cofactor.py): the reference's
        example scores NDCG(k=-1) beside top-20 metrics, so the order of a top-k ranking's tail is part of the metric."""
        return Recommender.rank(self, user_idx, item_indices, k, **kwargs)

    # ---- ANNMixin (recom_c2pf.py:300-336) ----------------------------------------------------------------------------
    def get_vector_measure(self):
        return MEASURE_DOT

    def get_user_vectors(self):
        if self.variant == "rc2pf":
            return np.concatenate((self.Theta, self.Theta), axis=1)
        return self.Theta

    def get_item_vectors(self):
        if self.variant == "rc2pf":
            return np.concatenate((self.Beta, self.Xi), axis=1)
        return self.Beta
