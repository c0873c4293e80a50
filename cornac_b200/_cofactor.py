"""The fit and rank() shared by the SoRec and MCF plug-ins (recom_sorec.py, recom_mcf.py).

Both reference loops (cornac/models/sorec/cython/sorec.pyx, cornac/models/mcf/cython/mcf.pyx) draw U, V and Z from one
generator and then run, per epoch, PMF's non-linear RMSProp update over the graph edges and then over the ratings.  The
epochs run as b200_cofactor_fit over one level schedule of both streams, with the reference's f64 arithmetic, so U, V
and Z are bit-identical to the reference's.
"""
import numpy as np
import torch

from cornac.models.recommender import Recommender
from cornac.utils import get_rng
from cornac.utils.init_utils import normal

from . import engine


class CofactorMixin:
    """Expects `k`, `max_iter`, `learning_rate`, `gamma`, `seed`, `verbose`, `U`, `V`, `Z` and `num_users` / `num_items`
    (set by Recommender.fit); `_COFACTOR` is "sorec" or "mcf"."""

    _B200_LOSS_BYTES = 256 << 20                # device budget of the per-update loss terms when verbose

    def _z_rows(self):
        return self.num_users if self._COFACTOR == "sorec" else self.num_items

    def _init_factors(self):
        """sorec.pyx:63-75 / mcf.pyx:66-78: U, then V, then Z from one generator, each only when init_params does not
        supply it.  Raises ValueError on a wrong dtype or shape, before any device work."""
        rng = get_rng(self.seed)
        out = []
        for name, n in (("U", self.num_users), ("V", self.num_items), ("Z", self._z_rows())):
            x = getattr(self, name)
            if x is None:
                x = normal((n, self.k), mean=0.0, std=0.001, random_state=rng, dtype=np.double)
            a = np.asarray(x)
            if a.dtype != np.float64:                         # what the reference's double[:, :] memoryview raises
                raise ValueError("Buffer dtype mismatch, expected 'double' but got '%s'" % a.dtype)
            if a.ndim != 2 or a.shape[0] < n or a.shape[1] != self.k:
                raise ValueError("%s must have shape (%d, %d), got %s" % (name, n, self.k, a.shape))
            out.append(x)
        return out

    def _fit_cofactor(self, net_a, net_b, net_val, uid, iid, rat, lambda_c, lambda_reg):
        """Train U, V, Z from the prepared triplets (int32 ids, f32 values, stored order) and print the reference's
        verbose lines."""
        U, V, Z = self._init_factors()
        engine.require_cuda()
        data = engine.CofactorData(self._COFACTOR, net_a, net_b, net_val, uid, iid, rat, self.num_users, self.num_items)
        dev = [engine.to_device(np.ascontiguousarray(x), torch.float64) for x in (U, V, Z)]
        caches = [torch.zeros_like(x) for x in dev]
        hyper = [float(np.float32(x)) for x in (lambda_c, lambda_reg, self.learning_rate, self.gamma)]
        n_total = data.n_edges + data.n_ratings
        if self.verbose and n_total > 0:
            # each update's loss term lands at its stored index (edges, then ratings); summing a row in stored order is
            # the reference's sum
            chunk = max(1, self._B200_LOSS_BYTES // (8 * n_total))
            for e0 in range(0, self.max_iter, chunk):
                n = min(chunk, self.max_iter - e0)
                terms = torch.empty((n, n_total), dtype=torch.float64, device="cuda")
                engine.cofactor_fit(data, *dev, *caches, n, *hyper, loss=terms)
                loss = np.add.accumulate(terms.cpu().numpy(), axis=1)[:, -1]
                for j in range(n):
                    print("epoch %i, loss: %f" % (e0 + j, loss[j]))
        elif self.verbose:
            for e in range(self.max_iter):
                print("epoch %i, loss: %f" % (e, 0.0))
        else:
            engine.cofactor_fit(data, *dev, *caches, self.max_iter, *hyper)
        # an f64 init_params array is trained in place, as through the reference's memoryview
        for x, d in zip((U, V, Z), dev):
            x[...] = d.cpu().numpy()
        self.U, self.V, self.Z = U, V, Z
        if U.shape == (self.num_users, self.k) and V.shape == (self.num_items, self.k):
            self._b200_dev = dict(U=dev[0], V=dev[1])           # the trained device factors score as they are

    def rank(self, user_idx, item_indices=None, k=-1, **kwargs):
        """Recommender.rank (cornac/models/recommender.py:475-530) as written, over the f64 score row of score(u): the head
        of k items sorted and the rest in argpartition's order, or the whole argsort reversed for k == -1.  The examples of
        both models score NDCG over the whole list (NDCG(k=-1)) beside top-20 metrics, so the order of the tail is part of
        the metric; ScoringMixin.rank would order it by item id.  rank_batch / recommend_batch keep the shared order."""
        return Recommender.rank(self, user_idx, item_indices, k, **kwargs)
