"""TEST INFRASTRUCTURE: scalar numpy restatement of the reference's neighbourhood kernels.

    similarity(...)  <- compute_similarity  cornac/models/knn/similarity.pyx:51-105
    score_row(...)   <- compute_score       cornac/models/knn/similarity.pyx:154-201 with SparseNeighbors / TopK of
                                            cornac/models/knn/similarity.h:15-89 (compute_score_single :109-150 is one entry)

The similarity keeps the reference's order of operations: S[r, x] is summed over the stored entries of row r in stored
order, every product and sum rounded on its own (numpy never fuses a multiply-add).  The denominator is the one the
compiled reference evaluates: it is built with -O3 -ffast-math (setup.py), under which gcc turns the source's
sqrt(D1) * sqrt(D2) into sqrt(D1 * D2); `denominator="source"` gives the formula as written, for comparison.
"""
import numpy as np


def similarity(indptr, indices, data, n_cols, denominator="compiled"):
    """Dense f64 [n, n] similarity of the n rows of the CSR weight matrix (indptr, indices, data)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    data = np.asarray(data, dtype=np.float64)
    n = len(indptr) - 1
    rows = np.repeat(np.arange(n), np.diff(indptr))
    order = np.lexsort((rows, indices))                  # the transpose: column c's entries in ascending row
    c_ptr = np.zeros(n_cols + 1, dtype=np.int64)
    np.add.at(c_ptr, indices + 1, 1)
    c_ptr = np.cumsum(c_ptr)
    c_idx, c_val = rows[order], data[order]
    S = np.zeros((n, n))
    for r in range(n):
        D1, D2, s = np.zeros(n), np.zeros(n), S[r]
        for p in range(indptr[r], indptr[r + 1]):
            c, w = indices[p], data[p]
            xs, v = c_idx[c_ptr[c]:c_ptr[c + 1]], c_val[c_ptr[c]:c_ptr[c + 1]]
            s[xs] = s[xs] + v * w                        # one term per x per column: the ordered sum
            both = (v != 0) & (w != 0)
            D1[xs[both]] = D1[xs[both]] + w * w
            D2[xs[both]] = D2[xs[both]] + v[both] * v[both]
        nz = s != 0
        if denominator == "compiled":
            s[nz] = s[nz] / np.sqrt(D1[nz] * D2[nz])
        else:
            s[nz] = s[nz] / (np.sqrt(D1[nz]) * np.sqrt(D2[nz]))
    return S


def amplify(sim, alpha):
    """recom_knn.py:48-55 on the non-zeros of a dense matrix."""
    out = np.array(sim, dtype=np.float64)
    if alpha == 1.0:
        return out
    pos, neg = out > 0, out < 0
    out[pos] = out[pos] ** alpha
    out[neg] = -((-out[neg]) ** alpha)
    return out


def select(candidates, k):
    """The pairs TopK keeps from `candidates` [(weight, value), ...] given in the order SparseNeighbors visits them
    (descending neighbour index): the first k are kept; after that a candidate is kept only if its weight is strictly
    greater than the smallest kept weight, and it replaces the smallest kept (weight, value) pair."""
    kept = []
    for w, v in candidates:
        if len(kept) < k:
            kept.append((w, v))
        elif w > min(kept)[0]:
            kept.remove(min(kept))
            kept.append((w, v))
    return kept


def weighted_average(kept):
    num = den = 0.0
    for w, v in kept:
        num = num + w * v
        den = den + abs(w)
    return num / (den + 1e-8)


def score_row(user_mode, sim_row, indptr, indices, data, k):
    """compute_score: one weighted average per row of (indptr, indices, data), without the user's mean.
    user_mode (UserKNN): sim_row = row u of the similarity, (indptr, indices, data) = the item-user matrix.
    item mode (ItemKNN): sim_row = row u of the user-item matrix, (indptr, indices, data) = the similarity in CSR."""
    out = np.zeros(len(indptr) - 1)
    for i in range(len(out)):
        cand = []
        for p in range(indptr[i + 1] - 1, indptr[i] - 1, -1):
            nn, s = indices[p], data[p]
            if sim_row[nn] != 0:
                cand.append((sim_row[nn], s) if user_mode else (s, sim_row[nn]))
        out[i] = weighted_average(select(cand, k))
    return out
