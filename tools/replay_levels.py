"""CPU analysis for the seeded (parity) mode: how much parallelism does the reference's sample stream allow?

A sample (u, i, j) must see every earlier update of its three rows; samples that share no row commute exactly.  The
dependency level of a sample = 1 + the largest level among earlier samples that touch one of its rows; all samples of
one level are independent, and the number of levels is the length of the critical path = the number of sequential steps
ANY exact schedule needs.  The scheduled replay kernel (bpr_replay_sched_kernel) resolves this inside phases of 1024
samples; this script measures what window sizes up to the whole epoch would allow.  Pure numpy + the host sampler of libb200cornac.so; no GPU."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from conftest import synth_csr  # noqa: E402
from cornac_b200 import engine  # noqa: E402


def levels(u, i, j, skip, n_users, n_items, window):
    """critical-path length summed over consecutive windows of `window` samples, and the mean parallelism"""
    total_levels = 0
    n = len(u)
    for a in range(0, n, window):
        lu = np.zeros(n_users, np.int32)
        li = np.zeros(n_items, np.int32)
        top = 0
        for t in range(a, min(n, a + window)):
            if skip[t]:
                continue
            lv = 1 + max(lu[u[t]], li[i[t]], li[j[t]])
            lu[u[t]] = li[i[t]] = li[j[t]] = lv
            top = max(top, lv)
        total_levels += top
    return total_levels, (n - int(skip.sum())) / max(total_levels, 1)


def main():
    for (n_users, n_items, nnz, label) in [(943, 1682, 100_000, "ML-100K sized"), (20_000, 5_000, 1_000_000, "20K x 5K x 1M")]:
        indptr, indices = synth_csr(n_users, n_items, nnz, seed=1)
        nnz = len(indices)
        coo = np.repeat(np.arange(n_users), np.diff(indptr))
        pos, neg = engine.MTSampler(11), engine.MTSampler(12)
        n = min(nnz, 200_000)
        ii = pos.fill(nnz - 1, n, dtype=np.int64)
        jj = neg.fill(n_items - 1, n, dtype=np.int32)
        u, i = coo[ii], indices[ii]
        key = set((coo.astype(np.int64) * n_items + indices).tolist())
        skip = np.fromiter(((int(a) * n_items + int(b)) in key for a, b in zip(u, jj)), dtype=bool, count=n)
        print("%s: %d samples, %.1f %% skipped" % (label, n, 100.0 * skip.mean()))
        for w in (32, 256, 1024, 8192, n):
            lv, par = levels(u, i, jj, skip, n_users, n_items, w)
            print("  window %7d: %7d sequential steps, mean parallelism %.1f" % (w, lv, par))


if __name__ == "__main__":
    main()
