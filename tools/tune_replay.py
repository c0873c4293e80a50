"""Seeded (deterministic) mode throughput: the scheduled replay kernel vs the serial kernel vs the oracle's
single-thread loop, on a mid-size matrix (dev tool, GPU box)."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from conftest import synth_csr  # noqa: E402
from cornac_b200 import engine  # noqa: E402
from oracle import oracle as O  # noqa: E402

for (n_users, n_items, nnz, k) in ((943, 1682, 80000, 10), (100_000, 20_000, 5_000_000, 64)):
    indptr, indices = synth_csr(n_users, n_items, nnz, seed=1)
    nnz = len(indices)
    rng = np.random.RandomState(0)
    U0 = rng.normal(0, 0.1, (n_users, k)).astype(np.float32)
    V0 = rng.normal(0, 0.1, (n_items, k)).astype(np.float32)
    B0 = np.zeros(n_items, np.float32)
    n = min(nnz, 2_000_000)
    ii = rng.randint(nnz, size=n).astype(np.int64)
    jj = rng.randint(n_items, size=n).astype(np.int32)
    data = engine.BprData.from_host(indptr, indices)
    di, dj = torch.from_numpy(ii).cuda(), torch.from_numpy(jj).cuda()
    res = {}
    for serial in ("1", "0"):
        os.environ["B200_REPLAY_SERIAL"] = serial
        U, V, B = (torch.from_numpy(x.copy()).cuda() for x in (U0, V0, B0))
        stats = torch.zeros(2, dtype=torch.int64, device="cuda")
        engine.bpr_epoch_replay(data, di[:1000], dj[:1000], U, V, B, 0.05, 0.01, True, stats)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        engine.bpr_epoch_replay(data, di, dj, U, V, B, 0.05, 0.01, True, stats)
        torch.cuda.synchronize()
        res[serial] = n / (time.perf_counter() - t0)
    Ur, Vr, Br = U0.copy(), V0.copy(), B0.copy()
    t0 = time.perf_counter()
    O.bpr_replay(ii, jj, indptr, indices, Ur, Vr, Br, 0.05, 0.01, True)
    cpu = n / (time.perf_counter() - t0)
    print("%d x %d x %d k=%d: scheduled (default; on-chip model when it fits) %.2f M/s, serial-warp %.2f M/s, "
          "oracle 1 thread %.2f M samples/s" % (n_users, n_items, nnz, k, res["0"] / 1e6, res["1"] / 1e6, cpu / 1e6), flush=True)
