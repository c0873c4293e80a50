"""EASE fit and ranking on the GPU at the MovieLens shapes, plus the reference's host fit where it is affordable.

    python tools/ease_bench.py OUTDIR [--shapes ml1m,ml10m,ml20m] [--reps 3]

Seeded synthetic ratings (1-5, Zipf 0.8 item popularity) at the ML-1M, ML-10M and ML-20M shapes.  Per shape: CUDA-event
medians (after one warm-up fit) of the Gram kernel (its inputs prepared and uploaded beforehand; that host preparation is
timed on its own, host clock), potrf, trtri, lauum, the weights pass and the B download; the achieved
FP64 rate of each factorisation phase from its n^3 / 3 flop against the H100 SXM data sheet's 67 TFLOP/s FP64 Tensor Core
rate (a 700 W card); fit() end to end; ranked users/s (score rows + top-100 with the training items excluded); and the
reference EASE.fit on the host for ML-1M and ML-10M.  Writes OUTDIR/ease_bench.json with the card's name, power limit and
max SM clock.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = os.path.join(ROOT, "oracle", "_ref")
if os.path.isdir(os.path.join(REF, "cornac")):
    sys.path.insert(0, REF)

from conftest import synth_csr  # noqa: E402
from cornac_b200 import _lib, engine  # noqa: E402

SHAPES = {"ml1m": (6040, 3706, 1_000_209), "ml10m": (69_878, 10_677, 10_000_054), "ml20m": (138_493, 26_744, 20_000_263)}
FP64_TC_PEAK = 67e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    name, power, clock = (s.strip() for s in q[0].split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def bench_shape(key, reps, with_ref):
    n_users, n, nnz = SHAPES[key]
    indptr, indices = synth_csr(n_users, n, nnz, 2024)
    X = sp.csr_matrix((np.random.RandomState(7).randint(1, 6, size=len(indices)).astype(np.float64), indices, indptr),
                      shape=(n_users, n))
    res = dict(shape=[n_users, n, int(X.nnz)])
    phases = {k: [] for k in ("gram_input", "gram", "potrf", "trtri", "lauum", "weights", "download", "fit")}
    A = torch.empty((n, n), dtype=torch.float64, device="cuda")
    ws = torch.empty(int(_lib.load().b200_spd_inverse_workspace_bytes(n)), dtype=torch.uint8, device="cuda")
    info = torch.zeros(1, dtype=torch.int32, device="cuda")
    host = torch.empty((n, n), dtype=torch.float64, pin_memory=False)
    for rep in range(reps + 1):
        t = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        inp = engine.EaseGramInput(X)
        torch.cuda.synchronize()
        t["gram_input"] = (time.perf_counter() - t0) * 1e3
        t["gram"], _ = timed(lambda: engine.ease_gram(inp, 500.0, A))
        del inp
        t["potrf"], _ = timed(lambda: engine.spd_inverse(A, _lib.SPD_POTRF, ws, info))
        t["trtri"], _ = timed(lambda: engine.spd_inverse(A, _lib.SPD_TRTRI, ws, info))
        t["lauum"], _ = timed(lambda: engine.spd_inverse(A, _lib.SPD_LAUUM, ws, info))
        t["weights"], _ = timed(lambda: engine.ease_weights(A, True))
        t["download"], _ = timed(lambda: host.copy_(A))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        B = engine.ease_fit(X, 500.0, True)
        Bh = B.cpu().numpy()
        t["fit"] = (time.perf_counter() - t0) * 1e3
        del B, Bh
        if rep:                                         # rep 0 is the warm-up
            for k, v in t.items():
                phases[k].append(v)
    res["ms"] = {k: float(np.median(v)) for k, v in phases.items()}
    flop = n ** 3 / 3.0
    res["tflops"] = {k: flop / (res["ms"][k] * 1e-3) / 1e12 for k in ("potrf", "trtri", "lauum")}
    res["share_of_fp64_tc_peak"] = {k: v * 1e12 / FP64_TC_PEAK for k, v in res["tflops"].items()}
    # ranked users/s: score rows + top-100 with the training items excluded, batches of 4096 users
    B = engine.ease_fit(X, 500.0, True)
    ratings = engine.EaseRatings(X)
    users = np.arange(min(n_users, 32768))
    batch = 4096

    def rank_all():
        for b0 in range(0, len(users), batch):
            ub = users[b0:b0 + batch]
            sub = X[ub]
            ep = engine.to_device(sub.indptr.astype(np.int64), torch.int64)
            ei = engine.to_device(sub.indices.astype(np.int32), torch.int32)
            engine.topk_rows_f64(engine.ease_score(B, ub, ratings), 100, ep, ei)

    rank_all()
    ms, _ = timed(rank_all)
    res["ranked_users_per_s"] = len(users) / (ms * 1e-3)
    del A, B, ws, host
    torch.cuda.empty_cache()
    if with_ref:
        from cornac.data import Dataset
        from cornac.models import EASE
        coo = X.tocoo()
        ds = Dataset.from_uir(list(zip(coo.row.astype(str), coo.col.astype(str), coo.data)), seed=None)
        t0 = time.perf_counter()
        EASE(lamb=500, posB=True, verbose=False).fit(ds)
        res["reference_fit_ms"] = (time.perf_counter() - t0) * 1e3
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--shapes", default="ml1m,ml10m,ml20m")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true")
    a = ap.parse_args()
    os.makedirs(a.outdir, exist_ok=True)
    engine.warmup()
    out = dict(card=card(), shapes={})
    for key in a.shapes.split(","):
        out["shapes"][key] = bench_shape(key, a.reps, with_ref=not a.no_ref and key in ("ml1m", "ml10m"))
        print(key, json.dumps(out["shapes"][key]), flush=True)
    with open(os.path.join(a.outdir, "ease_bench.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
