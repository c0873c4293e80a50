"""Time the PMF fit and the f64 rank on seeded rating sets; write one JSON file.

    python tools/pmf_bench.py OUTDIR [--epochs 100] [--runs 3]

Shapes (k = 10, ratings 1-5, Zipf 0.8 item popularity, ratings in shuffled order): ML-100K (943 x 1682 x 100 000),
ML-1M (6040 x 3706 x 1 000 209) and ML-10M (69 878 x 10 677 x 10 000 054), both variants.  For each: the level count
of the schedule and the mean level width, the schedule's host time, the fit's CUDA-event time (median of --runs after a
warm-up; --epochs epochs, 10 on ML-10M) and its ms per epoch, and the ranked users/s of score_batch_f64 + topk_rows_f64
(top-10, training items excluded).  The compiled reference's pmf_linear / pmf_non_linear (oracle/_ref) is timed on the
same host when importable, over fewer epochs on the larger shapes.  The card's name and power limit are read in the run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "oracle", "_ref"))

SHAPES = [("ml100k", 943, 1682, 100000, None, 100), ("ml1m", 6040, 3706, 1000209, None, 10),
          ("ml10m", 69878, 10677, 10000054, 10, 1)]     # name, users, items, nnz, GPU epochs cap, reference epochs


def synth(n_users, n_items, nnz, seed, zipf=0.8):
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** zipf
    p /= p.sum()
    key = np.unique(rng.randint(n_users, size=int(nnz * 1.4)).astype(np.int64) * n_items
                    + rng.choice(n_items, size=int(nnz * 1.4), p=p))
    key = rng.choice(key, size=min(nnz, len(key)), replace=False)       # shuffled order
    r = rng.randint(1, 6, size=len(key)).astype(np.float32)
    return (key // n_items).astype(np.int32), (key % n_items).astype(np.int32), r


def cuda_median(fn, runs):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return float(np.median(ts))


def run_shape(name, n_users, n_items, nnz, cap, ref_epochs, epochs, runs):
    import scipy.sparse as sp
    import torch
    from cornac_b200 import engine
    uid, iid, rat = synth(n_users, n_items, nnz, seed=1)
    out = dict(n_users=n_users, n_items=n_items, nnz=len(uid), k=10)
    t = time.perf_counter()
    data = engine.PmfData(uid, iid, rat, n_users, n_items)
    torch.cuda.synchronize()
    out["schedule_and_upload_s"] = time.perf_counter() - t
    out["levels_per_epoch"] = data.n_levels
    out["mean_level_width"] = len(uid) / data.n_levels
    out["max_item_degree"] = int(np.bincount(iid).max())
    ep = epochs if cap is None else min(epochs, cap)
    rng = np.random.RandomState(2)
    U0, V0 = rng.normal(0, 0.001, (n_users, 10)), rng.normal(0, 0.001, (n_items, 10))
    for variant in ("linear", "non_linear"):
        r = rat if variant == "linear" else (rat - np.float32(1)) / np.float32(4)
        d = engine.PmfData(uid, iid, r, n_users, n_items)
        U, V = engine.to_device(U0, torch.float64), engine.to_device(V0, torch.float64)
        cu, cv = torch.zeros_like(U), torch.zeros_like(V)
        fit_s = cuda_median(lambda: engine.pmf_fit(d, variant, U, V, cu, cv, ep, 0.001, 0.001, 0.9), runs)
        res = dict(epochs=ep, fit_s=fit_s, ms_per_epoch=1e3 * fit_s / ep)
        try:
            from cornac.models.pmf import pmf as cy
            fn = cy.pmf_linear if variant == "linear" else cy.pmf_non_linear
            t = time.perf_counter()
            fn(uid, iid, r, n_users=n_users, n_items=n_items, n_ratings=len(uid), k=10, n_epochs=ref_epochs,
               init_params={"U": U0.copy(), "V": V0.copy()}, seed=1)
            ref_s = time.perf_counter() - t
            res.update(reference_epochs=ref_epochs, reference_s=ref_s, reference_ms_per_epoch=1e3 * ref_s / ref_epochs,
                       speedup_per_epoch=(ref_s / ref_epochs) / (fit_s / ep))
        except ImportError as e:
            res["reference"] = "not importable: %s" % e
        out[variant] = res
        print(name, variant, json.dumps(res), flush=True)
    # ranked users/s: all users, top-10, training items excluded, batches of 4096 users
    X = sp.csr_matrix((np.ones(len(uid)), (uid, iid)), shape=(n_users, n_items))
    X.sort_indices()
    Ud, Vd = engine.to_device(U0, torch.float64), engine.to_device(V0, torch.float64)
    batches = []
    for b0 in range(0, n_users, 4096):
        sub = X[b0:b0 + 4096]
        batches.append((engine.to_device(np.arange(b0, b0 + sub.shape[0]), torch.int64),
                        engine.to_device(sub.indptr.astype(np.int64), torch.int64),
                        engine.to_device(sub.indices.astype(np.int32), torch.int32)))

    def rank_all():
        for users, ep_, ei in batches:
            engine.topk_rows_f64(engine.score_batch_f64(Ud, Vd, user_idx=users), 10, ep_, ei)

    rank_s = cuda_median(rank_all, runs)
    out["rank_users_per_s"] = n_users / rank_s
    print(name, "rank users/s %.3g" % out["rank_users_per_s"], flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    from cornac_b200 import engine
    engine.warmup()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q, runs=a.runs, host_cpus=os.cpu_count(), cases={})
    print(res["gpu"], q, flush=True)
    for name, nu, ni, nnz, cap, ref_ep in SHAPES:
        res["cases"][name] = run_shape(name, nu, ni, nnz, cap, ref_ep, a.epochs, a.runs)
    os.makedirs(a.outdir, exist_ok=True)
    with open(os.path.join(a.outdir, "pmf_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
