"""Time the NMF fit on seeded rating sets in CSR order; write one JSON file.

    python tools/nmf_bench.py OUTDIR [--epochs 20] [--runs 3]

Shapes (k = 15, ratings 1-5, Zipf 0.8 item popularity, CSR order as train_set.matrix stores them): ML-100K
(943 x 1682 x 100 000), ML-1M (6040 x 3706 x 1 000 000) and ML-10M (69 878 x 10 677 x 10 000 000), use_bias False and
True.  For each: the level count of the bias pass, the fit's ms per epoch (CUDA events, median of --runs after a
warm-up), the time per phase from torch.profiler in a run of its own (level pass, user sums + update, item sums +
update) and the level pass's us per level, and the compiled reference's serial _fit_sgd (oracle/_ref) on the same host
when importable.  The card's name and power limit are read in the run.
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

SHAPES = [("ml100k", 943, 1682, 100000, 3), ("ml1m", 6040, 3706, 1000000, 3), ("ml10m", 69878, 10677, 10000000, 1)]
K = 15                                                   # name, users, items, nnz, reference epochs


def synth_csr(n_users, n_items, nnz, seed, zipf=0.8):
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** zipf
    p /= p.sum()
    u = rng.randint(n_users, size=int(nnz * 1.3))
    i = rng.choice(n_items, size=len(u), p=p)
    key = np.unique(u.astype(np.int64) * n_items + i)
    if len(key) > nnz:
        key = np.sort(rng.choice(key, size=nnz, replace=False))
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    np.add.at(indptr, key // n_items + 1, 1)
    return np.cumsum(indptr).astype(np.int32), (key % n_items).astype(np.int32)


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


def phase_ms(fn, n_epochs):
    """Device time per epoch of each kernel family, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for tag in ("nmf_level_kernel", "nmf_user_kernel", "nmf_item_kernel"):
            if tag in ev.key:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[tag] = out.get(tag, 0.0) + t / 1e3 / n_epochs
    return out


def run_shape(name, n_users, n_items, nnz, ref_epochs, epochs, runs):
    import torch
    from cornac_b200 import engine
    indptr, indices = synth_csr(n_users, n_items, nnz, seed=1)
    rng = np.random.RandomState(2)
    val = rng.randint(1, 6, size=len(indices)).astype(np.float32)
    U0 = rng.uniform(0, 1, (n_users, K)).astype(np.float32)
    V0 = rng.uniform(0, 1, (n_items, K)).astype(np.float32)
    out = dict(n_users=n_users, n_items=n_items, nnz=len(indices), k=K,
               max_item_degree=int(np.bincount(indices).max()), max_user_degree=int(np.diff(indptr).max()))
    for use_bias in (False, True):
        mu = float(np.float32(val.mean())) if use_bias else 0.0
        t = time.perf_counter()
        data = engine.NmfData(indptr, indices, val, n_items, use_bias)
        torch.cuda.synchronize()
        res = dict(prepare_and_upload_s=time.perf_counter() - t, epochs=epochs)
        if use_bias:
            res["levels_per_epoch"] = data.n_levels
        d = [engine.to_device(a, torch.float32) for a in (U0, V0, np.zeros(n_users, np.float32),
                                                         np.zeros(n_items, np.float32))]
        work = torch.empty_like(d[0])
        fit = lambda n: engine.nmf_fit(data, *d, n, mu=mu, workspace=work)     # noqa: E731
        fit_s = cuda_median(lambda: fit(epochs), runs)
        res.update(fit_s=fit_s, ms_per_epoch=1e3 * fit_s / epochs)
        ph = phase_ms(lambda: fit(2), 2)
        res["phase_ms_per_epoch"] = ph
        if use_bias and data.n_levels:
            res["us_per_level"] = 1e3 * ph.get("nmf_level_kernel", float("nan")) / data.n_levels
        try:
            from cornac.models import NMF as RefNMF
            m = RefNMF(k=K, max_iter=ref_epochs, use_bias=use_bias, seed=1)
            m.num_users, m.num_items, m.global_mean = n_users, n_items, mu
            rid = np.repeat(np.arange(n_users, dtype=np.int32), np.diff(indptr))
            uc = np.diff(indptr).astype(np.int32)
            ic = np.bincount(indices, minlength=n_items).astype(np.int32)
            args = [U0.copy(), V0.copy(), np.zeros(n_users, np.float32), np.zeros(n_items, np.float32)]
            t = time.perf_counter()
            m._fit_sgd(rid, indices, val, uc, ic, *args)
            ref_s = time.perf_counter() - t
            res.update(reference_epochs=ref_epochs, reference_ms_per_epoch=1e3 * ref_s / ref_epochs,
                       speedup_per_epoch=(ref_s / ref_epochs) / (fit_s / epochs))
        except ImportError as e:
            res["reference"] = "not importable: %s" % e
        out["use_bias" if use_bias else "no_bias"] = res
        print(name, "use_bias=%s" % use_bias, json.dumps(res), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    from cornac_b200 import engine
    engine.warmup()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q, runs=a.runs, host_cpus=os.cpu_count(), cases={})
    print(res["gpu"], q, flush=True)
    for name, nu, ni, nnz, ref_ep in SHAPES:
        res["cases"][name] = run_shape(name, nu, ni, nnz, ref_ep, a.epochs, a.runs)
    os.makedirs(a.outdir, exist_ok=True)
    with open(os.path.join(a.outdir, "nmf_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
