"""Time the HPF / PF fit on seeded rating sets; write one JSON file.

    python tools/hpf_bench.py OUTDIR [--iters 10] [--runs 3] [--shapes ml1m,ml10m,ml20m] [--ks 5,10,50] [--ref-iters 1]

Shapes (ratings 1-5, Zipf 0.8 item popularity): ML-1M (6040 x 3706 x 1 000 000), ML-10M (69 878 x 10 677 x 10 000 000)
and ML-20M (138 493 x 26 744 x 20 000 000), k in --ks, both variants.  For each: the fit's ms per iteration (CUDA events,
median of --runs after a warm-up) and the device time per iteration of each kernel from torch.profiler in a run of its
own.  At the ML-1M shape with k = 10 it also times the compiled reference's hpf_cpp (oracle/_ref, single-threaded, on
the same host) for --ref-iters iterations, less a 0-iteration call that prices its input conversion.  The card's name
and power limit are read in the run.
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

SHAPES = {"ml1m": (6040, 3706, 1000000), "ml10m": (69878, 10677, 10000000), "ml20m": (138493, 26744, 20000000)}
KERNELS = (("expect", "hpf_expect_kernel"), ("quotient", "hpf_quotient_kernel"), ("colsum", "hpf_colsum_kernel"),
           ("dk", "hpf_dk_kernel"), ("user_pass", "hpf_pass_kernel<true>"), ("item_pass", "hpf_pass_kernel<false>"),
           ("rate", "hpf_rate_kernel"))


def synth(n_users, n_items, nnz, seed, zipf=0.8):
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** zipf
    p /= p.sum()
    u = rng.randint(n_users, size=int(nnz * 1.3))
    i = rng.choice(n_items, size=len(u), p=p)
    key = np.unique(u.astype(np.int64) * n_items + i)
    if len(key) > nnz:
        key = np.sort(rng.choice(key, size=nnz, replace=False))
    val = rng.randint(1, 6, size=len(key)).astype(np.float64)
    return (key // n_items).astype(np.int32), (key % n_items).astype(np.int32), val


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


def kernel_ms(fn, n_iter):
    """Device ms per iteration of each kernel family, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for tag, pat in KERNELS:
            if pat in ev.key:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[tag] = out.get(tag, 0.0) + t / 1e3 / n_iter
    return out


def reference_s_per_iter(rid, cid, val, n, d, k, iters):
    from cornac.models.hpf import hpf as cy
    tX = np.concatenate((np.stack([rid, cid]).T, val.astype(np.float32).reshape(-1, 1)), axis=1)
    ts = []
    for m in (0, iters):
        t = time.perf_counter()
        cy.hpf(tX, n, d, k, m, 1, {"G_s": None, "G_r": None, "L_s": None, "L_r": None})
        ts.append(time.perf_counter() - t)
    return (ts[1] - ts[0]) / iters, ts


def run_shape(name, ks, iters, runs, ref_iters):
    import torch
    from cornac_b200 import engine
    n, d, nnz = SHAPES[name]
    rid, cid, val = synth(n, d, nnz, seed=1)
    t = time.perf_counter()
    data = engine.HpfData(rid, cid, val, n, d)
    torch.cuda.synchronize()
    out = dict(n_users=n, n_items=d, nnz=len(val), prepare_and_upload_s=time.perf_counter() - t,
               max_item_degree=int(np.bincount(cid).max()), max_user_degree=int(np.bincount(rid).max()), cases={})
    rng = np.random.RandomState(2)
    for k in ks:
        for hier in (True, False):
            sh, sc = (100.0, 0.003) if hier else (0.3, 1 / 0.3)
            init = [rng.gamma(sh, sc, (n, k)), rng.gamma(sh, sc, (n, k)), rng.gamma(sh, sc, (d, k)),
                    rng.gamma(sh, sc, (d, k))]
            st = [engine.to_device(a, torch.float64) for a in init]
            Kr = torch.ones(n, dtype=torch.float64, device="cuda")
            Tr = torch.ones(d, dtype=torch.float64, device="cuda")
            fit = lambda m: engine.hpf_fit(data, hier, *st, Kr, Tr, m)      # noqa: E731
            fit_s = cuda_median(lambda: fit(iters), runs)
            res = dict(iters=iters, ms_per_iter=1e3 * fit_s / iters, kernel_ms_per_iter=kernel_ms(lambda: fit(3), 3))
            if name == "ml1m" and k == 10 and hier and ref_iters > 0:
                try:
                    ref, raw = reference_s_per_iter(rid, cid, val, n, d, k, ref_iters)
                    res.update(reference_iters=ref_iters, reference_s_per_iter=ref, reference_raw_s=raw,
                               speedup_per_iter=ref / (fit_s / iters))
                except ImportError as e:
                    res["reference"] = "not importable: %s" % e
            key = "%s_k%d" % ("hpf" if hier else "pf", k)
            out["cases"][key] = res
            print(name, key, json.dumps(res), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--shapes", default="ml1m,ml10m,ml20m")
    ap.add_argument("--ks", default="5,10,50")
    ap.add_argument("--ref-iters", type=int, default=1)
    a = ap.parse_args()
    import torch
    from cornac_b200 import engine
    engine.warmup()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q, runs=a.runs, host_cpus=os.cpu_count(), shapes={})
    print(res["gpu"], q, flush=True)
    ks = [int(x) for x in a.ks.split(",")]
    for name in a.shapes.split(","):
        res["shapes"][name] = run_shape(name, ks, a.iters, a.runs, a.ref_iters)
    os.makedirs(a.outdir, exist_ok=True)
    with open(os.path.join(a.outdir, "hpf_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
