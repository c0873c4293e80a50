"""Time the C2PF fit on seeded problems of the Amazon Office shape; write one JSON file.

    python tools/c2pf_bench.py OUTDIR [--iters 10] [--runs 5] [--shapes office,office10] [--ks 10,100] [--ref-iters 4]

Shapes (ratings 1-5, Zipf 0.8 item popularity, a symmetric context graph without self-loops): "office" is 3 703 users x
6 523 items x 53 282 ratings with 50 000 item pairs (100 000 stored edges; the output states the exact count), and
"office10" is ten times each.  For each shape, k in --ks and variant: the fit's ms per iteration with the second-phase
prior (CUDA events; --runs timed calls after a warm-up, the variants alternating within a run; median, min and max are
reported) and the device time per iteration of each kernel from torch.profiler in a run of its own.  At the "office"
shape it also times the compiled reference's c2pf_cpp (oracle/_ref, single-threaded, on the same host) at k = 10: a call
of c2pf.pyx with max_iter = --ref-iters (below 5 the second phase has no iteration), less a max_iter = 0 call that prices
its input conversion (the reference builds its sparse matrices entry by entry, twice per call of c2pf.pyx).  The card's name, power limit and clocks are read in the run.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "oracle", "_ref"))

from tools.hpf_bench import synth  # noqa: E402

SHAPES = {"office": (3703, 6523, 53282, 50000), "office10": (37030, 65230, 532820, 500000)}
VARIANTS = ("c2pf", "tc2pf", "rc2pf")
KERNELS = ("hpf_expect_kernel", "hpf_quotient_kernel", "hpf_colsum_kernel", "hpf_dk_kernel", "hpf_pass_kernel<true>",
           "hpf_pass_kernel<false>", "c2pf_add_kernel", "c2pf_lbu_kernel", "c2pf_sj_kernel", "c2pf_kappa_kernel",
           "c2pf_lb2_kernel", "c2pf_edge_sum_kernel", "c2pf_gr_terms_kernel", "c2pf_rate_kernel", "c2pf_context_kernel",
           "c2pf_edge_expect_kernel", "Memcpy")


def synth_graph(d, n_pairs, seed):
    """[2 * n_pairs', 3] triplets: both directions of distinct item pairs, value 1."""
    rng = np.random.RandomState(seed)
    a, b = rng.randint(d, size=(2, int(n_pairs * 1.05)))
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    key = np.unique(lo[lo != hi].astype(np.int64) * d + hi[lo != hi])[:n_pairs]
    a, b = key // d, key % d
    return np.column_stack([np.concatenate([a, b]), np.concatenate([b, a]), np.ones(2 * len(a))]).astype(np.float64)


def kernel_ms(fn, n_iter):
    """Device ms per iteration of each kernel, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for pat in KERNELS:
            if pat in ev.key:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[pat] = out.get(pat, 0.0) + t / 1e3 / n_iter
    return out


def reference_s_per_iter(rid, cid, val, n, d, C, k, iters):
    from cornac.models.c2pf import c2pf as cy
    tX = np.concatenate((np.stack([rid, cid]).T, val.astype(np.float32).reshape(-1, 1)), axis=1).astype(np.float64)
    ts = []
    for m in (0, iters):
        np.random.seed(1)
        t = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            cy.c2pf(tX, n, d, C, d, d, k, m, dict.fromkeys(("G_s", "G_r", "L_s", "L_r", "L2_s", "L2_r", "L3_s", "L3_r")))
        ts.append(time.perf_counter() - t)
    return (ts[1] - ts[0]) / iters, ts


def run_shape(name, ks, iters, runs, ref_iters):
    import torch
    from cornac_b200 import engine
    from cornac_b200.recom_c2pf import PHASE_TWO, ContextGraph
    n, d, nnz, n_pairs = SHAPES[name]
    rid, cid, val = synth(n, d, nnz, seed=1)
    C = synth_graph(d, n_pairs, seed=3)
    G = ContextGraph(C, d)
    dgraph = engine.C2pfGraph(engine.HpfData(rid, cid, val, n, d), G.ptr, G.row, G.mir, G.util)
    out = dict(n_users=n, n_items=d, nnz=len(val), n_edges=int(G.nnz), max_context_degree=int(np.diff(G.ptr).max()),
               cases={})
    rng = np.random.RandomState(2)
    for k in ks:
        fits = {}
        for v in VARIANTS:
            st = [engine.to_device(rng.gamma(100, 0.003, (rows, k)), torch.float64) for rows in (n, n, d, d, d, d)]
            st += [engine.to_device(rng.gamma(100, 0.005, G.nnz), torch.float64) for _ in range(2)]
            st += [torch.ones(d, dtype=torch.float64, device="cuda")]
            if v == "tc2pf":
                st[4] = st[5] = None
            if v == "rc2pf":
                st[2] = st[3] = None
            fits[v] = lambda m, v=v, st=st: engine.c2pf_fit(dgraph, v, *PHASE_TWO[v], st, m)      # noqa: E731
        ts = {v: [] for v in VARIANTS}
        for r in range(runs + 1):                              # run 0 warms up; the variants alternate within a run
            for v in VARIANTS:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fits[v](iters)
                b.record()
                b.synchronize()
                if r:
                    ts[v].append(a.elapsed_time(b) / iters)
        for v in VARIANTS:
            res = dict(iters=iters, ms_per_iter=float(np.median(ts[v])), ms_per_iter_min=float(min(ts[v])),
                       ms_per_iter_max=float(max(ts[v])), kernel_ms_per_iter=kernel_ms(lambda: fits[v](3), 3))
            if name == "office" and k == 10 and v == "c2pf" and ref_iters > 0:
                try:
                    ref, raw = reference_s_per_iter(rid, cid, val, n, d, C, k, ref_iters)
                    res.update(reference_iters=ref_iters, reference_s_per_iter=ref, reference_raw_s=raw,
                               speedup_per_iter=ref / (res["ms_per_iter"] / 1e3))
                except ImportError as e:
                    res["reference"] = "not importable: %s" % e
            out["cases"]["%s_k%d" % (v, k)] = res
            print(name, v, k, json.dumps(res), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--shapes", default="office,office10")
    ap.add_argument("--ks", default="10,100")
    ap.add_argument("--ref-iters", type=int, default=4)
    a = ap.parse_args()
    import torch
    from cornac_b200 import engine
    engine.warmup()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q, runs=a.runs, host_cpus=os.cpu_count(), shapes={})
    print(res["gpu"], q, flush=True)
    ks = [int(x) for x in a.ks.split(",")]
    for name in a.shapes.split(","):
        res["shapes"][name] = run_shape(name, ks, a.iters, a.runs, a.ref_iters)
    os.makedirs(a.outdir, exist_ok=True)
    with open(os.path.join(a.outdir, "c2pf_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
