"""Time the SoRec / MCF co-factor fit on seeded synthetic shapes; write one JSON file.

    python tools/cofactor_bench.py OUTDIR [--epochs 20] [--runs 3]

Shapes (k = 10, ratings 1-5 scaled to [0, 1], Zipf 0.8 item popularity, ratings and edges in shuffled order):
  filmtrust  SoRec, 1 508 users x 2 071 items x 35 497 ratings, 1 853 trust edges
  epinions   SoRec, 49 290 users x 139 738 items x 664 824 ratings, 487 181 trust edges
  mcf_ft     MCF on the filmtrust ratings with an item graph of 2 540 edges (the trust graph's edges per node)
  mcf_ep     MCF on the epinions ratings with an item graph of 1 381 087 edges (the same density)
Graph edges join distinct nodes, with Zipf 0.8 popularity of the target node.  For each shape: the level count of the
mixed schedule, how many edge and rating slots there are, the schedule's host time, the fit's CUDA-event time (median of
--runs after a warm-up) and its ms per epoch.  The compiled reference's sorec / mcf loop (oracle/_ref) is timed on the
same host when importable.  The card's name and power limit are read in the run.
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

SHAPES = [("filmtrust", "sorec", 1508, 2071, 35497, 1853), ("epinions", "sorec", 49290, 139738, 664824, 487181),
          ("mcf_ft", "mcf", 1508, 2071, 35497, 2540), ("mcf_ep", "mcf", 49290, 139738, 664824, 1381087)]


def _zipf(n, zipf=0.8):
    p = 1.0 / np.arange(1, n + 1) ** zipf
    return p / p.sum()


def synth(variant, n_users, n_items, n_ratings, n_edges, seed, order="shuffled"):
    """(net_a, net_b, net_val, uid, iid, rat): unique ratings in [0, 1] and unique edges between distinct nodes (users for
    "sorec", items for "mcf"), in shuffled stored order, or sorted by (row, column) with order="csr"."""
    rng = np.random.RandomState(seed)
    key = np.unique(rng.randint(n_users, size=int(n_ratings * 1.4)).astype(np.int64) * n_items
                    + rng.choice(n_items, size=int(n_ratings * 1.4), p=_zipf(n_items)))
    key = rng.choice(key, size=min(n_ratings, len(key)), replace=False)
    n = n_users if variant == "sorec" else n_items
    ek = rng.randint(n, size=int(n_edges * 1.4)).astype(np.int64) * n + rng.choice(n, size=int(n_edges * 1.4), p=_zipf(n))
    ek = np.unique(ek[ek // n != ek % n])
    ek = rng.choice(ek, size=min(n_edges, len(ek)), replace=False)
    if order == "csr":
        key, ek = np.sort(key), np.sort(ek)
    rat = (rng.randint(1, 6, size=len(key)).astype(np.float32) - np.float32(1)) / np.float32(4)
    net_val = np.ones(len(ek), dtype=np.float32)
    return ((ek // n).astype(np.int32), (ek % n).astype(np.int32), net_val, (key // n_items).astype(np.int32),
            (key % n_items).astype(np.int32), rat)


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


def run_shape(name, variant, n_users, n_items, n_ratings, n_edges, epochs, runs, ref_epochs):
    import torch
    from cornac_b200 import engine
    net_a, net_b, net_val, uid, iid, rat = synth(variant, n_users, n_items, n_ratings, n_edges, seed=1)
    out = dict(model=variant, n_users=n_users, n_items=n_items, n_ratings=len(uid), n_edges=len(net_a), k=10)
    t = time.perf_counter()
    data = engine.CofactorData(variant, net_a, net_b, net_val, uid, iid, rat, n_users, n_items)
    torch.cuda.synchronize()
    out["schedule_and_upload_s"] = time.perf_counter() - t
    order, level_ptr = engine.cofactor_schedule(variant, net_a, net_b, uid, iid, n_users, n_items)
    edge_slot = order < len(net_a)
    per_level_edges = np.add.reduceat(edge_slot.astype(np.int64), level_ptr[:-1]) if len(order) else np.zeros(0)
    out.update(levels_per_epoch=data.n_levels, mean_level_width=len(order) / max(1, data.n_levels),
               edge_slots=int(edge_slot.sum()), rating_slots=int((~edge_slot).sum()),
               levels_with_edges=int((per_level_edges > 0).sum()),
               levels_with_ratings=int((per_level_edges < np.diff(level_ptr)).sum()),
               levels_rating_pass_alone=int(engine.PmfData(uid, iid, rat, n_users, n_items).n_levels))
    rng = np.random.RandomState(2)
    n_z = n_users if variant == "sorec" else n_items
    U0, V0, Z0 = (rng.normal(0, 0.001, (n, 10)) for n in (n_users, n_items, n_z))
    dev = [engine.to_device(x, torch.float64) for x in (U0, V0, Z0)]
    caches = [torch.zeros_like(x) for x in dev]
    fit_s = cuda_median(lambda: engine.cofactor_fit(data, *dev, *caches, epochs, 10.0, 0.001, 0.001, 0.9), runs)
    out.update(epochs=epochs, fit_s=fit_s, ms_per_epoch=1e3 * fit_s / epochs)
    try:
        if variant == "sorec":
            from cornac.models.sorec import sorec as cy
            kw = dict(lambda_c=10.0, lambda_reg=0.001)
        else:
            from cornac.models.mcf import mcf as cy
            kw = dict(lamda=0.001)
        fn = getattr(cy, variant)
        t = time.perf_counter()
        fn(uid, iid, rat, net_a, net_b, net_val, k=10, n_users=n_users, n_items=n_items, n_ratings=len(uid),
           n_edges=len(net_a), n_epochs=ref_epochs, learning_rate=0.001, gamma=0.9,
           init_params={"U": U0.copy(), "V": V0.copy(), "Z": Z0.copy()}, seed=1, **kw)
        ref_s = time.perf_counter() - t
        out.update(reference_epochs=ref_epochs, reference_s=ref_s, reference_ms_per_epoch=1e3 * ref_s / ref_epochs,
                   speedup_per_epoch=(ref_s / ref_epochs) / (fit_s / epochs))
    except ImportError as e:
        out["reference"] = "not importable: %s" % e
    print(name, json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--ref-epochs", type=int, default=3)
    a = ap.parse_args()
    import torch
    from cornac_b200 import engine
    engine.warmup()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q, runs=a.runs, host_cpus=os.cpu_count(), cases={})
    print(res["gpu"], q, flush=True)
    for name, variant, nu, ni, nr, ne in SHAPES:
        res["cases"][name] = run_shape(name, variant, nu, ni, nr, ne, a.epochs, a.runs, a.ref_epochs)
    os.makedirs(a.outdir, exist_ok=True)
    with open(os.path.join(a.outdir, "cofactor_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
