"""Time the EFM fit and its aspect-weighted rank on seeded shapes; write one JSON file.

    python tools/efm_bench.py OUTDIR [--iters 20] [--runs 3]

Shapes (E = 40, L = 60, ratings 1-5, Zipf 0.8 item popularity, 200 aspects, 3 sentiment tuples per rating): the ML-1M
rating shape (6040 x 3706 x 1 000 000) and ten times it (60 400 x 37 060 x 10 000 000).  For each: the fit's ms per
iteration (CUDA events, median of --runs after a warm-up); the device time per iteration of the prediction kernel and of
the update launch, which runs the aspect, item and user passes together (torch.profiler); rank throughput (users/s, top-10, seen items excluded,
queries included); and at the small shape the compiled reference's serial _fit_efm (oracle/_ref) when importable.
The card's name and power limit are read in the run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "oracle", "_ref"))

SHAPES = [("ml1m", 6040, 3706, 1000000, True), ("ml1m_x10", 60400, 37060, 10000000, False)]
E, L, N_ASPECTS, TUPLES = 40, 60, 200, 3


def synth(n_users, n_items, nnz, seed):
    """(A, X, Y) CSR matrices of a seeded rating set with TUPLES sentiment tuples per rating over N_ASPECTS aspects
    (X, Y values in the reference's ranges; their exact formula does not change the work)."""
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** 0.8
    p /= p.sum()
    u = rng.randint(n_users, size=int(nnz * 1.3))
    i = rng.choice(n_items, size=len(u), p=p)
    key = np.unique(u.astype(np.int64) * n_items + i)
    if len(key) > nnz:
        key = np.sort(rng.choice(key, size=nnz, replace=False))
    uu, ii = key // n_items, key % n_items
    A = sp.csr_matrix((rng.randint(1, 6, size=len(key)).astype(np.float32), (uu, ii)), shape=(n_users, n_items))
    pa = 1.0 / np.arange(1, N_ASPECTS + 1) ** 0.7
    asp = rng.choice(N_ASPECTS, size=(len(key), TUPLES), p=pa / pa.sum())
    ua = np.unique(np.repeat(uu, TUPLES) * N_ASPECTS + asp.ravel())
    ia = np.unique(np.repeat(ii, TUPLES) * N_ASPECTS + asp.ravel())
    X = sp.csr_matrix((rng.uniform(1, 5, len(ua)).astype(np.float32), (ua // N_ASPECTS, ua % N_ASPECTS)),
                      shape=(n_users, N_ASPECTS))
    Y = sp.csr_matrix((rng.uniform(1, 5, len(ia)).astype(np.float32), (ia // N_ASPECTS, ia % N_ASPECTS)),
                      shape=(n_items, N_ASPECTS))
    return A, X, Y


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


def phase_ms(fn, n_iter):
    """Device time per iteration of each EFM kernel, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for tag in ("efm_pred_kernel", "efm_pass_kernel"):
            if tag in ev.key:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[tag] = out.get(tag, 0.0) + t / 1e3 / n_iter
    return out


def run_shape(name, n_users, n_items, nnz, with_ref, iters, runs):
    import torch
    from cornac_b200 import engine
    A, X, Y = synth(n_users, n_items, nnz, seed=1)
    rng = np.random.RandomState(2)
    high = np.sqrt(5.0 / (E + L))
    init = [rng.uniform(0, high, s).astype(np.float32)
            for s in ((n_users, E), (n_items, E), (N_ASPECTS, E), (n_users, L), (n_items, L))]
    out = dict(n_users=n_users, n_items=n_items, nnz_A=A.nnz, nnz_X=X.nnz, nnz_Y=Y.nnz, E=E, L=L, n_aspects=N_ASPECTS,
               longest_aspect_chain=int((X.getnnz(axis=0) + Y.getnnz(axis=0)).max()), iters=iters)
    t = time.perf_counter()
    data = engine.EfmData(A, X, Y)
    torch.cuda.synchronize()
    out["prepare_and_upload_s"] = time.perf_counter() - t
    d = [engine.to_device(x, torch.float32) for x in init]
    work = torch.empty(engine.efm_workspace_floats(n_users, n_items, N_ASPECTS, E, L), dtype=torch.float32, device="cuda")
    fit = lambda n: engine.efm_fit(data, *d, n, workspace=work)          # noqa: E731
    fit_s = cuda_median(lambda: fit(iters), runs)
    out.update(fit_s=fit_s, ms_per_iter=1e3 * fit_s / iters, phase_ms_per_iter=phase_ms(lambda: fit(2), 2))
    # rank throughput: queries + fused top-10 with the training items excluded
    from cornac_b200.recom_efm import EFM
    model = EFM(num_explicit_factors=E, num_latent_factors=L, trainable=False)
    model.U1, model.U2, model.V, model.H1, model.H2 = [x.cpu().numpy() for x in d]
    model.num_users, model.num_items, model.num_aspects = n_users, n_items, N_ASPECTS
    users = np.arange(n_users)

    def rank_all():
        model._b200_invalidate()
        model.rank_batch(users, 10, exclude=A)
    rank_s = cuda_median(rank_all, runs)
    out.update(rank_s=rank_s, rank_users_per_s=n_users / rank_s)
    if with_ref:
        try:
            from cornac.models import EFM as RefEFM
            m = RefEFM(num_explicit_factors=E, num_latent_factors=L, max_iter=1, seed=1)
            m.num_users, m.num_items, m.num_aspects = n_users, n_items, N_ASPECTS
            args = [x.copy() for x in init]
            cnt = lambda M, ax: np.asarray(M.getnnz(axis=ax), dtype=np.int32)       # noqa: E731
            rows = lambda M: np.repeat(np.arange(M.shape[0], dtype=np.int32), np.diff(M.indptr))   # noqa: E731
            t = time.perf_counter()
            m._fit_efm(1, A.data, rows(A), A.indices, cnt(A, 1), cnt(A, 0), X.data, rows(X), X.indices, cnt(X, 1),
                       cnt(X, 0), Y.data, rows(Y), Y.indices, cnt(Y, 1), cnt(Y, 0), *args)
            ref_s = time.perf_counter() - t
            out.update(reference_ms_per_iter=1e3 * ref_s, speedup_per_iter=ref_s / (fit_s / iters))
        except ImportError as e:
            out["reference"] = "not importable: %s" % e
    print(name, json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    from cornac_b200 import engine
    engine.warmup()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q, runs=a.runs, host_cpus=os.cpu_count(), cases={})
    print(res["gpu"], q, flush=True)
    for name, nu, ni, nnz, with_ref in SHAPES:
        res["cases"][name] = run_shape(name, nu, ni, nnz, with_ref, a.iters, a.runs)
    os.makedirs(a.outdir, exist_ok=True)
    with open(os.path.join(a.outdir, "efm_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
