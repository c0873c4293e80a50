"""Time the UserKNN / ItemKNN kernels and plug-ins on seeded rating matrices; write one JSON file.

    python tools/knn_bench.py OUTDIR [--runs 5] [--skip-large]

Shapes: an ML-1M shape (6040 x 3706 x 1 000 209, ratings 1-5, Zipf 0.8 item popularity) for ItemKNN and UserKNN, a
larger ItemKNN (100 K users x 20 K items x 10 M: a 3.2 GB dense similarity) and a UserKNN on 30 K users.  Kernel times
are CUDA-event medians of --runs runs after a warm-up; fit() / transform() are host-clock times ending in a device
synchronise.  On the ML-1M shape the compiled reference's compute_similarity (all host threads) and compute_score
(users/s over 100 users) are timed too when it is importable (oracle/_ref).
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


def synth(n_users, n_items, nnz, seed, zipf=0.8):
    import scipy.sparse as sp
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** zipf
    p /= p.sum()
    key = np.unique(rng.randint(n_users, size=int(nnz * 1.4)).astype(np.int64) * n_items
                    + rng.choice(n_items, size=int(nnz * 1.4), p=p))
    key = np.sort(rng.choice(key, size=min(nnz, len(key)), replace=False))
    r = rng.randint(1, 6, size=len(key)).astype(np.float64)
    return sp.csr_matrix((r, (key // n_items, key % n_items)), shape=(n_users, n_items))


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


class _DS:
    """The attributes of cornac.data.Dataset that the plug-ins' fit() reads."""

    def __init__(self, X):
        self.matrix = X
        self.num_users, self.num_items = X.shape
        self.total_users, self.total_items = X.shape
        self.min_rating, self.max_rating = float(X.data.min()), float(X.data.max())
        self.global_mean = float(X.data.mean())
        self.uid_map = {str(u): u for u in range(X.shape[0])}
        self.iid_map = {str(i): i for i in range(X.shape[1])}
        rows = np.repeat(np.arange(X.shape[0]), np.diff(X.indptr))
        self.uir_tuple = (rows, X.indices, X.data)

    def reset(self):
        return self


def run_case(name, cls_name, X, runs, reference=False):
    import torch
    import cornac_b200
    from cornac_b200 import engine
    from cornac_b200.recom_knn import _mean_centered
    user_mode = cls_name == "UserKNN"
    ui, mean = _mean_centered(X.copy())
    W = X if user_mode else X.T.tocsr()                      # cosine on the raw ratings
    cols = W.T.tocsr()
    n = W.shape[0]
    madds = int(np.sum(np.diff(cols.indptr).astype(np.int64) ** 2))
    out = dict(model=cls_name, n_users=X.shape[0], n_items=X.shape[1], nnz=int(X.nnz), k=20,
               sum_deg_sq_madds=madds, dense_bytes=n * n * 8)
    S_holder = {}

    def sim():
        S_holder["S"], S_holder["sim"] = engine.knn_similarity(W, 1.0)
    # similarity call = kernel + mirror + count + compaction + copies; the kernel time is taken from the profiler below
    out["similarity_call_s"] = cuda_median(sim, runs)
    S = S_holder["S"]
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sim()
        torch.cuda.synchronize()
    ks = {e.key: e.device_time_total / 1e6 for e in prof.key_averages() if "knn_" in e.key}
    out["kernel_s"] = ks
    out["sim_nnz"] = int(S_holder["sim"].nnz)
    R = engine.KnnRatings(ui.T.tocsr() if user_mode else ui, mean)
    users = np.arange(min(X.shape[0], 6040), dtype=np.int64)     # every user of the ML-1M shape, a sample of larger ones
    batch = max(1, (1 << 30) // (8 * X.shape[1]))

    def score_all():
        for b0 in range(0, len(users), batch):
            engine.knn_score(user_mode, S, users[b0:b0 + batch], R, 20)
    out["score_users"] = len(users)
    out["score_s"] = cuda_median(score_all, runs)
    out["score_users_per_s"] = len(users) / out["score_s"]
    del S, S_holder
    torch.cuda.empty_cache()
    ds = _DS(X)
    m = getattr(cornac_b200, cls_name)(k=20, verbose=False)
    t0 = time.perf_counter()
    m.fit(ds)
    torch.cuda.synchronize()
    out["fit_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    m.transform(ds)
    out["transform_s"] = time.perf_counter() - t0
    out["transform_cached"] = m._b200_eval_cache is not None
    del m
    torch.cuda.empty_cache()
    if reference:
        try:
            from cornac.models.knn.similarity import compute_score, compute_similarity
        except Exception as e:                              # the reference install is optional
            out["reference"] = "not importable: %s" % e
            return out
        threads = os.cpu_count()
        t0 = time.perf_counter()
        ref = compute_similarity(W, num_threads=threads, verbose=False)
        out["reference_similarity_s"] = time.perf_counter() - t0
        out["reference_threads"] = threads
        dense_row = np.zeros(n)
        sample = users[:100]
        t0 = time.perf_counter()
        for u in sample:
            o = np.zeros(X.shape[1])
            if user_mode:
                iu = ui.T.tocsr()
                dense_row[:] = ref[u].toarray().ravel()
                compute_score(True, dense_row, iu.indptr, iu.indices, iu.data, k=20, num_threads=threads, output=o)
            else:
                compute_score(False, ui[u].toarray().ravel(), ref.indptr, ref.indices, ref.data, k=20, num_threads=threads,
                              output=o)
        out["reference_score_users_per_s"] = len(sample) / (time.perf_counter() - t0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--skip-large", action="store_true")
    a = ap.parse_args()
    import torch
    from cornac_b200 import engine
    engine.warmup()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q, runs=a.runs, cases={})
    ml1m = synth(6040, 3706, 1000209, seed=1)
    res["cases"]["ml1m_itemknn"] = run_case("ml1m_itemknn", "ItemKNN", ml1m, a.runs, reference=True)
    res["cases"]["ml1m_userknn"] = run_case("ml1m_userknn", "UserKNN", ml1m, a.runs, reference=True)
    if not a.skip_large:
        res["cases"]["itemknn_100k_20k"] = run_case("itemknn_100k_20k", "ItemKNN", synth(100000, 20000, 10000000, seed=2), a.runs)
        res["cases"]["userknn_30k"] = run_case("userknn_30k", "UserKNN", synth(30000, 5000, 2000000, seed=3), a.runs)
    os.makedirs(a.outdir, exist_ok=True)
    with open(os.path.join(a.outdir, "knn_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
