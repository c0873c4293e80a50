"""LRPPM on the GPU: fit milliseconds per iteration (with the phase split) and rank users per second.

    python tools/lrppm_bench.py [--out DIR]

Shapes: a synthetic train set the size of the Amazon Toys data of examples/lrppm_example.py (19 412 users, 11 924 items,
167 597 ratings, 200 aspects) and ten times its users, items and ratings, with the reference's defaults (k = 8,
n_samples = 200, n_ranking_samples = 1000).  The fit runs a fixed number of iterations from uploaded draws with a small
lr, which keeps the parameters moving, so no iteration converges.  Prints one JSON line with the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "oracle", "_ref"))        # cornac, for the plug-in module's imports


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:                   # noqa: BLE001
        return "unknown (%s)" % e


def synth(n_users, n_items, nnz, n_aspects, seed):
    from cornac_b200.engine import LrppmData
    from cornac_b200.recom_lrppm import get_key, get_key3
    rng = np.random.RandomState(seed)
    key = np.unique(rng.randint(0, n_users * n_items, size=int(nnz * 1.1)))[:nnz]
    rng.shuffle(key)
    u, i = (key // n_items).astype(np.int32), (key % n_items).astype(np.int32)
    r = rng.randint(1, 6, size=len(key)).astype(np.float32)
    rev = rng.rand(len(key)) < 0.8
    n_t = rng.randint(1, 5, size=rev.sum())
    xu, xi = np.repeat(u[rev], n_t), np.repeat(i[rev], n_t)
    xa = rng.randint(0, n_aspects, size=len(xu))
    trip = np.unique((xu.astype(np.int64) * n_items + xi) * n_aspects + xa)
    xu, xi, xa = (trip // n_aspects // n_items).astype(np.int32), (trip // n_aspects % n_items).astype(np.int32), \
        (trip % n_aspects).astype(np.int32)
    rk = get_key(u, i)
    order = np.unique(rk, return_index=True)[1]
    return LrppmData(n_users=n_users, n_items=n_items, n_aspects=n_aspects, u_indices=u, i_indices=i, r_values=r,
                     X_uids=xu, X_iids=xi, X_aids=xa, X_l_ui=np.full(len(xu), 0.01, np.float32),
                     aspect_keys=np.unique(get_key3(xu, xi, xa)).astype(np.int32),
                     rating_keys=rk[order].astype(np.int32), rating_values=r[order])


def bench_fit(d, n_iter, k=8, n_s=200, n_r=1000):
    import torch
    from cornac_b200 import engine
    dd = engine.LrppmDeviceData(d)
    rng = np.random.RandomState(0)
    params = [torch.from_numpy(rng.uniform(0, 1, (n, k)).astype(np.float32)).cuda()
              for n in (d.n_users, d.n_items, d.n_aspects, d.n_aspects)]
    work = torch.zeros(engine.lrppm_workspace_bytes(dd, k, n_s, n_r), dtype=torch.uint8, device="cuda")
    dr = np.concatenate([rng.randint(0, len(d.r_values), (n_iter, n_s)), rng.randint(0, len(d.X_uids), (n_iter, n_r)),
                         rng.randint(0, d.n_aspects, (n_iter, n_r))], axis=1).astype(np.int32)
    draws = torch.from_numpy(dr).cuda()
    counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    phase = torch.zeros(3, dtype=torch.int64, device="cuda")
    kw = dict(lr=1e-3, reg=0.01, ld=1.0, counts=counts, workspace=work)
    engine.lrppm_fit(dd, params, draws, 10, n_s, n_r, **kw)
    torch.cuda.synchronize()
    counts.zero_()
    t0 = time.perf_counter()
    engine.lrppm_fit(dd, params, draws, n_iter, n_s, n_r, phase_ns=phase, **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    ran = int(counts[2].item())
    ph = (phase.cpu().numpy() / 1e6 / max(ran, 1)).tolist()
    return dict(iterations=ran, ms_per_iter=1e3 * dt / max(ran, 1), phase_ms=dict(zip(("predict", "del", "step"), ph)))


def bench_rank(d, n_top, k=8, n_users=4096):
    import scipy.sparse as sp
    import torch
    from cornac_b200 import engine
    rng = np.random.RandomState(1)
    dv = lambda x: torch.from_numpy(x).cuda()                                         # noqa: E731
    U, I = dv(rng.uniform(0, 1, (d.n_users, k)).astype(np.float32)), dv(rng.uniform(0, 1, (d.n_items, k)).astype(np.float32))
    UA, IA = (dv(rng.uniform(0, 1, (d.n_aspects, k)).astype(np.float32)) for _ in range(2))
    Q = sp.random(d.n_items, d.n_aspects, density=0.05, random_state=2, format="csr")
    q = engine.LrppmQuality(Q)
    users = dv(np.arange(n_users, dtype=np.int64) % d.n_users)
    rows = engine.lrppm_rank_rows(U, I, UA, IA, q, users[:256], n_top, 1.0, 5.0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in range(0, n_users, 256):
        rows = engine.lrppm_rank_rows(U, I, UA, IA, q, users[b:b + 256], n_top, 1.0, 5.0, out=rows)
        engine.topk_rows_f64(rows, 10)
    torch.cuda.synchronize()
    return n_users / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from cornac_b200 import engine
    engine.warmup()
    res = dict(card=card())
    for tag, scale in (("toys", 1), ("toys_x10", 10)):
        d = synth(19412 * scale, 11924 * scale, 167597 * scale, 200, 7)
        res["fit_" + tag] = bench_fit(d, a.iters)
        res["rank_users_per_s_" + tag] = dict(all=bench_rank(d, 200), top10=bench_rank(d, 10))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lrppm_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
