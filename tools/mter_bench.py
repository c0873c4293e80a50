"""MTER fit and rank timing on seeded synthetic data (not bench.py's workload).

    python tools/mter_bench.py [--iters 20] [--out mter_bench.json]

Shapes: the ML-1M rating shape (6 040 users x 3 706 items, 1 M ratings) and ten times it, with 200 aspects, 100
opinions and 3 sentiment tuples per rating; the reference's defaults otherwise (15/15/12/12 factors, 50 element and
1 000 BPR samples per iteration).  Reports, per shape: the exact (seeded) fit and the unordered (unseeded, Philox) fit in ms per
iteration (CUDA events, median of 5 calls of --iters iterations each); the exact fit's time per phase (the kernel's
own global-timer marks at its grid barriers, as block 0 sees them); the rank rate (top-10, seen items excluded) in
users/s.  At the ML-1M shape it also times the compiled reference's `_fit_mter` over --ref-iters iterations when the
reference install under oracle/_ref is present: seeded (one thread) and unseeded on every host thread.  Prints one JSON
line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cornac_b200 import engine  # noqa: E402


def synth(n_users, n_items, nnz, n_aspects, n_opinions, seed):
    rng = np.random.RandomState(seed)
    key = np.unique(rng.randint(0, n_users * n_items, size=int(nnz * 1.02)).astype(np.int64))[:nnz]
    u, i = (key // n_items).astype(np.int32), (key % n_items).astype(np.int32)
    nx, ny = 3 * len(key), 2 * len(key)
    ri = lambda hi, n: rng.randint(0, hi, n).astype(np.int32)       # noqa: E731
    return engine.MterData(n_users=n_users, n_items=n_items, n_aspects=n_aspects, n_opinions=n_opinions,
                    X=rng.uniform(1, 5, nx).astype(np.float32), X_uids=ri(n_users, nx), X_iids=ri(n_items, nx),
                    X_aids=ri(n_aspects + 1, nx), YU=rng.uniform(1, 5, ny).astype(np.float32), YU_uids=ri(n_users, ny),
                    YU_aids=ri(n_aspects, ny), YU_oids=ri(n_opinions, ny), YI=rng.uniform(1, 5, ny).astype(np.float32),
                    YI_iids=ri(n_items, ny), YI_aids=ri(n_aspects, ny), YI_oids=ri(n_opinions, ny),
                    indptr=np.concatenate([[0], np.cumsum(np.bincount(u, minlength=n_users))]).astype(np.int32),
                    indices=i, user_ids=u, pair_rating=rng.randint(1, 6, len(key)).astype(np.float32))


def run(name, data, iters, dims=(15, 15, 12, 12), n_el=50, n_bpr=1000):
    d1, d2, d3, d4 = dims
    rng = np.random.RandomState(1)
    shapes = ((data.n_users, d1), (data.n_items, d2), (data.n_aspects + 1, d3), (data.n_opinions, d4), (d1, d2, d3),
              (d1, d3, d4), (d2, d3, d4))
    dd = engine.MterDeviceData(data)
    params = [torch.from_numpy(rng.uniform(0, 1, s).astype(np.float32)).cuda() for s in shapes]
    sgrad = [torch.zeros_like(x) for x in params]
    work = torch.zeros(engine.mter_workspace_bytes(dd, dims, n_el, n_bpr), dtype=torch.uint8, device="cuda")
    draws = engine.MterDraws([11, 12, 13, 14, 15], data, n_el, n_bpr, iters)
    dev = draws.next(iters).clone()
    t0 = time.perf_counter()
    draws.draw(iters)
    host_ms = (time.perf_counter() - t0) * 1e3 / iters

    def timed(fit):
        fit()
        torch.cuda.synchronize()
        times = []
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fit()
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) / iters)
        return times

    times = timed(lambda: engine.mter_fit(dd, params, sgrad, dev, iters, n_el, n_bpr, workspace=work))
    phase = torch.zeros(4, dtype=torch.int64, device="cuda")
    engine.mter_fit(dd, params, sgrad, dev, iters, n_el, n_bpr, workspace=work, phase_ns=phase)
    names = ("predictions", "owners_and_stored_terms", "gradients", "adagrad")
    phases = {k: v / 1e6 / iters for k, v in zip(names, phase.cpu().tolist())}
    un = timed(lambda: engine.mter_fit(dd, params, sgrad, None, iters, n_el, n_bpr, workspace=work, unordered=True,
                                       philox_seed=99))
    uphase = torch.zeros(4, dtype=torch.int64, device="cuda")
    engine.mter_fit(dd, params, sgrad, None, iters, n_el, n_bpr, workspace=work, unordered=True, philox_seed=99,
                    phase_ns=uphase)
    uphases = {k: v / 1e6 / iters for k, v in zip(names, uphase.cpu().tolist()) if k != "owners_and_stored_terms"}
    # rank: Q = U . (G1 . A[-1]), then the shared fused top-10 with seen items excluded
    Q = engine.mter_queries(params[0], params[4], params[2])
    users = np.arange(data.n_users, dtype=np.int64)
    ex_ptr = torch.from_numpy(data.indptr.astype(np.int64)).cuda()
    ex_idx = torch.from_numpy(data.indices.astype(np.int32)).cuda()
    engine.rank_topk(Q, params[1], 10, user_idx=torch.from_numpy(users).cuda(), excl_indptr=ex_ptr, excl_indices=ex_idx)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
        engine.rank_topk(Q, params[1], 10, user_idx=torch.from_numpy(users).cuda(), excl_indptr=ex_ptr,
                         excl_indices=ex_idx)
    torch.cuda.synchronize()
    rank_rate = 3 * len(users) / (time.perf_counter() - t0)
    return dict(shape=name, exact_ms_per_iter_median=float(np.median(times)), exact_ms_per_iter_min=float(min(times)),
                exact_ms_per_iter_max=float(max(times)), exact_phase_ms_per_iter=phases,
                unordered_ms_per_iter_median=float(np.median(un)), unordered_ms_per_iter_min=float(min(un)),
                unordered_ms_per_iter_max=float(max(un)), unordered_phase_ms_per_iter=uphases,
                host_draw_ms_per_iter=host_ms, rank_users_per_s=rank_rate)


def reference_ms(data, n_threads, seed, iters, dims=(15, 15, 12, 12), n_el=50, n_bpr=1000):
    """ms per iteration of the compiled reference's _fit_mter on the same arrays (None without oracle/_ref)."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "cornac")):
        return None
    if ref not in sys.path:
        sys.path.insert(0, ref)
    from cornac.models.bpr.recom_bpr import RNGVector
    from cornac.models.mter.recom_mter import MTER as RefMTER
    from cornac.utils.fast_dict import IntFloatDict
    d1, d2, d3, d4 = dims
    m = RefMTER(n_user_factors=d1, n_item_factors=d2, n_aspect_factors=d3, n_opinion_factors=d4, n_threads=n_threads,
                seed=seed)
    m.num_users, m.num_items, m.num_aspects, m.num_opinions = data.n_users, data.n_items, data.n_aspects, data.n_opinions
    rng = np.random.RandomState(1)
    shapes = dict(U=(data.n_users, d1), I=(data.n_items, d2), A=(data.n_aspects + 1, d3), O=(data.n_opinions, d4),
                  G1=(d1, d2, d3), G2=(d1, d3, d4), G3=(d2, d3, d4))
    P = {k: rng.uniform(0, 1, v).astype(np.float32) for k, v in shapes.items()}
    u, i = data.user_ids.astype(np.int64), data.indices.astype(np.int64)
    keys = ((u + i) * (u + i + 1) // 2 + i).astype(np.intp)       # the reference's get_key; no overflow at this shape
    rd = IntFloatDict(keys, data.pair_rating.astype(np.float64))
    nt = m.n_threads
    streams = [RNGVector(nt, n - 1, s) for n, s in zip((len(data.X), len(data.YU), len(data.YI), len(data.indices),
                                                        data.n_items), range(21, 26))]
    order = ("G1", "G2", "G3", "U", "I", "A", "O")
    z = lambda: [np.zeros_like(P[k]) for k in order]          # noqa: E731
    sg, de, dr = z(), z(), z()
    args = (*streams, nt, data.X, data.X_uids, data.X_iids, data.X_aids, data.YU, data.YU_uids, data.YU_aids,
            data.YU_oids, data.YI, data.YI_iids, data.YI_aids, data.YI_oids, rd, data.user_ids, data.indices,
            np.arange(data.n_items, dtype=np.int32), data.indptr, *[P[k] for k in order], *sg, *de, *dr)
    m._fit_mter(*args)
    t0 = time.perf_counter()
    for _ in range(iters):
        m._fit_mter(*args)
    return (time.perf_counter() - t0) * 1e3 / iters, nt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ref-iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    engine.warmup()
    props = torch.cuda.get_device_properties(0)
    res = dict(gpu=props.name, results=[])
    for name, scale in (("ml1m", 1), ("ml1m_x10", 10)):
        data = synth(6040 * scale, 3706 * scale, 1_000_000 * scale, 200, 100, 7)
        res["results"].append(run(name, data, a.iters))
        if scale == 1 and a.ref_iters > 0:
            for tag, nt, seed in (("reference_seeded", 1, 123), ("reference_unseeded", 0, None)):
                r = reference_ms(data, nt, seed, a.ref_iters)
                if r is not None:
                    res["results"][-1][tag + "_ms_per_iter"], res["results"][-1][tag + "_threads"] = r
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
