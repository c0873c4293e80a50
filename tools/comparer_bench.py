"""ComparERSub fit, rank and pair-list timing on seeded synthetic data (not bench.py's workload).

    python tools/comparer_bench.py [--iters 20]

Fit and rank: MTER's benchmark shape (tools/mter_bench.py: ML-1M's 6 040 users x 3 706 items, 1 M ratings, 200
aspects, 100 opinions, 3 sentiment tuples per rating) plus 200 000 comparative pairs whose aspects follow a Zipf law
(the popular aspects' A rows are the long pair chains); the reference's defaults otherwise (8/8/8/8 factors, 50
element, 1 000 BPR and 1 000 pair samples per iteration).  Reports the exact (seeded) and unordered (unseeded) fit in ms
per iteration (CUDA events, median of 5 calls of --iters iterations) with the kernel's phase split, and the rank rate
(top-10, seen items excluded, the mean of the top 100 of 200 aspect scores) in users/s.  Pair list: the host time of
build_pairs against the reference's _build_chrono_purchased_pairs on a train set with timestamps and sentiment
(--pair-users users with 40 items each, 20 aspects, enum_window 10), when the reference install under oracle/_ref is
present.  Prints one JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cornac_b200 import engine  # noqa: E402
from mter_bench import synth  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        limit = limit.strip() or "not measured"
    except (OSError, subprocess.SubprocessError):
        limit = "not measured"
    return name, limit


def with_pairs(data, n_pairs, seed):
    rng = np.random.RandomState(seed)
    a = np.minimum(rng.zipf(1.3, n_pairs) - 1, data.n_aspects - 2)
    kw = dict(data.__dict__)
    kw.update(p_user_indices=rng.randint(0, data.n_users, n_pairs).astype(np.int32),
              earlier_indices=rng.randint(0, data.n_items, n_pairs).astype(np.int32),
              later_indices=rng.randint(0, data.n_items, n_pairs).astype(np.int32),
              aspect_indices=a.astype(np.int32), pair_freq=np.ones(n_pairs, np.int32))
    return engine.MterData(**kw)


def fit_and_rank(data, iters, dims=(8, 8, 8, 8), n_el=50, n_bpr=1000, n_pair=1000):
    d1, d2, d3, d4 = dims
    rng = np.random.RandomState(1)
    shapes = ((data.n_users, d1), (data.n_items, d2), (data.n_aspects + 1, d3), (data.n_opinions, d4), (d1, d2, d3),
              (d1, d3, d4), (d2, d3, d4))
    dd = engine.ComparerDeviceData(data)
    params = [torch.from_numpy(rng.uniform(0, 1, s).astype(np.float32)).cuda() for s in shapes]
    sgrad = [torch.zeros_like(x) for x in params]
    work = torch.zeros(engine.comparer_sub_workspace_bytes(dd, dims, n_el, n_bpr, n_pair), dtype=torch.uint8,
                       device="cuda")
    dev = engine.comparer_draws([11, 12, 13, 14, 15, 16], data, n_el, n_bpr, n_pair, iters).next(iters).clone()
    hy = dict(lr=0.5, lambda_reg=0.1, lambda_bpr=10.0, lambda_d=0.01, workspace=work)

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

    names = ("predictions", "owners_and_stored_terms", "gradients", "adagrad")
    out = {}
    for mode, kw in (("exact", dict(draws=dev)), ("unordered", dict(draws=None, unordered=True, philox_seed=99))):
        draws = kw.pop("draws")
        times = timed(lambda: engine.comparer_sub_fit(dd, params, sgrad, draws, iters, n_el, n_bpr, n_pair, **hy, **kw))
        phase = torch.zeros(4, dtype=torch.int64, device="cuda")
        engine.comparer_sub_fit(dd, params, sgrad, draws, iters, n_el, n_bpr, n_pair, phase_ns=phase, **hy, **kw)
        out[mode + "_ms_per_iter_median"] = float(np.median(times))
        out[mode + "_ms_per_iter_min_max"] = [float(min(times)), float(max(times))]
        out[mode + "_phase_ms_per_iter"] = {k: v / 1e6 / iters for k, v in zip(names, phase.cpu().tolist())}
    # rank: the aspect-mixed rows of every user (N = 100 of 200 aspects), then top-10 with seen items excluded
    U, I, A, G1 = params[0], params[1], params[2], params[4]
    users = torch.arange(data.n_users, dtype=torch.int64, device="cuda")
    ex_ptr = torch.from_numpy(data.indptr.astype(np.int64)).cuda()
    ex_idx = torch.from_numpy(data.indices.astype(np.int32)).cuda()
    batch = 1024
    buf = torch.empty((batch, data.n_items), dtype=torch.float32, device="cuda")

    def rank_all():
        for u0 in range(0, data.n_users, batch):
            ub = users[u0:u0 + batch]
            sc = engine.comparer_rank_rows(U, I, A, G1, ub, 100, 0.5, out=buf[: len(ub)])
            engine.topk_rows(sc, 10, ex_ptr[u0:u0 + len(ub) + 1] - ex_ptr[u0], ex_idx[int(ex_ptr[u0]):])
    rank_all()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(3):
        rank_all()
    b.record()
    b.synchronize()
    out["rank_users_per_s"] = 3 * data.n_users / (a.elapsed_time(b) / 1e3)
    a.record()
    engine.comparer_rank_rows(U, I, A, G1, users[:batch], 100, 0.5, out=buf)
    b.record()
    b.synchronize()
    out["rank_rows_kernel_ms_per_1024_users"] = a.elapsed_time(b)
    return out


def pair_build(n_users, seed=5):
    """Host seconds of build_pairs and of the reference's _build_chrono_purchased_pairs on one train set."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "cornac")):
        return {"pair_build": "not measured (no reference install)"}
    if ref not in sys.path:
        sys.path.insert(0, ref)
    from cornac.data import Dataset, SentimentModality
    from cornac.models import ComparERSub as RefComparERSub
    from cornac_b200.recom_comparer import build_pairs, item_quality
    from cornac_b200.recom_mter import build_data
    rng = np.random.RandomState(seed)
    n_items, per_user, n_aspects = 2000, 40, 20
    rows, reviews = [], []
    for u in range(n_users):
        for i in rng.choice(n_items, per_user, replace=False):
            rows.append(("u%d" % u, "i%d" % i, float(rng.randint(1, 6)), int(rng.randint(10 ** 6))))
            reviews.append(("u%d" % u, "i%d" % i, [("a%d" % rng.randint(n_aspects), "o%d" % rng.randint(50),
                                                     float(rng.choice([-1.0, 1.0, 0.5]))) for _ in range(3)]))
    ts = Dataset.from_uirt(rows, seed=1)
    md = SentimentModality(data=reviews)
    md.build(uid_map=ts.uid_map, iid_map=ts.iid_map, dok_matrix=ts.dok_matrix)
    ts.add_modalities(sentiment=md)
    ts.chrono_user_data
    data = build_data(ts, ts.num_users, ts.num_items, 5.0)
    t0 = time.perf_counter()
    Y = item_quality(ts.sentiment, ts.num_items, 5.0, True)
    mine = build_pairs(ts, data, ts.num_items, Y, 2, 1, 10)
    ours = time.perf_counter() - t0
    m = RefComparERSub(enum_window=10, max_iter=0)
    m.num_users, m.num_items, m.num_aspects = ts.num_users, ts.num_items, md.num_aspects
    uia = {(int(u), int(i), int(a)): float(v) for u, i, a, v in zip(data.X_uids, data.X_iids, data.X_aids, data.X64)}
    t0 = time.perf_counter()
    Yr = m._build_item_quality_matrix(ts, md)
    theirs = m._build_chrono_purchased_pairs(ts, uia, Yr)
    ref_s = time.perf_counter() - t0
    same = all(np.array_equal(a, b) for a, b in zip(mine, theirs))
    return dict(pair_build_users=n_users, pair_build_items_per_user=per_user, pair_build_enum_window=10,
                pair_list_len=int(len(mine[0])), pair_build_s=ours, pair_build_reference_s=ref_s,
                pair_build_equal=bool(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--pairs", type=int, default=200000)
    ap.add_argument("--pair-users", type=int, default=300)
    args = ap.parse_args()
    name, limit = card()
    data = with_pairs(synth(6040, 3706, 1000209, 200, 100, 7), args.pairs, 8)
    res = dict(card=name, power_limit=limit, shape="ml1m", n_aspects=200, n_pairs=args.pairs)
    res.update(fit_and_rank(data, args.iters))
    res.update(pair_build(args.pair_users))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
