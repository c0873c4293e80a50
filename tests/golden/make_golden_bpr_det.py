"""SHA-256 digests of the deterministic BPR epoch (engine.bpr_epoch(..., deterministic=True)) -> bpr_det_digests.json.

    python tests/golden/make_golden_bpr_det.py [OUT.json]      (needs a GPU)

Each case trains seeded factors for 3 epochs and records the SHA-256 of the bytes of U, V and B and the (correct, skipped)
counts of every epoch.  The deterministic mode repeats bit for bit, so any rewrite of its kernels must reproduce these
digests exactly; tests/test_bpr_det_gpu.py recomputes them with run_case().  The committed JSON was written by the
two-launch-per-round implementation with row-indexed accumulators (one NVIDIA H100 80GB HBM3).
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

EPOCHS = 3
SEED = 77

# shape: (n_users, n_items, nnz, zipf exponent of item popularity).  "mid" rounds are the full 16384 samples
# (min(n_users, n_items) / 4 > 16384); "small" rounds are max_groups = 75 samples.
SHAPES = {
    "mid": (100_000, 70_000, 1_000_000, 0.8),
    "zipf": (100_000, 70_000, 1_000_000, 1.1),      # head item in ~10 % of the interactions: hundreds of touches per round
    "small": (2_000, 300, 20_000, 0.8),
}


def _case(name, shape, k, **kw):
    c = dict(name=name, shape=shape, k=k, use_bias=True, blocked=False, part_mb=None, exact_exp=False, hinge=False,
             neg_weighted=False, unbounded=False, n_samples=None, sample_base=0)
    c.update(kw)
    return c


CASES = [
    _case("mid_k10", "mid", 10),
    _case("mid_k64", "mid", 64),
    _case("mid_k128", "mid", 128),
    _case("mid_k130", "mid", 130),
    _case("mid_k128_blocked", "mid", 128, blocked=True, part_mb=4),
    _case("mid_k64_blocked_nobias", "mid", 64, blocked=True, part_mb=2, use_bias=False),
    _case("mid_k64_nobias", "mid", 64, use_bias=False),
    _case("mid_k128_exact", "mid", 128, exact_exp=True),
    _case("mid_k64_hinge", "mid", 64, hinge=True),
    _case("mid_k130_hinge_blocked", "mid", 130, hinge=True, blocked=True, part_mb=4),
    _case("mid_k64_wbpr", "mid", 64, neg_weighted=True),
    _case("mid_k128_wbpr_blocked", "mid", 128, neg_weighted=True, blocked=True, part_mb=4),
    _case("zipf_k128", "zipf", 128),
    _case("zipf_k64_wbpr_unbounded", "zipf", 64, neg_weighted=True, unbounded=True),
    _case("small_k10", "small", 10),
    _case("small_k130_exact", "small", 130, exact_exp=True),
    _case("mid_k64_tail_base", "mid", 64, unbounded=True, n_samples=123_457, sample_base=987_654_321),
    _case("mid_k130_tail_base_blocked", "mid", 130, blocked=True, part_mb=4, n_samples=250_001, sample_base=12_345),
]


def synth_csr(n_users, n_items, nnz, seed, zipf):
    """Unique (u, i) pairs with Zipf(zipf) item popularity -> (indptr, indices) int32, rows sorted."""
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** zipf
    p /= p.sum()
    u = rng.randint(n_users, size=int(nnz * 1.3))
    i = rng.choice(n_items, size=len(u), p=p)
    key = np.unique(u.astype(np.int64) * n_items + i)
    if len(key) > nnz:
        key = np.sort(rng.choice(key, size=nnz, replace=False))
    u, i = key // n_items, key % n_items
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    np.add.at(indptr, u + 1, 1)
    return np.cumsum(indptr).astype(np.int32), i.astype(np.int32)


_DATA = {}


def _shape_data(shape):
    if shape not in _DATA:
        n_users, n_items, nnz, zipf = SHAPES[shape]
        _DATA[shape] = synth_csr(n_users, n_items, nnz, seed=len(shape) * 1000 + nnz % 997, zipf=zipf)
    return _DATA[shape]


def run_case(c):
    """{U, V, B: sha256 hex, stats: [[correct, skipped] per epoch]} of case `c` on the current CUDA device."""
    import torch
    from cornac_b200 import engine
    n_users, n_items, _, _ = SHAPES[c["shape"]]
    indptr, indices = _shape_data(c["shape"])
    k = c["k"]
    rng = np.random.RandomState(k * 7 + 1)
    U = torch.from_numpy(rng.normal(0, 0.1, (n_users, k)).astype(np.float32)).cuda()
    V = torch.from_numpy(rng.normal(0, 0.1, (n_items, k)).astype(np.float32)).cuda()
    B = torch.from_numpy(rng.normal(0, 0.1, n_items).astype(np.float32)).cuda()
    data = engine.BprData.from_host(indptr, indices)
    old = os.environ.get("B200_BPR_PART_MB")
    if c["part_mb"] is not None:
        os.environ["B200_BPR_PART_MB"] = str(c["part_mb"])
    stats_all = []
    try:
        for e in range(EPOCHS):
            stats = torch.zeros(2, dtype=torch.int64, device="cuda")
            engine.bpr_epoch(data, n_items, U, V, B, 0.05, 0.01, c["use_bias"], SEED, e, stats,
                             n_samples=c["n_samples"], sample_base=c["sample_base"] + e * 7919, exact_exp=c["exact_exp"],
                             unbounded=c["unbounded"], neg_weighted=c["neg_weighted"], hinge=c["hinge"],
                             blocked=c["blocked"], deterministic=True)
            stats_all.append([int(x) for x in stats.cpu().tolist()])
    finally:
        if old is None:
            os.environ.pop("B200_BPR_PART_MB", None)
        else:
            os.environ["B200_BPR_PART_MB"] = old
    torch.cuda.synchronize()
    digest = lambda t: hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()
    return {"U": digest(U), "V": digest(V), "B": digest(B), "stats": stats_all}


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("make_golden_bpr_det.py needs a CUDA device")
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "bpr_det_digests.json")
    res = {"device": torch.cuda.get_device_name(0), "epochs": EPOCHS, "seed": SEED, "cases": {}}
    for c in CASES:
        res["cases"][c["name"]] = run_case(c)
        print(c["name"], res["cases"][c["name"]]["stats"], flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
