#!/usr/bin/env python
"""Per-kernel breakdown of ONE deterministic BPR epoch on the bench's configs[2] model (N = 1).

    python tools/det_epoch_profile.py OUTDIR [--warmup W]

Builds the model with bench.py's own generator and initialisation (imported, not copied), runs W warm-up epochs, then
one deterministic epoch under torch.profiler (CUDA activity) and writes OUTDIR/det_epoch_profile.json:
  * per kernel: total time, launch count, mean time per launch and per round (round = one bpr_det_grad_kernel launch);
  * the epoch's first bpr_det_apply_kernel launch on its own: it only plans round 0, so it prices one round's plan;
  * the gaps between consecutive kernels of the epoch (idle device time between launches) and their overlaps;
  * the epoch's span on the device, its algorithmic bytes (bench.algorithmic_bytes) and the resulting GB/s;
  * the card's name, power limit and max SM clock.
It only calls engine.bpr_epoch(..., deterministic=True), so the same script profiles any build of the library.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def card_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:          # the device name from torch still identifies the card
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "max_sm_clock": None, "nvidia_smi": repr(e)}


def kernel_events(trace_path):
    with open(trace_path) as f:
        tr = json.load(f)
    ev = [e for e in tr.get("traceEvents", []) if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev.sort(key=lambda e: float(e["ts"]))
    return [(e["name"].split("(")[0].split("<")[0].replace("void ", "").replace("b200::", ""), float(e["ts"]),
             float(e["dur"])) for e in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("det_epoch_profile.py: no CUDA device (this tool profiles the H100 kernels; no CPU fallback)")
    from torch.profiler import ProfilerActivity, profile
    from cornac_b200 import engine

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    W = dict(bench.WORKLOADS["c3"])
    blocks = bench.rank_blocks(0, 1)
    t0 = time.time()
    indptr, indices = bench.synth_shard(W, blocks, dev)
    U = bench.init_user_factors(W, blocks, dev)
    V, B = bench.init_item_factors(W, dev)
    data = engine.BprData(indptr, indices)
    data.prepare()
    torch.cuda.synchronize()
    print("[det_epoch_profile] model ready in %.1f s" % (time.time() - t0), file=sys.stderr, flush=True)
    stats = torch.zeros(2, dtype=torch.int64, device=dev)
    key = 0xB200

    def epoch(e):
        engine.bpr_epoch(data, W["n_items"], U, V, B, W["lr"], W["reg"], W["use_bias"], key, e, stats, blocked=True,
                         deterministic=True)

    for e in range(args.warmup):
        epoch(e)
    torch.cuda.synchronize()
    stats.zero_()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ev0.record()
        epoch(args.warmup)
        ev1.record()
        torch.cuda.synchronize()
    epoch_ms = ev0.elapsed_time(ev1)
    correct, skipped = stats.cpu().tolist()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        kev = kernel_events(path)
    kev = [e for e in kev if e[0].startswith("bpr_")]
    if not kev:
        raise SystemExit("det_epoch_profile.py: the trace holds no bpr_* kernel")
    n_rounds = sum(1 for e in kev if e[0] == "bpr_det_grad_kernel")
    # the epoch's first bpr_det_apply_kernel launch applies nothing and only plans round 0: the cost of one round's plan
    first_apply = next((x for x, e in enumerate(kev) if e[0] == "bpr_det_apply_kernel"), None)
    prologue = None
    per = {}
    for x, (name, ts, dur) in enumerate(kev):
        if x == first_apply:
            prologue = {"kernel": name, "us": round(dur, 3)}
            continue
        d = per.setdefault(name, {"count": 0, "total_us": 0.0})
        d["count"] += 1
        d["total_us"] += dur
    for d in per.values():
        d["mean_us"] = round(d["total_us"] / d["count"], 3)
        d["us_per_round"] = round(d["total_us"] / max(n_rounds, 1), 3)
        d["total_us"] = round(d["total_us"], 1)
    # a launch that starts before the one before it has ended (programmatic dependent launch) gives a negative gap: the
    # overlap, during which the later launch may be waiting for the earlier one, so kernel times can add up to more than
    # the span
    gaps = [kev[x + 1][1] - (kev[x][1] + kev[x][2]) for x in range(len(kev) - 1)]
    gaps_pos = [g for g in gaps if g > 0]
    overlaps = [-g for g in gaps if g < 0]
    span_us = kev[-1][1] + kev[-1][2] - kev[0][1]
    busy_us = sum(e[2] for e in kev)
    nnz = int(data.nnz)
    mean_deg = W["nnz"] / W["n_users"]
    alg = bench.algorithmic_bytes(W["k"], nnz - skipped, skipped, mean_deg)
    out = {
        "card": card_info(),
        "workload": bench.workload_text(W, 1),
        "epoch": {"samples": nnz, "updates": nnz - skipped, "skipped": skipped, "correct": correct, "rounds": n_rounds,
                  "launches": len(kev), "event_ms_under_profiler": round(epoch_ms, 3),
                  "device_span_ms": round(span_us / 1e3, 3), "kernel_busy_ms": round(busy_us / 1e3, 3),
                  "us_per_round": round(span_us / max(n_rounds, 1), 3),
                  "algorithmic_bytes": alg, "algorithmic_gbs": round(alg / (span_us * 1e-6) / 1e9, 1)},
        "kernels": per,
        "prologue": prologue,
        "gaps": {"count": len(gaps), "total_us": round(sum(gaps_pos), 1),
                 "mean_us": round(sum(gaps_pos) / max(len(gaps), 1), 3),
                 "max_us": round(max(gaps) if gaps else 0.0, 3),
                 "overlaps": len(overlaps), "overlap_total_us": round(sum(overlaps), 1),
                 "overlap_mean_us": round(sum(overlaps) / max(len(overlaps), 1), 3)},
        "note": "kernel times and gaps from torch.profiler (CUDA activity) over one epoch after %d warm-up epoch(s); "
                "`kernels` leaves out the epoch's first bpr_det_apply_kernel launch (`prologue`: the plan of round 0 "
                "alone); algorithmic GB/s = bench.algorithmic_bytes over the device span of the epoch's kernels"
                % args.warmup,
    }
    os.makedirs(args.outdir, exist_ok=True)
    with open(os.path.join(args.outdir, "det_epoch_profile.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
