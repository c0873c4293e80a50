#!/usr/bin/env python
"""bench.py -- BPR triplet-updates/s and ranked-users/s on 1/2/4/8 H100 vs the reference CPU path.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference] [--workload c3|c2] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

Workload (default, BASELINE.json configs[2] -- the north_star target): ONE synthetic model of 10 M users x
1 M items x 1 B interactions, BPR k = 128.  The matrix is generated as 8 fixed user blocks (1.25 M users /
125 M interactions each, block b seeded 1234 + b, one shared item-popularity law), so it is THE SAME model
for every N; `--gpus N` shards it by interaction count: rank r owns blocks [8 r / N, 8 (r + 1) / N)
(STRONG scaling: total work fixed).  The 1 M-item matrix V (512 MB) and the biases are replicated and the
item changes are exchanged once per epoch inside the timed region (one fused NVLink peer-memory kernel per tensor, or
delta kernels + NCCL all-reduce with --exchange nccl; rule: mean over the ranks that changed a row).  N = 1 holds the
whole model on one GPU (about 35 GB of the 80 GB).

A "step" is one BPR epoch over the whole model = 1 B sampled triplets in total (what one call of the
reference's BPR._fit_sgd does, cornac/models/bpr/recom_bpr.pyx:208-269), i.e. nnz / N per rank.

value  = non-skipped triplet updates per second over all ranks, inputs resident in HBM (CUDA events on
         the launching stream, max over ranks);
e2e    = the same through the host-buffer entry the plug-in's fit() uses (engine.bpr_train_host):
         pinned-host CSR + factors -> H2D -> prepare -> one epoch -> D2H, per rank on its shard;
roofline / cpu_baseline / per_rank / rank (configs[4]: all 10 M users of the trained model ranked against
the 1 M items, top-100) / mf (configs[3]: MF k = 128 on the same 10 M x 1 M x 1 B rating list) ride along.
--impl reference times the reference's own Cython/OpenMP kernel (oracle/_ref) on the host cores the
process actually owns, on a bounded sample of the same workload.
--dump-outputs DIR writes, after the timed steps, what the last timed epoch left to its caller: a fixed, seeded
sample of rows of U and V, all of B and the (correct, skipped) counts, as DIR/<name>.npy (rank r > 0 adds _r<r>).
The inputs depend only on the arguments, so two builds can be compared output for output.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

N_BLOCKS = 8
WORKLOADS = {
    # BASELINE.json configs[2]
    "c3": dict(label="BASELINE.json configs[2]", n_users=10_000_000, n_items=1_000_000, nnz=1_000_000_000, k=128,
               lr=0.05, reg=0.01, use_bias=True),
    # BASELINE.json configs[1] (round-1 headline; kept for A/B runs)
    "c2": dict(label="BASELINE.json configs[1]", n_users=1_000_000, n_items=100_000, nnz=100_000_000, k=64,
               lr=0.05, reg=0.01, use_bias=True),
}
RANK_TOPK = 100
RANK_E2E_BATCH = 1_000_000                          # users per host request of the rank e2e leg
CPU_SAMPLE = dict(n_users=100_000)                  # bounded sample for the CPU legs: the first users of block 0
ITEM_SEED = 4321                                    # the item-popularity law is one property of the model, shared by all blocks


def log(*a):
    print(*a, file=sys.stderr, flush=True)


# --------------------------------------------------------------------------------------
# synthetic data (torch on the GPU is used as a fast array library here; not product code)
def synth_interactions(n_users, n_items, nnz, seed, device, item_seed=None):
    """Unique (u, i) pairs: user activity ~ log-normal (mean degree nnz/n_users), item
    popularity ~ Zipf(1.0); returns CSR (indptr int32, indices int32) on `device`.
    item_seed: seed of the popular-item permutation (None: drawn from `seed`)."""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    w_u = torch.exp(torch.randn(n_users, generator=g, device=device, dtype=torch.float64))
    cdf_u = torch.cumsum(w_u / w_u.sum(), 0)
    w_i = 1.0 / torch.arange(1, n_items + 1, device=device, dtype=torch.float64)
    if item_seed is None:
        perm = torch.randperm(n_items, generator=g, device=device)      # popular ids spread over the id range
    else:
        gi = torch.Generator(device=device)
        gi.manual_seed(item_seed)
        perm = torch.randperm(n_items, generator=gi, device=device)
    cdf_i = torch.cumsum(w_i / w_i.sum(), 0)
    keys = torch.empty(0, dtype=torch.int64, device=device)
    need = nnz
    while need > 0:
        m = int(need * 1.25) + 1024
        u = torch.searchsorted(cdf_u, torch.rand(m, generator=g, device=device, dtype=torch.float64)).clamp_(max=n_users - 1)
        i = perm[torch.searchsorted(cdf_i, torch.rand(m, generator=g, device=device, dtype=torch.float64)).clamp_(max=n_items - 1)]
        keys = torch.unique(torch.cat([keys, u * n_items + i]))
        del u, i
        need = nnz - keys.numel()
    if keys.numel() > nnz:
        drop = torch.randperm(keys.numel(), generator=g, device=device)[: keys.numel() - nnz]
        mask = torch.ones(keys.numel(), dtype=torch.bool, device=device)
        mask[drop] = False
        keys = keys[mask]
    u = keys // n_items
    indices = (keys % n_items).to(torch.int32)
    counts = torch.bincount(u, minlength=n_users)
    indptr = torch.zeros(n_users + 1, dtype=torch.int64, device=device)
    indptr[1:] = torch.cumsum(counts, 0)
    return indptr.to(torch.int32), indices.contiguous()


def block_shape(W):
    """(users, interactions) of one of the N_BLOCKS user blocks the model is generated in."""
    return W["n_users"] // N_BLOCKS, W["nnz"] // N_BLOCKS


def rank_blocks(rank, world):
    per = N_BLOCKS // world
    return list(range(rank * per, (rank + 1) * per))


def synth_shard(W, blocks, device):
    """CSR of the user blocks `blocks` (consecutive), user ids local to the shard."""
    import torch
    ub, nb = block_shape(W)
    ptrs, idxs, base = [], [], 0
    for b in blocks:
        ip, ix = synth_interactions(ub, W["n_items"], nb, seed=1234 + b, device=device, item_seed=ITEM_SEED)
        ptrs.append(ip[:-1].to(torch.int64) + base)
        base += int(ix.numel())
        idxs.append(ix)
        del ip, ix
    ptrs.append(torch.tensor([base], dtype=torch.int64, device=device))
    indptr = torch.cat(ptrs).to(torch.int32)
    indices = torch.cat(idxs) if len(idxs) > 1 else idxs[0]
    return indptr.contiguous(), indices.contiguous()


def init_user_factors(W, blocks, device):
    """(U[0,1) - 0.5) / k like BPR._init (recom_bpr.pyx:145-152), block b seeded 500 + b."""
    import torch
    ub, _ = block_shape(W)
    U = torch.empty((ub * len(blocks), W["k"]), dtype=torch.float32, device=device)
    for n, b in enumerate(blocks):
        g = torch.Generator(device=device)
        g.manual_seed(500 + b)
        U[n * ub:(n + 1) * ub] = (torch.rand((ub, W["k"]), generator=g, device=device) - 0.5) / W["k"]
    return U


def init_item_factors(W, device, seed=99):
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    V = (torch.rand((W["n_items"], W["k"]), generator=g, device=device) - 0.5) / W["k"]
    B = torch.zeros(W["n_items"], device=device)
    return V, B


# --------------------------------------------------------------------------------------
class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 20 ms; samples are stamped on arrival and
    only those inside the timed window are reported (fallback: all samples of the run)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx, self.proc, self.lines = gpu_index, None, []
        self.t0 = self.t1 = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.idx), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "20"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append((time.time(), line.strip()))

    def window_begin(self):
        self.t0 = time.time()

    def window_end(self):
        self.t1 = time.time()

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.1)
        self.proc.terminate()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]

        def digest(rows):
            sm, smax, pw, reasons = [], [], [], set()
            for _, l in rows:
                f = [x.strip() for x in l.split(",")]
                if len(f) < 9:
                    continue
                try:
                    sm.append(float(f[1])); smax.append(float(f[2])); pw.append(float(f[3]))
                except ValueError:
                    continue
                for nm, v in zip(names, f[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(nm)
            return sm, smax, pw, reasons
        inside = [r for r in self.lines if self.t0 is not None and self.t0 - 0.01 <= r[0] <= (self.t1 or 1e30) + 0.03]
        window = "timed region"
        if len(inside) < 2:
            inside, window = self.lines, "whole run (timed region shorter than the sampling period)"
        sm, smax, pw, reasons = digest(inside)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(smax) if smax else None,
                "power_w_max": max(pw) if pw else None, "samples": len(sm), "window": window, "reasons": sorted(reasons)}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "fallback (H100 SXM data sheet, HBM3)"


def tensor_peak():
    """dense 16-bit tensor TFLOP/s: the sustained figure of MEASURED_PEAKS.json (the kernel runs for many ms)."""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        for key in ("bf16_tflops_sustained", "bf16_tflops"):
            if key in d:
                return float(d[key]), "measured sustained (MEASURED_PEAKS.json)"
    return 989.0, "fallback (H100 SXM data sheet, dense FP16; not reached in practice)"


def algorithmic_bytes(k, updates, skipped, mean_deg):
    """SURVEY.md 8(d): 3 rows read + 3 written (24k B) + 4 biases R/W (16 B) + indices/coo/indptr
    (16 B) + 4*ceil(log2(deg+1)) B binary search per update; a skipped sample costs only the
    sampling + search bytes."""
    search = 4 * math.ceil(math.log2(mean_deg + 1))
    return updates * (24 * k + 16 + 16 + search) + skipped * (16 + search)


def host_cores():
    """The host cores this process may actually use: the scheduler affinity mask capped by the cgroup CPU quota
    (a 1-GPU lease of a 128-core box does not own 128 cores; 128 OpenMP threads on a 16-core quota run SLOWER
    than 16).  The reference's own rule is multiprocessing.cpu_count() (recom_bpr.pyx:134-137), which ignores both."""
    try:
        aff = len(os.sched_getaffinity(0))
    except Exception:
        aff = os.cpu_count() or 1
    quota = None
    try:
        f = open("/sys/fs/cgroup/cpu.max").read().split()                 # cgroup v2: "<quota> <period>" or "max <period>"
        if f[0] != "max":
            quota = float(f[0]) / float(f[1])
    except Exception:
        try:                                                                 # cgroup v1
            q = float(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            p = float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                quota = q / p
        except Exception:
            quota = None
    use = aff if quota is None else max(1, min(aff, int(quota + 0.5)))
    try:
        load1 = os.getloadavg()[0]
    except Exception:
        load1 = None
    return {"os_cpu_count": os.cpu_count(), "sched_affinity": aff, "cgroup_cpu_quota": quota, "threads_used": use,
            "omp_num_threads_env": os.environ.get("OMP_NUM_THREADS"), "loadavg_1m": load1}


def measured_traffic(workload, kernel_name, samples_per_launch):
    """DRAM bytes per launch of the timed kernel from the committed `ncu --set full` capture of THIS kernel on THIS
    workload shape (profiles/bpr_hogwild_dram_bytes.json: per-sample bytes, kernel name, commit, capture file);
    None when no capture of this kernel / shape exists."""
    p = os.path.join(ROOT, "profiles", "bpr_hogwild_dram_bytes.json")
    try:
        rec = json.load(open(p)).get("captures", {}).get(workload)
        if rec and rec.get("kernel") == kernel_name:
            return {"bytes_per_launch": rec["dram_bytes_per_sample"] * samples_per_launch,
                    "dram_bytes_per_sample": rec["dram_bytes_per_sample"], "capture": rec.get("capture"), "commit": rec.get("commit")}
    except Exception:
        pass
    return None


# --------------------------------------------------------------------------------------
def ref_path():
    return os.path.join(ROOT, "oracle", "_ref")


def reference_fit_sgd_runner(indptr, indices, n_items, k, lr, reg, n_threads):
    """Returns (run_epoch() -> (correct, skipped), kind, cores).  Uses the UNMODIFIED compiled
    reference (oracle/_ref: cornac.models.bpr.recom_bpr.BPR._fit_sgd + RNGVector) when it is
    importable, else the oracle's OpenMP port."""
    ref = ref_path()
    n_users = len(indptr) - 1
    rng = np.random.RandomState(1)
    U = ((rng.uniform(0, 1, (n_users, k)).astype(np.float32) - 0.5) / k)
    V = ((rng.uniform(0, 1, (n_items, k)).astype(np.float32) - 0.5) / k)
    B = np.zeros(n_items, np.float32)
    user_ids = np.repeat(np.arange(n_users), np.diff(indptr)).astype(np.int32)
    try:
        if ref not in sys.path:
            sys.path.insert(0, ref)
        from cornac.models.bpr.recom_bpr import BPR as RefBPR, RNGVector
        n_threads = n_threads or host_cores()["threads_used"]
        m = RefBPR(k=k, learning_rate=lr, lambda_reg=reg, use_bias=True)
        rp = RNGVector(n_threads, len(user_ids) - 1, 11)
        rn = RNGVector(n_threads, n_items - 1, 12)
        neg = np.arange(n_items, dtype=np.int32)

        def run():
            return m._fit_sgd(rp, rn, n_threads, user_ids, indices, neg, indptr, U, V, B)
        return run, "reference", n_threads
    except Exception as e:   # reference install absent: the oracle port, all threads
        log("[bench] reference install not importable (%s); using the oracle OpenMP port" % (e,))
        from oracle import oracle as O
        n_threads = n_threads or host_cores()["threads_used"]
        state = {"e": 0}

        def run():
            state["e"] += 1
            return O.bpr_epoch_omp(indptr, indices, n_items, U, V, B, lr, reg, True, n_threads, seed=state["e"])
        return run, "port", n_threads


def cpu_sample_csr(indptr_host, indices_host):
    """Bounded sample of the workload for the CPU legs: the first users of the same synthetic
    matrix (same k, same item catalogue, ~1 % of the interactions)."""
    n_u = CPU_SAMPLE["n_users"]
    n_u = min(n_u, len(indptr_host) - 1)
    end = int(indptr_host[n_u])
    return np.ascontiguousarray(indptr_host[: n_u + 1]), np.ascontiguousarray(indices_host[:end])


def time_cpu_epochs(run, nnz, min_seconds=8.0, max_epochs=6):
    run()                                             # warm-up epoch (page-in, thread pool)
    t_tot, upd, eps = 0.0, 0, 0
    while t_tot < min_seconds and eps < max_epochs:
        t0 = time.perf_counter()
        c, s = run()
        t_tot += time.perf_counter() - t0
        upd += nnz - s
        eps += 1
    return upd / t_tot, t_tot, eps


# --------------------------------------------------------------------------------------
def checked_item_sync(sync, tensors, world):
    """After the warm-up exchanges: if the peer-memory exchange reported a missing peer on ANY rank (its bounded waits expired),
    every rank drops it, the replicas are re-synchronised from rank 0 and the delta-kernel + NCCL path takes over; the JSON line
    says so.  Returns (sync, note)."""
    import torch
    import torch.distributed as dist
    if sync is None or not hasattr(sync, "failed"):
        return sync, None
    bad = torch.tensor([1 if sync.failed() else 0], device=tensors[0].device)
    dist.all_reduce(bad, op=dist.ReduceOp.MAX)
    if int(bad.item()) == 0:
        return sync, None
    from cornac_b200.parallel import ItemReplicaSync
    torch.cuda.synchronize()
    sync.close()
    for t in tensors:
        dist.broadcast(t, 0)
    log("[bench] the peer-memory exchange timed out on some rank during the warm-up: falling back to delta kernels + NCCL all-reduce")
    return ItemReplicaSync(tensors), "peer-memory exchange timed out during the warm-up; timed region ran delta kernels + NCCL all-reduce"


def workload_text(W, world):
    return ("%s: ONE model of %d users x %d items x %d interactions, BPR k=%d, lr=%g reg=%g use_bias; user activity "
            "log-normal, item popularity Zipf(1.0), unique pairs; generated as %d user blocks, rank r owns blocks "
            "[%d r, %d (r+1))" % (W["label"], W["n_users"], W["n_items"], W["nnz"], W["k"], W["lr"], W["reg"], N_BLOCKS,
                                  N_BLOCKS // world, N_BLOCKS // world))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--scale", type=float, default=1.0, help="shrink users and interactions (debug only; result then INVALID)")
    ap.add_argument("--workload", default="c3", choices=sorted(WORKLOADS),
                    help="c3 = BASELINE configs[2] (default, the north_star target); c2 = configs[1]")
    ap.add_argument("--atomic", type=int, default=1, help="Hogwild scatter: 1 red.global.add (default, what fit() uses), 0 plain racy stores")
    ap.add_argument("--deterministic", type=int, default=1,
                    help="1: the timed epochs run in deterministic rounds, so their outputs repeat run to run (default); the Hogwild "
                         "kernels are then timed in a separate leg (`hogwild`); 0: the timed epochs are Hogwild epochs")
    ap.add_argument("--blocked", type=int, default=1, help="1: cache-blocked sample order (default, what fit() uses), 0: i.i.d. order")
    ap.add_argument("--exchange", default="auto", choices=["auto", "p2p", "nccl"],
                    help="item-replica exchange at N > 1: p2p = one fused NVLink kernel per tensor, nccl = delta kernels + all-reduce")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-rank", action="store_true")
    ap.add_argument("--no-mf", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's outputs (sampled U / V rows, B, counts) as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0:
        raise SystemExit("bench.py: --steps must be >= 1 and --warmup >= 0")

    # stdout carries exactly ONE line, the JSON record: everything else any library prints to fd 1 (NCCL's INFO log goes
    # to stdout by default) is sent to stderr, where the NCCL init lines ("... nranks N ...") stay visible.
    real_stdout = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    os.environ.setdefault("NCCL_DEBUG", "INFO")
    os.environ.setdefault("NCCL_DEBUG_SUBSYS", "INIT")

    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    W = dict(WORKLOADS[args.workload])
    if args.scale != 1.0:
        W["n_users"] = max(8000, int(W["n_users"] * args.scale) // N_BLOCKS * N_BLOCKS)
        W["nnz"] = max(80000, int(W["nnz"] * args.scale) // N_BLOCKS * N_BLOCKS)
    k = W["k"]
    if world not in (1, 2, 4, 8):
        raise SystemExit("bench.py shards %d user blocks: --gpus must be 1, 2, 4 or 8" % N_BLOCKS)

    if args.impl == "reference":
        if rank != 0:
            return 0
        return run_reference_arm(args, W, world, real_stdout)

    assert torch.cuda.is_available(), "bench.py needs a GPU (no CPU fallback)"
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from cornac_b200 import engine
    from cornac_b200._lib import load
    from cornac_b200.parallel import make_item_sync
    L = load()

    # ---- data: this rank's user blocks of the ONE model; items shared
    t0 = time.time()
    blocks = rank_blocks(rank, world)
    indptr, indices = synth_shard(W, blocks, dev)
    U = init_user_factors(W, blocks, dev)
    V, B = init_item_factors(W, dev)
    if world > 1:
        dist.broadcast(V, 0); dist.broadcast(B, 0)
    data = engine.BprData(indptr, indices)
    nnz = data.nnz
    n_local = data.n_users
    mean_deg = W["nnz"] / W["n_users"]
    data.prepare()
    torch.cuda.synchronize()
    log("[bench] rank %d/%d data ready in %.1fs: blocks %s = %d users x %d items x %d nnz (%.1f GB allocated)"
        % (rank, world, time.time() - t0, blocks, n_local, W["n_items"], nnz, torch.cuda.memory_allocated() / 1e9))
    sync = make_item_sync([V, B], kind=args.exchange) if world > 1 else None
    exchange_kind = type(sync).__name__ if sync is not None else None
    stats = torch.zeros(2, dtype=torch.int64, device=dev)
    key = 0xB200

    def epoch(e):
        engine.bpr_epoch(data, W["n_items"], U, V, B, W["lr"], W["reg"], W["use_bias"], key + rank, e, stats,
                         atomic=bool(args.atomic), blocked=bool(args.blocked), deterministic=bool(args.deterministic))

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for e in range(args.warmup):
        epoch(e)
        if sync is not None:
            sync.exchange()
    barrier()
    sync, exchange_note = checked_item_sync(sync, [V, B], world)
    exchange_kind = type(sync).__name__ if sync is not None else None
    stats.zero_()
    clocks = ClockSampler(local_rank)
    if rank == 0:
        clocks.start()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    ev0, ev1 = ev(), ev()
    step_ev = [(ev(), ev(), ev()) for _ in range(args.steps)]
    barrier()
    launches0 = int(L.b200_kernel_launches())
    clocks.window_begin()
    ev0.record()
    for e in range(args.steps):
        a, b, c = step_ev[e]
        if e == args.steps - 1:
            stats_before_last = stats.clone()
        a.record()
        epoch(args.warmup + e)
        b.record()
        if sync is not None:
            sync.exchange()
        c.record()
    ev1.record()
    barrier()
    clocks.window_end()
    launches = int(L.b200_kernel_launches()) - launches0
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, U, V, B, stats - stats_before_last, rank, world)
    clk = clocks.stop() if rank == 0 else None
    ms_total = ev0.elapsed_time(ev1)
    kern_list = [a.elapsed_time(b) for a, b, _ in step_ev]
    xchg_list = [b.elapsed_time(c) for _, b, c in step_ev]
    kern_ms, xchg_ms = float(np.mean(kern_list)), float(np.mean(xchg_list))
    correct, skipped = stats.cpu().tolist()
    mine = torch.tensor([ms_total, float(nnz * args.steps - skipped), float(skipped), kern_ms, xchg_ms, float(launches),
                         float(np.min(kern_list)), float(np.max(kern_list))], dtype=torch.float64, device=dev)
    if world > 1:
        allr = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(allr, mine)
        allr = torch.stack(allr).cpu().numpy()
    else:
        allr = mine.cpu().numpy()[None, :]
    ms_total = float(allr[:, 0].max())
    updates, skipped_all = float(allr[:, 1].sum()), float(allr[:, 2].sum())
    value = updates / (ms_total * 1e-3)

    # ---- roofline of the dominant kernel, per rank (every rank launches the same kernel on nnz / N samples)
    peak, peak_src = measured_peaks()
    g_lanes = min(32, max(4, k // 4))
    hog_name = ("bpr_hogwild_stream_kernel<G=%d,%s,D=2>" if (k % 4 == 0 and g_lanes >= 32) else "bpr_hogwild_chunk_kernel<G=%d,NPL=1,VEC,%s>") \
        % (g_lanes, "ATOMIC" if args.atomic else "PLAIN")
    kernel_name = "bpr_det_grad_kernel + bpr_det_apply_kernel" if args.deterministic else hog_name
    fracs = []
    for r in range(world):
        upd_r, skp_r = allr[r, 1] / args.steps, allr[r, 2] / args.steps
        fracs.append(algorithmic_bytes(k, upd_r, skp_r, mean_deg) / (allr[r, 3] * 1e-3) / 1e9)
    slow = int(np.argmax(allr[:, 3]))
    roofline = {"kernel": kernel_name, "bound": "hbm", "achieved": round(fracs[slow], 1), "peak": peak, "unit": "GB/s",
                "frac": round(fracs[slow] / peak, 4), "traffic": None, "peak_source": peak_src,
                "algorithmic_bytes_per_update": 24 * k + 32 + 4 * math.ceil(math.log2(mean_deg + 1)),
                "kernel_ms": round(float(allr[slow, 3]), 3), "rank": slow,
                "note": "slowest rank's launches; achieved = algorithmic bytes of one launch / its mean CUDA-event duration",
                "frac_per_rank": [round(f / peak, 4) for f in fracs]}
    tr = measured_traffic(args.workload if args.scale == 1.0 else "scaled", kernel_name, nnz)
    if tr is not None:
        roofline["traffic"] = tr["bytes_per_launch"]
        roofline["traffic_source"] = tr
    per_rank = {"kernel_ms_mean": [round(float(x), 3) for x in allr[:, 3]],
                "kernel_ms_min": [round(float(x), 3) for x in allr[:, 6]],
                "kernel_ms_max": [round(float(x), 3) for x in allr[:, 7]],
                "exchange_ms_mean": [round(float(x), 3) for x in allr[:, 4]],
                "kernel_ms_min_med_max_over_ranks": [round(float(np.min(allr[:, 3])), 3), round(float(np.median(allr[:, 3])), 3),
                                                     round(float(np.max(allr[:, 3])), 3)],
                "exchange": ("none (single GPU)" if world == 1 else
                             ("%s: one fused NVLink peer-memory kernel per tensor (reduce-scatter + apply + all-gather of %d MB)"
                              if exchange_kind == "PeerItemExchange" else
                              "%s: delta_make -> NCCL all-reduce(%d MB, + the touched-by count) -> delta_apply") % (exchange_kind, (W["n_items"] * (k + 1) * 4) // 1000000))}

    if world > 1 and exchange_note:
        per_rank["exchange_note"] = exchange_note

    def over_ranks(ms):
        if world == 1:
            return ms
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # ---- the Hogwild kernels (what fit() runs) on the same model, continuing from the timed epochs: their results differ
    #      from run to run (samples read rows while others update them), so they are timed here but not dumped
    hogwild = None
    if args.deterministic:
        hev = [(ev(), ev()) for _ in range(args.steps)]
        stats.zero_()
        barrier()
        for e in range(args.steps):
            hev[e][0].record()
            engine.bpr_epoch(data, W["n_items"], U, V, B, W["lr"], W["reg"], W["use_bias"], key + rank, 1000 + e, stats,
                             atomic=bool(args.atomic), blocked=bool(args.blocked))
            hev[e][1].record()
        barrier()
        h_ms = over_ranks(float(np.mean([a.elapsed_time(b) for a, b in hev])))
        h_skipped = float(stats[1].item())
        h_upd = nnz * args.steps - h_skipped
        if world > 1:
            t = torch.tensor([h_upd], device=dev, dtype=torch.float64)
            dist.all_reduce(t)
            h_upd = float(t.item())
        h_gbs = algorithmic_bytes(k, h_upd / args.steps / world, h_skipped / args.steps, mean_deg) / (h_ms * 1e-3) / 1e9
        hogwild = {"value": round(h_upd / args.steps / (h_ms * 1e-3), 1), "unit": "updates/s", "ms_per_step": round(h_ms, 3),
                   "steps": args.steps, "kernel": hog_name,
                   "roofline": {"bound": "hbm", "achieved": round(h_gbs, 1), "peak": peak, "unit": "GB/s", "frac": round(h_gbs / peak, 4)},
                   "note": "Hogwild epochs (the kernels fit() runs) on the same model, after the timed epochs; max over ranks, "
                           "no item exchange; results differ from run to run, so they are not dumped"}

    # the pair store / membership table are only needed by the epochs
    data.pairs = data.table = None
    if sync is not None and hasattr(sync, "failed") and sync.failed():
        raise SystemExit("bench.py: a peer did not arrive in the NVLink item exchange (bounded wait expired)")
    if sync is not None and hasattr(sync, "close"):
        sync.close()
    sync = None
    torch.cuda.empty_cache()

    # ---- e2e: host buffers through the plug-in's training entry, copies inside the timed region
    e2e = None
    if not args.no_e2e:
        e2e = run_e2e(args, W, engine, indptr, indices, blocks, dev, world, rank)

    # ---- configs[4]: every user of the trained model ranked against the item catalogue (users stay sharded, no collective)
    rank_metric = None
    if not args.no_rank:
        rank_metric = run_rank(W, engine, L, data, U, V, B, dev, world, over_ranks)
    del U
    torch.cuda.empty_cache()

    # ---- configs[3]: MF on the same rating list, all ranks
    mf_metric = None
    if not args.no_mf:
        mf_metric = run_mf(W, engine, data, dev, world, over_ranks, exchange=args.exchange, steps=args.steps)

    # ---- CPU baseline on rank 0, N = 1 only
    cpu_baseline = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        ip, ix = cpu_sample_csr(indptr.cpu().numpy(), indices.cpu().numpy())
        run, kind, cores = reference_fit_sgd_runner(ip, ix, W["n_items"], k, W["lr"], W["reg"], 0)
        v, secs, eps = time_cpu_epochs(run, len(ix))
        cpu_baseline = {"value": round(v, 1), "unit": "triplet-updates/s", "cores": cores, "kind": kind,
                        "sample": "first %d users of the same matrix: %d interactions, %d items, k=%d, %d epoch(s) in %.1fs"
                                  % (len(ip) - 1, len(ix), W["n_items"], k, eps, secs),
                        "host": host_cores()}

    if rank == 0:
        out = {
            "metric": "BPR triplet-updates/sec", "value": round(value, 1), "unit": "updates/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms_total / args.steps, 3),
            "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": workload_text(W, world),
                       "step": "one epoch over the whole model = %d sampled triplets (%d per rank; Hogwild, on-device Philox sampling)"
                               % (W["nnz"], nnz),
                       "l2": "working set per rank (U %d MB + V %d MB + pair store %d MB + membership table) exceeds the 50 MB L2; no flush needed"
                             % (n_local * k * 4 // 1000000, W["n_items"] * k * 4 // 1000000, nnz * 8 // 1000000),
                       "parallelism": "users sharded x%d by interaction count, items replicated, 1 exchange of item changes per epoch (mean over the ranks that changed a row)" % world,
                       "scatter": ("deterministic rounds of <= 16384 samples, updates summed in 2^-40 fixed point" if args.deterministic
                                   else "red.global.add.v4.f32 (Hogwild)" if args.atomic else "st.global.cg.v4.f32 (Hogwild)"),
                       "sample_order": ("cache-blocked: %d windows of the interaction list x %d item blocks per rank (b200_bpr_block_plan); "
                                        "same per-epoch law as the i.i.d. order" % engine.bpr_block_plan(n_local, W["n_items"], k))
                                       if args.blocked else "i.i.d. (Philox counter order)"},
            "samples_per_s": round((W["nnz"] * args.steps) / (ms_total * 1e-3), 1),
            "skipped_frac": round(skipped_all / (W["nnz"] * args.steps), 5),
            "timed_region_s": round(ms_total * 1e-3, 3),
            "gpu_launches": int(allr[:, 5].sum()),
            "gpu_launches_note": "b200_kernel_launches() delta over the timed region, summed over ranks (NCCL's own kernels not counted)",
            "clocks": clk, "roofline": roofline, "per_rank": per_rank, "cpu_baseline": cpu_baseline, "e2e": e2e,
            "hogwild": hogwild, "rank": rank_metric, "mf": mf_metric, "host": host_cores(),
        }
        if args.scale != 1.0:
            out["INVALID"] = "scaled-down debug run (--scale %g)" % args.scale
        real_stdout.write(json.dumps(out) + "\n")
        real_stdout.flush()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


DUMP_ROWS = 32768                                   # sampled rows of U (over all ranks) and of V: 2 x 16 MB at k = 128


def dump_outputs(out_dir, U, V, B, last_stats, rank, world):
    """The arrays the timed BPR epochs leave to their caller, after the last timed step: a fixed sample of U's rows
    (seeded, independent of the build; DUMP_ROWS / world per rank), and on rank 0 only a fixed sample of V's rows and all
    of B (replicated on every rank), plus the (correct, skipped) counts of the last timed step, as float32 / float64 .npy."""
    import torch
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    sfx = "" if rank == 0 else "_r%d" % rank
    rng = np.random.RandomState(2024)
    u_rows = np.sort(rng.choice(U.shape[0], min(DUMP_ROWS // world, U.shape[0]), replace=False))
    v_rows = np.sort(rng.choice(V.shape[0], min(DUMP_ROWS, V.shape[0]), replace=False))
    pick = lambda T, rows: T.index_select(0, torch.from_numpy(rows).to(T.device)).cpu().numpy().astype(np.float32)
    arrays = {"U_sample": pick(U, u_rows), "U_sample_rows": u_rows.astype(np.float64),
              "stats": last_stats.cpu().numpy().astype(np.float64)}
    if rank == 0:
        arrays.update({"V_sample": pick(V, v_rows), "V_sample_rows": v_rows.astype(np.float64),
                       "B": B.cpu().numpy().astype(np.float32)})
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + sfx + ".npy"), a)
    log("[bench] wrote %s to %s" % (", ".join(sorted(arrays)), out_dir))


def run_e2e(args, W, engine, indptr, indices, blocks, dev, world, rank):
    import torch
    import torch.distributed as dist
    pin = lambda t: t.cpu().pin_memory()
    h_indptr, h_indices = pin(indptr), pin(indices)
    U = init_user_factors(W, blocks, dev)
    V, B = init_item_factors(W, dev, seed=7)
    hU, hV, hB = pin(U), pin(V), pin(B)
    del U, V, B
    torch.cuda.empty_cache()
    nnz = h_indices.numel()
    h2d = sum(t.numel() * t.element_size() for t in (h_indptr, h_indices, hU, hV, hB))
    d2h = sum(t.numel() * t.element_size() for t in (hU, hV, hB)) + 16
    steps = args.steps

    def one(e):
        hist, _ = engine.bpr_train_host(h_indptr.numpy(), h_indices.numpy(), W["n_items"], hU.numpy(), hV.numpy(),
                                        hB.numpy(), W["lr"], W["reg"], W["use_bias"], 1, key=77 + e + rank,
                                        atomic=bool(args.atomic), on_epoch=lambda *a: None, replica_sync=world > 1,
                                        blocked=bool(args.blocked))
        return hist[0]

    one(0)                                             # warm-up (allocator, pinned staging)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    upd = 0
    for e in range(steps):
        c, s = one(1 + e)
        upd += nnz - s
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    t = torch.tensor([dt, float(upd), float(h2d), float(d2h)], dtype=torch.float64, device=dev)
    if world > 1:
        tm = t.clone(); dist.all_reduce(tm, op=dist.ReduceOp.MAX)
        ts = t.clone(); dist.all_reduce(ts, op=dist.ReduceOp.SUM)
        dt, upd, h2d, d2h = tm[0].item(), ts[1].item(), ts[2].item(), ts[3].item()
    return {"value": round(upd / dt, 1), "unit": "updates/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h),
            "steps": steps, "ms_per_step": round(dt / steps * 1e3, 2),
            "path": "engine.bpr_train_host (the call BPR.fit makes) on every rank's shard: pinned host CSR + U/V/B -> H2D -> "
                    "prepare (pair store + membership table) -> 1 epoch" + (" -> item-delta all-reduce" if world > 1 else "")
                    + " -> D2H U/V/B + stats; bytes are summed over ranks"}


def reference_rank_users_per_s(U_host, V_host, B_host, topk, budget_s=8.0):
    """ranked users/s of the UNMODIFIED reference on the host cores: cornac.models.BPR.rank(user, k=topk) -- score() =
    copy(B) + fast_dot(U[u], V) (recom_bpr.pyx:272-297, OpenMP over the items) + argpartition top-k
    (recommender.py:476-530) -- called once per user like ranking_eval does, for a bounded number of users.
    Returns (users/s, users timed, seconds) or None when the compiled reference is not importable."""
    ref = ref_path()
    if not os.path.isdir(os.path.join(ref, "cornac")):
        return None
    if ref not in sys.path:
        sys.path.insert(0, ref)
    from cornac.models import BPR as RefBPR
    m = RefBPR(k=U_host.shape[1])
    m.num_users, m.num_items = U_host.shape[0], V_host.shape[0]
    m.u_factors = np.ascontiguousarray(U_host, dtype=np.float32)
    m.i_factors = np.ascontiguousarray(V_host, dtype=np.float32)
    m.i_biases = np.ascontiguousarray(B_host, dtype=np.float32)
    m.rank(0, k=topk)                                     # warm-up (thread pool, page faults)
    n, t0 = 0, time.perf_counter()
    while n < U_host.shape[0]:
        m.rank(n, k=topk)
        n += 1
        if (n & 15) == 0 and time.perf_counter() - t0 > budget_s:
            break
    secs = time.perf_counter() - t0
    return n / secs, n, secs


def run_rank(W, engine, L, data, U, V, B, dev, world=1, over_ranks=lambda ms: ms):
    """BASELINE.json configs[4] on the model the bench just trained: EVERY user of this rank's shard (10 M / N) is
    scored against all items (U x V^T + B on the tensor cores), the user's train positives are excluded, top-100 kept.
    `value` = device-resident request; `e2e` = host request -> H2D -> kernels -> D2H ids + scores."""
    import torch
    import torch.distributed as dist
    topk, k, n_items = RANK_TOPK, W["k"], W["n_items"]
    n_q = data.n_users
    ex_ptr = data.indptr.to(torch.int64).contiguous()
    ex_idx = data.indices
    nb = int(L.b200_rank_topk_workspace_bytes(n_q, n_items, k, topk))
    ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=dev)
    n_warm = min(n_q, 75776)
    engine.rank_topk(U[:n_warm], V, topk, item_base=B, excl_indptr=ex_ptr[: n_warm + 1].contiguous(), excl_indices=ex_idx, workspace=ws)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    launches0 = int(L.b200_kernel_launches())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ids, sc = engine.rank_topk(U, V, topk, item_base=B, excl_indptr=ex_ptr, excl_indices=ex_idx, workspace=ws)
    e1.record()
    torch.cuda.synchronize()
    launches = int(L.b200_kernel_launches()) - launches0
    ms = over_ranks(e0.elapsed_time(e1))
    filled = float((ids[: min(n_q, 100000)] >= 0).float().mean().item())
    del ids, sc
    torch.cuda.empty_cache()
    # end to end: pinned host request (user ids + their exclusion CSR) -> H2D -> kernels -> D2H ids + scores
    nb_e = min(n_q, RANK_E2E_BATCH)
    n_batches = 2 if n_q >= 2 * nb_e else 1
    reqs = []
    for b in range(n_batches):
        lo = b * nb_e
        p = ex_ptr[lo: lo + nb_e + 1]
        base = int(p[0].item())
        reqs.append((torch.arange(lo, lo + nb_e, dtype=torch.int64).pin_memory(), (p - base).cpu().pin_memory(),
                     ex_idx[base: int(p[-1].item())].cpu().pin_memory()))
    o_i = torch.empty((nb_e, topk), dtype=torch.int32).pin_memory()
    o_s = torch.empty((nb_e, topk), dtype=torch.float32).pin_memory()

    def go_host(r):
        engine.rank_topk_host(U, V, topk, r[0].numpy(), item_base=B, excl_indptr=r[1].numpy(), excl_indices=r[2].numpy(),
                              out_ids=o_i.numpy(), out_scores=o_s.numpy(), workspace=ws)
    go_host(reqs[0])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r in reqs:
        go_host(r)
    torch.cuda.synchronize()
    ms_h = over_ranks((time.perf_counter() - t0) * 1e3)
    h2d = sum(r[0].numel() * 8 + r[1].numel() * 8 + r[2].numel() * 4 for r in reqs) / len(reqs)
    cpu = None
    if world == 1:
        try:                                                # a reported baseline, never a reason for the bench line to fail
            r = reference_rank_users_per_s(U[:4096].cpu().numpy(), V.cpu().numpy(), B.cpu().numpy(), topk)
            if r is not None:
                cpu = {"value": round(r[0], 1), "unit": "users/s", "cores": host_cores()["threads_used"], "kind": "reference",
                       "sample": "cornac.models.BPR.rank(u, k=%d) of the compiled reference for %d users of the same model "
                                 "(%d items, k=%d) in %.1fs, no exclusion list (OpenMP default thread count)" % (topk, r[1], n_items, k, r[2])}
        except Exception as exc:                            # noqa: BLE001
            cpu = {"unavailable": "%s: %s" % (type(exc).__name__, exc)}
    tf_peak, tf_src = tensor_peak()
    users_all = n_q * world
    tfl = 2.0 * k * n_items * users_all / (ms * 1e-3) / 1e12
    return {"metric": "ranked users/sec", "value": round(users_all / (ms * 1e-3), 1), "unit": "users/s", "n_gpus": world,
            "config": "BASELINE.json configs[4] on the trained bench model: all %d users (%d per rank) x %d items, k=%d, top-%d, "
                      "each user's train positives excluded" % (users_all, n_q, n_items, k, topk),
            "ms": round(ms, 3), "filled_frac_of_lists": round(filled, 4), "gpu_launches": launches,
            "roofline": {"kernel": "rank_tc_kernel (wgmma fp16 -> f32) + finish + packs", "bound": "tensor", "achieved": round(tfl, 1),
                         "peak": tf_peak * world, "unit": "TFLOP/s", "frac": round(tfl / (tf_peak * world), 4), "peak_source": tf_src,
                         "note": "2*k*n_items flop per user over the WHOLE call (pack + tensor pass + exact finish), all ranks"},
            "cpu_baseline": cpu,
            "e2e": {"value": round(world * nb_e * len(reqs) / (ms_h * 1e-3), 1), "unit": "users/s",
                    "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(nb_e * topk * 8), "ms_per_step": round(ms_h / len(reqs), 3),
                    "steps": len(reqs),
                    "path": "engine.rank_topk_host per rank, %d users per request: pinned user ids + exclusion CSR -> H2D -> "
                            "b200_rank_topk -> D2H ids + scores" % nb_e}}


def reference_mf_ratings_per_s(rid, cid, val, n_users, n_items, k, budget_s=8.0):
    """ratings/s of the UNMODIFIED reference kernel backend_cpu.fit_sgd (cornac/models/mf/backend_cpu.pyx:35-97) with the
    host threads this process owns on a bounded rating sample.  Returns (ratings/s, threads, epochs, seconds) or None."""
    ref = ref_path()
    if not os.path.isdir(os.path.join(ref, "cornac")):
        return None
    if ref not in sys.path:
        sys.path.insert(0, ref)
    from cornac.models.mf import backend_cpu
    rng = np.random.RandomState(5)
    n_u = int(rid.max()) + 1 if len(rid) else 1
    U = rng.normal(0, 0.01, (n_u, k)).astype(np.float32)
    V = rng.normal(0, 0.01, (n_items, k)).astype(np.float32)
    Bu, Bi = np.zeros(n_u, np.float32), np.zeros(n_items, np.float32)
    rid64, cid64 = np.ascontiguousarray(rid, dtype=np.int64), np.ascontiguousarray(cid, dtype=np.int64)
    val32 = np.ascontiguousarray(val, dtype=np.float32)
    threads = host_cores()["threads_used"]
    backend_cpu.fit_sgd(rid64[:100000], cid64[:100000], val32[:100000], U, V, Bu, Bi, 0.01, 0.02, 3.0, 1, threads, True, False, False)
    epochs, t0 = 0, time.perf_counter()
    while epochs < 1 or time.perf_counter() - t0 < budget_s / 2:
        backend_cpu.fit_sgd(rid64, cid64, val32, U, V, Bu, Bi, 0.01, 0.02, 3.0, 1, threads, True, False, False)
        epochs += 1
    secs = time.perf_counter() - t0
    return epochs * len(val32) / secs, threads, epochs, secs


def run_mf(W, engine, data, dev, world=1, over_ranks=lambda ms: ms, exchange="auto", steps=3):
    """BASELINE.json configs[3]: MF ratings/s (b200_mf_epoch, Hogwild + atomic scatter), k = 128, on the rating list made
    of the model's interactions with synthetic ratings in {1..5}, stored by user (CSR order); every rank trains its
    shard, V / Bi are replicated and all-reduced once per epoch like BPR's."""
    import torch
    import torch.distributed as dist
    from cornac_b200.parallel import make_item_sync
    k = 128
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    n = data.nnz
    rid = data.coo_row
    cid = data.indices
    val = torch.randint(1, 6, (n,), generator=g, device=dev).float()
    U = torch.randn((data.n_users, k), generator=g, device=dev) * 0.01
    gv = torch.Generator(device=dev)
    gv.manual_seed(6)
    V = torch.randn((W["n_items"], k), generator=gv, device=dev) * 0.01
    Bu, Bi = torch.zeros(data.n_users, device=dev), torch.zeros(W["n_items"], device=dev)
    loss = torch.zeros(1, device=dev)
    sync = make_item_sync([V, Bi], kind=exchange) if world > 1 else None

    def step():
        engine.mf_epoch(rid, cid, val, U, V, Bu, Bi, 0.01, 0.02, 3.0, True, loss)

    for _ in range(2):
        step()
        if sync is not None:
            sync.exchange()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    sync, _ = checked_item_sync(sync, [V, Bi], world)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for a, b in ev:
        a.record()
        step()
        b.record()
        if sync is not None:
            sync.exchange()
    e1.record()
    torch.cuda.synchronize()
    ms = over_ranks(e0.elapsed_time(e1) / steps)
    kms = over_ranks(float(np.mean([a.elapsed_time(b) for a, b in ev])))
    peak, _ = measured_peaks()
    gbs = n * (16 * k + 28) / (kms * 1e-3) / 1e9
    if sync is not None and hasattr(sync, "close"):
        torch.cuda.synchronize()
        sync.close()
    cpu = None
    if world == 1:
        try:                                                # a reported baseline, never a reason for the bench line to fail
            n_s = min(n, 10_000_000)                        # bounded sample: the first 10 M ratings (users in CSR order)
            r = reference_mf_ratings_per_s(rid[:n_s].cpu().numpy(), cid[:n_s].cpu().numpy(), val[:n_s].cpu().numpy(),
                                           data.n_users, W["n_items"], k)
            if r is not None:
                cpu = {"value": round(r[0], 1), "unit": "ratings/s", "cores": r[1], "kind": "reference",
                       "sample": "backend_cpu.fit_sgd of the compiled reference, %d epoch(s) over the first %d ratings of the same "
                                 "list (%d items, k=%d) in %.1fs" % (r[2], n_s, W["n_items"], k, r[3])}
        except Exception as exc:                            # noqa: BLE001
            cpu = {"unavailable": "%s: %s" % (type(exc).__name__, exc)}
    return {"metric": "MF ratings/sec", "cpu_baseline": cpu, "value": round(world * n / (ms * 1e-3), 1), "unit": "ratings/s", "n_gpus": world,
            "config": "BASELINE.json configs[3]: %d users x %d items x %d ratings (%d per rank), k=%d, use_bias, Hogwild + red.global.add, "
                      "item replicas all-reduced once per epoch" % (W["n_users"], W["n_items"], W["nnz"], n, k),
            "ms_per_epoch": round(ms, 3), "steps": steps,
            "roofline": {"kernel": "mf_hogwild_kernel", "bound": "hbm", "achieved": round(gbs, 1), "peak": peak, "unit": "GB/s",
                         "frac": round(gbs / peak, 4), "kernel_ms": round(kms, 3), "algorithmic_bytes_per_rating": 16 * k + 28,
                         "note": "slowest rank's kernel launches"}}


def run_reference_arm(args, W, world, out_stream):
    """--impl reference: the reference's own CPU kernel on a bounded sample of the workload."""
    import torch
    k = W["k"]
    ub, nb = block_shape(W)
    if torch.cuda.is_available():
        indptr, indices = synth_interactions(ub, W["n_items"], nb, seed=1234, device=torch.device("cuda", 0), item_seed=ITEM_SEED)
        ip, ix = cpu_sample_csr(indptr.cpu().numpy(), indices.cpu().numpy())
        del indptr, indices
    else:   # no GPU: generate the sample directly at sample size
        n_u = min(CPU_SAMPLE["n_users"], ub)
        ipt, ixt = synth_interactions(n_u, W["n_items"], int(nb * (n_u / ub)), seed=1234, device=torch.device("cpu"), item_seed=ITEM_SEED)
        ip, ix = ipt.numpy(), ixt.numpy()
    run, kind, cores = reference_fit_sgd_runner(ip, ix, W["n_items"], k, W["lr"], W["reg"], 0)
    nnz = len(ix)
    for _ in range(max(1, min(args.warmup, 2))):
        run()
    t0 = time.perf_counter()
    upd = 0
    steps = args.steps
    for _ in range(steps):
        c, s = run()
        upd += nnz - s
    dt = time.perf_counter() - t0
    v = upd / dt
    sample = "first %d users of block 0 of the matrix: %d interactions, %d items, k=%d" % (len(ip) - 1, nnz, W["n_items"], k)
    out = {"impl": "reference", "metric": "BPR triplet-updates/sec", "value": round(v, 1), "unit": "updates/s",
           "n_gpus": args.gpus, "steps": steps, "warmup": args.warmup, "ms_per_step": round(dt / steps * 1e3, 2),
           "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
           "config": {"workload": workload_text(W, world) + "; each step = one _fit_sgd epoch over a bounded sample: " + sample},
           "cpu_baseline": {"value": round(v, 1), "unit": "updates/s", "cores": cores, "kind": kind, "sample": sample, "host": host_cores()},
           "e2e": {"value": round(v, 1), "unit": "updates/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
           "gpu_launches": 0}
    if args.scale != 1.0:
        out["INVALID"] = "scaled-down debug run (--scale %g)" % args.scale
    out_stream.write(json.dumps(out) + "\n")
    out_stream.flush()
    return 0


if __name__ == "__main__":
    sys.exit(main())
