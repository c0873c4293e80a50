"""The multi-GPU item-replica exchange, checked exactly on one GPU.

Both exchange paths set every replica to  snapshot + mean over the ranks that changed the element of (x_r - snapshot)
(mean_touched = 0: the plain sum):
  * b200_item_exchange (csrc/p2p.cu, parallel.PeerItemExchange, the default with NCCL).  Rank r's kernel reads and rewrites
    only its own slice [lo_r, hi_r) of every replica, and the slices are disjoint: the W rank kernels launched one after
    another on one stream, with all W replicas and flag buffers on this device, leave exactly the memory W concurrent ranks
    leave.  The flag waits are met without concurrency: before exchange `seq`, flag buffer b gets `seq` preset in the words
    of the ranks r' > b (in a concurrent run they would already have published; here they launch after b), and the kernels
    write the rest.  With correct code no wait spins; a missing publication runs into the kernel's own bound (~4 s) and
    sets the error word, which the emulation asserts on.
  * b200_delta_make / b200_delta_apply (csrc/api.cu, parallel.ItemReplicaSync) around an all-reduce.

Every result is compared bit for bit with a host restatement in float32, one IEEE operation at a time in the kernel's order
(the library is built without fast-math: IEEE division, subnormals kept, no multiply-add to contract).  The only slack is
a NaN's payload: the device's arithmetic NaN is not the host's.  Ordering and visibility across GPUs over NVLink, the IPC
mapping and the timeout path are not exercised here: they rest on tools/mgpu_check.py, run on a multi-GPU machine."""
import ctypes

import numpy as np
import pytest

from conftest import rel_err
from oracle import oracle as O

pytestmark = pytest.mark.gpu

F32 = np.float32
WORLDS = (1, 2, 3, 4, 5, 7, 8)
N_ITEMS, K = 1001, 33                    # a V-shaped vector (n_items x k, k odd) and its B-shaped bias vector
GUARD = 16                               # guard floats on each side of every replica
GUARD_BITS = 0x7FC0BEEF                  # a NaN payload no kernel writes
TINY = F32(2.0 ** -127)                  # subnormal
POOL = np.random.RandomState(0).standard_normal(1 << 21).astype(F32)      # local changes are cut from this


def _bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.uint32)


def _same(a, b):
    """Bit-equal, signed zeros included, except that any NaN matches any NaN."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(_bits(a)[~na], _bits(b)[~nb])


def _addr(t):
    """The device address of a view, also of an empty one (whose data_ptr() is 0)."""
    return t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()


def _replica(n, offset=0):
    """(buffer, view): a float32 CUDA view of n elements `offset` floats past a 16-byte boundary, between guard floats."""
    import torch
    buf = torch.full((n + 2 * GUARD + 3,), GUARD_BITS, dtype=torch.int32, device="cuda").view(torch.float32)
    view = buf[GUARD + offset:GUARD + offset + n]
    assert _addr(view) % 16 == 4 * offset
    return buf, view


def _guards_intact(buf, n, offset=0):
    b = _bits(buf.cpu().numpy())
    return (np.all(b[:GUARD + offset] == GUARD_BITS) and np.all(b[GUARD + offset + n:] == GUARD_BITS))


def _upload(view, host):
    import torch
    view.copy_(torch.from_numpy(np.ascontiguousarray(host, dtype=F32)))


class _Exchange:
    """PeerItemExchange's state for every rank of one tensor, all on this device: the replica and flag pointer arrays, each
    rank's slice and its snapshot of it.  exchange() launches the rank kernels 0 .. W-1 one after another."""

    def __init__(self, xs, mean_touched):
        import torch
        from cornac_b200 import _lib
        self.L, self.check = _lib.load(), _lib.check
        self.xs, self.world, self.n, self.mean = list(xs), len(xs), xs[0].numel(), int(mean_touched)
        self.flags = [torch.zeros(32, dtype=torch.int32, device="cuda") for _ in self.xs]
        self.x_ptrs = (ctypes.c_void_p * self.world)(*[_addr(x) for x in self.xs])
        self.f_ptrs = (ctypes.c_void_p * self.world)(*[f.data_ptr() for f in self.flags])
        self.slices, self.snaps = [], []
        for r, x in enumerate(self.xs):
            lo, hi = ctypes.c_int64(), ctypes.c_int64()
            self.check(self.L.b200_item_exchange_slice(r, self.world, self.n, ctypes.byref(lo), ctypes.byref(hi)),
                       "b200_item_exchange_slice")
            lo, hi = lo.value, hi.value
            self.slices.append((lo, hi))
            self.snaps.append(x.view(-1)[lo:hi].clone() if hi > lo else torch.zeros(4, device=x.device))
        # the slices tile [0, n) in rank order and start at multiples of 4 floats
        assert self.slices[0][0] == 0 and self.slices[-1][1] == self.n
        assert all(a[1] == b[0] for a, b in zip(self.slices, self.slices[1:]))
        assert all(lo % 4 == 0 or lo == self.n for lo, _ in self.slices)
        self.seq = 0

    def exchange(self):
        import torch
        from cornac_b200._lib import current_stream
        self.seq += 1
        W = self.world
        for b, f in enumerate(self.flags):       # what the ranks launched after b would already have published
            for phase in (0, 1):
                f[phase * 8 + b + 1:phase * 8 + W] = self.seq
        for r in range(W):
            self.check(self.L.b200_item_exchange(r, W, self.x_ptrs, self.f_ptrs, self.snaps[r].data_ptr(), self.n, self.seq,
                                                 self.mean, current_stream()), "b200_item_exchange")
        torch.cuda.synchronize()
        # every rank published both phases into every buffer (buffer W-1 had nothing preset), the done counters are back
        # at 0 and no wait ran out
        want = np.zeros(32, np.int32)
        want[:W] = want[8:8 + W] = self.seq
        for b, f in enumerate(self.flags):
            got = f.cpu().numpy()
            assert np.array_equal(got, want), (b, got.tolist())


class _DeltaExchange:
    """ItemReplicaSync's exchange for every rank of one tensor on this device: delta_make on each replica, the sum of the
    deltas and their touched count in rank order in float32 on the host (the all-reduce), the division, delta_apply on
    each replica.  The snapshots are full copies, as ItemReplicaSync keeps them."""

    def __init__(self, xs, mean_touched):
        import torch
        self.xs, self.mean = list(xs), bool(mean_touched)
        self.snaps = [x.clone() for x in self.xs]
        self.deltas = [torch.empty_like(x) for x in self.xs]

    def exchange(self):
        from cornac_b200 import engine
        for x, s, d in zip(self.xs, self.snaps, self.deltas):
            engine.delta_make(x, s, d)
        ds = [d.cpu().numpy() for d in self.deltas]
        tot, cnt = ds[0].copy(), (ds[0] != 0).astype(F32)
        with np.errstate(invalid="ignore", over="ignore"):
            for d in ds[1:]:
                tot = tot + d
                cnt = cnt + (d != 0).astype(F32)
            if self.mean:
                tot = tot / np.maximum(cnt, F32(1))
        for x, s, d in zip(self.xs, self.snaps, self.deltas):
            _upload(d, tot)
            engine.delta_apply(x, s, d)


def _rule(s, xs, mean_touched):
    """The exchange's element rule in float32, in the kernel's order."""
    s = np.asarray(s, F32)
    d, c = np.zeros_like(s), np.zeros_like(s)
    with np.errstate(invalid="ignore", over="ignore"):
        for x in xs:
            dx = x - s
            d = d + dx
            c = c + (dx != 0).astype(F32)
        if mean_touched:
            d = np.divide(d, c, out=d.copy(), where=c > 1)
        return s + d


def _rule_f64_ok(s, xs, mean_touched, got):
    """The rule in float64 (start + mean / sum of the changes) bounds the float32 result where every value is moderate."""
    s64, x64 = s.astype(np.float64), [x.astype(np.float64) for x in xs]
    with np.errstate(invalid="ignore", over="ignore"):
        dx = [x - s64 for x in x64]
        tot, cnt, mag = sum(dx, np.zeros_like(s64)), sum((d != 0 for d in dx), np.zeros_like(s64)), np.abs(s64)
        for d in dx:
            mag = mag + np.abs(d)
        want = s64 + (tot / np.maximum(cnt, 1) if mean_touched else tot)
        ok = np.isfinite(mag) & (mag < 1e20)
        err = np.abs(got.astype(np.float64) - want)
    tol = 16 * (len(xs) + 1) * np.finfo(F32).eps * mag
    return bool(np.all(err[ok] <= tol[ok]))


# ---- per-rank changes --------------------------------------------------------------------------------------------------
# Special elements: each kind sits at two positions per exchange, one near the head (in rank 0's float4 range) and one
# near the end, from the last element but one down (the first two kinds of exchange 1 land in the last slice's scalar
# tail when n % 4 == 3; the last element stays an ordinary one).  Outside their own exchange every rank leaves them alone.
def _k_equal(c, r, w, seq):          # the ranks write back the value they found (not a change); the last one changes it
    return c + F32(0.25) if r == w - 1 and w > 1 else c


def _k_pos_zero(c, r, w, seq):       # from +0: rank 0 writes -0 (not a change), the last rank 0.5 (the only change)
    return F32(0.5) if r == w - 1 and w > 1 else (-c if c == 0 else c)


def _k_neg_zero(c, r, w, seq):       # from -0 (+0 once an earlier exchange passed it): rank 0 flips the sign only
    return F32(-0.75) if r == w - 1 and w > 1 else (-c if c == 0 else c)


def _k_subnormal(c, r, w, seq):      # one rank changes the value by a subnormal difference: a change
    return c - TINY if r == seq % w else c


def _k_subnormal2(c, r, w, seq):     # two ranks' subnormal differences, averaged
    return c - TINY * F32(r + 1) if r in (0, w - 1) else c


def _k_cancel(c, r, w, seq):         # large changes that cancel; the sum's order decides whether the third one survives
    return {0: c + F32(3e37), 1: c - F32(3e37), 2: c + F32(1e30)}.get(r, c) if w > 1 else c + F32(3e37)


def _k_inf(c, r, w, seq):
    return F32(np.inf) if r == w - 1 else c


def _k_nan(c, r, w, seq):
    return F32(np.nan) if r == w - 1 else c


def _k_infs(c, r, w, seq):           # -inf and +inf into the same element: NaN (with one rank: +inf)
    return F32(np.inf) if r == w - 1 else (F32(-np.inf) if r == 0 else c)


KINDS = (_k_equal, _k_pos_zero, _k_neg_zero, _k_subnormal, _k_subnormal2, _k_cancel, _k_inf, _k_nan, _k_infs)
START = {_k_pos_zero: F32(0.0), _k_neg_zero: F32(-0.0), _k_subnormal: F32(1.5 * 2.0 ** -126), _k_subnormal2: F32(2.0 ** -125)}


def _positions(n, seq, j):
    h = (seq - 1) * len(KINDS) + j
    return sorted({h % n, (n - 2 - h) % n}) if n else []


def _reserved(n):
    return np.array(sorted({p for seq in (1, 2, 3) for j in range(len(KINDS)) for p in _positions(n, seq, j)}), np.int64)


def _start(n, seed=1):
    x = np.random.RandomState(seed).standard_normal(n).astype(F32)
    for seq in (1, 2, 3):
        for j, kind in enumerate(KINDS):
            for p in _positions(n, seq, j):
                if kind in START:
                    x[p] = START[kind]
    return x


def _local(cur, world, k, seq):
    """Every rank's replica after its local epoch of exchange `seq`, from the common value `cur`.  Whole k-rows change: row i
    by (i + seq) % (world + 1) of the ranks, a run of consecutive ranks starting at rank i % world, so that every count
    0 .. world occurs and the ranks change different rows; in exchange 2, rank 1 (rank 0 alone) changes nothing."""
    n = cur.size
    rows = np.arange(n) // k
    hits = (rows + seq) % (world + 1)
    res = _reserved(n)
    xs = []
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(world):
            x = cur.copy()
            if not (seq == 2 and r == 1 % world):
                mine = (r - rows) % world < hits
                off = (7919 * r + 104729 * seq) % (POOL.size - n + 1)
                x[mine] = cur[mine] + POOL[off:off + n][mine] * F32(0.01 * (r + 1))
                x[res] = cur[res]
                for j, kind in enumerate(KINDS):
                    for p in _positions(n, seq, j):
                        x[p] = kind(cur[p], r, world, seq)
            xs.append(x)
    return xs


def _n_cases():
    """(n, row width): empty and short slices, 4 * world - 1, the V- and B-shaped vectors, several blocks per rank."""
    return [("0", lambda w: (0, 1)), ("1", lambda w: (1, 1)), ("3", lambda w: (3, 1)), ("4w-1", lambda w: (4 * w - 1, 1)),
            ("V", lambda w: (N_ITEMS * K, K)), ("B", lambda w: (N_ITEMS, 1)), ("1000003", lambda w: (1_000_003, 1))]


def _run(world, n, k, mean, offsets=None):
    """Three exchanges of `world` emulated ranks from _start(n), each checked against the restatement; returns the common
    value after each exchange."""
    offsets = offsets or [0] * world
    cur = _start(n)
    reps = [_replica(n, o) for o in offsets]
    for _, x in reps:
        _upload(x, cur)
    ex = _Exchange([x for _, x in reps], mean)
    out = []
    for seq in (1, 2, 3):
        xs = _local(cur, world, k, seq)
        for (_, x), v in zip(reps, xs):
            _upload(x, v)
        ex.exchange()
        want = _rule(cur, xs, mean)
        got = [x.cpu().numpy() for _, x in reps]
        for r, g in enumerate(got):
            assert np.array_equal(_bits(g), _bits(got[0])), "replica %d differs from replica 0 after exchange %d" % (r, seq)
        assert _same(got[0], want), "exchange %d: %d elements differ from the restatement" % (
            seq, int(np.sum(_bits(got[0]) != _bits(want))))
        assert _rule_f64_ok(cur, xs, mean, got[0])
        for r, ((lo, hi), snap) in enumerate(zip(ex.slices, ex.snaps)):
            s = snap.cpu().numpy()
            assert np.array_equal(_bits(s), _bits(got[0][lo:hi]) if hi > lo else np.zeros(4, np.uint32)), (r, seq)
        for (buf, _), o in zip(reps, offsets):
            assert _guards_intact(buf, n, o)
        cur = got[0]
        out.append(cur)
    return out


@pytest.mark.parametrize("mean", [1, 0])
@pytest.mark.parametrize("case", [c for c, _ in _n_cases()])
@pytest.mark.parametrize("world", WORLDS)
def test_p2p_exchange_matches_float32_restatement(world, case, mean):
    n, k = dict(_n_cases())[case](world)
    _run(world, n, k, mean)


OFFSETS = {"all+1": lambda w: [1] * w, "all+2": lambda w: [2] * w, "all+3": lambda w: [3] * w,
           "mixed": lambda w: [r % 4 for r in range(w)], "last+3": lambda w: [0] * (w - 1) + [3]}


@pytest.mark.parametrize("world,pattern,case", [(w, p, c) for w in WORLDS for p in OFFSETS for c in ("4w-1", "V")
                                                if any(OFFSETS[p](w))] + [(w, "mixed", "1000003") for w in WORLDS[1:]])
def test_p2p_exchange_unaligned_replicas_match_aligned_run(world, pattern, case):
    """Replicas that are views at a storage offset (a bias vector carved out of a packed buffer) take the scalar loop:
    the result is bit-identical to the aligned run on the same values."""
    offsets = OFFSETS[pattern](world)
    n, k = dict(_n_cases())[case](world)
    aligned = _run(world, n, k, 1)
    shifted = _run(world, n, k, 1, offsets)
    for a, b in zip(aligned, shifted):
        assert np.array_equal(_bits(a), _bits(b))


# ---- the delta kernels -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offsets", [(0, 0, 0), (1, 1, 1), (2, 2, 2), (3, 3, 3), (1, 0, 0), (0, 2, 0), (0, 0, 3)])
@pytest.mark.parametrize("n", [1, 3, 4, 5, 1_000_003])
def test_delta_kernels_match_float32(n, offsets):
    """delta_make: delta = x - snapshot; delta_apply: x = snapshot = snapshot + delta, both over x.numel() elements.  The
    snapshot and delta buffers are longer than x: their excess is untouched.  A view off a 16-byte boundary in any of the
    three arguments takes the scalar loop."""
    from cornac_b200 import engine
    extra = 5
    (xb, x), (sb, s), (db, d) = _replica(n, offsets[0]), _replica(n + extra, offsets[1]), _replica(n + extra, offsets[2])
    s0 = np.concatenate([_start(n, seed=2), np.arange(1, extra + 1, dtype=F32)])
    x0 = _local(s0[:n], 3, 2, 1)[0]                    # rank 0's changes: rows, +0 -> -0, a subnormal step, -inf, ...
    if n > 4:
        x0[n // 2 + 1] = np.nan
    d0 = np.full(n + extra, 7.0, F32)
    for v, h in ((x, x0), (s, s0), (d, d0)):
        _upload(v, h)
    engine.delta_make(x, s, d)
    with np.errstate(invalid="ignore", over="ignore"):
        want_d = x0 - s0[:n]
    got_d = d.cpu().numpy()
    assert _same(got_d[:n], want_d) and np.array_equal(got_d[n:], d0[n:])
    assert np.array_equal(_bits(x.cpu().numpy()), _bits(x0)) and np.array_equal(_bits(s.cpu().numpy()), _bits(s0))
    # apply a reduced delta: halves, NaN and subnormals included
    with np.errstate(invalid="ignore", over="ignore"):
        red = np.concatenate([want_d * F32(0.5), np.full(extra, 9.0, F32)])
    red[n // 2] = TINY
    _upload(d, red)
    engine.delta_apply(x, s, d)
    with np.errstate(invalid="ignore", over="ignore"):
        want = s0[:n] + red[:n]
    got_x, got_s = x.cpu().numpy(), s.cpu().numpy()
    assert _same(got_x, want) and _same(got_s[:n], want) and np.array_equal(_bits(got_s[n:]), _bits(s0[n:]))
    assert np.array_equal(_bits(d.cpu().numpy()), _bits(red))
    for buf, m, o in ((xb, n, offsets[0]), (sb, n + extra, offsets[1]), (db, n + extra, offsets[2])):
        assert _guards_intact(buf, m, o)


# ---- the two paths agree -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mean", [1, 0])
@pytest.mark.parametrize("world", WORLDS)
def test_both_exchange_paths_agree_bit_for_bit(world, mean):
    """The peer-memory kernel and the delta kernels around a reduction give the same bits for the same local changes.  A
    real NCCL all-reduce sums in an order of its own choosing; the reduction here sums in rank order, the peer kernel's
    order, so that what is compared is the element rule the two device paths implement."""
    n, k = N_ITEMS * K + 2, K
    cur = _start(n)
    a, b = [_replica(n)[1] for _ in range(world)], [_replica(n)[1] for _ in range(world)]
    for x in a + b:
        _upload(x, cur)
    pa, pb = _Exchange(a, mean), _DeltaExchange(b, mean)
    for seq in (1, 2, 3):
        xs = _local(cur, world, k, seq)
        for x, y, v in zip(a, b, xs):
            _upload(x, v)
            _upload(y, v)
        pa.exchange()
        pb.exchange()
        got = a[0].cpu().numpy()
        assert _same(got, _rule(cur, xs, mean))
        for y, s in zip(b, pb.snaps):
            assert _same(y.cpu().numpy(), got) and _same(s.cpu().numpy(), got)
        cur = got


# ---- composition with the MF epoch -------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_mf_epochs_through_the_exchange(world):
    """parallel.mf_fit_sharded's epochs on one GPU: every rank runs the ordered MF epoch on its users' U / Bu rows and its
    own replica of V / Bi, then [V, Bi] go through the emulated peer exchange (and, on a second copy of everything, through
    the delta kernels).  Against the oracle's serial epoch per shard followed by the float32 rule."""
    import torch
    from cornac_b200 import engine, parallel
    rng = np.random.RandomState(11)
    n_users, n_items, k, n = 301, 1001, 10, 8000
    lr, reg, mu = 0.01, 0.02, 3.0
    pop = 1.0 / np.arange(1, n_items + 1) ** 0.9        # popular items trained by every shard, the tail by few
    rid = rng.randint(n_users, size=n).astype(np.int64)
    cid = rng.choice(n_items, size=n, p=pop / pop.sum()).astype(np.int64)
    val = rng.randint(1, 6, size=n).astype(F32)
    U0, V0, Bu0, Bi0 = O.mf_init(4, n_users, n_items, k)
    Bu0 = rng.normal(0, 0.1, n_users).astype(F32)
    Bi0 = rng.normal(0, 0.1, n_items).astype(F32)
    bounds = parallel.shard_ratings_by_user(rid, n_users, world)
    shards = [parallel.shard_ratings(rid, cid, val, bounds, r) for r in range(world)]
    dshards = [tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in s) for s in shards]
    dev = lambda a: torch.from_numpy(a.copy()).cuda()  # noqa: E731

    paths = []
    for kind in (_Exchange, _DeltaExchange):
        st = dict(U=[dev(U0) for _ in range(world)], Bu=[dev(Bu0) for _ in range(world)],
                  V=[dev(V0) for _ in range(world)], Bi=[dev(Bi0) for _ in range(world)],
                  loss=[torch.zeros(1, dtype=torch.float32, device="cuda") for _ in range(world)])
        st["sync"] = [kind([v.view(-1) for v in st["V"]], 1), kind(st["Bi"], 1)]
        paths.append(st)
    Uh, Buh = [U0.copy() for _ in range(world)], [Bu0.copy() for _ in range(world)]
    Vh, Bih = V0.copy(), Bi0.copy()
    for epoch in range(3):
        for st in paths:
            for r in range(world):
                lo, hi = int(bounds[r]), int(bounds[r + 1])
                engine.mf_epoch(*dshards[r], st["U"][r][lo:hi], st["V"][r], st["Bu"][r][lo:hi], st["Bi"][r], lr, reg, mu,
                                True, st["loss"][r], ordered=True)
            for sync in st["sync"]:
                sync.exchange()
        Vs, Bis, losses = [], [], []
        for r in range(world):
            lo, hi = int(bounds[r]), int(bounds[r + 1])
            Vr, Bir = Vh.copy(), Bih.copy()
            losses.append(O.mf_epoch(*shards[r], Uh[r][lo:hi], Vr, Buh[r][lo:hi], Bir, lr, reg, mu, True))
            Vs.append(Vr)
            Bis.append(Bir)
        Vh, Bih = _rule(Vh, Vs, 1), _rule(Bih, Bis, 1)
        p2p, delta = paths
        for name in ("V", "Bi", "U", "Bu"):
            for r in range(world):
                assert np.array_equal(_bits(p2p[name][r].cpu().numpy()), _bits(delta[name][r].cpu().numpy())), (epoch, name, r)
        V, Bi = p2p["V"][0].cpu().numpy(), p2p["Bi"][0].cpu().numpy()
        for r in range(1, world):
            assert np.array_equal(_bits(p2p["V"][r].cpu().numpy()), _bits(V))
            assert np.array_equal(_bits(p2p["Bi"][r].cpu().numpy()), _bits(Bi))
        assert rel_err(V, Vh) < 1e-4 and np.allclose(V, Vh, rtol=1e-4, atol=1e-6), epoch
        assert rel_err(Bi, Bih) < 1e-4, epoch
        for r in range(world):
            lo, hi = int(bounds[r]), int(bounds[r + 1])
            U, Bu = p2p["U"][r].cpu().numpy(), p2p["Bu"][r].cpu().numpy()
            assert rel_err(U[lo:hi], Uh[r][lo:hi]) < 1e-4 and rel_err(Bu[lo:hi], Buh[r][lo:hi]) < 1e-4
            outside = np.r_[0:lo, hi:n_users]
            assert np.array_equal(_bits(U[outside]), _bits(U0[outside])) and np.array_equal(_bits(Bu[outside]), _bits(Bu0[outside]))
            assert abs(0.5 * p2p["loss"][r].item() - losses[r]) <= 1e-4 * losses[r]
    # the exchange saw partial counts: some items were trained by some shards only
    seen = np.stack([np.bincount(s[1], minlength=n_items) > 0 for s in shards]).sum(axis=0)
    assert np.any(seen == 1) and np.any(seen == world) and np.any(seen == 0)
