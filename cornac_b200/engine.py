"""Device-side engine: thin, typed Python wrappers over the C ABI.

Everything here operates on torch CUDA tensors used as plain device buffers.  The
functions mirror the reference kernels one to one (see include/b200cornac.h):
    bpr_epoch / bpr_epoch_replay   <-> BPR._fit_sgd          (cornac/models/bpr/recom_bpr.pyx:208-269)
    MTSampler                      <-> RNGVector             (cornac/models/bpr/recom_bpr.pyx:54-62)
    mf_epoch                       <-> backend_cpu.fit_sgd   (cornac/models/mf/backend_cpu.pyx:58-83)
    score_batch                    <-> fast_dot              (cornac/utils/fast_dot.pyx:40-43)
    topk_rows / rank_topk          <-> Recommender.rank      (cornac/models/recommender.py:476-530)
    knn_similarity / knn_score     <-> compute_similarity / compute_score (cornac/models/knn/similarity.pyx)
    pmf_schedule / pmf_fit         <-> pmf_linear / pmf_non_linear (cornac/models/pmf/cython/pmf.pyx:55-173)
    cofactor_schedule / cofactor_fit <-> sorec / mcf (cornac/models/sorec/cython/sorec.pyx, cornac/models/mcf/cython/mcf.pyx)
    score_batch_f64 / topk_rows_f64 <-> PMF.score / Recommender.rank (cornac/models/pmf/recom_pmf.py:191-222)
    NmfData / nmf_fit              <-> NMF._fit_sgd          (cornac/models/nmf/recom_nmf.pyx:182-267)
    ease_fit / ease_score          <-> EASE.fit / EASE.score (cornac/models/ease/recom_ease.py:57-126)
    hpf_fit / hpf_update / hpf_expect <-> hpf_cpp / pf_cpp   (cornac/models/hpf/cpp/cpp_hpf.cpp:139-275)
    c2pf_fit / c2pf_update  <-> c2pf_cpp / tc2pf_cpp / rc2pf_cpp  (cornac/models/c2pf/cpp/cpp_c2pf.cpp)
    efm_fit / efm_queries   <-> EFM._fit_efm / EFM.rank  (cornac/models/efm/recom_efm.pyx:268-353, 471-528)
    mter_fit / mter_queries <-> MTER._fit_mter / MTER.score (cornac/models/mter/recom_mter.pyx:434-714)
    comparer_sub_fit / comparer_rank_rows <-> ComparERSub._fit_mter / rank (recom_comparer_sub.pyx:487-806)
    lrppm_fit / lrppm_rank_rows <-> LRPPM._fit / LRPPM.rank (cornac/models/lrppm/recom_lrppm.pyx:356-560)
"""
import ctypes

import numpy as np
import scipy.sparse as _sp
import torch

from . import _lib
from ._lib import B200Error, check, current_stream, ptr


def require_cuda():
    if not torch.cuda.is_available():
        raise B200Error("cornac_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    return _lib.load()


def warmup():
    """Create the CUDA context and load libb200cornac.so now instead of inside the first fit()/rank() (a fresh process
    pays seconds for the context; an experiment that times its models should not charge that to whichever runs first)."""
    L = require_cuda()
    torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    return L


class _AtLeast(int):
    """A minimum size in a shape _dev checks: the kernel reads only a prefix of that extent."""


def _fits(n, want):
    return want is None or (n >= want if type(want) is _AtLeast else n == want)


def _size_str(want):
    return "*" if want is None else (">=%d" if type(want) is _AtLeast else "%d") % want


def _dev(t, dtype, name, shape=None):
    """t, checked to be a contiguous CUDA tensor of `dtype` and, when `shape` is given, of that shape: a tuple with per
    dimension an exact size, an _AtLeast or None (any size); or one size (exact or _AtLeast), the element count of a
    flat buffer.  The C entry points take raw pointers: these are the only checks of the extents they index."""
    if isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous():
        if shape is None:
            return t
        if type(shape) is not tuple:
            if _fits(t.numel(), shape):
                return t
        elif len(t.shape) == len(shape) and all(map(_fits, t.shape, shape)):
            return t
    if shape is None:
        want = ""
    elif isinstance(shape, tuple):
        want = " and shape (%s)" % ", ".join(map(_size_str, shape))
    else:
        want = " and shape [%s elements]" % _size_str(shape)
    got = ("a %s tensor of dtype %s and shape %s" % (t.device, t.dtype, tuple(t.shape)) if isinstance(t, torch.Tensor)
           else type(t).__name__)
    raise B200Error("%s must be a contiguous CUDA tensor of dtype %s%s, got %s" % (name, dtype, want, got))


def _buf(t, dtype, name, shape, zero=False):
    """An optional caller buffer: t checked by _dev when given, else a new CUDA tensor of `shape` (zeros when `zero`;
    a flat buffer gets at least one element, as no device buffer here is zero-size)."""
    if t is None:
        return (torch.zeros if zero else torch.empty)(shape if isinstance(shape, tuple) else max(int(shape), 1),
                                                      dtype=dtype, device="cuda")
    return _dev(t, dtype, name, shape)


def _f32(x):
    """x rounded to f32, as the reference's C `float` / `floating` parameters hold it."""
    return float(np.float32(x))


def to_device(a, dtype=None, pinned=True):
    """H2D copy of a numpy array (through pinned memory) -> CUDA tensor."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if pinned:
        t = t.pin_memory()
    return t.cuda(non_blocking=True)


def _pad(a):
    """a, or one zero of its dtype when it is empty (no zero-size device buffers)."""
    return a if len(a) else np.zeros(1, a.dtype)


class BprData:
    """Device copy of train_set.matrix: the CSR arrays (indptr int32 [n_users+1], sorted indices
    int32 [nnz]) + the COO row array (BPR._prepare_data, recom_bpr.pyx:154-161) used by the
    parity kernel, and -- built on first use by b200_bpr_prepare -- the (pairs, membership
    table) store the throughput kernel gathers from."""

    def __init__(self, indptr, indices, coo_row=None):
        self.indptr = _dev(indptr, torch.int32, "indptr")
        self.indices = _dev(indices, torch.int32, "indices")
        self.n_users = self.indptr.numel() - 1
        self.nnz = self.indices.numel()
        self._coo_row = None if coo_row is None else _dev(coo_row, torch.int32, "coo_row", self.nnz)
        self.pairs = self.table = None

    @property
    def coo_row(self):
        if self._coo_row is None:
            counts = (self.indptr[1:] - self.indptr[:-1]).to(torch.int64)
            self._coo_row = torch.repeat_interleave(
                torch.arange(self.n_users, device=self.indptr.device, dtype=torch.int32), counts)
        return self._coo_row

    def prepare(self):
        """Build pairs + membership table (idempotent)."""
        if self.pairs is None:
            L = require_cuda()
            slots = int(L.b200_bpr_table_slots(self.nnz))
            pairs = torch.empty((max(self.nnz, 1), 2), dtype=torch.int32, device=self.indptr.device)
            table = torch.empty(slots, dtype=torch.int64, device=self.indptr.device)
            check(L.b200_bpr_prepare(ptr(self.indptr), ptr(self.indices), self.n_users, self.nnz, ptr(pairs),
                                     ptr(table), slots, current_stream()), "b200_bpr_prepare")
            self.pairs, self.table = pairs, table
        return self

    @classmethod
    def from_host(cls, indptr, indices):
        if len(indices) >= 2 ** 31:
            raise B200Error("nnz >= 2^31 per shard is not supported (int32 CSR offsets)")
        return cls(to_device(np.asarray(indptr), torch.int32), to_device(np.asarray(indices), torch.int32))


def bpr_epoch(data, n_neg, U, V, B, lr, reg, use_bias, seed, epoch, stats, n_samples=None,
              sample_base=0, atomic=True, exact_exp=False, unbounded=False, neg_weighted=False, hinge=False, blocked=False,
              deterministic=False):
    """One Hogwild BPR epoch on the current stream; `stats` (int64[2] CUDA) accumulates
    (correct, skipped).  deterministic=True: rounds of samples that read the factors as the previous round left them,
    their updates summed exactly -- the result repeats bit for bit from run to run."""
    L = require_cuda()
    k = _dev(U, torch.float32, "U", (_AtLeast(data.n_users), None)).shape[1]
    _dev(V, torch.float32, "V", (_AtLeast(n_neg), k)), _dev(B, torch.float32, "B", _AtLeast(n_neg))
    _dev(stats, torch.int64, "stats", _AtLeast(2))
    flags = ((_lib.SGD_ATOMIC if atomic else 0) | (_lib.SGD_EXACT_EXP if exact_exp else 0)
             | (_lib.SGD_UNBOUNDED if unbounded else 0) | (_lib.BPR_NEG_WEIGHTED if neg_weighted else 0)
             | (_lib.BPR_LOSS_HINGE if hinge else 0) | (_lib.BPR_BLOCKED if blocked else 0)
             | (_lib.BPR_DETERMINISTIC if deterministic else 0))
    n = data.nnz if n_samples is None else int(n_samples)
    data.prepare()
    check(L.b200_bpr_epoch(ptr(data.pairs), ptr(data.table), data.table.numel(), data.nnz, data.n_users, int(n_neg), n,
                           ptr(U), ptr(V), ptr(B), int(k), float(lr), float(reg), int(bool(use_bias)),
                           int(seed) & (2 ** 64 - 1), int(epoch), int(sample_base), flags, ptr(stats),
                           current_stream()), "b200_bpr_epoch")


def bpr_block_plan(n_users, n_neg, k):
    """(windows of the interaction list, item blocks) of the cache-blocked sample order for this model size."""
    import ctypes
    L = _lib.load()
    a, b = ctypes.c_uint32(), ctypes.c_uint32()
    check(L.b200_bpr_block_plan(int(n_users), int(n_neg), int(k), ctypes.byref(a), ctypes.byref(b)), "b200_bpr_block_plan")
    return a.value, b.value


def bpr_draw_host(seed, epoch, n, nnz, n_neg, sample_base=0, plan=(1, 1)):
    """The (i_index, j_id) stream that bpr_epoch(seed, epoch) consumes, computed on the host (plan = bpr_block_plan(...)
    for an epoch run with blocked=True)."""
    L = _lib.load()
    ii = np.empty(n, dtype=np.int64)
    jj = np.empty(n, dtype=np.int32)
    check(L.b200_bpr_draw_host2(int(seed) & (2 ** 64 - 1), int(epoch), int(sample_base), int(n), int(nnz), int(n_neg),
                                int(plan[0]), int(plan[1]), ii.ctypes.data, jj.ctypes.data), "b200_bpr_draw_host")
    return ii, jj


def bpr_epoch_replay(data, i_index, j_id, U, V, B, lr, reg, use_bias, stats, hinge=False):
    """Serial-equivalent application of an explicit sample stream (parity mode)."""
    L = require_cuda()
    n = _dev(i_index, torch.int64, "i_index").numel()
    _dev(j_id, torch.int32, "j_id", _AtLeast(n))
    k = _dev(U, torch.float32, "U", (_AtLeast(data.n_users), None)).shape[1]
    n_items = _dev(V, torch.float32, "V", (None, k)).shape[0]
    _dev(B, torch.float32, "B", _AtLeast(n_items)), _dev(stats, torch.int64, "stats", _AtLeast(2))
    check(L.b200_bpr_epoch_replay2(ptr(i_index), ptr(j_id), n, ptr(data.indptr), ptr(data.indices), ptr(data.coo_row),
                                   int(U.shape[0]), int(n_items), ptr(U), ptr(V), ptr(B), int(k), float(lr), float(reg),
                                   int(bool(use_bias)), _lib.BPR_LOSS_HINGE if hinge else 0, ptr(stats), current_stream()),
          "b200_bpr_epoch_replay")


def bpr_train_host(indptr, indices, n_neg, U, V, B, lr, reg, use_bias, max_iter, key=0, replay_seeds=None,
                   atomic=True, on_epoch=None, keep_device=False, replica_sync=False, weighted_seed=None,
                   neg_weighted=False, hinge=False, blocked=True, deterministic=False):
    """Host-buffer entry of BPR training (what BPR.fit calls): uploads the CSR matrix and the
    factors, runs `max_iter` epochs, writes the trained factors back INTO the given numpy
    arrays U, V, B (pinned staging both ways).

    replay_seeds = (seed_pos, seed_neg): deterministic mode -- per epoch the two mt19937 streams
    of the reference's RNGVector are drawn on the host and applied by the serial-equivalent
    replay kernel.  Otherwise Hogwild epochs with the on-device Philox sampler keyed by `key`.
    replica_sync=True (multi-GPU, one process per GPU, torch.distributed initialised): `indptr/indices/U`
    are this rank's USER SHARD, V/B are replicas; after every epoch the ranks exchange their item-side
    changes (parallel.ItemReplicaSync: make-delta -> NCCL all-reduce -> apply).
    Returns (per-epoch (correct, skipped) list or [], device tensors (U, V, B) if keep_device)."""
    require_cuda()
    data = BprData.from_host(indptr, indices)
    nnz = data.nnz
    if replay_seeds is None and weighted_seed is None:
        data.prepare()                  # pair store + membership table: runs while the factors are still copying
    # the factor matrices go up on a side stream so that the copy engine overlaps b200_bpr_prepare
    main = torch.cuda.current_stream()
    side = _copy_stream()               # no dependency on `main`: the uploads may start right away
    with torch.cuda.stream(side):
        dU, dV, dB = to_device(U, torch.float32), to_device(V, torch.float32), to_device(B, torch.float32)
    main.wait_stream(side)
    for t in (dU, dV, dB):
        t.record_stream(main)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    lr, reg = _f32(lr), _f32(reg)
    history = []
    sync = None
    if replica_sync:
        from .parallel import make_item_sync
        sync = make_item_sync([dV, dB])
    if weighted_seed is not None or replay_seeds is not None:
        # Deterministic mode.  BPR: the two mt19937 streams of the reference's RNGVector (recom_bpr.pyx:54-62).  WBPR:
        # ONE stream, each sample takes (pos draw, neg draw) from it and the negative is the item of the drawn
        # interaction (recom_wbpr.pyx:125-136).  The epochs are PIPELINED: the host draws epoch e + 1 while the GPU
        # applies epoch e (three pinned staging sets, fenced by events; per-epoch stats stay on the device and come
        # back once at the end), unless a per-epoch callback needs the numbers right away.
        n_sets = 3 if nnz <= (1 << 24) else 2
        if weighted_seed is not None:
            g = MTSampler(weighted_seed)
            h_ij = np.empty(2 * nnz, dtype=np.int64)
            host_indices = np.asarray(indices)
        else:
            g_pos, g_neg = MTSampler(replay_seeds[0]), MTSampler(replay_seeds[1])
        h_i = [torch.empty(nnz, dtype=torch.int64).pin_memory() for _ in range(n_sets)]
        h_j = [torch.empty(nnz, dtype=torch.int32).pin_memory() for _ in range(n_sets)]
        d_i = [torch.empty(nnz, dtype=torch.int64, device="cuda") for _ in range(n_sets)]
        d_j = [torch.empty(nnz, dtype=torch.int32, device="cuda") for _ in range(n_sets)]
        fence = [None] * n_sets
        stats_all = torch.zeros((max_iter, 2), dtype=torch.int64, device="cuda")
        for epoch in range(max_iter):
            b = epoch % n_sets
            if fence[b] is not None:
                fence[b].synchronize()          # the upload of the epoch that last used this staging set has finished
            if weighted_seed is not None:
                g.fill(nnz - 1, 2 * nnz, out=h_ij)
                h_i[b].numpy()[:] = h_ij[0::2]
                h_j[b].numpy()[:] = host_indices[h_ij[1::2]]
            else:
                g_pos.fill(nnz - 1, nnz, out=h_i[b].numpy())
                g_neg.fill(int(n_neg) - 1, nnz, out=h_j[b].numpy())
            d_i[b].copy_(h_i[b], non_blocking=True)
            d_j[b].copy_(h_j[b], non_blocking=True)
            fence[b] = torch.cuda.Event()
            fence[b].record()
            bpr_epoch_replay(data, d_i[b], d_j[b], dU, dV, dB, lr, reg, use_bias, stats_all[epoch], hinge=hinge)
            if on_epoch:
                on_epoch(epoch, *stats_all[epoch].cpu().tolist())
        history = [tuple(r) for r in stats_all.cpu().tolist()]
    else:
        for epoch in range(max_iter):
            stats.zero_()
            bpr_epoch(data, n_neg, dU, dV, dB, lr, reg, use_bias, key, epoch, stats, atomic=atomic,
                      neg_weighted=neg_weighted, hinge=hinge, blocked=blocked, deterministic=deterministic)
            if sync is not None:
                sync.exchange()
            if on_epoch:
                history.append(tuple(stats.cpu().tolist()))
                on_epoch(epoch, *history[-1])
    if sync is not None and hasattr(sync, "close"):
        torch.cuda.synchronize()
        sync.close()
    for host, dev in ((U, dU), (V, dV), (B, dB)):
        _to_host_into(host, dev)
    return history, ((dU, dV, dB) if keep_device else None)


def tri_train_host(kind, indptr, indices, aux, n_items, U, V, B, hyper, max_iter, key=0, replay_seeds=None, on_epoch=None,
                   keep_device=False):
    """Host-buffer entry of the BPR siblings with a third item per sample (csrc/bprx.cu), what VEBPR.fit / SBPR.fit call.

    kind "vebpr": aux = (view_indptr, view_indices) of the viewed-not-purchased CSR, hyper = dict(lr, reg, alpha), B = None,
                  replay_seeds = (pos, view, neg) mt19937 seeds of the three RNGVectors (recom_vebpr.pyx:198-200);
    kind "sbpr":  aux = (social_indptr, social_item_ids, social_item_counts), hyper = dict(lr, lambda_u, lambda_v, lambda_b,
                  use_bias), replay_seeds = (pos, neg) (recom_sbpr.pyx:173-174).
    replay_seeds given -> the seeded streams are drawn on the host in the reference's order (b200_*_draw_host) and applied
    by the serial-equivalent replay kernel, the host drawing epoch e + 1 while the GPU applies epoch e; else Hogwild epochs
    with on-device Philox sampling keyed by `key`.  Trained factors are written back INTO U, V (, B).
    Returns (per-epoch (correct, skipped) list, device tensors (U, V, B or None) if keep_device)."""
    L = require_cuda()
    assert kind in ("vebpr", "sbpr")
    data = BprData.from_host(indptr, indices)
    nnz = data.nnz
    coo = data.coo_row
    aux_dev = [to_device(np.ascontiguousarray(a, dtype=np.int32), torch.int32) if len(a) else
               torch.zeros(1, dtype=torch.int32, device="cuda") for a in aux]
    dU, dV = to_device(U, torch.float32), to_device(V, torch.float32)
    dB = to_device(B, torch.float32) if B is not None else None
    n_users, k = int(dU.shape[0]), int(dU.shape[1])
    max_iter = int(max_iter)
    stats_all = torch.zeros((max(max_iter, 1), 2), dtype=torch.int64, device="cuda")
    st = current_stream

    def hogwild(epoch):
        if kind == "vebpr":
            check(L.b200_vebpr_epoch(ptr(data.indptr), ptr(data.indices), ptr(coo), n_users, int(n_items), nnz,
                                     ptr(aux_dev[0]), ptr(aux_dev[1]), ptr(dU), ptr(dV), k, _f32(hyper["lr"]), _f32(hyper["reg"]),
                                     _f32(hyper["alpha"]), int(key) & ((1 << 64) - 1), epoch, nnz, ptr(stats_all[epoch]), st()),
                  "b200_vebpr_epoch")
        else:
            check(L.b200_sbpr_epoch(ptr(data.indptr), ptr(data.indices), ptr(coo), n_users, int(n_items), nnz,
                                    ptr(aux_dev[0]), ptr(aux_dev[1]), ptr(aux_dev[2]), len(aux[1]), ptr(dU), ptr(dV), ptr(dB), k,
                                    _f32(hyper["lr"]), _f32(hyper["lambda_u"]), _f32(hyper["lambda_v"]), _f32(hyper["lambda_b"]),
                                    int(bool(hyper["use_bias"])), int(key) & ((1 << 64) - 1), epoch, nnz, ptr(stats_all[epoch]), st()),
                  "b200_sbpr_epoch")

    if replay_seeds is None:
        for epoch in range(max_iter):
            hogwild(epoch)
            if on_epoch:
                on_epoch(epoch, *stats_all[epoch].cpu().tolist())
    else:
        gens = [MTSampler(s_) for s_ in replay_seeds]
        h_coo = np.repeat(np.arange(len(indptr) - 1, dtype=np.int32), np.diff(np.asarray(indptr)).astype(np.int64))
        h_aux = [np.ascontiguousarray(a, dtype=np.int32) for a in aux]
        third = torch.int32 if kind == "vebpr" else torch.int64
        n_sets = 2
        h_i = [torch.empty(nnz, dtype=torch.int64).pin_memory() for _ in range(n_sets)]
        h_j = [torch.empty(nnz, dtype=torch.int32).pin_memory() for _ in range(n_sets)]
        h_t = [torch.empty(nnz, dtype=third).pin_memory() for _ in range(n_sets)]
        d_i = [torch.empty(nnz, dtype=torch.int64, device="cuda") for _ in range(n_sets)]
        d_j = [torch.empty(nnz, dtype=torch.int32, device="cuda") for _ in range(n_sets)]
        d_t = [torch.empty(nnz, dtype=third, device="cuda") for _ in range(n_sets)]
        fence = [None] * n_sets
        for epoch in range(max_iter):
            b = epoch % n_sets
            if fence[b] is not None:
                fence[b].synchronize()
            if kind == "vebpr":
                check(L.b200_vebpr_draw_host(gens[0]._h, gens[1]._h, gens[2]._h, nnz, int(n_items), h_coo.ctypes.data,
                                             h_aux[0].ctypes.data, h_aux[1].ctypes.data, nnz, h_i[b].data_ptr(), h_t[b].data_ptr(),
                                             h_j[b].data_ptr()), "b200_vebpr_draw_host")
            else:
                check(L.b200_sbpr_draw_host(gens[0]._h, gens[1]._h, nnz, int(n_items), h_coo.ctypes.data, h_aux[0].ctypes.data, nnz,
                                            h_i[b].data_ptr(), h_j[b].data_ptr(), h_t[b].data_ptr()), "b200_sbpr_draw_host")
            d_i[b].copy_(h_i[b], non_blocking=True), d_j[b].copy_(h_j[b], non_blocking=True), d_t[b].copy_(h_t[b], non_blocking=True)
            fence[b] = torch.cuda.Event()
            fence[b].record()
            if kind == "vebpr":
                check(L.b200_vebpr_epoch_replay(ptr(d_i[b]), ptr(d_t[b]), ptr(d_j[b]), nnz, ptr(data.indptr), ptr(data.indices), ptr(coo),
                                                ptr(aux_dev[0]), ptr(aux_dev[1]), ptr(dU), ptr(dV), k, _f32(hyper["lr"]), _f32(hyper["reg"]),
                                                _f32(hyper["alpha"]), ptr(stats_all[epoch]), st()), "b200_vebpr_epoch_replay")
            else:
                check(L.b200_sbpr_epoch_replay(ptr(d_i[b]), ptr(d_j[b]), ptr(d_t[b]), nnz, ptr(data.indptr), ptr(data.indices), ptr(coo),
                                               ptr(aux_dev[0]), ptr(aux_dev[1]), ptr(aux_dev[2]), len(aux[1]), ptr(dU), ptr(dV), ptr(dB), k,
                                               _f32(hyper["lr"]), _f32(hyper["lambda_u"]), _f32(hyper["lambda_v"]), _f32(hyper["lambda_b"]),
                                               int(bool(hyper["use_bias"])), ptr(stats_all[epoch]), st()), "b200_sbpr_epoch_replay")
            if on_epoch:
                on_epoch(epoch, *stats_all[epoch].cpu().tolist())
    history = [tuple(r) for r in stats_all[:max_iter].cpu().tolist()]
    _to_host_into(U, dU)
    _to_host_into(V, dV)
    if B is not None:
        _to_host_into(B, dB)
    return history, ((dU, dV, dB) if keep_device else None)


_COPY_STREAMS = {}


def _copy_stream():
    dev = torch.cuda.current_device()
    if dev not in _COPY_STREAMS:
        _COPY_STREAMS[dev] = torch.cuda.Stream(device=dev)
    return _COPY_STREAMS[dev]


def _to_host_into(host, dev):
    """D2H into an existing numpy array (through pinned staging when it is not pinned itself)."""
    out = torch.from_numpy(host) if (host.flags["C_CONTIGUOUS"] and host.flags.writeable) else None
    if out is not None and out.dtype == dev.dtype and tuple(out.shape) == tuple(dev.shape):
        out.copy_(dev)
        return host
    raise B200Error("destination array must be a writable C-contiguous %s array of shape %s" % (dev.dtype, tuple(dev.shape)))


class MTSampler:
    """boost::random::mt19937 + uniform_int_distribution<long>(0, hi) on the host
    (RNGVector of the reference, one thread)."""

    def __init__(self, seed):
        self._L = _lib.load()
        self._h = self._L.b200_mt_sampler_create(int(seed) & 0xFFFFFFFF)
        if not self._h:
            raise B200Error("b200_mt_sampler_create failed")

    def fill(self, hi, n, dtype=np.int64, out=None):
        out = np.empty(n, dtype=dtype) if out is None else out
        fn = self._L.b200_mt_sampler_fill_i64 if out.dtype == np.int64 else self._L.b200_mt_sampler_fill_i32
        check(fn(self._h, int(hi), int(n), out.ctypes.data), "b200_mt_sampler_fill")
        return out

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200_mt_sampler_destroy(self._h)
            self._h = None


def mf_epoch(rid, cid, val, U, V, Bu, Bi, lr, reg, mu, use_bias, loss, ordered=False, atomic=True, unbounded=False):
    """One MF epoch; `loss` (float32[1] CUDA) receives sum(err^2).  U = V = None: the bias-only model
    (BaselineOnly), sized by Bu / Bi."""
    L = require_cuda()
    if rid.dtype not in (torch.int32, torch.int64) or cid.dtype != rid.dtype:
        raise B200Error("rid/cid must both be int32 or int64")
    if (U is None) != (V is None):
        raise B200Error("U and V must both be given or both be None")
    n = _dev(val, torch.float32, "val").numel()
    _dev(rid, rid.dtype, "rid", _AtLeast(n)), _dev(cid, rid.dtype, "cid", _AtLeast(n))
    n_users, n_items = _dev(Bu, torch.float32, "Bu").numel(), _dev(Bi, torch.float32, "Bi").numel()
    _dev(loss, torch.float32, "loss", _AtLeast(1))
    k = 0 if U is None else _dev(U, torch.float32, "U", (_AtLeast(n_users), None)).shape[1]
    if V is not None:
        _dev(V, torch.float32, "V", (_AtLeast(n_items), k))
    check(L.b200_mf_epoch(ptr(rid), ptr(cid), ptr(val), n, int(rid.dtype == torch.int32),
                          n_users, n_items, ptr(U), ptr(V), ptr(Bu), ptr(Bi), int(k), float(lr), float(reg), float(mu),
                          int(bool(use_bias)), int(bool(ordered)),
                          (_lib.SGD_ATOMIC if atomic else 0) | (_lib.SGD_UNBOUNDED if unbounded else 0), ptr(loss),
                          current_stream()), "b200_mf_epoch")


class WmfTrainer:
    """Device state of one WMF fit (the variables and Adam slots of the reference's TF-1 graph, wmf/wmf.py:34-55) and
    the step `sess.run([model.opt, model.loss], feed_dict)` of recom_wmf.py:197-199, one mini-batch of item ids at a
    time.  `csc` is train_set.csc_matrix (scipy); U, V numpy float32 arrays (copied up; read back with .download())."""

    BETA1, BETA2, EPS = 0.9, 0.999, 1e-8              # tf.train.AdamOptimizer defaults

    def __init__(self, csc, U, V, a, b, lambda_u, lambda_v, lr):
        require_cuda()
        csc = csc.tocsc()
        csc.sort_indices()
        if csc.nnz >= 2 ** 31:
            raise B200Error("nnz >= 2^31 is not supported (int32 CSC offsets)")
        self.n_users, self.n_items = (int(x) for x in csc.shape)
        self.U = _dev(to_device(np.ascontiguousarray(U, dtype=np.float32)), torch.float32, "U", (self.n_users, None))
        self.k = int(self.U.shape[1])
        self.V = _dev(to_device(np.ascontiguousarray(V, dtype=np.float32)), torch.float32, "V", (self.n_items, self.k))
        self.indptr = to_device(csc.indptr, torch.int32)
        self.rows = to_device(csc.indices if csc.nnz else np.zeros(1, np.int32), torch.int32)
        self.vals = to_device(np.asarray(csc.data if csc.nnz else np.zeros(1), dtype=np.float32), torch.float32)
        self.mU, self.vU = torch.zeros_like(self.U), torch.zeros_like(self.U)
        self.mV, self.vV = torch.zeros_like(self.V), torch.zeros_like(self.V)
        self.slot_of = torch.full((self.n_items,), -1, dtype=torch.int32, device="cuda")
        self.loss = torch.zeros(1, dtype=torch.float64, device="cuda")
        self.gV = None
        f32 = np.float32
        self.a, self.b, self.lambda_u, self.lambda_v = f32(a), f32(b), f32(lambda_u), f32(lambda_v)
        self.lr = f32(lr)
        self.b1_pow, self.b2_pow = f32(self.BETA1), f32(self.BETA2)     # beta^t for the step about to be taken (t = 1)

    def step(self, ids, want_loss=True):
        """One optimisation step on the item mini-batch `ids` (distinct item indices); returns the batch loss (float) or
        None.  Reading the loss synchronises with the device, like sess.run does."""
        L = _lib.load()
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        b = int(len(ids))
        if b == 0:
            return 0.0
        if ids.min() < 0 or ids.max() >= self.n_items:
            raise B200Error("item id out of range in the mini-batch")
        d_ids = to_device(ids, torch.int32, pinned=False)
        if self.gV is None or self.gV.numel() < b * self.k:
            self.gV = torch.empty(b * self.k, dtype=torch.float32, device="cuda")
        f32 = np.float32
        lr_t = self.lr * np.sqrt(f32(1) - self.b2_pow) / (f32(1) - self.b1_pow)          # AdamOptimizer._prepare / _apply_*
        check(L.b200_wmf_step(ptr(self.indptr), ptr(self.rows), ptr(self.vals), ptr(d_ids), b, self.n_users, self.n_items,
                              self.k, ptr(self.U), ptr(self.V), ptr(self.mU), ptr(self.vU), ptr(self.mV), ptr(self.vV),
                              float(self.a), float(self.b), float(self.lambda_u), float(self.lambda_v), _f32(lr_t),
                              self.BETA1, self.BETA2, self.EPS, ptr(self.slot_of), ptr(self.gV), ptr(self.loss),
                              current_stream()), "b200_wmf_step")
        self.b1_pow = f32(self.b1_pow * f32(self.BETA1))              # _finish: the beta powers advance once per step
        self.b2_pow = f32(self.b2_pow * f32(self.BETA2))
        return float(self.loss.item()) if want_loss else None

    def download(self):
        return self.U.cpu().numpy(), self.V.cpu().numpy()


def _csr_arrays(m, what):
    """int32 indptr / indices and f64 data of a scipy CSR matrix (copies only where the dtype differs)."""
    if m.nnz >= 2 ** 31:
        raise B200Error("%s: nnz >= 2^31 is not supported (int32 CSR offsets)" % what)
    return (np.ascontiguousarray(m.indptr, dtype=np.int32), np.ascontiguousarray(m.indices, dtype=np.int32),
            np.ascontiguousarray(m.data, dtype=np.float64))


def _upload_csr(m, what):
    ip, ix, dt = _csr_arrays(m, what)
    if len(ix) == 0:
        ix, dt = np.zeros(1, np.int32), np.zeros(1)
    return to_device(ip, torch.int32), to_device(ix, torch.int32), to_device(dt, torch.float64)


def _heaviest_rows_first(rows, cols):
    """The rows of `rows` in decreasing work (sum of the lengths of the rows of `cols` a row touches), so that the longest
    rows of an ordered row-pair sum start first."""
    ip, ix, _ = _csr_arrays(rows, "weight matrix")
    work = np.zeros(len(ip) - 1, dtype=np.int64)
    if len(ix):
        np.add.at(work, np.repeat(np.arange(len(ip) - 1), np.diff(ip)), np.diff(cols.indptr)[ix])
    return np.argsort(-work, kind="stable").astype(np.int32)


def knn_similarity(weight, amplify=1.0):
    """compute_similarity + the amplify map (cornac/models/knn/similarity.pyx:51-105, recom_knn.py:48-55) of the rows of
    the scipy CSR weight matrix.  Returns (S, sim_mat): the dense symmetric f64 [n, n] device similarity and the same
    matrix as a host scipy CSR (f64, zeros dropped).  Refuses before allocating when S does not fit the free device memory."""
    L = require_cuda()
    weight = weight.tocsr()
    n, n_cols = (int(x) for x in weight.shape)
    ws_bytes = int(L.b200_knn_similarity_workspace_bytes(n))
    need = n * n * 8
    free, _ = torch.cuda.mem_get_info()
    if need + ws_bytes > free:
        raise B200Error("the dense %d x %d f64 similarity needs %d bytes (+ %d bytes of workspace); the device has %d bytes free"
                        % (n, n, need, ws_bytes, free))
    cols = weight.T.tocsr()
    cols.sort_indices()
    order = _heaviest_rows_first(weight, cols)
    r_p, r_i, r_d = _upload_csr(weight, "weight matrix")
    c_p, c_i, c_d = _upload_csr(cols, "weight matrix")
    ws = torch.empty(max(ws_bytes, 8), dtype=torch.uint8, device="cuda")
    S = torch.empty((n, n), dtype=torch.float64, device="cuda")
    st = current_stream()
    check(L.b200_knn_similarity(n, ptr(r_p), ptr(r_i), ptr(r_d), n_cols, ptr(c_p), ptr(c_i), ptr(c_d),
                                ptr(to_device(order, torch.int32)), float(amplify), ptr(ws) if ws_bytes else None, ptr(S), st),
          "b200_knn_similarity")
    del ws
    counts = torch.empty(n, dtype=torch.int32, device="cuda")
    check(L.b200_knn_row_nnz(n, ptr(S), ptr(counts), st), "b200_knn_row_nnz")
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(counts.cpu().numpy(), out=indptr[1:])
    nnz = int(indptr[-1])
    if nnz >= 2 ** 31:
        raise B200Error("the similarity has %d non-zeros: nnz >= 2^31 is not supported (int32 CSR offsets)" % nnz)
    d_ptr = to_device(indptr, torch.int32)
    d_idx = torch.empty(max(nnz, 1), dtype=torch.int32, device="cuda")
    d_val = torch.empty(max(nnz, 1), dtype=torch.float64, device="cuda")
    check(L.b200_knn_compact(n, ptr(S), ptr(d_ptr), ptr(d_idx), ptr(d_val), st), "b200_knn_compact")
    sim = _sp.csr_matrix((d_val[:nnz].cpu().numpy(), d_idx[:nnz].cpu().numpy(), indptr.astype(np.int32)), shape=(n, n))
    return S, sim


def _csr_bytes(n_rows, nnz):
    """Device bytes of an int32 / int32 / f64 CSR copy (_upload_csr)."""
    return 4 * (n_rows + 1) + 12 * max(nnz, 1)


def ease_device_bytes(n_users, n_items, nnz):
    """Device bytes of ease_fit plus the rating copy the scores read: the n x n matrix, the Gram inputs (X^T and X as CSR,
    the row order) and workspace, the inverse workspace, the saved diagonal, and EaseRatings."""
    L = _lib.load()
    n = int(n_items)
    return (n * n * 8 + _csr_bytes(n, nnz) + _csr_bytes(n_users, nnz) + 4 * n + int(L.b200_ease_gram_workspace_bytes(n))
            + int(L.b200_spd_inverse_workspace_bytes(n)) + 8 * n + _csr_bytes(n_users, nnz))


class EaseGramInput:
    """The device inputs of b200_ease_gram for a scipy CSR rating matrix X (users x items): X^T as CSR with each item's
    users ascending (the order of scipy's sums), X as CSR with each user's items ascending, and the item rows in
    decreasing work.  Built once; ease_gram then only launches."""

    def __init__(self, X):
        require_cuda()
        X = X.tocsr().copy()
        X.sort_indices()
        self.n_users, self.n = (int(x) for x in X.shape)
        XT = X.T.tocsr()
        XT.sort_indices()
        self.rows = _upload_csr(XT, "rating matrix")
        self.cols = _upload_csr(X, "rating matrix")
        self.order = to_device(_heaviest_rows_first(XT, X), torch.int32)


def ease_gram(inp, lamb, out, workspace=None):
    """X.T.dot(X).toarray() + lamb on the diagonal into the f64 device tensor out [n_items, n_items], bit for bit (the
    raw mode of the KNN similarity kernel over the rows of X^T).  inp: EaseGramInput of X."""
    L = require_cuda()
    n = inp.n
    _dev(out, torch.float64, "out", (n, n))
    ws_bytes = int(L.b200_ease_gram_workspace_bytes(n))
    workspace = _buf(workspace, torch.uint8, "workspace", _AtLeast(ws_bytes))
    (r_p, r_i, r_d), (c_p, c_i, c_d) = inp.rows, inp.cols
    check(L.b200_ease_gram(n, ptr(r_p), ptr(r_i), ptr(r_d), max(inp.n_users, 1), ptr(c_p), ptr(c_i), ptr(c_d),
                           ptr(inp.order), float(lamb), ptr(workspace) if ws_bytes else None, ptr(out), current_stream()),
          "b200_ease_gram")
    return out


def spd_inverse(A, phases=_lib.SPD_ALL, workspace=None, info=None):
    """Replace the symmetric positive definite f64 device matrix A [n, n] (lower triangle read) by its inverse, in place, on
    the FP64 tensor cores (b200_spd_inverse).  `phases` runs a subset of potrf / trtri / lauum (in order, with the same
    workspace and info).  Raises numpy.linalg.LinAlgError naming the first failing column when A is not positive definite
    (checked after the factorisation; the call then synchronises with the device)."""
    L = require_cuda()
    n = _dev(A, torch.float64, "A", (None, None)).shape[0]
    _dev(A, torch.float64, "A", (n, n))
    workspace = _buf(workspace, torch.uint8, "workspace", _AtLeast(L.b200_spd_inverse_workspace_bytes(n)))
    info = _buf(info, torch.int32, "info", _AtLeast(1), zero=True)
    check(L.b200_spd_inverse(n, ptr(A), ptr(workspace), ptr(info), int(phases), current_stream()), "b200_spd_inverse")
    if phases & _lib.SPD_POTRF:
        bad = int(info.item())
        if bad:
            raise np.linalg.LinAlgError("the %d x %d Gram matrix is not positive definite: pivot of column %d is not a "
                                        "positive finite number (info = %d)" % (n, n, bad - 1, bad))
    return A


def ease_weights(P, posB, diag=None):
    """B = P / -diag(P), B[j, j] = 0, negatives to 0 under posB, in place on the f64 device matrix P (b200_ease_weights)."""
    L = require_cuda()
    n = _dev(P, torch.float64, "P", (None, None)).shape[0]
    _dev(P, torch.float64, "P", (n, n))
    diag = _buf(diag, torch.float64, "diag", _AtLeast(n))
    check(L.b200_ease_weights(n, ptr(P), ptr(diag), int(bool(posB)), current_stream()), "b200_ease_weights")
    return P


def ease_fit(X, lamb, posB):
    """EASE.fit (recom_ease.py:72-95) on the device: G = X^T X + lamb I, P = G^-1, B = P / -diag(P).  Returns B, the f64
    device [n_items, n_items] weight matrix.  Refuses before allocating when it does not fit the free device memory;
    raises numpy.linalg.LinAlgError when G is not positive definite (only possible for lamb <= 0)."""
    require_cuda()
    n_users, n = (int(x) for x in X.shape)
    need = ease_device_bytes(n_users, n, X.nnz)
    free, _ = torch.cuda.mem_get_info()
    free += torch.cuda.memory_reserved() - torch.cuda.memory_allocated()    # blocks torch's allocator holds but does not use
    if need > free:
        raise B200Error("the dense %d x %d f64 EASE matrix needs %d bytes with its inputs and workspaces (%d bytes in all); the "
                        "device has %d bytes free" % (n, n, n * n * 8, need, free))
    inp = EaseGramInput(X)
    B = torch.empty((n, n), dtype=torch.float64, device="cuda")
    ease_gram(inp, lamb, B)
    del inp
    spd_inverse(B)
    return ease_weights(B, posB)


class EaseRatings:
    """Device copy of the CSR rating matrix X that EASE's score rows read, in stored order."""

    def __init__(self, X):
        require_cuda()
        X = X.tocsr()
        self.n_rows, self.n_cols = (int(x) for x in X.shape)
        self.indptr, self.indices, self.data = _upload_csr(X, "rating matrix")


def ease_score(B, users, ratings, out=None):
    """out[q, :] = X[users[q], :] . B in scipy's order (b200_ease_score): f64 [n_q, n_items] device score rows.
    ratings: EaseRatings of X; B: f64 device [n_items, n_items]; users: indices of rows of X (host or int64 device)."""
    L = require_cuda()
    n = ratings.n_cols
    _dev(B, torch.float64, "B", (n, n))
    if isinstance(users, torch.Tensor):
        _dev(users, torch.int64, "users")
        lo, hi = (int(users.min()), int(users.max())) if users.numel() else (0, 0)
    else:
        host = np.asarray(users, dtype=np.int64)
        lo, hi = (int(host.min()), int(host.max())) if host.size else (0, 0)
        users = to_device(host, torch.int64)
    if lo < 0 or hi >= ratings.n_rows:
        raise B200Error("user index out of range [0, %d): %d" % (ratings.n_rows, lo if lo < 0 else hi))
    n_q = int(users.numel())
    out = _buf(out, torch.float64, "out", (n_q, n))
    check(L.b200_ease_score(ptr(users), n_q, n, ptr(ratings.indptr), ptr(ratings.indices), ptr(ratings.data), ptr(B),
                            ptr(out), current_stream()), "b200_ease_score")
    return out


def knn_dense(sim):
    """The dense f64 device matrix of a host scipy CSR similarity (after load(): the device state is not pickled)."""
    require_cuda()
    n = int(sim.shape[0])
    need = n * n * 8
    free, _ = torch.cuda.mem_get_info()
    if need > free:
        raise B200Error("the dense %d x %d f64 similarity needs %d bytes; the device has %d bytes free" % (n, n, need, free))
    coo = sim.tocoo()
    S = torch.zeros((n, n), dtype=torch.float64, device="cuda")
    S.view(-1)[to_device(coo.row.astype(np.int64) * n + coo.col, torch.int64)] = to_device(coo.data, torch.float64)
    return S


class KnnRatings:
    """Device copy of the CSR rating matrix the scores read: the user-item matrix (ItemKNN) or the item-user matrix
    (UserKNN), and the users' mean ratings."""

    def __init__(self, m, mean):
        require_cuda()
        m = m.tocsr().copy()
        m.sort_indices()                             # the candidates are visited in descending neighbour index
        self.n_rows, self.n_cols = (int(x) for x in m.shape)
        self.indptr, self.indices, self.data = _upload_csr(m, "rating matrix")
        self.mean = to_device(np.asarray(mean, dtype=np.float64), torch.float64)


def knn_score(user_mode, S, users, ratings, k):
    """compute_score (cornac/models/knn/similarity.pyx:154-201) plus the user's mean for each user of `users`:
    f64 [n_q, n_items] device scores.  user_mode: UserKNN (S is [n_users, n_users], ratings the item-user matrix);
    otherwise ItemKNN (S is [n_items, n_items], ratings the user-item matrix)."""
    L = require_cuda()
    n = ratings.n_cols                            # the similarity's rows and columns are the ratings' columns
    _dev(S, torch.float64, "S", (n, n))
    if k < 1:
        raise B200Error("k must be >= 1, got %d" % k)
    users = users if isinstance(users, torch.Tensor) else to_device(np.asarray(users, dtype=np.int64), torch.int64)
    _dev(users, torch.int64, "users")
    n_q = int(users.numel())
    n_users = n if user_mode else ratings.n_rows
    n_items = ratings.n_rows if user_mode else n
    out = torch.empty((n_q, n_items), dtype=torch.float64, device="cuda")
    ws_bytes = int(L.b200_knn_score_workspace_bytes(n_q, n_users if user_mode else 0, int(k)))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda") if ws_bytes else None
    if user_mode:
        rc = L.b200_knn_score_users(ptr(users), n_q, n_users, n_items, ptr(ratings.indptr), ptr(ratings.indices),
                                    ptr(ratings.data), ptr(S), ptr(ratings.mean), int(k), ptr(ws), ptr(out), current_stream())
    else:
        rc = L.b200_knn_score_items(ptr(users), n_q, n_items, ptr(ratings.indptr), ptr(ratings.indices), ptr(ratings.data),
                                    ptr(S), ptr(ratings.mean), int(k), ptr(ws), ptr(out), current_stream())
    check(rc, "b200_knn_score_users" if user_mode else "b200_knn_score_items")
    return out


def score_batch(U, V, user_idx=None, item_base=None, user_off=None, n_items=None, out=None):
    """out[q, i] = (item_base[i] + user_off[q]) + dot(U[user_idx[q]], V[i]) for i < n_items."""
    L = require_cuda()
    n_items, k, n_q = _score_args(U, V, user_idx, n_items, torch.float32, item_base, user_off)
    out = _buf(out, torch.float32, "out", (n_q, n_items))
    check(L.b200_score_batch(ptr(U), ptr(user_idx), n_q, ptr(V), n_items, k, ptr(item_base), ptr(user_off), ptr(out),
                             current_stream()), "b200_score_batch")
    return out


def _score_args(U, V, user_idx, n_items, dtype, item_base=None, user_off=None):
    """(n_items, k, n_q) of a score or rank call, checked: V [>= n_items (default all rows), k], U [*, k] (its rows the
    queries when user_idx is None), user_idx int64 [n_q], item_base [>= n_items] and user_off [>= n_q] when given."""
    k = _dev(V, dtype, "V", (None if n_items is None else _AtLeast(n_items), None)).shape[1]
    n_items = int(V.shape[0] if n_items is None else n_items)
    _dev(U, dtype, "U", (None, k))
    n_q = U.shape[0] if user_idx is None else _dev(user_idx, torch.int64, "user_idx").numel()
    if item_base is not None:
        _dev(item_base, dtype, "item_base", _AtLeast(n_items))
    if user_off is not None:
        _dev(user_off, dtype, "user_off", _AtLeast(n_q))
    return n_items, int(k), int(n_q)


def _exclusions(excl_indptr, excl_indices, n_q):
    """Checks the optional per-row exclusion CSR: excl_indptr int64 [>= n_q + 1], excl_indices int32."""
    if excl_indptr is not None:
        _dev(excl_indptr, torch.int64, "excl_indptr", _AtLeast(n_q + 1))
        _dev(excl_indices, torch.int32, "excl_indices")


def topk_rows(scores, topk, excl_indptr=None, excl_indices=None):
    """Exact top-k (score desc, id asc) of each row of `scores`, with per-row exclusions."""
    L = require_cuda()
    n_q, n_items = _dev(scores, torch.float32, "scores", (None, None)).shape
    ids = torch.empty((n_q, topk), dtype=torch.int32, device=scores.device)
    sc = torch.empty((n_q, topk), dtype=torch.float32, device=scores.device)
    _exclusions(excl_indptr, excl_indices, n_q)
    check(L.b200_topk_rows(ptr(scores), n_q, n_items, ptr(excl_indptr), ptr(excl_indices), int(topk), ptr(ids),
                           ptr(sc), current_stream()), "b200_topk_rows")
    return ids, sc


def score_batch_f64(U, V, user_idx=None, n_items=None, out=None):
    """out[q, i] = sum_f U[user_idx[q], f] * V[i, f] in f64 (f ascending, no FMA) for i < n_items."""
    L = require_cuda()
    n_items, k, n_q = _score_args(U, V, user_idx, n_items, torch.float64)
    out = _buf(out, torch.float64, "out", (n_q, n_items))
    check(L.b200_score_batch_f64(ptr(U), ptr(user_idx), n_q, ptr(V), n_items, k, ptr(out), current_stream()),
          "b200_score_batch_f64")
    return out


def topk_rows_f64(scores, topk, excl_indptr=None, excl_indices=None):
    """topk_rows over f64 score rows: exact top-k (score desc, id asc) with per-row exclusions."""
    L = require_cuda()
    n_q, n_items = _dev(scores, torch.float64, "scores", (None, None)).shape
    ids = torch.empty((n_q, topk), dtype=torch.int32, device=scores.device)
    sc = torch.empty((n_q, topk), dtype=torch.float64, device=scores.device)
    _exclusions(excl_indptr, excl_indices, n_q)
    check(L.b200_topk_rows_f64(ptr(scores), n_q, n_items, ptr(excl_indptr), ptr(excl_indices), int(topk), ptr(ids),
                               ptr(sc), current_stream()), "b200_topk_rows_f64")
    return ids, sc


def pmf_schedule(uid, iid, n_users, n_items):
    """Level schedule of PMF's ratings (host, no device needed): (order int32 [nnz], level_ptr int32 [n_levels + 1]).
    Slot s of the schedule is stored rating order[s]; level l is slots [level_ptr[l], level_ptr[l+1]), its ratings touch
    pairwise disjoint user and item rows, and inside a level the slots keep the stored order."""
    L = _lib.load()
    uid = np.ascontiguousarray(uid, dtype=np.int32)
    iid = np.ascontiguousarray(iid, dtype=np.int32)
    nnz = len(uid)
    if len(iid) != nnz:
        raise B200Error("uid and iid differ in length (%d, %d)" % (nnz, len(iid)))
    order = np.empty(nnz, dtype=np.int32)
    level_ptr = np.empty(nnz + 1, dtype=np.int32)
    n_levels = np.zeros(1, dtype=np.int32)
    check(L.b200_pmf_schedule(ptr(uid), ptr(iid), nnz, int(n_users), int(n_items), ptr(order), ptr(level_ptr),
                              ptr(n_levels)), "b200_pmf_schedule")
    return order, level_ptr[: int(n_levels[0]) + 1].copy()


class PmfData:
    """Device copy of PMF's ratings in schedule order (b200_pmf_schedule), built once per fit and used by every epoch."""

    def __init__(self, uid, iid, rat, n_users, n_items):
        require_cuda()
        self.nnz, self.n_users, self.n_items = len(uid), int(n_users), int(n_items)
        self.order_host, level_ptr = pmf_schedule(uid, iid, n_users, n_items)
        self.n_levels = len(level_ptr) - 1
        o = self.order_host
        self.uid = to_device(np.asarray(uid, dtype=np.int32)[o], torch.int32)
        self.iid = to_device(np.asarray(iid, dtype=np.int32)[o], torch.int32)
        self.rat = to_device(np.asarray(rat, dtype=np.float32)[o], torch.float32)
        self.level_ptr = to_device(level_ptr, torch.int32)
        self.order = to_device(o, torch.int32)


def pmf_fit(data, variant, U, V, cache_u, cache_v, n_epochs, lambda_reg, learning_rate, gamma, loss=None):
    """n_epochs epochs of pmf_linear / pmf_non_linear (pmf.pyx:55-173) over `data` (PmfData), updating the f64 device
    tensors U, V, cache_u, cache_v in place.  loss: optional f64 device tensor [n_epochs, nnz] that receives each rating's
    loss term at its stored index."""
    L = require_cuda()
    variants = {"linear": _lib.PMF_LINEAR, "non_linear": _lib.PMF_NON_LINEAR}
    if variant not in variants:
        raise B200Error('variant must be one of {"linear","non_linear"}, got %r' % (variant,))
    users, items = _AtLeast(data.n_users), _AtLeast(data.n_items)
    k = _dev(U, torch.float64, "U", (users, None)).shape[1]
    _dev(cache_u, torch.float64, "cache_u", (users, k))
    _dev(V, torch.float64, "V", (items, k)), _dev(cache_v, torch.float64, "cache_v", (items, k))
    if loss is not None:
        _dev(loss, torch.float64, "loss", (int(n_epochs), data.nnz))
    check(L.b200_pmf_fit(variants[variant], ptr(data.uid), ptr(data.iid), ptr(data.rat), ptr(data.level_ptr),
                         data.n_levels, data.nnz, int(k), ptr(U), ptr(V), ptr(cache_u), ptr(cache_v), int(n_epochs),
                         float(lambda_reg), float(learning_rate), float(gamma), ptr(loss),
                         ptr(data.order) if loss is not None else None, current_stream()), "b200_pmf_fit")


def pmf_sigmoid(z):
    """The reference PMF sigmoid (pmf.pyx:27-37, expf in f32) of a f32 device tensor, as b200_pmf_fit evaluates it."""
    L = require_cuda()
    _dev(z, torch.float32, "z")
    out = torch.empty_like(z)
    check(L.b200_pmf_sigmoid(ptr(z), z.numel(), ptr(out), current_stream()), "b200_pmf_sigmoid")
    return out


COFACTOR_VARIANTS = {"sorec": _lib.COFACTOR_SOREC, "mcf": _lib.COFACTOR_MCF}


def cofactor_schedule(variant, net_a, net_b, uid, iid, n_users, n_items):
    """Level schedule of a SoRec / MCF epoch (host, no device needed): the n_edges graph edges (net_a, net_b: user ids for
    "sorec", item ids for "mcf") then the ratings (uid, iid), one stream.  Returns (order int32 [n_edges + n_ratings],
    level_ptr int32 [n_levels + 1]); order holds stored indices, edge e at e and rating r at n_edges + r.  The updates of
    one level touch pairwise disjoint rows of U, V and Z, and inside a level the slots keep the stored order."""
    L = _lib.load()
    if variant not in COFACTOR_VARIANTS:
        raise B200Error('variant must be one of {"sorec","mcf"}, got %r' % (variant,))
    net_a, net_b, uid, iid = (np.ascontiguousarray(x, dtype=np.int32) for x in (net_a, net_b, uid, iid))
    if len(net_b) != len(net_a) or len(iid) != len(uid):
        raise B200Error("edge ids (%d, %d) or rating ids (%d, %d) differ in length"
                        % (len(net_a), len(net_b), len(uid), len(iid)))
    n = len(net_a) + len(uid)
    order = np.empty(n, dtype=np.int32)
    level_ptr = np.empty(n + 1, dtype=np.int32)
    n_levels = np.zeros(1, dtype=np.int32)
    check(L.b200_cofactor_schedule(COFACTOR_VARIANTS[variant], ptr(net_a), ptr(net_b), len(net_a), ptr(uid), ptr(iid),
                                   len(uid), int(n_users), int(n_items), ptr(order), ptr(level_ptr), ptr(n_levels)),
          "b200_cofactor_schedule")
    return order, level_ptr[: int(n_levels[0]) + 1].copy()


class CofactorData:
    """Device copy of a SoRec / MCF epoch in schedule order (b200_cofactor_schedule), built once per fit and used by
    every epoch: per slot the two row ids, the target (edge value or rating) and whether it is an edge."""

    def __init__(self, variant, net_a, net_b, net_val, uid, iid, rat, n_users, n_items):
        require_cuda()
        self.variant = variant
        self.n_edges, self.n_ratings = len(net_a), len(uid)
        self.n_users, self.n_items = int(n_users), int(n_items)
        if len(net_val) != self.n_edges or len(rat) != self.n_ratings:
            raise B200Error("net_val has %d values for %d edges, rat %d for %d ratings"
                            % (len(net_val), self.n_edges, len(rat), self.n_ratings))
        self.order_host, level_ptr = cofactor_schedule(variant, net_a, net_b, uid, iid, n_users, n_items)
        self.n_levels = len(level_ptr) - 1
        o = self.order_host
        cat = lambda x, y, t: np.concatenate([np.asarray(x, dtype=t), np.asarray(y, dtype=t)])[o]   # noqa: E731
        self.a_id = to_device(_pad(cat(net_a, uid, np.int32)), torch.int32)
        self.b_id = to_device(_pad(cat(net_b, iid, np.int32)), torch.int32)
        self.val = to_device(_pad(cat(net_val, rat, np.float32)), torch.float32)
        self.is_edge = to_device(_pad((o < self.n_edges).astype(np.uint8)), torch.uint8)
        self.level_ptr = to_device(level_ptr, torch.int32)
        self.order = to_device(_pad(o), torch.int32)


def cofactor_fit(data, U, V, Z, cache_u, cache_v, cache_z, n_epochs, lambda_c, lambda_reg, learning_rate, gamma,
                 loss=None):
    """n_epochs epochs of sorec / mcf (sorec.pyx:78-143, mcf.pyx:80-144) over `data` (CofactorData), updating the f64
    device tensors U, V, Z and their RMSProp caches in place.  lambda_c is used by SoRec only; the hyperparameters are
    the reference's C floats.  loss: optional f64 device tensor [n_epochs, n_edges + n_ratings] that receives each
    update's loss term at its stored index."""
    L = require_cuda()
    users, items = _AtLeast(data.n_users), _AtLeast(data.n_items)
    z_rows = users if data.variant == "sorec" else items             # SoRec's Z rows are users, MCF's items
    k = _dev(U, torch.float64, "U", (users, None)).shape[1]
    _dev(cache_u, torch.float64, "cache_u", (users, k))
    _dev(V, torch.float64, "V", (items, k)), _dev(cache_v, torch.float64, "cache_v", (items, k))
    _dev(Z, torch.float64, "Z", (z_rows, k)), _dev(cache_z, torch.float64, "cache_z", (z_rows, k))
    if loss is not None:
        _dev(loss, torch.float64, "loss", (int(n_epochs), data.n_edges + data.n_ratings))
    check(L.b200_cofactor_fit(COFACTOR_VARIANTS[data.variant], ptr(data.a_id), ptr(data.b_id), ptr(data.val),
                              ptr(data.is_edge), ptr(data.level_ptr), data.n_levels, data.n_edges, data.n_ratings, int(k),
                              ptr(U), ptr(V), ptr(Z), ptr(cache_u), ptr(cache_v), ptr(cache_z), int(n_epochs),
                              float(lambda_c), float(lambda_reg), float(learning_rate), float(gamma), ptr(loss),
                              ptr(data.order) if loss is not None else None, current_stream()), "b200_cofactor_fit")


def csc_map(indptr, indices, n_cols):
    """Host checks of a CSR and its stable CSC position map (b200_csc_map, no device needed): (csc_ptr int32
    [n_cols + 1], csc_pos int32 [nnz]); column c lists the CSR indices of its entries in stored order."""
    L = _lib.load()
    indptr = np.ascontiguousarray(indptr, dtype=np.int32)
    indices = np.ascontiguousarray(indices, dtype=np.int32)
    csc_ptr = np.empty(int(n_cols) + 1, dtype=np.int32)
    csc_pos = np.empty(len(indices), dtype=np.int32)
    check(L.b200_csc_map(ptr(indptr), ptr(indices), len(indptr) - 1, int(n_cols), len(indices), ptr(csc_ptr),
                         ptr(csc_pos)), "b200_csc_map")
    return csc_ptr, csc_pos


def longest_first(lengths):
    """The ids by decreasing length, ties in id order (int32): the order the fits launch their rows in."""
    return np.argsort(-np.asarray(lengths), kind="stable").astype(np.int32)


class SparseLayout:
    """Device copy of an n_rows x n_cols sparse matrix, as B200_SPARSE (include/b200cornac.h) passes it: the CSR (ptr,
    idx, val) with each entry's row, and its stable CSC transpose (csc_map) with the row, CSR index and value of each CSC
    entry.  The values are stored as dtype (np.float32 or np.float64); col_lengths (host) counts each column's entries."""

    def __init__(self, indptr, indices, values, n_cols, dtype):
        require_cuda()
        if len(indices) >= 2 ** 31:
            raise B200Error("nnz >= 2^31 is not supported (int32 offsets)")
        indptr = np.ascontiguousarray(indptr, dtype=np.int32)
        indices = np.ascontiguousarray(indices, dtype=np.int32)
        val = np.ascontiguousarray(values, dtype=dtype)
        self.n_rows, self.n_cols, self.nnz = len(indptr) - 1, int(n_cols), len(indices)
        if len(val) != self.nnz:
            raise B200Error("%d values for %d entries" % (len(val), self.nnz))
        cptr, cpos = csc_map(indptr, indices, self.n_cols)
        row = np.repeat(np.arange(self.n_rows, dtype=np.int32), np.diff(indptr))
        self.col_lengths = np.diff(cptr)
        self.ptr, self.cptr = to_device(indptr), to_device(cptr)
        self.idx, self.row, self.val = (to_device(_pad(a)) for a in (indices, row, val))
        self.crow, self.cpos, self.cval = (to_device(_pad(a)) for a in (row[cpos], cpos, val[cpos]))

    def args(self):
        """The nine arguments of B200_SPARSE."""
        return [ptr(self.ptr), ptr(self.idx), ptr(self.row), ptr(self.val), self.nnz, ptr(self.cptr), ptr(self.crow),
                ptr(self.cpos), ptr(self.cval)]


class NmfData:
    """Device copy of NMF's ratings, built once per fit and used by every epoch: the ratings as a SparseLayout (f32), the
    items by decreasing number of ratings and, only when the biases are trained, the ratings in the level order of
    b200_pmf_schedule."""

    def __init__(self, indptr, indices, rating, n_items, use_bias):
        self.ratings = r = SparseLayout(indptr, indices, rating, n_items, np.float32)
        self.n_users, self.n_items, self.nnz = r.n_rows, r.n_cols, r.nnz
        self.item_order = to_device(_pad(longest_first(r.col_lengths)))
        self.use_bias = bool(use_bias)
        self.n_levels = 0
        self.s_uid = self.s_iid = self.s_rat = self.s_pos = self.level_ptr = None
        if self.use_bias:
            uid = np.repeat(np.arange(self.n_users, dtype=np.int32), np.diff(indptr))
            indices = np.asarray(indices, dtype=np.int32)
            rating = np.asarray(rating, dtype=np.float32)
            order, level_ptr = pmf_schedule(uid, indices, self.n_users, self.n_items)
            self.n_levels = len(level_ptr) - 1
            self.s_uid = to_device(_pad(uid[order]), torch.int32)
            self.s_iid = to_device(_pad(indices[order]), torch.int32)
            self.s_rat = to_device(_pad(rating[order]), torch.float32)
            self.s_pos = to_device(_pad(order), torch.int32)
            self.level_ptr = to_device(level_ptr, torch.int32)
        self.rp = torch.empty(max(self.nnz, 1), dtype=torch.float32, device="cuda")


def nmf_fit(data, U, V, Bu, Bi, n_epochs, mu=0.0, learning_rate=0.005, lambda_u=0.06, lambda_v=0.06, lambda_bu=0.02,
            lambda_bi=0.02, loss=None, workspace=None):
    """n_epochs epochs of NMF._fit_sgd (recom_nmf.pyx:182-267) over `data` (NmfData), updating the f32 device tensors U,
    V, Bu, Bi in place, bit for bit as the reference's serial loop.  The biases are trained when data.use_bias; they enter
    the predictions either way.  The hyperparameters are rounded to f32.  loss: optional f64 device tensor [n_epochs]
    that receives each epoch's sum err^2 + lambda_u |U|^2 + lambda_v |V|^2 (f64, not the reference's f32 order).
    workspace: optional f32 device tensor of at least U.numel() floats, not U itself (allocated per call otherwise)."""
    L = require_cuda()
    k = _dev(U, torch.float32, "U", (data.n_users, _AtLeast(1))).shape[1]
    _dev(V, torch.float32, "V", (data.n_items, k))
    _dev(Bu, torch.float32, "Bu", data.n_users), _dev(Bi, torch.float32, "Bi", data.n_items)
    if loss is not None:
        _dev(loss, torch.float64, "loss", int(n_epochs))
    workspace = _buf(workspace, torch.float32, "workspace", _AtLeast(U.numel()))
    if workspace.data_ptr() == U.data_ptr():
        raise B200Error("workspace must not alias U")
    check(L.b200_nmf_fit(data.n_users, data.n_items, *data.ratings.args(), ptr(data.item_order), ptr(data.s_uid),
                         ptr(data.s_iid), ptr(data.s_rat), ptr(data.s_pos), ptr(data.level_ptr), data.n_levels, int(k), ptr(U),
                         ptr(V), ptr(Bu), ptr(Bi), ptr(data.rp), ptr(workspace), int(n_epochs), _f32(mu), _f32(learning_rate),
                         _f32(lambda_u), _f32(lambda_v), _f32(lambda_bu), _f32(lambda_bi), int(data.use_bias), ptr(loss),
                         current_stream()), "b200_nmf_fit")


class EfmData:
    """Device copy of EFM's three matrices, built once per fit and used by every iteration: A (users x items), X (users x
    aspects) and Y (items x aspects) as SparseLayouts (f32); the launch orders of the item and aspect rows (longest
    chains first); the prediction buffer."""

    def __init__(self, A, X, Y):
        A, X, Y = (_sp.csr_matrix(M) for M in (A, X, Y))
        self.n_users, self.n_items = A.shape
        self.n_aspects = X.shape[1]
        if X.shape[0] != self.n_users or Y.shape != (self.n_items, self.n_aspects):
            raise B200Error("A %s, X %s and Y %s do not agree in shape" % (A.shape, X.shape, Y.shape))
        self.a, self.x, self.y = (SparseLayout(M.indptr, M.indices, M.data, M.shape[1], np.float32) for M in (A, X, Y))
        self.item_order = to_device(_pad(longest_first(self.a.col_lengths + np.diff(Y.indptr))))
        self.aspect_order = to_device(_pad(longest_first(self.x.col_lengths + self.y.col_lengths)))
        self.pred = torch.empty(max(self.a.nnz + self.x.nnz + self.y.nnz, 1), dtype=torch.float32, device="cuda")

    def args(self):
        """B200_EFM_DATA of include/b200cornac.h."""
        return self.a.args() + self.x.args() + self.y.args() + [ptr(self.item_order), ptr(self.aspect_order),
                                                                  self.n_users, self.n_items, self.n_aspects]


def efm_fit(data, U1, U2, V, H1, H2, n_iter, lambda_x=1.0, lambda_y=1.0, lambda_u=0.01, lambda_h=0.01, lambda_v=0.01,
            loss=None, workspace=None):
    """n_iter iterations of EFM._fit_efm (recom_efm.pyx:268-353) over `data` (EfmData), updating the f32 device tensors
    U1, U2, V, H1, H2 in place, bit for bit as the reference.s serial loop with the defined dot.
    The hyperparameters are rounded to f32.  loss: optional f64 device tensor [n_iter] that receives each iteration's
    loss, summed in f64 (not the reference's f32 order).  workspace: optional f32 device tensor of
    efm_workspace_floats(...) floats (allocated per call otherwise)."""
    L_ = require_cuda()
    E = _dev(U1, torch.float32, "U1", (data.n_users, _AtLeast(1))).shape[1]
    Lw = _dev(H1, torch.float32, "H1", (data.n_users, _AtLeast(1))).shape[1]
    _dev(U2, torch.float32, "U2", (data.n_items, E)), _dev(V, torch.float32, "V", (data.n_aspects, E))
    _dev(H2, torch.float32, "H2", (data.n_items, Lw))
    if loss is not None:
        _dev(loss, torch.float64, "loss", int(n_iter))
    need = efm_workspace_floats(data.n_users, data.n_items, data.n_aspects, E, Lw)
    workspace = _buf(workspace, torch.float32, "workspace", _AtLeast(need))
    check(L_.b200_efm_fit(*data.args(), int(E), int(Lw), ptr(U1), ptr(U2), ptr(V), ptr(H1), ptr(H2), ptr(workspace), ptr(data.pred),
                          int(n_iter), _f32(lambda_x), _f32(lambda_y), _f32(lambda_u), _f32(lambda_h), _f32(lambda_v),
                          ptr(loss), current_stream()), "b200_efm_fit")


def efm_workspace_floats(n_users, n_items, n_aspects, E, L):
    """Floats of b200_efm_fit's workspace: the second buffer of each factor matrix."""
    return (int(n_users) + int(n_items)) * (int(E) + int(L)) + int(n_aspects) * int(E)


def efm_queries(U1, H1, V, num_most_cared, alpha, rating_scale, user_idx=None):
    """[n_q, E + L] f32 query vectors of the aspect-weighted rank (b200_efm_queries) of the users user_idx (int64 device
    tensor; None: every row of U1): Q[q] . [U2 | H2][i] is EFM.rank's row alpha * explicit + (1 - alpha) * score."""
    L_ = require_cuda()
    n_users, E = _dev(U1, torch.float32, "U1", (None, None)).shape
    Lw = _dev(H1, torch.float32, "H1", (n_users, None)).shape[1]
    if _dev(V, torch.float32, "V", (None, None)).shape[0]:           # without aspects V's width is never read
        _dev(V, torch.float32, "V", (None, E))
    if user_idx is None:
        user_idx = torch.arange(n_users, dtype=torch.int64, device=U1.device)
    _dev(user_idx, torch.int64, "user_idx")
    Q = torch.empty((user_idx.numel(), E + Lw), dtype=torch.float32, device=U1.device)
    check(L_.b200_efm_queries(ptr(user_idx), user_idx.numel(), ptr(U1), ptr(H1), ptr(V), int(V.shape[0]), E, Lw,
                              int(num_most_cared), float(alpha), float(rating_scale), ptr(Q), current_stream()),
          "b200_efm_queries")
    return Q


MTER_PARAMS = ("U", "I", "A", "O", "G1", "G2", "G3")
_MTER_DRAW_CHUNK = 1 << 24        # draws uploaded per chunk (64 MB of int32)


class MterData:
    """The arrays `fit` hands to `_fit_mter` (recom_mter.pyx:334-371), in the reference's order.

    X, YU, YI: f32 values; X_uids / X_iids / X_aids, YU_uids / YU_aids / YU_oids, YI_iids / YI_aids / YI_oids: int32
    indices.  indptr / indices: the rating CSR (sorted columns; repeated pairs summed, as scipy builds it); user_ids:
    the row of each CSR entry; pair_rating: the f32 rating of each entry's exact (user, item) pair, the last value a
    repeated pair has (what the reference's IntFloatDict keeps) -- the BPR skip and sign rule reads it."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class StreamDraws:
    """Seeded mt19937 sample streams (the reference's RNGVector, one thread each), drawn on the host in chunks of
    iterations and uploaded through two pinned buffers: chunk k + 1 is drawn while the GPU runs chunk k.  streams:
    (seed, hi, n) per stream, n draws in [0, hi] per iteration; an iteration's draws are the streams' in that order."""

    def __init__(self, streams, max_chunk):
        self.samplers = [MTSampler(int(s)) for s, _, _ in streams]
        self.hi = [int(hi) for _, hi, _ in streams]
        self.n = [int(n) for _, _, n in streams]
        self.per_iter = sum(self.n)
        self.chunk = max(1, min(int(max_chunk), _MTER_DRAW_CHUNK // max(self.per_iter, 1)))
        self.host = [torch.empty((self.chunk, self.per_iter), dtype=torch.int32).pin_memory() for _ in range(2)]
        self.dev = [torch.empty((self.chunk, self.per_iter), dtype=torch.int32, device="cuda") for _ in range(2)]
        self.done = [None, None]
        self.slot = 0

    def draw(self, n_iter):
        """Draws of the next n_iter iterations as one int64 array [n_iter, per_iter]."""
        cols = [s.fill(h, n_iter * n).reshape(n_iter, n) for s, h, n in zip(self.samplers, self.hi, self.n)]
        return np.concatenate(cols, axis=1)

    def next(self, n_iter):
        """Device draws of the next n_iter (<= chunk) iterations."""
        k = self.slot
        self.slot ^= 1
        if self.done[k] is not None:
            self.done[k].synchronize()                 # the last upload from this pinned buffer has finished
        host = self.host[k][:n_iter]
        host.numpy()[:] = self.draw(n_iter)
        dev = self.dev[k][:n_iter]
        dev.copy_(host, non_blocking=True)
        self.done[k] = torch.cuda.Event()
        self.done[k].record()
        return dev


class MterDraws(StreamDraws):
    """MTER's five seeded sample streams (uia, uao, iao, pos, neg) as StreamDraws.  `extra`: (seed, hi, n) of further
    streams, whose n draws of an iteration follow the five's."""

    def __init__(self, seeds, data, n_el, n_bpr, max_chunk, extra=()):
        his = [len(data.X) - 1, len(data.YU) - 1, len(data.YI) - 1, len(data.indices) - 1, data.n_items - 1]
        ns = [n_el, n_el, n_el, n_bpr, n_bpr]
        super().__init__(list(zip(seeds, his, ns)) + list(extra), max_chunk)


class MterDeviceData:
    """Device copy of MTER's training data (a recom_mter.MterData): the three sentiment tensors and the ratings' CSR
    with each entry's row and pair rating, uploaded once per fit."""

    def __init__(self, data):
        i32 = lambda a: to_device(_pad(np.asarray(a, dtype=np.int32)), torch.int32)      # noqa: E731
        f32 = lambda a: to_device(_pad(np.asarray(a, dtype=np.float32)), torch.float32)  # noqa: E731
        self.n_users, self.n_items = int(data.n_users), int(data.n_items)
        self.n_aspects, self.n_opinions = int(data.n_aspects), int(data.n_opinions)
        self.x = [f32(data.X), i32(data.X_uids), i32(data.X_iids), i32(data.X_aids)]
        self.yu = [f32(data.YU), i32(data.YU_uids), i32(data.YU_aids), i32(data.YU_oids)]
        self.yi = [f32(data.YI), i32(data.YI_iids), i32(data.YI_aids), i32(data.YI_oids)]
        self.n_x, self.n_yu, self.n_yi = len(data.X), len(data.YU), len(data.YI)
        self.csr = [i32(data.indptr), i32(data.indices), i32(data.user_ids), f32(data.pair_rating)]
        self.nnz = len(data.indices)

    def args(self):
        return [self.n_users, self.n_items, self.n_aspects, self.n_opinions]


def comparer_draws(seeds, data, n_el, n_bpr, n_pair, max_chunk):
    """ComparERSub's six seeded streams as an MterDraws.  `seeds` in the reference's order (uia, uao, iao, pair, pos,
    neg); an iteration's draws are MTER's five streams', then the n_pair draws of the pair stream over the pair list of
    `data` (ComparerData).  With n_pair = 0 the pair stream is seeded but never drawn from."""
    uia, uao, iao, pair, pos, neg = seeds
    extra = [(pair, len(data.p_user_indices) - 1, n_pair)] if n_pair > 0 else []
    return MterDraws([uia, uao, iao, pos, neg], data, n_el, n_bpr, max_chunk, extra=extra)


class ComparerDeviceData(MterDeviceData):
    """MterDeviceData plus ComparERSub's pair list (user, earlier, later, aspect), in the reference's order."""

    def __init__(self, data):
        super().__init__(data)
        i32 = lambda a: to_device(_pad(np.asarray(a, dtype=np.int32)), torch.int32)      # noqa: E731
        self.pairs = [i32(data.p_user_indices), i32(data.earlier_indices), i32(data.later_indices),
                      i32(data.aspect_indices)]
        self.n_plist = len(data.p_user_indices)


def mter_workspace_bytes(data, dims, n_el, n_bpr):
    L_ = require_cuda()
    return int(L_.b200_mter_workspace_bytes(data.n_users, data.n_items, data.n_aspects, data.n_opinions, *dims,
                                            int(n_el), int(n_bpr)))


def comparer_sub_workspace_bytes(data, dims, n_el, n_bpr, n_pair):
    L_ = require_cuda()
    return int(L_.b200_comparer_sub_workspace_bytes(data.n_users, data.n_items, data.n_aspects, data.n_opinions,
                                                    *dims, int(n_el), int(n_bpr), int(n_pair)))


def mter_fit(data, params, sgrad, draws, n_iter, n_el, n_bpr, lr=0.1, lambda_reg=0.1, lambda_bpr=10.0, counts=None,
             losses=None, workspace=None, unordered=False, philox_seed=None, iter0=0, phase_ns=None):
    """n_iter iterations of MTER._fit_mter (recom_mter.pyx:434-675) over `data` (MterDeviceData), bit for bit as the
    reference's serial f32 loop given the draws.  params / sgrad: sequences of the f32 device tensors U, I, A, O, G1,
    G2, G3 and their AdaGrad sums, updated in place.  draws: int32 device tensor [n_iter, 3 n_el + 2 n_bpr] (per
    iteration the uia, uao, iao, pos and neg draws).  counts: int64 device [2] (+= correct, skipped).  losses: f64
    device [2] or None (+= loss, bpr_loss, summed in f64).  workspace: uint8 device tensor of mter_workspace_bytes
    that is zero before its first use (the fit leaves the part it needs zero); allocated per call when None.
    unordered: sum the rows' gradients per sample with f32 atomics (no fixed order).  philox_seed: draw on the device
    from Philox4x32-10 with this key, iterations iter0, iter0 + 1, ... (draws is then ignored and may be None).
    phase_ns: int64 device [4] or None (+= nanoseconds of the predictions, owners + stored terms, gradients, AdaGrad)."""
    return _tensor_fit(data, params, sgrad, draws, n_iter, n_el, n_bpr, 0, lr, lambda_reg, lambda_bpr, 0.0, counts,
                       losses, workspace, unordered, philox_seed, iter0, phase_ns)


def comparer_sub_fit(data, params, sgrad, draws, n_iter, n_el, n_bpr, n_pair, lr=0.5, lambda_reg=0.1, lambda_bpr=10.0,
                     lambda_d=0.01, counts=None, losses=None, workspace=None, unordered=False, philox_seed=None, iter0=0,
                     phase_ns=None):
    """n_iter iterations of ComparERSub._fit_mter (recom_comparer_sub.pyx:487-760) over `data` (ComparerDeviceData):
    mter_fit plus n_pair samples per iteration from the pair list, bit for bit as the reference's serial f32 loop given
    the draws.  draws: int32 device tensor [n_iter, 3 n_el + 2 n_bpr + n_pair] (ComparerDraws' layout).  counts: int64
    device [3] (+= correct, skipped, aspect_correct).  losses: f64 device [3] or None (+= loss, bpr_loss,
    aspect_bpr_loss).  workspace: of comparer_sub_workspace_bytes.  The other arguments are mter_fit's."""
    if int(n_pair) < 0 or (int(n_pair) > 0 and data.n_plist == 0):
        raise B200Error("%d pair samples from a pair list of %d" % (int(n_pair), data.n_plist))
    return _tensor_fit(data, params, sgrad, draws, n_iter, n_el, n_bpr, int(n_pair), lr, lambda_reg, lambda_bpr,
                       lambda_d, counts, losses, workspace, unordered, philox_seed, iter0, phase_ns)


def _tensor_fit(data, params, sgrad, draws, n_iter, n_el, n_bpr, n_pair, lr, lambda_reg, lambda_bpr, lambda_d, counts,
                losses, workspace, unordered, philox_seed, iter0, phase_ns):
    """mter_fit (n_pair = 0, b200_mter_fit) and comparer_sub_fit (b200_comparer_sub_fit)."""
    L_ = require_cuda()
    comparer = isinstance(data, ComparerDeviceData)
    n_counts = 3 if comparer else 2
    G1, G2 = params[4:6]
    d1, d2, d3 = _dev(G1, torch.float32, "G1", (None, None, None)).shape
    d4 = _dev(G2, torch.float32, "G2", (d1, d3, None)).shape[2]
    dims = (d1, d2, d3, d4)
    shapes = ((data.n_users, d1), (data.n_items, d2), (data.n_aspects + 1, d3), (data.n_opinions, d4), (d1, d2, d3),
              (d1, d3, d4), (d2, d3, d4))
    for name, t, st, shape in zip(MTER_PARAMS, params, sgrad, shapes):
        _dev(t, torch.float32, name, shape), _dev(st, torch.float32, "sgrad_" + name, shape)
    if philox_seed is None:
        _dev(draws, torch.int32, "draws", _AtLeast(int(n_iter) * (3 * int(n_el) + 2 * int(n_bpr) + int(n_pair))))
    else:
        draws = None
    if phase_ns is not None:
        _dev(phase_ns, torch.int64, "phase_ns", _AtLeast(4))
    counts = _buf(counts, torch.int64, "counts", _AtLeast(n_counts), zero=True)
    if losses is not None:
        _dev(losses, torch.float64, "losses", _AtLeast(n_counts))
    need = (comparer_sub_workspace_bytes(data, dims, n_el, n_bpr, n_pair) if comparer else
            mter_workspace_bytes(data, dims, n_el, n_bpr))
    workspace = _buf(workspace, torch.uint8, "workspace", _AtLeast(need), zero=True)
    pp = (ctypes.c_void_p * 7)(*[ptr(t) for t in params])
    ps = (ctypes.c_void_p * 7)(*[ptr(t) for t in sgrad])
    head = [*data.args(), *dims, *[ptr(t) for t in data.x], data.n_x, *[ptr(t) for t in data.yu], data.n_yu,
            *[ptr(t) for t in data.yi], data.n_yi, *[ptr(t) for t in data.csr], data.nnz]
    flags = (_lib.MTER_UNORDERED if unordered else 0) | (0 if philox_seed is None else _lib.MTER_PHILOX)
    tail = [flags, int(philox_seed or 0) & (2 ** 64 - 1), int(iter0), ptr(counts), ptr(losses), ptr(phase_ns),
            current_stream()]
    if comparer:
        check(L_.b200_comparer_sub_fit(*head, *[ptr(t) for t in data.pairs], data.n_plist, int(n_el), int(n_bpr),
                                       int(n_pair), int(n_iter), ptr(draws), pp, ps, ptr(workspace), _f32(lr),
                                       _f32(lambda_reg), _f32(lambda_bpr), _f32(lambda_d), *tail),
              "b200_comparer_sub_fit")
    else:
        check(L_.b200_mter_fit(*head, int(n_el), int(n_bpr), int(n_iter), ptr(draws), pp, ps, ptr(workspace), _f32(lr),
                               _f32(lambda_reg), _f32(lambda_bpr), *tail),
              "b200_mter_fit")
    return counts


def mter_queries(U, G1, A):
    """[n_users, d2] f32 rank queries (b200_mter_queries): Q[u] . I[i] is MTER.score(u)[i] = einsum(G1, U[u], I[i],
    A[-1]) up to rounding.  M = G1 . A[-1] and Q = U . M are f64 sums in index order, each rounded once to f32."""
    L_ = require_cuda()
    d1, d2, d3 = _dev(G1, torch.float32, "G1", (None, None, None)).shape
    _dev(U, torch.float32, "U", (None, d1)), _dev(A, torch.float32, "A", (_AtLeast(1), d3))
    Q = torch.empty((U.shape[0], d2), dtype=torch.float32, device=U.device)
    check(L_.b200_mter_queries(ptr(U), int(U.shape[0]), ptr(G1), ptr(A[-1]), d1, d2, d3, ptr(Q), current_stream()),
          "b200_mter_queries")
    return Q


def comparer_rank_rows(U, I, A, G1, user_idx, n_top, alpha, n_items=None, out=None):
    """[n_q, n_items] f32 device rank rows of ComparERSub (b200_comparer_rank_rows): for each user u of user_idx
    (int64 device) and item i < n_items (default all rows of I), alpha * mean(the n_top largest ts3[i, a < n_aspects])
    + (1 - alpha) * ts3[i, n_aspects] with ts3[i, a] = sum_qr I[i, q] (sum_p G1[p, q, r] U[u, p]) A[a, r], every sum in
    f64 and one rounding to f32.  out: an optional [n_q, n_items] f32 device buffer to write."""
    L_ = require_cuda()
    d1, d2, d3 = _dev(G1, torch.float32, "G1", (None, None, None)).shape
    _dev(U, torch.float32, "U", (None, d1)), _dev(A, torch.float32, "A", (_AtLeast(2), d3))
    _dev(I, torch.float32, "I", (None if n_items is None else _AtLeast(n_items), d2))
    n_items = int(I.shape[0] if n_items is None else n_items)
    if n_items < 0:
        raise B200Error("n_items must be >= 0, got %d" % n_items)
    n_q = _dev(user_idx, torch.int64, "user_idx").numel()
    out = _buf(out, torch.float32, "out", (n_q, n_items))
    check(L_.b200_comparer_rank_rows(ptr(U), ptr(I), ptr(A), ptr(G1), ptr(user_idx), n_q, n_items, d1, d2, d3,
                                     int(A.shape[0]) - 1, int(n_top), float(alpha), ptr(out), current_stream()),
          "b200_comparer_rank_rows")
    return out


LRPPM_PARAMS = ("U", "I", "UA", "IA")


class LrppmData:
    """The arrays LRPPM.fit hands to `_fit` (recom_lrppm.pyx:289-303) and the lookups its loop makes, in the reference's
    order.  u_indices / i_indices / r_values: the train set's triples; X_uids / X_iids / X_aids / X_l_ui: the review
    triples and their weights; aspect_keys: the sorted distinct wrapped get_key3 keys of the triples; rating_keys /
    rating_values: the sorted distinct wrapped get_key(u, i) keys of the ratings with the f32 value the reference's
    IntFloatDict keeps; item_aspect_quality: the f64 item x aspect quality CSR."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class LrppmDeviceData:
    """Device copy of an LrppmData, uploaded once per fit."""

    def __init__(self, data):
        i32 = lambda a: to_device(_pad(np.asarray(a, dtype=np.int32)), torch.int32)      # noqa: E731
        f32 = lambda a: to_device(_pad(np.asarray(a, dtype=np.float32)), torch.float32)  # noqa: E731
        self.n_users, self.n_items, self.n_aspects = int(data.n_users), int(data.n_items), int(data.n_aspects)
        self.ratings = [i32(data.u_indices), i32(data.i_indices), f32(data.r_values)]
        self.n_r = len(data.r_values)
        self.triples = [i32(data.X_uids), i32(data.X_iids), i32(data.X_aids), f32(data.X_l_ui)]
        self.n_x = len(data.X_uids)
        self.akeys = i32(data.aspect_keys)
        self.n_akeys = len(data.aspect_keys)
        self.rkeys, self.rvals = i32(data.rating_keys), f32(data.rating_values)
        self.n_rkeys = len(data.rating_keys)


def lrppm_draws(seeds, data, n_samples, n_ranking_samples, max_chunk):
    """LRPPM's three seeded streams (pos, pos_uia, neg_uia; recom_lrppm.pyx:307-309) as StreamDraws."""
    pos, pos_uia, neg_uia = seeds
    return StreamDraws([(pos, len(data.r_values) - 1, n_samples), (pos_uia, len(data.X_uids) - 1, n_ranking_samples),
                        (neg_uia, data.n_aspects - 1, n_ranking_samples)], max_chunk)


def lrppm_workspace_bytes(data, k, n_samples, n_ranking_samples):
    L_ = require_cuda()
    return int(L_.b200_lrppm_workspace_bytes(data.n_users, data.n_items, data.n_aspects, int(k), int(n_samples),
                                             int(n_ranking_samples)))


def lrppm_fit(data, params, draws, n_iter, n_samples, n_ranking_samples, lr=0.1, reg=0.01, ld=1.0, counts=None,
              losses=None, workspace=None, philox_seed=None, iter0=0, phase_ns=None):
    """Up to n_iter iterations of LRPPM._fit (recom_lrppm.pyx:356-482) over `data` (LrppmDeviceData), bit for bit as the
    reference's compiled float loop given the draws; the fit stops after the first iteration that leaves every
    parameter isclose to its value before it (recom_lrppm.pyx:337-344).  params: the f32 device tensors U, I, UA, IA,
    updated in place.  draws: int32 device tensor [n_iter, n_samples + 2 n_ranking_samples] (pos, pos_uia, neg_uia).
    counts: int64 device [4] (+= correct, skipped, iterations run; [3] = 1 once converged).  losses: f64 device [3] or
    None (+= loss, ranking_loss, r_loss).  workspace: uint8 device tensor of lrppm_workspace_bytes that is zero before
    its first use.  philox_seed: draw on the device from Philox4x32-10 with this key, iterations iter0, iter0 + 1, ...
    (draws is then ignored).  phase_ns: int64 device [3] or None (+= nanoseconds of the predictions, del chains, dense
    step)."""
    L_ = require_cuda()
    k = _dev(params[0], torch.float32, "U", (data.n_users, None)).shape[1]
    for name, t, rows in zip(LRPPM_PARAMS, params, (data.n_users, data.n_items, data.n_aspects, data.n_aspects)):
        _dev(t, torch.float32, name, (rows, k))
    n_s, n_rk = int(n_samples), int(n_ranking_samples)
    if n_s < 0 or n_rk < 0:
        raise B200Error("n_samples and n_ranking_samples must not be negative")
    if philox_seed is None:
        _dev(draws, torch.int32, "draws", _AtLeast(int(n_iter) * (n_s + 2 * n_rk)))
    else:
        draws = None
    if phase_ns is not None:
        _dev(phase_ns, torch.int64, "phase_ns", _AtLeast(3))
    counts = _buf(counts, torch.int64, "counts", _AtLeast(4), zero=True)
    if losses is not None:
        _dev(losses, torch.float64, "losses", _AtLeast(3))
    workspace = _buf(workspace, torch.uint8, "workspace", _AtLeast(lrppm_workspace_bytes(data, k, n_s, n_rk)), zero=True)
    pp = (ctypes.c_void_p * 4)(*[ptr(t) for t in params])
    check(L_.b200_lrppm_fit(data.n_users, data.n_items, data.n_aspects, int(k), *[ptr(t) for t in data.ratings],
                            data.n_r, *[ptr(t) for t in data.triples], data.n_x, ptr(data.akeys), data.n_akeys,
                            ptr(data.rkeys), ptr(data.rvals), data.n_rkeys, n_s, n_rk, int(n_iter), ptr(draws), pp,
                            ptr(workspace), _f32(lr), _f32(reg), _f32(ld), 0 if philox_seed is None else _lib.LRPPM_PHILOX,
                            int(philox_seed or 0) & (2 ** 64 - 1), int(iter0), ptr(counts), ptr(losses), ptr(phase_ns),
                            current_stream()),
          "b200_lrppm_fit")
    return counts


class LrppmQuality:
    """Device copy of the f64 item x aspect quality CSR of a trained LRPPM."""

    def __init__(self, Q):
        Q = _sp.csr_matrix(Q)
        self.n_rows, self.n_aspects = Q.shape
        self.indptr = to_device(Q.indptr.astype(np.int32), torch.int32)
        self.indices = to_device(_pad(Q.indices.astype(np.int32)), torch.int32)
        self.data = to_device(_pad(Q.data.astype(np.float64)), torch.float64)


def lrppm_rank_rows(U, I, UA, IA, quality, user_idx, n_top, alpha, rating_scale, n_items=None, out=None):
    """[n_q, n_items] f64 device rank rows of LRPPM (b200_lrppm_rank_rows): for each user u of user_idx (int64 device)
    and item i < n_items (default all rows of I), alpha rating_scale mean(the n_top largest s[i, a], each times
    q[i, a]) + f32(f32(1 - alpha) f32(I[i] . U[u])), with s[i, a] = f32(f32(f32(UA[a] . U[u]) + f32(I[i] . IA[a])) +
    f32(I[i] . U[u])).  quality: an LrppmQuality.  out: an optional [n_q, n_items] f64 device buffer to write."""
    L_ = require_cuda()
    k = _dev(U, torch.float32, "U", (None, None)).shape[1]
    n_aspects = _dev(UA, torch.float32, "UA", (None, k)).shape[0]
    _dev(IA, torch.float32, "IA", (n_aspects, k))
    _dev(I, torch.float32, "I", (None if n_items is None else _AtLeast(n_items), k))
    n_items = int(I.shape[0] if n_items is None else n_items)
    if n_items < 0 or n_items > quality.n_rows or quality.n_aspects != n_aspects:
        raise B200Error("quality of shape (%d, %d) for %d items and %d aspects" % (quality.n_rows, quality.n_aspects,
                                                                                 n_items, n_aspects))
    n_q = _dev(user_idx, torch.int64, "user_idx").numel()
    out = _buf(out, torch.float64, "out", (n_q, n_items))
    check(L_.b200_lrppm_rank_rows(ptr(U), ptr(I), ptr(UA), ptr(IA), ptr(quality.indptr), ptr(quality.indices),
                                  ptr(quality.data), ptr(user_idx), n_q, n_items, int(k), int(n_aspects), int(n_top),
                                  float(alpha), float(rating_scale), ptr(out), current_stream()),
          "b200_lrppm_rank_rows")
    return out


class HpfData(SparseLayout):
    """Device copy of HPF's ratings, built once per fit and used by every iteration: a SparseLayout (f64) with items
    ascending in each row, and the scratch of the fit.  rid, cid, val: the stored (user, item, value) triplets, each pair
    at most once; zeros are the caller's to drop."""

    def __init__(self, rid, cid, val, n_users, n_items):
        rid = np.asarray(rid, dtype=np.int64)
        cid = np.asarray(cid, dtype=np.int64)
        val = np.asarray(val, dtype=np.float64)
        self.n_users, self.n_items, nnz = int(n_users), int(n_items), len(rid)
        if len(cid) != nnz or len(val) != nnz:
            raise B200Error("rid, cid and val differ in length (%d, %d, %d)" % (nnz, len(cid), len(val)))
        if nnz and (rid.min() < 0 or rid.max() >= self.n_users or cid.min() < 0 or cid.max() >= self.n_items):
            raise B200Error("a rating lies outside the %d x %d matrix" % (self.n_users, self.n_items))
        order = np.lexsort((cid, rid))                       # CSR: users, then items ascending
        rid, cid, val = rid[order], cid[order], val[order]
        if nnz > 1 and np.any((rid[1:] == rid[:-1]) & (cid[1:] == cid[:-1])):
            raise B200Error("a (user, item) pair is stored twice")
        indptr = np.zeros(self.n_users + 1, dtype=np.int64)
        np.cumsum(np.bincount(rid, minlength=self.n_users), out=indptr[1:])
        super().__init__(indptr, cid, val, self.n_items, np.float64)
        self._work = {}

    def workspace(self, k):
        """The device scratch of b200_hpf_fit / b200_hpf_update for k factors, allocated once per k."""
        if k not in self._work:
            nbytes = _lib.load().b200_hpf_workspace_bytes(self.n_users, self.n_items, self.nnz, int(k))
            if nbytes < 0:
                raise B200Error("bad HPF sizes")
            self._work = {k: torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")}
        return self._work[k]


def _hpf_state(data, Gs, Gr, Ls, Lr, Kr, Tr):
    """k of an HPF state, checked: Gs, Gr [n_users, k], Ls, Lr [n_items, k], Kr [n_users], Tr [n_items]."""
    k = _dev(Gs, torch.float64, "Gs", (data.n_users, _AtLeast(1))).shape[1]
    _dev(Gr, torch.float64, "Gr", (data.n_users, k))
    _dev(Ls, torch.float64, "Ls", (data.n_items, k)), _dev(Lr, torch.float64, "Lr", (data.n_items, k))
    _dev(Kr, torch.float64, "Kr", data.n_users), _dev(Tr, torch.float64, "Tr", data.n_items)
    return int(k)


def hpf_fit(data, hierarchical, Gs, Gr, Ls, Lr, Kr, Tr, max_iter):
    """max_iter iterations of hpf_cpp (hierarchical) or pf_cpp (cpp_hpf.cpp:139-275) over `data` (HpfData), updating the
    f64 device tensors Gs, Gr [n_users, k], Ls, Lr [n_items, k], Kr [n_users], Tr [n_items] in place.  Two calls of a and
    b iterations equal one call of a + b."""
    L = require_cuda()
    k = _hpf_state(data, Gs, Gr, Ls, Lr, Kr, Tr)
    if int(max_iter) < 0:
        raise B200Error("max_iter must be >= 0, got %d" % int(max_iter))
    check(L.b200_hpf_fit(int(bool(hierarchical)), data.n_users, data.n_items, k, *data.args(), ptr(Gs), ptr(Gr), ptr(Ls),
                         ptr(Lr), ptr(Kr), ptr(Tr), int(max_iter), ptr(data.workspace(k)), current_stream()),
          "b200_hpf_fit")


def hpf_update(data, hierarchical, Lt, Lb, Gs, Gr, Ls, Lr, Kr, Tr):
    """One iteration of the fit from given expectations Lt [n_users, k] and Lb [n_items, k] (f64 device tensors)."""
    L = require_cuda()
    k = _hpf_state(data, Gs, Gr, Ls, Lr, Kr, Tr)
    _dev(Lt, torch.float64, "Lt", (data.n_users, k)), _dev(Lb, torch.float64, "Lb", (data.n_items, k))
    check(L.b200_hpf_update(int(bool(hierarchical)), data.n_users, data.n_items, k, *data.args(), ptr(Lt), ptr(Lb),
                            ptr(Gs), ptr(Gr), ptr(Ls), ptr(Lr), ptr(Kr), ptr(Tr), ptr(data.workspace(k)), current_stream()),
          "b200_hpf_update")


def hpf_expect(shape, rate, out=None):
    """exp(digamma(shape) - log(rate)) element-wise on f64 device tensors, with HPF's stored-entry rules: a term whose
    argument is <= 0 is dropped, and an entry with both dropped is 0."""
    L = require_cuda()
    dims = tuple(_dev(shape, torch.float64, "shape").shape)
    _dev(rate, torch.float64, "rate", dims)
    out = _buf(out, torch.float64, "out", dims)
    check(L.b200_hpf_expect(ptr(shape), ptr(rate), shape.numel(), ptr(out), current_stream()), "b200_hpf_expect")
    return out


C2PF_VARIANTS = {"c2pf": 0, "tc2pf": 1, "rc2pf": 2}


class C2pfGraph:
    """Device copy of C2PF's context graph: a symmetric n_items x n_items CSC pattern (c_ptr int32[n_items + 1], c_row
    int32[n_edges], rows ascending in each column), the position c_mir of each entry's mirror, and util f64[n_items], the
    column sums of the graph's values.  `ratings` is the HpfData of the same items; the scratch is kept here."""

    def __init__(self, ratings, c_ptr, c_row, c_mir, util):
        require_cuda()
        self.ratings = ratings
        d = ratings.n_items
        c_ptr, c_row, c_mir = (np.asarray(x, dtype=np.int64) for x in (c_ptr, c_row, c_mir))
        self.n_edges = len(c_row)
        if len(c_ptr) != d + 1 or c_ptr[0] != 0 or c_ptr[-1] != self.n_edges or np.any(np.diff(c_ptr) < 0):
            raise B200Error("c_ptr is not the column pointer of a %d-column pattern with %d entries" % (d, self.n_edges))
        c_col = np.repeat(np.arange(d), np.diff(c_ptr))
        if len(c_mir) != self.n_edges or len(util) != d:
            raise B200Error("c_mir must hold %d values and util %d" % (self.n_edges, d))
        if self.n_edges and (c_row.min() < 0 or c_row.max() >= d or c_mir.min() < 0 or c_mir.max() >= self.n_edges or
                             not np.array_equal(c_row[c_mir], c_col) or not np.array_equal(c_col[c_mir], c_row)):
            raise B200Error("c_mir does not map every entry (r, i) to a stored (i, r)")
        self.c_ptr = to_device(c_ptr.astype(np.int32), torch.int32)
        self.c_row = to_device(_pad(c_row.astype(np.int32)), torch.int32)
        self.c_col = to_device(_pad(c_col.astype(np.int32)), torch.int32)
        self.c_mir = to_device(_pad(c_mir.astype(np.int32)), torch.int32)
        self.util = to_device(_pad(np.asarray(util, dtype=np.float64)), torch.float64)
        self._work = {}

    def workspace(self, k):
        if k not in self._work:
            r = self.ratings
            nbytes = _lib.load().b200_c2pf_workspace_bytes(r.n_users, r.n_items, r.nnz, self.n_edges, int(k))
            if nbytes < 0:
                raise B200Error("bad C2PF sizes")
            self._work = {k: torch.empty(nbytes // 8, dtype=torch.float64, device="cuda")}
        return self._work[k]


def _c2pf_args(graph, variant, at, bt, state):
    """The B200_C2PF_PARAMS of a call.  state = (Gs, Gr, Ls, Lr, L2s, L2r, L3s, L3r, T3r), f64 device tensors; None for the
    matrices the variant does not have (tc2pf: L2s, L2r; rc2pf: Ls, Lr)."""
    if variant not in C2PF_VARIANTS:
        raise B200Error("variant must be one of %s, got %r" % (sorted(C2PF_VARIANTS), variant))
    r = graph.ratings
    Gs, Gr, Ls, Lr, L2s, L2r, L3s, L3r, T3r = state
    k = _dev(Gs, torch.float64, "Gs", (r.n_users, _AtLeast(1))).shape[1]
    _dev(Gr, torch.float64, "Gr", (r.n_users, k))
    if variant == "rc2pf":
        Ls = Lr = None
    else:
        _dev(Ls, torch.float64, "Ls", (r.n_items, k)), _dev(Lr, torch.float64, "Lr", (r.n_items, k))
    if variant == "tc2pf":
        L2s = L2r = None
    else:
        _dev(L2s, torch.float64, "L2s", (r.n_items, k)), _dev(L2r, torch.float64, "L2r", (r.n_items, k))
    n_edges = max(graph.n_edges, 1)
    _dev(L3s, torch.float64, "L3s", n_edges), _dev(L3r, torch.float64, "L3r", n_edges)
    _dev(T3r, torch.float64, "T3r", r.n_items)
    return int(k), [C2PF_VARIANTS[variant], r.n_users, r.n_items, int(k), *r.args(), graph.n_edges, ptr(graph.c_ptr),
                    ptr(graph.c_row), ptr(graph.c_col), ptr(graph.c_mir), ptr(graph.util), float(at), float(bt),
                    *[ptr(t) for t in (Gs, Gr, Ls, Lr, L2s, L2r, L3s, L3r, T3r)]]


def c2pf_fit(graph, variant, at, bt, state, n_iter):
    """One call of c2pf_cpp / tc2pf_cpp / rc2pf_cpp (cpp_c2pf.cpp) with the kappa prior (at, bt): n_iter iterations over
    `graph` (C2pfGraph), updating the device state (see _c2pf_args) in place.  Two calls of a and b iterations with the
    same (at, bt) equal one call of a + b."""
    L = require_cuda()
    k, args = _c2pf_args(graph, variant, at, bt, state)
    if int(n_iter) < 0:
        raise B200Error("n_iter must be >= 0, got %d" % int(n_iter))
    check(L.b200_c2pf_fit(*args, int(n_iter), ptr(graph.workspace(k)), current_stream()), "b200_c2pf_fit")


def c2pf_update(graph, variant, at, bt, state, expectations, given=(None, None, None, None)):
    """One iteration from the expectations (Lt, Lb, L2b, L3b, Lb2) (f64 device tensors, None where the variant has none),
    which are replaced by those the iteration computes.  given = (Lt, Lb, L2b, L3b): tensors to take in place of the
    expectations the iteration would compute (None: compute)."""
    L = require_cuda()
    k, args = _c2pf_args(graph, variant, at, bt, state)
    r = graph.ratings
    absent = {"c2pf": None, "tc2pf": 2, "rc2pf": 1}[variant]             # L2b / Lb, which the variant has not
    sizes = (r.n_users * k, r.n_items * k, r.n_items * k, max(graph.n_edges, 1), r.n_items * k)
    exps = [None if j == absent else _dev(t, torch.float64, "expectation %d" % j, n)
            for j, (t, n) in enumerate(zip(expectations, sizes))]
    given = [None if t is None else _dev(t, torch.float64, "given expectation %d" % j, n)
             for j, (t, n) in enumerate(zip(given, sizes))]
    check(L.b200_c2pf_update(*args, *map(ptr, exps), *map(ptr, given), ptr(graph.workspace(k)), current_stream()),
          "b200_c2pf_update")


def rank_pack_items(V, item_base=None, n_items=None):
    """The item side of the fused rank packed once (b200_rank_pack_items): fp16 tile images of V[:n_items] with the item
    base folded in + the scaling scalars, as a uint8 CUDA tensor to pass to rank_topk(packed_items=...).  Valid as long as
    V / item_base do not change.  Returns None for shapes the tensor-core pass does not take."""
    L = require_cuda()
    k = _dev(V, torch.float32, "V", (None if n_items is None else _AtLeast(n_items), None)).shape[1]
    n_items = int(V.shape[0] if n_items is None else n_items)
    if item_base is not None:
        _dev(item_base, torch.float32, "item_base", _AtLeast(n_items))
    nbytes = int(L.b200_rank_items_bytes(n_items, k))
    if nbytes <= 0:
        return None
    packed = torch.empty(nbytes, dtype=torch.uint8, device=V.device)
    check(L.b200_rank_pack_items(ptr(V), n_items, k, ptr(item_base), ptr(packed), nbytes, current_stream()),
          "b200_rank_pack_items")
    return packed


def rank_topk(U, V, topk, user_idx=None, item_base=None, user_off=None, excl_indptr=None, excl_indices=None,
              n_items=None, workspace=None, packed_items=None):
    """Fused score + exclusion + top-k on device tensors (b200_rank_topk).  Returns (ids int32 [n_q, topk],
    scores f32 [n_q, topk]) CUDA tensors ordered by (score desc, item id asc); ids are -1 padded.
    packed_items: result of rank_pack_items(V, item_base, n_items) for the SAME V / item_base / n_items (skips the two
    passes over V that every call otherwise makes).  workspace: optional uint8 device scratch of at least
    b200_rank_topk_workspace_bytes(n_q, n_items, k, topk) bytes (allocated per call otherwise)."""
    L = require_cuda()
    n_items, k, n_q = _score_args(U, V, user_idx, n_items, torch.float32, item_base, user_off)
    _exclusions(excl_indptr, excl_indices, n_q)
    if packed_items is not None:                                   # built by rank_pack_items for this n_items and k
        _dev(packed_items, torch.uint8, "packed_items", int(L.b200_rank_items_bytes(n_items, k)))
    nbytes = int(L.b200_rank_topk_workspace_bytes(n_q, n_items, k, int(topk)))
    workspace = _buf(workspace, torch.uint8, "workspace", _AtLeast(max(nbytes, 16)))
    ids = torch.empty((n_q, topk), dtype=torch.int32, device=U.device)
    sc = torch.empty((n_q, topk), dtype=torch.float32, device=U.device)
    check(L.b200_rank_topk_packed(ptr(U), ptr(user_idx), n_q, ptr(V), n_items, k, ptr(item_base), ptr(user_off),
                                  ptr(excl_indptr), ptr(excl_indices), int(topk), ptr(ids), ptr(sc), ptr(packed_items),
                                  ptr(workspace), workspace.numel(), current_stream()), "b200_rank_topk")
    return ids, sc


def rank_topk_host(U, V, topk, user_idx, item_base=None, excl_indptr=None, excl_indices=None, out_ids=None,
                   out_scores=None, workspace=None, packed_items=None):
    """Host-buffer entry of the rank path (what the plug-ins' rank_batch calls): the factor matrices are
    device resident (model state), the REQUEST -- user indices and the per-user sorted exclusion lists in CSR
    form, numpy / pinned -- is copied in, ids + scores are copied back into numpy arrays."""
    uidx = to_device(np.asarray(user_idx, dtype=np.int64), torch.int64)
    ep = ei = None
    if excl_indptr is not None:
        ep = to_device(np.asarray(excl_indptr, dtype=np.int64), torch.int64)
        ei = to_device(np.asarray(excl_indices, dtype=np.int32), torch.int32) if len(excl_indices) else \
            torch.zeros(1, dtype=torch.int32, device="cuda")
    ids, sc = rank_topk(U, V, topk, user_idx=uidx, item_base=item_base, excl_indptr=ep, excl_indices=ei,
                        workspace=workspace, packed_items=packed_items)
    n_q = len(user_idx)
    out_ids = np.empty((n_q, topk), dtype=np.int32) if out_ids is None else out_ids
    out_scores = np.empty((n_q, topk), dtype=np.float32) if out_scores is None else out_scores
    torch.from_numpy(out_ids).copy_(ids)
    torch.from_numpy(out_scores).copy_(sc)
    return out_ids, out_scores


def topk_metrics(ids, pos_indptr, pos_indices, kinds, ks, user_idx=None, topk=None):
    """Per-user values of the @k ranking metrics for device ranked lists (b200_topk_metrics).
    ids int32 [n_q, >=topk] CUDA; pos_* the test-positives CSR (int64 / int32 CUDA); kinds / ks python lists.
    Returns a float64 CUDA tensor [n_metrics, n_q]."""
    L = require_cuda()
    n_q, stride = _dev(ids, torch.int32, "ids", (None, None if topk is None else _AtLeast(topk))).shape
    topk = stride if topk is None else int(topk)
    _dev(pos_indptr, torch.int64, "pos_indptr"), _dev(pos_indices, torch.int32, "pos_indices")
    if user_idx is not None:
        _dev(user_idx, torch.int64, "user_idx", _AtLeast(n_q))
    mk = torch.tensor(list(kinds), dtype=torch.int32).to(ids.device)
    kk = torch.tensor(list(ks), dtype=torch.int32).to(ids.device)
    out = torch.empty((len(kinds), n_q), dtype=torch.float64, device=ids.device)
    check(L.b200_topk_metrics(ptr(ids), n_q, topk, stride, ptr(user_idx), ptr(pos_indptr), ptr(pos_indices), ptr(mk),
                              ptr(kk), len(kinds), ptr(out), current_stream()), "b200_topk_metrics")
    return out


def rank_counts(scores, pos_indptr, pos_indices, user_idx=None, excl_indptr=None, excl_indices=None, less=None, pos_score=None):
    """The counts behind AUC / MAP / MRR for a batch of score rows (b200_rank_counts).  `scores` f32 [n_q, n_items] CUDA is
    MODIFIED (excluded entries become NaN).  pos_* = CSR of the test positives (int64 / int32 CUDA), row user_idx[q] for
    score row q.  Returns (less int64 [len(pos_indices)], pos_score f32 [len(pos_indices)], n_cand int64 [n_q],
    before_first int64 [n_q]); `less` / `pos_score` are filled only at the positions of the listed users' positives."""
    L = require_cuda()
    n_q, n_items = _dev(scores, torch.float32, "scores", (None, None)).shape
    _dev(pos_indptr, torch.int64, "pos_indptr")
    n_pos = _dev(pos_indices, torch.int32, "pos_indices").numel()
    if user_idx is not None:
        _dev(user_idx, torch.int64, "user_idx", _AtLeast(n_q))
    _exclusions(excl_indptr, excl_indices, n_q)
    less = _buf(less, torch.int64, "less", _AtLeast(n_pos), zero=True)
    pos_score = _buf(pos_score, torch.float32, "pos_score", _AtLeast(n_pos), zero=True)
    n_cand = torch.zeros(max(n_q, 1), dtype=torch.int64, device=scores.device)
    before = torch.zeros(max(n_q, 1), dtype=torch.int64, device=scores.device)
    check(L.b200_rank_counts(ptr(scores), n_q, n_items, ptr(excl_indptr), ptr(excl_indices), ptr(user_idx), ptr(pos_indptr),
                             ptr(pos_indices), ptr(less), ptr(pos_score), ptr(n_cand), ptr(before), current_stream()),
          "b200_rank_counts")
    return less, pos_score, n_cand[:n_q], before[:n_q]


def _delta_args(x, snapshot, delta):
    """The element count of a replica exchange step, checked: x, snapshot and delta f32 [>= n], n = x.numel()."""
    n = _dev(x, torch.float32, "x").numel()
    _dev(snapshot, torch.float32, "snapshot", _AtLeast(n)), _dev(delta, torch.float32, "delta", _AtLeast(n))
    return n


def delta_make(x, snapshot, delta):
    L = require_cuda()
    n = _delta_args(x, snapshot, delta)
    check(L.b200_delta_make(ptr(x), ptr(snapshot), ptr(delta), n, current_stream()), "b200_delta_make")


def delta_apply(x, snapshot, delta):
    L = require_cuda()
    n = _delta_args(x, snapshot, delta)
    check(L.b200_delta_apply(ptr(x), ptr(snapshot), ptr(delta), n, current_stream()), "b200_delta_apply")


def device_info():
    import ctypes
    L = require_cuda()
    a, b, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    check(L.b200_device_info(ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)), "b200_device_info")
    return dict(sm_count=a.value, cc=(b.value, c.value))
