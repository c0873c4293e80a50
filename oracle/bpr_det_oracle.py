"""ctypes front-end of oracle/bpr_det_oracle.c: a serial restatement of the deterministic BPR epoch
(engine.bpr_epoch(..., deterministic=True); bpr_det_grad_kernel + bpr_det_apply_kernel in cornac_b200/csrc/bpr.cu).

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  The sample stream comes from b200_bpr_draw_host2 (the host twin of the device
draw, no GPU needed); the round size and the per-delta bound are restated here from b200_bpr_epoch, so that tests pin
both rules.  Hinge (MMMF) and exact-exp epochs are bit-identical to the device; the fast __expf path is run with the
exact z and can only be compared with a tolerance.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "bpr_det_oracle.c")
_LIB_PATH = os.path.join(_HERE, "libbpr_det_oracle.so")
_CMD = ["/usr/bin/gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-Wall",
        "-Wextra", "-std=c11", "-o", _LIB_PATH, _SRC, "-lm"]

_p, _i64, _f32, _c_int = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int

DET_ROUND = 16384           # rounds hold at most this many samples (bpr.cu DET_ROUND)
INT64_MAX = 2 ** 63 - 1


def build(force=False):
    """Compile oracle/bpr_det_oracle.c (gcc, a second)."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
        subprocess.check_call(_CMD)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        L.bpr_det_epoch.argtypes = ([_p, _p, _i64, _i64, _p, _p, _p, _i64, _i64, _p, _p, _p, _c_int, _f32, _f32, _c_int,
                                     _c_int, _f32, _p, _p])
        L.bpr_det_epoch.restype = _c_int
        L.bpr_det_sum_apply.argtypes = [_f32, _p, _i64, _f32]
        L.bpr_det_sum_apply.restype = _f32
        _lib = L
    return _lib


def block_plan(n_users, n_neg, k, blocked, neg_weighted):
    """(windows, item blocks) of the epoch's sample order, as b200_bpr_epoch picks them (B200_BPR_PART_MB is read by
    b200_bpr_block_plan)."""
    if not blocked:
        return 1, 1
    from cornac_b200 import engine
    wn, bn = engine.bpr_block_plan(n_users, n_neg, k)
    return wn, (1 if neg_weighted else bn)


def round_size(n_users, n_neg, k, blocked=False, neg_weighted=False, unbounded=False):
    """Samples per round R of the deterministic epoch: min(max_groups, 16384), where max_groups is the Hogwild staleness
    bound of b200_bpr_epoch -- a quarter of the rows of the smaller factor matrix (at least 16), of one window / item
    block when the order is blocked, and unlimited with `unbounded`."""
    rows = min(n_users, n_neg)
    max_groups = max(16, rows // 4)
    if unbounded:
        max_groups = INT64_MAX // 1024
    wn, bn = block_plan(n_users, n_neg, k, blocked, neg_weighted)
    if wn > 1 or bn > 1:
        cap = max(16, min(n_users // wn, n_neg // bn) // 4)
        if not unbounded and cap < max_groups:
            max_groups = cap
    return min(max_groups, DET_ROUND)


def delta_bound(R):
    """Largest |d| a delta may have in a round of R samples: 2^(22 - ceil(log2 R)).  An element takes at most R deltas
    per round (a live sample touches each row once), so |Q| <= R 2^(62 - ceil(log2 R)) <= 2^62 and the int64 sum cannot
    wrap.  At R = 16384 the bound is 256."""
    c = 0
    while (1 << c) < R:
        c += 1
    return float(2.0 ** (22 - c))


def draw(indptr, indices, n_neg, seed, epoch, n, sample_base=0, plan=(1, 1), neg_weighted=False):
    """(u, i, j) int32 of the n samples the device epoch (seed, epoch, sample_base) draws under `plan`.  A WBPR negative
    is the item of the interaction range64(r.z, r.w, nnz): b200_bpr_draw_host2 with n_neg = nnz and one item block
    returns exactly that index."""
    from cornac_b200 import engine
    indices = np.asarray(indices, dtype=np.int32)
    nnz = len(indices)
    coo = np.repeat(np.arange(len(indptr) - 1, dtype=np.int32), np.diff(np.asarray(indptr, dtype=np.int64)))
    if neg_weighted:
        ii, jx = engine.bpr_draw_host(seed, epoch, n, nnz, nnz, sample_base=sample_base, plan=(plan[0], 1))
        jj = indices[jx.astype(np.int64)]
    else:
        ii, jj = engine.bpr_draw_host(seed, epoch, n, nnz, n_neg, sample_base=sample_base, plan=plan)
    return coo[ii], indices[ii], np.ascontiguousarray(jj, dtype=np.int32)


def epoch(indptr, indices, U, V, B, su, si, sj, R, lr, reg, use_bias, hinge, d_max=None):
    """One deterministic epoch of the samples (su, si, sj) in rounds of R, applied to the f32 U, V, B in place.
    d_max: the per-delta bound (default delta_bound(R)).  Returns (correct, skipped, largest finite |d|)."""
    indptr = np.ascontiguousarray(indptr, dtype=np.int32)
    indices = np.ascontiguousarray(indices, dtype=np.int32)
    for x in (U, V, B):
        assert x.dtype == np.float32 and x.flags.c_contiguous and x.flags.writeable
    k = U.shape[1]
    assert V.shape[1] == k and len(B) == V.shape[0] and len(indptr) == U.shape[0] + 1
    su, si, sj = (np.ascontiguousarray(a, dtype=np.int32) for a in (su, si, sj))
    stats = np.zeros(2, dtype=np.int64)
    max_d = ctypes.c_double(0.0)
    rc = lib().bpr_det_epoch(indptr.ctypes.data, indices.ctypes.data, U.shape[0], V.shape[0], su.ctypes.data,
                             si.ctypes.data, sj.ctypes.data, len(su), int(R), U.ctypes.data, V.ctypes.data, B.ctypes.data,
                             int(k), float(lr), float(reg), int(bool(use_bias or hinge)), int(bool(hinge)),
                             float(delta_bound(R) if d_max is None else d_max), stats.ctypes.data, ctypes.byref(max_d))
    if rc != 0:
        raise MemoryError("bpr_det_oracle: out of memory")
    return int(stats[0]), int(stats[1]), max_d.value


def train(indptr, indices, n_neg, U, V, B, lr, reg, use_bias, seed, epochs, n_samples=None, sample_base=0,
          base_step=0, epoch0=0, hinge=False, neg_weighted=False, blocked=False, unbounded=False, d_max=None):
    """`epochs` deterministic epochs with the arguments engine.bpr_epoch takes: epoch e = epoch0 + t draws from
    sample_base + t * base_step.  Returns ([[correct, skipped] per epoch], largest finite |d|)."""
    n_users, k = U.shape
    nnz = len(indices)
    n = nnz if n_samples is None else int(n_samples)
    R = round_size(n_users, n_neg, k, blocked, neg_weighted, unbounded)
    plan = block_plan(n_users, n_neg, k, blocked, neg_weighted)
    stats, max_d = [], 0.0
    for t in range(epochs):
        su, si, sj = draw(indptr, indices, n_neg, seed, epoch0 + t, n, sample_base + t * base_step, plan, neg_weighted)
        c, s, m = epoch(indptr, indices, U, V, B, su, si, sj, R, lr, reg, use_bias, hinge, d_max)
        stats.append([c, s])
        max_d = max(max_d, m)
    return stats, max_d


def sum_apply(x, deltas, d_max):
    """The rule for one element and one round: add.rn.ftz(x, (float)(Q 2^-40)), Q = wrapping sum of llrint(d 2^40)."""
    d = np.ascontiguousarray(deltas, dtype=np.float32)
    return float(np.float32(lib().bpr_det_sum_apply(float(x), d.ctypes.data, len(d), float(d_max))))
