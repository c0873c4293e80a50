"""Host restatement of the sample stream of the VEBPR / SBPR Hogwild epoch (csrc/bprx.cu, tri_hogwild_kernel).

TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/cornac_oracle.c header).

Sample s of epoch e under key `seed` is Philox4x32-10 of the counter (s_lo, s_hi, e_lo, 0x7813 + kind) under the key
(seed_lo, seed_hi), kind 0 = VEBPR, 1 = SBPR; its words (x, y, z, w) decode as
    i_index = floor((y:x) * nnz / 2^64),  j = mulhi32(z, n_items),  d3 = mulhi32(w, n_items),
    VEBPR: third item view[a_lo + d3 % n_views], none for a user without views; skipped when j is a purchase or a view
           of the user (views are only looked up when the user has some);
    SBPR:  position a_lo + floor(fl(fl(fl(d3) * fl(1 / n_items)) * n_social)) (float32, as the compiled reference,
           b200_sbpr_draw_host); the id at the position is read even when the user has no social item (then it belongs
           to a later user; past the end of the array there is none) and the sample is skipped when j is a purchase of
           the user or equals that id; the third item is that id for a user with social items, none past the end.
Everything here is exact integer / float32 arithmetic in numpy, vectorised over the samples.
"""
import numpy as np

KIND = {"vebpr": 0, "sbpr": 1}
_M32 = np.uint64(0xFFFFFFFF)


def _mulhi_lo(a, m):
    p = np.uint64(m) * a
    return p >> np.uint64(32), p & _M32


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) over uint64 arrays holding 32-bit words; returns (x, y, z, w)."""
    c = [np.asarray(v, np.uint64) & _M32 for v in (c0, c1, c2, c3)]
    c = list(np.broadcast_arrays(*c))
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    for _ in range(10):
        hi0, lo0 = _mulhi_lo(c[0], 0xD2511F53)
        hi1, lo1 = _mulhi_lo(c[2], 0xCD9E8D57)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return tuple(c)


def range64(lo, hi, n):
    """floor((hi:lo) * n / 2^64) exactly, for n < 2^32: (hi * n + ((lo * n) >> 32)) >> 32 never overflows 64 bits."""
    assert 1 <= int(n) < (1 << 32)
    n = np.uint64(n)
    return ((hi * n + ((lo * n) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)


def raw_words(kind, seed, epoch, n, sample_base=0):
    """The Philox words (x, y, z, w) of samples sample_base .. sample_base + n - 1 of the tri stream."""
    s = np.uint64(sample_base) + np.arange(n, dtype=np.uint64)
    seed = int(seed) & ((1 << 64) - 1)
    return philox4x32_10(s & _M32, s >> np.uint64(32), int(epoch) & 0xFFFFFFFF, 0x7813 + KIND[kind],
                         seed & 0xFFFFFFFF, seed >> 32)


def _member(indptr, indices, n_cols, u, col):
    """col in the sorted CSR row u (vectorised)."""
    keys = np.repeat(np.arange(len(indptr) - 1, dtype=np.int64), np.diff(indptr).astype(np.int64)) * n_cols + indices
    q = u.astype(np.int64) * n_cols + col
    pos = np.searchsorted(keys, q)
    return (pos < len(keys)) & (keys[np.minimum(pos, len(keys) - 1)] == q)


def tri_stream(kind, seed, epoch, n, indptr, indices, n_items, aux, sample_base=0):
    """Decode n samples of the tri stream exactly as tri_hogwild_kernel does.

    aux = (view_indptr, view_indices) for "vebpr", (social_indptr, social_item_ids, social_item_counts) for "sbpr".
    Returns a dict of arrays over the samples: i_index (int64), u, i, j, t (third item, -1 = none), t_count (SBPR),
    k_index (SBPR: the sampled position), skip (bool); v_id = t for VEBPR is what O.vebpr_replay takes."""
    indptr, indices = np.asarray(indptr), np.asarray(indices)
    nnz = len(indices)
    x, y, z, w = raw_words(kind, seed, epoch, n, sample_base)
    ii = range64(x, y, nnz)
    j = ((z * np.uint64(n_items)) >> np.uint64(32)).astype(np.int64)
    d3 = ((w * np.uint64(n_items)) >> np.uint64(32)).astype(np.int64)
    coo = np.repeat(np.arange(len(indptr) - 1, dtype=np.int64), np.diff(indptr).astype(np.int64))
    u = coo[ii]
    a_ptr = np.asarray(aux[0]).astype(np.int64)
    a_items = np.asarray(aux[1])
    a_lo, n_aux_u = a_ptr[u], a_ptr[u + 1] - a_ptr[u]
    skip = _member(indptr, indices, n_items, u, j)
    out = dict(i_index=ii, u=u, i=indices[ii].astype(np.int64), j=j)
    if kind == "vebpr":
        has = n_aux_u > 0
        pos = a_lo + d3 % np.maximum(n_aux_u, 1)
        t = np.where(has, a_items[np.minimum(pos, max(len(a_items) - 1, 0))] if len(a_items) else -1, -1).astype(np.int64)
        skip |= has & _member(a_ptr, a_items, n_items, u, j)
        out.update(t=t, t_count=np.zeros(n, np.int64), v_id=t.astype(np.int32))
    else:
        n_aux = len(a_items)
        inv = np.float32(1.0) / np.float32(n_items)
        kr = (d3.astype(np.float32) * inv) * n_aux_u.astype(np.float32)
        kidx = a_lo + np.floor(kr).astype(np.int64)
        inside = kidx < n_aux
        kid = np.where(inside, a_items[np.minimum(kidx, max(n_aux - 1, 0))] if n_aux else -1, -1).astype(np.int64)
        skip |= j == kid
        has = (n_aux_u > 0) & inside
        cnt = np.asarray(aux[2]).astype(np.int64)
        out.update(t=np.where(has, kid, -1), t_count=np.where(has, cnt[np.minimum(kidx, max(n_aux - 1, 0))] if n_aux else 0, 0),
                   k_index=kidx)
    out["skip"] = skip
    return out
