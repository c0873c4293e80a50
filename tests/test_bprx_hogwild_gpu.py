"""The VEBPR / SBPR Hogwild epoch (csrc/bprx.cu, tri_hogwild_kernel) against the serial oracle on the same Philox stream,
restated on the host by oracle/tri_stream.py.  Over a stretch of the stream whose samples share no row Hogwild has no
races, so the kernel must equal the oracle's serial replay there -- element by element on the change of every touched row,
within a bound derived from __expf's error and the reassociated dot products, at every (G, NPL, VEC) row layout and in
every update branch.  Over 2 M samples at lr = 0 the counts must equal the restatement's.  GPU only."""
import functools

import numpy as np
import pytest
import torch

from conftest import needs_cornac, rel_err, synth_csr
from oracle import oracle as O
from oracle import tri_stream as T

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24
# every (G, NPL) the dispatch picks: scalar rows (k % 4 != 0) G = 4, 8, 16, 32 then NPL = 2, 4; float4 rows likewise
SCALAR_K = [1, 3, 5, 9, 17, 31, 33, 63, 65, 126, 127]
VEC_K = [4, 20, 36, 64, 68, 128, 132, 256, 260, 384, 512]


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def _aux_lists(indptr, indices, n_items, frac, max_per, seed, empty_tail=0):
    """Per user a sorted list of items disjoint from the user's purchases (views / social items) and a count per entry; a fraction
    `1 - frac` of the users, and the last `empty_tail` users, have none."""
    rng = np.random.RandomState(seed)
    n_users = len(indptr) - 1
    per = np.where(rng.rand(n_users) < frac, rng.randint(1, max_per + 1, size=n_users), 0)
    if empty_tail:
        per[-empty_tail:] = 0
    u = np.repeat(np.arange(n_users, dtype=np.int64), per)
    key = np.unique(u * n_items + rng.randint(n_items, size=len(u)))
    own = np.repeat(np.arange(n_users, dtype=np.int64), np.diff(indptr)) * n_items + indices
    key = key[~np.isin(key, own)]
    ptr = np.zeros(n_users + 1, np.int64)
    np.add.at(ptr, key // n_items + 1, 1)
    return (np.cumsum(ptr).astype(np.int32), (key % n_items).astype(np.int32),
            rng.randint(1, 6, size=len(key)).astype(np.int32))


def _launch(kind, data, n_items, U, V, B, k, hy, seed, epoch, n):
    """b200_vebpr_epoch / b200_sbpr_epoch on device tensors; returns the stats (correct, skipped)."""
    from cornac_b200 import _lib
    from cornac_b200._lib import check, current_stream, ptr
    L = _lib.load()
    indptr, indices, aux = data
    nnz = len(indices)
    t = [_dev(indptr, torch.int32), _dev(indices, torch.int32), _dev(O.coo_rows(indptr), torch.int32)]
    t += [_dev(a, torch.int32) if len(a) else torch.zeros(1, dtype=torch.int32, device="cuda") for a in aux]
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    f32 = lambda x: float(np.float32(x))          # noqa: E731
    if kind == "vebpr":
        rc = L.b200_vebpr_epoch(ptr(t[0]), ptr(t[1]), ptr(t[2]), U.shape[0], n_items, nnz, ptr(t[3]), ptr(t[4]), ptr(U), ptr(V), k,
                                f32(hy["lr"]), f32(hy["reg"]), f32(hy["alpha"]), seed, epoch, n, ptr(stats), current_stream())
    else:
        rc = L.b200_sbpr_epoch(ptr(t[0]), ptr(t[1]), ptr(t[2]), U.shape[0], n_items, nnz, ptr(t[3]), ptr(t[4]), ptr(t[5]),
                               len(aux[1]), ptr(U), ptr(V), ptr(B), k, f32(hy["lr"]), f32(hy["lambda_u"]), f32(hy["lambda_v"]),
                               f32(hy["lambda_b"]), int(hy["use_bias"]), seed, epoch, n, ptr(stats), current_stream())
    check(rc, "b200_%s_epoch" % kind)
    return tuple(stats.cpu().tolist())


# ---------------------------------------------------------------------------------------------------------------------
# 1. Conflict-free stretches: Hogwild == the serial oracle
@functools.lru_cache(maxsize=None)
def _big_data(kind):
    """300 K items and 200 K users of 1-3 purchases: the first ~150 samples of most streams share no row."""
    rng = np.random.RandomState(21)
    n_users, n_items = 200_000, 300_000
    u = np.repeat(np.arange(n_users, dtype=np.int64), rng.randint(1, 4, size=n_users))
    key = np.unique(u * n_items + rng.randint(n_items, size=len(u)))
    indptr = np.zeros(n_users + 1, np.int64)
    np.add.at(indptr, key // n_items + 1, 1)
    indptr, indices = np.cumsum(indptr).astype(np.int32), (key % n_items).astype(np.int32)
    ptr, ids, cnt = _aux_lists(indptr, indices, n_items, 0.6, 3, seed=22)
    return (indptr, indices, (ptr, ids) if kind == "vebpr" else (ptr, ids, cnt)), n_items


@functools.lru_cache(maxsize=None)
def _conflict_free_stream(kind, want=128):
    """(seed, epoch, n, stream): the first n samples of the (seed, epoch) stream share no user or item row among the samples
    that are not skipped, and >= `want` of them are not skipped."""
    (indptr, indices, aux), n_items = _big_data(kind)
    for seed in range(1000, 1200):
        for epoch in (0, 5):
            s = T.tri_stream(kind, seed, epoch, 400, indptr, indices, n_items, aux)
            users, items, live = set(), set(), 0
            for q in range(400):
                if s["skip"][q]:
                    continue
                rows = [int(s["i"][q]), int(s["j"][q])] + ([int(s["t"][q])] if s["t"][q] >= 0 else [])
                if int(s["u"][q]) in users or items.intersection(rows):
                    break
                users.add(int(s["u"][q])), items.update(rows)
                live += 1
            if live >= want:
                return seed, epoch, q, {name: a[:q] for name, a in s.items()}
    raise AssertionError("no conflict-free stretch of %d samples" % want)


def _compact(kind, s, U0, V0, B0):
    """The stretch's non-skipped samples as a self-contained problem for the oracle: sample q owns user row q and item rows
    3q (i), 3q + 1 (j), 3q + 2 (third item, if any).  Purchases, views and social items are cut down to those rows, which
    keeps every membership test the samples make.  Returns (oracle inputs, row maps back into the full matrices)."""
    live = np.flatnonzero(~s["skip"])
    n = len(live)
    u, i, j, t, cnt = (s[f][live] for f in ("u", "i", "j", "t", "t_count"))
    has = t >= 0
    item_rows = np.stack([i, j, np.where(has, t, i)], 1).reshape(-1)       # row 3q + 2 of a sample without one: unused
    Uc = U0[torch.from_numpy(u).cuda()].cpu().numpy()
    Vc = V0[torch.from_numpy(item_rows).cuda()].cpu().numpy()
    Bc = B0[torch.from_numpy(item_rows).cuda()].cpu().numpy() if B0 is not None else None
    q = np.arange(n)
    indptr, indices = np.arange(n + 1, dtype=np.int32), (3 * q).astype(np.int32)
    a_ptr = np.concatenate([[0], np.cumsum(has)]).astype(np.int32)
    a_ids = (3 * q[has] + 2).astype(np.int32)
    st = dict(ii=q.astype(np.int64), j=(3 * q + 1).astype(np.int32), has=has, cnt=cnt[has].astype(np.int32),
              t=np.where(has, 3 * q + 2, -1).astype(np.int32), k_index=np.where(has, np.cumsum(has) - 1, -1).astype(np.int64),
              indptr=indptr, indices=indices, a_ptr=a_ptr, a_ids=a_ids)
    return st, (u, item_rows), (Uc, Vc, Bc)


def _oracle(kind, st, rows0, hy, counts_add=0):
    Uc, Vc, Bc = (None if a is None else a.copy() for a in rows0)
    if kind == "vebpr":
        c, sk = O.vebpr_replay(st["ii"], st["t"], st["j"], st["indptr"], st["indices"], st["a_ptr"], st["a_ids"], Uc, Vc,
                               hy["lr"], hy["reg"], hy["alpha"])
    else:
        c, sk = 0, O.sbpr_replay(st["ii"], st["j"], st["k_index"], st["indptr"], st["indices"], st["a_ids"], st["cnt"] + counts_add,
                                 st["a_ptr"], Uc, Vc, Bc, hy["lr"], hy["lambda_u"], hy["lambda_v"], hy["lambda_b"], hy["use_bias"])
    assert sk == 0
    return c, (Uc, Vc, Bc)


def _sig(x):
    return 1.0 / (1.0 + np.exp(x))


def _coef(x, s_abs, k, scale=1.0):
    """(d, bound on |d_device - d_oracle|) for d = scale * sigma(-x * scale), x a dot product of k terms plus a bias difference
    whose absolute terms sum to s_abs.
    * The device sums the terms by fmaf and a group shuffle tree, the oracle serially: each is within gamma = (k + 1) eps / (1 - (k + 1) eps)
      of s_abs of the exact sum (eps = 2^-24), so the two x differ by at most 2 gamma s_abs (+ 2 eps |x| for the product
      with s_uk, whose float value each side may round once differently).  sigma's slope is d (1 - d).
    * The device's sigma is __frcp_rn(1 + __expf(x)); __expf is within 2 + floor(1.173 |x|) ulp of e^x (CUDA C Programming
      Guide, intrinsic functions), i.e. (2 + 1.173 |x|) 2^-23 relative; 1 + e, the reciprocal and the oracle's own rounding
      add 3 eps.  1 / (1 + E) moves by at most the relative change of E, so d is within (4 + 1.173 |x|) 2^-23 of itself."""
    g = (k + 1) * EPS / (1 - (k + 1) * EPS)
    xs = x * scale
    d = _sig(xs)
    dx = scale * 2 * g * s_abs + 2 * EPS * np.abs(xs)
    return scale * d, scale * (d * (4 + 1.173 * np.abs(xs)) * 2.0 ** -23 + d * (1 - d) * dx)


def _bound(kind, st, rows0, hy, k):
    """Per element of the compact rows: the largest |(x_dev - x0) - (x_ora - x0)| the two roundings allow, before the final
    store (added by _check).  Each update is x += lr (sum_m c_m w_m - reg x) with coefficients c_m from the sigmoids above:
      lr sum_m err(c_m) |w_m|                                 the coefficients' difference, and
      2^-19 lr (sum_m |c_m| |w_m| + reg |x|)                  at most 16 roundings on each side (products, sums, lr *), each
                                                              within eps of the sum of the magnitudes of the terms."""
    U0, V0, B0 = (None if a is None else a.astype(np.float64) for a in rows0)
    n = len(st["ii"])
    q = np.arange(n)
    u, vi, vj, vt = U0, V0[3 * q], V0[3 * q + 1], V0[3 * q + 2]
    has = st["has"][:, None]
    lr = float(np.float32(hy["lr"]))
    tol = [np.zeros_like(U0), np.zeros_like(V0), None if B0 is None else np.zeros_like(B0)]
    borderline = np.zeros(n, bool)

    def add(which, rows, terms, reg, x0):
        e = sum(ec * np.abs(w) for _, ec, w in terms)
        m = sum(np.abs(c) * np.abs(w) for c, _, w in terms)
        tol[which][rows] += (lr * e + 2.0 ** -19 * lr * (m + reg * np.abs(x0))).reshape(tol[which][rows].shape)

    def dot(a, b):
        return np.sum(a * b, 1, keepdims=True), np.sum(np.abs(a * b), 1, keepdims=True)

    if kind == "vebpr":
        reg, al = float(np.float32(hy["reg"])), float(np.float32(hy["alpha"]))
        out = []
        for a, b in ((vi, vj), (vi, vt), (vt, vj)):
            x, s_abs = dot(u, a - b)
            d, e = _coef(np.clip(x, -50, 50), s_abs, k)
            out.append((d, e))
            borderline |= (np.abs(x) <= 2 * (k + 1) * EPS / (1 - (k + 1) * EPS) * s_abs + 2.0 ** -19)[:, 0] & (has[:, 0] | (a is vi and b is vj))
        (dij, eij), (div, eiv), (dvj, evj) = out
        z = np.zeros_like(dij)
        a_, ea = np.where(has, al * div, z), np.where(has, al * eiv, z)
        b_, eb = np.where(has, (1 - al) * dvj, z), np.where(has, (1 - al) * evj, z)
        add(0, q, [(dij, eij, vi - vj), (a_, ea, vi - vt), (b_, eb, vt - vj)], reg, u)
        add(1, 3 * q, [(dij, eij, u), (a_, ea, u)], reg, vi)
        add(1, 3 * q + 1, [(dij, eij, u), (b_, eb, u)], reg, vj)
        add(1, 3 * q + 2, [(a_, ea, u), (b_, eb, u)], reg, vt)
        return tol, borderline
    ru, rv, rb = (float(np.float32(hy[x])) for x in ("lambda_u", "lambda_v", "lambda_b"))
    bi, bj, bt = B0[3 * q, None], B0[3 * q + 1, None], B0[3 * q + 2, None]
    cnt = np.zeros(n)
    cnt[st["has"]] = st["cnt"]
    s_uk = (1.0 / (1.0 + cnt))[:, None]
    x, s_abs = dot(u, vi - vj)
    zb, eb_ = _coef(bi - bj + x, np.abs(bi - bj) + s_abs, k)                       # BPR fall-back
    x, s_abs = dot(u, vi - vt)
    zik, eik = _coef(bi - bt + x, np.abs(bi - bt) + s_abs, k, scale=s_uk)          # SBPR-2: z_ik s_uk and z_kj
    x, s_abs = dot(u, vt - vj)
    zkj, ekj = _coef(bt - bj + x, np.abs(bt - bj) + s_abs, k)
    z = np.zeros_like(zb)
    fb = lambda a: np.where(has, z, a)            # noqa: E731
    s2 = lambda a: np.where(has, a, z)            # noqa: E731
    one = np.ones_like(zb)
    add(0, q, [(fb(zb), fb(eb_), vi - vj), (s2(zik), s2(eik), vi - vt), (s2(zkj), s2(ekj), vt - vj)], ru, u)
    add(1, 3 * q, [(fb(zb), fb(eb_), u), (s2(zik), s2(eik), u)], rv, vi)
    add(1, 3 * q + 1, [(fb(zb), fb(eb_), u), (s2(zkj), s2(ekj), u)], rv, vj)
    add(1, 3 * q + 2, [(s2(zik), s2(eik), u), (s2(zkj), s2(ekj), u)], rv, vt)
    bias2 = 1.0 if hy["use_bias"] else 0.0                                      # the fall-back trains biases regardless
    add(2, 3 * q, [(fb(zb) + bias2 * s2(zik), fb(eb_) + bias2 * s2(eik), one)], rb, bi)
    add(2, 3 * q + 1, [(fb(zb) + bias2 * s2(zkj), fb(eb_) + bias2 * s2(ekj), one)], rb, bj)
    add(2, 3 * q + 2, [(bias2 * s2(zik) + bias2 * s2(zkj), bias2 * (s2(eik) + s2(ekj)), one)], rb, bt)
    return tol, borderline


def _violations(got, want, base, tol):
    """Elements whose change differs from the oracle's by more than tol plus the two final stores' roundings."""
    got, want, base = (np.asarray(a, np.float64) for a in (got, want, base))
    lim = tol + 2.0 ** -22 * np.maximum(np.abs(base), np.abs(want))
    return int(np.sum(np.abs((got - base) - (want - base)) > lim))


def _check(dev_rows, orc_rows, rows0, tol, used):
    return sum(_violations(g[m], w[m], b[m], t[m]) for g, w, b, t, m in zip(dev_rows, orc_rows, rows0, tol, used) if g is not None)


@pytest.mark.parametrize("k", SCALAR_K + VEC_K)
@pytest.mark.parametrize("variant", ["vebpr", "sbpr_bias", "sbpr_nobias"])
def test_hogwild_equals_serial_oracle_on_a_conflict_free_stretch(variant, k):
    """The first samples of the stream share no row: tri_hogwild_kernel must change every touched element as the oracle's
    serial replay of the restated stream does, within _bound; untouched rows come back bit-identical and the skipped count
    is the restatement's.  Users with and without views / social items (both branches of each model), alpha = 0.3,
    lambda_u != lambda_v != lambda_b, one VEBPR score past the +-50 clip.  The same check rejects the oracle run with a
    swapped alpha, no regularisation, a learning rate off by 2^-10, and for SBPR lambda_u <-> lambda_v, lambda_b = 0,
    use_bias flipped and social_item_counts + 1."""
    kind = "vebpr" if variant == "vebpr" else "sbpr"
    data, n_items = _big_data(kind)
    seed, epoch, n, s = _conflict_free_stream(kind)
    if kind == "vebpr":
        hy = dict(lr=0.05, reg=0.01, alpha=0.3)
    else:
        hy = dict(lr=0.05, lambda_u=0.01, lambda_v=0.02, lambda_b=0.03, use_bias=variant == "sbpr_bias")
    g = torch.Generator(device="cuda")
    g.manual_seed(1000 + k)
    n_users = len(data[0]) - 1
    U0 = torch.rand((n_users, k), generator=g, device="cuda") - 0.5
    V0 = torch.rand((n_items, k), generator=g, device="cuda") - 0.5
    B0 = (torch.rand(n_items, generator=g, device="cuda") - 0.5) if kind == "sbpr" else None
    live = np.flatnonzero(~s["skip"])
    has = s["t"][live] >= 0
    assert has.any() and (~has).any() and len(live) >= 128
    if kind == "vebpr":                                      # a score of 100: clipped to 50
        q = live[np.flatnonzero(has)[0]]
        w = V0[int(s["i"][q])] - V0[int(s["j"][q])]
        U0[int(s["u"][q])] = w * (100.0 / float(torch.dot(w, w)))
    st, (u_rows, v_rows), rows0 = _compact(kind, s, U0, V0, B0)
    U, V = U0.clone(), V0.clone()
    B = B0.clone() if B0 is not None else None
    stats = _launch(kind, data, n_items, U, V, B, k, hy, seed, epoch, n)
    c_ora, orc = _oracle(kind, st, rows0, hy)
    tol, borderline = _bound(kind, st, rows0, hy, k)
    if kind == "vebpr":
        qh = int(np.flatnonzero(st["has"])[0])
        assert float(rows0[0][qh].astype(np.float64) @ (rows0[1][3 * qh] - rows0[1][3 * qh + 1])) > 50
    assert stats[1] == int(s["skip"].sum())
    assert abs(stats[0] - c_ora) <= int(borderline.sum()) if kind == "vebpr" else stats[0] == 0
    ui, vi = torch.from_numpy(u_rows).cuda(), torch.from_numpy(v_rows).cuda()
    dev = (U[ui].cpu().numpy(), V[vi].cpu().numpy(), B[vi].cpu().numpy() if B is not None else None)
    used = [np.ones(len(u_rows), bool), np.ones(len(v_rows), bool), np.ones(len(v_rows), bool)]
    used[1][2::3] = used[2][2::3] = st["has"]                # row 3q + 2 of a sample without a third item is row i again
    assert _check(dev, orc, rows0, tol, used) == 0
    # untouched rows: bit-identical
    for X, X0, r in ((U, U0, ui), (V, V0, vi), (B, B0, vi)):
        if X is None:
            continue
        keep = torch.ones(X.shape[0], dtype=torch.bool, device="cuda")
        keep[r] = False
        assert torch.equal(X[keep], X0[keep])
    # the check has teeth: each perturbed oracle is rejected
    bad = [dict(hy, lr=float(np.float32(hy["lr"])) * (1 + 2.0 ** -10))]
    if kind == "vebpr":
        bad += [dict(hy, alpha=1 - hy["alpha"]), dict(hy, reg=0.0)]
    else:
        bad += [dict(hy, lambda_u=0.0, lambda_v=0.0, lambda_b=0.0), dict(hy, lambda_u=hy["lambda_v"], lambda_v=hy["lambda_u"]),
                dict(hy, lambda_b=0.0), dict(hy, use_bias=not hy["use_bias"])]
    for h in bad:
        assert _check(dev, _oracle(kind, st, rows0, h)[1], rows0, tol, used) > 0, h
    if kind == "sbpr":
        assert _check(dev, _oracle(kind, st, rows0, hy, counts_add=1)[1], rows0, tol, used) > 0


@pytest.mark.parametrize("k", [130, 516, 1024])
def test_unsupported_width_is_an_error_not_a_launch(k):
    from cornac_b200._lib import B200Error
    data, n_items = _big_data("vebpr")
    U = torch.zeros((len(data[0]) - 1, k), device="cuda")
    V = torch.zeros((n_items, k), device="cuda")
    with pytest.raises(B200Error, match="not supported"):
        _launch("vebpr", data, n_items, U, V, None, k, dict(lr=0.05, reg=0.01, alpha=0.3), 1, 0, 10)
    data, n_items = _big_data("sbpr")
    with pytest.raises(B200Error, match="not supported"):
        _launch("sbpr", data, n_items, U, V, torch.zeros(n_items, device="cuda"), k,
                dict(lr=0.05, lambda_u=0.01, lambda_v=0.02, lambda_b=0.03, use_bias=True), 1, 0, 10)


# ---------------------------------------------------------------------------------------------------------------------
# 2. Long streams at lr = 0: nothing moves and the counts are the restatement's
def _vebpr_count_bound(s, U, V, k):
    """(correct count of the oracle's serial replay at lr = 0, number of samples whose correctness the two roundings of a
    margin may flip: |x| within the _coef bound of 0 for one of the margins that decide it)."""
    live = np.flatnonzero(~s["skip"])
    correct, border = 0, 0
    for c in range(0, len(live), 1 << 17):
        q = live[c:c + (1 << 17)]
        u, vi, vj = (X[s[f][q]].astype(np.float64) for X, f in ((U, "u"), (V, "i"), (V, "j")))
        has = s["t"][q] >= 0
        vt = V[np.where(has, s["t"][q], s["j"][q])].astype(np.float64)
        ok, near = np.ones(len(q), bool), np.zeros(len(q), bool)
        for a, b, gate in ((vi, vj, np.ones_like(has)), (vi, vt, has), (vt, vj, has)):
            p = u * (a - b)
            x, s_abs = p.sum(1), np.abs(p).sum(1)
            ok &= ~gate | (x > 0)
            near |= gate & (np.abs(x) <= 2 * (k + 1) * EPS / (1 - (k + 1) * EPS) * s_abs + 2.0 ** -19)
        correct += int(ok.sum())
        border += int(near.sum())
    return correct, border


def _long_case(kind, small):
    if small:                                                # 50 items; the last 4000 of 20 000 users have no social item
        indptr, indices = synth_csr(20000, 50, 200000, seed=31)
        aux = _aux_lists(indptr, indices, 50, 0.5, 4, seed=32, empty_tail=4000)
        return indptr, indices, 50, aux
    indptr, indices = synth_csr(20000, 2000, 400000, seed=5)
    return indptr, indices, 2000, _aux_lists(indptr, indices, 2000, 0.7, 8, seed=6)


@pytest.mark.parametrize("kind,k,small", [("vebpr", 5, False), ("vebpr", 64, False), ("sbpr", 9, False), ("sbpr", 64, False),
                                          ("sbpr", 36, True)])
def test_hogwild_lr0_is_identity_and_counts_match_the_restated_stream(kind, k, small):
    """lr = 0 over 2 M samples: the factors come back bit-identical, the skipped count equals the restatement's exactly and
    VEBPR's correct count the oracle's up to samples whose margin lies within rounding of 0.  On 50 items with many users
    without social items the SBPR quirk (such a user's sampled entry is a later user's) decides thousands of skips."""
    indptr, indices, n_items, (ptr, ids, cnt) = _long_case(kind, small)
    aux = (ptr, ids) if kind == "vebpr" else (ptr, ids, cnt)
    rng = np.random.RandomState(k)
    U0 = rng.normal(0, 0.3, (len(indptr) - 1, k)).astype(np.float32)
    V0 = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    B0 = rng.normal(0, 0.3, n_items).astype(np.float32)
    U, V, B = _dev(U0, torch.float32), _dev(V0, torch.float32), _dev(B0, torch.float32)
    hy = dict(lr=0.0, reg=0.01, alpha=0.3) if kind == "vebpr" else dict(lr=0.0, lambda_u=0.01, lambda_v=0.02, lambda_b=0.03, use_bias=True)
    n, seed, epoch = 2_000_003, 0xDEADBEEF12345678, 9
    c, sk = _launch(kind, (indptr, indices, aux), n_items, U, V, B, k, hy, seed, epoch, n)
    assert np.array_equal(U.cpu().numpy(), U0) and np.array_equal(V.cpu().numpy(), V0) and np.array_equal(B.cpu().numpy(), B0)
    s = T.tri_stream(kind, seed, epoch, n, indptr, indices, n_items, aux)
    assert sk == int(s["skip"].sum())
    if kind == "vebpr":
        c_ref, border = _vebpr_count_bound(s, U0, V0, k)
        assert abs(c - c_ref) <= border, (c, c_ref, border)
        assert (s["t"] >= 0).any() and (s["t"] < 0).any()
    else:
        assert c == 0
        quirk = (s["k_index"] - ptr[s["u"]] == 0) & (ptr[s["u"] + 1] == ptr[s["u"]]) & (s["j"] == np.where(
            s["k_index"] < len(ids), ids[np.minimum(s["k_index"], len(ids) - 1)], -1)) & ~T._member(indptr, indices, n_items, s["u"], s["j"])
        if small:
            assert quirk.sum() > 2000 and (s["k_index"] == len(ids)).any()


# ---------------------------------------------------------------------------------------------------------------------
# 3. The plug-ins reach the kernel with their key and the epochs 0, 1, 2
def _dataset(indptr, indices, n_items):
    from collections import OrderedDict
    from cornac.data import Dataset
    n_users = len(indptr) - 1
    rows = np.repeat(np.arange(n_users), np.diff(indptr))
    uid_map = OrderedDict((str(u), u) for u in range(n_users))
    iid_map = OrderedDict((str(i), i) for i in range(n_items))
    return Dataset.build([(str(u), str(i), 1.0) for u, i in zip(rows, indices)], global_uid_map=uid_map, global_iid_map=iid_map)


@needs_cornac
@pytest.mark.parametrize("kind", ["vebpr", "sbpr"])
def test_plugin_hogwild_epochs_are_the_restated_streams(kind, monkeypatch):
    import scipy.sparse as sp
    from cornac_b200 import SBPR, VEBPR, engine
    indptr, indices = synth_csr(400, 300, 6000, seed=41)
    n_users, n_items = 400, 300
    ds = _dataset(indptr, indices, n_items)
    assert np.array_equal(ds.matrix.indptr, indptr) and np.array_equal(ds.matrix.indices, indices)
    calls = []
    real = engine.tri_train_host

    def record(*a, **kw):
        calls.append((a, kw))
        return real(*a, **kw)

    monkeypatch.setattr(engine, "tri_train_host", record)
    rng = np.random.RandomState(42)
    U0 = ((rng.rand(n_users, 20) - 0.5) / 20).astype(np.float32)
    V0 = ((rng.rand(n_items, 20) - 0.5) / 20).astype(np.float32)
    seed = 2024
    if kind == "vebpr":
        from cornac.data import PurchaseViewDataset
        vptr, vidx, _ = _aux_lists(indptr, indices, n_items, 0.7, 6, seed=43)
        ds = PurchaseViewDataset(ds, sp.csr_matrix((np.ones(len(vidx), np.float32), vidx, vptr), shape=(n_users, n_items)))
        m = VEBPR(k=20, max_iter=3, learning_rate=0.0, lambda_reg=0.01, alpha=0.3, seed=seed, mode="hogwild",
                  init_params=dict(U=U0.copy(), V=V0.copy())).fit(ds)
        r = np.random.RandomState(seed)                  # factors given: the three RNGVector seeds are the first draws
        s0, s1, s2 = (r.randint(2 ** 31) for _ in range(3))
        key = (int(s0) << 31) ^ (int(s1) << 15) ^ int(s2)
    else:
        from cornac.data import GraphModality
        edges = [(str(a), str((a * 7 + d) % n_users), 1.0) for a in range(n_users) for d in range(1, 1 + a % 4)]
        gm = GraphModality(data=edges)
        gm.build(id_map=ds.uid_map)
        ds.add_modalities(user_graph=gm)
        m = SBPR(k=20, max_iter=3, learning_rate=0.0, lambda_u=0.01, lambda_v=0.02, lambda_b=0.03, seed=seed, mode="hogwild",
                 init_params=dict(U=U0.copy(), V=V0.copy(), Bi=np.zeros(n_items, np.float32))).fit(ds)
        r = np.random.RandomState(seed)
        s_pos, s_neg = r.randint(2 ** 31), r.randint(2 ** 31)
        key = (int(s_pos) << 31) | int(s_neg)
    assert len(calls) == 1
    (_, c_indptr, c_indices, aux, c_items, *_), kw = calls[0]
    assert kw["key"] == key and kw.get("replay_seeds") is None
    assert c_items == n_items and np.array_equal(c_indptr, indptr) and np.array_equal(c_indices, indices)
    if kind == "sbpr":
        assert len(aux[1]) > 0 and (np.diff(aux[0]) == 0).any()
    assert len(m.epoch_stats) == 3
    for e in range(3):
        s = T.tri_stream(kind, key, e, len(indices), indptr, indices, n_items, aux)
        c, sk = m.epoch_stats[e]
        assert sk == int(s["skip"].sum())
        if kind == "vebpr":
            c_ref, border = _vebpr_count_bound(s, U0, V0, 20)
            assert abs(c - c_ref) <= border
        else:
            assert c == 0


# ---------------------------------------------------------------------------------------------------------------------
# 4. SBPR's position at the end of a user's list: the next user's entry and count, or past the array the BPR fall-back
@pytest.mark.parametrize("use_bias", [True, False])
def test_sbpr_replay_reads_position_at_the_end_of_the_list(use_bias):
    """k_index = a_hi (reachable in both modes once n_items >= 2^24 - 1): for a user followed by others with social items it
    is the next user's first entry and count, as the reference reads them -- possibly one of the user's own items, k == i,
    which the reference updates after i; for the last user, k_index = n_social, there is no entry and the sample is a BPR
    fall-back.  Kernel == oracle within the replay tolerance, skipped count exact."""
    from cornac_b200 import _lib
    from cornac_b200._lib import check, current_stream, ptr
    L = _lib.load()
    n_users, n_items, k = 200, 150, 16
    indptr, indices = synth_csr(n_users, n_items, 4000, seed=51)
    seed = 52
    s_ptr, s_ids, s_cnt = _aux_lists(indptr, indices, n_items, 0.7, 5, seed=seed)
    while s_ptr[-1] == s_ptr[-2]:                                    # the last user has social items
        seed += 1
        s_ptr, s_ids, s_cnt = _aux_lists(indptr, indices, n_items, 0.7, 5, seed=seed)
    coo = O.coo_rows(indptr)
    rng = np.random.RandomState(53)
    n = 3000
    ii = rng.randint(len(indices), size=n).astype(np.int64)
    u = coo[ii]
    ns = s_ptr[u + 1] - s_ptr[u]
    kidx = s_ptr[u].astype(np.int64) + np.floor(rng.rand(n) * ns).astype(np.int64)
    at_end = (rng.rand(n) < 0.3) & (ns > 0)
    kidx[at_end] = s_ptr[u + 1][at_end]                              # the position a_hi
    last = int(np.flatnonzero(coo == n_users - 1)[0])
    ii[:40], kidx[:40] = last, len(s_ids)                            # the last user, past the array
    # users whose next entry is one of their own items: a sample with that item as i has k == i
    alias = [(indptr[v] + int(np.searchsorted(indices[indptr[v]:indptr[v + 1]], s_ids[s_ptr[v + 1]])), s_ptr[v + 1])
             for v in range(n_users - 1) if s_ptr[v + 1] > s_ptr[v] and s_ids[s_ptr[v + 1]] in indices[indptr[v]:indptr[v + 1]]]
    assert len(alias) >= 5
    for r, (a_ii, a_k) in enumerate(alias):
        ii[40 + 7 * r], kidx[40 + 7 * r] = a_ii, a_k
    j = rng.randint(n_items, size=n).astype(np.int32)
    inside = (kidx == s_ptr[coo[ii] + 1]) & (kidx < len(s_ids))
    assert inside.sum() > 100
    U0 = (rng.rand(n_users, k) - 0.5).astype(np.float32)
    V0 = (rng.rand(n_items, k) - 0.5).astype(np.float32)
    B0 = (rng.rand(n_items) - 0.5).astype(np.float32)
    Uo, Vo, Bo = U0.copy(), V0.copy(), B0.copy()
    sk = O.sbpr_replay(ii, j, kidx, indptr, indices, s_ids, s_cnt, s_ptr, Uo, Vo, Bo, 0.05, 0.02, 0.03, 0.04, use_bias)
    dU, dV, dB = _dev(U0, torch.float32), _dev(V0, torch.float32), _dev(B0, torch.float32)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    t = [_dev(ii, torch.int64), _dev(j, torch.int32), _dev(kidx, torch.int64), _dev(indptr, torch.int32), _dev(indices, torch.int32),
         _dev(coo, torch.int32), _dev(s_ptr, torch.int32), _dev(s_ids, torch.int32), _dev(s_cnt, torch.int32)]
    check(L.b200_sbpr_epoch_replay(ptr(t[0]), ptr(t[1]), ptr(t[2]), n, ptr(t[3]), ptr(t[4]), ptr(t[5]), ptr(t[6]), ptr(t[7]), ptr(t[8]),
                                   len(s_ids), ptr(dU), ptr(dV), ptr(dB), k, 0.05, 0.02, 0.03, 0.04, int(use_bias), ptr(stats),
                                   current_stream()), "replay")
    assert int(stats[1].item()) == sk
    assert rel_err(dU.cpu().numpy(), Uo) < 1e-5 and rel_err(dV.cpu().numpy(), Vo) < 1e-5 and rel_err(dB.cpu().numpy(), Bo) < 1e-5
