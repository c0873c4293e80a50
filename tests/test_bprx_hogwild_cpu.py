"""The host restatement of the VEBPR / SBPR Hogwild sample stream (oracle/tri_stream.py) against the library's own Philox,
and the oracle's SBPR fall-back for a sampled position past the social-item array.  No GPU needed."""
import numpy as np
import pytest

from conftest import synth_csr
from oracle import tri_stream as T


def test_philox_restatement_matches_known_answers():
    """Random123's known-answer vectors for philox4x32-10 (counter, key) -> output."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        got = T.philox4x32_10(*[np.array([c], np.uint64) for c in ctr], *key)
        assert tuple(int(g[0]) for g in got) == want


@pytest.mark.parametrize("kind", ["vebpr", "sbpr"])
@pytest.mark.parametrize("seed,epoch,base,nnz", [
    (5, 0, 0, 1),
    (0x9E3779B97F4A7C15, 3, 0, 1_234_567),
    ((1 << 62) + 11, 0xFFFFFFFF, (1 << 32) - 70_000, 4_000_000_007),      # sample indices across 2^32; nnz > 2^31
    (77, 12, (5 << 40) + 3, (1 << 32) - 1),
])
def test_tri_stream_is_the_library_philox_stream(kind, seed, epoch, base, nnz):
    """b200_bpr_draw_host with epoch = e | (0x7813 + kind) << 32 runs Philox on the tri kernel's counter: its i_index is the tri
    stream's, and with n_neg = 2^32 its j is the raw fourth word w (the word behind the third item's draw)."""
    from cornac_b200 import engine
    n = 100_000
    ii, jj = engine.bpr_draw_host(seed, (epoch & 0xFFFFFFFF) | ((0x7813 + T.KIND[kind]) << 32), n, nnz, 1 << 32, sample_base=base)
    x, y, z, w = T.raw_words(kind, seed, epoch, n, sample_base=base)
    assert np.array_equal(T.range64(x, y, nnz), ii)
    assert np.array_equal(w.astype(np.uint32), jj.view(np.uint32))


def test_tri_stream_decode_on_a_small_catalogue():
    """The decode rules themselves: j and the third draw are mulhi32 of z and w; VEBPR's view is d3 % n_views (none for a user
    without views); SBPR's position is the float32 product and reads a later user's entry for a user without social items."""
    indptr, indices = synth_csr(300, 40, 3000, seed=2)
    rng = np.random.RandomState(3)
    rows = [np.setdiff1d(rng.randint(40, size=rng.randint(0, 4)), indices[indptr[u]:indptr[u + 1]]) for u in range(300)]
    vptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    vidx = np.concatenate(rows).astype(np.int32)          # sorted rows, disjoint from the purchases
    n = 5000
    x, y, z, w = T.raw_words("vebpr", 9, 1, n)
    s = T.tri_stream("vebpr", 9, 1, n, indptr, indices, 40, (vptr, vidx))
    d3 = (w * np.uint64(40)) >> np.uint64(32)
    assert np.array_equal(s["j"], (z * np.uint64(40)) >> np.uint64(32))
    for q in range(0, n, 37):
        u = s["u"][q]
        row, views = indices[indptr[u]:indptr[u + 1]], vidx[vptr[u]:vptr[u + 1]]
        assert s["i"][q] == indices[s["i_index"][q]] and indptr[u] <= s["i_index"][q] < indptr[u + 1]
        assert s["t"][q] == (views[int(d3[q]) % len(views)] if len(views) else -1)
        assert s["skip"][q] == (s["j"][q] in row or (len(views) > 0 and s["j"][q] in views))
    sptr, sids, scnt = vptr, vidx, rng.randint(1, 6, size=len(vidx)).astype(np.int32)
    x, y, z, w = T.raw_words("sbpr", 9, 1, n)
    s = T.tri_stream("sbpr", 9, 1, n, indptr, indices, 40, (sptr, sids, scnt))
    d3 = ((w * np.uint64(40)) >> np.uint64(32)).astype(np.float32)
    for q in range(0, n, 37):
        u = s["u"][q]
        ns = sptr[u + 1] - sptr[u]
        pos = sptr[u] + int(np.floor(np.float32(d3[q] * (np.float32(1) / np.float32(40))) * np.float32(ns)))
        kid = sids[pos] if pos < len(sids) else -1
        assert s["k_index"][q] == pos
        assert s["skip"][q] == (s["j"][q] in indices[indptr[u]:indptr[u + 1]] or s["j"][q] == kid)
        assert s["t"][q] == (kid if ns > 0 else -1) and s["t_count"][q] == (scnt[pos] if ns > 0 else 0)


def test_sbpr_float_position_reaches_the_end_of_the_list():
    """fl(d3 * fl(1 / n)) rounds to 1.0 for d3 = n - 1 once n >= 2^24 - 1: the sampled position is then a_hi, past the user's
    list -- for the last user with social items, past the whole array."""
    n = 16_777_215
    for n_social in (1, 3, 7):
        pos = np.floor((np.float32(n - 1) * (np.float32(1) / np.float32(n))) * np.float32(n_social))
        assert pos == n_social
    n = 1 << 20
    assert np.floor((np.float32(n - 1) * (np.float32(1) / np.float32(n))) * np.float32(7)) == 6


def _sbpr_case(seed=4):
    from oracle import oracle as O
    indptr, indices = synth_csr(30, 50, 300, seed=seed)
    rng = np.random.RandomState(seed)
    sptr, sids, scnt = [0], [], []
    for u in range(30):
        if u % 3 != 1:                                      # users 1, 4, ... have no social item; the last one (29) has
            it = np.setdiff1d(rng.choice(50, size=4, replace=False), indices[indptr[u]:indptr[u + 1]])
            sids.extend(it.tolist()), scnt.extend(rng.randint(1, 5, size=len(it)).tolist())
        sptr.append(len(sids))
    k = 6
    U0 = (rng.rand(30, k) - 0.5).astype(np.float32)
    V0 = (rng.rand(50, k) - 0.5).astype(np.float32)
    B0 = (rng.rand(50) - 0.5).astype(np.float32)
    coo = O.coo_rows(indptr)
    return indptr, indices, coo, (np.asarray(sptr, np.int32), np.asarray(sids, np.int32), np.asarray(scnt, np.int32)), U0, V0, B0


def _unpurchased(indptr, indices, u, avoid=()):
    return next(j for j in range(50) if j not in indices[indptr[u]:indptr[u + 1]] and j not in avoid)


@pytest.mark.parametrize("use_bias", [False, True])
def test_oracle_sbpr_past_the_array_is_the_bpr_fall_back(use_bias):
    """A user with social items whose position is past the whole social array (k_index = n_social) has no third item: the
    oracle applies the BPR branch, bit for bit what it applies to the same sample of a user without social items."""
    from oracle import oracle as O
    indptr, indices, coo, (sptr, sids, scnt), U0, V0, B0 = _sbpr_case()
    u = 29
    assert sptr[u + 1] > sptr[u] and sptr[u + 1] == len(sids)
    ii = np.array([indptr[u]], np.int64)
    j = np.array([_unpurchased(indptr, indices, u)], np.int32)
    hy = (0.05, 0.02, 0.03, 0.04, use_bias)
    U1, V1, B1 = U0.copy(), V0.copy(), B0.copy()
    sk = O.sbpr_replay(ii, j, np.array([len(sids)], np.int64), indptr, indices, sids, scnt, sptr, U1, V1, B1, *hy)
    cut = int(sptr[u])                                       # the same user without social items
    sptr2 = sptr.copy()
    sptr2[u + 1] = cut
    U2, V2, B2 = U0.copy(), V0.copy(), B0.copy()
    sk2 = O.sbpr_replay(ii, j, np.array([cut], np.int64), indptr, indices, sids[:cut], scnt[:cut], sptr2, U2, V2, B2, *hy)
    assert sk == sk2 == 0
    assert np.array_equal(U1, U2) and np.array_equal(V1, V2) and np.array_equal(B1, B2)
    i = indices[ii[0]]
    moved = np.flatnonzero(np.any(V1 != V0, axis=1))
    assert set(moved.tolist()) == {i, int(j[0])}
    assert set(np.flatnonzero(B1 != B0).tolist()) == {i, int(j[0])}      # the fall-back trains biases whatever use_bias
