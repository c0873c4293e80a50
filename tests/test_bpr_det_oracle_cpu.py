"""The deterministic BPR epoch's committed digests recomputed without a GPU by the serial oracle
(oracle/bpr_det_oracle.c), and unit tests of the oracle's round rule.

Every committed case whose z can be restated exactly (hinge and exact exp) is replayed on the CPU from the inputs
tests/golden/make_golden_bpr_det.py uses; the SHA-256 of U, V, B and the per-epoch (correct, skipped) counts must equal
the committed ones.  So the digests are proven to be the output of the specified rule, not only of some earlier kernel.
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import make_golden_bpr_det as M  # noqa: E402
from oracle import bpr_det_oracle as DO  # noqa: E402

with open(os.path.join(GOLDEN, "bpr_det_digests.json")) as _f:
    DIGESTS = json.load(_f)

RESTATED = ["mid_k128_exact", "mid_k64_hinge", "mid_k130_hinge_blocked", "small_k130_exact"]
_CASES = {c["name"]: c for c in M.CASES}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_case_oracle(c, monkeypatch):
    """make_golden_bpr_det.run_case on the oracle: same data, seeds, hyperparameters and epoch arguments."""
    n_users, n_items, _, _ = M.SHAPES[c["shape"]]
    indptr, indices = M._shape_data(c["shape"])
    k = c["k"]
    rng = np.random.RandomState(k * 7 + 1)
    U = rng.normal(0, 0.1, (n_users, k)).astype(np.float32)
    V = rng.normal(0, 0.1, (n_items, k)).astype(np.float32)
    B = rng.normal(0, 0.1, n_items).astype(np.float32)
    if c["part_mb"] is not None:
        monkeypatch.setenv("B200_BPR_PART_MB", str(c["part_mb"]))
    assert not c["exact_exp"] or not c["hinge"]
    stats, max_d = DO.train(indptr, indices, n_items, U, V, B, 0.05, 0.01, c["use_bias"], M.SEED, M.EPOCHS,
                            n_samples=c["n_samples"], sample_base=c["sample_base"], base_step=7919, hinge=c["hinge"],
                            neg_weighted=c["neg_weighted"], blocked=c["blocked"], unbounded=c["unbounded"])
    return {"U": _sha(U), "V": _sha(V), "B": _sha(B), "stats": stats}, max_d


def test_restated_cases_are_the_ones_with_an_exact_z():
    for name in RESTATED:
        c = _CASES[name]
        assert c["hinge"] or c["exact_exp"], name
    assert sorted(n for n, c in _CASES.items() if c["hinge"] or c["exact_exp"]) == sorted(RESTATED)


@pytest.mark.parametrize("name", RESTATED)
def test_oracle_reproduces_committed_digest(name, monkeypatch):
    got, max_d = run_case_oracle(_CASES[name], monkeypatch)
    want = DIGESTS["cases"][name]
    print("%s: largest |d| = %.6g" % (name, max_d))
    assert got["stats"] == want["stats"]
    for x in ("U", "V", "B"):
        assert got[x] == want[x], x
    # no delta of the committed cases comes near the per-delta bound, so tightening it cannot change a digest
    assert 0.0 < max_d < 1e-3 * DO.delta_bound(DO.DET_ROUND)


def test_round_size_rule(monkeypatch):
    """R = min(max(16, min(rows) / 4) [per window / block when blocked], 16384), unlimited staleness -> 16384."""
    assert DO.round_size(100_000, 70_000, 64) == 16384
    assert DO.round_size(2_000, 300, 10) == 75
    assert DO.round_size(200, 40, 8) == 16
    assert DO.round_size(200, 40, 8, unbounded=True) == 16384
    monkeypatch.setenv("B200_BPR_PART_MB", "4")
    assert DO.block_plan(100_000, 70_000, 130, True, False) == (13, 9)
    assert DO.round_size(100_000, 70_000, 130, blocked=True) == 1923
    assert DO.round_size(100_000, 70_000, 128, blocked=True, neg_weighted=True) == min(100_000 // 13, 70_000) // 4
    assert DO.round_size(100_000, 70_000, 130, blocked=True, unbounded=True) == 16384


def test_delta_bound_keeps_every_round_sum_in_range():
    assert DO.delta_bound(16384) == 256.0
    assert DO.delta_bound(16) == 2.0 ** 18 and DO.delta_bound(75) == 2.0 ** 15 and DO.delta_bound(1) == 2.0 ** 22
    for R in (1, 2, 3, 16, 75, 1923, 16383, 16384):
        b = DO.delta_bound(R)
        assert R * b <= 2.0 ** 22 < 2 * R * b      # R deltas just under the bound sum to < 2^62 fixed-point units
        d = np.full(R, np.nextafter(np.float32(b), np.float32(0)), np.float32)
        want = np.float32(np.float32(0.5) + np.float32(float(R) * float(d[0])))
        assert DO.sum_apply(0.5, d, b) == want


def test_round_sum_is_order_independent():
    rng = np.random.RandomState(3)
    d = (rng.standard_normal(5000) * 10.0 ** rng.uniform(-9, 2, 5000)).astype(np.float32)
    x = np.float32(0.3)
    ref = DO.sum_apply(x, d, 256.0)
    for _ in range(5):
        assert DO.sum_apply(x, rng.permutation(d), 256.0) == ref
    # the exact sum: integer fixed-point, then one rounding to f32
    q = sum(int(np.rint(np.float64(v) * 2.0 ** 40)) for v in d)
    assert ref == np.float32(np.float32(x) + np.float32(q * 2.0 ** -40))


def test_zero_sum_writes_nothing():
    # deltas that cancel exactly leave x untouched, even a subnormal or negative zero that the add would flush / change
    for x in (np.float32(1e-40), np.float32(-0.0), np.float32(0.7)):
        got = DO.sum_apply(x, np.array([0.25, -0.25], np.float32), 256.0)
        assert np.float32(got).tobytes() == x.tobytes()
    # a delta below 2^-41 quantises to zero: no write
    assert DO.sum_apply(1e-40, np.array([2.0 ** -42], np.float32), 256.0) == np.float32(1e-40)


def test_subnormal_x_takes_the_update_as_zero():
    """add.rn.ftz reads a subnormal x as zero.  A written update is at least 2^-40 in magnitude, so x + y is never
    subnormal and a subnormal x is far below half an ulp of y: the result is y itself, with or without the flush."""
    for x in (np.float32(1e-40), np.float32(-1e-40), np.float32(2.0 ** -149)):
        for y in (2.0 ** -40, -(2.0 ** -40), 3.0 * 2.0 ** -40, -0.75):
            got = np.float32(DO.sum_apply(x, np.array([y], np.float32), 256.0))
            assert got.tobytes() == np.float32(y).tobytes()


def test_delta_at_the_bound_is_nan():
    assert np.isnan(DO.sum_apply(0.5, np.array([256.0], np.float32), 256.0))
    assert np.isnan(DO.sum_apply(0.5, np.array([1.0, np.inf, -1.0], np.float32), 256.0))
    assert np.isnan(DO.sum_apply(0.5, np.array([np.nan], np.float32), 256.0))
    assert DO.sum_apply(0.5, np.array([np.nextafter(np.float32(256), np.float32(0))], np.float32), 256.0) == \
        np.float32(0.5 + float(np.nextafter(np.float32(256), np.float32(0))))


def test_deltas_under_the_old_bound_wrapped_to_a_finite_value():
    """The former bound (|d| < 2^22 alone) let three deltas of 2^21.5 overflow the int64 sum into a finite, wrong value;
    under delta_bound(R) they turn the element into NaN."""
    d = np.full(3, np.float32(2.0 ** 21.5), np.float32)
    wrapped = DO.sum_apply(0.0, d, 2.0 ** 22)
    assert np.isfinite(wrapped) and wrapped < 0          # 3 * 2^61.5 wraps past 2^63 to a negative sum
    assert np.isnan(DO.sum_apply(0.0, d, DO.delta_bound(16384)))
    assert np.isnan(DO.sum_apply(0.0, d, DO.delta_bound(16)))


def _tiny_problem(seed, n_users=30, n_items=12, k=5):
    rng = np.random.RandomState(seed)
    dense = rng.rand(n_users, n_items) < 0.3
    indptr = np.concatenate([[0], np.cumsum(dense.sum(1))]).astype(np.int32)
    indices = np.nonzero(dense)[1].astype(np.int32)
    U = rng.normal(0, 0.3, (n_users, k)).astype(np.float32)
    V = rng.normal(0, 0.3, (n_items, k)).astype(np.float32)
    B = rng.normal(0, 0.3, n_items).astype(np.float32)
    return rng, indptr, indices, U, V, B


def test_epoch_is_order_independent_within_a_round():
    rng, indptr, indices, U, V, B = _tiny_problem(5)
    n = 64
    coo = np.repeat(np.arange(30, dtype=np.int32), np.diff(indptr))
    ii = rng.randint(len(indices), size=n)
    su, si, sj = coo[ii], indices[ii], rng.randint(12, size=n).astype(np.int32)
    outs = []
    for perm in (np.arange(n), rng.permutation(n), rng.permutation(n)):
        Ux, Vx, Bx = U.copy(), V.copy(), B.copy()
        st = DO.epoch(indptr, indices, Ux, Vx, Bx, su[perm], si[perm], sj[perm], n, 0.1, 0.01, True, False)
        outs.append((Ux.tobytes(), Vx.tobytes(), Bx.tobytes(), st))
    assert outs[0] == outs[1] == outs[2]
    # rounds are not interchangeable: the second half reads what the first half wrote
    Ux, Vx, Bx = U.copy(), V.copy(), B.copy()
    DO.epoch(indptr, indices, Ux, Vx, Bx, su, si, sj, n // 2, 0.1, 0.01, True, False)
    assert Ux.tobytes() != outs[0][0]


def test_epoch_matches_a_float64_restatement_of_one_round():
    """One round against numpy: the same reads of the round's starting factors, deltas summed in f64."""
    rng, indptr, indices, U, V, B = _tiny_problem(9, k=40)
    n = 50
    coo = np.repeat(np.arange(30, dtype=np.int32), np.diff(indptr))
    ii = rng.randint(len(indices), size=n)
    su, si, sj = coo[ii], indices[ii], rng.randint(12, size=n).astype(np.int32)
    Uo, Vo, Bo = U.copy(), V.copy(), B.copy()
    c, s, _ = DO.epoch(indptr, indices, Uo, Vo, Bo, su, si, sj, n, 0.1, 0.01, True, False)
    dU, dV, dB = np.zeros(U.shape), np.zeros(V.shape), np.zeros(B.shape)
    n_skip = n_corr = 0
    for u, i, j in zip(su, si, sj):
        if j in indices[indptr[u]:indptr[u + 1]]:
            n_skip += 1
            continue
        x = float(B[i]) - float(B[j]) + float(U[u].astype(np.float64) @ (V[i].astype(np.float64) - V[j]))
        z = 1.0 / (1.0 + np.exp(x))
        n_corr += z < 0.5
        dU[u] += 0.1 * (z * (V[i].astype(np.float64) - V[j]) - 0.01 * U[u])
        dV[i] += 0.1 * (z * U[u].astype(np.float64) - 0.01 * V[i])
        dV[j] += 0.1 * (-z * U[u].astype(np.float64) - 0.01 * V[j])
        dB[i] += 0.1 * (z - 0.01 * B[i])
        dB[j] += 0.1 * (-z - 0.01 * B[j])
    assert s == n_skip and c == n_corr and n_skip < n
    for got, x0, d in ((Uo, U, dU), (Vo, V, dV), (Bo, B, dB)):
        assert np.max(np.abs(got - (x0 + d))) <= 1e-6 * max(1.0, np.max(np.abs(x0)))
