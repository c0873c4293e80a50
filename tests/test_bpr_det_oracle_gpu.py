"""The deterministic BPR epoch (engine.bpr_epoch(..., deterministic=True)) against the serial oracle
(oracle/bpr_det_oracle.c), bit for bit: U, V, B bytes and the per-epoch (correct, skipped) counts over 2-3 epochs, at
shapes and edges the committed digests do not reach -- k around the warp width and the register-resident 128 elements,
rounds of 16 samples, a partial last round of one sample, a user with 30 % of the interactions, a Zipf-1.6 item,
rounds where every sample is skipped, WBPR, blocked orders, a sample base across 2^32 and an epoch beyond 2^32.  The
fast __expf path is compared with the oracle's exact z within a bound derived from the __expf error.  GPU only."""
import numpy as np
import pytest
import torch

from oracle import bpr_det_oracle as DO

pytestmark = pytest.mark.gpu

SEED = 1234
LR, REG = 0.05, 0.01


def _csr(n_users, n_items, u, i):
    key = np.unique(np.asarray(u, np.int64) * n_items + np.asarray(i, np.int64))
    u, i = key // n_items, key % n_items
    indptr = np.zeros(n_users + 1, np.int64)
    np.add.at(indptr, u + 1, 1)
    return np.cumsum(indptr).astype(np.int32), i.astype(np.int32)


def _synth(n_users, n_items, nnz, seed, zipf=0.8):
    rng = np.random.RandomState(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** zipf
    p /= p.sum()
    u = rng.randint(n_users, size=nnz)
    return _csr(n_users, n_items, u, rng.choice(n_items, size=nnz, p=p))


def _hot_user(n_users, n_items, nnz, seed, frac=0.3):
    """User 0 holds `frac` of the interactions: a user row with thousands of terms in a round of 16384."""
    rng = np.random.RandomState(seed)
    n_hot = int(frac * nnz)
    u = np.concatenate([np.zeros(n_hot, np.int64), rng.randint(1, n_users, size=nnz - n_hot)])
    i = np.concatenate([rng.choice(n_items, size=n_hot, replace=False), rng.randint(n_items, size=nnz - n_hot)])
    return _csr(n_users, n_items, u, i)


def _full_rows_first(n_users, n_items, n_full, seed):
    """Users 0..n_full-1 hold every item (each of their samples is skipped); the others one item each."""
    rng = np.random.RandomState(seed)
    u = np.concatenate([np.repeat(np.arange(n_full), n_items), np.arange(n_full, n_users)])
    i = np.concatenate([np.tile(np.arange(n_items), n_full), rng.randint(n_items, size=n_users - n_full)])
    return _csr(n_users, n_items, u, i)


DATA = {
    "S": lambda: (_synth(1500, 400, 15000, 1), 400),             # R = 100
    "T": lambda: (_synth(200, 40, 2500, 2), 40),                 # R = 16 from a 40-item catalogue
    "H": lambda: (_hot_user(2000, 20000, 40000, 3), 20000),      # with unbounded: R = 16384, user 0 ~ 4900 terms a round
    "Z": lambda: (_synth(20000, 5000, 60000, 4, zipf=1.6), 5000),
    "F": lambda: (_full_rows_first(9000, 40, 300, 5), 40),       # part_mb=1, k=64: 3 windows, window 0 all skipped
    "A": lambda: (_full_rows_first(100, 30, 100, 6), 30),        # every sample skipped
    "BB": lambda: (_synth(6000, 6000, 60000, 7), 6000),          # part_mb=1: 2 x 2 runs (R = 750) at k = 64, 3 x 3 at 128
}
_CACHE = {}


def _data(name):
    if name not in _CACHE:
        _CACHE[name] = DATA[name]()
    return _CACHE[name]


def _case(name, data, k, mode, epochs=3, **kw):
    c = dict(name=name, data=data, k=k, mode=mode, epochs=epochs, use_bias=True, neg_weighted=False, blocked=False,
             unbounded=False, part_mb=None, n_samples=None, sample_base=0, base_step=7919, epoch0=0)
    c.update(kw)
    return pytest.param(c, id=name)


EXACT_CASES = (
    [_case("k%d_%s" % (k, m), "S", k, m) for k in (1, 31, 32, 33, 127, 128, 129, 256) for m in ("hinge", "exact")]
    + [
        _case("r16_last_round_one", "T", 33, "exact", n_samples=16 * 37 + 1),
        _case("r16_multiple_of_round", "T", 33, "hinge", n_samples=16 * 40),
        _case("r16_below_one_round", "T", 33, "exact", n_samples=10),
        _case("hot_user_exact", "H", 64, "exact", unbounded=True),
        _case("hot_user_hinge_k129", "H", 129, "hinge", epochs=2, unbounded=True),
        _case("zipf16_exact", "Z", 32, "exact", unbounded=True),
        _case("zipf16_hinge_k130", "Z", 130, "hinge", epochs=2, unbounded=True),
        _case("skipped_rounds_blocked", "F", 64, "exact", blocked=True, part_mb=1),
        _case("all_skipped", "A", 8, "hinge", epochs=2),
        _case("nobias_exact", "S", 64, "exact", use_bias=False),
        _case("nobias_k130_exact", "S", 130, "exact", use_bias=False),
        _case("wbpr_exact", "S", 64, "exact", neg_weighted=True),
        _case("wbpr_hinge_blocked", "BB", 64, "hinge", neg_weighted=True, blocked=True, part_mb=1),
        _case("blocked_exact", "BB", 64, "exact", blocked=True, part_mb=1),
        _case("blocked_hinge_k128", "BB", 128, "hinge", epochs=2, blocked=True, part_mb=1),
        _case("base_across_2p32", "S", 32, "hinge", sample_base=2 ** 32 - 7000, n_samples=15000),
        _case("zero_init_hinge_ties", "S", 16, "hinge", init="zeros"),      # scores of exactly 0 are not "correct"
        _case("epoch_beyond_2p32_blocked", "BB", 64, "exact", epochs=2, blocked=True, part_mb=1, epoch0=2 ** 32 + 1),
    ]
)


def _init(n_users, n_items, k, seed):
    rng = np.random.RandomState(seed)
    return (rng.normal(0, 0.1, (n_users, k)).astype(np.float32), rng.normal(0, 0.1, (n_items, k)).astype(np.float32),
            rng.normal(0, 0.1, n_items).astype(np.float32))


def _run_device(c, indptr, indices, n_items, U0, V0, B0):
    from cornac_b200 import engine
    U, V, B = (torch.from_numpy(x.copy()).cuda() for x in (U0, V0, B0))
    data = engine.BprData.from_host(indptr, indices)
    stats = []
    for t in range(c["epochs"]):
        st = torch.zeros(2, dtype=torch.int64, device="cuda")
        engine.bpr_epoch(data, n_items, U, V, B, c.get("lr", LR), c.get("reg", REG), c["use_bias"], SEED, c["epoch0"] + t,
                         st, n_samples=c["n_samples"], sample_base=c["sample_base"] + t * c["base_step"],
                         exact_exp=c["mode"] == "exact", unbounded=c["unbounded"], neg_weighted=c["neg_weighted"], hinge=c["mode"] == "hinge",
                         blocked=c["blocked"], deterministic=True)
        stats.append([int(x) for x in st.cpu().tolist()])
    torch.cuda.synchronize()
    return U.cpu().numpy(), V.cpu().numpy(), B.cpu().numpy(), stats


def _run_oracle(c, indptr, indices, n_items, U0, V0, B0, d_max=None):
    U, V, B = U0.copy(), V0.copy(), B0.copy()
    stats, max_d = DO.train(indptr, indices, n_items, U, V, B, c.get("lr", LR), c.get("reg", REG), c["use_bias"], SEED,
                            c["epochs"], n_samples=c["n_samples"], sample_base=c["sample_base"], base_step=c["base_step"],
                            epoch0=c["epoch0"], hinge=c["mode"] == "hinge", neg_weighted=c["neg_weighted"],
                            blocked=c["blocked"], unbounded=c["unbounded"], d_max=d_max)
    return U, V, B, stats, max_d


def _run_both(c, monkeypatch):
    if c["part_mb"] is not None:
        monkeypatch.setenv("B200_BPR_PART_MB", str(c["part_mb"]))
    (indptr, indices), n_items = _data(c["data"])
    n_users, k = len(indptr) - 1, c["k"]
    U0, V0, B0 = _init(n_users, n_items, k, seed=k * 31 + len(c["name"]))
    if c.get("init") == "zeros":
        U0, V0, B0 = np.zeros_like(U0), np.zeros_like(V0), np.zeros_like(B0)
    dev = _run_device(c, indptr, indices, n_items, U0, V0, B0)
    orc = _run_oracle(c, indptr, indices, n_items, U0, V0, B0)
    return (indptr, indices, n_items, U0, V0, B0), dev, orc


def _first_diff(got, want):
    bad = np.flatnonzero(got.view(np.uint32).ravel() != want.view(np.uint32).ravel())
    if len(bad) == 0:
        return None
    f = int(bad[0])
    return "%d elements differ; first at flat index %d: %r (device) vs %r (oracle)" % (
        len(bad), f, got.ravel()[f], want.ravel()[f])


@pytest.mark.parametrize("c", EXACT_CASES)
def test_device_epoch_equals_oracle_bit_for_bit(c, monkeypatch):
    (indptr, indices, n_items, U0, V0, B0), dev, orc = _run_both(c, monkeypatch)
    U, V, B, stats = dev
    Uo, Vo, Bo, stats_o, max_d = orc
    assert stats == stats_o
    for name, g, w in (("U", U, Uo), ("V", V, Vo), ("B", B, Bo)):
        assert _first_diff(g, w) is None, (name, _first_diff(g, w))
    assert not (U.tobytes() == U0.tobytes() and B.tobytes() == B0.tobytes()) or c["data"] == "A"
    if c["data"] == "A":          # every sample skipped: nothing changes
        assert U.tobytes() == U0.tobytes() and V.tobytes() == V0.tobytes() and B.tobytes() == B0.tobytes()
        assert all(s == [0, len(indices) if c["n_samples"] is None else c["n_samples"]] for s in stats)


def test_the_edge_cases_reach_their_edges(monkeypatch):
    """The shapes above produce the rounds they are named for."""
    (indptr, indices), n_items = _data("T")
    assert DO.round_size(len(indptr) - 1, n_items, 33) == 16
    (indptr, indices), n_items = _data("H")
    assert np.diff(indptr)[0] >= 0.29 * len(indices) and DO.round_size(2000, n_items, 64, unbounded=True) == 16384
    (indptr, indices), n_items = _data("Z")
    assert np.bincount(indices).max() > 0.2 * len(indices)
    monkeypatch.setenv("B200_BPR_PART_MB", "1")
    (indptr, indices), n_items = _data("BB")
    assert DO.block_plan(len(indptr) - 1, n_items, 64, True, False) == (2, 2)
    assert DO.round_size(len(indptr) - 1, n_items, 64, blocked=True) == 750
    (indptr, indices), n_items = _data("F")
    n_users = len(indptr) - 1
    plan = DO.block_plan(n_users, n_items, 64, True, False)
    R = DO.round_size(n_users, n_items, 64, blocked=True)
    assert plan[0] > 1 and R == 16
    su, si, sj = DO.draw(indptr, indices, n_items, SEED, 0, len(indices), plan=plan)
    skip = np.array([j in indices[indptr[u]:indptr[u + 1]] for u, j in zip(su, sj)])
    n_r = len(skip) // R
    per_round = skip[:n_r * R].reshape(n_r, R).all(axis=1)
    assert per_round.any() and not per_round.all()


def test_k_above_256_is_rejected():
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    (indptr, indices), n_items = _data("T")
    U = torch.zeros((len(indptr) - 1, 257), device="cuda")
    V = torch.zeros((n_items, 257), device="cuda")
    B = torch.zeros(n_items, device="cuda")
    st = torch.zeros(2, dtype=torch.int64, device="cuda")
    with pytest.raises(B200Error, match="k=257"):
        engine.bpr_epoch(engine.BprData.from_host(indptr, indices), n_items, U, V, B, LR, REG, True, SEED, 0, st,
                         exact_exp=True, deterministic=True)


def test_deltas_that_would_wrap_the_round_sum_make_nan(monkeypatch):
    """A hot item collects many deltas of about 2^21.5 in one round, each below the former per-delta bound 2^22.  Three
    of them overflow the int64 sum; the element must come out NaN, not a finite wrapped value."""
    rng = np.random.RandomState(11)
    n_users, n_items, k = 200, 50, 8
    u = np.concatenate([np.arange(n_users), rng.randint(n_users, size=800)])
    i = np.concatenate([np.zeros(n_users, np.int64), rng.randint(1, n_items, size=800)])
    indptr, indices = _csr(n_users, n_items, u, i)     # item 0 is in every row: it is a positive, never a negative
    U0, V0, B0 = _init(n_users, n_items, k, seed=12)
    U0[:, 0] = 3.0e6                                    # z * u = 3e6 ~ 2^21.5 on element 0 of every positive
    V0[:, 0] = 0.0                                      # ... which does not move the scores
    c = dict(name="wrap", k=k, mode="hinge", epochs=1, use_bias=True, neg_weighted=False, blocked=False,
             unbounded=True, part_mb=None, n_samples=len(indices), sample_base=0, base_step=0, epoch0=0, lr=1.0, reg=0.0)
    R = DO.round_size(n_users, n_items, k, unbounded=True)
    assert len(indices) <= R                             # one round: every sample reads the initial factors
    U, V, B, stats = _run_device(c, indptr, indices, n_items, U0, V0, B0)
    Uo, Vo, Bo, stats_o, max_d = _run_oracle(c, indptr, indices, n_items, U0, V0, B0)
    assert stats[0][1] == stats_o[0][1]                  # (correct counts may differ: a sample may read a NaN store)
    assert 2.0 ** 21 < max_d < 2.0 ** 22
    assert np.isnan(Vo[0, 0]) and np.isnan(V[0, 0])
    # every element the oracle turns into NaN is NaN on the device (the device may spread NaN further within the round:
    # other samples can read a NaN stored into a shared row)
    for g, w in ((U, Uo), (V, Vo), (B, Bo)):
        assert np.all(np.isnan(g[np.isnan(w)]))
    # what the former bound gave: the same deltas summed into a finite, wrong value
    Uw, Vw, Bw, _, _ = _run_oracle(c, indptr, indices, n_items, U0, V0, B0, d_max=2.0 ** 22)
    assert np.isfinite(Vw[0, 0])


FAST_CASES = [
    _case("fast_k64", "S", 64, "fast"),
    _case("fast_k130_nobias", "S", 130, "fast", use_bias=False),
    _case("fast_k128_blocked", "BB", 128, "fast", epochs=2, blocked=True, part_mb=1),
    _case("fast_zipf16_k32", "Z", 32, "fast", unbounded=True),
]


@pytest.mark.parametrize("c", FAST_CASES)
def test_fast_exp_epoch_within_expf_error_of_exact_oracle(c, monkeypatch):
    """The fast path computes z = __frcp_rn(1 + __expf(score)).  __expf has at most 2 + floor(1.173 |x|) ulp of error
    (CUDA C Programming Guide, intrinsic functions), so with |score| < 4 and the two roundings of 1 + e and of the
    reciprocal, z (the scores here are O(0.1)) is within 8 ulp = 2^-20 (relative) of the exact f32 z.  To first order a row's difference from the
    exact oracle is then at most 2^-20 of the row's total change; the margin 2^4 covers the feedback of the perturbed
    rows into later samples (each round's reads), which contracts at these step sizes.  Once two values differ, each
    round's f32 add may round them one ulp apart: at most 2^-24 of the row's norm per round of the run."""
    (indptr, indices, n_items, U0, V0, B0), dev, orc = _run_both(c, monkeypatch)
    U, V, B, stats = dev
    Uo, Vo, Bo, stats_o, _ = orc
    n = len(indices) if c["n_samples"] is None else c["n_samples"]
    R = DO.round_size(len(indptr) - 1, n_items, c["k"], c["blocked"], c["neg_weighted"], c["unbounded"])
    n_rounds = c["epochs"] * -(-n // R)
    for (cg, sg), (cw, sw) in zip(stats, stats_o):
        assert sg == sw                                     # the skip test does not read the factors
        assert abs(cg - cw) <= 2 + n // 1000                # z flips across 1/2 only within 2^-20 of it
    for g, w, x0 in ((U, Uo, U0), (V, Vo, V0)):
        diff = np.linalg.norm(g.astype(np.float64) - w, axis=1)
        change = np.linalg.norm(w.astype(np.float64) - x0, axis=1)
        size = np.linalg.norm(w.astype(np.float64), axis=1)
        bound = 2.0 ** -16 * change + n_rounds * 2.0 ** -24 * size
        assert np.all(diff <= bound), float(np.max(diff / np.maximum(bound, 1e-30)))
        assert np.all(np.isfinite(g))
    if c["use_bias"]:
        assert np.all(np.abs(B.astype(np.float64) - Bo) <= 2.0 ** -16 * np.abs(Bo.astype(np.float64) - B0)
                      + n_rounds * 2.0 ** -24 * np.abs(Bo))
    else:
        assert B.tobytes() == B0.tobytes()
