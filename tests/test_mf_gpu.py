"""MF kernels (through the C ABI) against the oracle and the golden vectors.  GPU only."""
import numpy as np
import pytest

from conftest import golden, rel_err
from oracle import oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _dev(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).cuda()


@pytest.mark.parametrize("ids32", [False, True])
@pytest.mark.parametrize("name", ["mf_small_k10", "mf_mid_k32", "mf_nobias_k16"])
def test_ordered_fit_matches_reference_golden(name, ids32):
    import torch
    from cornac_b200 import engine
    g = golden(name)
    k = int(g["k"])
    U0, V0, Bu0, Bi0 = O.mf_init(int(g["seed"]), int(g["num_users"]), int(g["num_items"]), k)
    idt = torch.int32 if ids32 else torch.int64
    rid, cid, val = _dev(g["rid"], idt), _dev(g["cid"], idt), _dev(g["val"])
    U, V, Bu, Bi = _dev(U0), _dev(V0), _dev(Bu0), _dev(Bi0)
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    ref = O.mf_fit(g["rid"], g["cid"], g["val"], int(g["num_users"]), int(g["num_items"]), k, int(g["max_iter"]),
                   float(g["lr"]), float(g["reg"]), bool(g["use_bias"]), False, int(g["seed"]), float(g["global_mean"]))
    for ep in range(int(g["max_iter"])):
        engine.mf_epoch(rid, cid, val, U, V, Bu, Bi, float(g["lr"]), float(g["reg"]), float(g["mu"]),
                        bool(g["use_bias"]), loss, ordered=True)
        assert abs(0.5 * loss.item() - ref["losses"][ep]) <= 1e-5 * abs(ref["losses"][ep])
    for got, want in ((U, g["U"]), (V, g["V"])):
        got = got.cpu().numpy()
        assert rel_err(got, want) < TOL and np.allclose(got, want, rtol=1e-4, atol=1e-6)
    if bool(g["use_bias"]):
        assert rel_err(Bu.cpu().numpy(), g["Bu"]) < TOL and rel_err(Bi.cpu().numpy(), g["Bi"]) < TOL
    else:
        assert np.all(Bu.cpu().numpy() == 0) and np.all(Bi.cpu().numpy() == 0)


@pytest.mark.parametrize("atomic", [False, True])
@pytest.mark.parametrize("k", [4, 10, 16, 32, 64, 100, 128, 256])
def test_hogwild_equals_sequential_when_conflict_free(k, atomic):
    """Ratings with pairwise distinct users and items: no races, any order gives the same result."""
    import torch
    from cornac_b200 import engine
    n = 3001
    rng = np.random.RandomState(k)
    rid = rng.permutation(5000)[:n].astype(np.int64)
    cid = rng.permutation(4000)[:n].astype(np.int64)
    val = rng.randint(1, 6, size=n).astype(np.float32)
    U0 = rng.normal(0, 0.2, (5000, k)).astype(np.float32)
    V0 = rng.normal(0, 0.2, (4000, k)).astype(np.float32)
    Bu0 = rng.normal(0, 0.2, 5000).astype(np.float32)
    Bi0 = rng.normal(0, 0.2, 4000).astype(np.float32)
    Ur, Vr, Bur, Bir = U0.copy(), V0.copy(), Bu0.copy(), Bi0.copy()
    loss_ref = O.mf_epoch(rid, cid, val, Ur, Vr, Bur, Bir, 0.01, 0.02, 3.0, True)
    U, V, Bu, Bi = _dev(U0), _dev(V0), _dev(Bu0), _dev(Bi0)
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    engine.mf_epoch(_dev(rid), _dev(cid), _dev(val), U, V, Bu, Bi, 0.01, 0.02, 3.0, True, loss, ordered=False,
                    atomic=atomic)
    assert abs(0.5 * loss.item() - loss_ref) < 1e-4 * loss_ref
    for got, want in ((U, Ur), (V, Vr), (Bu, Bur), (Bi, Bir)):
        got = got.cpu().numpy()
        assert rel_err(got, want) < 1e-6 and np.allclose(got, want, rtol=2e-5, atol=1e-6)


def test_hogwild_lr0_identity_and_loss():
    import torch
    from cornac_b200 import engine
    n, k = 1_000_003, 64
    rng = np.random.RandomState(3)
    rid = rng.randint(20000, size=n).astype(np.int32)
    cid = rng.randint(5000, size=n).astype(np.int32)
    val = rng.randint(1, 6, size=n).astype(np.float32)
    U0 = rng.normal(0, 0.1, (20000, k)).astype(np.float32)
    V0 = rng.normal(0, 0.1, (5000, k)).astype(np.float32)
    Bu0 = rng.normal(0, 0.1, 20000).astype(np.float32)
    Bi0 = rng.normal(0, 0.1, 5000).astype(np.float32)
    U, V, Bu, Bi = _dev(U0), _dev(V0), _dev(Bu0), _dev(Bi0)
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    engine.mf_epoch(_dev(rid), _dev(cid), _dev(val), U, V, Bu, Bi, 0.0, 0.02, 3.0, True, loss)
    assert np.array_equal(U.cpu().numpy(), U0) and np.array_equal(V.cpu().numpy(), V0)
    pred = 3.0 + Bu0[rid] + Bi0[cid] + np.einsum("nk,nk->n", U0[rid].astype(np.float64), V0[cid].astype(np.float64))
    want = float(((val - pred) ** 2).sum())
    assert abs(loss.item() - want) < 1e-4 * want


def test_hogwild_training_tracks_cpu_hogwild():
    import torch
    from cornac_b200 import engine
    rng = np.random.RandomState(5)
    n_users, n_items, k, n = 4000, 1500, 16, 200000
    P, Q = rng.normal(0, 0.5, (n_users, 4)), rng.normal(0, 0.5, (n_items, 4))
    rid = rng.randint(n_users, size=n).astype(np.int64)
    cid = rng.randint(n_items, size=n).astype(np.int64)
    val = (3.0 + np.einsum("nk,nk->n", P[rid], Q[cid]) + rng.normal(0, 0.1, n)).astype(np.float32)
    U0, V0, Bu0, Bi0 = O.mf_init(1, n_users, n_items, k)
    Uc, Vc, Buc, Bic = U0.copy(), V0.copy(), Bu0.copy(), Bi0.copy()
    mu = float(val.mean())
    cpu = [O.mf_epoch(rid, cid, val, Uc, Vc, Buc, Bic, 0.02, 0.01, mu, True, n_threads=O.n_threads()) for _ in range(20)]
    U, V, Bu, Bi = _dev(U0), _dev(V0), _dev(Bu0), _dev(Bi0)
    d = (_dev(rid), _dev(cid), _dev(val))
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    gpu = []
    for _ in range(20):
        engine.mf_epoch(*d, U, V, Bu, Bi, 0.02, 0.01, mu, True, loss)
        gpu.append(0.5 * loss.item())
    assert gpu[-1] < 0.5 * gpu[0]
    assert abs(gpu[-1] - cpu[-1]) < 0.25 * cpu[-1]      # Hogwild vs Hogwild: same regime, not the same trajectory


@pytest.mark.parametrize("hot", [False, True])
def test_windowed_ordered_epoch_is_bit_identical_to_serial(hot, monkeypatch):
    import torch
    from cornac_b200 import engine
    n_users, n_items = (30, 9) if hot else (4000, 2500)
    n, k = 20007, 20
    rng = np.random.RandomState(8)
    rid = rng.randint(n_users, size=n).astype(np.int64)
    cid = rng.randint(n_items, size=n).astype(np.int64)
    val = rng.randint(1, 6, size=n).astype(np.float32)
    U0, V0, Bu0, Bi0 = O.mf_init(3, n_users, n_items, k)
    outs = []
    for serial in ("1", "0"):
        monkeypatch.setenv("B200_REPLAY_SERIAL", serial)
        U, V, Bu, Bi = _dev(U0), _dev(V0), _dev(Bu0), _dev(Bi0)
        loss = torch.zeros(1, dtype=torch.float32, device="cuda")
        for _ in range(2):
            engine.mf_epoch(_dev(rid), _dev(cid), _dev(val), U, V, Bu, Bi, 0.01, 0.02, 3.0, True, loss, ordered=True)
        outs.append((U.cpu().numpy(), V.cpu().numpy(), Bu.cpu().numpy(), Bi.cpu().numpy(), loss.item()))
    for a, b in zip(outs[0][:4], outs[1][:4]):
        assert np.array_equal(a, b)
    assert outs[0][4] == outs[1][4]
    Ur, Vr, Bur, Bir = U0.copy(), V0.copy(), Bu0.copy(), Bi0.copy()
    for _ in range(2):
        l_ref = O.mf_epoch(rid, cid, val, Ur, Vr, Bur, Bir, 0.01, 0.02, 3.0, True)
    assert rel_err(outs[1][0], Ur) < 1e-5 and abs(0.5 * outs[1][4] - l_ref) < 1e-4 * l_ref


def test_mf_fit_sharded_single_process_trains_like_plain_epochs():
    """parallel.mf_fit_sharded with no process group (world 1): the whole rating list is this rank's shard; the
    result must be in the same regime as the oracle's sequential epochs and be written back into the host arrays."""
    from cornac_b200 import parallel
    rng = np.random.RandomState(8)
    n_users, n_items, k, n = 3000, 1000, 16, 120000
    P, Q = rng.normal(0, 0.5, (n_users, 4)), rng.normal(0, 0.5, (n_items, 4))
    rid = rng.randint(n_users, size=n).astype(np.int64)
    cid = rng.randint(n_items, size=n).astype(np.int64)
    val = (3.0 + np.einsum("nk,nk->n", P[rid], Q[cid]) + rng.normal(0, 0.1, n)).astype(np.float32)
    U0, V0, Bu0, Bi0 = O.mf_init(2, n_users, n_items, k)
    Uc, Vc, Buc, Bic = U0.copy(), V0.copy(), Bu0.copy(), Bi0.copy()
    mu = float(val.mean())
    cpu = [O.mf_epoch(rid, cid, val, Uc, Vc, Buc, Bic, 0.02, 0.01, mu, True) for _ in range(10)]
    U, V, Bu, Bi = U0.copy(), V0.copy(), Bu0.copy(), Bi0.copy()
    bounds, losses = parallel.mf_fit_sharded(rid, cid, val, U, V, Bu, Bi, 0.02, 0.01, mu, True, max_iter=10)
    assert bounds.tolist() == [0, n_users] and len(losses) == 10
    assert losses[-1] < losses[0] and abs(losses[0] - cpu[0]) < 0.02 * cpu[0] and abs(losses[-1] - cpu[-1]) < 0.02 * cpu[-1]
    assert np.abs(U - U0).max() > 1e-4 and np.abs(V - V0).max() > 1e-4 and np.abs(Bi - Bi0).max() > 1e-3
