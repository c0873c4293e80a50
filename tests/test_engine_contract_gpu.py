"""The engine wrappers refuse a mis-sized or mis-typed device argument before any launch: the C entry points take raw
pointers, so an extent the wrapper does not check becomes an out-of-bounds device access.  Each case passes one bad
tensor and expects a B200Error that names it, no kernel launched by the library, and a clean device afterwards."""
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_USERS, N_ITEMS, K = 6, 5, 4
INDPTR = np.array([0, 2, 3, 3, 5, 6, 8], dtype=np.int32)
INDICES = np.array([0, 3, 1, 2, 4, 0, 1, 4], dtype=np.int32)


def f32(*shape):
    return torch.zeros(shape, dtype=torch.float32, device="cuda")


def f64(*shape):
    return torch.zeros(shape, dtype=torch.float64, device="cuda")


def i64(*shape):
    return torch.zeros(shape, dtype=torch.int64, device="cuda")


def i32(*shape):
    return torch.zeros(shape, dtype=torch.int32, device="cuda")


def users(n):
    return torch.arange(n, dtype=torch.int64, device="cuda")


def excl(n_q):
    return torch.zeros(n_q + 1, dtype=torch.int64, device="cuda"), i32(1)


def bpr_data():
    from cornac_b200 import engine
    return engine.BprData.from_host(INDPTR, INDICES)


def bpr_epoch(**bad):
    from cornac_b200 import engine
    a = dict(U=f32(N_USERS, K), V=f32(N_ITEMS, K), B=f32(N_ITEMS), stats=i64(2))
    a.update(bad)
    engine.bpr_epoch(bpr_data(), N_ITEMS, a["U"], a["V"], a["B"], 0.05, 0.01, True, 1, 0, a["stats"])


def bpr_epoch_replay(**bad):
    from cornac_b200 import engine
    a = dict(i_index=i64(8), j_id=i32(8), U=f32(N_USERS, K), V=f32(N_ITEMS, K), B=f32(N_ITEMS), stats=i64(2))
    a.update(bad)
    engine.bpr_epoch_replay(bpr_data(), a["i_index"], a["j_id"], a["U"], a["V"], a["B"], 0.05, 0.01, True, a["stats"])


def mf_epoch(**bad):
    from cornac_b200 import engine
    a = dict(rid=i32(8), cid=i32(8), val=f32(8), U=f32(N_USERS, K), V=f32(N_ITEMS, K), Bu=f32(N_USERS), Bi=f32(N_ITEMS),
             loss=f32(1))
    a.update(bad)
    engine.mf_epoch(a["rid"], a["cid"], a["val"], a["U"], a["V"], a["Bu"], a["Bi"], 0.01, 0.02, 3.0, True, a["loss"])


def score_batch(**bad):
    from cornac_b200 import engine
    a = dict(U=f32(N_USERS, K), V=f32(N_ITEMS, K), user_idx=users(3), item_base=f32(N_ITEMS), user_off=f32(3),
             out=f32(3, N_ITEMS))
    a.update(bad)
    engine.score_batch(**a)


def score_batch_f64(**bad):
    from cornac_b200 import engine
    a = dict(U=f64(N_USERS, K), V=f64(N_ITEMS, K), user_idx=users(3), out=f64(3, N_ITEMS))
    a.update(bad)
    engine.score_batch_f64(**a)


def rank_topk(**bad):
    from cornac_b200 import engine
    ep, ei = excl(3)
    a = dict(U=f32(N_USERS, K), V=f32(N_ITEMS, K), user_idx=users(3), item_base=f32(N_ITEMS), user_off=f32(3),
             excl_indptr=ep, excl_indices=ei)
    a.update(bad)
    engine.rank_topk(a.pop("U"), a.pop("V"), 2, **a)


def topk_rows(**bad):
    from cornac_b200 import engine
    ep, ei = excl(3)
    a = dict(scores=f32(3, N_ITEMS), excl_indptr=ep, excl_indices=ei)
    a.update(bad)
    engine.topk_rows(a.pop("scores"), 2, **a)


def rank_counts(**bad):
    from cornac_b200 import engine
    pos_indptr = torch.tensor([0, 1, 2, 3], dtype=torch.int64, device="cuda")
    a = dict(scores=f32(3, N_ITEMS), pos_indptr=pos_indptr, pos_indices=i32(3), user_idx=users(3), less=i64(3),
             pos_score=f32(3))
    a.update(bad)
    engine.rank_counts(**a)


def delta_make(**bad):
    from cornac_b200 import engine
    a = dict(x=f32(10), snapshot=f32(10), delta=f32(10))
    a.update(bad)
    engine.delta_make(**a)


def delta_apply(**bad):
    from cornac_b200 import engine
    a = dict(x=f32(10), snapshot=f32(10), delta=f32(10))
    a.update(bad)
    engine.delta_apply(**a)


def pmf_fit(**bad):
    from cornac_b200 import engine
    uid = np.repeat(np.arange(N_USERS, dtype=np.int32), np.diff(INDPTR))
    data = engine.PmfData(uid, INDICES, np.ones(len(INDICES), np.float32), N_USERS, N_ITEMS)
    a = dict(U=f64(N_USERS, K), V=f64(N_ITEMS, K), cache_u=f64(N_USERS, K), cache_v=f64(N_ITEMS, K))
    a.update(bad)
    engine.pmf_fit(data, "linear", a["U"], a["V"], a["cache_u"], a["cache_v"], 1, 0.01, 0.01, 0.9)


def cofactor_fit(**bad):
    from cornac_b200 import engine
    uid = np.repeat(np.arange(N_USERS, dtype=np.int32), np.diff(INDPTR))
    net = np.array([0, 1, 2], dtype=np.int32)
    data = engine.CofactorData("sorec", net, net[::-1].copy(), np.ones(3, np.float32), uid, INDICES,
                               np.ones(len(INDICES), np.float32), N_USERS, N_ITEMS)
    a = dict(U=f64(N_USERS, K), V=f64(N_ITEMS, K), Z=f64(N_USERS, K))
    a.update(bad)
    engine.cofactor_fit(data, a["U"], a["V"], a["Z"], f64(N_USERS, K), f64(N_ITEMS, K), f64(N_USERS, K), 1, 1.0, 0.01,
                        0.01, 0.9)


def nmf_fit(**bad):
    from cornac_b200 import engine
    data = engine.NmfData(INDPTR, INDICES, np.ones(len(INDICES), np.float32), N_ITEMS, False)
    a = dict(U=f32(N_USERS, K), V=f32(N_ITEMS, K), Bu=f32(N_USERS), Bi=f32(N_ITEMS), workspace=f32(N_USERS, K))
    a.update(bad)
    engine.nmf_fit(data, a["U"], a["V"], a["Bu"], a["Bi"], 1, workspace=a["workspace"])


def hpf_fit(**bad):
    from cornac_b200 import engine
    rid = np.repeat(np.arange(N_USERS), np.diff(INDPTR))
    data = engine.HpfData(rid, INDICES, np.ones(len(INDICES)), N_USERS, N_ITEMS)
    a = dict(Gs=f64(N_USERS, K), Gr=f64(N_USERS, K), Ls=f64(N_ITEMS, K), Lr=f64(N_ITEMS, K), Kr=f64(N_USERS),
             Tr=f64(N_ITEMS))
    a.update(bad)
    engine.hpf_fit(data, True, a["Gs"], a["Gr"], a["Ls"], a["Lr"], a["Kr"], a["Tr"], 1)


def efm_fit(**bad):
    import scipy.sparse as sp
    from cornac_b200 import engine
    A = sp.csr_matrix((np.ones(len(INDICES)), INDICES, INDPTR), shape=(N_USERS, N_ITEMS))
    data = engine.EfmData(A, sp.random(N_USERS, 3, density=0.5, random_state=0),
                          sp.random(N_ITEMS, 3, density=0.5, random_state=1))
    a = dict(U1=f32(N_USERS, K), U2=f32(N_ITEMS, K), V=f32(3, K), H1=f32(N_USERS, 2), H2=f32(N_ITEMS, 2))
    a.update(bad)
    engine.efm_fit(data, a["U1"], a["U2"], a["V"], a["H1"], a["H2"], 1)


def mter_fit(**bad):
    from cornac_b200 import engine
    one_f, one_i = np.ones(1, np.float32), np.zeros(1, np.int32)
    data = engine.MterDeviceData(engine.MterData(
        n_users=N_USERS, n_items=N_ITEMS, n_aspects=3, n_opinions=2, X=one_f, X_uids=one_i, X_iids=one_i, X_aids=one_i,
        YU=one_f, YU_uids=one_i, YU_aids=one_i, YU_oids=one_i, YI=one_f, YI_iids=one_i, YI_aids=one_i, YI_oids=one_i,
        indptr=INDPTR, indices=INDICES, user_ids=np.repeat(np.arange(N_USERS, dtype=np.int32), np.diff(INDPTR)),
        pair_rating=np.ones(len(INDICES), np.float32)))
    d = 2
    params = [f32(N_USERS, d), f32(N_ITEMS, d), f32(4, d), f32(2, d), f32(d, d, d), f32(d, d, d), f32(d, d, d)]
    a = dict(draws=i32(1, 3 * 4 + 2 * 4), counts=i64(2))
    a.update(bad)
    engine.mter_fit(data, params, [torch.zeros_like(p) for p in params], a["draws"], 1, 4, 4, counts=a["counts"])


def comparer_rank_rows(**bad):
    from cornac_b200 import engine
    d = 2
    a = dict(out=f32(3, N_ITEMS))
    a.update(bad)
    engine.comparer_rank_rows(f32(N_USERS, d), f32(N_ITEMS, d), f32(4, d), f32(d, d, d), users(3), 2, 0.5, out=a["out"])


def ease_score(**bad):
    import scipy.sparse as sp
    from cornac_b200 import engine
    X = sp.csr_matrix((np.ones(len(INDICES)), INDICES, INDPTR), shape=(N_USERS, N_ITEMS))
    a = dict(B=f64(N_ITEMS, N_ITEMS), out=f64(2, N_ITEMS))
    a.update(bad)
    engine.ease_score(a["B"], [0, 1], engine.EaseRatings(X), out=a["out"])


def ease_gram(**bad):
    import scipy.sparse as sp
    from cornac_b200 import engine
    X = sp.csr_matrix((np.ones(len(INDICES)), INDICES, INDPTR), shape=(N_USERS, N_ITEMS))
    a = dict(out=f64(N_ITEMS, N_ITEMS), workspace=None)
    a.update(bad)
    engine.ease_gram(engine.EaseGramInput(X), 1.0, a["out"], workspace=a["workspace"])


def spd_inverse(**bad):
    from cornac_b200 import engine
    engine.spd_inverse(bad.get("A", f64(4, 4)))


def knn_score(**bad):
    import scipy.sparse as sp
    from cornac_b200 import engine
    X = sp.csr_matrix((np.ones(len(INDICES)), INDICES, INDPTR), shape=(N_USERS, N_ITEMS))
    engine.knn_score(False, bad.get("S", f64(N_ITEMS, N_ITEMS)), [0, 1], engine.KnnRatings(X, np.zeros(N_USERS)), 2)


CASES = [
    # (wrapper, bad argument, bad value); the value is built on the device when the case runs
    (score_batch, "U", lambda: f32(N_USERS, K + 1)),                   # k is V's width
    (score_batch, "out", lambda: f32(3, N_ITEMS - 1)),                 # would be written past its end
    (score_batch, "item_base", lambda: f32(N_ITEMS - 1)),
    (score_batch, "user_off", lambda: f32(2)),
    (score_batch, "user_idx", lambda: i32(3)),
    (score_batch_f64, "U", lambda: f64(N_USERS, K + 1)),
    (score_batch_f64, "out", lambda: f64(2, N_ITEMS)),
    (rank_topk, "U", lambda: f32(N_USERS, K - 1)),
    (rank_topk, "user_idx", lambda: i32(3)),
    (rank_topk, "excl_indptr", lambda: i32(4)),                        # would be read as int64
    (rank_topk, "excl_indptr", lambda: i64(3)),
    (rank_topk, "excl_indices", lambda: i64(1)),
    (rank_topk, "item_base", lambda: f32(N_ITEMS - 1)),
    (rank_topk, "user_off", lambda: f32(2)),
    (bpr_epoch, "V", lambda: f32(N_ITEMS, K + 1)),                     # k is U's width
    (bpr_epoch, "V", lambda: f32(N_ITEMS - 1, K)),                     # fewer rows than n_neg, the negatives' range
    (bpr_epoch, "B", lambda: f32(N_ITEMS - 1)),
    (bpr_epoch, "U", lambda: f32(N_USERS - 1, K)),                     # fewer rows than the data has users
    (bpr_epoch, "stats", lambda: i64(1)),
    (bpr_epoch_replay, "V", lambda: f32(N_ITEMS, K + 1)),
    (bpr_epoch_replay, "j_id", lambda: i32(7)),
    (mf_epoch, "V", lambda: f32(N_ITEMS, K + 1)),
    (mf_epoch, "cid", lambda: i32(7)),
    (pmf_fit, "U", lambda: f64(N_USERS - 1, K)),
    (pmf_fit, "cache_v", lambda: f64(N_ITEMS - 1, K)),
    (cofactor_fit, "Z", lambda: f64(N_USERS - 1, K)),
    (cofactor_fit, "V", lambda: f64(N_ITEMS - 1, K)),
    (ease_score, "out", lambda: f64(2, N_ITEMS - 1)),
    (ease_score, "B", lambda: f64(N_ITEMS, N_ITEMS - 1)),
    (rank_counts, "less", lambda: i64(2)),                             # indexed like pos_indices
    (rank_counts, "pos_score", lambda: f32(2)),
    (rank_counts, "user_idx", lambda: users(2)),
    (delta_make, "snapshot", lambda: f32(9)),
    (delta_make, "delta", lambda: f64(10)),
    (delta_apply, "x", lambda: f32(10).cpu()),
    (delta_apply, "delta", lambda: f32(9)),
    (topk_rows, "excl_indptr", lambda: i64(3)),
    (nmf_fit, "workspace", lambda: f32(N_USERS * K - 1)),
    (nmf_fit, "Bi", lambda: f32(N_ITEMS + 1)),
    (hpf_fit, "Kr", lambda: f64(N_ITEMS)),
    (hpf_fit, "Ls", lambda: f64(N_ITEMS, K + 1)),
    (efm_fit, "U2", lambda: f32(N_ITEMS + 1, K)),
    (mter_fit, "draws", lambda: i32(1, 19)),
    (mter_fit, "counts", lambda: i64(1)),
    (comparer_rank_rows, "out", lambda: f32(3, N_ITEMS + 1)),
    (ease_gram, "workspace", lambda: f32(1 << 20)),
    (spd_inverse, "A", lambda: f64(4, 3)),
    (knn_score, "S", lambda: f64(N_ITEMS + 1, N_ITEMS + 1)),
]


@pytest.mark.parametrize("call, name, bad", CASES,
                         ids=["%s-%s-%d" % (c.__name__, n, i) for i, (c, n, _) in enumerate(CASES)])
def test_bad_argument_is_refused_before_any_launch(call, name, bad):
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    L = engine.require_cuda()
    value = bad()
    torch.cuda.synchronize()
    launches = int(L.b200_kernel_launches())
    with pytest.raises(B200Error, match="^%s must be a contiguous CUDA tensor" % re.escape(name)):
        call(**{name: value})
    assert int(L.b200_kernel_launches()) == launches
    torch.cuda.synchronize()


def test_refusal_names_the_expected_and_the_actual_shape():
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    engine.require_cuda()
    with pytest.raises(B200Error, match=r"^out must be a contiguous CUDA tensor of dtype torch.float32 and shape "
                                        r"\(3, %d\), got a cuda:\d+ tensor of dtype torch.float32 and shape \(3, %d\)$"
                                        % (N_ITEMS, N_ITEMS - 1)):
        score_batch(out=f32(3, N_ITEMS - 1))
    with pytest.raises(B200Error, match=r"^U must be .* got a cpu tensor"):
        score_batch(U=f32(N_USERS, K).cpu())
    with pytest.raises(B200Error, match=r"shape \(>=%d, %d\)" % (N_ITEMS, K)):
        bpr_epoch(V=f32(N_ITEMS - 1, K))
    with pytest.raises(B200Error, match=r"shape \[>=%d elements\]" % (N_USERS * K)):
        nmf_fit(workspace=f32(3))
