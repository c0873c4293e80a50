"""The scoring half of the Recommender contract, model by model: score(u) rows, rank(), the transform() cache,
rank_batch / recommend_batch and a save / load round trip, each against a host restatement built from score(u).

The rules restated here (cornac/models/recommender.py:476-530 with the total order score desc, item id asc):
  * the row is score(u); a ScoreException scores every item default_score(); unknown items get the row's minimum;
  * k == -1, k >= len(candidates) or k > 4096: every candidate, sorted;
  * otherwise the top k sorted, then the other candidates in candidate order;
  * SoRec and MCF rank with Recommender.rank itself, UserKNN and ItemKNN sort every candidate for every k.
The split has users and items that only the test set holds, so total_users > num_users and total_items > num_items."""
from collections import OrderedDict

import numpy as np
import pytest

from conftest import needs_cornac

pytestmark = [pytest.mark.gpu, needs_cornac]

F32 = ("BPR", "WBPR", "MMMF", "VEBPR", "SBPR", "MF", "NMF", "WMF", "BaselineOnly")
F64 = ("PMF", "HPF", "PF", "EASE", "SoRec", "MCF", "UserKNN", "ItemKNN")
NAMES = F32 + F64
ROW_BEYOND_RAISES = ("BPR", "WBPR", "MMMF", "VEBPR", "SBPR")      # score(u) reads the factor row of any user index
KS = (1, 10, None, -1, 5000)                                      # None: len(candidates)


def _data():
    from cornac.data import Dataset, GraphModality
    rng = np.random.RandomState(5)
    n_users, n_items = 150, 120
    tr = []
    for u in range(n_users):
        for i in rng.choice(n_items, size=rng.randint(8, 25), replace=False):
            tr.append(("u%d" % u, "i%d" % i, float(rng.randint(1, 6))))
    tr += [("u%d" % (i % n_users), "i%d" % i, 3.0) for i in range(n_items)]          # every item is a train item
    tr = list(OrderedDict(((a, b), (a, b, r)) for a, b, r in tr).values())
    te = []
    for u in range(0, n_users, 2):
        for i in rng.choice(n_items + 15, size=4, replace=False):                    # items >= n_items: test-only
            te.append(("u%d" % u, "i%d" % i, float(rng.randint(1, 6))))
    te += [("new%d" % u, "i%d" % rng.randint(n_items), 4.0) for u in range(6)]       # test-only users
    uid_map, iid_map = OrderedDict(), OrderedDict()
    train = Dataset.build(tr, global_uid_map=uid_map, global_iid_map=iid_map, seed=123)
    test = Dataset.build(te, global_uid_map=uid_map, global_iid_map=iid_map, seed=123, exclude_unknowns=False)
    assert train.num_users == n_users and train.num_items == n_items
    assert len(uid_map) > n_users and len(iid_map) > n_items
    users = ["u%d" % u for u in range(n_users)]
    items = ["i%d" % i for i in range(n_items)]
    ugm = GraphModality(data=[(users[a], users[b], 1.0) for a, b in rng.randint(n_users, size=(600, 2)) if a != b])
    ugm.build(id_map=train.uid_map)
    igm = GraphModality(data=[(items[a], items[b], float(rng.randint(1, 4)))
                              for a, b in rng.randint(n_items, size=(500, 2)) if a != b])
    igm.build(id_map=train.iid_map)
    train.add_modalities(user_graph=ugm, item_graph=igm)
    return train, test, rng


def _model(name):
    import cornac_b200 as cb
    if name in ("BPR", "WBPR", "MMMF", "VEBPR", "SBPR"):
        return getattr(cb, name)(k=8, max_iter=5, learning_rate=0.05, seed=1)
    return dict(MF=lambda: cb.MF(k=8, max_iter=5, seed=1),
                NMF=lambda: cb.NMF(k=8, max_iter=5, use_bias=True, seed=1),
                WMF=lambda: cb.WMF(k=8, max_iter=3, verbose=False, seed=1),
                BaselineOnly=lambda: cb.BaselineOnly(max_iter=5, seed=1),
                PMF=lambda: cb.PMF(k=5, max_iter=10, seed=1),
                HPF=lambda: cb.HPF(k=5, max_iter=10, seed=1),
                PF=lambda: cb.HPF(k=5, max_iter=10, hierarchical=False, seed=1),
                EASE=lambda: cb.EASE(verbose=False),
                SoRec=lambda: cb.SoRec(k=5, max_iter=10, seed=1),
                MCF=lambda: cb.MCF(k=5, max_iter=10, seed=1),
                UserKNN=lambda: cb.UserKNN(k=10, verbose=False),
                ItemKNN=lambda: cb.ItemKNN(k=10, verbose=False))[name]()


def _fit(name, train):
    m = _model(name)
    if name == "VEBPR":
        import scipy.sparse as sp
        from cornac.data import PurchaseViewDataset
        rng = np.random.RandomState(9)
        W = sp.random(train.num_users, train.num_items, density=0.05, format="csr", random_state=rng, dtype=np.float32)
        W.data[:] = 1
        train = PurchaseViewDataset(train, W)
    return m.fit(train)


def _row(m, name, u):
    """score(u) as Recommender.rank reads it, in the dtype rank() orders."""
    from cornac.exception import ScoreException
    dtype = np.float32 if name in F32 else np.float64
    try:
        return np.asarray(m.score(u), dtype=dtype).ravel()
    except ScoreException:
        return np.full(m.total_items, m.default_score(), dtype=dtype)


def _want(m, name, u, cand, k):
    """The host restatement of rank(u, cand, k)."""
    from cornac.models.recommender import Recommender
    if name in ("SoRec", "MCF"):
        return Recommender.rank(m, u, cand, k)
    row = _row(m, name, u)
    if len(row) < m.total_items:
        full = np.full(m.total_items, row.min(), dtype=row.dtype)
        full[: len(row)] = row
        row = full
    cand = np.arange(m.num_items) if cand is None else np.asarray(cand)
    sc = row[cand]
    order = np.lexsort((cand, -sc.astype(np.float64)))
    if name in ("UserKNN", "ItemKNN") or k == -1 or k >= len(cand) or k > 4096:
        return cand[order], sc
    top = cand[order[:k]]
    return np.concatenate([top, cand[~np.isin(cand, top)]]), sc


def _call(f, *args):
    """f(*args), or the type of the ValueError it raises (Recommender.rank rejects k > len(candidates))."""
    try:
        return f(*args)
    except ValueError as e:
        return type(e)


def _same(got, want):
    if isinstance(want, type) or isinstance(got, type):
        assert got is want
        return
    assert np.array_equal(got[0], want[0]) and got[1].dtype == want[1].dtype and np.array_equal(got[1], want[1])


def _calls(m, users, rng, n_total):
    """(user, candidates, k) cases: no candidates, a sorted subset, an unsorted subset with test-only items."""
    out = []
    for u in users:
        for cand in (None, np.sort(rng.choice(m.num_items, size=70, replace=False)),
                     rng.choice(n_total, size=90, replace=False)):
            n = m.num_items if cand is None else len(cand)
            out += [(u, cand, n if k is None else k) for k in KS]
    return out


@pytest.mark.parametrize("name", NAMES)
def test_rank_score_and_transform_follow_the_contract(name, tmp_path):
    from cornac.models.recommender import Recommender
    from cornac_b200 import engine
    train, test, rng = _data()
    m = _fit(name, train)
    n_total = m.total_items
    known = [u for u in sorted(set(test.uir_tuple[0])) if u < m.num_users][:12]
    calls = _calls(m, known, rng, n_total)

    # known users, uncached
    cold = [_call(m.rank, u, cand, k) for u, cand, k in calls]
    for (u, cand, k), got in zip(calls, cold):
        _same(got, _call(_want, m, name, u, cand, k))
    rows = {u: m.score(u) for u in known}

    # test-only users and a user past every row: sorted candidates (for a row of equal scores the order of an
    # unsorted tail is not part of the contract)
    for u in (m.num_users, m.total_users):
        if name in ROW_BEYOND_RAISES and u >= m.total_users:
            with pytest.raises(IndexError):
                m.rank(u, None, 10)
            with pytest.raises(IndexError):
                m.score(u)
            continue
        for cand in (None, np.sort(rng.choice(n_total, size=60, replace=False))):
            for k in (1, 10, -1):
                _same(m.rank(u, cand, k), _want(m, name, u, cand, k))

    # the transform() cache: identical answers, and no kernel for a cached user
    m.transform(test)
    if name == "BaselineOnly":
        assert m._b200_eval_cache is None
    else:
        assert m._b200_eval_cache is not None
        L = engine.require_cuda()
        launches = L.b200_kernel_launches()
        warm = [_call(m.rank, u, cand, k) for u, cand, k in calls]
        for u in known:
            assert np.array_equal(m.score(u), rows[u]) and m.score(u).dtype == rows[u].dtype
        assert L.b200_kernel_launches() == launches
        for a, b in zip(cold, warm):
            _same(b, a)

    # batched entry points
    if name in ("UserKNN", "ItemKNN"):
        assert not hasattr(m, "rank_batch") and not hasattr(m, "recommend_batch")
    else:
        excl = train.csr_matrix
        for k in (1, 10):
            ids, sc = m.rank_batch(np.asarray(known), k, exclude=excl)
            for q, u in enumerate(known):
                row = _row(m, name, u)
                cand = np.setdiff1d(np.arange(len(row)), excl[u].indices)
                want = cand[np.lexsort((cand, -row[cand].astype(np.float64)))[:k]]
                if name == "BaselineOnly":              # device f32 sums against the host row: equal up to rounding
                    assert np.allclose(row[ids[q]], row[want], rtol=1e-6, atol=1e-6)
                    continue
                assert np.array_equal(ids[q], want), (u, k, ids[q], want)
                if name in F32:
                    assert np.allclose(sc[q], row[want], rtol=1e-6, atol=1e-6)
                else:
                    assert np.array_equal(sc[q], row[want])
        uids = [m.user_ids[u] for u in known]
        for remove_seen in (False, True):
            got = m.recommend_batch(uids, k=10, remove_seen=remove_seen, train_set=train)
            want = [list(m.recommend(uid, k=10, remove_seen=remove_seen, train_set=train)) for uid in uids]
            if name == "BaselineOnly":
                for u, a, b in zip(known, got, want):
                    row = _row(m, name, u)
                    assert np.allclose(row[[m.iid_map[i] for i in a]], row[[m.iid_map[i] for i in b]], rtol=1e-6, atol=1e-6)
            else:
                assert got == want

    # save / load
    loaded = Recommender.load(m.save(str(tmp_path / name)))
    assert getattr(loaded, "_b200_dev", None) is None
    for u, cand, k in calls[:15]:
        _same(_call(loaded.rank, u, cand, k), _call(m.rank, u, cand, k))
    assert np.array_equal(loaded.score(known[0]), rows[known[0]])
