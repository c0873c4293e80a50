"""NMF on the GPU: b200_nmf_fit bit-identical to the compiled reference's fixtures and to the serial oracle (both use_bias
modes, shared-memory and global bias paths, several k), and the plug-in through init_params, scores, ranking, save /
load and an unchanged Experiment."""
import tempfile

import numpy as np
import pytest
import torch

from conftest import golden, needs_cornac, synth_csr
from oracle import nmf_oracle as NO

pytestmark = pytest.mark.gpu

FIT_CASES = ["nmf_default_k15", "nmf_bias_k10", "nmf_lambda_reg_k8", "nmf_init_u_bi_k6", "nmf_k1", "nmf_bias_k1",
             "nmf_mid_k12"]


def device_fit(indptr, indices, val, init, n_epochs, use_bias, split=None, **hyper):
    from cornac_b200 import engine
    data = engine.NmfData(indptr, indices, val, init[1].shape[0], use_bias)
    d = [engine.to_device(np.ascontiguousarray(a), torch.float32) for a in init]
    if split is None:
        engine.nmf_fit(data, *d, n_epochs, **hyper)
    else:                                                     # two calls of a and b epochs == one call of a + b
        engine.nmf_fit(data, *d, split, **hyper)
        engine.nmf_fit(data, *d, n_epochs - split, **hyper)
    return [t.cpu().numpy() for t in d]


def _hyper(g):
    return dict(mu=float(g["mu"]), learning_rate=float(g["learning_rate"]), lambda_u=float(g["lambda_u"]),
                lambda_v=float(g["lambda_v"]), lambda_bu=float(g["lambda_bu"]), lambda_bi=float(g["lambda_bi"]))


def _oracle(indptr, indices, val, init, n_epochs, use_bias, **h):
    out = [a.copy() for a in init]
    NO.nmf_fit(indptr, indices, val, *out, n_epochs, mu=h["mu"], lr=h["learning_rate"], lambda_u=h["lambda_u"],
               lambda_v=h["lambda_v"], lambda_bu=h["lambda_bu"], lambda_bi=h["lambda_bi"], use_bias=use_bias)
    return out


def _dataset(u, i, r):
    from cornac.data import Dataset
    return Dataset.from_uir([(str(a), str(b), float(c)) for a, b, c in zip(u, i, r)], seed=None)


@pytest.mark.parametrize("split", [None, 3])
@pytest.mark.parametrize("name", FIT_CASES)
def test_fit_is_bit_identical_to_the_reference(name, split):
    g = golden(name)
    init = [g[x] for x in ("U0", "V0", "Bu0", "Bi0")]
    got = device_fit(g["indptr"], g["indices"], g["data"], init, int(g["max_iter"]), bool(g["use_bias"]), split=split,
                     **_hyper(g))
    for a, key in zip(got, ("U", "V", "Bu", "Bi")):
        assert np.array_equal(a, g[key]), key


def _synth(n_users, n_items, nnz, k, seed):
    indptr, indices = synth_csr(n_users, n_items, nnz, seed=seed)
    rng = np.random.RandomState(seed)
    val = rng.randint(1, 6, size=len(indices)).astype(np.float32)
    init = [rng.uniform(0, 1, (n_users, k)).astype(np.float32), rng.uniform(0, 1, (n_items, k)).astype(np.float32),
            np.zeros(n_users, np.float32), np.zeros(n_items, np.float32)]
    return indptr, indices, val, init


HYPER = dict(learning_rate=0.005, lambda_u=0.06, lambda_v=0.06, lambda_bu=0.02, lambda_bi=0.02)


@pytest.mark.parametrize("use_bias", [False, True])
def test_ml1m_shape_is_bit_identical_to_the_oracle(use_bias):
    indptr, indices, val, init = _synth(6040, 3706, 1000000, 15, 3)
    h = dict(HYPER, mu=float(np.float32(val.mean())) if use_bias else 0.0)
    got = device_fit(indptr, indices, val, init, 3, use_bias, **h)
    want = _oracle(indptr, indices, val, init, 3, use_bias, **h)
    for a, b, key in zip(got, want, ("U", "V", "Bu", "Bi")):
        assert np.array_equal(a, b), key


@pytest.mark.parametrize("use_bias", [False, True])
def test_biases_beyond_shared_memory_are_bit_identical_to_the_oracle(use_bias):
    """70 000 users + 5 000 items: 300 KB of biases, more than a CTA's shared memory holds (the global-memory path)."""
    indptr, indices, val, init = _synth(70000, 5000, 600000, 15, 4)
    rng = np.random.RandomState(9)
    init[2], init[3] = rng.normal(0, 0.1, 70000).astype(np.float32), rng.normal(0, 0.1, 5000).astype(np.float32)
    h = dict(HYPER, mu=3.0 if use_bias else 0.0)
    got = device_fit(indptr, indices, val, init, 2, use_bias, **h)
    want = _oracle(indptr, indices, val, init, 2, use_bias, **h)
    for a, b, key in zip(got, want, ("U", "V", "Bu", "Bi")):
        assert np.array_equal(a, b), key


@pytest.mark.parametrize("use_bias", [False, True])
@pytest.mark.parametrize("k", [1, 20, 64, 130])
def test_factor_widths_are_bit_identical_to_the_oracle(k, use_bias):
    indptr, indices, val, init = _synth(400, 300, 12000, k, k)
    h = dict(HYPER, mu=3.0 if use_bias else 0.0)
    got = device_fit(indptr, indices, val, init, 4, use_bias, **h)
    want = _oracle(indptr, indices, val, init, 4, use_bias, **h)
    for a, b, key in zip(got, want, ("U", "V", "Bu", "Bi")):
        assert np.array_equal(a, b), key


def test_loss_output_and_bad_arguments():
    from cornac_b200 import engine
    from cornac_b200._lib import B200Error
    indptr, indices, val, init = _synth(300, 200, 6000, 8, 5)
    data = engine.NmfData(indptr, indices, val, 200, True)
    d = [engine.to_device(a, torch.float32) for a in init]
    loss = torch.zeros(3, dtype=torch.float64, device="cuda")
    engine.nmf_fit(data, *d, 3, mu=3.0, loss=loss, **HYPER)
    # epoch 0's loss from the initial parameters: sum err^2 + lambda_u |U0|^2 + lambda_v |V0|^2
    U0, V0 = init[0].astype(np.float64), init[1].astype(np.float64)
    assert float(loss[0]) > 0 and np.isfinite(loss.cpu().numpy()).all()
    assert float(loss[0]) > 0.06 * (np.sum(U0 * U0) + np.sum(V0 * V0))
    with pytest.raises(B200Error, match="outside"):
        engine.NmfData(np.array([0, 1]), np.array([7]), np.ones(1), 3, False)
    with pytest.raises(B200Error, match="shape"):
        engine.nmf_fit(data, d[1], d[0], d[2], d[3], 1)


@needs_cornac
@pytest.mark.parametrize("name", ["nmf_default_k15", "nmf_bias_k10", "nmf_lambda_reg_k8", "nmf_k1"])
def test_plugin_fit_and_scores_match_the_reference(name):
    from cornac_b200 import NMF
    g = golden(name)
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    kw = dict(k=int(g["k"]), max_iter=int(g["max_iter"]), learning_rate=float(g["learning_rate"]),
              lambda_reg=float(g["lambda_reg"]), use_bias=bool(g["use_bias"]), seed=int(g["seed"]))
    if float(g["lambda_reg"]) <= 0:
        kw.update(lambda_u=float(g["lambda_u"]), lambda_v=float(g["lambda_v"]), lambda_bu=float(g["lambda_bu"]),
                  lambda_bi=float(g["lambda_bi"]))
    m = NMF(**kw).fit(ds)
    for a, key in ((m.u_factors, "U"), (m.i_factors, "V"), (m.u_biases, "Bu"), (m.i_biases, "Bi")):
        assert np.array_equal(a, g[key]), key
    single = np.array([m.score(int(u), int(i)) for u, i in g["single_pairs"]])
    assert single.dtype == g["single_scores"].dtype and np.array_equal(single, g["single_scores"])


@needs_cornac
def test_init_params_are_trained_in_place_and_f64_is_refused():
    from cornac_b200 import NMF
    g = golden("nmf_init_u_bi_k6")
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    U, Bi = g["U0"].copy(), g["Bi0"].copy()
    m = NMF(k=6, max_iter=int(g["max_iter"]), seed=int(g["seed"]), init_params={"U": U, "Bi": Bi}).fit(ds)
    assert m.u_factors is U and np.array_equal(U, g["U"]) and np.array_equal(m.i_factors, g["V"])
    assert m.i_biases is Bi and np.array_equal(Bi, g["Bi"])
    with pytest.raises(ValueError, match="Buffer dtype mismatch, expected 'float' but got 'double'"):
        NMF(k=6, max_iter=1, init_params={"U": g["U0"].astype(np.float64)}).fit(ds)
    m = NMF(k=6, trainable=False, init_params={"U": U, "V": g["V"]}).fit(ds)
    assert m.u_factors is U and m.global_mean == 0.0


@needs_cornac
@pytest.mark.parametrize("use_bias", [False, True])
def test_scores_and_rank_follow_the_device_row(use_bias):
    from cornac_b200 import NMF
    from oracle import oracle as O
    g = golden("nmf_mid_k12")
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    m = NMF(k=12, max_iter=5, seed=1, use_bias=use_bias).fit(ds)
    base = (m.global_mean + m.i_biases).astype(np.float32)
    users = np.array([0, 17, ds.num_users - 1])
    want = O.score_batch(m.u_factors[users], m.i_factors, base, m.u_biases[users])
    n = ds.num_items
    rng = np.random.RandomState(0)
    for cached in (False, True):
        if cached:
            m.transform(ds)
        for q, u in enumerate(users):
            row = m.score(int(u))
            assert row.dtype == np.float32 and np.array_equal(row, want[q])
            full = np.lexsort((np.arange(n), -row.astype(np.float64)))
            ranked, sc = m.rank(int(u))
            assert np.array_equal(ranked, full) and np.array_equal(sc, row)
            ranked, _ = m.rank(int(u), k=10)
            assert np.array_equal(ranked[:10], full[:10]) and np.array_equal(np.sort(ranked), np.arange(n))
            cand = np.sort(rng.choice(n, size=50, replace=False))
            ranked, sc = m.rank(int(u), cand, k=5)
            w = cand[np.lexsort((cand, -row[cand].astype(np.float64)))]
            assert np.array_equal(ranked[:5], w[:5]) and np.array_equal(np.sort(ranked), cand)
    ranked, sc = m.rank(ds.num_users + 3, k=5)                 # unknown user: the base row
    assert np.array_equal(sc, (m.global_mean + m.i_biases)[np.arange(n)].astype(np.float32))
    batch = np.arange(0, ds.num_users, 7)
    ids, top = m.rank_batch(batch, 20, exclude=ds.csr_matrix)
    for q, u in enumerate(batch):
        row = m.score(int(u))
        cand = np.setdiff1d(np.arange(n), ds.csr_matrix[u].indices)
        w = cand[np.lexsort((cand, -row[cand].astype(np.float64)))][:20]
        assert np.array_equal(ids[q], w) and np.array_equal(top[q], row[w])
    recs = m.recommend_batch([ds.user_ids[0], ds.user_ids[3]], k=5, remove_seen=True, train_set=ds)
    assert recs == [m.recommend(ds.user_ids[0], k=5, remove_seen=True, train_set=ds)[:5],
                    m.recommend(ds.user_ids[3], k=5, remove_seen=True, train_set=ds)[:5]]


@needs_cornac
def test_save_load_round_trip():
    from cornac_b200 import NMF
    g = golden("nmf_bias_k10")
    ds = _dataset(g["uir_u"], g["uir_i"], g["uir_r"])
    m = NMF(k=10, max_iter=10, use_bias=True, seed=2).fit(ds)
    with tempfile.TemporaryDirectory() as d:
        path = m.save(d)
        m2 = NMF.load(path)
    for attr in ("u_factors", "i_factors", "u_biases", "i_biases"):
        assert np.array_equal(getattr(m2, attr), getattr(m, attr))
    assert m2.global_mean == m.global_mean
    assert np.array_equal(m2.score(3), m.score(3)) and m2.score(3, 4) == m.score(3, 4)
    assert np.array_equal(m2.rank(3, k=10)[0][:10], m.rank(3, k=10)[0][:10])


@needs_cornac
def test_experiment_metrics_equal_the_reference():
    import cornac
    import cornac_b200
    from cornac.eval_methods import RatioSplit
    from cornac.eval_methods.base_method import ranking_eval as ref_ranking_eval
    from cornac.metrics import AUC, MAE, NDCG, RMSE, Precision, Recall
    from cornac_b200.evaluation import ranking_eval
    g = golden("nmf_experiment")
    data = [(str(a), str(b), float(c)) for a, b, c in zip(g["uir_u"], g["uir_i"], g["uir_r"])]
    rs = RatioSplit(data=data, test_size=0.2, rating_threshold=4.0, exclude_unknowns=True, seed=123, verbose=False)
    hyper = dict(k=15, max_iter=50, learning_rate=0.005, lambda_u=0.06, lambda_v=0.06, lambda_bu=0.02, lambda_bi=0.02,
                 seed=123)
    metrics = [MAE(), RMSE(), Recall(k=20), Precision(k=20), NDCG(), AUC()]
    model = cornac_b200.NMF(use_bias=False, **hyper)
    exp = cornac.Experiment(eval_method=rs, models=[model], metrics=metrics, user_based=True, verbose=False)
    exp.run()
    res = exp.result[0].metric_avg_results
    names = [str(n) for n in g["metric_names"]]
    got = np.array([res[n] for n in names])
    assert np.array_equal(got[:2], g["plain"][:2])                      # MAE, RMSE: exactly
    # NDCG over the full list depends on the order of tied scores: NMF drives many item rows to exact zeros, and the
    # reference orders ties by numpy's unstable argsort while the plug-in orders them by item id
    top = [j for j, n in enumerate(names) if not n.startswith("NDCG")]
    assert np.all(np.abs(got[top] - g["plain"][top]) <= 1e-12), dict(zip(names, got))
    ranking = [Recall(k=20), Precision(k=20), NDCG(k=20), AUC()]
    mine, _ = ranking_eval(model, ranking, rs.train_set, rs.test_set, rating_threshold=4.0, exclude_unknowns=True)
    ref, _ = ref_ranking_eval(model, ranking, rs.train_set, rs.test_set, rating_threshold=4.0, exclude_unknowns=True)
    assert np.all(np.abs(np.array(mine) - np.array(ref)) <= 1e-12)
    exp = cornac.Experiment(eval_method=rs, models=[cornac_b200.NMF(use_bias=True, **hyper)], metrics=[MAE(), RMSE()],
                            user_based=True, verbose=False)
    exp.run()
    res = exp.result[0].metric_avg_results
    assert np.array_equal(np.array([res[str(n)] for n in g["bias_metric_names"]]), g["bias"])
