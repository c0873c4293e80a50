"""Batched, device-side evaluation and recommendation with the GPU plug-ins (needs a GPU + the cornac package).

    python examples/batched_eval.py

`cornac.Experiment` calls `model.rank()` once per test user from a Python loop.  The plug-ins also offer the batched
forms that loop has no use for:
  * `model.rank_batch(users, k, exclude=csr)`            top-k ids + scores of many users in one fused kernel call
  * `cornac_b200.evaluation.ranking_eval(...)`            drop-in for cornac.eval_methods.base_method.ranking_eval: every
                                                          test user ranked at once, @k metrics reduced on the GPU
Both return exactly what the per-user reference path returns (same ids, same metric values).
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))
ref = os.path.join(ROOT, "oracle", "_ref")
if os.path.isdir(os.path.join(ref, "cornac")):
    sys.path.insert(0, ref)

import numpy as np  # noqa: E402
from cornac.eval_methods import RatioSplit  # noqa: E402
from cornac.eval_methods.base_method import ranking_eval as reference_ranking_eval  # noqa: E402
from cornac.metrics import NDCG, Precision, Recall  # noqa: E402

import cornac_b200  # noqa: E402
from bpr_experiment import ml100k_like  # noqa: E402
from cornac_b200.evaluation import ranking_eval as batched_ranking_eval  # noqa: E402

if __name__ == "__main__":
    rs = RatioSplit(data=ml100k_like(), test_size=0.2, rating_threshold=4.0, exclude_unknowns=True, seed=123, verbose=False)
    model = cornac_b200.BPR(k=32, max_iter=50, learning_rate=0.05, lambda_reg=0.01).fit(rs.train_set)
    metrics = [NDCG(k=10), Precision(k=10), Recall(k=10), Recall(k=50)]

    t0 = time.perf_counter()
    ref_avg, _ = reference_ranking_eval(model, metrics, rs.train_set, rs.test_set, rating_threshold=4.0)
    t1 = time.perf_counter()
    b_avg, _ = batched_ranking_eval(model, metrics, rs.train_set, rs.test_set, rating_threshold=4.0)
    t2 = time.perf_counter()
    for m, a, b in zip(metrics, ref_avg, b_avg):
        print("%-14s per-user loop %.6f   batched %.6f" % (m.name, a, b))
    print("per-user loop %.2f s, batched %.3f s" % (t1 - t0, t2 - t1))

    # recommendations for every user at once, items seen in training removed
    users = np.arange(rs.train_set.num_users)
    ids, scores = model.rank_batch(users, 10, exclude=rs.train_set.csr_matrix)
    print("top-10 of user 0:", ids[0].tolist())
    assert ids[0].tolist() == [i for i in model.rank(0, k=rs.train_set.num_items)[0]
                               if i not in set(rs.train_set.csr_matrix[0].indices)][:10]
