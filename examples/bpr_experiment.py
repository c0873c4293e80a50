"""cornac.Experiment with the GPU plug-ins next to the reference models (needs a GPU + the cornac package).

    python examples/bpr_experiment.py

The reference's own example (examples/bpr_netflix.py) downloads a data set; there is no network here, so the
script builds a MovieLens-100K-shaped synthetic rating list (943 users x 1682 items x 100K ratings, BASELINE.json
configs[0]) and runs BPR / WBPR / MF from both implementations through the SAME unchanged cornac pipeline.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ref = os.path.join(ROOT, "oracle", "_ref")
if os.path.isdir(os.path.join(ref, "cornac")):
    sys.path.insert(0, ref)

import cornac  # noqa: E402
from cornac.eval_methods import RatioSplit  # noqa: E402
from cornac.metrics import AUC, MAP, NDCG, Precision, Recall  # noqa: E402

import cornac_b200  # noqa: E402


def ml100k_like(seed=123):
    rng = np.random.RandomState(seed)
    n_users, n_items, nnz = 943, 1682, 100_000
    taste = rng.normal(0, 1, (n_users, 8))
    style = rng.normal(0, 1, (n_items, 8))
    pop = 1.0 / np.arange(1, n_items + 1) ** 0.9
    pairs = set()
    while len(pairs) < nnz:
        u = rng.randint(n_users, size=nnz)
        i = rng.choice(n_items, size=nnz, p=pop / pop.sum())
        for a, b in zip(u, i):
            if len(pairs) < nnz:
                pairs.add((int(a), int(b)))
    data = []
    for u, i in sorted(pairs):
        r = 3.0 + 0.8 * float(taste[u] @ style[i]) / np.sqrt(8) + rng.normal(0, 0.5)
        data.append((str(u), str(i), float(np.clip(np.rint(r), 1, 5))))
    rng.shuffle(data)
    return data


if __name__ == "__main__":
    # CUDA context + library load happen here, not inside the first GPU model's fit(): Train (s) then compares training
    cornac_b200.engine.warmup()
    rs = RatioSplit(data=ml100k_like(), test_size=0.2, rating_threshold=4.0, exclude_unknowns=True, seed=123, verbose=True)
    models = [
        cornac.models.BPR(k=10, max_iter=200, learning_rate=0.001, lambda_reg=0.01, seed=123, name="BPR (reference, seeded)"),
        cornac_b200.BPR(k=10, max_iter=200, learning_rate=0.001, lambda_reg=0.01, seed=123, name="BPR (GPU, seeded replay)"),
        cornac_b200.BPR(k=10, max_iter=200, learning_rate=0.001, lambda_reg=0.01, name="BPR (GPU, Hogwild)"),
        cornac_b200.WBPR(k=10, max_iter=200, learning_rate=0.001, lambda_reg=0.01, name="WBPR (GPU, Hogwild)"),
        cornac.models.MF(k=10, max_iter=25, learning_rate=0.01, lambda_reg=0.02, use_bias=True, seed=123, name="MF (reference, seeded)"),
        cornac_b200.MF(k=10, max_iter=25, learning_rate=0.01, lambda_reg=0.02, use_bias=True, seed=123, name="MF (GPU, ordered)"),
    ]
    metrics = [AUC(), MAP(), NDCG(k=10), Precision(k=10), Recall(k=10)]
    cornac.Experiment(eval_method=rs, models=models, metrics=metrics, user_based=True).run()
