"""Host half of the batched ranking_eval (cornac_b200/evaluation.py): the per-user tie counts of the positives that MAP
and AUC need, and the test-positives CSR, each against a brute-force restatement.  CPU only: no kernel is launched."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import needs_cornac

pytestmark = needs_cornac


def _evaluation():
    from cornac_b200 import evaluation
    return evaluation


def _brute_less(seg, score):
    """per entry: entries of the same segment with a strictly smaller score (float compare: -0.0 == +0.0)"""
    return np.array([int(np.sum((seg == g) & (score < s))) for g, s in zip(seg, score)], dtype=np.int64)


def _score_cases():
    rng = np.random.RandomState(7)
    levels = np.array([-np.inf, -1.5, -0.0, 0.0, 0.25, 2.0, np.inf], dtype=np.float32)
    cases = {
        "single": (np.array([3]), np.array([1.0], np.float32)),
        "all_tied": (np.zeros(9, np.int64), np.full(9, 0.5, np.float32)),
        "signed_zeros": (np.array([0, 0, 0, 1, 1, 2]), np.array([-0.0, 0.0, -0.0, 0.0, -0.0, -0.0], np.float32)),
        "infinities": (np.array([0, 0, 0, 0, 1, 1]), np.array([np.inf, -np.inf, np.inf, 1.0, -np.inf, -np.inf], np.float32)),
        # the largest score of one segment equals the smallest of the next: ties must not run across the boundary
        "boundary_ties": (np.array([0, 0, 1, 1, 2, 2]), np.array([1.0, 2.0, 2.0, 3.0, 3.0, 3.0], np.float32)),
        "length_one_segments": (np.arange(50)[::-1].copy(), rng.choice(levels, 50)),
    }
    seg = np.repeat(np.arange(300), rng.randint(1, 12, size=300))
    cases["quantised_sorted"] = (seg, rng.choice(levels, len(seg)))
    perm = rng.permutation(len(seg))
    cases["quantised_shuffled"] = (seg[perm], rng.choice(levels, len(seg)))
    cases["continuous"] = (seg[perm], rng.standard_normal(len(seg)).astype(np.float32))
    return cases


@pytest.mark.parametrize("name", sorted(_score_cases()))
def test_rank_within_segments_equals_a_brute_force_count(name):
    seg, score = _score_cases()[name]
    got = _evaluation()._rank_within_segments(seg, score)
    assert got.dtype == np.int64
    assert np.array_equal(got, _brute_less(seg, score)), name


def test_rank_within_segments_of_nothing_is_empty():
    got = _evaluation()._rank_within_segments(np.zeros(0, np.int64), np.zeros(0, np.float32))
    assert got.dtype == np.int64 and got.shape == (0,)


@pytest.mark.parametrize("threshold", [-1.0, 0.0, 1.0, 3.5, 4.0, 6.0])
@pytest.mark.parametrize("shape", [(40, 30), (25, 30), (40, 12), (13, 7), (60, 50)])
def test_positives_keeps_the_entries_at_the_threshold_inside_the_new_shape(threshold, shape):
    rng = np.random.RandomState(int(threshold * 10) + shape[0])
    keep = rng.rand(40, 30) < 0.4
    rows, cols = np.nonzero(keep)
    vals = rng.choice([0.0, 1.0, 2.5, 3.5, 4.0, 5.0], size=len(rows))       # 0.0: an explicitly stored zero rating
    mat = sp.csr_matrix((vals, (rows, cols)), shape=(40, 30))
    assert np.any(mat.data == 0.0)
    n_rows, n_cols = shape
    got = _evaluation()._positives(mat, threshold, n_rows, n_cols)
    assert got.shape == (n_rows, n_cols) and got.dtype == np.int8 and sp.isspmatrix_csr(got)
    want = np.zeros((n_rows, n_cols), dtype=np.int8)
    coo = mat.tocoo()
    for r, c, v in zip(coo.row, coo.col, coo.data):
        if v >= threshold and r < n_rows and c < n_cols:
            want[r, c] = 1
    assert np.array_equal(got.toarray(), want)
    assert np.all(got.data == 1)
