"""The deterministic BPR epoch against committed digests of its output (tests/golden/bpr_det_digests.json, written by
tests/golden/make_golden_bpr_det.py).  The mode promises the same bytes for the same arguments, so every case must
reproduce U, V, B and the per-epoch counts exactly.  GPU only."""
import json
import os
import sys

import pytest

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import make_golden_bpr_det as M  # noqa: E402

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, "bpr_det_digests.json")) as _f:
    DIGESTS = json.load(_f)


def test_digest_file_covers_every_case():
    assert sorted(DIGESTS["cases"]) == sorted(c["name"] for c in M.CASES)
    assert DIGESTS["epochs"] == M.EPOCHS and DIGESTS["seed"] == M.SEED


@pytest.mark.parametrize("case", M.CASES, ids=[c["name"] for c in M.CASES])
def test_deterministic_epoch_matches_digest(case):
    got = M.run_case(case)
    want = DIGESTS["cases"][case["name"]]
    assert got["stats"] == want["stats"]
    for name in ("U", "V", "B"):
        assert got[name] == want[name], name
