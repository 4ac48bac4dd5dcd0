"""The oracle's batch_objects closes batches at the dispatch limit exactly as batching.rs:194-209 does: tiny worlds against batch
tables worked out by hand (tests/batch_split_cases.py).  CPU only."""
import pytest

from rend3_b200.backend import CAMERA_VIEWPORT

from batch_split_cases import CASES, assert_same_tables, expected_tables, load
from oracle import load_oracle_backend


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_splits_batches_at_the_dispatch_limit(name):
    c = CASES[name]
    orc = load_oracle_backend()
    load(orc, c)
    got_b, got_r = orc.readback_batches(CAMERA_VIEWPORT)
    want_b, want_r = expected_tables(c)
    assert_same_tables(got_b, got_r, want_b, want_r, name)
    assert orc.batching_info(CAMERA_VIEWPORT)["batches"] == len(want_b)
