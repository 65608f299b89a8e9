"""Window planning / stitching of jukebox_b200.sample against the UNMODIFIED reference's own loop
(jukebox/sample.py:17-96), both driven with the same recording dummy prior on the CPU.  The reference's results
are stored in tests/golden/sample_level.json (oracle/make_golden_sample_plan.py)."""
import itertools
import json
import os

import pytest

from golden_util import GOLDEN
from oracle.make_golden_sample_plan import CASES, case_key, run_case
from jukebox_b200.sample import plan_windows, Window
from jukebox_b200.utils.sample_utils import get_starts

with open(os.path.join(GOLDEN, "sample_level.json")) as _f:
    REF = json.load(_f)


@pytest.mark.parametrize("total,n_ctx,hop,have,bs,mbs", CASES)
def test_sample_level_matches_reference(total, n_ctx, hop, have, bs, mbs):
    import jukebox_b200.sample as ours
    if total >= n_ctx and have > total:
        pytest.skip("more tokens than the level holds")
    case = (total, n_ctx, hop, have, bs, mbs)
    ref = REF[case_key(case)]
    got = json.loads(json.dumps(run_case(ours.sample_level, case)))     # tuples -> lists, as stored
    if "error" in ref:
        assert "error" in got, got
        return
    assert "error" not in got, got
    assert got["codes"] == ref["codes"]
    assert got["calls"] == ref["calls"]


def test_plan_windows_shapes():
    assert plan_windows(0, 40, 16, 8) == [Window(s, 16) for s in get_starts(40, 16, 8)]
    assert plan_windows(0, 10, 16, 8) == [Window(0, 10)]
    assert plan_windows(12, 10, 16, 8) == [Window(6, 16)]
    for total, n_ctx, hop in itertools.product((16, 17, 31, 64), (16,), (4, 8, 16)):
        wins = plan_windows(0, total, n_ctx, hop)
        assert wins[0].start == 0 and wins[-1].start + n_ctx == total
        assert all(b.start - a.start <= hop for a, b in zip(wins, wins[1:]))
