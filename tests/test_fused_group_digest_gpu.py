"""The fused conv kernel's generator-group launches at the benchmarked Kokoro shape write exactly the bytes recorded in
tests/golden/fused_group_digest.json (tests/golden/make_fused_group_digest.py): outputs and statistics of all 12 launches."""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))


@pytest.mark.gpu
def test_generator_groups_match_the_recorded_digests():
    from make_fused_group_digest import OUT, generator_group_digests
    with open(OUT) as f:
        want = json.load(f)
    got = generator_group_digests()
    assert [g["launch"] for g in got] == [w["launch"] for w in want]
    bad = [g["launch"] for g, w in zip(got, want) if g["sha256"] != w["sha256"]]
    assert not bad, f"{len(bad)} of {len(want)} generator-group launches changed their output bytes: {bad}"
