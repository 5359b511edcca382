"""The BiLSTM recurrence (csrc/lstm.cu) writes exactly the bytes recorded in tests/golden/lstm_digest.json
(tests/golden/make_lstm_digest.py), follows the float64 oracle, and gives the same bytes replayed in a CUDA graph as launched eagerly."""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

pytestmark = pytest.mark.gpu


def _rel_err(case, y):
    import make_lstm_digest as M
    ref = M.oracle(case)
    return float((M.result(case, y).double().cpu() - ref).abs().max() / ref.abs().max())


def test_lstm_matches_the_recorded_digests():
    import make_lstm_digest as M
    with open(M.OUT) as f:
        want = json.load(f)
    assert [w["case"] for w in want] == [M.label(c) for c in M.CASES]
    bad = []
    for case, w in zip(M.CASES, want):
        y = M.run(case)
        if M.digest(y) != w["sha256"]:
            bad.append(f"{w['case']} (max error vs float64 relative to max |h|: {_rel_err(case, y):.2e})")
    assert not bad, f"{len(bad)} of {len(want)} cases changed their output bytes: {bad}"


@pytest.mark.parametrize("index", range(7))
def test_lstm_follows_the_float64_oracle(index):
    import make_lstm_digest as M
    case = M.CASES[index]
    y = M.run(case)
    assert _rel_err(case, y) < 5e-6          # fp32 with SFU exp / division: ~4e-7 measured
    if case[2] is not None:                 # nothing outside the column slice is written
        sl = case[2]
        outside = y.clone()
        outside[:, :, sl[1]:sl[1] + 2 * M.H] = -7.0
        assert bool((outside == -7.0).all())


@pytest.mark.parametrize("B", [1, 2])
def test_lstm_graph_replay_matches_eager(B):
    import torch
    import make_lstm_digest as M
    from mlx_audio_b200 import ops
    xproj, wh = M.inputs((B, 130, None))
    xproj, wh = xproj.cuda(), wh.cuda().contiguous()
    eager = ops.lstm_bidir(xproj, wh).clone()
    out = torch.full_like(eager, float("nan"))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.lstm_bidir(xproj, wh, out=out)                      # warm-up outside the capture
        s.synchronize()
        out.fill_(float("nan"))
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.lstm_bidir(xproj, wh, out=out)
        out.fill_(float("nan"))
        g.replay()
        g.replay()
    s.synchronize()
    assert torch.equal(out, eager)
