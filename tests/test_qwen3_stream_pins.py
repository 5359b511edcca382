"""Qwen3-TTS streaming protocol pinned to the reference's own code: tests/golden/qwen3_stream_golden.npz holds the events of the reference's
``Model.generate(stream=True)`` (custom-voice and base paths, incremental decoder), executed through the NumPy stand-in by
tests/golden/make_qwen3_stream_golden.py.  ``oracle.qwen3_stream.generate_stream`` must reproduce every event: frames, token counts,
sample counts, flags and segment index identical, audio to float32 storage precision."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(HERE))
FIXTURE = "qwen3_stream_golden.npz"
WTOL = 2e-7                                        # waveforms are stored as float32 in the fixture

IDS = dict(codec_nothink_id=1004, codec_think_id=1003, codec_think_bos_id=1005, codec_think_eos_id=1006, codec_pad_id=1001, codec_bos_id=1002)
LANG, SPK = {"english": 1010, "german": 1011}, {"amy": 1020, "bob": 1021}


def _load():
    if HERE not in sys.path:
        sys.path.insert(0, HERE)
    import synth_params
    g = np.load(os.path.join(HERE, FIXTURE), allow_pickle=False)
    P = {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g["talker_params"]).items()}
    PT = {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g["tok_params"]).items()}
    return g, P, PT, json.loads(str(g["cfg"])), json.loads(str(g["tok_cfg"]))


@pytest.mark.parametrize("tag", ["cv_exact", "cv_rem", "cv_one", "base_two"])
def test_oracle_stream_events_match_the_reference_generate(tag):
    from oracle import qwen3 as Q
    from oracle import qwen3_stream as QS
    g, P, PT, cfg, tcfg = _load()
    m = json.loads(str(g[f"{tag}_meta"]))
    u = torch.as_tensor(g[f"{tag}_u"])
    mt = m["max_tokens"]
    want = []
    for idx, text_ids in enumerate(m["text_ids"]):
        spk = SPK[m["voice"]] if m["voice"] else None
        ie, tr, pad = Q.prepare_generation_inputs_from_ids(P, text_ids, (112, 113, 111), IDS, LANG.get(m["lang_code"]), spk)
        want += QS.generate_stream(P, PT, ie, tr, pad, u[idx * mt:(idx + 1) * mt], mt, m["interval"], cfg=cfg, tcfg=tcfg,
                                   segment_idx=idx if m["kind"] == "base" else 0)
    ev = g[f"{tag}_events"]
    assert len(want) == ev.shape[0]
    got = np.array([[e["token_count"], e["samples"], int(e["is_streaming_chunk"]), int(e["is_final_chunk"]), e["segment_idx"]] for e in want])
    assert np.array_equal(got, ev)
    for i, e in enumerate(want):
        assert np.array_equal(e["codes"].T[None].numpy(), g[f"{tag}_ev{i}_codes"]), i
        assert np.abs(e["audio"].numpy() - g[f"{tag}_ev{i}_audio"]).max() < WTOL, i
    if tag == "cv_exact":                          # frame count a multiple of the chunk size: no final event at all
        assert not ev[:, 3].any()
    if tag == "base_two":
        assert ev[:, 4].tolist() == [0, 0, 1, 1] and ev[:, 3].tolist() == [0, 1, 0, 1]


@pytest.mark.skipif(not os.path.isdir("/root/reference/mlx_audio"), reason="the reference source is only present in the build container")
def test_stream_fixture_is_what_the_reference_code_produces(tmp_path):
    env = dict(os.environ, GOLDEN_OUT=str(tmp_path), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(HERE, "make_qwen3_stream_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    new, old = np.load(tmp_path / FIXTURE), np.load(os.path.join(HERE, FIXTURE))
    assert sorted(new.files) == sorted(old.files)
    for k in old.files:
        a, b = new[k], old[k]
        assert a.dtype == b.dtype and a.shape == b.shape, k
        if a.dtype.kind == "f":
            assert np.abs(a - b).max(initial=0.0) <= 1e-12 * max(1.0, float(np.abs(b).max(initial=0.0))), k
        else:
            assert np.array_equal(a, b), k
