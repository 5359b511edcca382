"""Qwen3-TTS continuous-batching session pinned to the reference's own code: tests/golden/qwen3_session_golden.npz holds a staggered run of
the reference's ``Qwen3TTSBatchSession`` (admissions at different steps, a cancelled active row, rows ending on EOS, on max_tokens and on
their first frame), executed through the NumPy stand-in by tests/golden/make_qwen3_session_golden.py.  ``oracle.qwen3_session`` restates
that schedule over the single-sequence loop and must reproduce it: events and codes identical, audio to float32 storage precision.  The
same fixture pins the tts/continuous.py dataclasses and the supports_tts_batch / supports_tts_continuous_batch truth table."""
import dataclasses
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(HERE))
FIXTURE = "qwen3_session_golden.npz"
WTOL = 2e-7                                        # waveforms are stored as float32 in the fixture

IDS = dict(codec_nothink_id=1004, codec_think_id=1003, codec_think_bos_id=1005, codec_think_eos_id=1006, codec_pad_id=1001, codec_bos_id=1002)
SPK = {"amy": 1020, "bob": 1021}


def _load():
    if HERE not in sys.path:
        sys.path.insert(0, HERE)
    import synth_params
    g = np.load(os.path.join(HERE, FIXTURE), allow_pickle=False)
    P = {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g["talker_params"]).items()}
    PT = {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g["tok_params"]).items()}
    return g, P, PT, json.loads(str(g["cfg"])), json.loads(str(g["tok_cfg"]))


def test_oracle_session_schedule_matches_the_reference_session():
    from oracle import qwen3 as Q
    from oracle import qwen3_session as QS
    g, P, PT, cfg, tcfg = _load()
    P["codec_head.weight"] = P["codec_head.weight"].clone()
    P["codec_head.weight"][cfg["codec_eos_token_id"]] *= float(g["eos_gain"])
    m = json.loads(str(g["meta"]))
    us, mt = torch.as_tensor(g["u"]), m["max_tokens"]
    codes = {}
    for i, it in enumerate(m["items"]):
        ie, tr, pad = Q.prepare_generation_inputs_from_ids(P, m["text_ids"][i], (112, 113, 111), IDS, None, SPK[it["voice"]], m["instruct_ids"][i])
        codes[i] = Q.generate_codes(P, ie, tr, pad, us[i], mt, cfg=cfg)
    script = {int(k): [(kind, arg) for kind, arg in v] for k, v in m["script"].items()}
    events, cancelled = QS.run_schedule(codes, script, m["max_batch_size"], mt)
    ev = g["events"]
    assert [(s, i, n) for s, i, n in events] == [(int(r[0]), int(r[1]), int(r[3])) for r in ev]
    assert cancelled == {0: 5}
    for s, i, n in events:
        if n == 0:
            assert not any(k == f"codes_{i}" for k in g.files)
            continue
        assert np.array_equal(codes[i].numpy(), g[f"codes_{i}"]), i
        audio = Q.decode_generated_codes(PT, codes[i], tcfg).numpy()
        assert audio.shape[0] == int(ev[[r[1] for r in ev].index(i), 2]) and np.abs(audio - g[f"audio_{i}"]).max() < WTOL, i
    kinds = {n for _, _, n in events}
    assert 0 in kinds and mt in kinds and any(0 < n < mt for n in kinds)     # first-frame EOS, max_tokens and EOS are all exercised


def test_batch_types_and_support_hooks_match_the_reference():
    from mlx_audio.tts import continuous as CT
    from mlx_audio_b200.tts.models.qwen3_tts import Model
    g, _, _, _, _ = _load()
    want = json.loads(str(g["dataclasses"]))
    for cls in (CT.TTSBatchOptions, CT.TTSBatchItem, CT.TTSBatchEvent):
        got = [[f.name, None if f.default is dataclasses.MISSING else f.default] for f in dataclasses.fields(cls)]
        assert got == want[cls.__name__], cls.__name__
    assert dataclasses.fields(CT.TTSBatchOptions) and CT.TTSBatchOptions.__dataclass_params__.frozen
    m = Model.__new__(Model)                           # the hooks read only the config and the speech tokenizer

    class _Cfg:
        tts_model_type = "base"

    class _Tok:
        has_encoder = True
    m.config = _Cfg()
    for kind, has_tok, stream, voice, instruct, ref, speed, batch, cont in json.loads(str(g["truth_table"])):
        m.config.tts_model_type = kind
        m.speech_tokenizer = _Tok() if has_tok else None
        kw = dict(stream=stream, voice=voice, instruct=instruct, speed=speed, ref_audio=np.zeros(4) if ref in ("audio", "both") else None,
                  ref_text="words" if ref in ("text", "both") else None)
        assert (m.supports_tts_batch(**kw), m.supports_tts_continuous_batch(**kw)) == (batch, cont), (kind, has_tok, stream, voice, instruct, ref, speed)


@pytest.mark.skipif(not os.path.isdir("/root/reference/mlx_audio"), reason="the reference source is only present in the build container")
def test_session_fixture_is_what_the_reference_code_produces(tmp_path):
    env = dict(os.environ, GOLDEN_OUT=str(tmp_path), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(HERE, "make_qwen3_session_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
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
