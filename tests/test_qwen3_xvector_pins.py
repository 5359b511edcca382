"""Qwen3-TTS x-vector voice cloning pinned to the reference's own code: tests/golden/qwen3_xvector_golden.npz holds the reference's
``Model.generate(text, ref_audio=...)`` on a base model (alone and reaching EOS, with a preset voice and a language, over two segments,
streamed, and with ref_text when the speech tokenizer has no encoder), executed through the NumPy stand-in by
tests/golden/make_qwen3_xvector_golden.py.  ``oracle.qwen3_xvector`` must reproduce every run: the speaker embedding (the oracle's
filterbank emulates float32: 1e-5, as in test_oracle_pins.py), the prompt built from the reference's embedding to 1e-12, codes and stream
flags identical, audio to float32 storage precision."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(HERE))
FIXTURE = "qwen3_xvector_golden.npz"
WTOL = 2e-7

IDS = dict(codec_nothink_id=1004, codec_think_id=1003, codec_think_bos_id=1005, codec_think_eos_id=1006, codec_pad_id=1001, codec_bos_id=1002)
LANG = {"english": 1010, "german": 1011}
TAGS = ["alone", "voice", "two_seg", "stream", "ref_text"]


def _load():
    if HERE not in sys.path:
        sys.path.insert(0, HERE)
    import synth_params
    g = np.load(os.path.join(HERE, FIXTURE), allow_pickle=False)
    P, PT, PS = ({k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g[n]).items()} for n in ("talker_params", "tok_params", "spk_params"))
    cfg = json.loads(str(g["cfg"]))
    P["codec_head.weight"] = P["codec_head.weight"].clone()
    P["codec_head.weight"][cfg["codec_eos_token_id"]] *= float(g["gen_eos_gain"])
    return g, P, PT, PS, cfg, json.loads(str(g["tok_cfg"])), json.loads(str(g["spk_cfg"]))


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_xvector_runs_match_the_reference_generate(tag):
    from oracle import qwen3 as Q
    from oracle import qwen3_stream as QS
    from oracle import qwen3_xvector as QX
    g, P, PT, PS, cfg, tcfg, scfg = _load()
    m = json.loads(str(g[f"{tag}_meta"]))
    rng = np.random.default_rng(m["seed"])
    ref_audio = 0.3 * rng.standard_normal(2 * 1920 + 700)
    u = torch.as_tensor(g[f"{tag}_u"])
    assert np.array_equal(u.numpy(), rng.random(u.shape))
    emb = QX.speaker_embedding(PS, ref_audio, scfg)
    mt, row, events = m["max_tokens"], 0, []
    for s, text_ids in enumerate(m["text_ids"]):
        want_emb = g[f"{tag}_s{s}_speaker_embed"]
        assert want_emb.shape == (1, scfg["enc_dim"]) and np.abs(emb.numpy() - want_emb).max() < 1e-5
        ie, tr, pad = QX.prepare_generation_inputs_from_embed(P, text_ids, (112, 113, 111), IDS, LANG.get(m["lang_code"]),
                                                              torch.as_tensor(want_emb))
        for x, k in ((ie, "input_embeds"), (tr, "trailing"), (pad, "pad")):
            assert x.shape == g[f"{tag}_s{s}_{k}"].shape and np.abs(x.numpy() - g[f"{tag}_s{s}_{k}"]).max() < 1e-12, (s, k)
        codes = Q.generate_codes(P, ie, tr, pad, u[row:], mt, cfg=cfg)
        row += codes.shape[0] + (1 if codes.shape[0] < mt else 0)         # the EOS frame draws its uniforms too
        if m.get("stream"):
            events += QS.stream_events(PT, codes, m["interval"], tcfg, segment_idx=s)
            continue
        assert np.array_equal(codes.numpy(), g[f"{tag}_s{s}_codes"]), s
        wav, ln = Q.speech_tokenizer_decode(PT, codes[None], tcfg)
        want = g[f"{tag}_s{s}_audio"]
        assert int(ln[0]) == want.shape[0] and np.abs(wav[0, :int(ln[0])].numpy() - want).max() < WTOL, s
    assert row * u.shape[1] + m["draws_left"] == u.numel()                 # every uniform the reference drew is accounted for
    if m.get("stream"):
        ev = g[f"{tag}_events"]
        got = np.array([[e["token_count"], e["samples"], int(e["is_streaming_chunk"]), int(e["is_final_chunk"]), e["segment_idx"]] for e in events])
        assert np.array_equal(got, ev) and ev[:, 0].tolist() == [3, 3, 1]
        for i, e in enumerate(events):
            assert np.array_equal(e["codes"].T[None].numpy(), g[f"{tag}_ev{i}_codes"]), i
            assert np.abs(e["audio"].numpy() - g[f"{tag}_ev{i}_audio"]).max() < WTOL, i
    if tag == "alone":
        assert m["draws_left"] > 0                                         # stopped on EOS, not on max_tokens
    if tag == "two_seg":
        assert len(m["text_ids"]) == 2


@pytest.mark.skipif(not os.path.isdir("/root/reference/mlx_audio"), reason="the reference source is only present in the build container")
def test_xvector_fixture_is_what_the_reference_code_produces(tmp_path):
    env = dict(os.environ, GOLDEN_OUT=str(tmp_path), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(HERE, "make_qwen3_xvector_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True,
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
