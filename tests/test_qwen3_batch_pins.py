"""Qwen3-TTS ``batch_generate`` on the host: its request checks against the reference's own errors, and the float64 oracle against the
reference's own batch loop (tests/golden/qwen3_batch_golden.npz, written by tests/golden/make_qwen3_batch_golden.py, waveforms kept at
every ``audio_stride``-th sample): in-context (ICL) cloning from one shared reference with per-row frame caps, its stream, and the
stream of a batch without a reference.

The stream rule and the cap rule live here (``stream_schedule``, ``capped``) on top of oracle/qwen3.py, and the GPU tests
(test_qwen3_batch_gpu.py) use the same functions.  Rows of the static batch loop do not interact (per-row attention masks, per-row
uniforms), so a row capped at c frames is the first c frames of the uncapped row."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import qwen3 as Q

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CFG_IDS = dict(codec_nothink_id=1004, codec_think_id=1003, codec_think_bos_id=1005, codec_think_eos_id=1006, codec_pad_id=1001, codec_bos_id=1002)
STREAM_CONTEXT = 25          # qwen3_tts.py:1847: the batch stream's context, whatever streaming_context_size says


def capped(rows, caps):
    """The ICL cap rule (qwen3_tts.py:1818-1823, 1925-1932) applied to the rows of an uncapped run."""
    return [r[: int(c)] for r, c in zip(rows, caps)]


def stream_schedule(lengths, caps, max_tokens, chunk):
    """The emission rule of the batch stream (qwen3_tts.py:1861-2029) from each row's frame count.  A row is finished after the frame
    that sampled its EOS (frame ``length``) or, with caps, after its cap-th frame; the loop breaks before emitting once every row is
    finished.  Otherwise every row that recorded this frame and has ``chunk`` undecoded frames emits them; after the loop every row emits
    its remainder as the final chunk.  Returns [(row, decoded, end, final)] in emission order."""
    B = len(lengths)
    done_at = [c if caps is not None and n == c else n + 1 for n, c in zip(lengths, caps if caps is not None else [None] * B)]
    decoded, events = [0] * B, []
    for n in range(1, max_tokens + 1):
        if all(d <= n for d in done_at):
            break
        for b in range(B):
            if lengths[b] >= n and n - decoded[b] >= chunk:
                events.append((b, decoded[b], n, False))
                decoded[b] = n
    events += [(b, decoded[b], lengths[b], True) for b in range(B) if lengths[b] > decoded[b]]
    return events


def stream_audio(PT, rows, events, tcfg):
    """Each event's audio: chunked_decode of up to 25 frames of context + the new frames, the context's samples dropped."""
    up = int(np.prod(tcfg["upsample_rates"]) * np.prod(tcfg["upsampling_ratios"]))
    out = []
    for b, dec, end, _ in events:
        ctx = min(STREAM_CONTEXT, dec)
        wav = Q.chunked_decode(PT, rows[b][dec - ctx: end].T[None], cfg=tcfg)[0, 0]
        out.append(wav[ctx * up:] if ctx * up < wav.shape[0] else wav)
    return out


def _golden():
    if HERE not in sys.path:
        sys.path.insert(0, HERE)
    import synth_params
    g = np.load(os.path.join(HERE, "qwen3_batch_golden.npz"))
    P, PT, PS = ({k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g[n]).items()} for n in ("talker_params", "tok_params", "spk_params"))
    return g, P, PT, PS


def _check_events(g, tag, rows, caps, max_tokens, interval, PT, tcfg):
    m = json.loads(str(g[f"{tag}_meta"]))
    chunk = max(1, int(interval * 12.5))
    events = stream_schedule([int(r.shape[0]) for r in rows], caps, max_tokens, chunk)
    want = [(e["sequence_idx"], e["token_count"], e["is_final_chunk"]) for e in m["events"]]
    assert [(b, end - dec, final) for b, dec, end, final in events] == want
    assert all(e["is_streaming_chunk"] for e in m["events"])
    for i, a in enumerate(stream_audio(PT, rows, events, tcfg)):
        want = g[f"{tag}_audio_{i}"]
        assert a.shape[0] == m["events"][i]["samples"] and np.abs(a.numpy()[:: int(g["audio_stride"])] - want).max() < 2e-7, i
    return events


def test_oracle_icl_batch_matches_the_reference_batch_generate():
    """ICL batch, stream=False and stream=True: reference encoded once, per-row in-context prompts left-padded into one batch, repetition
    penalty 1.5, rows 0 and 1 stopped by their caps (75, 78), row 2 by EOS after 20 frames; [ref | generated] decoded per row."""
    g, P, PT, PS = _golden()
    cfg, tcfg, ecfg = (json.loads(str(g[k])) for k in ("cfg", "tok_cfg", "tok_enc_cfg"))
    m = json.loads(str(g["icl_meta"]))
    ref_audio = 0.3 * np.random.default_rng(m["ref_seed"]).standard_normal(3 * 1920 + 500)
    rc = Q.tokenizer_encode(PT, torch.as_tensor(ref_audio)[None, None], ecfg)
    assert np.array_equal(rc.numpy(), g["icl_ref_codes"])
    assert m["caps"] == [min(m["max_tokens"], max(75, 6 * n)) for n in m["raw_text_lens"]] == [75, 78, 80]
    spk = torch.as_tensor(g["icl_speaker_embed"])
    rows = [Q.prepare_icl_generation_inputs_from_ids(P, t, m["ref_ids"], rc, (112, 113, 111), CFG_IDS, 1011, spk, cfg) for t in m["target_ids"]]
    assert len({r[0].shape[1] for r in rows}) == 3                                  # three prompt lengths: left padding
    got = capped(Q.generate_codes_batch(P, [r[0] for r in rows], [r[1] for r in rows], rows[0][2], torch.as_tensor(g["icl_u"]), m["max_tokens"],
                                        repetition_penalty=m["repetition_penalty"], cfg=cfg), m["caps"])
    assert [int(r.shape[0]) for r in got] == [75, 78, 20] and m["order"] == [0, 1, 2]
    for b, r in enumerate(got):
        assert np.array_equal(r.numpy(), g[f"icl_codes_{b}"]), b
        wav = Q.decode_icl_generated_codes(PT, r, rc, tcfg).numpy()
        assert m["events"][b]["token_count"] == r.shape[0] and wav.shape[0] == m["events"][b]["samples"]
        assert np.abs(wav[:: int(g["audio_stride"])] - g[f"icl_audio_{b}"]).max() < 2e-7, b
    events = _check_events(g, "icl_stream", got, m["caps"], m["max_tokens"], m["streaming_interval"], PT, tcfg)
    # row 0 completes a chunk at its cap while row 1 runs on (no final chunk), row 1 flushes 3 frames, row 2 ends on a chunk boundary
    assert [e for e in events if e[3]] == [(1, 75, 78, True)]


def test_oracle_plain_batch_stream_matches_the_reference_batch_generate():
    """batch_generate(stream=True) without a reference: the static loop (clamp-pad trailing rule) with a chunk per row every 4 frames and
    the 2-frame remainders as final chunks."""
    g, P, PT, _ = _golden()
    cfg, tcfg = json.loads(str(g["cfg"])), json.loads(str(g["tok_cfg"]))
    m = json.loads(str(g["plain_meta"]))
    rows = [Q.prepare_generation_inputs_from_ids(P, ids, (112, 113, 111), CFG_IDS, 1010) for ids in m["target_ids"]]
    got = Q.generate_codes_batch(P, [r[0] for r in rows], [r[1] for r in rows], rows[0][2], torch.as_tensor(g["plain_u"]), m["max_tokens"], cfg=cfg)
    events = _check_events(g, "plain", got, None, m["max_tokens"], m["streaming_interval"], PT, tcfg)
    assert sum(not e[3] for e in events) == 9 and sum(e[3] for e in events) == 3


def test_stream_schedule_without_caps_emits_at_max_tokens():
    """Without caps a row is never finished by max_tokens, so a chunk completed on the last frame is emitted in the loop, not as a final
    chunk; with caps the loop breaks first and the same frames come out as the final chunk."""
    assert stream_schedule([8, 8], None, 8, 4) == [(0, 0, 4, False), (1, 0, 4, False), (0, 4, 8, False), (1, 4, 8, False)]
    assert stream_schedule([8, 8], [8, 8], 8, 4) == [(0, 0, 4, False), (1, 0, 4, False), (0, 4, 8, True), (1, 4, 8, True)]
    assert stream_schedule([3, 0], None, 8, 4) == [(0, 0, 3, True)]


@pytest.mark.parametrize("name", [row[0] for row in json.loads(str(np.load(os.path.join(HERE, "qwen3_batch_golden.npz"))["errors"]))])
def test_batch_request_errors_match_the_reference(name):
    """Model._batch_request raises what the reference's batch_generate raises (type and message) for each malformed request."""
    from mlx_audio_b200.tts.models.qwen3_tts import Model
    errors = {row[0]: row[1:] for row in json.loads(str(np.load(os.path.join(HERE, "qwen3_batch_golden.npz"))["errors"]))}
    kw, kind, msg = errors[name]
    sym = {"A": np.zeros(4000), "B": np.ones(4000)}                   # two distinct arrays, as in the generator
    kw = {k: ([sym.get(x, x) for x in v] if isinstance(v, list) else sym.get(v, v)) for k, v in kw.items()}
    with pytest.raises({"ValueError": ValueError, "TypeError": TypeError}[kind]) as e:
        Model._batch_request(2, has_encoder=name != "no_encoder", **kw)
    assert str(e.value) == msg


def test_batch_request_routes():
    """The shared reference comes from the scalar arguments or from per-text lists naming the same reference; file paths compare by
    string and are refused (decoding files is outside the accelerated path)."""
    from pathlib import Path
    from mlx_audio_b200.tts.models.qwen3_tts import Model
    a = np.zeros(100)
    assert Model._batch_request(2, has_encoder=True) == ([None, None], [None, None], None, None, False)
    v, i, ra, rt, icl = Model._batch_request(2, ref_audios=[a, a], ref_texts=["t", "t"], has_encoder=True)
    assert ra is a and rt == "t" and icl
    assert Model._batch_request(2, ref_audio=a, ref_text="t", ref_audios=[None, None], has_encoder=True)[4]
    with pytest.raises(NotImplementedError, match="file decoding"):
        Model._batch_request(2, ref_audios=["x.wav", Path("x.wav")], ref_texts=["t", "t"], has_encoder=True)
