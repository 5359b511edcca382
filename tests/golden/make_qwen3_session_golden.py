"""Golden vectors of the REFERENCE'S OWN continuous-batching session, ``Qwen3TTSBatchSession`` (tts/models/qwen3_tts/continuous_batching.py),
driven step by step with staggered admissions and executed in float64 with NumPy standing in for MLX.  Same synthetic tree, stand-in
and EOS boost as make_qwen3_golden.py (whose setup this reuses), and its per-row uniform-stream convention (session_cases): every
request draws from its own stream u[request, frame, group], whichever batch it is in.
Run from the repo root in the build container:  python tests/golden/make_qwen3_session_golden.py  ->  tests/golden/qwen3_session_golden.npz

Schedule: max_batch_size 2, max_tokens 12; requests 0-3 (four prompt lengths: voice and instruct differ) added before step 0, request 4
added after the third step, request 0 cancelled while active before step 5.  Recorded: per request its uniforms, the codes handed to
_decode_generated_codes, the event's audio and token count; the event sequence (step, sequence id, samples, token count); the fields
and defaults of the tts/continuous.py dataclasses; and the supports_tts_batch / supports_tts_continuous_batch truth table."""
import dataclasses
import itertools
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_qwen3_golden as G        # noqa: E402  (installs the NumPy stand-in for MLX and the reference packages)
import synth_params                  # noqa: E402

mx, C = G.mx, G.C

ITEMS = [dict(text="Hello there, world.", voice="amy", instruct="calm and slow"), dict(text="Short one", voice="bob", instruct=None),
         dict(text="A middle sentence", voice="amy", instruct="sad"), dict(text="Hi", voice="bob", instruct=None),
         dict(text="Late arrival.", voice="amy", instruct=None)]
SCRIPT = {0: [("add", [0, 1, 2, 3])], 3: [("add", [4])], 5: [("cancel", 0)]}
MAX_TOKENS, MAX_BATCH = 12, 2


def truth_table(model, tok):
    rows = []
    for kind, has_tok, stream, voice, instruct, ref, speed in itertools.product(("base", "custom_voice", "voice_design"), (True, False),
                                                                                 (False, True), (None, "amy"), (None, "calm"),
                                                                                 ("none", "audio", "text", "both"), (1.0, 1.5)):
        model.config.tts_model_type = kind
        model.speech_tokenizer = tok if has_tok else None
        kw = dict(stream=stream, voice=voice, instruct=instruct, speed=speed, ref_audio=np.zeros(4) if ref in ("audio", "both") else None,
                  ref_text="words" if ref in ("text", "both") else None)
        rows.append([kind, has_tok, stream, voice, instruct, ref, speed, bool(model.supports_tts_batch(**kw)),
                     bool(model.supports_tts_continuous_batch(**kw))])
    model.config.tts_model_type = "custom_voice"
    model.speech_tokenizer = tok
    return rows


def main():
    from mlx_audio.tts import continuous as CT
    from mlx_audio.tts.models.qwen3_tts import continuous_batching as CB
    from mlx_audio.tts.models.qwen3_tts import qwen3_tts as QM
    from mlx_audio.tts.models.qwen3_tts import speech_tokenizer as S
    out = {"cfg": json.dumps(G.ORACLE_CFG), "tok_cfg": json.dumps(G.ORACLE_TOK)}
    tok = S.Qwen3TTSSpeechTokenizer(C.Qwen3TTSTokenizerConfig(decoder_config=C.Qwen3TTSTokenizerDecoderConfig(**G.TOKDEC),
                                                              encoder_config=C.Qwen3TTSTokenizerEncoderConfig(**G.TOKENC)))
    names = G.fill(tok, rule=lambda n: "small" if n.endswith((".alpha", ".beta")) else ("scale0.08" if n == "decoder.decoder.6.conv.weight" else None))
    out["tok_params"] = synth_params.manifest(names)
    cfg = C.ModelConfig(talker_config=dict(G.TALKER), tts_model_type="custom_voice", tts_pad_token_id=111, tts_bos_token_id=112, tts_eos_token_id=113)
    model = QM.Model(cfg)
    out["talker_params"] = synth_params.manifest(G.fill(model.talker))
    gain = 2.0
    w = np.array(model.talker.codec_head.weight)
    w[G.TALKER["codec_eos_token_id"]] *= gain                        # makes EOS reachable within a few frames
    model.talker.codec_head.weight = mx.array(w)
    out["eos_gain"] = gain
    model.load_speech_tokenizer(tok)
    model.tokenizer = G.CharTokenizer()
    g, n = G.TALKER["num_code_groups"], len(ITEMS)
    us = np.random.default_rng(71).random((n, MAX_TOKENS, g))
    state = {"rows": [], "frame": {b: 0 for b in range(n)}, "group": 0}

    def draw(shape):
        rows = state["rows"]
        assert shape == (len(rows),), (shape, rows)
        v = np.array([us[r, state["frame"][r], state["group"]] for r in rows])
        state["group"] += 1
        if state["group"] == g:
            state["group"] = 0
            for r in rows:
                state["frame"][r] += 1
        return v
    admit, advance = CB.Qwen3TTSBatchSession._admit_pending, CB.Qwen3TTSBatchSession._advance_active

    def admit_spy(self):
        state["rows"] = [it.sequence_id for it in self._pending[: min(self.available_slots, len(self._pending))]]
        return admit(self)

    def advance_spy(self):
        state["rows"] = [st.sequence_id for st in self._active]
        return advance(self)
    CB.Qwen3TTSBatchSession._admit_pending, CB.Qwen3TTSBatchSession._advance_active = admit_spy, advance_spy
    decoded = []
    real = model._decode_generated_codes

    def decode_spy(codes, **k):
        decoded.append(np.concatenate([np.asarray(c) for c in codes], axis=0))
        return real(codes, **k)
    model._decode_generated_codes = decode_spy
    mx.random.strict = True
    mx.random.queue[:] = [("categorical", draw)] * (n * MAX_TOKENS * g)
    session = model.create_tts_batch_session(CT.TTSBatchOptions(max_tokens=MAX_TOKENS, max_batch_size=MAX_BATCH))
    items = [CT.TTSBatchItem(sequence_id=i, **it) for i, it in enumerate(ITEMS)]
    events, cancelled_active = [], []
    for step in range(200):
        for kind, arg in SCRIPT.get(step, []):
            if kind == "add":
                session.add([items[i] for i in arg])
            else:
                cancelled_active += [st.sequence_id for st in session._active if st.sequence_id == arg]
                session.cancel(arg)
        if session.idle and step > max(SCRIPT):
            break
        for e in session.step():
            events.append((step, e))
    CB.Qwen3TTSBatchSession._admit_pending, CB.Qwen3TTSBatchSession._advance_active = admit, advance
    del model.__dict__["_decode_generated_codes"]
    mx.random.queue[:] = []
    mx.random.strict = False
    assert cancelled_active == [0], "request 0 must be active when it is cancelled"
    counts = [e.token_count for _, e in events]
    assert len(decoded) == sum(c > 0 for c in counts), counts              # an empty event (EOS on the first frame) decodes nothing
    assert MAX_TOKENS in counts and any(0 < c < MAX_TOKENS for c in counts), ("need one row on max_tokens and one on EOS", counts)
    out["meta"] = json.dumps({"items": ITEMS, "script": {str(k): v for k, v in SCRIPT.items()}, "max_tokens": MAX_TOKENS,
                              "max_batch_size": MAX_BATCH, "lang_code": "auto",
                              "text_ids": [G.CharTokenizer().encode(f"<|im_start|>assistant\n{it['text']}<|im_end|>\n<|im_start|>assistant\n") for it in ITEMS],
                              "instruct_ids": [G.CharTokenizer().encode(f"<|im_start|>user\n{it['instruct']}<|im_end|>\n") if it["instruct"] else None
                                               for it in ITEMS]})
    out["u"] = us
    out["events"] = np.array([[s, e.sequence_id, e.samples, e.token_count] for s, e in events], dtype=np.int64)
    for (s, e), c in zip([ev for ev in events if ev[1].token_count > 0], decoded):
        out[f"codes_{e.sequence_id}"] = c.astype(np.int64)
        out[f"audio_{e.sequence_id}"] = np.asarray(e.audio, dtype=np.float32)
    out["dataclasses"] = json.dumps({cls.__name__: [[f.name, None if f.default is dataclasses.MISSING else f.default] for f in dataclasses.fields(cls)]
                                     for cls in (CT.TTSBatchOptions, CT.TTSBatchItem, CT.TTSBatchEvent)})
    out["truth_table"] = json.dumps(truth_table(model, tok))
    print("events", out["events"].tolist())
    np.savez_compressed(os.path.join(os.environ.get("GOLDEN_OUT", HERE), "qwen3_session_golden.npz"), **out)


if __name__ == "__main__":
    main()
