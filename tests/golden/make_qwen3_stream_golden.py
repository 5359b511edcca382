"""Golden vectors of the REFERENCE'S OWN streaming generation loop, ``Model.generate(stream=True)`` (qwen3_tts.py:1316-1521 base path,
:2264-2446 custom-voice path) with the incremental decoder ``streaming_step`` (speech_tokenizer.py:882-930), executed in float64 with
NumPy standing in for MLX.  Same synthetic tree, stand-in and injected uniforms as make_qwen3_golden.py (whose setup this reuses).
Run from the repo root in the build container:  python tests/golden/make_qwen3_stream_golden.py  ->  tests/golden/qwen3_stream_golden.npz

Cases (no EOS boost, so every segment runs to max_tokens; the generator asserts it):
  cv_exact   custom voice, 8 frames in chunks of 4 -> two chunks and NO final event;
  cv_rem     custom voice, 7 frames in chunks of 3 -> 3 + 3 + a final chunk of 1;
  cv_one     custom voice, 5 frames in 1-frame chunks (history longer than a chunk);
  base_two   base model, two '\\n' segments of 6 frames in chunks of 4 (4 + final 2 each), segment_idx 0 and 1.
Per event: audio (float32), token_count, samples, is_streaming_chunk, is_final_chunk, segment_idx, and the codes handed to that
streaming_step (captured by a spy)."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_qwen3_golden as G        # noqa: E402  (installs the NumPy stand-in for MLX and the reference packages)
import synth_params                  # noqa: E402

mx, C = G.mx, G.C

CASES = [dict(tag="cv_exact", kind="custom_voice", texts=["Stream me."], voice="amy", lang_code="english", max_tokens=8, interval=0.32, seed=61),
         dict(tag="cv_rem", kind="custom_voice", texts=["Another one"], voice="bob", lang_code="auto", max_tokens=7, interval=0.24, seed=62),
         dict(tag="cv_one", kind="custom_voice", texts=["Tiny"], voice="amy", lang_code="german", max_tokens=5, interval=0.08, seed=63),
         dict(tag="base_two", kind="base", texts=["First part.", "Second part"], voice=None, lang_code="auto", max_tokens=6, interval=0.32, seed=64)]


def main():
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
    model.load_speech_tokenizer(tok)
    model.tokenizer = G.CharTokenizer()
    captured = []
    real_step = tok.decoder.streaming_step

    def spy(codes):
        captured.append(np.asarray(codes))
        return real_step(codes)
    tok.decoder.streaming_step = spy
    mx.random.strict = True
    g = G.TALKER["num_code_groups"]
    for c in CASES:
        model.config.tts_model_type = c["kind"]
        n_seg = len(c["texts"])
        us = np.random.default_rng(c["seed"]).random((n_seg * c["max_tokens"], g))
        mx.random.queue[:] = [("categorical", np.array([v])) for v in us.reshape(-1)]
        model.tokenizer.calls.clear()
        captured.clear()
        events = list(model.generate(text="\n".join(c["texts"]), voice=c["voice"], lang_code=c["lang_code"], max_tokens=c["max_tokens"],
                                     stream=True, streaming_interval=c["interval"]))
        assert not mx.random.queue, "a segment stopped on EOS before max_tokens; pick another seed"
        assert len(captured) == len(events)
        t = c["tag"]
        out[f"{t}_meta"] = json.dumps({k: v for k, v in c.items() if k != "seed"} | {"text_ids": list(model.tokenizer.calls)})
        out[f"{t}_u"] = us
        out[f"{t}_events"] = np.array([[e.token_count, e.samples, int(e.is_streaming_chunk), int(e.is_final_chunk), e.segment_idx] for e in events],
                                      dtype=np.int64)
        for i, (e, cc) in enumerate(zip(events, captured)):
            out[f"{t}_ev{i}_audio"] = np.asarray(e.audio, dtype=np.float32)
            out[f"{t}_ev{i}_codes"] = cc.astype(np.int64)
        print(t, "events", out[f"{t}_events"].tolist())
    mx.random.queue[:] = []
    mx.random.strict = False
    np.savez_compressed(os.path.join(os.environ.get("GOLDEN_OUT", HERE), "qwen3_stream_golden.npz"), **out)


if __name__ == "__main__":
    main()
