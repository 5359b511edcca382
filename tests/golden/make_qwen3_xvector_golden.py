"""Golden vectors of the REFERENCE'S OWN x-vector voice cloning, ``Model.generate(text, ref_audio=...)`` on a base model
(qwen3_tts.py:1227-1298, ``_prepare_generation_inputs`` :326-484, ``extract_speaker_embedding`` :285-324, speaker_encoder.py), executed in
float64 with NumPy standing in for MLX.  Same synthetic trees, configs, stand-in and injected uniforms as make_qwen3_golden.py, whose
setup (TALKER / TOKDEC / SPK, ``fill``, ``CharTokenizer``) this imports.  The speech tokenizer is decoder-only, so ``has_encoder`` is
False and ``ref_audio`` + ``ref_text`` takes the x-vector route too (:1233-1237).
Run from the repo root in the build container:  python tests/golden/make_qwen3_xvector_golden.py  ->  tests/golden/qwen3_xvector_golden.npz

Runs (EOS row of the codec head scaled by EOS_GAIN so that ``alone`` stops on EOS before max_tokens; the generator asserts it):
  alone      ref_audio alone, reaching EOS;
  voice      ref_audio with voice="amy" (the x-vector wins) and lang_code="english";
  two_seg    two '\\n' segments (the embedding is recomputed per segment, as the reference does);
  stream     stream=True, 7 frames in chunks of 3;
  ref_text   ref_audio + ref_text with a speech tokenizer that has no encoder.
Per run: per segment the prompt (input_embeds, trailing, pad), text ids, speaker embedding, codes and audio (float32); for ``stream``
the events (token_count, samples, is_streaming_chunk, is_final_chunk, segment_idx) with each event's audio."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_qwen3_golden as G        # noqa: E402  (installs the NumPy stand-in for MLX and the reference packages)
import synth_params                  # noqa: E402

mx, C = G.mx, G.C

RUNS = [dict(tag="alone", text="Clone this voice.", voice=None, lang_code="auto", max_tokens=24, seed=71),
        dict(tag="voice", text="With a voice", voice="amy", lang_code="english", max_tokens=6, seed=72),
        dict(tag="two_seg", text="First bit.\nSecond bit", voice=None, lang_code="german", max_tokens=5, seed=73),
        dict(tag="stream", text="Streamed clone", voice=None, lang_code="auto", max_tokens=7, seed=74, stream=True, interval=0.24),
        dict(tag="ref_text", text="Words too", voice=None, lang_code="auto", max_tokens=5, seed=75, ref_text="Reference words")]


def main():
    from mlx_audio.tts.models.qwen3_tts import qwen3_tts as QM
    from mlx_audio.tts.models.qwen3_tts import speech_tokenizer as S
    QM.load_audio = lambda a, sample_rate=None: a                     # callers hand 24 kHz samples, not a file
    gain = float(os.environ.get("EOS_GAIN", "2.0"))
    out = {"cfg": json.dumps(G.ORACLE_CFG), "tok_cfg": json.dumps(G.ORACLE_TOK), "spk_cfg": json.dumps(G.SPK), "gen_eos_gain": gain}
    mx.random.strict = False                                         # parameter initialisers draw while the modules are built
    tok = S.Qwen3TTSSpeechTokenizer(C.Qwen3TTSTokenizerConfig(decoder_config=C.Qwen3TTSTokenizerDecoderConfig(**G.TOKDEC)))
    assert not tok.has_encoder
    names = G.fill(tok, rule=lambda n: "small" if n.endswith((".alpha", ".beta")) else ("scale0.08" if n == "decoder.decoder.6.conv.weight" else None))
    out["tok_params"] = synth_params.manifest(names)
    cfg = C.ModelConfig(talker_config=dict(G.TALKER), speaker_encoder_config=dict(G.SPK), tts_model_type="base", tts_pad_token_id=111,
                        tts_bos_token_id=112, tts_eos_token_id=113)
    model = QM.Model(cfg)
    out["talker_params"] = synth_params.manifest(G.fill(model.talker))
    out["spk_params"] = synth_params.manifest(G.fill(model.speaker_encoder, prefix="speaker_encoder."))
    eos = G.TALKER["codec_eos_token_id"]
    w = np.array(model.talker.codec_head.weight)
    w[eos] *= gain
    model.talker.codec_head.weight = mx.array(w)
    model.load_speech_tokenizer(tok)
    model.tokenizer = G.CharTokenizer()
    # spies: prompts, embeddings, codes handed to the decoder
    cap = {"prompts": [], "embeds": [], "codes": [], "steps": []}
    real_prep, real_embed, real_decode, real_step = (model._prepare_generation_inputs, model.extract_speaker_embedding, tok.decode,
                                                     tok.decoder.streaming_step)

    def prep(*a, **k):
        r = real_prep(*a, **k)
        cap["prompts"].append([np.asarray(x) for x in r])
        return r

    def embed(*a, **k):
        r = real_embed(*a, **k)
        cap["embeds"].append(np.asarray(r))
        return r

    def decode(codes):
        cap["codes"].append(np.asarray(codes))
        return real_decode(codes)

    def step(codes):
        cap["steps"].append(np.asarray(codes))
        return real_step(codes)
    model._prepare_generation_inputs, model.extract_speaker_embedding, tok.decode, tok.decoder.streaming_step = prep, embed, decode, step
    mx.random.strict = True
    g = G.TALKER["num_code_groups"]
    for r in RUNS:
        t = r["tag"]
        rng = np.random.default_rng(r["seed"])
        ref_audio = 0.3 * rng.standard_normal(2 * 1920 + 700)                     # regenerated by the test from the seed
        n_seg = len(r["text"].split("\n"))
        us = rng.random((n_seg * r["max_tokens"], g))
        mx.random.queue[:] = [("categorical", np.array([v])) for v in us.reshape(-1)]
        model.tokenizer.calls.clear()
        for v in cap.values():
            v.clear()
        res = list(model.generate(text=r["text"], voice=r["voice"], lang_code=r["lang_code"], max_tokens=r["max_tokens"], ref_audio=mx.array(ref_audio),
                                  ref_text=r.get("ref_text"), stream=r.get("stream", False), streaming_interval=r.get("interval", 2.0)))
        draws_left = len(mx.random.queue)
        if t == "alone":
            assert draws_left > 0, "no EOS before max_tokens; pick another seed or EOS_GAIN"
        assert len(cap["prompts"]) == len(cap["embeds"]) == n_seg
        out[f"{t}_meta"] = json.dumps({k: v for k, v in r.items() if k != "seed"} | {"seed": r["seed"], "text_ids": list(model.tokenizer.calls),
                                                                                   "draws_left": draws_left})
        out[f"{t}_u"] = us
        for s in range(n_seg):
            out[f"{t}_s{s}_input_embeds"], out[f"{t}_s{s}_trailing"], out[f"{t}_s{s}_pad"] = cap["prompts"][s]
            out[f"{t}_s{s}_speaker_embed"] = cap["embeds"][s]
        if r.get("stream"):
            out[f"{t}_events"] = np.array([[e.token_count, e.samples, int(e.is_streaming_chunk), int(e.is_final_chunk), e.segment_idx] for e in res],
                                          dtype=np.int64)
            for i, (e, cc) in enumerate(zip(res, cap["steps"])):
                out[f"{t}_ev{i}_audio"], out[f"{t}_ev{i}_codes"] = np.asarray(e.audio), cc.astype(np.int64)
        else:
            assert len(res) == len(cap["codes"]) == n_seg
            for s, (e, cc) in enumerate(zip(res, cap["codes"])):
                out[f"{t}_s{s}_codes"], out[f"{t}_s{s}_audio"] = cc[0].astype(np.int64), np.asarray(e.audio)
        print(t, "segments", n_seg, "results", [e.token_count for e in res], "draws left", draws_left)
    mx.random.queue[:] = []
    mx.random.strict = False
    for k in list(out):                                              # waveforms are stored as float32 (|x| <= 1: 6e-8 absolute)
        if k.endswith("_audio"):
            out[k] = np.asarray(out[k], dtype=np.float32)
    np.savez_compressed(os.path.join(os.environ.get("GOLDEN_OUT", HERE), "qwen3_xvector_golden.npz"), **out)


if __name__ == "__main__":
    main()
