"""Batched in-context voice cloning (Qwen3-TTS ``batch_generate(texts, ref_audio=..., ref_text=...)``) against one ``generate(text,
ref_audio=..., ref_text=...)`` call per text, at released sizes with synthetic weights (28 + 5 layer talker, speech-tokenizer encoder and
decoder, ECAPA speaker encoder), a 10 s reference and targets of 20-40 text tokens, for B = 1, 4 and 8 texts, alternating in one process:

- wall time to the last result, frames/s and audio-s/s of both;
- the batch call split into encoder + x-vector, prefill, frame loop and joint decode (each stage timed on its own, synchronised);
- for ``stream=True`` the time to the first chunk.

The reference cache is cleared before every timed call, so each call encodes its reference once.  Prints the card's name and power limit
with the numbers, then one JSON line.  Needs a GPU (no fallback).

    python tools/qwen3_batch_icl_bench.py [--reps 3] [--frames 50]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from mlx_audio_b200 import synth                                               # noqa: E402
from mlx_audio_b200.configs import QWEN3_TALKER, QWEN3_TOKENIZER_DECODER, QWEN3_TOKENIZER_ENCODER             # noqa: E402
from mlx_audio_b200.tts.models.qwen3_tts import (Model, ModelConfig, Qwen3TTSSpeechTokenizer, Qwen3TTSTalkerCodePredictorConfig,  # noqa: E402
                                                 Qwen3TTSTalkerConfig, Qwen3TTSTokenizerConfig, Qwen3TTSTokenizerEncoderConfig)
from qwen3_icl_bench import card                                               # noqa: E402
from speaker_encoder_bench import SPEAKER_ENCODER                              # noqa: E402


class CharTokenizer:
    """Chat markers are single ids, every other character one id (10-109): a text of n characters is n tokens."""
    MARK = {"<|im_start|>": 1, "<|im_end|>": 2, "assistant": 3, "user": 4, "\n": 5}

    def encode(self, text):
        ids, i = [], 0
        while i < len(text):
            for m, v in self.MARK.items():
                if text.startswith(m, i):
                    ids.append(v)
                    i += len(m)
                    break
            else:
                ids.append(10 + (ord(text[i]) % 100))
                i += 1
        return ids


def sync_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def split(model, texts, ref_audio, ref_text, frames):
    """The stages of the batch call, each synchronised: encoder + x-vector, prompt assembly + prefill frame, frame loop, joint decode."""
    tok = model.tokenizer
    (codes, spk), enc = sync_ms(lambda: (model.encode_reference(ref_audio), model.extract_speaker_embedding(ref_audio)))
    ref_ids = tok.encode(f"<|im_start|>assistant\n{ref_text}<|im_end|>\n")
    targets = [tok.encode(f"<|im_start|>assistant\n{t}<|im_end|>\n<|im_start|>assistant\n") for t in texts]
    caps = [min(frames, max(75, 6 * len(tok.encode(t)))) for t in texts]
    (x, trailing, pad, left), prep = sync_ms(lambda: model._pad_batch([model.prepare_icl_generation_inputs_from_ids(t, ref_ids, codes, None, spk)
                                                                      for t in targets]))
    gen = dict(max_tokens=frames, repetition_penalty=1.5, seed=1, left_padding=left, batch_mode=True, caps=caps)
    _, first = sync_ms(lambda: model.generate_codes(x, trailing, pad, **dict(gen, max_tokens=1, caps=[1] * len(texts))))
    (out, lengths), loop = sync_ms(lambda: model.generate_codes(x, trailing, pad, **gen))
    _, dec = sync_ms(lambda: model._decode_icl_batch([out[b, : int(lengths[b])] for b in range(len(texts))], codes))
    return {"encoder_xvector_ms": enc, "prefill_ms": prep + first, "frame_loop_ms": loop - first, "joint_decode_ms": dec,
            "frames": [int(v) for v in lengths]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=50, help="max_tokens of every call")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qwen3_batch_icl_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    flat = dict(QWEN3_TALKER)
    P = synth.qwen3_talker_weights(flat, seed=11)
    P.update(synth.qwen3_speaker_encoder_weights(dict(SPEAKER_ENCODER)))
    cp = Qwen3TTSTalkerCodePredictorConfig(num_hidden_layers=flat["cp_num_hidden_layers"])
    tc = Qwen3TTSTalkerConfig(code_predictor_config=cp, num_hidden_layers=flat["num_hidden_layers"], text_vocab_size=512,
                              codec_eos_token_id=flat["codec_eos_token_id"])
    model = Model(ModelConfig(talker_config=tc, tts_model_type="base", tts_pad_token_id=500, tts_bos_token_id=501, tts_eos_token_id=502),
                  dev).load_weights(P)
    st = Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(encoder_config=Qwen3TTSTokenizerEncoderConfig()), dev)
    st.load_weights(synth.qwen3_tokenizer_weights(dict(QWEN3_TOKENIZER_DECODER), seed=12, encoder=dict(QWEN3_TOKENIZER_ENCODER)))
    model.load_speech_tokenizer(st)
    model.tokenizer = CharTokenizer()
    rng = np.random.default_rng(5)
    ref_audio = torch.as_tensor(0.3 * rng.standard_normal(10 * 24000), dtype=torch.float32).to(dev)
    ref_text = "the words that were spoken in the reference recording, forty"
    letters = np.array(list("abcdefghijklmnopqrstuvwxyz     "))
    texts = ["".join(rng.choice(letters, size=int(n))) for n in rng.integers(20, 41, size=8)]
    res = {"card": card(), "frames_cap": args.frames, "batch": {}}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    for B in (1, 4, 8):
        row = {"batch_ms": [], "sequential_ms": [], "first_chunk_ms": []}
        for rep in range(args.reps + 1):                             # rep 0 warms up every shape
            model._icl_cache.clear()
            out, ms_b = sync_ms(lambda: list(model.batch_generate(texts[:B], ref_audio=ref_audio, ref_text=ref_text, max_tokens=args.frames, seed=rep)))
            model._icl_cache.clear()
            seq, ms_s = sync_ms(lambda: [r for t in texts[:B] for r in model.generate(t, ref_audio=ref_audio, ref_text=ref_text,
                                                                                      max_tokens=args.frames, seed=rep)])
            model._icl_cache.clear()
            stream = model.batch_generate(texts[:B], ref_audio=ref_audio, ref_text=ref_text, max_tokens=args.frames, seed=rep, stream=True,
                                          streaming_interval=2.0)
            _, ms_f = sync_ms(lambda: next(stream))
            stream.close()
            if rep:
                row["batch_ms"].append(ms_b)
                row["sequential_ms"].append(ms_s)
                row["first_chunk_ms"].append(ms_f)
                frames_b, audio_b = sum(r.token_count for r in out), sum(r.samples for r in out) / 24000
                frames_s, audio_s = sum(r.token_count for r in seq), sum(r.samples for r in seq) / 24000
        med = {k: float(np.median(v)) for k, v in row.items()}
        med.update(batch_frames=frames_b, batch_frames_per_s=frames_b / med["batch_ms"] * 1e3, batch_audio_s_per_s=audio_b / med["batch_ms"] * 1e3,
                   sequential_frames=frames_s, sequential_frames_per_s=frames_s / med["sequential_ms"] * 1e3,
                   sequential_audio_s_per_s=audio_s / med["sequential_ms"] * 1e3)
        split(model, texts[:B], ref_audio, "warm-up", args.frames)
        med["split"] = split(model, texts[:B], ref_audio, ref_text, args.frames)
        res["batch"][B] = med
        s = med["split"]
        print(f"B={B}: batch_generate {med['batch_ms']:.0f} ms ({med['batch_frames_per_s']:.0f} frames/s, {med['batch_audio_s_per_s']:.2f} audio-s/s), "
              f"{B} x generate {med['sequential_ms']:.0f} ms ({med['sequential_frames_per_s']:.0f} frames/s, {med['sequential_audio_s_per_s']:.2f} audio-s/s), "
              f"stream first chunk {med['first_chunk_ms']:.0f} ms | split: encoder + x-vector {s['encoder_xvector_ms']:.1f} ms, prefill "
              f"{s['prefill_ms']:.1f} ms, frame loop {s['frame_loop_ms']:.1f} ms ({max(s['frames'])} frames), joint decode {s['joint_decode_ms']:.1f} ms",
              flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
