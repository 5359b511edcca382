"""In-context voice cloning (Qwen3-TTS ``generate(text, ref_audio=..., ref_text=...)``) at released sizes with synthetic weights:

- speech-tokenizer encoder time for 3 / 10 / 30 s of reference audio;
- talker prefill time at the resulting ICL prompt lengths, attention on ``attn_decode`` (one CTA per query row) against the tensor-core
  ``attn_prefill``, alternating in one process, and the largest difference of their logits;
- time to the first streamed chunk of ``generate_icl_from_ids(..., stream=True)`` and the whole non-streaming call.

Prints the card's name and power limit with the numbers, then one JSON line.  CUDA events / host clocks around synchronised work;
every timed shape is warmed up first.  Needs a GPU (no fallback).

    python tools/qwen3_icl_bench.py [--reps 5] [--frames 50]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from mlx_audio_b200 import synth                                               # noqa: E402
from mlx_audio_b200.configs import QWEN3_TALKER, QWEN3_TOKENIZER_DECODER, QWEN3_TOKENIZER_ENCODER             # noqa: E402
from mlx_audio_b200.tts.models.qwen3_tts import (Model, ModelConfig, Qwen3TTSSpeechTokenizer, Qwen3TTSTalkerCodePredictorConfig,  # noqa: E402
                                                 Qwen3TTSTalkerConfig, Qwen3TTSTokenizerConfig, Qwen3TTSTokenizerEncoderConfig)
from mlx_audio_b200.tts.models.qwen3_tts import talker as T                    # noqa: E402
from speaker_encoder_bench import SPEAKER_ENCODER                              # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, reps):
    """median ms of ``reps`` calls (CUDA events), after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=50, help="max_tokens of the generate calls")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qwen3_icl_bench: needs a CUDA device")
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
    g = torch.Generator().manual_seed(3)
    target = [1, 3, 5] + torch.randint(10, 500, (30,), generator=g).tolist() + [2, 5, 1, 3, 5]          # ~30 text tokens to say
    ref = [1, 3, 5] + torch.randint(10, 500, (40,), generator=g).tolist() + [2, 5]                      # the reference's transcript
    res = {"card": card(), "encoder_ms": {}, "prefill": {}}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    default_min = T.PREFILL_TC_MIN_ROWS
    for sec in (3, 10, 30):
        audio = torch.as_tensor(0.3 * np.random.default_rng(sec).standard_normal(sec * 24000), dtype=torch.float32).to(dev)
        res["encoder_ms"][sec] = timed(lambda: model.encode_reference(audio), args.reps)
        codes = model.encode_reference(audio)
        spk = model.extract_speaker_embedding(audio)
        x, _, _ = model.prepare_icl_generation_inputs_from_ids(target, ref, codes, 2050, spk)
        S = int(x.shape[1])

        def prefill():
            model.talker.reset_cache(1, S + 64)
            return model.talker(x)[0]
        row = {}
        logits = {}
        for rep in range(2):                                     # alternate the two routes, twice
            for name, thr in (("attn_decode", 1 << 30), ("attn_prefill", default_min)):
                T.PREFILL_TC_MIN_ROWS = thr
                ms = timed(prefill, args.reps)
                row.setdefault(name, []).append(ms)
                logits[name] = prefill().clone()
        T.PREFILL_TC_MIN_ROWS = default_min
        row = {k: float(np.median(v)) for k, v in row.items()}
        row["logit_max_abs_diff"] = float((logits["attn_decode"] - logits["attn_prefill"]).abs().max())
        row["prompt_rows"] = S
        res["prefill"][sec] = row
        print(f"ref {sec:2d} s: encoder {res['encoder_ms'][sec]:.2f} ms, prompt {S} rows, talker prefill attn_decode {row['attn_decode']:.2f} ms"
              f" / attn_prefill {row['attn_prefill']:.2f} ms (logits differ by {row['logit_max_abs_diff']:.2e})", flush=True)
    audio10 = torch.as_tensor(0.3 * np.random.default_rng(10).standard_normal(10 * 24000), dtype=torch.float32).to(dev)
    kw = dict(ref_audio=audio10, language_id=2050, max_tokens=args.frames, seed=1)
    ttfc, whole, frames = [], [], 0
    for i in range(args.reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        next(iter(model.generate_icl_from_ids(target, ref, stream=True, streaming_interval=0.32, **kw)))
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        out = list(model.generate_icl_from_ids(target, ref, **kw))
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if i:                                                    # the first pass warms up every shape
            ttfc.append((t1 - t0) * 1e3)
            whole.append((t2 - t1) * 1e3)
            frames = out[0].token_count if out else 0
    res["ttfc_ms_10s_ref"] = float(np.median(ttfc))
    res["whole_call_ms_10s_ref"] = float(np.median(whole))
    res["whole_call_frames"] = frames
    print(f"10 s reference: first streamed chunk (4 frames) after {res['ttfc_ms_10s_ref']:.1f} ms; whole call ({frames} frames) "
          f"{res['whole_call_ms_10s_ref']:.1f} ms", flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
