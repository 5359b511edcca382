"""Qwen3-TTS streaming: what the incremental speech-tokenizer decoder costs per chunk, and what streaming does to time-to-first-audio.

Full-size synthetic checkpoints (``synth.qwen3_tokenizer_weights``, ``synth.qwen3_talker_weights``, the public 0.6B shapes).  Prints one
JSON object with the card's name and power limit:
  - ``streaming_step``: time per chunk (median and max, CUDA events) over a 250-frame stream in 1-, 6- and 25-frame chunks, next to the
    same chunks re-decoded with 25 frames of left context (``decoder(codes[start - 25 : end])``, what ``streaming_decode`` does);
  - ``generate``: time to the first chunk of ``generate_from_ids(stream=True)`` at ``streaming_interval`` 0.5 and 2.0 s, and the total
    time of the same call with ``stream=False`` (host clock; every chunk ends in a device synchronise).

    python tools/qwen3_stream_bench.py [--frames 250] [--gen-frames 60] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:                                  # the timing does not depend on it; report what failed
        return f"unknown ({e})", "unknown"


def _stats(ms):
    return {"median_ms": round(statistics.median(ms), 3), "max_ms": round(max(ms), 3), "chunks": len(ms)}


def _timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def bench_decoder(st, codes, sizes=(1, 6, 25), ctx=25):
    dec, T = st.decoder, codes.shape[-1]
    out = {}
    for n in sizes:
        spans = [(s, min(s + n, T)) for s in range(0, T, n)]
        for rep in range(2):                                 # rep 0 warms every shape the timed pass uses
            dec.reset_streaming_state()
            step = [_timed(lambda s=s, e=e: dec.streaming_step(codes[:, :, s:e])) for s, e in spans]
            redo = [_timed(lambda s=s, e=e: dec(codes[:, :, max(0, s - ctx):e])) for s, e in spans]
        dec.reset_streaming_state()
        out[f"{n}_frames"] = {"streaming_step": _stats(step), "redecode_ctx25": _stats(redo),
                              "median_ratio": round(statistics.median(step) / statistics.median(redo), 3)}
    return out


def bench_generate(model, ids, n_frames, seed=7):
    import torch
    from mlx_audio_b200 import configs
    u = torch.rand(n_frames, configs.QWEN3_TALKER["num_code_groups"], 1, generator=torch.Generator().manual_seed(seed))
    dev = model.device

    def first_chunk(interval):
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        it = model.generate_from_ids(ids, max_tokens=n_frames, u=u, stream=True, streaming_interval=interval)
        first = next(it)
        t1 = time.perf_counter()
        rest = list(it)
        torch.cuda.synchronize(dev)
        return t1 - t0, time.perf_counter() - t0, first.token_count, first.token_count + sum(r.token_count for r in rest)

    def whole():
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        res = list(model.generate_from_ids(ids, max_tokens=n_frames, u=u))
        torch.cuda.synchronize(dev)
        return time.perf_counter() - t0, res[0].token_count if res else 0

    out = {}
    whole()                                                  # warm-up: graph capture, every decoder shape
    for interval in (0.5, 2.0):
        first_chunk(interval)
        t_first, t_total, n_first, n = first_chunk(interval)
        out[f"stream_interval_{interval}"] = {"first_chunk_s": round(t_first, 4), "first_chunk_frames": n_first, "total_s": round(t_total, 4),
                                              "frames": n}
    t, n = whole()
    out["stream_false"] = {"total_s": round(t, 4), "frames": n}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=250)
    ap.add_argument("--gen-frames", type=int, default=60)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("qwen3_stream_bench: needs a CUDA device")
    from mlx_audio_b200 import configs, synth
    from mlx_audio_b200.tts.models.qwen3_tts import (Model, ModelConfig, Qwen3TTSSpeechTokenizer, Qwen3TTSTalkerCodePredictorConfig,
                                                     Qwen3TTSTalkerConfig, Qwen3TTSTokenizerConfig)
    dev = torch.device("cuda:0")
    name, power = _card()
    tflat = dict(configs.QWEN3_TOKENIZER_DECODER)
    st = Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(), dev).load_weights(synth.qwen3_tokenizer_weights(tflat, seed=12))
    codes = synth.qwen3_codes(tflat, a.frames, batch=1, seed=1).to(dev)
    res = {"card": name, "power_limit": power, "stream_frames": a.frames, "decoder": bench_decoder(st, codes)}
    flat = dict(configs.QWEN3_TALKER)
    cp = Qwen3TTSTalkerCodePredictorConfig(num_hidden_layers=flat["cp_num_hidden_layers"])
    tc = Qwen3TTSTalkerConfig(code_predictor_config=cp, num_hidden_layers=flat["num_hidden_layers"], text_vocab_size=512,
                              codec_eos_token_id=flat["codec_eos_token_id"])
    model = Model(ModelConfig(talker_config=tc, tts_pad_token_id=500, tts_bos_token_id=501, tts_eos_token_id=502), dev)
    model.load_weights(synth.qwen3_talker_weights(flat, seed=11))
    model.load_speech_tokenizer(st)
    ids = torch.randint(0, 500, (40,), generator=torch.Generator().manual_seed(4)).tolist()
    res["generate"] = bench_generate(model, ids, a.gen_frames)
    line = json.dumps(res)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
