"""Qwen3-TTS x-vector cloning: what the speaker encoder costs, and what it adds to time-to-first-audio.

Released-size synthetic checkpoints (``synth.qwen3_speaker_encoder_weights`` at the 512 / 1536-channel ECAPA-TDNN config,
``synth.qwen3_talker_weights`` / ``synth.qwen3_tokenizer_weights`` at the public 0.6B shapes).  Prints one JSON object with the card's
name and power limit, read in the same run:
  - ``extract_speaker_embedding``: B = 1 at 3, 10 and 30 s of audio, CUDA events after warm-up (median and max over ``--reps``), and
    the kernel launches per call (``ops.LAUNCHES``);
  - ``generate``: time to the first chunk of ``generate_from_ids(stream=True, ref_audio=3 s)`` against the same call without
    ``ref_audio`` (host clock; every chunk ends in a device synchronise).

    python tools/speaker_encoder_bench.py [--reps 20] [--gen-frames 30] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from qwen3_stream_bench import _card, _timed    # noqa: E402

SPEAKER_ENCODER = {"mel_dim": 128, "enc_dim": 1024, "enc_channels": [512, 512, 512, 512, 1536], "enc_kernel_sizes": [5, 3, 3, 3, 1],
                   "enc_dilations": [1, 2, 3, 4, 1], "enc_attention_channels": 128, "enc_res2net_scale": 8, "enc_se_channels": 128}


def bench_extract(model, reps):
    import numpy as np
    from mlx_audio_b200 import ops
    out = {}
    for sec in (3, 10, 30):
        audio = (0.3 * np.random.default_rng(sec).standard_normal(24000 * sec)).astype(np.float32)
        for _ in range(3):
            model.extract_speaker_embedding(audio)
        l0 = ops.LAUNCHES[0]
        model.extract_speaker_embedding(audio)
        launches = ops.LAUNCHES[0] - l0
        ms = [_timed(lambda: model.extract_speaker_embedding(audio)) for _ in range(reps)]
        out[f"{sec}s"] = {"median_ms": round(statistics.median(ms), 3), "max_ms": round(max(ms), 3), "reps": reps, "launches": launches}
    return out


def bench_first_chunk(model, ids, n_frames, seed=7):
    import numpy as np
    import torch
    u = torch.rand(n_frames, 16, 1, generator=torch.Generator().manual_seed(seed))
    ref = (0.3 * np.random.default_rng(5).standard_normal(72000)).astype(np.float32)
    dev = model.device

    def first(ref_audio):
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        it = model.generate_from_ids(ids, max_tokens=n_frames, u=u, stream=True, streaming_interval=0.5, ref_audio=ref_audio)
        next(it)
        t1 = time.perf_counter()
        list(it)
        torch.cuda.synchronize(dev)
        return t1 - t0

    out = {}
    for tag, ra in (("without_ref_audio", None), ("ref_audio_3s", ref)):
        first(ra)                                            # warm-up: graph capture, decoder shapes, encoder shapes
        t = sorted(first(ra) for _ in range(3))
        out[tag] = {"first_chunk_s_median": round(t[1], 4), "first_chunk_s_max": round(t[2], 4)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--gen-frames", type=int, default=30)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("speaker_encoder_bench: needs a CUDA device")
    from mlx_audio_b200 import configs, synth
    from mlx_audio_b200.tts.models.qwen3_tts import (Model, ModelConfig, Qwen3TTSSpeechTokenizer, Qwen3TTSTalkerCodePredictorConfig,
                                                     Qwen3TTSTalkerConfig, Qwen3TTSTokenizerConfig)
    dev = torch.device("cuda:0")
    name, power = _card()
    flat = dict(configs.QWEN3_TALKER)
    cp = Qwen3TTSTalkerCodePredictorConfig(num_hidden_layers=flat["cp_num_hidden_layers"])
    tc = Qwen3TTSTalkerConfig(code_predictor_config=cp, num_hidden_layers=flat["num_hidden_layers"], text_vocab_size=512,
                              codec_eos_token_id=flat["codec_eos_token_id"])
    model = Model(ModelConfig(talker_config=tc, speaker_encoder_config=SPEAKER_ENCODER, tts_pad_token_id=500, tts_bos_token_id=501,
                              tts_eos_token_id=502), dev)
    w = synth.qwen3_talker_weights(flat, seed=11)
    w.update(synth.qwen3_speaker_encoder_weights(SPEAKER_ENCODER))
    model.load_weights(w)
    tflat = dict(configs.QWEN3_TOKENIZER_DECODER)
    model.load_speech_tokenizer(Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(), dev).load_weights(synth.qwen3_tokenizer_weights(tflat, seed=12)))
    res = {"card": name, "power_limit": power, "extract_speaker_embedding": bench_extract(model, a.reps)}
    ids = torch.randint(0, 500, (40,), generator=torch.Generator().manual_seed(4)).tolist()
    res["generate_stream_first_chunk"] = bench_first_chunk(model, ids, a.gen_frames)
    line = json.dumps(res)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
