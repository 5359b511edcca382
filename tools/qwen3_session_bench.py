"""Continuous batching vs static batches for Qwen3-TTS on one GPU: released-size synthetic weights (28 + 5-layer talker, released
speech-tokenizer decoder), a seeded arrival trace of requests with 20-120 target frames each.

- session: ``Model.create_tts_batch_session(max_batch_size=8)``; arrived requests are added before every step, each request's
  frame cap is its target (``TTSBatchItem.extra["max_tokens"]``);
- static: the same requests in arrival order, as groups of 8 through ``batch_generate_from_ids(stream=False)``; a group starts once
  its last request has arrived and the previous group is done, and runs until its longest request's target (a static batch has no
  per-row cap: its rows run on until the longest one ends).

Both include the audio decode.  A request may end earlier on EOS (the synthetic weights sample it now and then); frames/s and audio-s/s
count the frames each request returned, over wall time from the first arrival to the last completion.  Step time: one ``step()`` of
the session; for the static path, a group's call time over its frames.  The two modes run alternately, ``--rounds`` times each, in one
process; one JSON line per run, with the card's name and power limit.

    python tools/qwen3_session_bench.py --requests 32 --rounds 2
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class _Ids:
    """The request's text is the decimal index of its prepared token ids."""

    def __init__(self, ids):
        self.ids = ids

    def encode(self, text):
        return self.ids[int(text.split("\n")[1].split("<|im_end|>")[0])]


def build(seed=0):
    from mlx_audio_b200 import configs, synth
    from mlx_audio_b200.tts.models.qwen3_tts import (Model, ModelConfig, Qwen3TTSSpeechTokenizer, Qwen3TTSTalkerCodePredictorConfig,
                                                     Qwen3TTSTalkerConfig, Qwen3TTSTokenizerConfig)
    flat = dict(configs.QWEN3_TALKER)
    P = synth.qwen3_talker_weights(flat, seed=11)
    tc = Qwen3TTSTalkerConfig(code_predictor_config=Qwen3TTSTalkerCodePredictorConfig(num_hidden_layers=flat["cp_num_hidden_layers"]),
                              num_hidden_layers=flat["num_hidden_layers"], text_vocab_size=512, codec_eos_token_id=flat["codec_eos_token_id"])
    model = Model(ModelConfig(talker_config=tc, tts_pad_token_id=500, tts_bos_token_id=501, tts_eos_token_id=502), "cuda").load_weights(P)
    st = Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(), "cuda").load_weights(synth.qwen3_tokenizer_weights(dict(configs.QWEN3_TOKENIZER_DECODER), seed=12))
    model.load_speech_tokenizer(st)
    return model


def trace(n, seed, rate):
    g = torch.Generator().manual_seed(seed)
    targets = torch.randint(20, 121, (n,), generator=g).tolist()
    n_ids = torch.randint(8, 60, (n,), generator=g).tolist()
    ids = [torch.randint(10, 500, (k,), generator=g).tolist() for k in n_ids]
    gaps = torch.empty(n).exponential_(rate, generator=g).tolist()
    t, arrivals = 0.0, []
    for gp in gaps:
        arrivals.append(t)
        t += gp
    return targets, ids, arrivals


def run_session(model, targets, arrivals, max_tokens):
    from mlx_audio_b200.tts.continuous import TTSBatchItem, TTSBatchOptions
    s = model.create_tts_batch_session(TTSBatchOptions(max_tokens=max_tokens, max_batch_size=8))
    n, added, done = len(targets), 0, {}
    step_ms = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    while len(done) < n:
        now = time.perf_counter() - t0
        while added < n and arrivals[added] <= now:
            s.add([TTSBatchItem(sequence_id=added, text=str(added), extra={"max_tokens": targets[added]})])
            added += 1
        if s.idle:
            time.sleep(max(0.0, arrivals[added] - now))
            continue
        a = time.perf_counter()
        for e in s.step():
            done[e.sequence_id] = (time.perf_counter() - t0, e.token_count)
        step_ms.append((time.perf_counter() - a) * 1e3)
    return done, step_ms, s.captures


def run_static(model, ids, targets, arrivals):
    n, done, step_ms = len(targets), {}, []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for g0 in range(0, n, 8):
        grp = list(range(g0, min(n, g0 + 8)))
        wait = arrivals[grp[-1]] - (time.perf_counter() - t0)
        if wait > 0:
            time.sleep(wait)
        frames = max(targets[i] for i in grp)
        a = time.perf_counter()
        res = list(model.batch_generate_from_ids([ids[i] for i in grp], max_tokens=frames, seed=g0))
        torch.cuda.synchronize()
        step_ms.append((time.perf_counter() - a) * 1e3 / frames)
        for r in res:
            done[grp[r.sequence_idx]] = (time.perf_counter() - t0, r.token_count)
    return done, step_ms


def summary(mode, done, step_ms, targets, arrivals, extra=None):
    wall = max(t for t, _ in done.values()) - min(arrivals)
    frames = sum(n for _, n in done.values())
    lat = [done[i][0] - arrivals[i] for i in range(len(targets))]
    r = {"mode": mode, "requests": len(targets), "frames": frames, "target_frames": sum(targets), "wall_s": round(wall, 3), "frames_per_s": round(frames / wall, 1),
         "audio_s_per_s": round(frames / 12.5 / wall, 2), "step_ms_median": round(statistics.median(step_ms), 2),
         "step_ms_max": round(max(step_ms), 2), "completion_s_median": round(statistics.median(lat), 3), "completion_s_max": round(max(lat), 3),
         "completion_s": [round(v, 3) for v in lat]}
    r.update(extra or {})
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--rate", type=float, default=4.0, help="mean arrivals per second")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out", default=None, help="write the JSON lines here as well")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qwen3_session_bench: needs a CUDA GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    model = build()
    targets, ids, arrivals = trace(a.requests, a.seed, a.rate)
    model.tokenizer = _Ids(ids)
    # warm-up: both paths once on a short trace (module loads, graph capture paths, decoder shapes)
    run_session(model, [20] * 8, [0.0] * 8, 120)
    run_static(model, ids[:8], [20] * 8, [0.0] * 8)
    lines = []
    for rnd in range(a.rounds):
        done, sms, caps = run_session(model, targets, arrivals, 120)
        lines.append(summary("session", done, sms, targets, arrivals, {"round": rnd, "captures": caps, "card": card}))
        done, sms = run_static(model, ids, targets, arrivals)
        lines.append(summary("static", done, sms, targets, arrivals, {"round": rnd, "card": card}))
    for l in lines:
        print(json.dumps(l))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()
