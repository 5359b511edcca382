"""Mimi streaming: what one incremental ``decode_step`` / ``encode_step`` costs, and how that depends on the position in the stream.

Released-size synthetic weights (``synth.mimi_weights(MIMI_202407)``), B = 1.  Prints one JSON object with the card's name and power limit:
  - ``decode_step``: per-frame time (median and max of ``--frames`` single-frame calls, CUDA events) at stream positions of about 10, 250,
    1000 and 3000 frames, through the captured CUDA graph and eagerly; the stream is brought to each position in 128-frame chunks;
  - ``redecode``: the same frames through the route ``decode_step`` replaces, a one-shot ``decode(codes[:, :, :t])`` sliced (median of 3);
  - ``eager_breakdown``: one eager single-frame step at position ~250 split by launch label (ops.PROFILE_TAGS), the largest first -- the
    transformer's 2-row linears are the ``[1x2x...]`` conv entries;
  - ``encode_step``: per 1920-sample chunk over a 200-frame stream.

    python tools/mimi_stream_bench.py [--frames 20] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

POSITIONS = (10, 250, 1000, 3000)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:                                  # the timing does not depend on it; report what failed
        return f"unknown ({e})", "unknown"


def _stats(ms):
    return {"median_ms": round(statistics.median(ms), 3), "max_ms": round(max(ms), 3), "n": len(ms)}


def _timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def _advance_to(model, codes, t):
    """Reset and stream frames [0, t) in 128-frame chunks (state identical to any other chunking)."""
    model.reset_state()
    for a in range(0, t, 128):
        model.decode_step(codes[:, :, a:min(a + 128, t)])


def bench_decode(model, codes, n):
    from mlx_audio_b200.codec.models import mimi as MM
    out = {}
    for graph in (True, False):
        MM.GRAPH_SINGLE_FRAME[0] = graph
        res = {}
        for p in POSITIONS:
            _advance_to(model, codes, p)
            model.decode_step(codes[:, :, p:p + 1])          # the eager warm-up step (graph mode captures at the next one)
            model.decode_step(codes[:, :, p + 1:p + 2])
            ms = [_timed(lambda t=t: model.decode_step(codes[:, :, t:t + 1])) for t in range(p + 2, p + 2 + n)]
            res[str(p)] = _stats(ms)
        out["graph" if graph else "eager"] = res
    MM.GRAPH_SINGLE_FRAME[0] = True
    red = {}
    for p in POSITIONS:
        model.decode(codes[:, :, :p + 1])
        red[str(p)] = _stats([_timed(lambda: model.decode(codes[:, :, :p + 1])[..., -1920:]) for _ in range(3)])
    out["redecode"] = red
    return out


def eager_breakdown(model, codes, p=250):
    import torch
    from mlx_audio_b200 import ops
    from mlx_audio_b200.codec.models import mimi as MM
    MM.GRAPH_SINGLE_FRAME[0] = False
    _advance_to(model, codes, p)
    model.decode_step(codes[:, :, p:p + 1])
    ops.PROFILE, ops.PROFILE_TAGS = {}, {}
    try:
        model.decode_step(codes[:, :, p + 1:p + 2])
        torch.cuda.synchronize()
        tot = {}
        for kind, evs in ops.PROFILE.items():
            for (a, b), tag in zip(evs, ops.PROFILE_TAGS.get(kind, [None] * len(evs))):
                key = f"{kind}: {tag or '(stream / ring kernels)'}"
                tot[key] = tot.get(key, 0.0) + a.elapsed_time(b)
    finally:
        ops.PROFILE, ops.PROFILE_TAGS = None, None
        MM.GRAPH_SINGLE_FRAME[0] = True
    rows = sorted(tot.items(), key=lambda kv: -kv[1])
    return {"sum_ms": round(sum(tot.values()), 3), "by_label_ms": {k: round(v, 4) for k, v in rows[:12]}, "labels": len(rows)}


def bench_encode(model, pcm):
    model.reset_state()
    for a in range(0, 1920 * 5, 1920):                      # warm-up
        model.encode_step(pcm[:, :, a:a + 1920])
    model.reset_state()
    ms = [_timed(lambda a=a: model.encode_step(pcm[:, :, a:a + 1920])) for a in range(0, pcm.shape[-1], 1920)]
    return _stats(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mimi_stream_bench: needs a CUDA device")
    from mlx_audio_b200 import configs, synth
    from mlx_audio_b200.codec import Mimi, mimi_202407
    dev = torch.device("cuda:0")
    name, power = _card()
    model = Mimi(mimi_202407(32), device=dev).load_weights(synth.mimi_weights(configs.MIMI_202407, encoder=True))
    codes = synth.mimi_codes(configs.MIMI_202407, max(POSITIONS) + a.frames + 4, 1).to(dev)
    res = {"card": name, "power_limit": power, "batch": 1, "decode_step": bench_decode(model, codes, a.frames),
           "eager_breakdown": eager_breakdown(model, codes)}
    pcm = (torch.randn(1, 1, 1920 * 200, generator=torch.Generator().manual_seed(3)) * 0.3).to(dev)
    res["encode_step_1920"] = bench_encode(model, pcm)
    line = json.dumps(res)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
