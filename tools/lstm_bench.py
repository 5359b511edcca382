"""Kokoro's bidirectional LSTM recurrence (`ops.lstm_bidir`, csrc/lstm.cu) on its own: time per launch and per sequential step.

At each (B, T) of --shapes, 20 launches on the same inputs are captured in one CUDA graph; the graph is replayed --reps times between
CUDA events and the median replay is reported.  A launch runs T sequential steps (both directions concurrently, B clusters per
direction), so `us_per_step` = launch time / T is the recurrence's step latency.  Prints one JSON object with the card's name, power
limit and SM clock, read in the same run right after the timing.

    python tools/lstm_bench.py [--reps 10] [--shapes 1x130,1x390,2x130] [--json OUT]
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

H = 256
LAUNCHES = 20


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, sm, sm_max = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return {"card": name, "power_limit": power, "clocks_sm": sm, "clocks_max_sm": sm_max}
    except Exception as e:                                  # the timing does not depend on it; report what failed
        return {"card": f"unknown ({e})"}


def bench(B, T, reps, dev):
    import torch
    from mlx_audio_b200 import ops
    g = torch.Generator().manual_seed(7)
    xproj = (torch.randn(B, T, 8 * H, generator=g) * 1.3).to(dev)
    wh = (torch.randn(2, 4 * H, H, generator=g) * 0.08).to(dev).contiguous()
    out = torch.empty(B, T, 2 * H, device=dev)
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        for _ in range(3):                                  # module load and warm-up outside the capture
            ops.lstm_bidir(xproj, wh, out=out)
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(LAUNCHES):
                ops.lstm_bidir(xproj, wh, out=out)
        graph.replay()
        s.synchronize()
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            graph.replay()
            e1.record(s)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
    us = statistics.median(ms) * 1e3 / LAUNCHES
    return {"B": B, "T": T, "us_per_launch": round(us, 2), "us_per_step": round(us / T, 4),
            "us_per_launch_min": round(min(ms) * 1e3 / LAUNCHES, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--shapes", default="1x130,1x390,2x130")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lstm_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    shapes = [tuple(int(v) for v in s.split("x")) for s in a.shapes.split(",")]
    res = {"launches_per_graph": LAUNCHES, "shapes": [bench(B, T, a.reps, dev) for B, T in shapes]}
    res.update(_card())
    line = json.dumps(res)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
