"""Where Kokoro's text-side graph spends its time: per-launch in-graph times grouped by ALBERT stage.

Builds the cfg2 model as bench.py does (synthetic checkpoint, 128 phonemes -> T = 130), captures ONLY the text-side CUDA graph with an
external event node around every launch, replays it and prints, per stage, the launches per ALBERT layer and their in-graph time, then
the text-graph replay time and its launch count.  Stages are read off the line of `Model._text_side` that issued each launch, so the
script attributes any version of that function.  The sum of in-graph times over-counts wall time where the text-encoder branch runs
concurrently on its side stream; the replay time is the wall time.  When ALBERT runs as the persistent kernel, eager calls of its
timeline build then give each stage's time per layer and the barrier wait in front of it.

    python tools/text_side_profile.py [--reps 20] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import linecache
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (stage, substring of the issuing source line); first match wins
STAGES = [("ALBERT (persistent)", "albert_encoder"), ("attention", "attention"), ("qkv", 'W["qkv"]'), ("attn_out", 'W["attn_out"]'), ("attn_ln", 'W["attn_ln"]'),
          ("ffn_out", 'W["ffn_out"]'), ("ffn", 'W["ffn"]'), ("full_ln", 'W["full_ln"]'),
          ("embedding", 'W["emb_ln"]'), ("embedding", 'W["map_in"]'), ("embedding", 'W["word_emb"]'),
          ("text encoder branch", "text_branch"), ("bert_encoder", 'W["bert_encoder"]'), ("duration LSTMs + AdaLN", "dur_lstms"),
          ("duration LSTMs + AdaLN", "adaln"), ("duration head", "pred_lstm"), ("duration head", 'W["dur_')]
ALBERT = ["ALBERT (persistent)", "qkv", "attention", "attn_out", "attn_ln", "ffn", "ffn_out", "full_ln"]
KERNEL_STAGES = ["qkv", "attention", "attn_out", "attn_ln", "ffn", "ffn_out", "full_ln"]      # csrc/albert.cu, per layer


def albert_timeline(model, ids, ref_s, layers, reps):
    """Per-stage times of the persistent kernel from its timeline build: globaltimer at the start (after the grid barrier) and end of
    every stage of every CTA.  Returns {stage: (us from the first CTA's start to the last CTA's end, mean us a CTA waits at the
    barrier in front of it)} averaged over layers and eager calls."""
    import torch
    from mlx_audio_b200 import ops
    nsm = torch.cuda.get_device_properties(model.device).multi_processor_count
    tl = torch.zeros(layers * 7, nsm, 2, dtype=torch.int64, device=model.device)
    orig = ops.albert_encoder
    span = [0.0] * 7
    wait = [0.0] * 7
    ops.albert_encoder = lambda *a, **k: orig(*a, **k, timeline=tl)
    try:
        for _ in range(reps + 1):
            model._text_side(ids, ref_s)
            torch.cuda.synchronize()
            t = tl.double().cpu()
            if _ == 0:
                continue                                               # warm-up
            for k in range(layers * 7):
                span[k % 7] += float(t[k, :, 1].max() - t[k, :, 0].min()) / 1e3
                if k:
                    wait[k % 7] += float((t[k, :, 0] - t[k - 1, :, 1]).mean()) / 1e3
    finally:
        ops.albert_encoder = orig
    n = reps * layers
    return {st: (span[i] / n, wait[i] / n) for i, st in enumerate(KERNEL_STAGES)}


def _stage() -> str:
    f = sys._getframe(2)
    while f is not None:
        if f.f_code.co_name == "_text_side":
            line = linecache.getline(f.f_code.co_filename, f.f_lineno)
            for name, key in STAGES:
                if key in line:
                    return name
            return "other"
        f = f.f_back
    return "other"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("text_side_profile.py needs a CUDA device")
    from mlx_audio_b200 import ops, synth
    from mlx_audio_b200.configs import KOKORO_82M
    from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig

    dev = torch.device("cuda", 0)
    P = synth.kokoro_weights(KOKORO_82M, seed=0)
    model = Model(ModelConfig.from_dict(KOKORO_82M), device=dev).load_weights(list(P.items()))
    ids, ref_s = synth.kokoro_inputs(128, seed=1)
    T = ids.shape[1]
    layers = KOKORO_82M["plbert"]["num_hidden_layers"]

    rec = []                                   # (stage, entry point, kernels, start event, end event) of the captured launches
    orig = ops._call

    def traced(kind, fn, n, *a):
        if not torch.cuda.is_current_stream_capturing():
            return orig(kind, fn, n, *a)
        e0 = torch.cuda.Event(enable_timing=True, external=True)
        e1 = torch.cuda.Event(enable_timing=True, external=True)
        e0.record()
        orig(kind, fn, n, *a)
        e1.record()
        rec.append((_stage(), getattr(fn, "__name__", kind), n, e0, e1))

    ops._call = traced
    try:
        ent = model._text_graph(T, 1.0, False)
    finally:
        ops._call = orig
    ent["ids"].copy_(ids[0].to(dev))
    ent["ref_s"].copy_(ref_s.to(dev))
    g = ent["graph"]

    per = [0.0] * len(rec)
    base = torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        g.replay()
    for _ in range(args.reps):
        base.record()
        g.replay()
        torch.cuda.synchronize(dev)
        for i, (_, _, _, e0, e1) in enumerate(rec):
            per[i] += base.elapsed_time(e1) - base.elapsed_time(e0)
    per = [1e3 * t / args.reps for t in per]                                    # us

    plain = torch.cuda.CUDAGraph()                  # replay time of the uninstrumented graph
    with torch.cuda.graph(plain, pool=model._graph_pool if model.share_graph_pool else None):
        model._text_side(ent["ids"], ent["ref_s"], 1.0, None)
    for _ in range(3):
        plain.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(dev)
    a.record()
    for _ in range(args.reps):
        plain.replay()
    b.record()
    torch.cuda.synchronize(dev)
    replay_ms = a.elapsed_time(b) / args.reps

    stages = {}
    for (st, fn, n, _, _), us in zip(rec, per):
        d = stages.setdefault(st, {"kernels": 0, "us": 0.0, "entry_points": {}})
        d["kernels"] += n
        d["us"] += us
        e = d["entry_points"].setdefault(fn, {"kernels": 0, "us": 0.0})
        e["kernels"] += n
        e["us"] += us
    name = torch.cuda.get_device_name(dev)
    print(f"device: {name}; text-side graph of cfg2 (T = {T}), {args.reps} replays")
    print(f"{'stage':<24}{'kernels/layer':>14}{'us/layer':>10}{'us total':>10}   entry points (kernels, us total)")
    albert_us = albert_k = 0
    for st in ALBERT + sorted(k for k in stages if k not in ALBERT):
        if st not in stages:
            continue
        d = stages[st]
        div = layers if st in ALBERT else 1
        if st in ALBERT:
            albert_us += d["us"]
            albert_k += d["kernels"]
        eps = ", ".join(f"{k} ({v['kernels']}, {v['us']:.0f})" for k, v in sorted(d["entry_points"].items()))
        kl = f"{d['kernels'] / div:.0f}" if st in ALBERT else "-"
        ul = f"{d['us'] / div:.1f}" if st in ALBERT else "-"
        print(f"{st:<24}{kl:>14}{ul:>10}{d['us']:>10.1f}   {eps}")
    n_kernels = sum(n for _, _, n, _, _ in rec)
    print(f"ALBERT layers: {albert_k / layers:.0f} kernels and {albert_us / layers:.1f} us per layer, {albert_us:.1f} us in all")
    print(f"text graph: {n_kernels} kernels, replay {replay_ms:.3f} ms")
    timeline = None
    if "ALBERT (persistent)" in stages:
        timeline = albert_timeline(model, ids[0].to(dev), ref_s.to(dev), layers, args.reps)
        print("persistent ALBERT kernel, timeline build (eager calls), per layer:")
        print(f"{'stage':<12}{'us':>8}{'barrier wait us':>17}")
        for st, (us, w) in timeline.items():
            print(f"{st:<12}{us:>8.1f}{w:>17.1f}")
        print(f"{'sum':<12}{sum(v[0] for v in timeline.values()):>8.1f}{sum(v[1] for v in timeline.values()):>17.1f}")
    res = {"device": name, "T": T, "reps": args.reps, "text_graph_ms": round(replay_ms, 4), "text_graph_kernels": n_kernels,
           "albert_kernels_per_layer": albert_k / layers, "albert_us_per_layer": round(albert_us / layers, 2),
           "stages": {k: {"kernels": v["kernels"], "us": round(v["us"], 1),
                          "entry_points": {e: {"kernels": x["kernels"], "us": round(x["us"], 1)} for e, x in v["entry_points"].items()}}
                      for k, v in stages.items()},
           "albert_timeline_us": None if timeline is None else {k: {"us": round(v[0], 2), "barrier_wait_us": round(v[1], 2)}
                                                               for k, v in timeline.items()}}
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
