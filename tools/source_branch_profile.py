"""Where Kokoro's acoustic side spends the time between its fork and its join: the harmonic-source branch against the decoder branch.

Builds the cfg2 model as bench.py does (synthetic checkpoint, 128 phonemes), lets `bench.kokoro_graph_profile` capture both CUDA graphs with
an event node around every launch, and records for each captured launch the stream it was issued on and whether it falls between the
acoustic side's `ops.fork` and `ops.join`.  Launches on the side stream there are the source branch (`ops.kokoro_source`, the two
noise convs, their statistics, the noise-resblock launches); launches on the main stream are the decoder branch (asr / F0 / N
inputs, encode and decode blocks).  After further replays it prints each branch launch's in-graph time, each branch's summed launch
time and its span (first launch start to last launch end), and the fork-to-join span.  The two branches share the SMs, so the summed
times of both exceed the fork-to-join span wherever they overlap.

    python tools/source_branch_profile.py [--reps 20] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("source_branch_profile.py needs a CUDA device")
    import bench
    from mlx_audio_b200 import ops, synth
    from mlx_audio_b200.configs import KOKORO_82M
    from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig

    dev = torch.device("cuda", 0)
    P = synth.kokoro_weights(KOKORO_82M, seed=0)
    model = Model(ModelConfig.from_dict(KOKORO_82M), device=dev).load_weights(list(P.items()))
    model.seed(1234)
    ids, ref_s = synth.kokoro_inputs(bench.N_PHONEMES, seed=1)
    ids_d, ref_d = ids[0].to(dev), ref_s.to(dev)
    audio, _ = model.synthesize_ids(ids_d, ref_d)
    torch.cuda.synchronize(dev)
    F = audio.shape[0] // 600

    log = []                      # ("fork" | "join", None, ...) markers and ("launch", label, stream, kernels, (start, end)) of captured calls
    twins = []
    orig_call, orig_fork, orig_join, orig_synth = ops._call, ops.fork, ops.join, Model.synthesize_ids

    def traced(kind, fn, n, *a):
        label = ops.TAG[0] or f"{sys._getframe(1).f_code.co_name} ({kind})"
        orig_call(kind, fn, n, *a)
        if torch.cuda.is_current_stream_capturing() and ops.PROFILE is not None:
            log.append(("launch", label, torch.cuda.current_stream().cuda_stream, n, ops.PROFILE[kind][-1]))

    def fork(device, n=1):
        if torch.cuda.is_current_stream_capturing():
            log.append(("fork",))
        return orig_fork(device, n)

    def join(device, streams):
        orig_join(device, streams)
        if torch.cuda.is_current_stream_capturing():
            log.append(("join",))

    def synth_ids(self, *a, **k):
        if self is not model and not any(t is self for t in twins):
            twins.append(self)
        return orig_synth(self, *a, **k)

    ops._call, ops.fork, ops.join, Model.synthesize_ids = traced, fork, join, synth_ids
    try:
        bench.kokoro_graph_profile(model, ops, torch, ids_d, ref_d, dev)
    finally:
        ops._call, ops.fork, ops.join, Model.synthesize_ids = orig_call, orig_fork, orig_join, orig_synth
    if not twins:
        raise RuntimeError("bench.kokoro_graph_profile built no second model")

    # the acoustic fork: the last captured fork whose side stream issues ops.kokoro_source before the next join
    seg = None
    for i, e in enumerate(log):
        if e[0] != "fork":
            continue
        j = next((j for j in range(i + 1, len(log)) if log[j][0] == "join"), None)
        if j is not None and any(x[0] == "launch" and x[1].startswith("kokoro_source") for x in log[i + 1:j]):
            seg = (i, j)
    if seg is None:
        raise RuntimeError("no captured fork / join pair around ops.kokoro_source")
    launches = [x for x in log[seg[0] + 1:seg[1]] if x[0] == "launch"]
    src_stream = next(x[2] for x in launches if x[1].startswith("kokoro_source"))
    for _ in range(3):
        twins[0].synthesize_ids(ids_d, ref_d)
    torch.cuda.synchronize(dev)
    base = torch.cuda.Event(enable_timing=True)
    t = [[0.0, 0.0] for _ in launches]
    span = 0.0
    for _ in range(args.reps):
        base.record()
        twins[0].synthesize_ids(ids_d, ref_d)
        torch.cuda.synchronize(dev)
        for i, x in enumerate(launches):
            t[i][0] += base.elapsed_time(x[4][0])
            t[i][1] += base.elapsed_time(x[4][1])
    t = [(s / args.reps, e / args.reps) for s, e in t]
    t0 = min(s for s, _ in t)
    out = {"device": torch.cuda.get_device_name(dev), "frames": F, "reps": args.reps, "branches": {}}
    for name, on_src in (("source", True), ("decoder", False)):
        rows = [(x[1], x[3], (s - t0) * 1e3, (e - s) * 1e3) for x, (s, e) in zip(launches, t) if (x[2] == src_stream) == on_src]
        out["branches"][name] = {"launches": [{"label": l, "kernels": n, "start_us": round(s, 1), "us": round(d, 1)} for l, n, s, d in rows],
                                 "sum_us": round(sum(r[3] for r in rows), 1),
                                 "span_us": round(max(r[2] + r[3] for r in rows) - min(r[2] for r in rows), 1)}
    out["fork_to_join_us"] = round((max(e for _, e in t) - t0) * 1e3, 1)

    print(f"device: {out['device']}; acoustic-side graph of cfg2 (F = {F}), {args.reps} replays; times in us from the first branch launch")
    for name, b in out["branches"].items():
        print(f"\n{name} branch: {len(b['launches'])} calls, summed {b['sum_us']:.1f} us, span {b['span_us']:.1f} us")
        print(f"{'start':>8}{'us':>8}   launch")
        for r in b["launches"]:
            print(f"{r['start_us']:8.1f}{r['us']:8.1f}   {r['label']}")
    print(f"\nfork to join: {out['fork_to_join_us']:.1f} us")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
