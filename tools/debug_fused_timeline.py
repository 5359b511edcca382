#!/usr/bin/env python
"""Per-launch attribution of csrc/conv_fused.cu on the launches Kokoro actually makes (run on the GPU box).

The problem lists come from the model: one eager `Model.forward_ids` at bench.py's cfg2 (128 phonemes, F = 390, synthetic checkpoint)
is run with `ops.conv_fused` wrapped, and every launch of `_acoustic_side_fused` is kept, inputs, statistics and residuals included.
By default the 3-problem launches (the generator stages' k = 3 / 7 / 11 resblock groups) are reported; --all reports every launch,
--only SUBSTR those whose label contains SUBSTR.  Per launch:

  us        un-instrumented: 20 launches of the same problems in one CUDA graph, CUDA events
  TFLOP/s   2 M N Cin taps x products (hi*hi + lo*hi [+ hi*lo]) over that time, both planes counted
  MMA       the DBG build's per-CTA mean of the MMA warpgroups' wait cycles: on `full` (weight stage), `a_full` (A chunk), `tempty`
            (output tile), and inside wgmma.wait_group, as a share of the CTA's lifetime
  workers   mean per-CTA cycles converting / in epilogues, and waiting on a_empty / tfull; the producer's wait on `empty`
  CTA end   spread of the CTAs' last timestamps (the scheduling tail)

--probe runs the largest generator group once more with parts of the workers' work switched off (B2A_FUSED_DBGFLAGS, results
garbage, see PROBES): with conversion and epilogue both off, the rate the MMA and the weight feed reach alone, to set against the card.
The card's name, power limit and clocks are read in the same run.
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from mlx_audio_b200 import ops, _lib, synth
from mlx_audio_b200.configs import KOKORO_82M
from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig

DEV = "cuda:0"
# B2A_FUSED_DBGFLAGS of the rate probes (csrc/conv_fused.cu FParams::dbg_flags); 48 is the MMA and weight feed alone
PROBES = {48: "no conversion, no epilogue", 16: "no conversion", 32: "no epilogue", 1: "conversion without its global loads",
          2: "conversion without its shared-memory stores", 4: "conversion without the proxy fence"}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def max_sm_mhz():
    try:
        return float(card().split(",")[3].split()[0])
    except (IndexError, ValueError):
        return 1980.0


def record():
    """[(label, [FusedProblem])] of every fused launch of one acoustic side at cfg2."""
    P = synth.kokoro_weights(KOKORO_82M, seed=0)
    model = Model(ModelConfig.from_dict(KOKORO_82M), device=DEV).load_weights(list(P.items()))
    model.seed(1234)
    ids, ref_s = synth.kokoro_inputs(128, seed=1)
    launches, on = [], [False]
    orig_launch, orig_side = ops.conv_fused, model._acoustic_side_fused

    def launch(problems):
        if on[0]:
            launches.append([problems] if isinstance(problems, ops.FusedProblem) else list(problems))
        return orig_launch(problems)

    def side(*a, **k):
        on[0] = True
        try:
            return orig_side(*a, **k)
        finally:
            on[0] = False

    ops.conv_fused, model._acoustic_side_fused = launch, side
    try:
        with torch.no_grad():
            model.forward_ids(ids[0].to(DEV), ref_s.to(DEV))
        torch.cuda.synchronize()
    finally:
        ops.conv_fused = orig_launch
    out = []
    for i, probs in enumerate(launches):
        parts = []
        for pr in probs:
            q = pr.p
            dil = q.shifts[1] - q.shifts[0] if q.taps > 1 else 1
            parts.append(f"{q.L}x{q.Cin}->{q.N} k{q.taps}" + (f" d{dil}" if dil != 1 else "") + (f" up{q.up_stride}" if q.up_stride else ""))
        out.append((f"#{i:02d} " + " + ".join(parts), probs))
    return out


def flops(probs):
    prod = 2 if ops.TC_MODE[0] == "x2" else 1
    f = 0
    for pr in probs:
        q = pr.p
        rows = q.L + q.taps - 1 if q.up_stride else q.Lout
        f += 2 * rows * q.N * q.Cin * q.taps * (prod + (1 if q.w_lo else 0))
    return f


def time_launch(probs, n=20):
    for _ in range(3):
        ops.conv_fused(probs)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            ops.conv_fused(probs)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def attribute(probs, mhz):
    stamps = torch.zeros(132, 32, dtype=torch.int64, device=DEV)
    _lib.lib().b2a_conv1d_fused_debug(stamps.data_ptr())
    ops.conv_fused(probs)
    torch.cuda.synchronize()
    _lib.lib().b2a_conv1d_fused_debug(None)
    s = stamps.cpu()
    live = s[:, 0] > 0
    t0 = int(s[live, 0].min())
    life_us = (s[live, 13] - s[live, 0]).double().mean().item() / 1e3
    cyc = s[live].double().mean(dim=0) / mhz                    # SM cycles -> us at the card's maximum SM clock
    mma = cyc[26:30] / 2                                        # per MMA warpgroup
    pct = lambda v: 100.0 * v / life_us
    end = ((s[live, 13] - t0).double() / 1e3)
    print(f"    MMA waits per CTA (lifetime {life_us:.1f} us): full {mma[0]:.1f} ({pct(mma[0]):.0f}%), a_full {mma[1]:.1f} ({pct(mma[1]):.0f}%), "
          f"tempty {mma[2]:.1f} ({pct(mma[2]):.0f}%), wgmma.wait_group {mma[3]:.1f} ({pct(mma[3]):.0f}%)")
    print(f"    workers: convert {cyc[24]:.1f} (a_empty {cyc[19]:.1f}), epilogue {cyc[25]:.1f} (tfull {cyc[20]:.1f}); producer loop {cyc[21]:.1f} "
          f"(empty {cyc[22]:.1f}) us")
    print(f"    CTA end: min {end.min():.1f} median {end.median():.1f} max {end.max():.1f} us (instrumented run)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--all", action="store_true", help="every fused launch of the acoustic side, not only the generator groups")
    ap.add_argument("--only", default=None, help="launches whose label contains this string")
    ap.add_argument("--probe", action="store_true", help="also run the no-conversion rate probe (in a child process)")
    ap.add_argument("--probe-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    ops.TC_MODE[0] = os.environ.get("TC", "x2")
    launches = record()
    if args.probe_child:
        label, probs = max((l for l in launches if len(l[1]) == 3), key=lambda l: flops(l[1]))
        us = time_launch(probs)
        what = PROBES[int(os.environ["B2A_FUSED_DBGFLAGS"])]
        print(f"probe ({what}) {label}: {us:.1f} us, {flops(probs) / us / 1e6:.0f} TFLOP/s; card after: {card()}")
        return
    print(f"card: {card()}; tensor-core mode {ops.TC_MODE[0]}")
    mhz = max_sm_mhz()
    sel = [l for l in launches if (args.all or len(l[1]) == 3) and (args.only is None or args.only in l[0])]
    total = 0.0
    for label, probs in sel:
        us = time_launch(probs)
        total += us
        print(f"== {label}: {us:.1f} us, {flops(probs) / us / 1e6:.0f} TFLOP/s")
        attribute(probs, mhz)
    print(f"sum over {len(sel)} launches: {total:.1f} us (each timed on its own, warm L2)")
    if args.probe:
        for flags in PROBES:
            env = dict(os.environ, B2A_FUSED_DBGFLAGS=str(flags))
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--probe-child"], env=env, stdout=subprocess.PIPE,
                               stderr=subprocess.STDOUT, text=True)
            print(r.stdout.strip().splitlines()[-1] if r.stdout.strip() else f"probe {flags} failed ({r.returncode})")
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
