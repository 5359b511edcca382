"""BigVGAN: what a vocoder call costs on the GPU, where the time goes, and what the one-pass anti-aliased activation buys.

Released-size synthetic weights (``synth.bigvgan_weights``), the 22 kHz / 80-band / 256x and 44 kHz / 128-band / 512x configurations of
the reference's tests, B = 1 and B = 4, 800 mel frames.  Prints one JSON object with the card's name and power limit; timings are the
median and max of ``--reps`` calls (CUDA events, after warm-up):
  - ``call``: the whole ``model(mel)`` and the audio-seconds it makes per second;
  - ``stages``: one profiled call split by up-sampling stage (and conv_pre / the final activation + conv_post), each stage's time by
    kernel kind: ``conv_tc`` (tensor cores), ``conv`` / ``other`` (CUDA cores), ``prep`` (bf16 operand split), ``aa_act`` (activation);
  - ``activation``: ``ops.aa_snakebeta`` alone at every stage's shape (B = 1, 22 kHz), its achieved bytes/s (one fp32 read and one fp32
    write per element) against the 3.35 TB/s of the H100 SXM data sheet, alternated call by call with the reference's four-pass route in
    torch ops (edge pad, grouped conv_transpose1d, SnakeBeta, edge pad + strided grouped conv1d), and the two routes' largest difference.
There is no CPU fall-back: without a GPU the script fails.

    python tools/bigvgan_bench.py [--reps 10] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RESBLOCKS = dict(resblock="1", resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
                 activation="snakebeta", snake_logscale=True)
CONFIGS = {"bigvgan_22khz_80band_256x": (dict(num_mels=80, upsample_rates=[4, 4, 2, 2, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4, 4, 4],
                                              upsample_initial_channel=1536, use_bias_at_final=True, use_tanh_at_final=True, **RESBLOCKS), 22050),
           "bigvgan_44khz_128band_512x": (dict(num_mels=128, upsample_rates=[8, 4, 2, 2, 2, 2], upsample_kernel_sizes=[16, 8, 4, 4, 4, 4],
                                               upsample_initial_channel=1536, use_bias_at_final=False, use_tanh_at_final=False, **RESBLOCKS), 44100)}
FRAMES = 800
HBM_BYTES_PER_S = 3.35e12


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:                                  # the timing does not depend on it; report what failed
        return f"unknown ({e})", "unknown"


def _timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def _stats(ms, audio_s=None):
    med = statistics.median(ms)
    out = {"median_ms": round(med, 3), "max_ms": round(max(ms), 3), "n": len(ms)}
    if audio_s:
        out["audio_s_per_s"] = round(audio_s / (med * 1e-3), 1)
    return out


def _alternate(fns, reps, warm=2):
    """Time several routes call by call in turn, so that drift of the shared machine lands on all of them alike."""
    for _ in range(warm):
        for f in fns.values():
            f()
    ms = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            ms[k].append(_timed(f))
    return ms


def stages(model, mel):
    """One call with every launch bracketed by events (ops.PROFILE), the launches grouped by the stage that issued them."""
    import torch
    from mlx_audio_b200 import ops
    W, out = model._W, []

    def run(name, fn):
        ops.PROFILE = {}
        try:
            r = fn()
            torch.cuda.synchronize()
            kinds = {k: round(sum(a.elapsed_time(b) for a, b in v), 3) for k, v in ops.PROFILE.items()}
        finally:
            ops.PROFILE = None
        out.append({"stage": name, "ms": round(sum(kinds.values()), 3), "by_kind": kinds})
        return r

    with torch.no_grad():
        x = run("conv_pre", lambda: ops.conv1d(mel.transpose(1, 2).contiguous(), W["pre"], pad_left=3))
        for i, st in enumerate(W["stages"]):
            def stage(x=x, st=st):
                u, k, L = st["u"], st["k"], x.shape[1]
                p = (k - u) // 2
                y = ops.conv1d(x, st["up"], stride=u, pad_left=p, lout=(L - 1) * u - 2 * p + k, transpose=True)
                acc = torch.empty_like(y)
                for j, blk in enumerate(st["blocks"]):
                    model._amp(y, blk, acc, j > 0)
                return acc
            x = run(f"stage{i} [{x.shape[1] * st['u']} rows x {st['up'].cout} ch]", stage)
        run("activation_post + conv_post", lambda: ops.conv1d(ops.aa_snakebeta(x, *W["post_act"]), W["post"], pad_left=3))
    return out


def activation(model, reps):
    """aa_snakebeta at each stage's shape against the reference's four-pass route in torch ops, alternated."""
    import torch
    import torch.nn.functional as F
    from mlx_audio_b200 import ops
    res = []
    L = FRAMES
    g = torch.Generator().manual_seed(1)
    for st in model._W["stages"]:
        L *= st["u"]
        a, ib, fu, fd = st["blocks"][0]["units"][0]["a1"]
        C = a.numel()
        x = torch.randn(1, L, C, generator=g).cuda()
        xc = x.transpose(1, 2).contiguous()                                    # the torch route runs channels-first: [B, C, L]
        wu, wd = fu.reshape(1, 1, 12).expand(C, 1, 12).contiguous(), fd.reshape(1, 1, 12).expand(C, 1, 12).contiguous()
        a3, ib3 = a.reshape(1, C, 1), ib.reshape(1, C, 1)

        def four_pass():
            # torch's conv_transpose1d is the same scatter as MLX's, y[2i + k] += x[i] w[k], with no flip
            u = 2 * F.conv_transpose1d(F.pad(xc, (5, 5), mode="replicate"), wu, stride=2, groups=C)[:, :, 15:-15]
            v = u + ib3 * torch.sin(a3 * u) ** 2
            return F.conv1d(F.pad(v, (5, 6), mode="replicate"), wd, stride=2, groups=C)

        ours = ops.aa_snakebeta(x, a, ib, fu, fd)
        ref = four_pass().transpose(1, 2)
        ms = _alternate({"one_pass": lambda: ops.aa_snakebeta(x, a, ib, fu, fd), "four_pass_torch": four_pass}, reps)
        med = statistics.median(ms["one_pass"])
        nbytes = 2 * L * C * 4
        res.append({"rows": L, "channels": C, "one_pass": _stats(ms["one_pass"]), "four_pass_torch": _stats(ms["four_pass_torch"]),
                    "one_pass_GB_per_s": round(nbytes / (med * 1e-3) / 1e9, 1), "share_of_3.35TB_per_s": round(nbytes / (med * 1e-3) / HBM_BYTES_PER_S, 3),
                    "speedup": round(statistics.median(ms["four_pass_torch"]) / med, 2),
                    "max_diff_rel": float((ours - ref).abs().max() / ref.abs().max())})
        del x, xc
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bigvgan_bench.py needs a GPU: it measures the CUDA path and has no fall-back")
    from mlx_audio_b200 import synth
    from mlx_audio_b200.codec import BigVGAN, BigVGANConfig
    name, power = _card()
    reps = max(10, args.reps)
    res = {"card": name, "power_limit": power, "reps": reps, "mel_frames": FRAMES}
    for tag, (cfg, sr) in CONFIGS.items():
        c = BigVGANConfig(**cfg)
        model = BigVGAN(c, device="cuda").load_weights(synth.bigvgan_weights(c))
        hop = math.prod(cfg["upsample_rates"])
        r = {"sample_rate": sr, "audio_s_per_item": round(FRAMES * hop / sr, 3)}
        for B in (1, 4):
            mel = torch.randn(B, cfg["num_mels"], FRAMES, generator=torch.Generator().manual_seed(B)).cuda()
            for _ in range(2):
                model(mel)
            r[f"call_B{B}"] = _stats([_timed(lambda: model(mel)) for _ in range(reps)], B * FRAMES * hop / sr)
            if B == 1:
                r["stages_B1"] = stages(model, mel)
        if tag.startswith("bigvgan_22khz"):
            r["activation_B1"] = activation(model, reps)
        res[tag] = r
        del model
        torch.cuda.empty_cache()
    text = json.dumps(res, indent=1)
    print(text)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
