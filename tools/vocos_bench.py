"""Vocos: what a vocoder call costs on the GPU, where the time goes, and what the two fused kernels buy.

Released-size synthetic weights (``synth.vocos_weights``) for the mel checkpoint (512 / 1536 / 8 layers, n_fft 1024, hop 256) and the
EnCodec-feature one (384 / 1152 / 8 layers with AdaLayerNorm, n_fft 1280, hop 320), 10 s at 24 kHz, B = 1, 8 and 32.  Prints one JSON
object with the card's name and power limit; timings are the median and max of ``--reps`` calls (CUDA events, after warm-up):
  - ``calls``: ``model(audio)`` and ``model.decode(features)``, audio-seconds per second, kernel launches per call (``ops.LAUNCHES``);
  - ``split``: one profiled call of each by kernel kind: ``logmel``, ``vocos_norm`` (dwnorm), ``conv_tc`` (tensor-core GEMMs and the
    embedding conv), ``vocos_head``, everything else;
  - ``dwnorm``: ``ops.vocos_dwnorm`` (planes out) at a block's shape, alternated call by call with the two-launch route it replaces
    (``ops.conv1d`` depthwise + ``ops.layernorm(planes=True)``);
  - ``head``: ``ops.vocos_istft_head`` alternated with spectrum formation in torch ops + ``dsp.istft``, and the largest difference.
There is no CPU fall-back: without a GPU the script fails.

    python tools/vocos_bench.py [--reps 10] [--json OUT]
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

SR, SECONDS = 24_000, 10.0


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
    out = {"median_ms": round(statistics.median(ms), 4), "max_ms": round(max(ms), 4)}
    if audio_s:
        out["audio_s_per_s"] = round(audio_s / (statistics.median(ms) / 1e3), 1)
    return out


def _split(fn):
    import torch
    from mlx_audio_b200 import ops
    ops.PROFILE = {}
    fn()
    torch.cuda.synchronize()
    prof, ops.PROFILE = ops.PROFILE, None
    return {k: round(sum(a.elapsed_time(b) for a, b in v), 4) for k, v in sorted(prof.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from mlx_audio_b200 import dsp, ops, synth
    from mlx_audio_b200.configs import VOCOS_ENCODEC_24K, VOCOS_MEL_24K
    from mlx_audio_b200.codec import Vocos
    from mlx_audio_b200.codec.models.vocos import hanning

    name, power = _card()
    res = {"card": name, "power_limit": power, "seconds_of_audio": SECONDS, "reps": args.reps, "calls": {}, "split": {}}
    n = int(SR * SECONDS)
    g = torch.Generator().manual_seed(0)
    mel = Vocos.from_hparams(VOCOS_MEL_24K).load_weights(synth.vocos_weights(VOCOS_MEL_24K))
    enc = Vocos.from_hparams(VOCOS_ENCODEC_24K).load_weights(synth.vocos_weights(VOCOS_ENCODEC_24K))
    for B in (1, 8, 32):
        audio = (0.3 * torch.randn(B, n, generator=g)).cuda()
        feats = mel.feature_extractor(audio)
        efeats = torch.randn(B, n // 320, 128, generator=g).cuda()
        cond = torch.tensor([[3.0, 3.0, 3.0, 3.0]]).cuda()
        for tag, fn in (("mel_call", lambda: mel(audio)), ("mel_decode", lambda: mel.decode(feats)),
                        ("encodec_decode", lambda: enc.decode(efeats, bandwidth_id=cond))):
            for _ in range(3):
                fn()
            l0 = ops.LAUNCHES[0]
            fn()
            launches = ops.LAUNCHES[0] - l0
            ms = [_timed(fn) for _ in range(args.reps)]
            res["calls"][f"{tag}_B{B}"] = dict(_stats(ms, B * SECONDS), launches=launches)
            res["split"][f"{tag}_B{B}"] = _split(fn)

    # dwnorm against conv1d (depthwise) + layernorm(planes=True), at a block's shape of the mel model
    blk = mel.backbone._W["blocks"][0]
    w, b = blk["norm"]
    dwn = {}
    for B in (1, 8, 32):
        x = torch.randn(B, n // 256, 512, generator=g).cuda()
        fused = lambda: ops.vocos_dwnorm(x, blk["dw"], w, b, fp32=False, planes=True)
        comp = lambda: ops.layernorm(ops.conv1d(x, blk["dw"], pad_left=3), w, b, eps=1e-6, planes=True)
        for _ in range(3):
            fused(), comp()
        tf, tc = [], []
        for _ in range(args.reps):
            tf.append(_timed(fused))
            tc.append(_timed(comp))
        dwn[f"B{B}"] = {"fused": _stats(tf), "conv1d_plus_layernorm": _stats(tc)}
    res["dwnorm"] = dwn

    # head kernel against spectrum formation in torch ops + the existing dsp.istft route
    head = {}
    for n_fft, hop, m in ((1024, 256, mel), (1280, 320, enc)):
        win = torch.from_numpy(hanning(n_fft)).float().cuda()
        nb = n_fft // 2 + 1
        for B in (1, 8, 32):
            T = n // hop + 1
            h = torch.randn(B, T, -(-(n_fft + 2) // 64) * 64, generator=g).cuda()
            h[..., :nb] -= 0.5

            def comp():
                mag = torch.clamp(torch.exp(h[..., :nb]), max=100.0).transpose(1, 2)
                p = h[..., nb:2 * nb].transpose(1, 2)
                S = torch.complex(mag * torch.cos(p), mag * torch.sin(p))
                return torch.stack([dsp.istft(S[i], hop_length=hop, win_length=n_fft, window=win) for i in range(B)])
            fused = lambda: ops.vocos_istft_head(h, n_fft, hop, win)
            for _ in range(2):
                fused(), comp()
            tf, tc = [], []
            for _ in range(args.reps):
                tf.append(_timed(fused))
                tc.append(_timed(comp))
            diff = float((fused() - comp()).abs().max())
            head[f"{n_fft}_B{B}"] = {"fused": _stats(tf), "torch_spectrum_plus_dsp_istft": _stats(tc), "max_abs_diff": diff}
    res["head"] = head
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
