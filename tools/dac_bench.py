"""Descript Audio Codec: what each stage costs on the GPU, and whether the one-launch quantiser and the batched windows pay.

Released-size synthetic weights (``synth.dac_weights``), the 44.1 kHz (9 code books) and 24 kHz (32 code books) shapes, B = 1 and B = 8,
10 s of audio.  Prints one JSON object with the card's name and power limit; every entry is the median and max of ``--reps`` timed
calls (CUDA events, after warm-up) and the audio-seconds it processes per second:
  - ``encoder``, ``decoder``: the conv stacks alone;
  - ``quantizer``: the fused kernel and the level-by-level route on the encoder's latent, alternated call by call;
  - ``from_codes``: the kernel against the torch gather + 1x1 projection loop the reference's code amounts to;
  - ``compress`` / ``decompress`` of 60 s in 1 s windows: all windows as one batch against one window at a time;
  - ``conv_paths``: the kernel every distinct conv shape of one encode + decode took (CUDA-core path or tensor-core tiling).
There is no CPU fall-back: without a GPU the script fails.

    python tools/dac_bench.py [--reps 10] [--json OUT]
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


DAC_44K = dict(encoder_dim=64, encoder_rates=[2, 4, 8, 8], decoder_dim=1536, decoder_rates=[8, 8, 4, 2], n_codebooks=9, codebook_size=1024,
               codebook_dim=8, sample_rate=44100)
DAC_24K = dict(encoder_dim=64, encoder_rates=[2, 4, 5, 8], decoder_dim=1536, decoder_rates=[8, 5, 4, 2], n_codebooks=32, codebook_size=1024,
               codebook_dim=8, sample_rate=24000)


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


def _stats(ms, audio_s):
    med = statistics.median(ms)
    return {"median_ms": round(med, 3), "max_ms": round(max(ms), 3), "n": len(ms), "audio_s_per_s": round(audio_s / (med * 1e-3), 1)}


def _bench(fn, reps, audio_s, warm=2):
    for _ in range(warm):
        fn()
    return _stats([_timed(fn) for _ in range(reps)], audio_s)


def _alternate(fns, reps, audio_s, warm=2):
    """Time several routes call by call in turn, so that drift of the shared machine lands on all of them alike."""
    for _ in range(warm):
        for f in fns.values():
            f()
    ms = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            ms[k].append(_timed(f))
    return {k: _stats(v, audio_s) for k, v in ms.items()}


def conv_paths(model, x):
    """One encode + decode with ops.conv1d wrapped: per distinct layer shape, the kernel it ran on and its time."""
    import torch
    from mlx_audio_b200 import ops
    seen, real = {}, ops.conv1d

    def spy(xx, cw, **kw):
        torch.cuda.synchronize()
        box = []
        ms = _timed(lambda: box.append(real(xx, cw, **kw)))
        after = (ops.conv1d_cl_last_path(), ops.conv1d_tc_last_config())
        key = f"[{xx.shape[0]}x{xx.shape[1]}x{cw.cin}->{cw.cout} k{cw.K} s{kw.get('stride', 1)} d{kw.get('dilation', 1)}{' T' if kw.get('transpose') else ''}]"
        tc = ops._tc_eligible(cw, xx.shape[1], kw.get("stride", 1), kw.get("transpose", False), 0, kw.get("dilation", 1))
        path = {"tensor_core": after[1]} if tc else {"cuda_core": after[0]}
        if key not in seen:
            seen[key] = dict(path, ms=round(ms, 3), calls=1)
        else:
            seen[key]["calls"] += 1
        return box[0]
    ops.conv1d = spy
    try:
        z = model.encode(x)[0]
        model.decode(z)
    finally:
        ops.conv1d = real
    return seen


def bench_shape(cfg, name, reps, seconds=10.0, long_seconds=60.0):
    import torch
    from mlx_audio_b200 import synth
    from mlx_audio_b200.codec import DAC
    from mlx_audio_b200.codec.models import dac as M
    dev = "cuda:0"
    model = DAC(**cfg, device=dev).load_weights(synth.dac_weights(cfg, encoder=True))
    sr, q = cfg["sample_rate"], model.quantizer
    out = {}
    g = torch.Generator().manual_seed(0)

    def levels_route(z):
        M.FUSED_RVQ[0] = False
        try:
            return q.quantize_cl(z)
        finally:
            M.FUSED_RVQ[0] = True

    def torch_from_codes(codes):
        zq = None
        for i in range(codes.shape[1]):
            lv = q._levels[i]
            zi = lv["cb"][codes[:, i]] @ lv["w_out"] + lv["b_out"]
            zq = zi if zq is None else zq + zi
        return zq

    for B in (1, 8):
        x = model.preprocess((0.3 * torch.randn(B, 1, int(seconds * sr), generator=g)).to(dev), sr)
        audio_s = B * seconds
        z = model.encode_latent(x)
        zq, codes, _, _ = q.quantize_cl(z)
        r = {"frames": int(z.shape[1]), "routes_same_codes": bool(torch.equal(codes, levels_route(z)[1])),
             "from_codes_max_diff": float((q.from_codes_cl(codes)[0] - torch_from_codes(codes)).abs().max()),
             "encoder": _bench(lambda: model.encode_latent(x), reps, audio_s),
             "quantizer": _alternate({"fused": lambda: q.quantize_cl(z), "level_by_level": lambda: levels_route(z)}, reps, audio_s),
             "from_codes": _alternate({"kernel": lambda: q.from_codes_cl(codes), "torch_loop": lambda: torch_from_codes(codes)}, reps, audio_s),
             "decoder": _bench(lambda: model.decode_cl(zq), reps, audio_s)}
        out[f"B{B}"] = r
        if B == 1:
            out["conv_paths"] = conv_paths(model, x)
        del x, z, zq
    sig = (0.05 * torch.randn(int(long_seconds * sr), generator=g)).to(dev)
    f = model.compress(sig)

    def compress_serial():
        win = f.chunk_length * model.hop_length
        xs = sig * float(10.0 ** ((-16 - f.input_db) / 20))
        xs = torch.nn.functional.pad(xs, (0, -xs.numel() % win))
        return torch.cat([model.encode(xs[i:i + win].reshape(1, 1, -1))[1] for i in range(0, xs.numel(), win)], dim=-1)

    def decompress_serial():
        cl = f.chunk_length
        return torch.cat([model.decode_cl(q.from_codes_cl(f.codes[:, :, i:i + cl])[0]) for i in range(0, f.codes.shape[-1], cl)], dim=1)

    out["compress_60s"] = dict(_alternate({"batched": lambda: model.compress(sig), "one_window_at_a_time": compress_serial}, reps, long_seconds),
                               windows=int(f.codes.shape[-1] // f.chunk_length), codes_equal=bool(torch.equal(compress_serial(), f.codes)))
    out["decompress_60s"] = _alternate({"batched": lambda: model.decompress(f), "one_window_at_a_time": decompress_serial}, reps, long_seconds)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/dac_bench.py needs a GPU: it measures the CUDA path and has no fall-back")
    name, power = _card()
    res = {"card": name, "power_limit": power, "reps": max(10, args.reps), "seconds": 10.0}
    for tag, cfg in (("dac_44khz", DAC_44K), ("dac_24khz", DAC_24K)):
        res[tag] = bench_shape(cfg, tag, max(10, args.reps))
    text = json.dumps(res, indent=1)
    print(text)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
