"""EnCodec timings on the GPU with synthetic float32 weights at the released widths: 24 kHz at 10 s (B = 1 and 8: encoder, quantiser at
1.5 / 6 / 24 kbps, decoder, LSTM microseconds per step) and 48 kHz stereo at 10 s (chunked encode and decode, all chunks as one batch
against chunk by chunk, alternated in the same call).  CUDA events, warm-up, median of --reps (>= 10).  The batched and the chunk-by-chunk
routes are checked against each other at the timed size (codes identical, largest sample difference reported); agreement with the float64
oracle is tests/test_encodec_gpu.py's job (tools do not import oracle/).  Prints the card and its power limit beside the numbers.

    python tools/encodec_bench.py [--reps 10] [--out results/encodec_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mlx_audio_b200 import configs, ops, synth  # noqa: E402
from mlx_audio_b200.codec import Encodec  # noqa: E402
from mlx_audio_b200.codec.models.encodec import preprocess_audio  # noqa: E402


def timed(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:                                                  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encodec_bench: needs a CUDA device")
    res = {"card": card(), "reps": a.reps}
    print("card:", res["card"])
    g = torch.Generator().manual_seed(0)

    # ---- 24 kHz, 10 s
    cfg = configs.ENCODEC_24K
    P = synth.encodec_weights(cfg)
    m = Encodec(cfg).load_weights(P)
    n = 240_000
    for B in (1, 8):
        x = (0.1 * torch.randn(B, n, 1, generator=g)).to("cuda")
        emb = m.encode_latent(x)
        r = {"encoder_ms": timed(lambda: m.encode_latent(x), a.reps)}
        for bw in (1.5, 6.0, 24.0):
            nq = m.get_num_quantizers_for_bandwidth(bw)
            r[f"quantiser_{bw}kbps_ms"] = timed(lambda: m._quantize(emb, nq), a.reps)
        codes = m._quantize(emb, 32)
        r["decoder_ms"] = timed(lambda: m.decode_frames(codes), a.reps)
        H, T = 512, emb.shape[1]
        xp = (0.5 * torch.randn(B, T, 4 * H, generator=g)).to("cuda")
        wh = m._W["enc"]["lstm"][0]["wh"]
        err = torch.zeros(1, device="cuda", dtype=torch.int32)
        r["lstm_us_per_step"] = 1000 * timed(lambda: ops.encodec_lstm(xp, wh, err), a.reps) / T
        res[f"24k_B{B}"] = r
        print(f"24 kHz B={B}:", json.dumps(r))

    # ---- 48 kHz stereo, 10 s
    cfg = configs.ENCODEC_48K
    P = synth.encodec_weights(cfg, seed=16)
    m = Encodec(cfg).load_weights(P)
    x = 0.1 * torch.randn(480_000, 2, generator=g)
    inp, mask = preprocess_audio([x], 48000, m.chunk_length, m.chunk_stride)
    cl, st = m.chunk_length, m.chunk_stride
    offsets = list(range(0, inp.shape[1] - (cl - st), st))

    def by_chunk_encode():
        return [m.encode_frames(inp[:, o:o + cl].contiguous(), mask[:, o:o + cl].contiguous(), 4) for o in offsets]

    codes, scales = m.encode(inp, mask, bandwidth=6.0)
    single = by_chunk_encode()
    assert all(torch.equal(c, codes[k]) for k, (c, _) in enumerate(single))

    def by_chunk_decode():
        frames = torch.cat([m.decode_frames(codes[k]) for k in range(len(offsets))])
        return ops.encodec_ola(frames, 1, torch.cat([s.reshape(-1) for s in scales]), m.chunk_stride, mask.shape[1])

    y = m.decode(codes, scales, mask)
    r = {"chunks": len(offsets), "decode_batched_vs_by_chunk_max_abs": float((by_chunk_decode() - y).abs().max())}
    tb_e, tc_e, tb_d, tc_d = [], [], [], []
    for _ in range(a.reps):                                                  # alternated in the same call
        tb_e.append(timed(lambda: m.encode(inp, mask, bandwidth=6.0), 1, warm=1))
        tc_e.append(timed(by_chunk_encode, 1, warm=1))
        tb_d.append(timed(lambda: m.decode(codes, scales, mask), 1, warm=1))
        tc_d.append(timed(by_chunk_decode, 1, warm=1))
    r.update(encode_batched_ms=float(np.median(tb_e)), encode_by_chunk_ms=float(np.median(tc_e)), decode_batched_ms=float(np.median(tb_d)),
             decode_by_chunk_ms=float(np.median(tc_d)))
    res["48k_stereo_10s"] = r
    print("48 kHz stereo 10 s:", json.dumps(r))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
