"""SHA-256 digests of what `ops.lstm_bidir` (csrc/lstm.cu) writes on seeded inputs.

Kokoro's durations are rounded from this recurrence's output, so a last-bit change could move a frame boundary: a rewrite of the kernel
must reproduce these bytes.  Inputs are generated on the CPU from fixed seeds at the scales of
test_ops_gpu.py::test_lstm_bidir_matches_reference_recurrence (input projections of std ~1.3, W_h of std 0.08); a few time steps are
scaled up so that their gates saturate.  One case writes into a column slice of a wider buffer (out_ld > 2H); its digest covers the
whole buffer, so it also pins that nothing outside the slice is written.

Run on an H100 from the repository root:  python tests/golden/make_lstm_digest.py
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "lstm_digest.json")

H = 256
# (B, T, out columns: None = a fresh [B, T, 2H] tensor, else (buffer width, first column))
CASES = [(1, 130, None), (1, 390, None), (2, 57, None), (3, 1, None), (1, 2, None), (8, 130, None), (2, 57, (640, 64))]


def label(case) -> str:
    B, T, sl = case
    return f"B{B} T{T}" + (f" out[..., {sl[1]}:{sl[1] + 2 * H}] of {sl[0]}" if sl else "")


def inputs(case):
    """(xproj [B, T, 8H], wh [2, 4H, H]) as float32 CPU tensors."""
    import torch
    B, T, _ = case
    g = torch.Generator().manual_seed(1000 * B + T)
    xproj = torch.randn(B, T, 8 * H, generator=g) * 1.3
    hot = torch.randint(0, T, (max(1, T // 16),), generator=g)          # saturating steps
    xproj[:, hot] *= 12.0
    wh = torch.randn(2, 4 * H, H, generator=g) * 0.08
    return xproj, wh


def run(case, dev="cuda:0"):
    """The kernel's output on `case`: the [B, T, 2H] result, or the whole wider buffer it was written into."""
    import torch
    from mlx_audio_b200 import ops
    B, T, sl = case
    xproj, wh = inputs(case)
    xproj, wh = xproj.to(dev), wh.to(dev).contiguous()
    if sl is None:
        return ops.lstm_bidir(xproj, wh)
    buf = torch.full((B, T, sl[0]), -7.0, device=dev)
    ops.lstm_bidir(xproj, wh, out=buf[:, :, sl[1]:sl[1] + 2 * H])
    return buf


def result(case, y):
    """The [B, T, 2H] result inside what run() returned."""
    sl = case[2]
    return y if sl is None else y[:, :, sl[1]:sl[1] + 2 * H]


def oracle(case):
    """oracle.kokoro.lstm_bi in float64 on the same projections: x = xproj, Wx = [I | 0] / [0 | I], zero biases."""
    import torch
    from oracle import kokoro as OK
    xproj, wh = inputs(case)
    eye = torch.eye(4 * H, dtype=torch.float64)
    zero = torch.zeros(4 * H, 4 * H, dtype=torch.float64)
    P = {}
    for di, d in enumerate(("forward", "backward")):
        P[f"l.Wx_{d}"] = torch.cat([eye, zero] if di == 0 else [zero, eye], 1)
        P[f"l.Wh_{d}"] = wh[di].double()
        P[f"l.bias_ih_{d}"] = torch.zeros(4 * H, dtype=torch.float64)
        P[f"l.bias_hh_{d}"] = torch.zeros(4 * H, dtype=torch.float64)
    return OK.lstm_bi(P, "l", xproj.double())


def digest(y) -> str:
    import torch
    torch.cuda.synchronize()
    return hashlib.sha256(y.contiguous().cpu().numpy().tobytes()).hexdigest()


def digests(dev="cuda:0") -> list:
    return [{"case": label(c), "sha256": digest(run(c, dev))} for c in CASES]


if __name__ == "__main__":
    d = digests()
    with open(OUT, "w") as f:
        json.dump(d, f, indent=1)
        f.write("\n")
    print(f"{len(d)} cases -> {OUT}")
