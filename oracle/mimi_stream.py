"""Oracle for Mimi's incremental API (codec/models/mimi/mimi.py:164-176): ``decode_step`` / ``encode_step`` streams restated as slices of
the one-shot ``oracle.codec.mimi_decode`` / ``mimi_encode``.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Pinned against the reference's own step functions executed through the NumPy stand-in
(tests/golden/make_mimi_stream_golden.py -> mimi_stream_golden.npz, tests/test_mimi_stream_pins.py)."""
from __future__ import annotations

import math

import torch

from . import codec as OC


def frame_samples(cfg=OC.MIMI_202407) -> int:
    """Samples per code frame: the SEANet hop times the down-sampling stride (1920 at 24 kHz / 12.5 Hz)."""
    return math.prod(cfg["ratios"]) * cfg["upsample_stride"]


def decode_stream(P, codes: torch.Tensor, chunks, cfg=OC.MIMI_202407):
    """Outputs of ``decode_step`` over ``codes`` [B, nq, T] fed in ``chunks`` (frame counts summing to T): each is the matching slice of
    one one-shot decode, [B, 1, hop * chunk]."""
    assert sum(chunks) == codes.shape[-1]
    pcm, hop = OC.mimi_decode(P, codes, cfg), frame_samples(cfg)
    out, a = [], 0
    for c in chunks:
        out.append(pcm[..., a * hop:(a + c) * hop])
        a += c
    return out


def encode_stream(P, pcm: torch.Tensor, chunks, cfg=OC.MIMI_202407):
    """Outputs of ``encode_step`` over ``pcm`` [B, 1, n] fed in ``chunks`` (sample counts summing to n): call i returns the frames that the
    samples up to its end complete -- frame f needs samples [0, hop (f + 1)) (every conv is causal; the encoder transformer and the stride-2
    down-sampler see position 2f + 1 last) -- i.e. those frames of one one-shot encode of the complete frames."""
    assert sum(chunks) == pcm.shape[-1]
    hop = frame_samples(cfg)
    n_frames = pcm.shape[-1] // hop
    codes = OC.mimi_encode(P, pcm[..., :n_frames * hop], cfg) if n_frames else None
    out, done, seen = [], 0, 0
    for c in chunks:
        seen += c
        f = seen // hop
        out.append(codes[..., done:f] if f > done else torch.zeros(pcm.shape[0], cfg["nq"], 0, dtype=torch.int64))
        done = f
    return out
