"""Oracle for Qwen3-TTS streaming generation: the event sequence of ``Model.generate(stream=True)`` (qwen3_tts.py:1316-1521 base path,
:2264-2446 custom-voice / voice-design paths), restated from ``oracle.qwen3.generate_codes`` and the incremental decoder
``oracle.qwen3.tokenizer_decode(..., stream_boundaries=...)``.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Pinned against the reference's own streaming loop executed through the NumPy stand-in
(tests/golden/make_qwen3_stream_golden.py -> qwen3_stream_golden.npz, tests/test_qwen3_stream_pins.py)."""
from __future__ import annotations

import torch

from . import qwen3 as Q


def stream_chunk_size(streaming_interval: float) -> int:
    """qwen3_tts.py:1317: frames per streamed chunk (12.5 frames per second)."""
    return max(1, int(streaming_interval * 12.5))


def stream_spans(n_frames: int, chunk: int):
    """(start, end, is_final) of every event for ``n_frames`` recorded frames: a chunk each time ``chunk`` frames are undecoded, then the
    remainder as the final chunk -- only if there is one (an exact multiple ends without an ``is_final_chunk`` event)."""
    spans, start = [], 0
    while n_frames - start >= chunk:
        spans.append((start, start + chunk, False))
        start += chunk
    if n_frames > start:
        spans.append((start, n_frames, True))
    return spans


def stream_events(PT, codes, streaming_interval: float, tcfg=Q.TOKENIZER_DECODER, segment_idx: int = 0):
    """Events of one segment whose generated frames are ``codes`` [n, 16]: a list of dicts with the chunk's codes [k, 16], audio
    [1920 k] (the incremental decoder: reset at the start of the segment, one ``streaming_step`` per event), ``token_count``,
    ``samples``, ``is_streaming_chunk``, ``is_final_chunk`` and ``segment_idx``."""
    spans = stream_spans(codes.shape[0], stream_chunk_size(streaming_interval))
    if not spans:
        return []
    up = 1
    for r in list(tcfg["upsample_rates"]) + list(tcfg["upsampling_ratios"]):
        up *= r
    wav = Q.tokenizer_decode(PT, codes.T[None].contiguous(), tcfg, stream_boundaries=tuple(s for s, _, _ in spans[1:]))[0, 0]
    return [{"codes": codes[s:e], "audio": wav[s * up: e * up], "token_count": e - s, "samples": (e - s) * up, "is_streaming_chunk": True,
             "is_final_chunk": final, "segment_idx": segment_idx} for s, e, final in spans]


def generate_stream(P, PT, input_embeds, trailing_text_hidden, tts_pad_embed, u, max_tokens, streaming_interval: float = 2.0,
                    temperature=0.9, top_k=50, top_p=1.0, repetition_penalty=1.05, cfg=Q.TALKER, tcfg=Q.TOKENIZER_DECODER,
                    segment_idx: int = 0):
    """One segment of ``Model.generate(stream=True)``: the frame loop (``oracle.qwen3.generate_codes``, same injected uniforms ``u``
    [max_tokens, 16]) and its streamed events (``stream_events``)."""
    codes = Q.generate_codes(P, input_embeds, trailing_text_hidden, tts_pad_embed, u, max_tokens, temperature, top_k, top_p,
                             repetition_penalty, cfg)
    return stream_events(PT, codes, streaming_interval, tcfg, segment_idx)


def concat_audio(events):
    return torch.cat([e["audio"] for e in events]) if events else torch.zeros(0, dtype=torch.float64)
