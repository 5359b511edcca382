"""Oracle for Qwen3-TTS x-vector voice cloning: ``Model.generate(text, ref_audio=...)`` on a base model (qwen3_tts.py:1227-1298 with
``_prepare_generation_inputs`` :326-484): the reference audio's ECAPA-TDNN embedding (``oracle.qwen3.speaker_encoder`` on
``oracle.dsp.qwen3_mel_spectrogram``, :285-324) takes the speaker row of the codec prefix, cast to the talker's dtype (:429-432); the
frame loop, decode and streaming are the base path's (``oracle.qwen3`` / ``oracle.qwen3_stream``).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Pinned against the reference's own ``Model.generate`` executed through the NumPy
stand-in (tests/golden/make_qwen3_xvector_golden.py -> qwen3_xvector_golden.npz, tests/test_qwen3_xvector_pins.py)."""
from __future__ import annotations

import numpy as np
import torch

from . import dsp as D
from . import nn as N
from . import qwen3 as Q


def speaker_embedding(PS, audio, scfg=Q.SPEAKER_ENCODER) -> torch.Tensor:
    """Model.extract_speaker_embedding (qwen3_tts.py:285-324): samples [n] or [B, n] at 24 kHz -> [B, enc_dim] float64."""
    mel = torch.as_tensor(np.asarray(D.qwen3_mel_spectrogram(audio))).double()
    return Q.speaker_encoder(PS, mel, scfg)


def prepare_generation_inputs_from_embed(P, input_ids, tts_ids, cfg_ids, language_id=None, speaker_embed=None, embed_dtype=None):
    """Model._prepare_generation_inputs (qwen3_tts.py:326-484) after tokenisation, with the speaker row given as an EMBEDDING
    ``speaker_embed`` [enc_dim] / [1, enc_dim] (the x-vector; ``None``: no speaker row).  ``embed_dtype`` = the talker's dtype the
    embedding is cast to first (:429-432; ``None`` or float64 / float32: no rounding beyond float32's).  Same returns as
    ``oracle.qwen3.prepare_generation_inputs_from_ids``."""
    def text_projection(x):                                            # ResizeMLP (talker.py:339-364), silu
        h = torch.nn.functional.silu(N.linear(x, P["text_projection.linear_fc1.weight"], P["text_projection.linear_fc1.bias"]))
        return N.linear(h, P["text_projection.linear_fc2.weight"], P["text_projection.linear_fc2.bias"])
    te, ce = P["model.text_embedding.weight"], P["model.codec_embedding.weight"]
    ids = torch.as_tensor(input_ids, dtype=torch.int64).reshape(1, -1)
    text_embed = text_projection(te[ids])
    tts = text_projection(te[torch.tensor([list(tts_ids)])])
    tts_bos, tts_eos, tts_pad = tts[:, 0:1], tts[:, 1:2], tts[:, 2:3]
    if language_id is None:
        prefill = [cfg_ids["codec_nothink_id"], cfg_ids["codec_think_bos_id"], cfg_ids["codec_think_eos_id"]]
    else:
        prefill = [cfg_ids["codec_think_id"], cfg_ids["codec_think_bos_id"], language_id, cfg_ids["codec_think_eos_id"]]
    parts = [ce[torch.tensor([prefill])]]
    if speaker_embed is not None:
        e = torch.as_tensor(speaker_embed).double().reshape(1, 1, -1)
        if embed_dtype is not None:
            e = e.to(embed_dtype).double()
        parts.append(e.to(ce.dtype))
    parts.append(ce[torch.tensor([[cfg_ids["codec_pad_id"], cfg_ids["codec_bos_id"]]])])
    codec = torch.cat(parts, dim=1)
    combined = torch.cat([tts_pad.expand(1, codec.shape[1] - 2, -1), tts_bos], dim=1) + codec[:, :-1]
    first_text = text_embed[:, 3:4] + codec[:, -1:]
    input_embeds = torch.cat([text_embed[:, :3], combined, first_text], dim=1)
    trailing = torch.cat([text_embed[:, 4:-5], tts_eos], dim=1)
    return input_embeds, trailing, tts_pad


def segment_ids(encode, text: str, split_pattern: str = "\n"):
    """Token ids of every segment of the base path (split AND stripped, qwen3_tts.py:1268-1271), through the chat template (:336-338)."""
    segs = [s.strip() for s in text.split(split_pattern) if s.strip()] if split_pattern else [text]
    return [encode(f"<|im_start|>assistant\n{s}<|im_end|>\n<|im_start|>assistant\n") for s in segs]
