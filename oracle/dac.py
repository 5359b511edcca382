"""Oracle for the Descript Audio Codec (codec/models/descript/{dac,base}.py, nn/{layers,quantize}.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).  torch-CPU in the dtype of the weights dict (float64 in the tests).  Parameter names are
the reference's MLX parameter tree; activations are channels-last inside, the reference's [B, D, T] at the interface.

Quirks kept (and pinned against the reference by tests/golden/make_dac_golden.py):
  * WNConvTranspose1d passes ``groups`` in conv_transpose1d's ``output_padding`` slot (nn/layers.py:108-110): one extra sample per stage;
  * CodecMixin collects nn.Conv1d / nn.ConvTranspose1d instances and DAC has none (base.py:62-121): delay = 0, get_output_length(n) = n,
    compress cuts non-overlapping windows and decompress concatenates untrimmed decodes.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import nn as N

DAC_44K = {"encoder_dim": 64, "encoder_rates": [2, 4, 8, 8], "decoder_dim": 1536, "decoder_rates": [8, 8, 4, 2], "n_codebooks": 9,
           "codebook_size": 1024, "codebook_dim": 8, "sample_rate": 44100}
DAC_24K = {"encoder_dim": 64, "encoder_rates": [2, 4, 5, 8], "decoder_dim": 1536, "decoder_rates": [8, 5, 4, 2], "n_codebooks": 32,
           "codebook_size": 1024, "codebook_dim": 8, "sample_rate": 24000}
DAC_16K = {"encoder_dim": 64, "encoder_rates": [2, 4, 5, 8], "decoder_dim": 1536, "decoder_rates": [8, 5, 4, 2], "n_codebooks": 12,
           "codebook_size": 1024, "codebook_dim": 8, "sample_rate": 16000}


def hop(cfg):
    return math.prod(cfg["encoder_rates"])


def latent_dim(cfg):
    return cfg.get("latent_dim") or cfg["encoder_dim"] * 2 ** len(cfg["encoder_rates"])


def codebook_dims(cfg):
    cd = cfg["codebook_dim"]
    return [cd] * cfg["n_codebooks"] if isinstance(cd, int) else list(cd)


def _wn(P, pre, except_dim=0):
    """nn/layers.py:7-12,56: g * v / ||v||, the norm over every axis but ``except_dim``."""
    v, g = P[pre + ".weight_v"], P[pre + ".weight_g"]
    axes = tuple(i for i in range(v.ndim) if i != except_dim)
    return g * v / torch.sqrt((v * v).sum(dim=axes, keepdim=True))


def wnconv(P, pre, x, stride=1, padding=0, dilation=1):
    return N.conv1d(x, _wn(P, pre), stride, padding, dilation, 1, P.get(pre + ".bias"))


def wnconvtr(P, pre, x, stride, padding):
    """nn/layers.py:63-113: weight (out, K, in) normalised per INPUT channel; output_padding = 1 through the positional slot."""
    return N.conv_transpose1d(x, _wn(P, pre, except_dim=2), stride, padding, 1, 1, 1, P.get(pre + ".bias"))


def snake(x, alpha):
    """nn/layers.py:116-119 with alpha [1, 1, C] on channels-last x."""
    return x + (1.0 / (alpha + 1e-9)) * torch.sin(alpha * x) ** 2


def residual_unit(P, pre, x, dilation):
    y = snake(x, P[pre + ".block.layers.0.alpha"])
    y = wnconv(P, pre + ".block.layers.1", y, padding=3 * dilation, dilation=dilation)
    y = snake(y, P[pre + ".block.layers.2.alpha"])
    return x + wnconv(P, pre + ".block.layers.3", y)


def encoder(P, x, cfg):
    """dac.py:57-80 on channels-last x [B, n, 1] -> [B, T, latent]."""
    pre = "encoder.block.layers"
    x = wnconv(P, f"{pre}.0", x, padding=3)
    for i, stride in enumerate(cfg["encoder_rates"]):
        bp = f"{pre}.{i + 1}.block.layers"
        for bi, d in enumerate((1, 3, 9)):
            x = residual_unit(P, f"{bp}.{bi}", x, d)
        x = snake(x, P[f"{bp}.3.alpha"])
        x = wnconv(P, f"{bp}.4", x, stride=stride, padding=math.ceil(stride / 2))
    n = len(cfg["encoder_rates"])
    return wnconv(P, f"{pre}.{n + 2}", snake(x, P[f"{pre}.{n + 1}.alpha"]), padding=1)


def decoder(P, z, cfg):
    """dac.py:104-129 on channels-last z [B, T, latent] -> [B, T_out, 1]."""
    pre = "decoder.model.layers"
    x = wnconv(P, f"{pre}.0", z, padding=3)
    for i, stride in enumerate(cfg["decoder_rates"]):
        bp = f"{pre}.{i + 1}.block.layers"
        x = wnconvtr(P, f"{bp}.1", snake(x, P[f"{bp}.0.alpha"]), stride, math.ceil(stride / 2))
        for bi, d in enumerate((1, 3, 9)):
            x = residual_unit(P, f"{bp}.{2 + bi}", x, d)
    n = len(cfg["decoder_rates"])
    return torch.tanh(wnconv(P, f"{pre}.{n + 2}", snake(x, P[f"{pre}.{n + 1}.alpha"]), padding=3))


def _normalize(x):
    return x / torch.clamp(torch.sqrt((x.abs() ** 2).sum(1, keepdim=True)), min=1e-12)


def decode_latents(P, q, z_e, with_margin=False):
    """VectorQuantize.decode_latents (quantize.py:45-63) on channels-last z_e [B, T, cd] -> (codebook rows [B, T, cd], indices [B, T]
    [, arg-min margin [B, T]: second-lowest minus lowest distance])."""
    cb = P[f"quantizer.quantizers.{q}.codebook.weight"]
    e, c = _normalize(z_e.reshape(-1, z_e.shape[-1])), _normalize(cb)
    dist = (e ** 2).sum(1, keepdim=True) - 2 * e @ c.T + (c ** 2).sum(1, keepdim=True).T
    idx = (-dist).argmax(1).reshape(z_e.shape[:2])
    if not with_margin:
        return cb[idx], idx
    two = torch.topk(dist, 2, dim=1, largest=False).values
    return cb[idx], idx, (two[:, 1] - two[:, 0]).reshape(z_e.shape[:2])


def quantize(P, z, cfg, n_quantizers=None, with_margin=False):
    """ResidualVectorQuantize.__call__ (quantize.py:87-120) on z [B, D, T] -> (z_q [B, D, T], codes [B, nq, T], latents [B, sum cd, T],
    commitment_loss, codebook_loss [, margins [B, nq, T]])."""
    n = cfg["n_codebooks"] if n_quantizers is None else min(n_quantizers, cfg["n_codebooks"])
    residual, zq, codes, latents, margins, loss = z.transpose(1, 2), 0.0, [], [], [], 0.0
    for i in range(n):
        pre = f"quantizer.quantizers.{i}"
        z_e = wnconv(P, pre + ".in_proj", residual)
        e, idx, m = decode_latents(P, i, z_e, with_margin=True)
        loss = loss + ((z_e - e) ** 2).mean(dim=(1, 2)).mean()
        zqi = wnconv(P, pre + ".out_proj", z_e + (e - z_e))                                  # straight-through form, kept literally
        zq, residual = zq + zqi, residual - zqi
        codes.append(idx); latents.append(z_e.transpose(1, 2)); margins.append(m)
    out = (zq.transpose(1, 2), torch.stack(codes, 1), torch.cat(latents, 1), loss, loss)
    return out + (torch.stack(margins, 1),) if with_margin else out


def from_codes(P, codes, cfg):
    """quantize.py:122-131: the first codes.shape[1] code books -> (z_q [B, D, T], z_p [B, sum cd, T], codes)."""
    zq, zp = 0.0, []
    for i in range(codes.shape[1]):
        pre = f"quantizer.quantizers.{i}"
        e = P[pre + ".codebook.weight"][codes[:, i]]                                          # [B, T, cd]
        zp.append(e.transpose(1, 2))
        zq = zq + wnconv(P, pre + ".out_proj", e)
    return zq.transpose(1, 2), torch.cat(zp, 1), codes


def from_latents(P, latents, cfg):
    """quantize.py:133-151: as many code books as the latent channels cover -> (z_q, z_p, codes)."""
    dims = np.cumsum([0] + codebook_dims(cfg))
    n = int(np.where(dims <= latents.shape[1])[0].max())
    zq, zp, codes = 0.0, [], []
    for i in range(n):
        e, idx = decode_latents(P, i, latents[:, dims[i]:dims[i + 1]].transpose(1, 2))
        zp.append(e.transpose(1, 2)); codes.append(idx)
        zq = zq + wnconv(P, f"quantizer.quantizers.{i}.out_proj", e)
    return zq.transpose(1, 2), torch.cat(zp, 1), torch.stack(codes, 1)


def preprocess(audio, cfg):
    """dac.py:182-191: right-pad [B, 1, n] to a multiple of the hop."""
    return torch.nn.functional.pad(audio, (0, -audio.shape[-1] % hop(cfg)))


def encode(P, audio, cfg, n_quantizers=None):
    """dac.py:193-202: audio [B, 1, n] -> (z, codes, latents, commitment_loss, codebook_loss)."""
    return quantize(P, encoder(P, audio.transpose(1, 2), cfg).transpose(1, 2), cfg, n_quantizers)


def decode(P, z, cfg):
    """dac.py:204-205: z [B, D, T] -> [B, T_out, 1]."""
    return decoder(P, z.transpose(1, 2), cfg)


def forward(P, audio, cfg, n_quantizers=None):
    """dac.py:219-249 (use_rvq=True).  ``audio`` is sliced on the LAST axis of a [B, T_out, 1] tensor, i.e. not trimmed."""
    length = audio.shape[-1]
    z, codes, latents, cl, bl = encode(P, preprocess(audio, cfg), cfg, n_quantizers)
    return {"audio": decode(P, z, cfg)[..., :length], "z": z, "codes": codes, "latents": latents, "vq/commitment_loss": cl, "vq/codebook_loss": bl}


def output_length(cfg, frames):
    """Samples the decoder makes of ``frames`` frames (output_padding = 1 at every stage)."""
    L = frames
    for s in cfg["decoder_rates"]:
        L = (L - 1) * s - 2 * math.ceil(s / 2) + 2 * s + 1
    return L


def window_samples(cfg, win_duration):
    return int(math.ceil(int(win_duration * cfg["sample_rate"]) / hop(cfg)) * hop(cfg))


def compress(P, audio, cfg, win_duration=1.0, normalize_db=-16, n_quantizers=None):
    """CodecMixin.compress (base.py:123-196) on a 1-D sample tensor, window by window as the reference does -> dict with the DACFile fields."""
    nt = audio.shape[-1]
    duration = nt / cfg["sample_rate"]
    input_db = 20 * torch.log10(torch.sqrt((audio ** 2).mean(-1) + 1e-12) / 1.0 + 1e-12)
    if normalize_db is not None:
        audio = audio * 10 ** ((normalize_db - input_db) / 20)
    x = audio[None, None, :]
    win_duration = duration if win_duration is None else win_duration
    if duration <= win_duration:
        padding, n_samples = True, nt
    else:
        padding, n_samples = False, window_samples(cfg, win_duration)       # delay = 0: nothing is padded in front
    codes = []
    for i in range(0, nt, n_samples):                                      # hop = get_output_length(n_samples) = n_samples
        w = x[..., i:i + n_samples]
        w = torch.nn.functional.pad(w, (0, max(0, n_samples - w.shape[-1])))
        codes.append(encode(P, preprocess(w, cfg), cfg, n_quantizers)[1])
    return {"codes": torch.cat(codes, -1), "chunk_length": codes[-1].shape[-1], "original_length": duration, "input_db": float(input_db),
            "channels": 1, "sample_rate": cfg["sample_rate"], "padding": padding}


def decompress(P, f, cfg):
    """CodecMixin.decompress (base.py:198-231) on compress's dict -> [1, n]."""
    recons = []
    for i in range(0, f["codes"].shape[-1], f["chunk_length"]):
        recons.append(decode(P, from_codes(P, f["codes"][..., i:i + f["chunk_length"]], cfg)[0], cfg))
    return torch.cat(recons, 1).squeeze(-1) * 10 ** ((f["input_db"] - (-16)) / 20)
