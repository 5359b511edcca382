"""Oracle for the BigVGAN vocoder (codec/models/bigvgan/{bigvgan,amp,activation,resample,conv}.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).  torch-CPU in the dtype of the weights dict (float64 in the tests).  Parameter names are
the reference's MLX parameter tree (MLX layouts); activations are channels-last inside, the reference's [B, C, T] at the interface.
Activation1d is restated op by op -- edge pads, grouped transposed conv (MLX scatter rule, no flip), crop, SnakeBeta, edge pads,
strided grouped conv -- and pinned against the reference's own code by tests/golden/make_bigvgan_golden.py.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import nn as N

BIGVGAN_22K = dict(num_mels=80, upsample_rates=[4, 4, 2, 2, 2, 2], upsample_kernel_sizes=[8, 8, 4, 4, 4, 4], upsample_initial_channel=1536,
                   resblock="1", resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
                   activation="snakebeta", snake_logscale=True, use_bias_at_final=True, use_tanh_at_final=True)
BIGVGAN_44K = dict(num_mels=128, upsample_rates=[8, 4, 2, 2, 2, 2], upsample_kernel_sizes=[16, 8, 4, 4, 4, 4], upsample_initial_channel=1536,
                   resblock="1", resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
                   activation="snakebeta", snake_logscale=True, use_bias_at_final=False, use_tanh_at_final=False)


def output_length(cfg, frames):
    """bigvgan.py:40-53: each WNConvTranspose1d(k, u, padding=(k - u) // 2) maps L rows to (L-1) u - 2 ((k-u)//2) + k rows."""
    L = frames
    for u, k in zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"]):
        L = (L - 1) * u - 2 * ((k - u) // 2) + k
    return L


def kaiser_sinc_filter1d(cutoff, half_width, kernel_size):
    """resample.py:17-46, float64 [kernel_size]."""
    even = kernel_size % 2 == 0
    half_size = kernel_size // 2
    A = 2.285 * (half_size - 1) * math.pi * (4 * half_width) + 7.95
    beta = 0.1102 * (A - 8.7) if A > 50.0 else (0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0) if A >= 21.0 else 0.0)
    window = torch.from_numpy(np.kaiser(kernel_size, beta=beta))
    time = torch.arange(-half_size, half_size, dtype=torch.float64) + 0.5 if even else torch.arange(kernel_size, dtype=torch.float64) - half_size
    if cutoff == 0:
        return torch.zeros(kernel_size, dtype=torch.float64)
    x = 2 * cutoff * time
    f = 2 * cutoff * window * torch.where(x == 0, torch.ones_like(x), torch.sin(math.pi * x) / math.pi / x)
    return f / f.sum()


def _edge(x, left, right):
    """mx.pad(mode="edge") on the time axis of [B, L, C]."""
    return F.pad(x.transpose(1, 2), (left, right), mode="replicate").transpose(1, 2)


def upsample(x, f, ratio=2):
    """UpSample1d (resample.py:101-136): x [B, L, C], f [K] -> [B, ratio L, C]."""
    C, K = x.shape[2], f.numel()
    pad = K // ratio - 1
    pad_left = pad * ratio + (K - ratio) // 2
    pad_right = pad * ratio + (K - ratio + 1) // 2
    w = f.to(x.dtype).reshape(1, K, 1).expand(C, K, 1)
    y = ratio * N.conv_transpose1d(_edge(x, pad, pad), w, stride=ratio, groups=C)
    return y[:, pad_left: y.shape[1] - pad_right]


def lowpass(x, f, stride=2):
    """LowPassFilter1d (resample.py:49-98) with padding=True, padding_mode="edge": x [B, n, C], f [K]."""
    C, K = x.shape[2], f.numel()
    even = K % 2 == 0
    w = f.to(x.dtype).reshape(1, K, 1).expand(C, K, 1)
    return N.conv1d(_edge(x, K // 2 - int(even), K // 2), w, stride=stride, groups=C)


def snakebeta(x, alpha, beta, logscale):
    """activation.py:42-51."""
    if logscale:
        alpha, beta = torch.exp(alpha), torch.exp(beta)
    return x + (1.0 / (beta + 1e-9)) * torch.sin(x * alpha) ** 2


def _filters(P, pre):
    default = kaiser_sinc_filter1d(0.25, 0.3, 12)
    return P.get(pre + ".upsample.filter", default).reshape(-1), P.get(pre + ".downsample.lowpass.filter", default).reshape(-1)


def activation1d(P, pre, x, logscale):
    """Activation1d(SnakeBeta) (resample.py:157-177) with the parameters under ``pre``."""
    fu, fd = _filters(P, pre)
    y = snakebeta(upsample(x, fu), P[pre + ".act.alpha"].reshape(-1), P[pre + ".act.beta"].reshape(-1), logscale)
    return lowpass(y, fd)


def _wn(P, pre, except_dim=0):
    """conv.py:7-12,56,103-107: g * v / ||v||, the norm over every axis but ``except_dim``."""
    v, g = P[pre + ".weight_v"], P[pre + ".weight_g"]
    axes = tuple(i for i in range(v.ndim) if i != except_dim)
    return g * v / torch.sqrt((v * v).sum(dim=axes, keepdim=True))


def wnconv(P, pre, x, padding=0, dilation=1):
    return N.conv1d(x, _wn(P, pre), 1, padding, dilation, 1, P.get(pre + ".bias"))


def amp_block(P, pre, x, cfg, k, dilations):
    """AMPBlock1 (amp.py:52-58) / AMPBlock2 (amp.py:92-96)."""
    ls = cfg["snake_logscale"]
    for m, d in enumerate(dilations):
        if cfg["resblock"] == "1":
            t = wnconv(P, f"{pre}.convs1.{m}", activation1d(P, f"{pre}.activations.{2 * m}", x, ls), (k - 1) * d // 2, d)
            x = x + wnconv(P, f"{pre}.convs2.{m}", activation1d(P, f"{pre}.activations.{2 * m + 1}", t, ls), (k - 1) // 2)
        else:
            x = x + wnconv(P, f"{pre}.convs.{m}", activation1d(P, f"{pre}.activations.{m}", x, ls), (k - 1) * d // 2, d)
    return x


def forward(P, mel, cfg):
    """bigvgan.py:97-122: mel [B, num_mels, T] -> [B, 1, T * prod(upsample_rates)]."""
    x = wnconv(P, "conv_pre", mel.transpose(1, 2), 3)
    nk = len(cfg["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        pre = f"ups.{i}.0"
        x = N.conv_transpose1d(x, _wn(P, pre, except_dim=2), u, (k - u) // 2, 1, 0, 1, P.get(pre + ".bias"))
        xs = None
        for j, (kr, dil) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            y = amp_block(P, f"resblocks.{i * nk + j}", x, cfg, kr, dil)
            xs = y if xs is None else xs + y
        x = xs / nk
    x = wnconv(P, "conv_post", activation1d(P, "activation_post", x, cfg["snake_logscale"]), 3)
    x = torch.tanh(x) if cfg["use_tanh_at_final"] else torch.clamp(x, -1.0, 1.0)
    return x.transpose(1, 2)
