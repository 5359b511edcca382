"""BigVGAN vocoder on H100 (reference: codec/models/bigvgan/{bigvgan,amp,activation,resample,conv}.py).

``BigVGAN(config)(mel)``: mel [B, num_mels, T] -> audio [B, 1, T * prod(upsample_rates)], channels-first as the reference returns it.
Weight norm is folded once at load.  The dense, dilated and polyphase transposed convs run on ``ops.conv1d``; every residual add, the
sum of a stage's AMP blocks over ``num_kernels`` and the final tanh / clip are conv epilogues.  Each anti-aliased SnakeBeta
(``Activation1d``: 2x up-sampling, SnakeBeta, low-pass and 2x down-sampling) is one ``ops.aa_snakebeta`` launch, which writes the next
conv's bf16 operand planes directly where that conv runs on the tensor cores.

``activation="snake"`` is not supported: the reference's ``Snake`` indexes ``alpha[None, :, None]`` against a (B, T, C) tensor
(activation.py:18), which fails to broadcast unless T == C and then scales along time; every released checkpoint uses ``snakebeta``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Literal

import numpy as np
import torch

from ... import ops
from ...ops import ACT
from .descript_layers import wnconv


@dataclass
class BigVGANConfig:
    """bigvgan.py:14-26."""
    num_mels: int
    upsample_rates: list[int]
    upsample_kernel_sizes: list[int]
    upsample_initial_channel: int
    resblock: Literal["1", "2"]
    resblock_kernel_sizes: list[int]
    resblock_dilation_sizes: list[list[int]]
    activation: Literal["snakebeta", "snake"]
    snake_logscale: bool
    use_bias_at_final: bool = True  # compatability
    use_tanh_at_final: bool = True  # compatability


def kaiser_sinc_filter1d(cutoff: float, half_width: float, kernel_size: int) -> torch.Tensor:
    """resample.py:17-46 in float64: the windowed-sinc low-pass, [kernel_size]."""
    even = kernel_size % 2 == 0
    half_size = kernel_size // 2
    A = 2.285 * (half_size - 1) * math.pi * (4 * half_width) + 7.95
    if A > 50.0:
        beta = 0.1102 * (A - 8.7)
    elif A >= 21.0:
        beta = 0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21.0)
    else:
        beta = 0.0
    window = torch.from_numpy(np.kaiser(kernel_size, beta=beta))
    time = (torch.arange(-half_size, half_size, dtype=torch.float64) + 0.5) if even else torch.arange(kernel_size, dtype=torch.float64) - half_size
    if cutoff == 0:
        return torch.zeros(kernel_size, dtype=torch.float64)
    t = 2 * cutoff * time
    sinc = torch.where(t == 0, torch.ones_like(t), torch.sin(math.pi * t) / math.pi / t)
    f = 2 * cutoff * window * sinc
    return f / f.sum()


def _stage_channels(cfg: BigVGANConfig, i: int) -> int:
    return cfg.upsample_initial_channel // (2 ** i)


def param_shapes(cfg: BigVGANConfig) -> dict:
    """The reference's MLX parameter tree (bigvgan.py:29-95, amp.py, conv.py, resample.py): name -> shape."""
    S = {}

    def wn(pre, cout, k, cin, bias=True, except_dim=0):
        S[pre + ".weight_g"] = (cout, 1, 1) if except_dim == 0 else (1, 1, cin)
        S[pre + ".weight_v"] = (cout, k, cin)
        if bias:
            S[pre + ".bias"] = (cout,)

    def act(pre, c):
        S[pre + ".act.alpha"], S[pre + ".act.beta"] = (c,), (c,)
        S[pre + ".upsample.filter"] = S[pre + ".downsample.lowpass.filter"] = (1, 12, 1)

    wn("conv_pre", cfg.upsample_initial_channel, 7, cfg.num_mels)
    nk = len(cfg.resblock_kernel_sizes)
    for i, (u, k) in enumerate(zip(cfg.upsample_rates, cfg.upsample_kernel_sizes)):
        c = _stage_channels(cfg, i + 1)
        wn(f"ups.{i}.0", c, k, _stage_channels(cfg, i), except_dim=2)
        for j, (kr, dil) in enumerate(zip(cfg.resblock_kernel_sizes, cfg.resblock_dilation_sizes)):
            bp = f"resblocks.{i * nk + j}"
            for m in range(len(dil)):
                if cfg.resblock == "1":
                    wn(f"{bp}.convs1.{m}", c, kr, c)
                    wn(f"{bp}.convs2.{m}", c, kr, c)
                    act(f"{bp}.activations.{2 * m}", c)
                    act(f"{bp}.activations.{2 * m + 1}", c)
                else:
                    wn(f"{bp}.convs.{m}", c, kr, c)
                    act(f"{bp}.activations.{m}", c)
    c = _stage_channels(cfg, len(cfg.upsample_rates))
    act("activation_post", c)
    wn("conv_post", 1, 7, c, bias=cfg.use_bias_at_final)
    return S


def _perm(v, axes):
    return v.permute(*axes) if isinstance(v, torch.Tensor) else np.transpose(v, axes)


class BigVGAN:
    def __init__(self, config: BigVGANConfig, device="cuda"):
        if config.activation != "snakebeta":
            raise NotImplementedError("BigVGAN: activation='snake' is not supported -- the reference's Snake broadcasts alpha along time "
                                      "(activation.py:18) and fails unless T == C; released checkpoints use 'snakebeta'")
        if config.resblock not in ("1", "2"):
            raise ValueError(f"BigVGAN: resblock must be '1' or '2', got {config.resblock!r}")
        self.config = config
        self.num_kernels = len(config.resblock_kernel_sizes)
        self.num_upsamples = len(config.upsample_rates)
        self.use_tanh_at_final = config.use_tanh_at_final
        self.device = torch.device(device)
        self._W = None

    def _ensure_weights(self):
        """The reference's constructor leaves a randomly initialised, usable model (its own tests run one); here the random weights are
        made on first use, so that a model whose weights are loaded never pays for them."""
        if self._W is None:
            from ... import synth
            self.load_weights(synth.bigvgan_weights(self.config))

    def sanitize(self, weights):
        """bigvgan.py:124-149 on a torch-layout checkpoint (torch tensors or NumPy arrays): drops ``num_batches_tracked``, moves conv and
        filter weights to (out, K, in) and the transposed convs' (in, out, K) to (out, K, in) where the shape differs from the model's."""
        shapes = param_shapes(self.config)
        new_weights = {}
        for key, value in dict(weights).items():
            if "num_batches_tracked" in key:
                continue
            if "conv" in key or "lowpass.filter" in key or "upsample.filter" in key:
                if value.ndim == 3 and tuple(value.shape) != shapes[key]:
                    value = _perm(value, (0, 2, 1))
                elif value.ndim == 4 and tuple(value.shape) != shapes[key]:
                    value = _perm(value, (0, 2, 3, 1))
            if "ups." in key and value.ndim == 3 and tuple(value.shape) != shapes[key]:
                value = _perm(value, (1, 2, 0))
            new_weights[key] = value
        return new_weights

    def load_weights(self, weights):
        """The sanitized, MLX-layout parameters (``sanitize`` output or ``synth.bigvgan_weights``).  Filters missing from the dict are the
        constructor's Kaiser-sinc filters, computed in float64 and rounded once to fp32."""
        P = {k: torch.as_tensor(v) for k, v in dict(weights).items()}
        cfg, dev = self.config, self.device
        f = lambda t: t.float().to(dev).contiguous()
        kaiser = kaiser_sinc_filter1d(0.25, 0.3, 12)                       # UpSample1d / DownSample1d at ratio 2 (resample.py:117-119, :146-151)

        def act(pre):
            alpha, beta = P[pre + ".act.alpha"].double().reshape(-1), P[pre + ".act.beta"].double().reshape(-1)
            if cfg.snake_logscale:
                alpha, beta = torch.exp(alpha), torch.exp(beta)
            fu, fd = P.get(pre + ".upsample.filter", kaiser), P.get(pre + ".downsample.lowpass.filter", kaiser)
            return f(alpha), f(1.0 / (beta + 1e-9)), f(fu.reshape(-1)), f(fd.reshape(-1))

        W = {"pre": wnconv(P, "conv_pre", dev), "stages": []}
        for i, (u, k) in enumerate(zip(cfg.upsample_rates, cfg.upsample_kernel_sizes)):
            blocks = []
            for j, (kr, dil) in enumerate(zip(cfg.resblock_kernel_sizes, cfg.resblock_dilation_sizes)):
                bp = f"resblocks.{i * self.num_kernels + j}"
                if cfg.resblock == "1":
                    units = [{"d": d, "c1": wnconv(P, f"{bp}.convs1.{m}", dev), "c2": wnconv(P, f"{bp}.convs2.{m}", dev),
                              "a1": act(f"{bp}.activations.{2 * m}"), "a2": act(f"{bp}.activations.{2 * m + 1}")} for m, d in enumerate(dil)]
                else:
                    units = [{"d": d, "c1": wnconv(P, f"{bp}.convs.{m}", dev), "a1": act(f"{bp}.activations.{m}")} for m, d in enumerate(dil)]
                blocks.append({"k": kr, "units": units})
            W["stages"].append({"u": u, "k": k, "up": wnconv(P, f"ups.{i}.0", dev, except_dim=2), "blocks": blocks})
        W["post_act"], W["post"] = act("activation_post"), wnconv(P, "conv_post", dev)
        self._W = W
        return self

    @staticmethod
    def _act(x, act, cw, dilation):
        """Activation1d in front of conv ``cw``: bf16 planes when that conv takes the tensor-core path at this length, fp32 otherwise."""
        if cw.w_tc is not None and not cw.f16 and ops._tc_eligible(cw, x.shape[1], 1, False, 0, dilation):
            return ops.aa_snakebeta(x, *act, planes_for=cw)
        return ops.aa_snakebeta(x, *act)

    def _amp(self, x, blk, out, accumulate):
        """AMPBlock1 / AMPBlock2 (amp.py:52-58, :92-96); the last residual add writes (x + conv(...)) / num_kernels into ``out``, or adds
        it there (``accumulate``): the stage's sum over its AMP blocks (bigvgan.py:108-112)."""
        k, units = blk["k"], blk["units"]
        for m, u in enumerate(units):
            last = dict(out=out, accumulate=accumulate, out_scale=1.0 / self.num_kernels) if m == len(units) - 1 else {}
            d = u["d"]
            t = ops.conv1d(self._act(x, u["a1"], u["c1"], d), u["c1"], dilation=d, pad_left=(k - 1) * d // 2,
                           **({} if "c2" in u else dict(res=x, **last)))
            if "c2" in u:
                t = ops.conv1d(self._act(t, u["a2"], u["c2"], 1), u["c2"], pad_left=(k - 1) // 2, res=x, **last)
            x = t
        return x

    @torch.no_grad()
    def __call__(self, x: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        """bigvgan.py:97-122: mel [B, num_mels, T] -> audio [B, 1, T * prod(upsample_rates)] in [-1, 1]."""
        self._ensure_weights()
        W = self._W
        if x.dim() != 3 or x.shape[1] != self.config.num_mels:
            raise ValueError(f"BigVGAN: expected mel [B, {self.config.num_mels}, T], got {tuple(x.shape)}")
        x = x.to(device=self.device, dtype=torch.float32).transpose(1, 2).contiguous()
        x = ops.conv1d(x, W["pre"], pad_left=3)
        for st in W["stages"]:
            u, k, L = st["u"], st["k"], x.shape[1]
            p = (k - u) // 2
            x = ops.conv1d(x, st["up"], stride=u, pad_left=p, lout=(L - 1) * u - 2 * p + k, transpose=True)
            acc = torch.empty_like(x)
            for j, blk in enumerate(st["blocks"]):
                self._amp(x, blk, acc, j > 0)
            x = acc
        x = ops.aa_snakebeta(x, *W["post_act"])
        y = ops.conv1d(x, W["post"], pad_left=3, post_act=ACT["tanh"] if self.use_tanh_at_final else ACT["clip1"])
        return y.transpose(1, 2)
