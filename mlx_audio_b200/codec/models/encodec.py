"""EnCodec on H100 (reference: codec/models/encodec/encodec.py).

``Encodec(config)`` with the reference's surface: ``encode(input_values, padding_mask=None, bandwidth=None)`` -> (codes [chunks, B, nq, T],
scales), ``decode(audio_codes, audio_scales, padding_mask=None)`` -> audio [B, n, C], ``from_pretrained(local_dir)`` -> (model,
processor), ``preprocess_audio``, ``channels`` / ``sampling_rate`` / ``chunk_length`` / ``chunk_stride``.  Tensors are CUDA and
channels-last, as in the reference.

Per EncodecConv1d the input side (reflect / zero padding, the previous GroupNorm and ELU) is one ``ops.encodec_pad`` launch and the conv
runs on ``ops.conv1d`` with no padding (unpadded k = 1 convs take ELU in their prologue and the residual add in their epilogue); with
``time_group_norm`` the statistics are ``ops.encodec_gn_coeffs`` and the normalised tensor is written by the next ``encodec_pad``.  Each
LSTM layer is a tensor-core input projection (``ops.linear``; fp32 checkpoints run in split-weight mode) plus one ``ops.encodec_lstm``
launch, the last one adding EncodecLSTM's skip.  The quantiser is ``rvq_encode`` mode 0 / ``rvq_decode``.  A chunked encode sends all
chunks of all rows through the encoder and quantiser as ONE batch, and decode runs them as one batch into ``ops.encodec_ola``.

Kept from the reference: the ``"Expected one frame"`` check of a non-chunked decode looks at axis 1 of the codes (the batch), so B > 1
decodes only through a chunked model, exactly as there; the shortcut conv always exists (``use_conv_shortcut`` is not a config field).
Divergences: the LSTM runs every batch row independently (the reference's Metal kernel indexes rows > 0 wrongly); reflect padding of at
least the input's length raises ``ValueError`` (the reference builds a short pad); ``num_residual_layers > 1`` raises
``NotImplementedError`` (the reference pads dilated convs by the undilated kernel size and then fails on mismatched lengths);
``from_pretrained`` takes a local directory only.
"""
from __future__ import annotations

import functools
import json
import math
from dataclasses import asdict, dataclass, fields
from pathlib import Path
from typing import List, Optional, Union

import numpy as np
import torch

from ... import ops
from ...ops import ACT, Pre


@dataclass
class EncodecConfig:
    model_type: str = "encodec"
    audio_channels: int = 1
    num_filters: int = 32
    kernel_size: int = 7
    num_residual_layers: int = 1
    dilation_growth_rate: int = 2
    codebook_size: int = 1024
    codebook_dim: int = 128
    hidden_size: int = 128
    num_lstm_layers: int = 2
    residual_kernel_size: int = 3
    use_causal_conv: bool = True
    normalize: bool = False
    pad_mode: str = "reflect"
    norm_type: str = "weight_norm"
    last_kernel_size: int = 7
    trim_right_ratio: float = 1.0
    compress: int = 2
    upsampling_ratios: List[int] = None
    target_bandwidths: List[float] = None
    sampling_rate: int = 24000
    chunk_length_s: Optional[float] = None
    overlap: Optional[float] = None
    architectures: List[str] = None


def filter_dataclass_fields(data_dict, dataclass_type):
    valid = {f.name for f in fields(dataclass_type)}
    return {k: v for k, v in data_dict.items() if k in valid}


def preprocess_audio(raw_audio, sampling_rate: int = 24000, chunk_length: Optional[int] = None, chunk_stride: Optional[int] = None,
                     device="cuda"):
    """encodec.py:49-86: a clip [n] / [n, C] or a list of them -> (inputs [B, max, C] float32, masks bool [B, max]) on ``device``; with
    chunking the length is padded so that the chunks tile it."""
    if not isinstance(raw_audio, list):
        raw_audio = [raw_audio]
    clips = [torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a).to(device=device, dtype=torch.float32) for a in raw_audio]
    clips = [a[:, None] if a.dim() == 1 else a for a in clips]
    m = max(a.shape[0] for a in clips)
    if chunk_length is not None:
        m += chunk_length - (m % chunk_stride)
    inputs = torch.stack([torch.nn.functional.pad(a, (0, 0, 0, m - a.shape[0])) for a in clips])
    masks = torch.stack([torch.arange(m, device=device) < a.shape[0] for a in clips])
    return inputs, masks


def param_shapes(cfg) -> dict:
    """name -> shape of every parameter of the MLX-layout checkpoint (the reference's module tree)."""
    cfg = asdict(cfg) if isinstance(cfg, EncodecConfig) else dict(asdict(EncodecConfig()), **cfg)
    S = {}
    gn = cfg["norm_type"] == "time_group_norm"

    def conv(pre, cin, cout, k):
        S[pre + ".conv.weight"], S[pre + ".conv.bias"] = (cout, k, cin), (cout,)
        if gn:
            S[pre + ".norm.weight"], S[pre + ".norm.bias"] = (cout,), (cout,)

    def res(pre, dim):
        hid = dim // cfg["compress"]
        conv(pre + ".block.1", dim, hid, cfg["residual_kernel_size"])
        conv(pre + ".block.3", hid, dim, 1)
        conv(pre + ".shortcut", dim, dim, 1)

    def lstm(pre, dim):
        for j in range(cfg["num_lstm_layers"]):
            S[f"{pre}.lstm.{j}.Wx"], S[f"{pre}.lstm.{j}.Wh"], S[f"{pre}.lstm.{j}.bias"] = (4 * dim, dim), (4 * dim, dim), (4 * dim,)

    nf, R = cfg["num_filters"], cfg["upsampling_ratios"]
    i, scale = 0, 1
    conv(f"encoder.layers.{i}", cfg["audio_channels"], nf, cfg["kernel_size"])
    i += 1
    for ratio in reversed(R):
        for _ in range(cfg["num_residual_layers"]):
            res(f"encoder.layers.{i}", scale * nf)
            i += 1
        i += 1                                                              # ELU
        conv(f"encoder.layers.{i}", scale * nf, 2 * scale * nf, 2 * ratio)
        i += 1
        scale *= 2
    lstm(f"encoder.layers.{i}", scale * nf)
    conv(f"encoder.layers.{i + 2}", scale * nf, cfg["hidden_size"], cfg["last_kernel_size"])
    i = 0
    conv(f"decoder.layers.{i}", cfg["hidden_size"], scale * nf, cfg["kernel_size"])
    lstm("decoder.layers.1", scale * nf)
    i = 2
    for ratio in R:
        i += 1                                                              # ELU
        conv(f"decoder.layers.{i}", scale * nf, scale * nf // 2, 2 * ratio)
        i += 1
        for _ in range(cfg["num_residual_layers"]):
            res(f"decoder.layers.{i}", scale * nf // 2)
            i += 1
        scale //= 2
    conv(f"decoder.layers.{i + 1}", nf, cfg["audio_channels"], cfg["last_kernel_size"])
    for q in range(int(1000 * cfg["target_bandwidths"][-1] // (math.ceil(cfg["sampling_rate"] / int(np.prod(R))) * 10))):
        S[f"quantizer.layers.{q}.codebook.embed"] = (cfg["codebook_size"], cfg["codebook_dim"])
    return S


class Encodec:
    def __init__(self, config: Union[EncodecConfig, dict], device="cuda"):
        self.config = EncodecConfig(**filter_dataclass_fields(config, EncodecConfig)) if isinstance(config, dict) else config
        c = self.config
        if c.num_residual_layers != 1:
            raise NotImplementedError("EnCodec: num_residual_layers > 1 uses dilated convs whose padding the reference derives from the "
                                      "undilated kernel size, so the residual branch and the shortcut differ in length; only 1 is supported")
        if c.norm_type not in ("weight_norm", "time_group_norm"):
            raise NotImplementedError(f"EnCodec: norm_type {c.norm_type!r} (weight_norm or time_group_norm)")
        self.device = torch.device(device)
        hop = int(np.prod(c.upsampling_ratios))
        self.frame_rate = math.ceil(c.sampling_rate / hop)
        self.num_quantizers = int(1000 * c.target_bandwidths[-1] // (self.frame_rate * 10))
        self._W = None
        self._err = None

    # ---- reference properties
    @property
    def channels(self):
        return self.config.audio_channels

    @property
    def sampling_rate(self):
        return self.config.sampling_rate

    @property
    def chunk_length(self):
        return None if self.config.chunk_length_s is None else int(self.config.chunk_length_s * self.config.sampling_rate)

    @property
    def chunk_stride(self):
        if self.config.chunk_length_s is None or self.config.overlap is None:
            return None
        return max(1, int((1.0 - self.config.overlap) * self.chunk_length))

    def get_num_quantizers_for_bandwidth(self, bandwidth: Optional[float] = None) -> int:
        """encodec.py:506-514."""
        n = self.num_quantizers
        if bandwidth is not None and bandwidth > 0.0:
            n = int(max(1, math.floor(bandwidth * 1000 / (math.log2(self.config.codebook_size) * self.frame_rate))))
        return n

    # ---- weights
    @classmethod
    def from_pretrained(cls, path: str, device="cuda"):
        """encodec.py:710-738 for a LOCAL directory (config.json + model.safetensors, MLX layout): -> (model, processor)."""
        from safetensors.torch import load_file
        p = Path(path)
        if not p.is_dir():
            raise FileNotFoundError(f"Encodec.from_pretrained: {path} is not a local directory with config.json and model.safetensors")
        with open(p / "config.json") as f:
            config = EncodecConfig(**filter_dataclass_fields(json.load(f), EncodecConfig))
        model = cls(config, device=device).load_weights(load_file(str(p / "model.safetensors")))
        processor = functools.partial(preprocess_audio, sampling_rate=config.sampling_rate, chunk_length=model.chunk_length,
                                      chunk_stride=model.chunk_stride, device=device)
        return model, processor

    def load_weights(self, weights, strict: bool = True):
        """MLX-layout parameters (``encoder.layers.0.conv.weight`` [out, k, in], ``...lstm.0.Wx``, ``quantizer.layers.0.codebook.embed``, ...)."""
        P = dict(weights)
        c, dev = self.config, self.device
        gn = c.norm_type == "time_group_norm"
        f = lambda t: torch.as_tensor(np.asarray(t) if not isinstance(t, torch.Tensor) else t).float().to(dev).contiguous()
        used = set()

        def get(k):
            used.add(k)
            return P[k]

        def host(k):
            v = get(k)
            return torch.as_tensor(np.asarray(v) if not isinstance(v, torch.Tensor) else v).float()

        def conv(pre):
            w = host(pre + ".conv.weight")
            L = {"cw": ops.pack_conv(w, f(get(pre + ".conv.bias")), 1, dev), "k": w.shape[1]}
            L["gn"] = (f(get(pre + ".norm.weight")), f(get(pre + ".norm.bias"))) if gn else None
            return L

        def res(pre):
            return {"c1": conv(pre + ".block.1"), "c2": conv(pre + ".block.3"), "sc": conv(pre + ".shortcut")}

        def lstm(pre):
            out = []
            for j in range(c.num_lstm_layers):
                q = f"{pre}.lstm.{j}"
                wx = host(q + ".Wx")
                out.append({"wx": ops.pack_linear(wx, f(get(q + ".bias")), dev), "wh": f(get(q + ".Wh"))})
            return out

        R = list(c.upsampling_ratios)
        E = {"in": conv("encoder.layers.0"), "blocks": []}
        i = 1
        for ratio in reversed(R):
            E["blocks"].append({"res": res(f"encoder.layers.{i}"), "down": conv(f"encoder.layers.{i + 2}"), "stride": ratio})
            i += 3
        E["lstm"], E["out"] = lstm(f"encoder.layers.{i}"), conv(f"encoder.layers.{i + 2}")
        D = {"in": conv("decoder.layers.0"), "lstm": lstm("decoder.layers.1"), "blocks": []}
        i = 2
        for ratio in R:
            D["blocks"].append({"up": conv(f"decoder.layers.{i + 1}"), "res": res(f"decoder.layers.{i + 2}"), "stride": ratio})
            i += 3
        D["out"] = conv(f"decoder.layers.{i + 1}")
        cbs = [f(get(f"quantizer.layers.{q}.codebook.embed")) for q in range(self.num_quantizers)]
        cb = torch.stack(cbs).contiguous()
        Q = {"cb": cb, "c2": ((cb.double() ** 2).sum(-1) / 2).contiguous()}
        if strict and set(P) - used:
            raise ValueError(f"Encodec.load_weights: unexpected parameters {sorted(set(P) - used)[:5]}")
        self._W = {"enc": E, "dec": D, "q": Q}
        return self

    def _ensure_weights(self):
        """The reference's constructor leaves a usable (randomly initialised) model; here random weights are made on first use."""
        if self._W is None:
            from ... import synth
            self.load_weights(synth.encodec_weights(asdict(self.config)))

    def _err_word(self):
        if self._err is None:
            self._err = torch.zeros(1, device=self.device, dtype=torch.int32)
        return self._err

    def _check_err(self):
        if self._err is not None and int(self._err.item()) != 0:
            self._err.zero_()
            raise RuntimeError("Encodec: an LSTM recurrence step waited more than 10 s for its cluster; the output is invalid")

    # ---- layers (x [R, T, C] fp32 channels-last)
    def _pads(self, L, k, stride):
        pt = k - stride
        extra = -(-(L - k + pt) // stride) * stride + k - pt - L
        if self.config.use_causal_conv:
            return pt, extra
        return pt - pt // 2, pt // 2 + extra

    def _finish(self, y, L, res=None):
        """GroupNorm (if any) applied, plus ``res``: the materialised output of an EncodecConv1d."""
        if L["gn"] is None:
            return y if res is None else ops.encodec_pad(y, 0, 0, reflect=False, res=res)
        return ops.encodec_pad(y, 0, 0, reflect=False, coeffs=ops.encodec_gn_coeffs(y, *L["gn"]), res=res)

    def _conv(self, x, L, *, stride=1, elu=False, res=None):
        pl, pr = self._pads(x.shape[1], L["k"], stride)
        gn = L["gn"] is not None
        if pl or pr:
            x = ops.encodec_pad(x, pl, pr, reflect=self.config.pad_mode == "reflect", elu=elu)
            pre = None
        else:
            pre = Pre(act=ACT["elu"]) if elu else None
        if gn:
            return self._finish(ops.conv1d(x, L["cw"], stride=stride, pre=pre), L, res)
        return ops.conv1d(x, L["cw"], stride=stride, pre=pre, res=res)

    def _conv_transpose(self, x, L, stride):
        k = L["k"]
        pt = k - stride
        pr = math.ceil(pt * self.config.trim_right_ratio) if self.config.use_causal_conv else pt // 2
        pl = pt - pr
        full = (x.shape[1] - 1) * stride + k
        pre = Pre(act=ACT["elu"])
        if L["gn"] is None:
            return ops.conv1d(x, L["cw"], stride=stride, transpose=True, pad_left=pl, lout=full - pl - pr, pre=pre)
        y = ops.conv1d(x, L["cw"], stride=stride, transpose=True, pad_left=0, lout=full, pre=pre)
        return ops.encodec_pad(y[:, pl:full - pr], 0, 0, reflect=False, coeffs=ops.encodec_gn_coeffs(y, *L["gn"]))

    def _res(self, x, Rb):
        h = self._conv(x, Rb["c1"], elu=True)
        sc = self._conv(x, Rb["sc"])
        return self._conv(h, Rb["c2"], elu=True, res=sc)

    def _lstm(self, x, layers):
        x = x.contiguous()
        h = x
        for j, ly in enumerate(layers):
            h = ops.encodec_lstm(ops.linear(h, ly["wx"]), ly["wh"], self._err_word(), skip=x if j == len(layers) - 1 else None)
        return h

    def _encoder(self, x):
        E = self._W["enc"]
        h = self._conv(x, E["in"])
        for blk in E["blocks"]:
            h = self._res(h, blk["res"])
            h = self._conv(h, blk["down"], stride=blk["stride"], elu=True)
        h = self._lstm(h, E["lstm"])
        return self._conv(h, E["out"], elu=True)

    def _decoder(self, z):
        D = self._W["dec"]
        h = self._conv(z, D["in"])
        h = self._lstm(h, D["lstm"])
        for blk in D["blocks"]:
            h = self._conv_transpose(h, blk["up"], blk["stride"])
            h = self._res(h, blk["res"])
        return self._conv(h, D["out"], elu=True)

    def _quantize(self, emb, nq):
        R, T, Dm = emb.shape
        Q = self._W["q"]
        codes = ops.rvq_encode(emb.reshape(R * T, Dm), Q["cb"][:nq], Q["c2"][:nq])
        return codes.reshape(R, T, nq).permute(0, 2, 1).contiguous()

    def _dequantize(self, codes):
        return ops.rvq_decode(codes.contiguous(), self._W["q"]["cb"][: codes.shape[1]].contiguous())

    # ---- public surface
    @torch.no_grad()
    def encode_latent(self, frames: torch.Tensor) -> torch.Tensor:
        """The encoder alone: [R, n, C] -> embeddings [R, T, hidden_size]."""
        self._ensure_weights()
        return self._encoder(frames.to(device=self.device, dtype=torch.float32))

    @torch.no_grad()
    def encode_frames(self, frames: torch.Tensor, masks: Optional[torch.Tensor], nq: int):
        """``_encode_frame`` on a batch of chunk rows: frames [R, L, C] -> (codes [R, nq, T], scale [R] or None)."""
        self._ensure_weights()
        scale = None
        if self.config.normalize:
            frames, scale = ops.encodec_normalize(frames, None if masks is None else masks.to(torch.uint8).contiguous())
        codes = self._quantize(self._encoder(frames), nq)
        self._check_err()
        return codes, scale

    def _chunks(self, input_values, padding_mask, bandwidth):
        c = self.config
        if bandwidth is None:
            bandwidth = c.target_bandwidths[0]
        if bandwidth not in c.target_bandwidths:
            raise ValueError(f"This model doesn't support the bandwidth {bandwidth}. Select one of {c.target_bandwidths}.")
        x = torch.as_tensor(np.asarray(input_values) if not isinstance(input_values, torch.Tensor) else input_values)
        x = x.to(device=self.device, dtype=torch.float32)
        B, n, C = x.shape
        if C < 1 or C > 2:
            raise ValueError(f"Number of audio channels must be 1 or 2, but got {C}")
        cl, st = self.chunk_length, self.chunk_stride
        if cl is None:
            cl = st = n
        step = cl - st
        if n % st != step:
            raise ValueError("The input length is not properly padded for batched chunked encoding. Make sure to pad the input correctly.")
        if padding_mask is None:
            padding_mask = torch.ones(B, n, dtype=torch.bool, device=self.device)
        m = torch.as_tensor(np.asarray(padding_mask) if not isinstance(padding_mask, torch.Tensor) else padding_mask).to(self.device).bool()
        offsets = list(range(0, n - step, st))
        return x, m, offsets, cl, self.get_num_quantizers_for_bandwidth(bandwidth)

    @torch.no_grad()
    def encode(self, input_values, padding_mask=None, bandwidth: Optional[float] = None):
        """encodec.py:585-652: input_values [B, n, C] -> (codes int64 [chunks, B, nq, T], scales: per chunk None or [B, 1, 1]).  All
        chunks of all rows run as one batch."""
        x, m, offsets, cl, nq = self._chunks(input_values, padding_mask, bandwidth)
        B = x.shape[0]
        N = len(offsets)
        if N == 1 and offsets[0] == 0 and cl == x.shape[1]:
            frames, masks = x, m
        else:
            frames = torch.stack([x[:, o:o + cl] for o in offsets]).reshape(N * B, cl, x.shape[2])
            masks = torch.stack([m[:, o:o + cl] for o in offsets]).reshape(N * B, cl)
        codes, scale = self.encode_frames(frames.contiguous(), masks, nq)
        codes = codes.reshape(N, B, nq, -1)
        scales = [None] * N if scale is None else [scale[k * B:(k + 1) * B].reshape(B, 1, 1) for k in range(N)]
        return codes, scales

    @torch.no_grad()
    def decode_frames(self, codes: torch.Tensor) -> torch.Tensor:
        """``_decode_frame`` without the scale on a batch of chunk rows: codes [R, nq, T] -> [R, L, C]."""
        self._ensure_weights()
        y = self._decoder(self._dequantize(codes.to(device=self.device, dtype=torch.int64)))
        self._check_err()
        return y

    @torch.no_grad()
    def decode(self, audio_codes, audio_scales, padding_mask=None):
        """encodec.py:740-777: codes [chunks, B, nq, T] -> audio [B, n, C]; chunked models overlap-add the chunk decodes (one batch)."""
        codes = torch.as_tensor(np.asarray(audio_codes) if not isinstance(audio_codes, torch.Tensor) else audio_codes).to(self.device)
        if self.chunk_length is None:
            if codes.shape[1] != 1:
                raise ValueError(f"Expected one frame, got {len(codes)}")
            rows, stride, scales = codes[:, 0], None, [audio_scales[0]]
        else:
            N, B = codes.shape[:2]
            rows, stride, scales = codes.reshape(N * B, codes.shape[2], codes.shape[3]), self.chunk_stride or 1, list(audio_scales)[:N]
        y = self.decode_frames(rows)
        R, L, _ = y.shape
        B = R if stride is None else codes.shape[1]
        s = None
        if scales and all(v is not None for v in scales):
            s = torch.cat([torch.as_tensor(v).to(device=self.device, dtype=torch.float32).reshape(-1) for v in scales]).contiguous()
        if stride is None:
            total = L
            if s is not None:
                y = ops.encodec_ola(y, R, s, L, L)
        else:
            total = stride * (R // B - 1) + L
        n_out = total if padding_mask is None or padding_mask.shape[1] >= total else padding_mask.shape[1]
        if stride is not None:
            return ops.encodec_ola(y, B, s, stride, n_out)
        return y[:, :n_out]
