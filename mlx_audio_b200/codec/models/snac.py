"""SNAC multi-scale RVQ codec, decode side, on H100 (reference: codec/models/snac/{snac,layers,vq}.py).

``SNAC(**config).load_weights(...)``, ``decode(codes) -> [B, T_out, 1]`` with the reference's
signature (snac.py:101-104).  Weight-norm is folded once at load; every Snake, bias, residual add
and NoiseBlock gain is a conv prologue/epilogue; the three codebook levels are gathered, projected,
repeat-interleaved and summed by one kernel (b2a_snac_from_codes).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch

from ... import ops
from ...ops import ACT
from .descript_layers import downsample, fold_wn, res_unit, res_units, snake, snapshot_dir, upsample, vq_level, wnconv


class SNAC:
    def __init__(self, sampling_rate=44100, encoder_dim=64, encoder_rates=(3, 3, 7, 7), latent_dim=None, decoder_dim=1536,
                 decoder_rates=(7, 7, 3, 3), attn_window_size=32, codebook_size=4096, codebook_dim=8, vq_strides=(8, 4, 2, 1),
                 noise=True, depthwise=True, device="cuda"):
        self.sampling_rate = sampling_rate
        self.encoder_dim, self.encoder_rates = encoder_dim, list(encoder_rates)
        self.decoder_dim, self.decoder_rates = decoder_dim, list(decoder_rates)
        self.latent_dim = latent_dim or encoder_dim * (2 ** len(encoder_rates))
        self.hop_length = math.prod(encoder_rates)
        self.codebook_size, self.codebook_dim, self.vq_strides = codebook_size, codebook_dim, list(vq_strides)
        self.n_codebooks = len(vq_strides)
        self.attn_window_size, self.noise, self.depthwise = attn_window_size, noise, depthwise
        if attn_window_size is not None:
            raise NotImplementedError("SNAC LocalMHA (attn_window_size) is outside the accelerated configs (24 kHz model has none)")
        self.device = torch.device(device)
        self._w = None

    @classmethod
    def from_config(cls, config, device="cuda"):
        """snac.py:177-182: ``config`` = path of a config.json (as in the reference) or the already parsed dict."""
        if not isinstance(config, dict):
            import json
            with open(config, "r") as f:
                config = json.load(f)
        return cls(**config, device=device)

    @classmethod
    def from_pretrained(cls, repo_id, device="cuda", **kwargs):
        """snac.py:184-199 for a LOCAL snapshot directory (config.json + model.safetensors, already in the module-tree layout); a hub id
        is resolved through huggingface_hub only when that package can reach it."""
        path = snapshot_dir(repo_id)
        from safetensors.torch import load_file
        model = cls.from_config(path / "config.json", device=device)
        return model.load_weights(list(load_file(str(path / "model.safetensors")).items()))

    @property
    def sample_rate(self):
        return self.sampling_rate

    def load_weights(self, weights, strict=True):
        P = dict(weights)
        dev = self.device
        W = {"q": [vq_level(P, f"quantizer.quantizers.{i}", dev) for i in range(self.n_codebooks)]}
        W["from_codes"] = [[q[k] for q in W["q"]] for k in ("cb", "w_out", "b_out")]           # snac_from_codes' per-level tables
        pre = "decoder.model.layers"
        li = 0
        if self.depthwise:
            W["in_dw"] = wnconv(P, f"{pre}.{li}", dev, groups=self.latent_dim); li += 1
            W["in_pw"] = wnconv(P, f"{pre}.{li}", dev); li += 1
        else:
            W["in_pw"] = wnconv(P, f"{pre}.{li}", dev); li += 1
        W["blocks"] = []
        for i, stride in enumerate(self.decoder_rates):
            cout = self.decoder_dim // (2 ** (i + 1))
            bp = f"{pre}.{li}.block.layers"; li += 1
            blk = {"stride": stride, "snake": snake(P, f"{bp}.0.alpha", dev)}
            wt = fold_wn(P[f"{bp}.1.weight_v"], P[f"{bp}.1.weight_g"], except_dim=0).permute(2, 1, 0)     # (in,K,out)->(out,K,in)
            blk["up"] = ops.pack_conv(wt, P.get(f"{bp}.1.bias"), 1, dev)
            bi = 2
            if self.noise:
                blk["noise"] = wnconv(P, f"{bp}.{bi}.linear", dev); bi += 1
            blk["res"] = res_units(P, bp, bi, cout if self.depthwise else 1, dev)
            W["blocks"].append(blk)
        W["out_snake"] = snake(P, f"{pre}.{li}.alpha", dev); li += 1
        W["out_conv"] = wnconv(P, f"{pre}.{li}", dev)
        self._w = W
        self._enc = None
        if "encoder.block.layers.0.weight_v" in P:                     # encode side (snac/layers.py:133-158, vq.py:22-109)
            E = {"in": wnconv(P, "encoder.block.layers.0", dev), "blocks": []}
            pre, li, d = "encoder.block.layers", 1, self.encoder_dim
            for stride in self.encoder_rates:
                bp = f"{pre}.{li}.block.layers"; li += 1
                E["blocks"].append({"stride": stride, "res": res_units(P, bp, 0, d if self.depthwise else 1, dev),
                                    "snake": snake(P, f"{bp}.3.alpha", dev), "down": wnconv(P, f"{bp}.4", dev)})
                d *= 2
            E["out"] = wnconv(P, f"{pre}.{li}", dev, groups=d if self.depthwise else 1)
            self._enc = E
        return self

    @torch.no_grad()
    def decode(self, codes: List[torch.Tensor], noises: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
        """snac.py:101-104.  codes[l] int64 [B, T/stride_l] -> audio [B, T_out, 1].
        ``noises[i]`` [B,1,C_i] injects the NoiseBlock draw (one per channel, layers.py:261-267); None draws it."""
        W, dev = self._w, self.device
        codes = [c.to(device=dev, dtype=torch.int64).contiguous() for c in codes]
        z = ops.snac_from_codes(codes, self.vq_strides, *W["from_codes"], self.latent_dim)                   # [B,T,latent]
        B = z.shape[0]
        x = ops.conv1d(z, W["in_dw"], pad_left=3) if self.depthwise else z
        x = ops.conv1d(x, W["in_pw"], pad_left=0 if self.depthwise else 3)
        for i, blk in enumerate(W["blocks"]):
            x = upsample(x, blk)
            if self.noise:
                nz = noises[i] if noises is not None else torch.randn(B, 1, x.shape[2], device=dev)
                nz = nz.to(device=dev, dtype=torch.float32).reshape(B, -1).contiguous()
                x = ops.conv1d(x, blk["noise"], cscale=nz, res=x)                   # x + noise * linear(x)
            for ru in blk["res"]:
                x = res_unit(x, ru)
        return ops.conv1d(x, W["out_conv"], pad_left=3, pre=W["out_snake"], post_act=ACT["tanh"])

    # halo (in finest-level frames) that makes a span decode EXACT: first conv +-3, per block the transposed conv (+-1) and three residual
    # units of kernel 7 with dilations 1 / 3 / 9 (+-39 samples at that block's rate: 39/8 + 39/64 + ... < 6 frames), last conv +-3/512.
    SPAN_HALO = 16

    @torch.no_grad()
    def decode_span(self, codes: List[torch.Tensor], start: int, end: int, noises: Optional[List[torch.Tensor]] = None, halo: int = SPAN_HALO):
        """Audio of the finest-level frames [start, end) of a stream, decoded from those frames plus ``halo`` frames on each side: the decoder
        is convolutional, so this equals the corresponding slice of ``decode(codes)`` (SURVEY.md section 8e: one stream sharded across
        GPUs; the per-channel NoiseBlock draws ``noises`` must be the same on every shard).  ``start`` / ``end`` / ``halo`` are multiples of
        the coarsest code stride.  Returns [B, (end - start) * hop (+ the decoder's 75-sample tail when ``end`` is the stream's end), 1]."""
        top = max(self.vq_strides)
        T = codes[-1].shape[1] * self.vq_strides[-1]
        if start % top or (end % top and end != T) or halo % top or not 0 <= start < end <= T:
            raise ValueError(f"decode_span: start / end / halo must be multiples of {top} inside [0, {T}]")
        rs, re = max(0, start - halo), min(T, end + halo)
        part = [c[:, rs // st: -(-re // st)] for c, st in zip(codes, self.vq_strides)]
        y = self.decode(part, noises=noises)
        hop = math.prod(self.decoder_rates)
        lo = (start - rs) * hop
        hi = y.shape[1] if end == T else lo + (end - start) * hop
        return y[:, lo:hi]

    def decode_stream(self, codes: List[torch.Tensor], prev_codes: Optional[List[torch.Tensor]] = None, context_frames: int = 8, noises=None):
        """snac.py:106-162, literally: the first call decodes ``codes``; later calls prepend ``max(1, context_frames // stride_l)`` frames of
        context per level and decode the combination.  Kept quirk: the reference trims the context with ``full_audio[..., n:]`` on an audio
        tensor whose LAST axis is the channel ([B, T, 1]), so nothing is trimmed and the context's audio is returned again.
        -> (audio [B, T, 1], new context)."""
        new_context = [c[:, -context_frames:] if c.shape[1] > context_frames else c for c in codes]
        if prev_codes is None:
            return self.decode(codes, noises=noises), new_context
        combined = []
        for stride, prev, new in zip(self.vq_strides, prev_codes, codes):
            keep = max(1, context_frames // stride)
            prev = prev[:, -keep:] if prev.shape[1] > keep else prev
            combined.append(torch.cat([prev.to(new.device), new], dim=1))
        full_audio = self.decode(combined, noises=noises)
        context_samples = context_frames * self.hop_length
        audio = full_audio[..., context_samples:] if full_audio.shape[-1] > context_samples else full_audio
        return audio, new_context

    def preprocess(self, audio_data: torch.Tensor) -> torch.Tensor:
        """snac.py:67-84: right-pad [B, 1, n] to a multiple of hop x lcm(vq_strides)."""
        lcm = 1
        for v in self.vq_strides:
            lcm = lcm * v // math.gcd(lcm, v)
        pad_to = self.hop_length * lcm
        n = audio_data.shape[-1]
        return torch.nn.functional.pad(audio_data, (0, -n % pad_to))

    @torch.no_grad()
    def encode(self, audio_data: torch.Tensor) -> List[torch.Tensor]:
        """snac.py:95-99: audio [B, 1, n] -> codes, coarse to fine: [B, T/4], [B, T/2], [B, T] for the 24 kHz model.

        Encoder = the decoder's building blocks mirrored (k7 conv; per rate three Snake -> depthwise k7 (dilation 1 / 3 / 9) -> Snake -> 1x1
        residual units, Snake, strided conv k = 2s; depthwise k7 out conv), then per level of the residual quantiser: average-pool by the
        level's stride, 1x1 projection to 8 dims, cosine nearest-code search (`rvq_encode_kernel`, first index on ties), project the code
        back, repeat by the stride, subtract from the residual (vq.py:22-109).  Needs a checkpoint that carries the encoder."""
        residual = self.encode_latent(audio_data)                                                              # [B, T, latent]
        B, T, D = residual.shape
        codes = []
        for i, stride in enumerate(self.vq_strides):
            q = self._w["q"][i]
            xl = residual
            if stride > 1:
                t_ = (T - stride) // stride + 1
                xl = (residual[:, : t_ * stride].reshape(B, t_, stride, D).sum(dim=2) / stride).contiguous()
            ze = ops.conv1d(xl, q["in_proj"])                                                                  # [B, T', cd]
            idx = ops.rvq_encode(ze.reshape(-1, ze.shape[-1]), q["cbn"][None], q["c2"][None], mode=1)[:, 0].reshape(B, -1).contiguous()
            codes.append(idx)
            if i + 1 < len(self.vq_strides):
                zq = ops.snac_from_codes([idx], [stride], [q["cb"]], [q["w_out"]], [q["b_out"]], D, check=False)
                residual = residual - zq[:, :T] if zq.shape[1] >= T else residual - torch.nn.functional.pad(zq, (0, 0, 0, T - zq.shape[1]))
        return codes

    @torch.no_grad()
    def encode_latent(self, audio_data: torch.Tensor) -> torch.Tensor:
        """The encoder alone (snac/layers.py:133-158): audio [B, 1, n] -> z [B, T, latent] in front of the quantiser."""
        if self._enc is None:
            raise ValueError("SNAC.encode: the loaded weights have no encoder (encoder.block.layers.*)")
        E, dev = self._enc, self.device
        x = self.preprocess(audio_data.to(device=dev, dtype=torch.float32))
        x = x.reshape(x.shape[0], -1, 1)                                                                       # [B, 1, n] -> [B, n, 1] (one channel: same memory)
        y = ops.conv1d(x, E["in"], pad_left=3)
        for blk in E["blocks"]:
            y = downsample(y, blk)
        return ops.conv1d(y, E["out"], pad_left=3)
