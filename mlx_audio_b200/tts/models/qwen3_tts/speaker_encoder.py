"""Qwen3-TTS ECAPA-TDNN speaker encoder on H100 (reference: tts/models/qwen3_tts/speaker_encoder.py).

mel [B, T, mel_dim] -> x-vector [B, enc_dim], the voice of x-vector cloning (qwen3_tts.py:285-324, 381-432).  Per SE-Res2Net block:
tdnn1 (1x1 conv), the whole Res2Net chain in ONE launch (csrc/speaker.cu: the scale-1 dependent dilated convs with their reflect pads,
halo recomputed per time tile), tdnn2, the squeeze-excitation gate (fixed-order channel mean + one gate kernel) and ``y * gate +
residual`` written straight into the block's channel slice of the MFA buffer [B, T, 3C] (the concatenation of :293-295).  The dense
layers run on the tensor-core conv; a reflect-padded ("same") layer gets its operand from ``ops.spk_reflect_pad`` -- bf16 planes with
the reflected halo rows -- and then runs unpadded.  Attentive statistics pooling splits its 3C -> A TDNN as W_x.x + (W_m.mean + W_s.std
+ b), so the [T, 3C] concatenation is never built.  Layers too small for the tensor cores (the test configurations) take the CUDA-core
conv; every launch goes through ``ops``.
"""
from __future__ import annotations

from typing import Dict

import torch

from .... import ops

_RELU = ops.ACT["lrelu"]            # leaky ReLU with slope 0


class Qwen3TTSSpeakerEncoder:
    def __init__(self, config, device="cuda"):
        self.config = config
        self.device = torch.device(device)
        self.channels = list(config.enc_channels)
        self.loaded = False

    # ------------------------------------------------------------------ weights
    @staticmethod
    def sanitize(weights: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """speaker_encoder.py:309-332: keep ``speaker_encoder.*``, strip the prefix, conv weights [out, in, K] -> [out, K, in] unless
        already MLX-layout (the reference's shape heuristic, check_array_shape_qwen3)."""
        from .speech_tokenizer import check_array_shape_qwen3
        out = {}
        for k, v in weights.items():
            if not k.startswith("speaker_encoder."):
                continue
            nk = k.replace("speaker_encoder.", "")
            if nk.endswith(".weight") and v.dim() == 3:
                v = v if check_array_shape_qwen3(v) else v.permute(0, 2, 1)
            out[nk] = v
        return out

    def load_weights(self, weights: Dict[str, torch.Tensor]):
        """MLX-layout weights without the ``speaker_encoder.`` prefix (``sanitize``'s output) -> packed device weights."""
        cfg, dev = self.config, self.device
        w = {k: torch.as_tensor(v) for k, v in weights.items()}
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        conv = lambda pre: ops.pack_conv(w[pre + ".weight"].float(), w[pre + ".bias"].float(), 1, dev)
        ch, ks, dl, sc = self.channels, cfg.enc_kernel_sizes, cfg.enc_dilations, cfg.enc_res2net_scale
        self.b0 = (conv("blocks.0.conv"), ks[0], dl[0])
        self.blocks = []
        for i in range(1, len(ch) - 1):
            p = f"blocks.{i}"
            rw = [w[f"{p}.res2net_block.blocks.{j}.conv.weight"].float().permute(1, 2, 0) for j in range(sc - 1)]    # [K, in, out]
            rb = [w[f"{p}.res2net_block.blocks.{j}.conv.bias"].float() for j in range(sc - 1)]
            self.blocks.append(dict(
                tdnn1=conv(p + ".tdnn1.conv"), tdnn2=conv(p + ".tdnn2.conv"), k=ks[i], d=dl[i],
                res_w=f32(torch.stack(rw)), res_b=f32(torch.stack(rb)),
                se_w1=f32(w[p + ".se_block.conv1.weight"][:, 0]), se_b1=f32(w[p + ".se_block.conv1.bias"]),
                se_w2=f32(w[p + ".se_block.conv2.weight"][:, 0]), se_b2=f32(w[p + ".se_block.conv2.bias"])))
        self.mfa = (conv("mfa.conv"), ks[-1], dl[-1])
        C = ch[-1]
        wa = w["asp.tdnn.conv.weight"].float()[:, 0]                                      # [A, 3C]: x | mean | std columns
        self.asp_wx = ops.pack_conv(wa[:, None, :C], None, 1, dev)
        self.asp_wms, self.asp_b = f32(wa[:, C:]), f32(w["asp.tdnn.conv.bias"])
        self.asp_conv = conv("asp.conv")
        self.fc_w, self.fc_b = f32(w["fc.weight"].float()[:, 0]), f32(w["fc.bias"])
        self.loaded = True
        return self

    # ------------------------------------------------------------------ forward
    def min_frames(self) -> int:
        """Shortest mel the reference's reflect pads accept (pad < T for every TimeDelayNetBlock)."""
        cfg = self.config
        return 1 + max((k - 1) * d // 2 for k, d in zip(cfg.enc_kernel_sizes, cfg.enc_dilations))

    @staticmethod
    def _tdnn(x: torch.Tensor, cw: ops.ConvW, k: int, d: int, out=None) -> torch.Tensor:
        """TimeDelayNetBlock (speaker_encoder.py:29-57): reflect "same" padding, conv, ReLU."""
        pad = (k - 1) * d // 2
        if pad == 0:
            return ops.conv1d(x, cw, post_act=_RELU, out=out)
        T = x.shape[1]
        if not cw.f16 and ops._tc_eligible(cw, T + 2 * pad, 1, False, 0, d):            # reflected bf16 planes straight into the TC conv
            xp = ops.spk_reflect_pad(x, pad, cw.cin_pad, 2 if ops.TC_MODE[0] == "x2" else 1)
        else:
            xp = ops.spk_reflect_pad(x, pad)
        return ops.conv1d(xp, cw, dilation=d, lout=T, post_act=_RELU, out=out)

    @torch.no_grad()
    def __call__(self, mel: torch.Tensor) -> torch.Tensor:
        """speaker_encoder.py:277-307: mel [B, T, mel_dim] -> [B, enc_dim] (float32)."""
        if not self.loaded:
            raise ValueError("speaker encoder weights are not loaded")
        x = mel if mel.dim() == 3 else mel[None]
        if x.dtype != torch.float32 or x.device != self.device or x.stride(2) != 1:
            x = x.to(device=self.device, dtype=torch.float32).contiguous()
        B, T, D = x.shape
        if D != self.config.mel_dim:
            raise ValueError(f"speaker encoder: expected {self.config.mel_dim} mel bins, got {D}")
        if T < self.min_frames():
            raise ValueError(f"speaker encoder: {T} mel frames are too few for its reflect padding (needs at least {self.min_frames()})")
        h = self._tdnn(x, *self.b0)
        widths = self.channels[1:-1]
        cat = torch.empty(B, T, sum(widths), device=self.device, dtype=torch.float32)     # MFA input: the blocks write their slices
        off = 0
        for blk, Ci in zip(self.blocks, widths):
            y = self._tdnn(h, blk["tdnn1"], 1, 1)
            z = ops.spk_res2net(y, blk["res_w"], blk["res_b"], self.config.enc_res2net_scale, blk["d"])
            y = self._tdnn(z, blk["tdnn2"], 1, 1, out=y)
            gate = ops.spk_se_gate(ops.spk_channel_stats(y, False), blk["se_w1"], blk["se_b1"], blk["se_w2"], blk["se_b2"])
            h = ops.spk_se_apply(y, gate, h, cat[:, :, off:off + Ci])
            off += Ci
        x = self._tdnn(cat, *self.mfa)
        ms = ops.spk_channel_stats(x, True, 1e-12)                                        # [B, 2C]: mean | std
        cb = ops.spk_gemv(ms, self.asp_wms, self.asp_b)                                   # W_m.mean + W_s.std + b
        a = ops.spk_asp_act(ops.conv1d(x, self.asp_wx), cb)
        pooled = ops.spk_asp_pool(ops.conv1d(a, self.asp_conv), x, 1e-12)
        return ops.spk_gemv(pooled, self.fc_w, self.fc_b)
