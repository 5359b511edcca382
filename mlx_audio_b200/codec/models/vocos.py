"""Vocos vocoder on H100 (reference: codec/models/vocos/{vocos,mel}.py, dsp.py:385-513).

``Vocos(audio)``: log-mel -> ConvNeXt backbone -> iSTFT head; ``Vocos.decode(features, bandwidth_id=None)`` starts at the backbone.  Per
call (mel model, at least 32 frames): one log-mel launch (``ops.vocos_logmel``), the embedding conv, the backbone norm, then per ConvNeXt
block the depthwise conv + LayerNorm / AdaLayerNorm as one ``ops.vocos_dwnorm`` launch writing the bf16 planes of pwconv1, pwconv1 with
GELU writing the planes of pwconv2, and pwconv2 with ``gamma`` and the residual in its epilogue; the final LayerNorm writes the head
linear's planes, and ``ops.vocos_istft_head`` turns the linear's output into the waveform in one launch.  AdaLayerNorm's scale / shift of
every layer come from one linear over the condition vector.

Kept from the reference: the backbone transposes its input when ``x.shape[-1] != input_channels`` (ambiguous when T == C: such an input is
taken as [B, T, C]); the head's and the feature extractor's ``padding`` are ignored; ``gamma`` defaults to ``layer_scale_init_value or
1 / num_layers``.  Extension: B > 1 everywhere (the reference's head squeezes axis 0); B = 1 returns the reference's 1-D waveform, B > 1
returns [B, samples].  Divergences: audio of <= n_fft // 2 samples raises ``ValueError`` (the reference's reflect pad silently builds a short
pad); only the released mel front end (n_fft 1024, hop 256) runs on the GPU; ``EncodecFeatures`` never loads an EnCodec model by itself
(the reference downloads one from the hub when it is constructed): audio input and ``decode_from_codes`` work once a model is attached
with ``encodec=`` (an ``Encodec`` or a local checkpoint directory) on ``EncodecFeatures``, ``from_hparams`` or ``from_pretrained``, and
raise ``NotImplementedError`` otherwise; ``decode(features, bandwidth_id=...)`` works either way.
"""
from __future__ import annotations

import math
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from ... import ops
from ...ops import ACT


def hanning(n: int) -> np.ndarray:
    """dsp.py:40-50, the symmetric window the head and the log-mel use, in float64."""
    return 0.5 * (1 - np.cos(2 * math.pi * np.arange(n) / (n - 1)))


def mel_filters_htk(sample_rate: int, n_fft: int, n_mels: int) -> np.ndarray:
    """dsp.py:519-609 with norm=None, mel_scale="htk", in float64: [n_mels, n_fft // 2 + 1]."""
    hz_to_mel = lambda f: 2595.0 * math.log10(1.0 + f / 700.0)
    all_freqs = np.linspace(0, sample_rate // 2, n_fft // 2 + 1)
    f_pts = 700.0 * (10.0 ** (np.linspace(hz_to_mel(0.0), hz_to_mel(sample_rate / 2), n_mels + 2) / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    return np.ascontiguousarray(np.maximum(0.0, np.minimum(-slopes[:, :-2] / f_diff[:-1], slopes[:, 2:] / f_diff[1:])).T)


_MEL_TABLES = {}


def _audio_rows(audio, device) -> torch.Tensor:
    a = torch.as_tensor(np.asarray(audio) if not isinstance(audio, torch.Tensor) else audio)
    a = a.to(device=device, dtype=torch.float32)
    return (a[None] if a.dim() == 1 else a).contiguous()


def log_mel_spectrogram(audio, sample_rate: int = 24_000, n_mels: int = 100, n_fft: int = 1024, hop_length: int = 256, padding: int = 0,
                        device="cuda") -> torch.Tensor:
    """mel.py:8-33 on the GPU: audio [n] -> [1, n // 256, n_mels] as the reference returns it; [B, n] -> [B, n // 256, n_mels]."""
    if n_fft != 1024 or hop_length != 256:
        raise NotImplementedError(f"Vocos log-mel: only n_fft 1024 / hop 256 (the released mel checkpoint) runs on the GPU, got {n_fft} / {hop_length}")
    x = _audio_rows(audio, device)
    if padding > 0:
        x = torch.nn.functional.pad(x, (0, padding)).contiguous()
    if x.shape[1] <= n_fft // 2:
        raise ValueError(f"Vocos log-mel: the centre reflect padding of {n_fft // 2} samples needs more than {n_fft // 2} samples, got {x.shape[1]}")
    key = (sample_rate, n_mels, x.device)
    if key not in _MEL_TABLES:
        _MEL_TABLES[key] = (torch.from_numpy(hanning(n_fft)).float().to(x.device).contiguous(),
                            torch.from_numpy(mel_filters_htk(sample_rate, n_fft, n_mels)).float().to(x.device).contiguous())
    window, filters = _MEL_TABLES[key]
    return ops.vocos_logmel(x, window, filters)


class MelSpectrogramFeatures:
    """vocos.py:25-51: ``padding`` must be "center" or "same" and is otherwise ignored (the reference passes padding=0)."""

    def __init__(self, sample_rate=24_000, n_fft=1024, hop_length=256, n_mels=100, padding="center", device="cuda"):
        if padding not in ["center", "same"]:
            raise ValueError("Padding must be 'center' or 'same'.")
        if n_fft != 1024 or hop_length != 256:
            raise NotImplementedError(f"Vocos log-mel: only n_fft 1024 / hop 256 (the released mel checkpoint) runs on the GPU, got {n_fft} / {hop_length}")
        self.padding, self.sample_rate, self.n_fft, self.hop_length, self.n_mels = padding, sample_rate, n_fft, hop_length, n_mels
        self.device = torch.device(device)

    def __call__(self, audio, **kwargs):
        return log_mel_spectrogram(audio, self.sample_rate, self.n_mels, self.n_fft, self.hop_length, 0, self.device)


class EncodecFeatures:
    """vocos.py:54-116 on an EnCodec model attached explicitly (``encodec=``: an ``Encodec``, or a local directory for
    ``Encodec.from_pretrained``).  Constructing one without a model builds nothing (``from_hparams`` on an EnCodec config builds the
    backbone and head, so ``decode(features, bandwidth_id=...)`` works); using it then raises ``NotImplementedError``."""

    def __init__(self, encodec_model="encodec_24khz", bandwidths=(1.5, 3.0, 6.0, 12.0), train_codebooks=False, encodec=None, device="cuda", **_):
        if encodec_model not in ("encodec_24khz", "encodec_48khz"):
            raise ValueError(f"Unsupported encodec_model: {encodec_model}. Supported options are 'encodec_24khz' and 'encodec_48khz'.")
        self.encodec_model, self.bandwidths = encodec_model, list(bandwidths)
        self.encodec = self.preprocessor = None
        if encodec is not None:
            self.attach(encodec, device)

    def attach(self, encodec, device="cuda"):
        """Use ``encodec`` (an ``Encodec`` or a local checkpoint directory) as this extractor's model."""
        from .encodec import Encodec, preprocess_audio
        import functools
        if isinstance(encodec, Encodec):
            self.encodec = encodec
            self.preprocessor = functools.partial(preprocess_audio, sampling_rate=encodec.sampling_rate, chunk_length=encodec.chunk_length,
                                                  chunk_stride=encodec.chunk_stride, device=encodec.device)
        else:
            self.encodec, self.preprocessor = Encodec.from_pretrained(encodec, device=device)
        self.num_q = self.encodec.get_num_quantizers_for_bandwidth(max(self.bandwidths))
        return self

    def _need(self):
        if self.encodec is None:
            raise NotImplementedError("Vocos EncodecFeatures: no EnCodec model attached; pass encodec=<Encodec or local directory> to "
                                      "EncodecFeatures / Vocos.from_hparams / Vocos.from_pretrained (decode(features, bandwidth_id=...) "
                                      "with precomputed features works without one)")

    def get_encodec_codes(self, audio, bandwidth_id):
        """audio [n] -> codes int64 [nq, 1, T] at ``bandwidths[bandwidth_id]`` (a list or tensor id: its first entry, as the reference)."""
        self._need()
        features, mask = self.preprocessor(audio)
        if isinstance(bandwidth_id, (torch.Tensor, np.ndarray)):
            bandwidth_id = int(np.asarray(torch.as_tensor(bandwidth_id).cpu()).reshape(-1)[0])
        elif isinstance(bandwidth_id, (list, tuple)):
            bandwidth_id = bandwidth_id[0]
        codes, _ = self.encodec.encode(features, mask, bandwidth=self.bandwidths[int(bandwidth_id)])
        return codes.reshape(codes.shape[-2], 1, codes.shape[-1])

    def get_features_from_codes(self, codes):
        """codes [nq <= num_q, B, T] -> the sum of their code vectors [B, T, codebook_dim] (one rvq_decode)."""
        self._need()
        codes = torch.as_tensor(np.asarray(codes) if not isinstance(codes, torch.Tensor) else codes).to(self.encodec.device, torch.int64)
        if codes.dim() != 3 or not 1 <= codes.shape[0] <= self.num_q:
            raise ValueError(f"EncodecFeatures: codes must be [1..{self.num_q}, B, T], got {tuple(codes.shape)}")
        return self.encodec._dequantize(codes.permute(1, 0, 2))

    def __call__(self, audio, **kwargs):
        self._need()
        bandwidth_id = kwargs.get("bandwidth_id")
        if bandwidth_id is None:
            raise ValueError("The 'bandwidth_id' argument is required")
        return self.get_features_from_codes(self.get_encodec_codes(audio, bandwidth_id))


class VocosBackbone:
    """vocos.py:217-275.  Weights through ``load(P, prefix)`` (MLX layout); ``__call__(x, bandwidth_id=None)``: [B, T, C] or [B, C, T]."""

    def __init__(self, input_channels, dim, intermediate_dim, num_layers, layer_scale_init_value=None, adanorm_num_embeddings=None,
                 bias=True, input_kernel_size=7, dw_kernel_size=7, device="cuda"):
        if dw_kernel_size % 2 == 0 or dw_kernel_size > 15:
            raise NotImplementedError(f"VocosBackbone: dw_kernel_size must be odd and <= 15, got {dw_kernel_size}")
        if dim % 4 or dim > 1024:
            raise NotImplementedError(f"VocosBackbone: dim must be a multiple of 4 and <= 1024, got {dim}")
        self.input_channels, self.dim, self.intermediate_dim, self.num_layers = input_channels, dim, intermediate_dim, num_layers
        self.adanorm_num_embeddings, self.adanorm = adanorm_num_embeddings, adanorm_num_embeddings is not None
        self.layer_scale_init_value = layer_scale_init_value or 1 / num_layers
        self.bias, self.input_kernel_size, self.dw_kernel_size = bias, input_kernel_size, dw_kernel_size
        self.device = torch.device(device)
        self._W = None

    def param_shapes(self, prefix="backbone.") -> dict:
        d, S = self.dim, {}
        S[prefix + "embed.weight"], S[prefix + "embed.bias"] = (d, self.input_kernel_size, self.input_channels), (d,)

        def norm(pre):
            if self.adanorm:
                for p in ("scale", "shift"):
                    S[f"{pre}.{p}.weight"], S[f"{pre}.{p}.bias"] = (d, self.adanorm_num_embeddings), (d,)
            else:
                S[pre + ".weight"], S[pre + ".bias"] = (d,), (d,)
        norm(prefix + "norm")
        for i in range(self.num_layers):
            pre = f"{prefix}convnext.{i}"
            S[pre + ".dwconv.weight"], S[pre + ".dwconv.bias"] = (d, self.dw_kernel_size, 1), (d,)
            norm(pre + ".norm")
            S[pre + ".pwconv1.weight"], S[pre + ".pwconv1.bias"] = (self.intermediate_dim, d), (self.intermediate_dim,)
            S[pre + ".pwconv2.weight"], S[pre + ".pwconv2.bias"] = (d, self.intermediate_dim), (d,)
            S[pre + ".gamma"] = (d,)
        S[prefix + "final_layer_norm.weight"] = (d,)
        if self.bias:
            S[prefix + "final_layer_norm.bias"] = (d,)
        return S

    def load(self, P: dict, prefix="backbone."):
        dev, d = self.device, self.dim
        f = lambda t: None if t is None else torch.as_tensor(t).float().to(dev).contiguous()
        W = {"embed": ops.pack_conv(torch.as_tensor(P[prefix + "embed.weight"]).float(), f(P[prefix + "embed.bias"]), 1, dev)}
        norms = [prefix + "norm"] + [f"{prefix}convnext.{i}.norm" for i in range(self.num_layers)]
        if self.adanorm:                     # every AdaLayerNorm's scale and shift linear stacked: one GEMM per call
            ws = [torch.as_tensor(P[f"{n}.{p}.weight"]).float() for n in norms for p in ("scale", "shift")]
            bs = [torch.as_tensor(P[f"{n}.{p}.bias"]).float() for n in norms for p in ("scale", "shift")]
            W["ada"] = ops.pack_linear(torch.cat(ws), torch.cat(bs), dev)
            W["norm"] = (None, None)
        else:
            W["norm"] = (f(P[prefix + "norm.weight"]), f(P[prefix + "norm.bias"]))
        W["blocks"] = []
        for i in range(self.num_layers):
            pre = f"{prefix}convnext.{i}"
            W["blocks"].append({
                "dw": ops.pack_conv(torch.as_tensor(P[pre + ".dwconv.weight"]).float(), f(P[pre + ".dwconv.bias"]), d, dev),
                "norm": (None, None) if self.adanorm else (f(P[pre + ".norm.weight"]), f(P[pre + ".norm.bias"])),
                "pw1": ops.pack_linear(torch.as_tensor(P[pre + ".pwconv1.weight"]).float(), f(P[pre + ".pwconv1.bias"]), dev),
                "pw2": ops.pack_linear(torch.as_tensor(P[pre + ".pwconv2.weight"]).float(), f(P[pre + ".pwconv2.bias"]), dev),
                "gamma": f(P[pre + ".gamma"]) if pre + ".gamma" in P else f(torch.full((d,), float(self.layer_scale_init_value))),
            })
        W["final"] = (f(P[prefix + "final_layer_norm.weight"]), f(P.get(prefix + "final_layer_norm.bias")) if self.bias else None)
        self._W = W
        return self

    def _ensure_weights(self):
        if self._W is None:
            from ... import synth
            self.load(synth.vocos_backbone_weights(self))

    def _cond(self, bandwidth_id, B):
        if not self.adanorm:
            return None
        if bandwidth_id is None:
            raise ValueError("VocosBackbone: an AdaLayerNorm backbone needs bandwidth_id (vocos.py:186, :266 assert it)")
        c = torch.as_tensor(np.asarray(bandwidth_id) if not isinstance(bandwidth_id, torch.Tensor) else bandwidth_id)
        c = c.to(device=self.device, dtype=torch.float32).reshape(-1, self.adanorm_num_embeddings)
        if c.shape[0] == 1 and B > 1:
            c = c.expand(B, -1)
        if c.shape[0] != B:
            raise ValueError(f"VocosBackbone: bandwidth_id has {c.shape[0]} rows for a batch of {B}")
        return ops.linear(c.contiguous(), self._W["ada"])          # [B, (num_layers + 1) * 2 dim]: (scale | shift) per norm

    def forward(self, x, bandwidth_id=None, planes_for: Optional[ops.ConvW] = None):
        """x [B, T, C] / [B, C, T] / [T, C], or the bf16 ``Planes`` of the embed conv -> [B, T, dim] fp32, or the bf16 planes of
        ``planes_for`` (the head linear) when that layer runs on the tensor cores."""
        self._ensure_weights()
        W, d = self._W, self.dim
        if not isinstance(x, ops.Planes):                            # Planes: the embed conv's operand, already split by its producer
            x = torch.as_tensor(x).to(device=self.device, dtype=torch.float32)
            if x.dim() == 2:
                x = x[None]
            if x.shape[-1] != self.input_channels:                  # vocos.py:259-261, ambiguous when T == C
                x = x.transpose(1, 2)
            x = x.contiguous()
        B, T, _ = x.shape
        ada = self._cond(bandwidth_id, B)
        a = lambda i: None if ada is None else ada[:, 2 * d * i: 2 * d * (i + 1)]
        k = self.input_kernel_size
        x = ops.conv1d(x, W["embed"], pad_left=k // 2, lout=T + 2 * (k // 2) - k + 1)
        x = ops.vocos_dwnorm(x, None, *W["norm"], ada=a(0))
        for i, blk in enumerate(W["blocks"]):
            if ops.emit_tc_eligible(blk["pw1"], T) and d % 64 == 0 and ops.emit_tc_eligible(blk["pw2"], T):
                pl = ops.vocos_dwnorm(x, blk["dw"], *blk["norm"], ada=a(i + 1), fp32=False, planes=True)
                _, h = ops.linear(pl, blk["pw1"], planes=True, post_act=ACT["gelu"])
            else:
                h = ops.linear(ops.vocos_dwnorm(x, blk["dw"], *blk["norm"], ada=a(i + 1)), blk["pw1"], post_act=ACT["gelu"])
            x = ops.linear(h, blk["pw2"], cscale=blk["gamma"], res=x)
        if planes_for is not None and d % 64 == 0 and ops._tc_eligible(planes_for, T, 1, False, 0) and not planes_for.f16:
            return ops.vocos_dwnorm(x, None, *W["final"], fp32=False, planes=True)
        return ops.vocos_dwnorm(x, None, *W["final"])

    @torch.no_grad()
    def __call__(self, x, bandwidth_id=None, **kwargs):
        return self.forward(x, bandwidth_id)


class ISTFTHead:
    """vocos.py:119-140.  The linear's n_fft + 2 outputs are zero-padded to a multiple of 64 at load so that it runs on the tensor cores;
    the head kernel reads the true columns at that row stride.  ``padding`` is ignored, as in the reference."""

    def __init__(self, dim, n_fft, hop_length, padding="center", device="cuda"):
        if n_fft % 2 or n_fft > 2048:
            raise NotImplementedError(f"ISTFTHead: even n_fft <= 2048 only, got {n_fft}")
        self.dim, self.n_fft, self.hop_length, self.padding = dim, n_fft, hop_length, padding
        self.device = torch.device(device)
        self._W = None

    def param_shapes(self, prefix="head.") -> dict:
        return {prefix + "out.weight": (self.n_fft + 2, self.dim), prefix + "out.bias": (self.n_fft + 2,)}

    def load(self, P: dict, prefix="head."):
        n = self.n_fft + 2
        npad = -(-n // 64) * 64
        w = torch.zeros(npad, self.dim)
        b = torch.zeros(npad)
        w[:n], b[:n] = torch.as_tensor(P[prefix + "out.weight"]).float(), torch.as_tensor(P[prefix + "out.bias"]).float()
        self._W = {"out": ops.pack_linear(w, b, self.device), "window": torch.from_numpy(hanning(self.n_fft)).float().to(self.device).contiguous()}
        return self

    def _ensure_weights(self):
        if self._W is None:
            from ... import synth
            self.load(synth.vocos_head_weights(self))

    def waveform(self, x) -> torch.Tensor:
        """[B, T, dim] fp32 or the linear's bf16 planes -> [B, (T - 1) hop]."""
        self._ensure_weights()
        T = x.shape[1]
        if T == 1:
            return torch.empty(x.shape[0], 0, device=self.device, dtype=torch.float32)
        return ops.vocos_istft_head(ops.linear(x, self._W["out"]), self.n_fft, self.hop_length, self._W["window"])

    @torch.no_grad()
    def __call__(self, x):
        y = self.waveform(torch.as_tensor(x).to(device=self.device, dtype=torch.float32).contiguous())
        return y[0] if y.shape[0] == 1 else y


class Vocos:
    """vocos.py:278-375."""

    def __init__(self, feature_extractor, backbone: VocosBackbone, head: ISTFTHead):
        self.feature_extractor, self.backbone, self.head = feature_extractor, backbone, head

    @classmethod
    def from_hparams(cls, config: dict, device="cuda", encodec=None) -> "Vocos":
        """``encodec``: the EnCodec model (or local directory) an ``EncodecFeatures`` extractor uses; nothing is loaded without it."""
        fe_cfg = config["feature_extractor"]
        if "MelSpectrogramFeatures" in fe_cfg["class_path"]:
            fe = MelSpectrogramFeatures(**fe_cfg.get("init_args", {}), device=device)
        elif "EncodecFeatures" in fe_cfg["class_path"]:
            fe = EncodecFeatures(**fe_cfg.get("init_args", {}), encodec=encodec, device=device)
        else:
            raise ValueError(f"Vocos: unknown feature extractor {fe_cfg['class_path']!r}")
        return cls(fe, VocosBackbone(**config["backbone"]["init_args"], device=device), ISTFTHead(**config["head"]["init_args"], device=device))

    @staticmethod
    def sanitize(weights: dict) -> dict:
        """vocos.py:331-347 on a torch-layout checkpoint (torch tensors or NumPy arrays): drops the two stored windows (both deletions sit
        in one ``try``, so without the mel window nothing is dropped), moves backbone.embed and every dwconv weight from [out, in, k]
        to [out, k, in]."""
        w = dict(weights)
        if "feature_extractor.mel_spec.spectrogram.window" in w:
            del w["feature_extractor.mel_spec.spectrogram.window"]
            w.pop("head.istft.window", None)
        out = {}
        for k, v in w.items():
            base, pname = k.rsplit(".", 1)
            if pname == "weight" and ("backbone.embed" in base or "dwconv" in base):
                v = v.transpose(1, 2) if isinstance(v, torch.Tensor) else np.swapaxes(v, 1, 2)
            out[k] = v
        return out

    def load_weights(self, weights, strict: bool = False):
        """MLX-layout parameters (``sanitize`` output or ``synth.vocos_weights``); keys the model does not have (``feature_extractor.*``)
        are ignored, as the reference's non-strict load ignores them."""
        P = dict(weights)
        self.backbone.load(P)
        self.head.load(P)
        return self

    @classmethod
    def from_pretrained(cls, path_or_repo: str, device="cuda", encodec=None) -> "Vocos":
        """vocos.py:307-354 for a LOCAL directory (config.yaml + model.safetensors); a hub id is resolved through huggingface_hub only
        when that package can reach it."""
        import yaml
        from safetensors.torch import load_file
        path = Path(path_or_repo)
        if not path.exists():
            from huggingface_hub import snapshot_download
            path = Path(snapshot_download(repo_id=path_or_repo, allow_patterns=["*.yaml", "*.safetensors"]))
        with open(path / "config.yaml") as f:
            config = yaml.safe_load(f)
        model = cls.from_hparams(config, device=device, encodec=encodec)
        return model.load_weights(cls.sanitize(load_file(str(path / "model.safetensors"))))

    @torch.no_grad()
    def decode(self, features_input, bandwidth_id=None, **kwargs) -> torch.Tensor:
        """features [B, T, C] (or [B, C, T], or [T, C]) -> waveform [(T - 1) hop] for B = 1, [B, (T - 1) hop] otherwise."""
        self.head._ensure_weights()
        x = self.backbone.forward(features_input, bandwidth_id, planes_for=self.head._W["out"])
        y = self.head.waveform(x)
        return y[0] if y.shape[0] == 1 else y

    @torch.no_grad()
    def __call__(self, audio_input, **kwargs) -> torch.Tensor:
        return self.decode(self.feature_extractor(audio_input, **kwargs), **kwargs)

    def get_encodec_codes(self, audio_input, bandwidth_id):
        if not isinstance(self.feature_extractor, EncodecFeatures):
            raise ValueError("This model does not support getting encodec codes.")
        return self.feature_extractor.get_encodec_codes(audio_input, bandwidth_id)

    def decode_from_codes(self, codes, **kwargs):
        return self.decode(self.feature_extractor.get_features_from_codes(codes), **kwargs)
