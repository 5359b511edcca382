"""Oracle for Vocos (codec/models/vocos/vocos.py, mel.py with dsp.py:385-513): float64 restatement.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Parameters are the MLX-layout tree of the reference (``backbone.embed.weight`` [dim, k, in],
``backbone.convnext.{i}.dwconv.weight`` [dim, k, 1], ``...pwconv1.weight`` [inter, dim], ``head.out.weight`` [n_fft + 2, dim], ...).
Audio and features may carry a batch axis; the reference's head squeezes it (B = 1 only), here every row is computed independently.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import dsp as D

# The released mel checkpoint (codec/tests/test_vocos.py config_mel) and the EnCodec-feature one (config_encodec).
CONFIG_MEL = {
    "feature_extractor": {"class_path": "vocos.feature_extractors.MelSpectrogramFeatures",
                          "init_args": {"sample_rate": 24000, "n_fft": 1024, "hop_length": 256, "n_mels": 100}},
    "backbone": {"class_path": "vocos.models.VocosBackbone", "init_args": {"input_channels": 100, "dim": 512, "intermediate_dim": 1536, "num_layers": 8}},
    "head": {"class_path": "vocos.heads.ISTFTHead", "init_args": {"dim": 512, "n_fft": 1024, "hop_length": 256}},
}
CONFIG_ENCODEC = {
    "feature_extractor": {"class_path": "vocos.feature_extractors.EncodecFeatures",
                          "init_args": {"encodec_model": "encodec_24khz", "bandwidths": [1.5, 3.0, 6.0, 12.0, 24.0]}},
    "backbone": {"class_path": "vocos.models.VocosBackbone",
                 "init_args": {"input_channels": 128, "dim": 384, "intermediate_dim": 1152, "num_layers": 8, "adanorm_num_embeddings": 4}},
    "head": {"class_path": "vocos.heads.ISTFTHead", "init_args": {"dim": 384, "n_fft": 1280, "hop_length": 320, "padding": "same"}},
}


def backbone_args(cfg: dict) -> dict:
    """VocosBackbone's constructor arguments with the reference's defaults filled in (vocos.py:218-254)."""
    a = dict(layer_scale_init_value=None, adanorm_num_embeddings=None, bias=True, input_kernel_size=7, dw_kernel_size=7)
    a.update(cfg["backbone"]["init_args"])
    return a


def default_gamma(args: dict) -> float:
    """vocos.py:243: ``layer_scale_init_value or 1 / num_layers`` (a 0 falls through to 1 / num_layers as well)."""
    return args["layer_scale_init_value"] or 1 / args["num_layers"]


def mel_filters_htk(sample_rate: int, n_fft: int, n_mels: int) -> np.ndarray:
    """dsp.py:519-609 with norm=None, mel_scale="htk", in float64: [n_mels, n_fft // 2 + 1]."""
    n_freqs = n_fft // 2 + 1
    all_freqs = np.linspace(0, sample_rate // 2, n_freqs)
    m_pts = np.linspace(D._hz_to_mel(0.0, "htk"), D._hz_to_mel(sample_rate / 2, "htk"), n_mels + 2)
    f_pts = D._mel_to_hz(m_pts, "htk")
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    fb = np.maximum(0.0, np.minimum(-slopes[:, :-2] / f_diff[:-1], slopes[:, 2:] / f_diff[1:]))
    return np.ascontiguousarray(fb.T)


def log_mel_spectrogram(audio, sample_rate=24000, n_mels=100, n_fft=1024, hop_length=256) -> torch.Tensor:
    """mel.py:8-33 per row: symmetric Hann, centre reflect pad n_fft // 2, |X| of all frames but the last, HTK filters, log(max(., 1e-5)).
    audio [n] -> [1, n // hop, n_mels] as the reference returns it; [B, n] -> [B, n // hop, n_mels]."""
    a = np.asarray(torch.as_tensor(audio, dtype=torch.float64))
    rows = a[None] if a.ndim == 1 else a
    fb = mel_filters_htk(sample_rate, n_fft, n_mels)
    out = []
    for x in rows:
        mag = np.abs(D.stft(x, n_fft=n_fft, hop_length=hop_length, window=D.hanning(n_fft))[:-1])
        out.append(np.log(np.maximum(mag @ fb.T, 1e-5)))
    return torch.from_numpy(np.stack(out))


def _layer_norm(x, w, b, eps=1e-6):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    y = (x - mu) / torch.sqrt(var + eps)
    if w is not None:
        y = y * w
    if b is not None:
        y = y + b
    return y


def _norm(P, pre, x, cond, adanorm):
    """nn.LayerNorm(eps 1e-6) or AdaLayerNorm (vocos.py:198-214: scale / shift are Linear(cond), per batch row)."""
    if adanorm:
        scale = cond @ P[pre + ".scale.weight"].T + P[pre + ".scale.bias"]
        shift = cond @ P[pre + ".shift.weight"].T + P[pre + ".shift.bias"]
        return _layer_norm(x, None, None) * scale[:, None, :] + shift[:, None, :]
    return _layer_norm(x, P.get(pre + ".weight"), P.get(pre + ".bias"))


def _conv_same(x, w, b, groups=1):
    """MLX Conv1d with padding k // 2 on channels-last x [B, T, C]; w [out, k, in / groups]."""
    k = w.shape[1]
    y = torch.nn.functional.conv1d(x.transpose(1, 2), w.permute(0, 2, 1), b, padding=k // 2, groups=groups)
    return y.transpose(1, 2)


def backbone(P: dict, x, cfg: dict, bandwidth_id=None) -> torch.Tensor:
    """vocos.py:256-275: x [B, T, C] or [B, C, T] (transposed when its last dim is not input_channels) -> [B, T, dim]."""
    a = backbone_args(cfg)
    P = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in P.items()}
    x = torch.as_tensor(x, dtype=torch.float64)
    if x.shape[-1] != a["input_channels"]:
        x = x.transpose(1, 2)
    adanorm = a["adanorm_num_embeddings"] is not None
    cond = None
    if adanorm:
        assert bandwidth_id is not None
        cond = torch.as_tensor(bandwidth_id, dtype=torch.float64).reshape(-1, a["adanorm_num_embeddings"])
    dim = a["dim"]
    x = _conv_same(x, P["backbone.embed.weight"], P["backbone.embed.bias"])
    x = _norm(P, "backbone.norm", x, cond, adanorm)
    for i in range(a["num_layers"]):
        pre = f"backbone.convnext.{i}"
        r = x
        h = _conv_same(x, P[pre + ".dwconv.weight"], P[pre + ".dwconv.bias"], groups=dim)
        h = _norm(P, pre + ".norm", h, cond, adanorm)
        h = h @ P[pre + ".pwconv1.weight"].T + P[pre + ".pwconv1.bias"]
        h = 0.5 * h * (1 + torch.erf(h / math.sqrt(2)))
        h = h @ P[pre + ".pwconv2.weight"].T + P[pre + ".pwconv2.bias"]
        if pre + ".gamma" in P:
            h = P[pre + ".gamma"] * h
        x = r + h
    return _layer_norm(x, P["backbone.final_layer_norm.weight"], P.get("backbone.final_layer_norm.bias"))


def head_spectrum(P: dict, x, n_fft: int):
    """vocos.py:127-133: the complex spectra [B, n_fft / 2 + 1, T] and the fraction of bins clipped at 100."""
    P = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in P.items()}
    y = torch.as_tensor(x, dtype=torch.float64) @ P["head.out.weight"].T + P["head.out.bias"]
    return spectrum(y, n_fft)


def spectrum(y, n_fft: int):
    """The linear's output [B, T, >= n_fft + 2] -> (S [B, n_fft / 2 + 1, T] complex, clipped fraction)."""
    y = torch.as_tensor(y, dtype=torch.float64)
    nb = n_fft // 2 + 1
    mag, p = y[..., :nb].transpose(1, 2), y[..., nb:2 * nb].transpose(1, 2)
    m = torch.exp(mag)
    clipped = float((m > 100).double().mean())
    return torch.clamp(m, max=100.0) * torch.complex(torch.cos(p), torch.sin(p)), clipped


def istft(S, n_fft: int, hop: int) -> torch.Tensor:
    """dsp.py:436-513 with window=hanning(n_fft) (symmetric), win_length=n_fft, per row: [B, n_fft / 2 + 1, T] -> [B, (T - 1) hop]."""
    w = D.hanning(n_fft)
    return torch.from_numpy(np.stack([D.istft(s, hop_length=hop, win_length=n_fft, window=w) for s in np.asarray(S)]))


def head(P: dict, x, n_fft: int, hop: int) -> torch.Tensor:
    """ISTFTHead (vocos.py:119-140): [B, T, dim] -> [B, (T - 1) hop]."""
    S, _ = head_spectrum(P, x, n_fft)
    return istft(S, n_fft, hop)


def decode(P: dict, features, cfg: dict, bandwidth_id=None) -> torch.Tensor:
    h = cfg["head"]["init_args"]
    return head(P, backbone(P, features, cfg, bandwidth_id), h["n_fft"], h["hop_length"])


def forward(P: dict, audio, cfg: dict) -> torch.Tensor:
    """Vocos.__call__ for a MelSpectrogramFeatures model: audio [n] or [B, n] -> [B, samples]."""
    fe = dict(sample_rate=24000, n_fft=1024, hop_length=256, n_mels=100)
    fe.update({k: v for k, v in cfg["feature_extractor"]["init_args"].items() if k != "padding"})
    mel = log_mel_spectrogram(audio, fe["sample_rate"], fe["n_mels"], fe["n_fft"], fe["hop_length"])
    return decode(P, mel, cfg)


def output_length(cfg: dict, n_samples: int = None, frames: int = None) -> int:
    """Samples out of the mel model for n audio samples, or out of decode for ``frames`` feature frames."""
    h = cfg["head"]["init_args"]
    if frames is None:
        frames = n_samples // cfg["feature_extractor"]["init_args"].get("hop_length", 256)
    return (frames - 1) * h["hop_length"]


def sanitize(weights: dict) -> dict:
    """vocos.py:331-347: drop the two stored windows; moveaxis(1, 2) on backbone.embed and every dwconv weight (torch [out, in, k] ->
    MLX [out, k, in]).  Quirk kept: both deletions sit in one ``try``, so without the mel window the head's window stays (and is then
    ignored by the non-strict load)."""
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
