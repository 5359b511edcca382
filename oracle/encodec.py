"""Oracle for EnCodec (codec/models/encodec/encodec.py): float64 restatement.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Parameters are the MLX-layout tree of the reference (``encoder.layers.{i}.conv.weight``
[out, k, in], ``...norm.weight`` / ``.bias`` for time_group_norm, ``...lstm.{j}.Wx`` / ``.Wh`` [4H, H] / ``.bias`` [4H], transposed convs
[out, k, in], ``quantizer.layers.{i}.codebook.embed`` [bins, dim]).  Audio is channels-last [B, n, C].  The LSTM runs every batch row
independently (the reference's Metal kernel is only right for B = 1; see tests/golden/make_encodec_golden.py).
"""
from __future__ import annotations

import math

import numpy as np
import torch

# The two released families (mlx-community/encodec-{24,48}khz-float32 config.json).
CONFIG_24K = dict(model_type="encodec", audio_channels=1, num_filters=32, kernel_size=7, num_residual_layers=1, dilation_growth_rate=2,
                  codebook_size=1024, codebook_dim=128, hidden_size=128, num_lstm_layers=2, residual_kernel_size=3, use_causal_conv=True,
                  normalize=False, pad_mode="reflect", norm_type="weight_norm", last_kernel_size=7, trim_right_ratio=1.0, compress=2,
                  upsampling_ratios=[8, 5, 4, 2], target_bandwidths=[1.5, 3.0, 6.0, 12.0, 24.0], sampling_rate=24000,
                  chunk_length_s=None, overlap=None)
CONFIG_48K = dict(CONFIG_24K, audio_channels=2, use_causal_conv=False, normalize=True, norm_type="time_group_norm",
                  target_bandwidths=[3.0, 6.0, 12.0, 24.0], sampling_rate=48000, chunk_length_s=1.0, overlap=0.01)

DEFAULTS = dict(CONFIG_24K, upsampling_ratios=None, target_bandwidths=None)


def full_config(cfg: dict) -> dict:
    c = dict(DEFAULTS)
    c.update(cfg)
    return c


def chunk_length(cfg):
    return None if cfg["chunk_length_s"] is None else int(cfg["chunk_length_s"] * cfg["sampling_rate"])


def chunk_stride(cfg):
    if cfg["chunk_length_s"] is None or cfg["overlap"] is None:
        return None
    return max(1, int((1.0 - cfg["overlap"]) * chunk_length(cfg)))


def frame_rate(cfg):
    return math.ceil(cfg["sampling_rate"] / int(np.prod(cfg["upsampling_ratios"])))


def num_quantizers(cfg):
    return int(1000 * cfg["target_bandwidths"][-1] // (frame_rate(cfg) * 10))


def num_quantizers_for_bandwidth(cfg, bandwidth=None):
    n = num_quantizers(cfg)
    if bandwidth is not None and bandwidth > 0.0:
        n = int(max(1, math.floor(bandwidth * 1000 / (math.log2(cfg["codebook_size"]) * frame_rate(cfg)))))
    return n


def param_shapes(cfg) -> dict:
    """name -> shape of every parameter the reference's Encodec holds, in its flattening order per module."""
    cfg = full_config(cfg)
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
    for q in range(num_quantizers(cfg)):
        S[f"quantizer.layers.{q}.codebook.embed"] = (cfg["codebook_size"], cfg["codebook_dim"])
    return S


def _t(v):
    return torch.as_tensor(np.asarray(v) if not isinstance(v, torch.Tensor) else v).to(torch.float64)


def elu(x):
    return torch.where(x > 0, x, torch.expm1(torch.clamp(x, max=0.0)))


def pad1d(x, pl, pr, mode):
    """encodec.py:212-227; reflect padding of at least the input's length raises (the reference would build a short pad)."""
    if mode != "reflect":
        return torch.nn.functional.pad(x, (0, 0, pl, pr))
    L = x.shape[1]
    if max(pl, pr) >= L:
        raise ValueError(f"EnCodec reflect padding ({pl}, {pr}) needs more than {max(pl, pr)} frames, got {L}")
    pre = x[:, 1:pl + 1].flip(1)
    suf = x[:, L - pr - 1:L - 1].flip(1)
    return torch.cat([pre, x, suf], dim=1)


def group_norm(P, pre, y, eps=1e-5):
    m = y.mean(dim=(1, 2), keepdim=True)
    v = ((y - m) ** 2).mean(dim=(1, 2), keepdim=True)
    return (y - m) / torch.sqrt(v + eps) * _t(P[pre + ".norm.weight"]) + _t(P[pre + ".norm.bias"])


def conv_pads(cfg, L, k, stride):
    """EncodecConv1d's (left, right) padding for an input of L frames (encodec.py:200-245); kernel dilation 1."""
    pt = k - stride
    n_frames = -(-(L - k + pt) // stride)
    extra = n_frames * stride + k - pt - L
    if cfg["use_causal_conv"]:
        return pt, extra
    return pt - pt // 2, pt // 2 + extra


def conv(P, pre, x, cfg, stride=1):
    w = _t(P[pre + ".conv.weight"])
    k = w.shape[1]
    pl, pr = conv_pads(cfg, x.shape[1], k, stride)
    xp = pad1d(x, pl, pr, cfg["pad_mode"])
    y = torch.nn.functional.conv1d(xp.transpose(1, 2), w.permute(0, 2, 1), _t(P[pre + ".conv.bias"]), stride=stride).transpose(1, 2)
    return group_norm(P, pre, y) if cfg["norm_type"] == "time_group_norm" else y


def conv_transpose(P, pre, x, cfg, stride):
    w = _t(P[pre + ".conv.weight"])                                         # [out, k, in]
    k = w.shape[1]
    y = torch.nn.functional.conv_transpose1d(x.transpose(1, 2), w.permute(2, 0, 1), _t(P[pre + ".conv.bias"]), stride=stride).transpose(1, 2)
    if cfg["norm_type"] == "time_group_norm":
        y = group_norm(P, pre, y)
    pt = k - stride
    pr = math.ceil(pt * cfg["trim_right_ratio"]) if cfg["use_causal_conv"] else pt // 2
    return y[:, pt - pr: y.shape[1] - pr]


def lstm_layer(P, pre, x):
    """One LSTM layer, every row independently, h0 = c0 = 0: x [B, T, H] -> [B, T, H]."""
    Wx, Wh, b = _t(P[pre + ".Wx"]), _t(P[pre + ".Wh"]), _t(P[pre + ".bias"])
    H = Wh.shape[1]
    xp = x @ Wx.T + b
    h = torch.zeros(x.shape[0], H, dtype=torch.float64)
    c = torch.zeros_like(h)
    out = []
    for t in range(x.shape[1]):
        g = xp[:, t] + h @ Wh.T
        i, f, gg, o = torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H]), torch.tanh(g[:, 2 * H:3 * H]), torch.sigmoid(g[:, 3 * H:])
        c = f * c + i * gg
        h = o * torch.tanh(c)
        out.append(h)
    return torch.stack(out, dim=1)


def lstm_block(P, pre, x, cfg):
    h = x
    for j in range(cfg["num_lstm_layers"]):
        h = lstm_layer(P, f"{pre}.lstm.{j}", h)
    return h + x


def resnet_block(P, pre, x, cfg):
    h = conv(P, pre + ".block.1", elu(x), cfg)
    h = conv(P, pre + ".block.3", elu(h), cfg)
    return conv(P, pre + ".shortcut", x, cfg) + h


def check_config(cfg):
    if cfg["num_residual_layers"] != 1:
        raise NotImplementedError("EnCodec: num_residual_layers > 1 uses dilated convs whose padding the reference derives from the "
                                  "undilated kernel size, so the residual branch and the shortcut differ in length; only 1 is supported")


def encoder(P, x, cfg):
    """[B, n, C] -> embeddings [B, T, hidden_size]."""
    cfg = full_config(cfg)
    check_config(cfg)
    h = conv(P, "encoder.layers.0", _t(x), cfg)
    i = 1
    for ratio in reversed(cfg["upsampling_ratios"]):
        h = resnet_block(P, f"encoder.layers.{i}", h, cfg)
        h = conv(P, f"encoder.layers.{i + 2}", elu(h), cfg, stride=ratio)
        i += 3
    h = lstm_block(P, f"encoder.layers.{i}", h, cfg)
    return conv(P, f"encoder.layers.{i + 2}", elu(h), cfg)


def decoder(P, z, cfg):
    """embeddings [B, T, hidden_size] -> audio [B, n, C]."""
    cfg = full_config(cfg)
    check_config(cfg)
    h = conv(P, "decoder.layers.0", _t(z), cfg)
    h = lstm_block(P, "decoder.layers.1", h, cfg)
    i = 2
    for ratio in cfg["upsampling_ratios"]:
        h = conv_transpose(P, f"decoder.layers.{i + 1}", elu(h), cfg, ratio)
        h = resnet_block(P, f"decoder.layers.{i + 2}", h, cfg)
        i += 3
    return conv(P, f"decoder.layers.{i + 1}", elu(h), cfg)


def codebooks(P, n):
    return [_t(P[f"quantizer.layers.{q}.codebook.embed"]) for q in range(n)]


def quantize(P, emb, n, with_margin=False):
    """Residual quantiser (encodec.py:452-533): emb [B, T, D] -> codes int64 [B, n, T]; ``with_margin``: also the smallest gap, per
    frame over all levels, between the best and second-best squared distance."""
    r = _t(emb)
    codes, margin = [], torch.full(r.shape[:2], float("inf"), dtype=torch.float64)
    for e in codebooks(P, n):
        d = (e * e).sum(1) - 2 * r @ e.T                                    # |x|^2 dropped: the same for every code
        two = torch.topk(d, 2, dim=-1, largest=False).values
        margin = torch.minimum(margin, two[..., 1] - two[..., 0])
        idx = torch.argmin(d, dim=-1)
        codes.append(idx)
        r = r - e[idx]
    c = torch.stack(codes, dim=1)
    return (c, margin) if with_margin else c


def dequantize(P, codes):
    """codes [B, n, T] -> [B, T, D]."""
    cbs = codebooks(P, codes.shape[1])
    return sum(cbs[q][codes[:, q]] for q in range(codes.shape[1]))


def check_bandwidth(cfg, bandwidth):
    if bandwidth is None:
        bandwidth = cfg["target_bandwidths"][0]
    if bandwidth not in cfg["target_bandwidths"]:
        raise ValueError(f"This model doesn't support the bandwidth {bandwidth}. Select one of {cfg['target_bandwidths']}.")
    return bandwidth


def chunk_offsets(cfg, n):
    cl, st = chunk_length(cfg), chunk_stride(cfg)
    if cl is None:
        cl = st = n
    step = cl - st
    if n % st != step:
        raise ValueError("The input length is not properly padded for batched chunked encoding. Make sure to pad the input correctly.")
    return list(range(0, n - step, st)), cl


def normalize(x, mask):
    """encodec.py:574-579: (x * mask / scale, scale [B, 1, 1])."""
    x = x * _t(mask)[..., None]
    mono = x.sum(2, keepdim=True) / x.shape[2]
    scale = torch.sqrt((mono ** 2).mean(1, keepdim=True)) + 1e-8
    return x / scale, scale


def encode(P, x, cfg, padding_mask=None, bandwidth=None, return_embeddings=False):
    """Encodec.encode: x [B, n, C] -> (codes int64 [chunks, B, nq, T], scales: per chunk None or [B, 1, 1])."""
    cfg = full_config(cfg)
    bandwidth = check_bandwidth(cfg, bandwidth)
    x = _t(x)
    B, n, C = x.shape
    if C < 1 or C > 2:
        raise ValueError(f"Number of audio channels must be 1 or 2, but got {C}")
    if padding_mask is None:
        padding_mask = torch.ones(B, n, dtype=torch.bool)
    padding_mask = torch.as_tensor(np.asarray(padding_mask)).bool()
    offsets, cl = chunk_offsets(cfg, n)
    nq = num_quantizers_for_bandwidth(cfg, bandwidth)
    codes, scales, embs = [], [], []
    for off in offsets:
        frame = x[:, off:off + cl]
        scale = None
        if cfg["normalize"]:
            frame, scale = normalize(frame, padding_mask[:, off:off + cl])
        e = encoder(P, frame, cfg)
        embs.append(e)
        codes.append(quantize(P, e, nq))
        scales.append(scale)
    out = (torch.stack(codes), scales)
    return out + (embs,) if return_embeddings else out


def linear_overlap_add(frames, stride):
    """encodec.py:654-677 in float64: frames list of [B, L, C]."""
    B, L, C = frames[0].shape
    total = stride * (len(frames) - 1) + frames[-1].shape[1]
    tv = torch.linspace(0, 1, L + 2, dtype=torch.float64)[1:-1]
    w = (0.5 - (tv - 0.5).abs())[:, None]
    out = torch.zeros(B, total, C, dtype=torch.float64)
    sw = torch.zeros(total, 1, dtype=torch.float64)
    off = 0
    for f in frames:
        n = f.shape[1]
        out[:, off:off + n] += w[:n] * f
        sw[off:off + n] += w[:n]
        off += stride
    return out / sw


def decode(P, codes, scales, cfg, padding_mask=None):
    """Encodec.decode: codes [chunks, B, nq, T] -> audio [B, n, C]."""
    cfg = full_config(cfg)
    codes = torch.as_tensor(np.asarray(codes) if not isinstance(codes, torch.Tensor) else codes).long()
    if chunk_length(cfg) is None:
        if codes.shape[1] != 1:
            raise ValueError(f"Expected one frame, got {len(codes)}")
        s = scales[0]
        y = decoder(P, dequantize(P, codes[:, 0]), cfg)
        audio = y if s is None else y * _t(s)
    else:
        frames = []
        for c, s in zip(codes, scales):
            y = decoder(P, dequantize(P, c), cfg)
            frames.append(y if s is None else y * _t(s))
        audio = linear_overlap_add(frames, chunk_stride(cfg) or 1)
    if padding_mask is not None and padding_mask.shape[1] < audio.shape[1]:
        audio = audio[:, :padding_mask.shape[1]]
    return audio


def preprocess_audio(raw_audio, sampling_rate=24000, chunk_length=None, chunk_stride=None):
    """encodec.py:49-86: clips [n] or [n, C] -> (inputs [B, max, C], masks bool [B, max])."""
    if not isinstance(raw_audio, list):
        raw_audio = [raw_audio]
    raw = [_t(a) for a in raw_audio]
    raw = [a[:, None] if a.dim() == 1 else a for a in raw]
    m = max(a.shape[0] for a in raw)
    if chunk_length is not None:
        m += chunk_length - (m % chunk_stride)
    inputs = torch.stack([torch.nn.functional.pad(a, (0, 0, 0, m - a.shape[0])) for a in raw])
    masks = torch.stack([torch.arange(m) < a.shape[0] for a in raw])
    return inputs, masks


def encoded_frames(cfg, n):
    """Frames the encoder makes from n samples (every conv rounds up by its extra padding)."""
    cfg = full_config(cfg)
    L = n
    L = L + sum(conv_pads(cfg, L, cfg["kernel_size"], 1)) - cfg["kernel_size"] + 1
    for r in reversed(cfg["upsampling_ratios"]):
        pl, pr = conv_pads(cfg, L, 2 * r, r)
        L = (L + pl + pr - 2 * r) // r + 1
    return L
