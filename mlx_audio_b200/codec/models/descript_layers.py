"""The weight-normed Snake layers SNAC and DAC are both built from (reference: codec/models/snac/{layers,vq}.py,
codec/models/descript/nn/{layers,quantize}.py -- near copies of each other).

Loaders take the checkpoint dict ``P`` and a device and return packed layers: a weight-normed conv is an ``ops.ConvW`` folded once at
load, a Snake is a ready ``ops.Pre`` conv prologue.  Forwards take channels-last [B, L, C] tensors and block dicts made of those.
"""
from __future__ import annotations

import math
from pathlib import Path

import torch

from ... import ops
from ...ops import ACT, Pre


def fold_wn(v, g, except_dim=0):
    """snac/layers.py:9-14,57: g * v / ||v||, folded once at load in the checkpoint's dtype (SNAC checkpoints are
    float32 and the reference does not cast them, snac.py:184-199), so no rounding is applied."""
    v, g = v.double(), g.double()
    axes = tuple(i for i in range(v.dim()) if i != except_dim)
    return (g * v / torch.sqrt((v * v).sum(dim=axes, keepdim=True))).float()


def wnconv(P, pre, dev, groups=1, except_dim=0) -> ops.ConvW:
    """The weight-normed conv ``pre`` (``.weight_v``, ``.weight_g``, optional ``.bias``), MLX layout [Cout, K, Cin/groups]."""
    return ops.pack_conv(fold_wn(P[pre + ".weight_v"], P[pre + ".weight_g"], except_dim), P.get(pre + ".bias"), groups, dev)


def snake(P, name, dev) -> Pre:
    """Snake with the alpha ``name`` as a conv prologue: x + sin(a x)^2 / (a + 1e-9) (snac/layers.py:124-130, nn/layers.py:116-119)."""
    a = P[name].float().reshape(-1)
    return Pre(act=ACT["snake"], a=a.to(dev).contiguous(), b=(1.0 / (a + 1e-9)).to(dev).contiguous())


def res_units(P, block_prefix, first, groups, dev):
    """The three residual units ``{block_prefix}.{first}`` .. ``{first + 2}`` at dilations 1, 3 and 9 (snac/layers.py:208-231,
    descript/dac.py:16-33); ``groups`` is the k7 conv's (its channel count for a depthwise unit, else 1)."""
    units = []
    for i, d in enumerate((1, 3, 9)):
        rp = f"{block_prefix}.{first + i}.block.layers"
        units.append({"d": d, "s1": snake(P, rp + ".0.alpha", dev), "c1": wnconv(P, rp + ".1", dev, groups),
                      "s2": snake(P, rp + ".2.alpha", dev), "c2": wnconv(P, rp + ".3", dev)})
    return units


def res_unit(y, ru):
    """Snake -> k7 conv at dilation d -> Snake -> 1x1 conv, plus the input."""
    c1, c2, d = ru["c1"], ru["c2"], ru["d"]
    if c1.groups > 1 and c2.w_tc is not None and ops.emit_eligible(c1, y, y.shape[1], dilation=d) \
            and c2.cin_pad == c1.cout and c2.cin * c2.K >= ops.TC_MIN_K:
        # depthwise conv writes Snake2(t) as the 1x1 conv's bf16 planes: no fp32 t, no prologue pass
        t = ops.conv1d(y, c1, dilation=d, pad_left=3 * d, pre=ru["s1"], emit=ru["s2"])
        return ops.conv1d(t, c2, res=y)
    t = ops.conv1d(y, c1, dilation=d, pad_left=3 * d, pre=ru["s1"])
    return ops.conv1d(t, c2, pre=ru["s2"], res=y)


def upsample(x, blk):
    """Snake -> transposed conv (kernel 2s, stride s, cropped ceil(s / 2) per side).  The reference passes ``groups`` (= 1) in
    ``conv_transpose1d``'s ``output_padding`` slot (snac/layers.py:105-121, nn/layers.py:102-113), so every stage yields one sample more."""
    s, L = blk["stride"], x.shape[1]
    p = math.ceil(s / 2)
    lout = (L - 1) * s - 2 * p + (2 * s - 1) + 1 + 1
    return ops.conv1d(x, blk["up"], stride=s, pad_left=p, lout=lout, pre=blk["snake"], transpose=True)


def downsample(y, blk):
    """The residual units, Snake, then the strided conv (kernel 2s) padded ceil(s / 2) per side (snac/layers.py:234-253)."""
    for ru in blk["res"]:
        y = res_unit(y, ru)
    s = blk["stride"]
    return ops.conv1d(y, blk["down"], stride=s, pad_left=math.ceil(s / 2), pre=blk["snake"])


def vq_level(P, prefix, dev):
    """One residual-quantiser level (snac/vq.py:9-80, nn/quantize.py:15-64): ``cb`` the codebook [bins, cd], ``w_out`` [cd, D] and
    ``b_out`` the folded out-projection; when the level has an in-projection, also ``in_proj`` (its ConvW), ``cbn`` the L2-normalised
    codebook the cosine search runs on and ``c2`` its squared row norms (float64)."""
    f = lambda t: t.float().to(dev).contiguous()
    cb = P[prefix + ".codebook.weight"]
    lv = {"cb": f(cb), "w_out": f(fold_wn(P[prefix + ".out_proj.weight_v"], P[prefix + ".out_proj.weight_g"])[:, 0, :].t()),
          "b_out": f(P[prefix + ".out_proj.bias"])}
    if prefix + ".in_proj.weight_v" in P:
        cn = (cb.double() / cb.double().norm(dim=1, keepdim=True).clamp(min=1e-12)).float()
        lv.update(in_proj=wnconv(P, prefix + ".in_proj", dev), cbn=f(cn), c2=(cn.double() ** 2).sum(1).to(dev).contiguous())
    return lv


def snapshot_dir(repo_id) -> Path:
    """``repo_id`` when it is a local snapshot directory (config.json + model.safetensors); otherwise the hub id resolved through
    huggingface_hub, which works only when that package can reach the hub."""
    path = Path(repo_id)
    if not path.exists():
        from huggingface_hub import snapshot_download
        path = Path(snapshot_download(repo_id=repo_id, allow_patterns=["*.safetensors", "*.json"]))
    return path
