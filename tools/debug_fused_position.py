#!/usr/bin/env python
"""Is one fused conv layer position independent?  y(x)[a+h : b-h] vs y(x[a:b])[h : -h] (run on the GPU box)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from mlx_audio_b200 import ops
dev = "cuda:0"
g = torch.Generator().manual_seed(0)
def check(name, C, N, K, dil, L, a, b, act=None, exact_w=False, stride=1, transpose=False):
    x = torch.randn(1, L, C, generator=g).to(dev)
    w = torch.randn(N, K, C, generator=g) * 0.05
    if exact_w: w = w.to(torch.bfloat16).float()
    cw = ops.pack_conv(w, None, 1, dev)
    pad = (K - 1) * dil // 2
    kw = dict(dilation=dil, pad_left=pad)
    if act == "snake":
        al = (1 + 0.2 * torch.randn(C, generator=g)).abs().to(dev)
        kw["pre"] = ops.PreStats(None, None, 1e-5, ops.ACT["snake"], 0.0, al, 1.0 / al) if False else None
    yf = ops.conv_fused(ops.FusedProblem(x, cw, dilation=dil, pad_left=pad))[0]
    yp = ops.conv_fused(ops.FusedProblem(x[:, a:b].contiguous(), cw, dilation=dil, pad_left=pad))[0]
    h = pad + 1
    d = (yf[:, a + h:b - h] - yp[:, h:-h]).abs()
    print(f"{name}: max diff {float(d.max()):.3e} (ref max {float(yf.abs().max()):.2f}), nonzero {int((d > 0).sum())} of {d.numel()}")
check("C128 k7 L1000 slice 200:800", 128, 128, 7, 1, 1000, 200, 800)
check("C128 k7 L1000 slice 256:768 (tile aligned)", 128, 128, 7, 1, 1000, 256, 768)
check("C128 k7 L1000 slice 200:800 bf16-exact w", 128, 128, 7, 1, 1000, 200, 800, exact_w=True)
check("C512 k3 L300 slice 50:250", 512, 256, 3, 1, 300, 50, 250)
check("C128 k1 L20000 slice 5000:15000", 128, 128, 1, 1, 20000, 5000, 15000)
check("C128 k7 L40000 slice 5000:35000 (no split-K either way)", 128, 128, 7, 1, 40000, 5000, 35000)

print("--- through ops.conv1d (dispatcher), SNAC-shaped layers")
from mlx_audio_b200.ops import Pre, ACT
import math
def snake(C):
    al = (1 + 0.2 * torch.randn(C, generator=g)).abs().to(dev)
    return al, (1.0 / al)
def check_up(name, C, N, s, L, a, b):
    x = torch.randn(1, L, C, generator=g).to(dev)
    w = torch.randn(N, 2 * s, C, generator=g) * 0.05
    cw = ops.pack_conv(w, torch.randn(N, generator=g) * 0.1, 1, dev)
    al, ia = snake(C)
    p = math.ceil(s / 2)
    def up(xx):
        L_ = xx.shape[1]
        lout = (L_ - 1) * s - 2 * p + (2 * s - 1) + 1 + 1
        return ops.conv1d(xx, cw, stride=s, pad_left=p, lout=lout, pre=Pre(act=ACT["snake"], a=al, b=ia), transpose=True)
    yf, yp = up(x), up(x[:, a:b].contiguous())
    h = 3 * s
    d = (yf[:, a * s + h:b * s - h] - yp[:, h:(b - a) * s - h]).abs()
    print(f"{name}: max diff {float(d.max()):.3e} (ref max {float(yf.abs().max()):.2f}), nonzero {int((d > 0).sum())} of {d.numel()}")
def check_pw(name, C, N, L, a, b, cscale=False, res=False, pre=False):
    x = torch.randn(1, L, C, generator=g).to(dev)
    cw = ops.pack_conv(torch.randn(N, 1, C, generator=g) * 0.05, torch.randn(N, generator=g) * 0.1, 1, dev)
    nz = torch.randn(1, N, generator=g).to(dev) if cscale else None
    al, ia = snake(C)
    def f(xx):
        kw = {}
        if cscale: kw["cscale"] = nz
        if res: kw["res"] = xx
        if pre: kw["pre"] = Pre(act=ACT["snake"], a=al, b=ia)
        return ops.conv1d(xx, cw, **kw)
    yf, yp = f(x), f(x[:, a:b].contiguous())
    d = (yf[:, a:b] - yp).abs()
    print(f"{name}: max diff {float(d.max()):.3e} (ref max {float(yf.abs().max()):.2f}), nonzero {int((d > 0).sum())} of {d.numel()}")
check_up("up 1024->512 s8 L236 slice 104:236", 1024, 512, 8, 236, 104, 236)
check_up("up 512->256 s8 L1888 slice 800:1888", 512, 256, 8, 1888, 800, 1888)
check_up("up 256->128 s4 L15104 slice 6000:15104", 256, 128, 4, 15104, 6000, 15104)
check_up("up 128->64 s2 L60416 slice 30000:60416", 128, 64, 2, 60416, 30000, 60416)
check_pw("pw 512 noise cscale+res L1888", 512, 512, 1888, 800, 1888, cscale=True, res=True)
check_pw("pw 512 snake pre + res L1888", 512, 512, 1888, 800, 1888, res=True, pre=True)
check_pw("pw 768->1024 L236 (in_pw)", 768, 1024, 236, 104, 236)
check_pw("pw 64 snake pre + res L120832", 64, 64, 120832, 60000, 120832, res=True, pre=True)
