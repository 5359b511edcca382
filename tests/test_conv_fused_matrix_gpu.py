"""Fused conv kernel (csrc/conv_fused.cu: b2a_conv1d_fused) against float64, one host decision at a time.

The host code picks, per problem, an N tile (BN 128 / 96 / 64 / 32, each its own mma_tile variant), one of eleven A-chunk converter
bodies (16-bit type x number of summed inputs x prologue activation), a prologue (none, scale / shift, or AdaIN / InstanceNorm
coefficients derived from binned statistics, tabled per CTA when Cin <= 1280) and a K split (none, several CTAs, or none because the
workspace is full).  Every case runs through ops.conv_fused, asserts the tiling the launch reports (ops.conv1d_fused_last_config) against
_plan, a restatement of the host rules, and compares the output with a float64 CPU reference: the prologue, the convolution (or the
polyphase scatter plus crop; rows past the crop get the epilogue alone) and the epilogue in epilogue_tile's order (bias, post_act,
cscale * out_scale, + res[l / res_div] * out_scale, + previous y).

x is a channel slice of a NaN-filled buffer (rows above and below NaN too), and so are the summed inputs; y is a channel slice of a
NaN-filled buffer with guard rows; residuals carry NaN rows past the ones the layer may read.  A read outside the layer's span poisons
the result and a write past Lout or Cout shows up as a lost NaN.

Errors are max |y - ref| / max |ref|: x2 (hi + lo activation planes) <= 2e-5 for every weight kind, x1 within its plane's rounding
(TOL_X1, as in test_gemm_tc_matrix_gpu.py).  fp16 inputs stay inside the RMS range that file shows to be fp32-grade (2^-7 .. 2^10).
Output statistics are within 1e-6 of the float64 sums of what was written and bit-identical on a repeat run."""
import dataclasses
import os
import subprocess
import sys
import zlib
from typing import Optional

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import nn as ON

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL_X2 = 2e-5
TOL_X1 = {"bf16": 4e-3, "fp16": 5e-4, "fp32": 4e-3}      # test_gemm_tc_matrix_gpu.py
STATS_TOL = 1e-6
GUARD = 2                                               # NaN rows above and below the output, per batch row
PRE_P0, POST_P0, EPS = 0.15, 0.2, 1e-5
LRELU, SNAKE, ELU = 1, 2, 3                             # B2A_ACT_* (include/b200audio.h)
ACT = {"lrelu": 1, "snake": 2, "elu": 3, "gelu": 4, "gelu_tanh": 5, "tanh": 6, "sigmoid": 7, "silu": 8, "clip1": 9}   # ops.ACT
RUNTIME_ACTS = ("gelu", "gelu_tanh", "tanh", "sigmoid", "silu", "clip1")
TM, TK, CT_MAX, MAXG = 128, 64, 1280, 4                 # conv_fused.cu: row tile, K chunk, coefficient-table channels, problems

# ------------------------------------------------------------------------------------------------------------------------ branch keys
BODIES = {"plain", "add1", "add2", "snake", "lrelu", "elu", "act", "f16_plain", "f16_add1", "f16_add2", "f16_act"}
PRE_KINDS = ("scale", "stats", "stats_gb", "stats_gbb")
BRANCHES = {
    *[("tile", bn, kind) for bn in (128, 96, 64, 32) for kind in ("dense", "poly")],
    *[("body", b) for b in BODIES],
    ("pre", "none"), *[("pre", k, t) for k in PRE_KINDS for t in ("tabled", "untabled")],
    *[("split", s) for s in ("1", "k", "fallback")],
}


def _act_ref(name, v, p0, a=None, b=None):
    if name == "snake":
        return v + (1.0 if b is None else b) * torch.sin((1.0 if a is None else a) * v) ** 2
    return {"lrelu": lambda: ON.leaky_relu(v, p0), "elu": lambda: ON.elu(v), "gelu": lambda: ON.gelu(v),
            "gelu_tanh": lambda: ON.gelu_approx(v), "tanh": lambda: torch.tanh(v), "sigmoid": lambda: torch.sigmoid(v),
            "silu": lambda: F.silu(v), "clip1": lambda: v.clamp(-1.0, 1.0)}[name]()


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    B: int
    L: int
    Cin: int
    Cout: int
    K: int
    dil: int = 1
    pad: Optional[int] = None        # pad_left (dense) or left crop (transposed); default (K - 1) * dil // 2, transposed 0
    stride: int = 1                  # transposed only: polyphase with N = stride * Cout
    transpose: bool = False
    lout: Optional[int] = None       # default: L (dense), (L - 1) * stride + K - 2 * pad (transposed)
    wkind: str = "bf16"              # weights exact in bf16, exact in fp16, or fp32 (bf16 hi + lo planes)
    mode: str = "x2"                 # activation planes: "x2" hi + lo, "x1" hi only
    pre: Optional[str] = None        # None, "scale" ([B, Cin] scale / shift), "stats" (InstanceNorm), "stats_gb" (AdaIN), "stats_gbb" ([1, 2Cin] rows)
    act: Optional[str] = None        # prologue activation
    nadd: int = 0                    # x_add tensors summed into x
    in_scale: float = 1.0
    x_scale: float = 1.0
    a_range: tuple = (0.5, 1.5)      # Snake alpha ~ U(a_range); beta = 1 / alpha
    bias: bool = True
    post: Optional[str] = None
    cscale: Optional[str] = None     # "c": [Cout]; "bc": [B, Cout]
    res: Optional[str] = None        # "full": [B, ., Cout]; "bcast": [1, ., Cout]
    res_div: int = 1
    out_scale: float = 1.0
    accumulate: bool = False
    stats_out: bool = False
    x_off: Optional[int] = 4         # channel offset of x in its NaN-guarded buffer (a multiple of 4); None: contiguous
    y_off: int = 4

    @property
    def padl(self):
        if self.pad is not None:
            return self.pad
        return 0 if self.transpose else (self.K - 1) * self.dil // 2

    @property
    def taps(self):
        return self.K // self.stride if self.transpose else self.K

    @property
    def span(self):
        return self.taps - 1 if self.transpose else (self.K - 1) * self.dil

    @property
    def N(self):
        return self.stride * self.Cout if self.transpose else self.Cout

    @property
    def Lout(self):
        if self.lout is not None:
            return self.lout
        return (self.L - 1) * self.stride + self.K - 2 * self.padl if self.transpose else self.L

    @property
    def mrows(self):
        """GEMM rows: every output row (dense), or every polyphase row that reaches an output row below Lout."""
        if self.transpose:
            return max(self.L + self.taps - 1, -(-(self.Lout + self.padl) // self.stride))
        return self.Lout

    @property
    def cin_pad(self):
        return -(-self.Cin // TK) * TK

    @property
    def bn(self):
        return next(c for c in (128, 96, 64, 32) if self.N % c == 0 and self.Cout % c == 0)

    @property
    def body(self):
        act = ACT[self.act] if self.act else 0
        if self.wkind == "fp16":
            if self.nadd == 0 and act == 0:
                return "f16_plain"
            return {2: "f16_add2", 1: "f16_add1", 0: "f16_act"}[self.nadd]
        if self.nadd:
            return f"add{self.nadd}"
        return {0: "plain", SNAKE: "snake", LRELU: "lrelu", ELU: "elu"}.get(act, "act")


# ------------------------------------------------------------------------------------------------------------ the host rules, restated
@dataclasses.dataclass
class Plan:
    grid: int
    BN: list          # caller order
    ksplit: list
    kper: list
    fallback: list
    tiles: int


def _nsm():
    from mlx_audio_b200 import _lib
    return _lib.lib().b2a_device_sm_count()


def _plan(cases, nsm, ws_bytes) -> Plan:
    """b2a_conv1d_fused's tiling: heaviest problem first (taps x cin_pad), K split when the whole launch has at most nsm / 2 output
    tiles and the problem at least 4 K chunks, each split problem's partial tiles and counters placed in the workspace in that order."""
    n = len(cases)
    base = [-(-c.mrows // TM) * (c.N // c.bn) * c.B for c in cases]
    sum_base = sum(base)
    cost = [c.taps * c.cin_pad for c in cases]
    order = list(range(n))
    for i in range(n):                                  # the host's selection sort (ties keep no particular order)
        for j in range(i + 1, n):
            if cost[order[j]] > cost[order[i]]:
                order[i], order[j] = order[j], order[i]
    ks, kp, fb = [1] * n, [0] * n, [False] * n
    ws_used, cnt_used, tiles = 0, 0, 0
    for i in order:
        c = cases[i]
        kchunks = c.cin_pad // TK
        k = 1
        if sum_base * 2 <= nsm and kchunks >= 4 and ws_bytes:
            k = min(nsm // sum_base, 8, kchunks // 2)
            k = k if k >= 2 else 1
        kper = -(-kchunks // k)
        k = -(-kchunks // kper)
        if k > 1:
            nbytes = base[i] * k * TM * c.bn * 4
            if 4096 + ws_used + nbytes > ws_bytes or cnt_used + base[i] > 1024:
                k, kper, fb[i] = 1, kchunks, True
            else:
                ws_used += nbytes
                cnt_used += base[i]
        ks[i], kp[i] = k, kper
        tiles += base[i] * k
    return Plan(min(tiles, nsm), [c.bn for c in cases], ks, kp, fb, tiles)


def _keys(c: Case, plan: Plan, i: int = 0) -> set:
    pre = ("pre", "none") if c.pre is None else ("pre", c.pre, "tabled" if c.Cin <= CT_MAX else "untabled")
    split = "fallback" if plan.fallback[i] else ("k" if plan.ksplit[i] > 1 else "1")
    return {("tile", c.bn, "poly" if c.transpose else "dense"), ("body", c.body), pre, ("split", split)}


# --------------------------------------------------------------------------------------------------------------------------- cases
def _poly(name, B, L, Cin, C, K, stride, pad, **kw):
    return Case(name, B, L, Cin, C, K, stride=stride, pad=pad, transpose=True, **kw)


BRANCH_CASES = [
    # ---- N tiles: dense at each BN; polyphase at each BN (the tile divides C), all with a left crop
    Case("bn128_dense", 2, 300, 160, 256, 3, act="lrelu"),
    Case("bn96_dense", 1, 200, 100, 288, 3, pre="scale"),
    Case("bn64_dense", 2, 129, 64, 320, 5, dil=2, act="elu"),
    Case("bn32_dense", 1, 250, 65, 160, 3),
    _poly("bn128_poly_c256", 2, 60, 128, 256, 4, 2, 1, act="lrelu", stats_out=True),
    _poly("bn96_poly_c96", 2, 50, 64, 96, 6, 2, 2, act="snake"),
    _poly("bn64_poly_c64", 1, 70, 100, 64, 4, 2, 1, pre="scale", act="lrelu"),
    _poly("bn32_poly_c32_s4", 2, 40, 64, 32, 8, 4, 2, act="elu"),
    # ---- converter bodies: bf16 x {two inputs, one input, plain, Snake, LeakyReLU, ELU, runtime activation}, fp16 x {plain, two, one, runtime}
    Case("body_add2_snake_runtime", 2, 200, 96, 128, 3, nadd=2, in_scale=1 / 3, act="snake"),
    Case("body_add1_lrelu", 1, 180, 130, 128, 5, nadd=1, in_scale=0.5, act="lrelu"),
    Case("body_add1_plain_stats", 2, 140, 64, 96, 3, nadd=1, in_scale=0.5, pre="stats"),
    Case("body_plain_contiguous_x", 1, 200, 128, 128, 3, x_off=None),
    Case("body_snake_stats_gb", 2, 160, 96, 128, 7, dil=3, pre="stats_gb", act="snake"),
    Case("body_lrelu_scale_in_scale", 2, 150, 70, 64, 3, pre="scale", in_scale=0.7, act="lrelu"),
    Case("body_elu", 1, 210, 128, 128, 3, act="elu"),
    *[Case(f"body_act_{a}", 1, 150, 72, 64, 3, act=a, x_scale=2.0) for a in RUNTIME_ACTS],
    Case("body_f16_plain", 1, 200, 96, 128, 3, wkind="fp16"),
    Case("body_f16_add2_elu", 1, 170, 64, 96, 3, wkind="fp16", nadd=2, in_scale=1 / 3, act="elu"),
    Case("body_f16_add1", 2, 140, 100, 64, 3, wkind="fp16", nadd=1),
    Case("body_f16_act_gelu", 1, 160, 64, 128, 5, wkind="fp16", act="gelu", pre="scale"),
    # ---- prologues: scale / shift and statistics with per-batch, broadcast or no gamma|beta rows, tabled (Cin <= 1280) and not
    Case("pre_scale_tabled_1280", 2, 130, 1280, 64, 3, pre="scale", act="snake"),
    Case("pre_scale_untabled_1281", 2, 130, 1281, 64, 3, pre="scale", in_scale=0.5, act="lrelu"),
    Case("pre_stats_tabled", 3, 140, 1280, 32, 1, pre="stats", in_scale=2.0),
    Case("pre_stats_untabled", 3, 140, 1281, 32, 1, pre="stats", act="elu"),
    Case("pre_stats_gb_tabled", 2, 130, 1280, 64, 3, pre="stats_gb", act="snake"),
    Case("pre_stats_gb_untabled", 2, 130, 1281, 64, 3, pre="stats_gb", act="snake", in_scale=0.5),
    Case("pre_stats_gbb_tabled", 3, 200, 96, 128, 3, pre="stats_gbb", act="lrelu"),
    Case("pre_stats_gbb_untabled", 3, 100, 1281, 32, 1, pre="stats_gbb"),
    # ---- K split with the statistics prologue, and the precisions under it
    Case("split_fp32_x2", 1, 200, 512, 128, 3, wkind="fp32"),
    Case("split_fp16_x1", 1, 200, 512, 128, 3, wkind="fp16", mode="x1"),
    Case("split_bf16_x1_stats", 1, 150, 400, 64, 3, mode="x1", pre="stats_gb", act="snake"),
]

GEOMETRY_CASES = [
    # ---- lengths at the 128-row tile edges
    *[Case(f"len_{L}", 2, L, 64, 128, 3, pre="scale", act="lrelu") for L in (37, 127, 128, 129)],
    # ---- several waves of persistent CTAs, each meeting tiles of another batch row with other coefficients
    Case("waves_scale_b3", 3, 44 * 128 + 37, 64, 256, 3, pre="scale", act="lrelu"),
    Case("waves_stats_gb_b3", 3, 44 * 128 + 37, 64, 256, 3, pre="stats_gb", act="snake"),
    # ---- tap spans 0, 63 and 64, with negative shifts and asymmetric left padding
    Case("span0_linear", 2, 150, 64, 64, 1),
    Case("span63_asym", 1, 300, 64, 128, 8, dil=9, pad=10),
    Case("span64_all_negative", 1, 300, 64, 128, 5, dil=16, pad=64),
    Case("span64_all_positive", 1, 300, 64, 96, 2, dil=64, pad=0),
    Case("span64_centered_stats", 2, 200, 96, 64, 3, dil=32, pre="stats", act="elu"),
    # ---- input widths
    Case("cin1_k32", 2, 300, 1, 64, 32, dil=2),
    Case("cin2_k16", 1, 260, 2, 64, 16, dil=4, act="snake"),
    Case("cin3_k11", 1, 260, 3, 32, 11, dil=6, pre="scale"),
    Case("cin60", 1, 200, 60, 64, 3),
    Case("cin64", 1, 200, 64, 64, 3, act="lrelu"),
    Case("cin65", 1, 200, 65, 64, 3, pre="stats_gb"),
    Case("cin1281_b1", 1, 140, 1281, 32, 1, act="lrelu"),
    # ---- Snake arguments |a x| up to ~5e3 on the specialised body (b2a_sin_fast) and the runtime body (b2a_sin)
    Case("snake_big_fast", 1, 300, 64, 128, 3, act="snake", x_scale=300.0, a_range=(1.0, 4.0)),
    Case("snake_big_runtime_f16", 1, 300, 64, 128, 3, act="snake", x_scale=300.0, a_range=(1.0, 4.0), wkind="fp16"),
    Case("snake_big_runtime_add1", 1, 300, 64, 128, 3, act="snake", x_scale=150.0, a_range=(1.0, 4.0), nadd=1),
]

# Each epilogue field alone, then all together, on dense BN 128 with split K, dense BN 32 without, and polyphase (BN 64).  The bases
# have no bias and B = 3 so that the per-batch forms differ from the shared ones; every case also writes output statistics.
POSTS = ("lrelu", "snake", "elu", "gelu", "gelu_tanh", "tanh", "sigmoid", "silu", "clip1")
EPILOGUES = {
    "bare": {}, "bias": dict(bias=True), **{f"post_{a}": dict(post=a) for a in POSTS},
    "cscale": dict(cscale="c"), "cscale_per_batch": dict(cscale="bc"), "res": dict(res="full"), "res_bcast": dict(res="bcast"),
    "res_div2": dict(res="full", res_div=2), "out_scale_neg": dict(out_scale=-0.7), "accumulate": dict(accumulate=True),
    "all": dict(bias=True, post="silu", cscale="bc", res="bcast", res_div=2, out_scale=-0.7, accumulate=True),
}
EPILOGUE_BASES = [
    Case("ep_dense128_splitk", 3, 200, 320, 128, 3, bias=False, stats_out=True, act="lrelu"),
    Case("ep_dense32", 3, 150, 60, 32, 5, dil=2, bias=False, stats_out=True),
    _poly("ep_poly64", 3, 40, 64, 64, 6, 2, 2, bias=False, stats_out=True, act="lrelu"),
]
EPILOGUE_CASES = [dataclasses.replace(b, name=f"{b.name}-{e}", **f) for b in EPILOGUE_BASES for e, f in EPILOGUES.items()]

# Groups: caller order is not the heaviest-first order, problems differ in BN, span, Cin, prologue and dense / polyphase.
GROUPS = {
    "g2_dense_poly": [
        _poly("g2_poly_bn64", 2, 60, 96, 64, 4, 2, 1, act="lrelu", stats_out=True),
        Case("g2_dense_bn128_span54", 1, 300, 160, 128, 7, dil=9, pre="scale", act="snake"),
    ],
    "g2_split_pair": [
        Case("g2s_shortcut_k1", 1, 200, 512, 128, 1, stats_out=True),
        Case("g2s_conv_k3", 1, 200, 512, 128, 3, pre="stats", act="lrelu"),
    ],
    "g3_resblock_like": [
        Case("g3_k3_bn96_stats_gb", 2, 150, 64, 96, 3, pre="stats_gb", act="snake"),
        Case("g3_k7_span54_bn128", 2, 150, 200, 256, 7, dil=9, act="snake", stats_out=True),
        Case("g3_k1_cin1281_bn32", 2, 150, 1281, 32, 1, pre="scale", act="lrelu"),
    ],
    "g4_mixed": [
        Case("g4_dense_bn64", 1, 129, 64, 320, 3, pre="stats", act="elu"),
        _poly("g4_poly_bn32_s4", 2, 40, 64, 32, 8, 4, 2, act="lrelu"),
        Case("g4_dense_span64", 1, 200, 96, 128, 5, dil=16, pad=32, pre="stats_gbb", act="snake", stats_out=True),
        _poly("g4_poly_bn128", 1, 50, 128, 256, 4, 2, 1),
    ],
}


# --------------------------------------------------------------------------------------------------------------------- reference
def _inputs(c: Case) -> dict:
    g = torch.Generator().manual_seed(zlib.crc32(c.name.encode()))

    def r(*shape, scale=1.0):
        return torch.randn(*shape, generator=g) * scale
    # per-batch offset and spread: batch rows need different statistics and coefficients
    bscale = (1 + 0.25 * torch.arange(c.B, dtype=torch.float32))[:, None, None]
    boff = (0.2 * torch.arange(c.B, dtype=torch.float32))[:, None, None]
    x = (r(c.B, c.L, c.Cin) * bscale + boff) * c.x_scale
    w = r(c.Cout, c.K, c.Cin, scale=0.5 / (c.Cin * c.taps) ** 0.5)
    if c.wkind == "bf16":
        w = w.to(torch.bfloat16).float()
    elif c.wkind == "fp16":
        w = w.half().float()
    lo, hi = c.a_range
    a = lo + (hi - lo) * torch.rand(c.Cin, generator=g)
    nres = -(-c.Lout // c.res_div)
    return dict(x=x, xa=[r(c.B, c.L, c.Cin, scale=c.x_scale) for _ in range(c.nadd)], w=w, bias=r(c.Cout, scale=0.3), a=a, b=1.0 / a,
                scale=1 + 0.3 * r(c.B, c.Cin), shift=0.2 * r(c.B, c.Cin), gb=0.3 * r(c.B if c.pre != "stats_gbb" else 1, 2 * c.Cin),
                cscale=1 + 0.5 * r(c.B if c.cscale == "bc" else 1, c.Cout), res=r(c.B if c.res == "full" else 1, nres, c.Cout, scale=0.5),
                y0=r(c.B, c.Lout, c.Cout))


def _reference(c: Case, t: dict, stats_val: Optional[torch.Tensor]) -> torch.Tensor:
    """float64: prologue -> conv (scatter + crop) -> epilogue.  stats_val: float64 [B, Cin, 2] of the statistics the kernel reads."""
    v = t["x"].double()
    for xa in t["xa"]:
        v = v + xa.double()
    v = v * c.in_scale
    if c.pre == "scale":
        v = v * t["scale"].double()[:, None] + t["shift"].double()[:, None]
    elif c.pre:
        mean = stats_val[..., 0] / c.L
        var = (stats_val[..., 1] / c.L - mean ** 2).clamp(min=0)
        s, be = 1.0 / torch.sqrt(var + EPS), torch.zeros_like(mean)
        if c.pre != "stats":
            gb = t["gb"].double()
            s, be = s * (1 + gb[:, :c.Cin]), be + gb[:, c.Cin:]
        v = v * s[:, None] + (be - s * mean)[:, None]
    if c.act:
        v = _act_ref(c.act, v, PRE_P0, t["a"].double(), t["b"].double())
    w = t["w"].double()
    if c.transpose:
        full = ON.conv_transpose1d(v, w, c.stride, 0, 1, 0, 1)
        y = torch.zeros(c.B, c.Lout, c.Cout, dtype=torch.float64)
        n = max(0, min(c.Lout, full.shape[1] - c.padl))
        y[:, :n] = full[:, c.padl:c.padl + n]
    else:
        right = max(0, c.Lout + c.span - c.padl - c.L)
        xp = F.pad(v.transpose(1, 2), (c.padl, right)).transpose(1, 2)
        y = ON.conv1d(xp, w, 1, 0, c.dil, 1)[:, :c.Lout]
    if c.bias:
        y = y + t["bias"].double()
    if c.post:
        y = _act_ref(c.post, y, POST_P0)
    if c.cscale:
        y = y * t["cscale"].double()[:, None, :]
    if c.res:
        y = y + t["res"].double()[:, torch.arange(c.Lout) // c.res_div]
    y = y * c.out_scale
    if c.accumulate:
        y = y + t["y0"].double()
    return y


def rel_err(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _tol(c: Case):
    return TOL_X2 if c.mode == "x2" else TOL_X1[c.wkind]


def _guarded(B, rows, cols, off, nan_rows=GUARD):
    """A NaN-filled [B, rows + 2 nan_rows, width] buffer (width a multiple of 4, >= 3 NaN channels past the slice) and the view
    [:, nan_rows : nan_rows + rows, off : off + cols] of it."""
    width = -(-(off + cols + 3) // 4) * 4
    buf = torch.full((B, rows + 2 * nan_rows, width), float("nan"), device=DEV)
    return buf, buf[:, nan_rows:nan_rows + rows, off:off + cols]


def _outside_is_nan(buf, view_rows, off, cols, nan_rows=GUARD):
    inside = torch.zeros(buf.shape, dtype=torch.bool)
    inside[:, nan_rows:nan_rows + view_rows, off:off + cols] = True
    return bool(buf.cpu()[~inside].isnan().all())


class Prob:
    """One case's device tensors, its FusedProblem and (once computed) its float64 reference."""

    def __init__(self, ops, c: Case):
        self.c, t = c, _inputs(c)
        self.t = t

        def xin(src):
            if c.x_off is None:
                return src.to(DEV).contiguous()
            _, v = _guarded(c.B, c.L, c.Cin, c.x_off, nan_rows=1)
            return v.copy_(src)
        x, xa = xin(t["x"]), [xin(s) for s in t["xa"]]
        cw = ops.pack_conv(t["w"], t["bias"] if c.bias else None, 1, DEV)
        assert cw.w_tc is not None and cw.f16 == (c.wkind == "fp16") and (cw.w_tc_lo is not None) == (c.wkind == "fp32")
        a, b = (t["a"].to(DEV), t["b"].to(DEV)) if c.act == "snake" else (None, None)
        actv = ACT[c.act] if c.act else 0
        pre, self.stats_val = None, None
        if c.pre == "scale":
            pre = ops.Pre(t["scale"].to(DEV), t["shift"].to(DEV), actv, PRE_P0, a, b)
        elif c.pre:
            st = ops.new_stats(c.B, c.Cin, DEV)
            ops.channel_stats(t["x"].to(DEV), [st])                   # InstanceNorm statistics of x, per batch row
            self.stats_val = ops.stats_value(st).cpu()
            pre = ops.PreStats(st, None if c.pre == "stats" else t["gb"].to(DEV), EPS, actv, PRE_P0, a, b)
        elif c.act:
            pre = ops.Pre(act=actv, p0=PRE_P0, a=a, b=b)
        cscale = None
        if c.cscale:
            cscale = t["cscale"].to(DEV).reshape(-1) if c.cscale == "c" else t["cscale"].to(DEV)
        res = None
        if c.res:                                                    # the rows the layer may read, then NaN rows
            rbuf = torch.full((t["res"].shape[0], t["res"].shape[1] + GUARD, c.Cout), float("nan"), device=DEV)
            rbuf[:, :t["res"].shape[1]] = t["res"].to(DEV)
            res = rbuf[:, :t["res"].shape[1]]
        self.ybuf, self.y = _guarded(c.B, c.Lout, c.Cout, c.y_off)
        if c.accumulate:
            self.y.copy_(t["y0"])
        self.st = ops.new_stats(c.B, c.Cout, DEV) if c.stats_out else None
        self.fp = ops.FusedProblem(x, cw, stride=c.stride, dilation=c.dil, pad_left=c.padl, lout=c.Lout, pre=pre, x_add=xa,
                                   in_scale=c.in_scale, post_act=ACT[c.post] if c.post else 0, post_p0=POST_P0, cscale=cscale, res=res,
                                   res_div=c.res_div, out_scale=c.out_scale, out=self.y, accumulate=c.accumulate,
                                   transpose=c.transpose, stats_out=self.st)

    def check(self, tol=None):
        c = self.c
        assert _outside_is_nan(self.ybuf, c.Lout, c.y_off, c.Cout), f"{c.name}: write outside the output's rows / channels"
        ref = _reference(c, self.t, self.stats_val)
        e = rel_err(self.y, ref)
        assert e <= (tol or _tol(c)), (c.name, e)
        if self.st is not None:
            from mlx_audio_b200 import ops
            yd = self.y.double().cpu()
            want = torch.stack([yd.sum(dim=1), (yd ** 2).sum(dim=1)], dim=-1)
            es = rel_err(ops.stats_value(self.st), want)
            assert es <= STATS_TOL, (c.name, "statistics", es)
        return e


def _launch(ops, probs):
    ops.conv_fused([p.fp for p in probs])
    torch.cuda.synchronize()


def _assert_plan(ops, cases, ws_bytes=None):
    from mlx_audio_b200 import ops as _ops
    plan = _plan(cases, _nsm(), _ops.FUSED_WS_BYTES if ws_bytes is None else ws_bytes)
    cfg = ops.conv1d_fused_last_config()
    assert cfg == {"grid": plan.grid, "BN": plan.BN, "ksplit": plan.ksplit}, (cfg, plan)
    return plan


@pytest.fixture
def ops():
    """The fused kernel with the case's activation planes; the module's switches restored afterwards."""
    from mlx_audio_b200 import ops as _ops
    old = _ops.TC_MODE[0], _ops.FUSED[0], _ops.FUSED_DISPATCH[0]
    _ops.FUSED[0], _ops.FUSED_DISPATCH[0] = True, False
    yield _ops
    _ops.TC_MODE[0], _ops.FUSED[0], _ops.FUSED_DISPATCH[0] = old


def _run_case(ops, c: Case, repeat=False):
    ops.TC_MODE[0] = c.mode
    p = Prob(ops, c)
    _launch(ops, [p])
    plan = _assert_plan(ops, [c])
    p.check()
    if repeat or c.stats_out:                                        # the same launch again: the same bits, output and statistics
        q = Prob(ops, c)
        _launch(ops, [q])
        assert torch.equal(q.ybuf.nan_to_num(7.0), p.ybuf.nan_to_num(7.0)), c.name
        if p.st is not None:
            assert torch.equal(q.st, p.st), c.name
    return p, plan


@pytest.mark.parametrize("case", BRANCH_CASES, ids=lambda c: c.name)
def test_branch_vs_float64(case, ops):
    _run_case(ops, case)


@pytest.mark.parametrize("case", GEOMETRY_CASES, ids=lambda c: c.name)
def test_geometry_vs_float64(case, ops):
    _, plan = _run_case(ops, case)
    if case.name.startswith("waves"):
        assert plan.tiles >= 2 * _nsm(), plan                        # every CTA meets tiles of more than one batch row


def _consumer_check(ops, p: Prob):
    """The written output's statistics feed an InstanceNorm prologue (PreStats without gamma|beta) of a 1x1 consumer."""
    c = p.c
    w = (torch.randn(32, 1, c.Cout, generator=torch.Generator().manual_seed(5)) / c.Cout ** 0.5).to(torch.bfloat16).float()
    cw = ops.pack_conv(w, None, 1, DEV)
    z = ops.conv_fused(ops.FusedProblem(p.y, cw, pre=ops.PreStats(p.st, None, EPS)))[0]
    yd = p.y.double().cpu()
    mean, var = yd.mean(dim=1, keepdim=True), yd.var(dim=1, unbiased=False, keepdim=True)
    ref = ON.conv1d((yd - mean) / torch.sqrt(var + EPS), w.double())
    assert rel_err(z, ref) < 5e-5, (c.name, rel_err(z, ref))


@pytest.mark.parametrize("case", EPILOGUE_CASES, ids=lambda c: c.name)
def test_epilogue_vs_float64(case, ops):
    p, _ = _run_case(ops, case)
    _consumer_check(ops, p)


def test_every_branch_has_a_case():
    """Every branch key the host code can reach is taken by some single-problem case, and every case's key is listed.  Each case
    asserts the tiling it got, so together with them this fails when a dispatch change leaves a branch without a test."""
    nsm = _nsm()
    seen = set()
    for c in BRANCH_CASES + GEOMETRY_CASES + EPILOGUE_CASES:
        seen |= _keys(c, _plan([c], nsm, 16 << 20))
    for c, ks in FALLBACK_CASES:
        plan = _plan(c, nsm, ks)
        for i, ci in enumerate(c):
            seen |= _keys(ci, plan, i)
    assert not BRANCHES - seen, sorted(BRANCHES - seen)
    assert not seen - BRANCHES, sorted(seen - BRANCHES)
    names = [c.name for c in BRANCH_CASES + GEOMETRY_CASES + EPILOGUE_CASES + [p for g in GROUPS.values() for p in g]]
    assert len(names) == len(set(names))


# ------------------------------------------------------------------------------------------------------------------------------ groups
@pytest.mark.parametrize("group", list(GROUPS), ids=str)
def test_group_vs_float64_and_alone(group, ops):
    """Each problem of a grouped launch against float64; bit-identical to the same problem launched alone whenever both launches give
    it the same K split; last_config lists each problem's BN and K split in caller order."""
    cases = GROUPS[group]
    ops.TC_MODE[0] = "x2"
    probs = [Prob(ops, c) for c in cases]
    _launch(ops, probs)
    plan = _assert_plan(ops, cases)
    order = sorted(range(len(cases)), key=lambda i: -cases[i].taps * cases[i].cin_pad)
    assert order != list(range(len(cases))) or len(set(c.taps * c.cin_pad for c in cases)) == 1, "caller order is already heaviest-first"
    for p in probs:
        p.check()
    compared = 0
    for i, c in enumerate(cases):
        alone = Prob(ops, c)
        _launch(ops, [alone])
        solo = _assert_plan(ops, [c])
        if (solo.ksplit[0], solo.kper[0]) == (plan.ksplit[i], plan.kper[i]):
            assert torch.equal(alone.ybuf.nan_to_num(7.0), probs[i].ybuf.nan_to_num(7.0)), c.name
            if alone.st is not None:
                assert torch.equal(alone.st, probs[i].st), c.name
            compared += 1
    assert compared >= 1


# ------------------------------------------------------------------------------------------------------------------- split-K fallback
_FB_A = [Case("fb_shortcut_k1", 1, 200, 512, 128, 1, pre="stats", stats_out=True), Case("fb_conv_k3", 1, 200, 512, 128, 3, act="lrelu")]
_FB_B = [Case("fb_single_3_tiles", 1, 300, 512, 128, 3, stats_out=True)]
FB_WS = 4096 + 3 * 4 * TM * 128 * 4          # the 3-tile problem's partial tiles at K split 4; the pair needs twice 2 tiles x 4
FALLBACK_CASES = [(_FB_A, FB_WS), (_FB_B, FB_WS)]


@pytest.fixture
def small_ws(ops):
    """Replace this stream's split-K workspace with a zeroed FB_WS-byte buffer for the test; the original is restored afterwards."""
    key = (torch.empty(0, device=DEV).device, torch.cuda.current_stream().cuda_stream)
    old = ops._FUSED_WS.get(key)
    ops._FUSED_WS[key] = torch.zeros(FB_WS, device=DEV, dtype=torch.uint8)
    yield ops
    if old is None:
        del ops._FUSED_WS[key]
    else:
        ops._FUSED_WS[key] = old


def test_split_k_workspace_fallback_and_rearm(small_ws):
    """The heaviest problem of the pair takes the small workspace, the other finds it full and runs unsplit; a launch with another tile
    count reuses the same counters.  Alternating the two launches checks that the arrival counters re-arm after every tile."""
    ops = small_ws
    ops.TC_MODE[0] = "x2"
    plans = [_plan(c, _nsm(), FB_WS) for c, _ in FALLBACK_CASES]
    assert plans[0].fallback == [True, False] and plans[0].ksplit[1] > 1 and plans[1].ksplit[0] > 1, plans
    first = {}
    for it in range(3):
        for k, (cases, _) in enumerate(FALLBACK_CASES):
            probs = [Prob(ops, c) for c in cases]
            _launch(ops, probs)
            _assert_plan(ops, cases, FB_WS)
            for p in probs:
                if it == 0:
                    p.check()
                    first[p.c.name] = p
                else:
                    assert torch.equal(p.ybuf.nan_to_num(7.0), first[p.c.name].ybuf.nan_to_num(7.0)), (it, p.c.name)
                    if p.st is not None:
                        assert torch.equal(p.st, first[p.c.name].st), (it, p.c.name)


# --------------------------------------------------------------------------------------------------------------- per-process switches
# B2A_PDL is read once per process, so it runs in a child process that writes its results to a file.
_PDL_CHAIN = Case("pdl_chain", 1, 300, 256, 256, 3)


def _pdl_chain() -> dict:
    """A dependent chain of split-K launches (6 output tiles, 4 K chunks)."""
    from mlx_audio_b200 import ops
    ops.TC_MODE[0] = "x2"
    out = {}
    t = _inputs(_PDL_CHAIN)
    cw = ops.pack_conv(t["w"], t["bias"], 1, DEV)
    y = t["x"].to(DEV)
    for _ in range(8):
        y = ops.conv_fused(ops.FusedProblem(y, cw, pad_left=1, post_act=ACT["tanh"]))[0]
    out["ksplit"] = np.array(ops.conv1d_fused_last_config()["ksplit"])
    torch.cuda.synchronize()
    out["y"] = y.cpu().numpy()
    return out


def _switch_child(path: str):
    np.savez(path, **_pdl_chain())


def _run_child(env, tmp_path):
    path = str(tmp_path / "pdl.npz")
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
            f"import test_conv_fused_matrix_gpu as m\nm._switch_child({path!r})\n")
    subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), check=True, timeout=600)
    return dict(np.load(path))


def test_pdl_switch_off_identical(ops, tmp_path):
    """B2A_PDL=0: a dependent chain launched without programmatic dependent launch gives the same bits."""
    default = _pdl_chain()
    child = _run_child({"B2A_PDL": "0"}, tmp_path)
    assert default["ksplit"][0] > 1 and np.isfinite(default["y"]).all()
    assert np.array_equal(child["y"], default["y"])


# ----------------------------------------------------------------------------------------------------------------------------- routing
def _marker(ops):
    """A two-problem launch whose record a later single-problem fused launch replaces."""
    x = torch.randn(1, 64, 64, device=DEV)
    cw = ops.pack_conv(torch.randn(32, 1, 64).to(torch.bfloat16).float(), None, 1, DEV)
    ops.conv_fused([ops.FusedProblem(x, cw), ops.FusedProblem(x, cw)])
    assert len(ops.conv1d_fused_last_config()["BN"]) == 2


# (case, runs on the fused kernel): the eligibility edges of ops.fused_eligible
ROUTES = [
    (Case("route_span64", 1, 200, 64, 128, 5, dil=16, pad=32), True),
    (Case("route_span65", 1, 200, 64, 128, 2, dil=65, pad=32, lout=200), False),
    (Case("route_cin_k_32", 1, 200, 8, 64, 4, pad=1, lout=200, x_off=None), True),
    (Case("route_x1", 1, 200, 160, 128, 3, mode="x1"), True),
    (Case("route_fp32_span54_bn128", 1, 200, 128, 128, 7, dil=9, wkind="fp32"), False),     # two weight stages do not fit
    (Case("route_fp32_span54_bn96", 1, 200, 128, 96, 7, dil=9, wkind="fp32"), True),
    (Case("route_fp32_span24_bn128", 1, 200, 128, 128, 3, dil=12, wkind="fp32"), True),
    (Case("route_fp32_span25_bn128", 1, 200, 128, 128, 2, dil=25, pad=12, lout=200, wkind="fp32"), False),
    (Case("route_fp32_span54_bn128_x1", 1, 200, 128, 128, 7, dil=9, wkind="fp32", mode="x1"), True),
]


@pytest.mark.parametrize("case,fused", ROUTES, ids=lambda v: v.name if isinstance(v, Case) else str(v))
def test_dispatch_routing_at_eligibility_edges(case, fused, ops):
    """ops.conv1d under fused_dispatch(): each layer runs (on the fused kernel when fused_eligible says so, else on the split-plane
    GEMM) and matches float64."""
    c = case
    ops.TC_MODE[0] = c.mode
    p = Prob(ops, c)
    x = p.fp.keep[0]
    cw = p.fp.keep[2]
    assert ops.fused_eligible(x, cw, 1, c.dil) == fused
    _marker(ops)
    with ops.fused_dispatch(True):
        out = ops.conv1d(x, cw, dilation=c.dil, pad_left=c.padl, lout=c.Lout, out=p.y)
    torch.cuda.synchronize()
    assert out.data_ptr() == p.y.data_ptr()
    assert (len(ops.conv1d_fused_last_config()["BN"]) == 1) == fused
    p.check()


@pytest.mark.parametrize("span,K,dil", [(24, 3, 12), (25, 2, 25), (54, 7, 9), (64, 5, 16)])
def test_fused_eligible_agrees_with_the_launch(span, K, dil, ops):
    """For split (fp32) and single-plane weights, both activation modes and BN 128 / 96: fused_eligible is true exactly when the
    launch finds room for two weight stages, and a launch it refuses writes nothing."""
    for mode in ("x2", "x1"):
        for wkind in ("fp32", "bf16"):
            for cout in (128, 96):
                c = Case(f"fits_{span}_{mode}_{wkind}_{cout}", 1, 100, 64, cout, K, dil=dil, pad=0, lout=100, wkind=wkind, mode=mode)
                ops.TC_MODE[0] = mode
                p = Prob(ops, c)
                eligible = ops.fused_eligible(p.fp.keep[0], p.fp.keep[2], 1, dil)
                try:
                    _launch(ops, [p])
                    ran = True
                except NotImplementedError as e:
                    assert "weight stages" in str(e), e
                    ran = False
                assert ran == eligible, (c.name, ran, eligible)
                if ran:
                    p.check()
                else:
                    assert bool(p.ybuf.isnan().all())


def test_dac_decode_under_fused_dispatch():
    """A DAC decoder at half width (768: its first block's residual units are 384-channel k = 7 convs at dilation 9 with split fp32
    weights) decodes under fused_dispatch(True) as on the default route, within test_dac_gpu.py's tolerance."""
    from mlx_audio_b200 import ops, synth
    from mlx_audio_b200.codec import DAC
    from oracle import dac as OD
    cfg = dict(OD.DAC_44K, encoder_dim=16, decoder_dim=768)
    model = DAC(**cfg, device=DEV).load_weights(synth.dac_weights(cfg, encoder=False))
    codes = torch.randint(0, cfg["codebook_size"], (1, cfg["n_codebooks"], 13), generator=torch.Generator().manual_seed(3))
    zq = model.quantizer.from_codes(codes)[0]
    y0 = model.decode(zq)
    with ops.fused_dispatch(True):
        y1 = model.decode(zq)
    torch.cuda.synchronize()
    a, b = y1.double().cpu().reshape(-1), y0.double().cpu().reshape(-1)
    e = float(torch.sqrt(((a - b) ** 2).mean()) / torch.sqrt((b ** 2).mean()))
    assert e < 2e-3, e


# -------------------------------------------------------------------------------------- polyphase rows past the GEMM rows (lout > scatter)
# (L, K, stride, crop, extra rows past the full scatter length minus the crop)
PAST_ROWS = [(40, 4, 2, 0, 3), (40, 4, 2, 1, 3), (33, 8, 4, 2, 9)]


@pytest.mark.parametrize("L,K,stride,crop,extra", PAST_ROWS)
@pytest.mark.parametrize("path", ["gemm_tc", "fused"])
def test_polyphase_rows_past_the_scatter(path, L, K, stride, crop, extra, ops):
    """lout past the last row any tap reaches (output_padding > crop): those rows hold the epilogue alone (bias, activation, residual),
    the rule of the CUDA-core kernel and of test_conv_cuda_core_matrix_gpu.py's reference."""
    lout = (L - 1) * stride + K - 2 * crop + extra
    c = _poly(f"past_{path}_{L}_{K}_{stride}_{crop}", 2, L, 64, 64 if stride == 2 else 32, K, stride, crop, lout=lout, post="gelu",
              res="full", out_scale=0.5, stats_out=path == "fused", act="lrelu")
    ops.TC_MODE[0] = "x2"
    p = Prob(ops, c)
    if path == "fused":
        _launch(ops, [p])
        _assert_plan(ops, [c])
    else:
        ops.FUSED[0] = False
        x, cw = p.fp.keep[0], p.fp.keep[2]
        t = p.t
        res = torch.full((c.B, lout + GUARD, c.Cout), float("nan"), device=DEV)
        res[:, :lout] = t["res"].to(DEV)
        ops.conv1d(x, cw, stride=stride, pad_left=crop, lout=lout, transpose=True, pre=ops.Pre(act=ACT["lrelu"], p0=PRE_P0),
                   post_act=ACT["gelu"], post_p0=POST_P0, res=res[:, :lout], out_scale=0.5, out=p.y)
        torch.cuda.synchronize()
        cfg = ops.conv1d_tc_last_config()
        assert cfg["grid"] == (-(-c.mrows // TM), c.N // cfg["BN"], c.B), cfg
    p.check()


# ------------------------------------------------------------------------------------------------------------ host argument errors
def test_host_argument_errors(ops):
    """Taps spanning 65 rows are refused with a clean error before anything launches; so are five problems."""
    ops.TC_MODE[0] = "x2"
    _marker(ops)
    before = ops.conv1d_fused_last_config()
    c = Case("span65_refused", 1, 200, 64, 128, 2, dil=65, pad=0, lout=200)
    p = Prob(ops, c)
    assert not ops.fused_eligible(p.fp.keep[0], p.fp.keep[2], 1, 65)
    with pytest.raises(NotImplementedError, match="span 65"):
        ops.conv_fused(p.fp)
    torch.cuda.synchronize()
    assert ops.conv1d_fused_last_config() == before
    assert bool(p.ybuf.isnan().all())
    q = Prob(ops, Case("five_problems", 1, 64, 64, 32, 1))
    with pytest.raises(ValueError, match="1..4"):
        ops.conv_fused([q.fp] * 5)
    assert ops.conv1d_fused_last_config() == before
