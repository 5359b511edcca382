"""CUDA-core conv family (csrc/conv.cu: b2a_conv1d_cl, b2a_convtr1d_cl) against float64, one dispatch branch at a time.

Each entry point picks one of about thirty kernel instantiations from shape, stride, alignment, activation and shared-memory
predicates.  Every case below runs through ops.conv1d with the tensor cores and the fused kernel switched off, asserts which
instantiation ran (ops.conv1d_cl_last_path) and compares the result with a float64 CPU reference: oracle/nn.py's conv1d /
conv_transpose1d, the prologue (scale/shift, then LReLU / Snake / ELU / GELU) and the epilogue in the order of epilogue_store
(bias, post_act, cscale, res[l / res_div], out_scale, accumulate).  Errors are max |y - ref| / max |ref| <= 2e-5, as in test_ops_gpu.py.

The input is a channel slice of a wider buffer whose other channels and rows are NaN, and the output a channel slice of a wider
NaN-filled buffer with guard rows above and below; residuals carry NaN rows past the ones the layer may read.  So a read outside the
layer's span poisons the result, and a write past Lout or Cout shows up as a lost NaN.

Lengths sit at the kernels' tile edges (BM = 64 dense rows, DW_TL = 128 staged depthwise rows, NW_TL = 256 narrow-head rows,
TRDW_ROWS = 16 transposed depthwise rows): one tile minus one row (which falls to the next kernel in line), one tile, one tile plus
one, and several tiles with a ragged tail."""
import ctypes as C
import dataclasses
import zlib
from typing import Optional

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import nn as ON

TOL = 2e-5
DEV = "cuda:0"
PRE_P0, POST_P0 = 0.15, 0.2
LRELU, SNAKE, ELU = 1, 2, 3          # B2A_ACT_* (include/b200audio.h)
GUARD = 2                            # NaN rows above and below the output, per batch row

# Every instantiation the two dispatchers can launch, as ops.conv1d_cl_last_path reports it: (kernel, v1, v2, v3).
BRANCHES = {
    ("linear_rows", 0, 0, 0),
    *[("narrow", act, 0, v4) for act in (-1, 0, LRELU, SNAKE, ELU) for v4 in (0, 1)],        # prologue ACT, vector staging
    *[("dense", bn, ci, 0) for bn in (64, 16) for ci in (32, 16, 8)],                         # BN, CI
    *[("dw_tiled4", cw, kt, snake) for kt, snake in ((7, 1), (7, 0), (0, 0)) for cw in (128, 64)],   # CW, KT, SNAKE
    ("dw_tiled", 7, 0, 0), ("dw_tiled", 0, 0, 0),                                             # KT
    ("dw", 0, 0, 0),
    ("convtr_dense", 64, 16, 0), ("convtr_dense", 64, 8, 0),                                  # BN, CI
    ("convtr_dw", 0, 0, 0),
}

POST_REF = {"gelu": ON.gelu, "tanh": torch.tanh, "silu": F.silu, "clip1": lambda v: v.clamp(-1.0, 1.0),
            "lrelu": lambda v: ON.leaky_relu(v, POST_P0)}


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    path: tuple                      # the instantiation the dispatcher must pick
    B: int
    L: int
    Cin: int
    Cout: int
    K: int
    lout: Optional[int] = None       # default: L for stride-1 convs, else ops.conv1d's formula
    stride: int = 1
    dil: int = 1
    pad: Optional[int] = None        # default: (K - 1) * dil // 2; transposed: 0 (left crop)
    dw: bool = False
    transpose: bool = False
    pad_mode: int = 0
    pre: Optional[str] = None        # "snake", "snake_a" (no b: b = 1), "lrelu", "elu", "gelu", "scale", "scale+<act>"
    bias: bool = True
    post: Optional[str] = None
    cscale: Optional[str] = None     # "c": [Cout]; "bc": [B, Cout]
    res: Optional[str] = None        # "full": [B, ., Cout]; "bcast": [1, ., Cout]
    res_div: int = 1
    out_scale: float = 1.0
    accumulate: bool = False
    x_off: Optional[int] = 4         # channel offset of x in its NaN-guarded buffer; None: a contiguous tensor
    y_off: int = 4                   # channel offset of y in its NaN-guarded buffer (4: 16-byte aligned)

    @property
    def padl(self):
        if self.pad is not None:
            return self.pad
        return 0 if self.transpose else (self.K - 1) * self.dil // 2

    @property
    def Lout(self):
        if self.lout is not None:
            return self.lout
        if self.transpose:
            return (self.L - 1) * self.stride + self.K - 2 * self.padl
        if self.stride == 1:
            return self.L
        return (self.L + 2 * self.padl - self.dil * (self.K - 1) - 1) // self.stride + 1


def _dw(name, path, B, L, C, K, **kw):
    return Case(name, path, B, L, C, C, K, dw=True, **kw)


BRANCH_CASES = [
    # ---- linear_rows: K = 1, B*L <= 8 rows, Cout >= 256, rows * Cin * 4 <= 48 KB, no prologue / cscale / res / accumulate
    Case("lr_one_row", ("linear_rows", 0, 0, 0), 1, 1, 96, 300, 1, x_off=None),
    Case("lr_8_rows", ("linear_rows", 0, 0, 0), 2, 4, 64, 257, 1, post="gelu", out_scale=0.5),
    Case("lr_9_rows", ("dense", 64, 32, 0), 3, 3, 64, 257, 1, post="gelu", out_scale=0.5),
    Case("lr_cout_256", ("linear_rows", 0, 0, 0), 1, 2, 40, 256, 1, post="tanh"),
    Case("lr_cout_255", ("dense", 64, 32, 0), 1, 2, 40, 255, 1, post="tanh"),
    Case("lr_smem_48k", ("linear_rows", 0, 0, 0), 2, 4, 1536, 256, 1, out_scale=0.5),
    Case("lr_smem_over_48k", ("dense", 64, 32, 0), 2, 4, 1537, 256, 1, out_scale=0.5),
    # ---- narrow heads: stride 1, Cout <= 4, Lout >= 256; ACT specialised unless pre_scale or another activation; v4 staging
    Case("nw_snake_v4_one_tile", ("narrow", SNAKE, 0, 1), 3, 256, 64, 1, 7, pad=6, pre="snake"),
    Case("nw_snake_scalar_cin33", ("narrow", SNAKE, 0, 0), 1, 257, 33, 2, 7, pad=6, pre="snake"),
    Case("nw_none_v4_edge_pad", ("narrow", 0, 0, 1), 2, 773, 64, 3, 5, pad=4, pad_mode=1, post="clip1"),
    Case("nw_none_scalar_cin30", ("narrow", 0, 0, 0), 1, 512, 30, 4, 3, x_off=None),
    Case("nw_elu_v4_dil3", ("narrow", ELU, 0, 1), 1, 600, 96, 1, 7, dil=3, pad=18, pre="elu", post="tanh"),
    Case("nw_elu_scalar_unaligned_x", ("narrow", ELU, 0, 0), 2, 300, 48, 1, 7, pad=3, pre="elu", x_off=2),
    Case("nw_lrelu_v4_dil5", ("narrow", LRELU, 0, 1), 1, 1000, 64, 4, 7, dil=5, pad=30, pre="lrelu", x_off=None),
    Case("nw_lrelu_scalar_edge_pad", ("narrow", LRELU, 0, 0), 3, 256, 21, 2, 3, pad=2, pad_mode=1, pre="lrelu"),
    Case("nw_scale_snake_generic_v4", ("narrow", -1, 0, 1), 2, 400, 64, 1, 7, pad=6, pre="scale+snake"),
    Case("nw_gelu_generic_scalar", ("narrow", -1, 0, 0), 1, 257, 35, 2, 5, pad=4, pre="gelu"),
    Case("nw_scale_only_edge_pad", ("narrow", -1, 0, 1), 1, 300, 64, 1, 7, pad=6, pad_mode=1, pre="scale"),
    Case("nw_snake_without_b", ("narrow", -1, 0, 1), 1, 300, 40, 1, 7, pad=6, pre="snake_a"),
    Case("nw_lout_255", ("dense", 16, 16, 0), 1, 255, 64, 1, 7, pad=6, pre="snake"),
    Case("nw_halo_over_160k", ("dense", 16, 16, 0), 1, 300, 256, 1, 7, dil=20, pad=120, pre="snake"),
    # ---- dense implicit GEMM: CI = 32 / 16 / 8 for K <= 4 / <= 12 / more; BN = 64 unless Cout <= 16
    Case("d64_ci32_lout63", ("dense", 64, 32, 0), 1, 63, 40, 70, 3),
    Case("d64_ci32_lout64", ("dense", 64, 32, 0), 3, 64, 33, 65, 3, pre="lrelu", x_off=None),
    Case("d64_ci32_lout65_edge_pad", ("dense", 64, 32, 0), 1, 65, 48, 100, 4, pad=2, pad_mode=1),
    Case("d64_ci32_cout17", ("dense", 64, 32, 0), 2, 100, 24, 17, 3),
    Case("d64_ci16_ragged_dil3", ("dense", 64, 16, 0), 3, 209, 50, 100, 7, dil=3, pre="scale+lrelu"),
    Case("d64_ci16_s3_edge_pad", ("dense", 64, 16, 0), 2, 190, 40, 32, 6, stride=3, pad=3, pad_mode=1),
    Case("d64_ci8_s8_downsampler", ("dense", 64, 8, 0), 3, 1000, 24, 48, 16, stride=8, pad=4),
    Case("d64_ci8_dil4", ("dense", 64, 8, 0), 1, 200, 20, 33, 20, dil=4, pad=38, pre="elu"),
    Case("d16_ci32_s2", ("dense", 16, 32, 0), 1, 150, 20, 13, 3, stride=2, pad=1, x_off=None),
    Case("d16_ci16_cout16", ("dense", 16, 16, 0), 3, 100, 17, 16, 9, pre="elu", post="gelu"),
    Case("d16_ci8", ("dense", 16, 8, 0), 1, 255, 64, 3, 13, pad=12),
    # ---- staged depthwise, vectorised: stride 1, K <= 16, Lout >= 128, C % 4 == 0, aligned x / w / bias, (128 + halo) * 512 B <= 160 KB
    _dw("t4_k7_cw128_snake_one_tile", ("dw_tiled4", 128, 7, 1), 3, 128, 132, 7, dil=3, pre="snake"),
    _dw("t4_k7_cw64_snake_dil9", ("dw_tiled4", 64, 7, 1), 1, 129, 64, 7, dil=9, pre="snake"),
    _dw("t4_k7_cw128_convnext", ("dw_tiled4", 128, 7, 0), 1, 255, 256, 7, x_off=None),
    _dw("t4_k7_cw64_lrelu_edge_pad", ("dw_tiled4", 64, 7, 0), 2, 300, 68, 7, pre="lrelu", pad_mode=1),
    _dw("t4_k7_scale_edge_pad", ("dw_tiled4", 128, 7, 0), 1, 260, 128, 7, pre="scale", pad_mode=1),
    _dw("t4_k7_unaligned_y", ("dw_tiled4", 64, 7, 0), 2, 200, 64, 7, y_off=1),
    _dw("t4_k5_cw128_scale_snake_ragged", ("dw_tiled4", 128, 0, 0), 1, 391, 128, 5, dil=2, pre="scale+snake"),
    _dw("t4_k16_cw64_wide_halo", ("dw_tiled4", 64, 0, 0), 1, 130, 40, 16, dil=12, pre="elu"),
    _dw("t4_k3_cw64_gelu_c96", ("dw_tiled4", 64, 0, 0), 3, 256, 96, 3, pre="gelu"),
    _dw("t4_lout127", ("dw", 0, 0, 0), 1, 127, 64, 7),
    # ---- staged depthwise, scalar: as above when the vectorised kernel is not eligible, (128 + halo) * 128 B <= 96 KB
    _dw("tl_k7_snake_one_tile", ("dw_tiled", 7, 0, 0), 3, 128, 37, 7, pre="snake"),
    _dw("tl_k7_halo_over_tiled4", ("dw_tiled", 7, 0, 0), 1, 200, 64, 7, dil=50),
    _dw("tl_k5_scale_edge_pad", ("dw_tiled", 0, 0, 0), 1, 129, 33, 5, dil=3, pre="scale", pad_mode=1),
    _dw("tl_k16_unaligned_x", ("dw_tiled", 0, 0, 0), 2, 257, 36, 16, pre="lrelu", x_off=1),
    _dw("tl_k3_dil100", ("dw_tiled", 0, 0, 0), 3, 300, 30, 3, dil=100, x_off=None),
    _dw("tl_lout127", ("dw", 0, 0, 0), 1, 127, 37, 7),
    _dw("tl_halo_over_96k", ("dw", 0, 0, 0), 1, 300, 33, 5, dil=200),
    # ---- depthwise, one thread per output: strided, K > 16, or short
    _dw("dw_s2", ("dw", 0, 0, 0), 1, 400, 33, 4, stride=2, pad=1),
    _dw("dw_k20_snake", ("dw", 0, 0, 0), 2, 300, 40, 20, pre="snake"),
    _dw("dw_s3_edge_pad", ("dw", 0, 0, 0), 1, 200, 64, 5, stride=3, pad=2, pad_mode=1),
    # ---- transposed dense (polyphase gather): CI = 16 for K <= 12, else 8; 64 x 64 tiles
    Case("ctd_ci16_lout63", ("convtr_dense", 64, 16, 0), 1, 11, 22, 40, 12, stride=6, pad=3, lout=63, transpose=True),
    Case("ctd_ci16_lout64", ("convtr_dense", 64, 16, 0), 3, 17, 32, 64, 8, stride=4, pad=2, lout=64, transpose=True, pre="lrelu"),
    Case("ctd_ci8_lout65", ("convtr_dense", 64, 8, 0), 1, 8, 96, 70, 20, stride=10, pad=5, lout=65, transpose=True),
    Case("ctd_ci8_ragged_opad", ("convtr_dense", 64, 8, 0), 3, 30, 40, 33, 16, stride=8, pad=4, lout=241, transpose=True,
         pre="lrelu"),
    Case("ctd_k7_s3_snake", ("convtr_dense", 64, 16, 0), 2, 40, 24, 24, 7, stride=3, pad=2, transpose=True, pre="snake"),
    Case("ctd_s1", ("convtr_dense", 64, 16, 0), 1, 70, 20, 20, 5, pad=2, transpose=True, x_off=None),
    # ---- transposed depthwise: 16-row x 128-channel blocks
    _dw("ctdw_lout15", ("convtr_dw", 0, 0, 0), 1, 9, 130, 4, stride=2, pad=1, lout=15, transpose=True),
    _dw("ctdw_lout16", ("convtr_dw", 0, 0, 0), 3, 9, 130, 4, stride=2, pad=1, lout=16, transpose=True),
    _dw("ctdw_lout17_snake", ("convtr_dw", 0, 0, 0), 1, 9, 64, 3, stride=2, pad=1, lout=17, transpose=True, pre="snake"),
    _dw("ctdw_ragged_opad", ("convtr_dw", 0, 0, 0), 3, 43, 37, 3, stride=2, pad=1, lout=87, transpose=True, x_off=None),
]

# Each epilogue field alone on one case per kernel, then all of them together.  The bases carry no bias and B = 3, so that the
# per-batch cscale and the batch-broadcast residual differ from their shared forms.
EPILOGUES = {
    "bare": {}, "bias": dict(bias=True), "post_act": dict(post="gelu"), "cscale": dict(cscale="c"), "cscale_per_batch": dict(cscale="bc"),
    "res": dict(res="full"), "res_bcast": dict(res="bcast"), "res_div": dict(res="full", res_div=3), "out_scale": dict(out_scale=-0.7),
    "accumulate": dict(accumulate=True),
    "all": dict(bias=True, post="silu", cscale="bc", res="bcast", res_div=2, out_scale=0.7, accumulate=True),
}
EPILOGUE_BASES = [
    Case("dense64", ("dense", 64, 16, 0), 3, 150, 24, 70, 5, dil=2, bias=False),
    Case("dense16", ("dense", 16, 32, 0), 3, 70, 20, 13, 3, stride=2, bias=False),
    Case("narrow", ("narrow", SNAKE, 0, 1), 3, 300, 32, 3, 7, pad=6, pre="snake", bias=False),
    _dw("dw_tiled4_snake", ("dw_tiled4", 128, 7, 1), 3, 300, 132, 7, pre="snake", bias=False),
    _dw("dw_tiled4_k5", ("dw_tiled4", 64, 0, 0), 3, 200, 64, 5, dil=2, bias=False),
    _dw("dw_tiled", ("dw_tiled", 0, 0, 0), 3, 200, 37, 5, bias=False),
    _dw("dw", ("dw", 0, 0, 0), 3, 100, 37, 4, stride=2, pad=1, bias=False),
    Case("convtr_dense", ("convtr_dense", 64, 16, 0), 3, 30, 24, 40, 8, stride=4, transpose=True, bias=False),
    _dw("convtr_dw", ("convtr_dw", 0, 0, 0), 3, 40, 130, 3, stride=2, pad=1, transpose=True, bias=False),
]
LINEAR_ROWS_BASE = Case("linear_rows", ("linear_rows", 0, 0, 0), 2, 3, 64, 300, 1, bias=False)
LINEAR_ROWS_EPILOGUES = {k: EPILOGUES[k] for k in ("bare", "bias", "post_act", "out_scale")}
LINEAR_ROWS_EPILOGUES["all"] = dict(bias=True, post="tanh", out_scale=0.7)     # the only fields that keep the layer on linear_rows

EPILOGUE_CASES = [dataclasses.replace(b, name=f"{b.name}-{e}", **f) for b in EPILOGUE_BASES for e, f in EPILOGUES.items()]
EPILOGUE_CASES += [dataclasses.replace(LINEAR_ROWS_BASE, name=f"linear_rows-{e}", **f) for e, f in LINEAR_ROWS_EPILOGUES.items()]
ALL_CASES = BRANCH_CASES + EPILOGUE_CASES


@pytest.fixture
def cuda_core():
    """Route every ops.conv1d call to csrc/conv.cu: no tensor-core path, no fused kernel."""
    from mlx_audio_b200 import ops
    old = ops.TC_MODE[0], ops.FUSED_DISPATCH[0]
    ops.TC_MODE[0], ops.FUSED_DISPATCH[0] = "off", False
    yield ops
    ops.TC_MODE[0], ops.FUSED_DISPATCH[0] = old


def _last_path(ops):
    r = ops.conv1d_cl_last_path()
    return (r["kernel"], *r["variant"])


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _inputs(c: Case) -> dict:
    g = torch.Generator().manual_seed(zlib.crc32(c.name.encode()))

    def r(*shape, scale=1.0):
        return torch.randn(*shape, generator=g) * scale
    a = (1 + 0.2 * r(c.Cin)).abs() + 0.1
    return dict(x=r(c.B, c.L, c.Cin), w=r(c.Cout, c.K, 1 if c.dw else c.Cin, scale=0.3 if c.dw else 0.1), bias=r(c.Cout, scale=0.5),
                a=a, b=1.0 / a, scale=1 + 0.3 * r(c.B, c.Cin), shift=0.2 * r(c.B, c.Cin),
                cscale=1 + 0.5 * r(c.B if c.cscale == "bc" else 1, c.Cout),
                res=r(c.B if c.res == "full" else 1, c.Lout + GUARD, c.Cout, scale=0.5),
                y0=r(c.B, c.Lout, c.Cout))


def _reference(c: Case, t: dict) -> torch.Tensor:
    v = t["x"].double()
    if c.pre and c.pre.startswith("scale"):
        v = v * t["scale"].double()[:, None, :] + t["shift"].double()[:, None, :]
    act = c.pre.split("+")[-1] if c.pre else None
    if act in ("snake", "snake_a"):
        v = v + (t["b"].double() if act == "snake" else 1.0) * torch.sin(t["a"].double() * v) ** 2
    elif act == "lrelu":
        v = ON.leaky_relu(v, PRE_P0)
    elif act == "elu":
        v = ON.elu(v)
    elif act == "gelu":
        v = ON.gelu(v)
    w, groups, lout = t["w"].double(), c.Cin if c.dw else 1, c.Lout
    if c.transpose:                      # scatter output, then the left crop; rows past it (output padding) get only the epilogue
        full = ON.conv_transpose1d(v, w, c.stride, 0, 1, 0, groups)
        y = torch.zeros(c.B, lout, c.Cout, dtype=torch.float64)
        n = max(0, min(lout, full.shape[1] - c.padl))
        y[:, :n] = full[:, c.padl:c.padl + n]
    else:                                # zero or edge padding of the transformed input on both sides, as far as the outputs reach
        right = max(0, (lout - 1) * c.stride + (c.K - 1) * c.dil + 1 - c.padl - c.L)
        xp = F.pad(v.transpose(1, 2), (c.padl, right), mode="replicate" if c.pad_mode else "constant").transpose(1, 2)
        y = ON.conv1d(xp, w, c.stride, 0, c.dil, groups)[:, :lout]
    if c.bias:
        y = y + t["bias"].double()
    if c.post:
        y = POST_REF[c.post](y)
    if c.cscale:
        y = y * t["cscale"].double()[:, None, :]
    if c.res:
        y = y + t["res"].double()[:, torch.arange(lout) // c.res_div]
    y = y * c.out_scale
    if c.accumulate:
        y = y + t["y0"].double()
    return y


def _guarded(B, rows, cols, off, nan_rows=GUARD):
    """A NaN-filled [B, rows + 2 * nan_rows, width] buffer (width a multiple of 4, >= 3 NaN channels past the slice) and the view
    [:, nan_rows : nan_rows + rows, off : off + cols] of it."""
    width = -(-(off + cols + 3) // 4) * 4
    buf = torch.full((B, rows + 2 * nan_rows, width), float("nan"), device=DEV)
    return buf, buf[:, nan_rows:nan_rows + rows, off:off + cols]


def _outside_is_nan(buf, view_rows, off, cols, nan_rows=GUARD):
    inside = torch.zeros(buf.shape, dtype=torch.bool)
    inside[:, nan_rows:nan_rows + view_rows, off:off + cols] = True
    return bool(buf.cpu()[~inside].isnan().all())


def _run(ops, c: Case, t: dict):
    """ops.conv1d on c's device tensors; returns (y view, its guarded buffer)."""
    if c.x_off is None:
        x = t["x"].to(DEV)
    else:
        _, x = _guarded(c.B, c.L, c.Cin, c.x_off, nan_rows=1)
        x.copy_(t["x"])
    cw = ops.pack_conv(t["w"], t["bias"] if c.bias else None, c.Cin if c.dw else 1, DEV)
    pre = None
    if c.pre:
        act = c.pre.split("+")[-1]
        sc = c.pre.startswith("scale")
        pre = ops.Pre(t["scale"].to(DEV) if sc else None, t["shift"].to(DEV) if sc else None,
                      ops.ACT["snake" if act == "snake_a" else act] if act != "scale" else 0, PRE_P0,
                      t["a"].to(DEV), t["b"].to(DEV) if act == "snake" else None)
    cscale = None
    if c.cscale:
        cscale = t["cscale"].to(DEV).reshape(-1) if c.cscale == "c" else t["cscale"].to(DEV)
    res = None
    if c.res:                           # the rows the layer may read (ceil(Lout / res_div)), then NaN rows to Lout + GUARD
        nres = -(-c.Lout // c.res_div)
        rbuf = t["res"].to(DEV)
        rbuf[:, nres:] = float("nan")
        res = rbuf[:, :nres]
    ybuf, y = _guarded(c.B, c.Lout, c.Cout, c.y_off)
    if c.accumulate:
        y.copy_(t["y0"])
    out = ops.conv1d(x, cw, stride=c.stride, dilation=c.dil, pad_left=c.padl, lout=c.Lout, pad_mode=c.pad_mode, pre=pre,
                     post_act=ops.ACT[c.post] if c.post else 0, post_p0=POST_P0, cscale=cscale, res=res, res_div=c.res_div,
                     out_scale=c.out_scale, out=y, accumulate=c.accumulate, transpose=c.transpose)
    assert out.data_ptr() == y.data_ptr()
    return y, ybuf


def _check(ops, c: Case):
    t = _inputs(c)
    ref = _reference(c, t)
    y, ybuf = _run(ops, c, t)
    path = _last_path(ops)
    assert path in BRANCHES, path
    assert path == c.path, (path, c.path)
    assert _outside_is_nan(ybuf, c.Lout, c.y_off, c.Cout), "write outside the output's rows / channels"
    e = rel_err(y, ref)
    assert e <= TOL, (c.name, path, e)


@pytest.mark.parametrize("case", BRANCH_CASES, ids=lambda c: c.name)
def test_branch_vs_float64(case, cuda_core):
    _check(cuda_core, case)


@pytest.mark.parametrize("case", EPILOGUE_CASES, ids=lambda c: c.name)
def test_epilogue_vs_float64(case, cuda_core):
    _check(cuda_core, case)


def test_every_branch_has_a_case():
    """Every instantiation in BRANCHES is the expected path of some case, and every case expects a listed one.  Each case asserts the
    path it took, so together with them this fails when a dispatch change leaves a kernel without a test."""
    expected = {c.path for c in ALL_CASES}
    assert not BRANCHES - expected, sorted(BRANCHES - expected)
    assert not expected - BRANCHES, sorted(expected - BRANCHES)
    names = [c.name for c in ALL_CASES]
    assert len(names) == len(set(names))


@pytest.mark.parametrize("C,K,pre", [(256, 7, None), (132, 7, "snake"), (64, 5, "snake")])
def test_dw_tiled4_store_paths_agree(C, K, pre, cuda_core):
    """The vectorised depthwise kernel's 16-byte store, its per-element epilogue accumulating onto zeros, and the same epilogue into
    an unaligned y give the same bytes."""
    ops = cuda_core
    c = _dw(f"tiled4_store_{C}_{K}", None, 2, 300, C, K, pre=pre, out_scale=0.5)
    t = _inputs(c)
    x = t["x"].to(DEV)
    cw = ops.pack_conv(t["w"], t["bias"], C, DEV)
    p = ops.Pre(act=ops.ACT["snake"], a=t["a"].to(DEV), b=t["b"].to(DEV)) if pre else None

    def conv(**kw):
        out = ops.conv1d(x, cw, pad_left=c.padl, lout=c.Lout, pre=p, out_scale=0.5, **kw)
        assert _last_path(ops)[:3] == ("dw_tiled4", 128 if C >= 128 else 64, 7 if K == 7 else 0)
        return out
    fast = conv()
    acc = conv(out=torch.zeros(2, c.Lout, C, device=DEV), accumulate=True)
    _, unaligned = _guarded(2, c.Lout, C, 1)
    conv(out=unaligned)
    assert torch.equal(acc, fast)
    assert torch.equal(unaligned, fast)
    assert rel_err(fast, _reference(c, t)) <= TOL


# ---------------------------------------------------------------------------------------------------------------- argument checks
def _params(ops, x, y, w, K, groups, Cout):
    p = ops.Conv1dParams()
    p.x, p.x_bs, p.x_ld = x.data_ptr(), x.stride(0), x.stride(1)
    p.B, p.L, p.Cin = x.shape
    p.w = w.data_ptr()
    p.y, p.y_bs, p.y_ld = y.data_ptr(), y.stride(0), y.stride(1)
    p.Lout, p.Cout = y.shape[1], Cout
    p.K, p.stride, p.dilation, p.groups = K, 1, 1, groups
    p.res_div, p.out_scale = 1, 1.0
    return p


def _refused(ops, fn, p, exc, match):
    """fn(p) raises exc before launching anything: the path record and the output stay as they were."""
    from mlx_audio_b200 import _lib
    before = _last_path(ops)
    with pytest.raises(exc, match=match):
        _lib.check(fn(C.byref(p), ops._stream()))
    assert _last_path(ops) == before


def test_unsupported_groups_refused(cuda_core):
    """groups other than 1 or Cin == Cout (pack_conv already refuses such weights, so the parameters are built by hand)."""
    from mlx_audio_b200 import _lib
    ops = cuda_core
    _check(ops, BRANCH_CASES[0])                        # a known record to compare against
    x = torch.randn(1, 16, 4, device=DEV)
    w = torch.randn(3, 4, 8, device=DEV)
    for fn in (_lib.lib().b2a_conv1d_cl, _lib.lib().b2a_convtr1d_cl):
        for groups, cout in ((2, 4), (4, 8), (3, 4)):
            y = torch.full((1, 16, cout), float("nan"), device=DEV)
            _refused(ops, fn, _params(ops, x, y, w, 3, groups, cout), NotImplementedError, "groups")
            assert bool(y.isnan().all())


def test_plane_emission_refused_off_depthwise(cuda_core):
    from mlx_audio_b200 import _lib
    ops = cuda_core
    _check(ops, BRANCH_CASES[0])
    x = torch.randn(1, 200, 64, device=DEV)
    w = torch.randn(7, 64, 64, device=DEV)
    y = torch.full((1, 200, 64), float("nan"), device=DEV)
    hi = torch.zeros(1, 200, 64, device=DEV, dtype=torch.bfloat16)
    p = _params(ops, x, y, w, 7, 1, 64)
    p.emit_hi, p.emit_ld, p.emit_act = hi.data_ptr(), 64, SNAKE
    _refused(ops, _lib.lib().b2a_conv1d_cl, p, NotImplementedError, "depthwise")
    _refused(ops, _lib.lib().b2a_convtr1d_cl, p, ValueError, "plane emission")
    assert bool(y.isnan().all()) and not bool(hi.float().abs().max())


def test_dense_tile_over_shared_memory_refused(cuda_core):
    """K = 16 at dilation 1500 spans 22 564 input rows per 64-row tile (812 KB staged); the transposed tile with K = 100 holds 200 KB of
    weights alone.  Both exceed the 200 KB the kernels are built for and are refused, not launched."""
    ops = cuda_core
    _check(ops, BRANCH_CASES[0])
    before = _last_path(ops)
    x = torch.randn(1, 22600, 4, device=DEV)
    cw = ops.pack_conv(torch.randn(8, 16, 4), None, 1, DEV)
    with pytest.raises(NotImplementedError, match="shared memory"):
        ops.conv1d(x, cw, dilation=1500)
    cwt = ops.pack_conv(torch.randn(8, 100, 4), None, 1, DEV)
    with pytest.raises(NotImplementedError, match="shared memory"):
        ops.conv1d(x[:, :50], cwt, transpose=True)
    assert _last_path(ops) == before
