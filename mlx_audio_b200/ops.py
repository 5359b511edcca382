"""Host-side wrappers: torch CUDA tensors -> C-ABI calls on torch's current stream.

torch is plumbing only (device memory, streams); every compute op here is one of our sm_90a
kernels.  All activations are float32 channels-last ``[B, L, C]``; tensors may be channel-slice
views of wider buffers (row stride = ``stride(1)``), which is how concatenations are avoided.
"""
from __future__ import annotations

import ctypes as C
import math
import contextlib
import os
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib
from ._lib import AttnParams, Conv1dParams, ConvFParams

ACT = {"none": 0, "lrelu": 1, "snake": 2, "elu": 3, "gelu": 4, "gelu_tanh": 5, "tanh": 6, "sigmoid": 7,
       "silu": 8, "clip1": 9}

LAUNCHES = [0]        # kernels launched through this module (bench.py reports it as gpu_launches)


PROFILE = None        # dict kind -> [(start_event, end_event)] when bench.py instruments a pass
PROFILE_TAGS = None   # dict kind -> [label] parallel to PROFILE (bench.py's per-launch table); TAG[0] is the label of the next call
TAG = [None]
PROFILE_EXTERNAL = False   # True while an instrumented CUDA graph is captured: the events become event-record NODES of the graph, so
                           # every replay re-stamps them and the per-launch times are those of the replayed graph (not of an eager pass)


def _call(kind, fn, n_launches, *args):
    """Invoke a C-ABI entry point, map its status to an exception, count its kernel launches and (when
    bench.py asks) bracket it with CUDA events on the launching stream."""
    if PROFILE is not None:
        a = torch.cuda.Event(enable_timing=True, external=PROFILE_EXTERNAL)
        b = torch.cuda.Event(enable_timing=True, external=PROFILE_EXTERNAL)
        a.record()
        rc = fn(*args)
        b.record()
        PROFILE.setdefault(kind, []).append((a, b))
        if PROFILE_TAGS is not None:
            PROFILE_TAGS.setdefault(kind, []).append(TAG[0])
        TAG[0] = None
    else:
        rc = fn(*args)
    _lib.check(rc)
    LAUNCHES[0] += n_launches


_SIDE_POOL = {}      # device -> [streams];  _SIDE_BUSY: streams handed out by fork() and not yet joined
_SIDE_BUSY = set()


def fork(device, n: int = 1):
    """Start ``n`` concurrent branches: returns side streams that wait on the current stream's present point.  Use
    ``with torch.cuda.stream(s): ...`` for each branch, then ``join(device, streams)``.  Inside a CUDA-graph capture
    the branches become parallel graph paths.  Tensors that cross branches must be allocated BEFORE the fork (on the
    joining stream); branch temporaries stay stream-local, and because every fork waits on the forking stream and every
    join waits on the branches, block reuse by the caching allocator stays ordered."""
    device = torch.device(device)
    cur = torch.cuda.current_stream(device)
    pool = _SIDE_POOL.setdefault(device, [])
    out = []
    for s in pool:
        if len(out) == n:
            break
        if s not in _SIDE_BUSY and s != cur:
            out.append(s)
    while len(out) < n:
        s = torch.cuda.Stream(device=device)
        pool.append(s)
        out.append(s)
    for s in out:
        _SIDE_BUSY.add(s)
        s.wait_stream(cur)
    return out


def join(device, streams) -> None:
    cur = torch.cuda.current_stream(torch.device(device))
    for s in streams:
        cur.wait_stream(s)
        _SIDE_BUSY.discard(s)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _chk3(x: torch.Tensor, name: str):
    if x.dtype != torch.float32 or not x.is_cuda or x.dim() != 3 or x.stride(2) != 1:
        raise ValueError(f"{name}: expected a CUDA float32 [B, L, C] tensor with unit channel stride, got "
                         f"{tuple(x.shape)} {x.dtype} {x.device} strides {x.stride()}")


@dataclass
class Pre:
    """Input transform fused into a conv: x*scale[b,c]+shift[b,c] then an activation."""
    scale: Optional[torch.Tensor] = None
    shift: Optional[torch.Tensor] = None
    act: int = 0
    p0: float = 0.0
    a: Optional[torch.Tensor] = None
    b: Optional[torch.Tensor] = None


@dataclass
class ConvW:
    """Packed conv weights: ``w`` float32 [K, Cin/groups, Cout] (depthwise: [K, C]), optional bias [Cout];
    ``w_tc`` bf16 [K, Cout, cin_pad] for the tensor-core path (dense layers only)."""
    w: torch.Tensor
    bias: Optional[torch.Tensor]
    K: int
    cin: int
    cout: int
    groups: int = 1
    w_tc: Optional[torch.Tensor] = None
    cin_pad: int = 0
    f16: bool = False          # w_tc is IEEE fp16 (fp16 checkpoints) instead of bf16
    w_tc_lo: Optional[torch.Tensor] = None   # fp32 checkpoints: w = w_tc + w_tc_lo (both bf16), kept to ~2^-17


# Tensor-core dispatch policy: "off" = CUDA-core fp32 everywhere; "x2" = wgmma with (hi, lo) bf16 activation planes
# (fp32-grade products); "x1" = wgmma with a single bf16 plane.
TC_MODE = [os.environ.get("B2A_TC", "x2")]
ATTN_MODE = [os.environ.get("B2A_ATTN", "tc")]      # "tc": wgmma flash attention for head_dim 64; "cuda": CUDA-core kernel
TC_MIN_K = 32                          # reduction length (Cin*K) below which the layer stays on the CUDA-core kernel


def _tc_eligible(cw: "ConvW", L: int, stride: int, transpose: bool, pad_mode: int, dilation: int = 1) -> bool:
    if TC_MODE[0] == "off" or cw.w_tc is None or pad_mode != 0 or cw.cout % 32 != 0 or L < 32:
        return False
    if transpose:                      # polyphase form: K = taps * stride, every phase is a `taps`-tap stride-1 conv
        return dilation == 1 and cw.K % stride == 0 and cw.cin * (cw.K // stride) >= TC_MIN_K
    return stride == 1 and cw.cin * cw.K >= TC_MIN_K


def _tc_transposed_weights(cw: "ConvW", stride: int):
    """([J, stride*Cout, cin_pad] hi, lo-or-None) with W[j, r*Cout + co, ci] = w[k = r + j*stride][ci][co] (cached per stride)."""
    cache = cw.__dict__.setdefault("_w_tc_tr", {})
    if stride not in cache:
        J = cw.K // stride
        w = cw.w.reshape(J, stride, cw.cin, cw.cout).permute(0, 1, 3, 2).reshape(J, stride * cw.cout, cw.cin)   # k = j*stride + r
        wt = torch.zeros(J, stride * cw.cout, cw.cin_pad, device=cw.w.device, dtype=cw.w_tc.dtype)
        wt[:, :, :cw.cin] = w.to(cw.w_tc.dtype)
        wl = None
        if cw.w_tc_lo is not None:
            wl = torch.zeros_like(wt)
            wl[:, :, :cw.cin] = (w - wt[:, :, :cw.cin].float()).to(wt.dtype)
        cache[stride] = (wt.contiguous(), None if wl is None else wl.contiguous())
    return cache[stride]


@dataclass
class Planes:
    """A tensor-core A operand already split by its producer: bf16 hi / lo planes [B, L, cin_pad] (what prep_bf16 would make)."""
    hi: torch.Tensor
    lo: Optional[torch.Tensor]
    C: int

    @property
    def shape(self):
        return (self.hi.shape[0], self.hi.shape[1], self.C)


def pack_conv(w_mlx: torch.Tensor, bias=None, groups=1, device="cuda") -> ConvW:
    """MLX-layout conv weight [Cout, K, Cin/g] -> packed [K, Cin/g, Cout]."""
    cout, k, cin_g = w_mlx.shape
    if groups == 1:
        w = w_mlx.permute(1, 2, 0).contiguous()
        cin = cin_g
    else:
        if not (cin_g == 1 and groups == cout):
            raise NotImplementedError("only dense or depthwise convolutions are on the hot path")
        w = w_mlx[:, :, 0].t().contiguous()              # [K, C]
        cin = cout
    cwo = ConvW(w.to(device=device, dtype=torch.float32), None if bias is None else bias.to(device=device, dtype=torch.float32).contiguous(),
                k, cin, cout, groups)
    if groups == 1 and cout % 32 == 0 and torch.device(device).type == "cuda":
        for dt in (torch.bfloat16, torch.float16):                     # 16-bit-exact weights only (bf16 / fp16 checkpoints)
            wb = w_mlx.float().to(dt)
            if torch.equal(wb.float(), w_mlx.float()):
                cpad = -(-cin // 64) * 64
                wt = torch.zeros(k, cout, cpad, dtype=dt)
                wt[:, :, :cin] = wb.permute(1, 0, 2)
                cwo.w_tc, cwo.cin_pad, cwo.f16 = wt.to(device).contiguous(), cpad, dt == torch.float16
                break
        else:                                                          # fp32 checkpoint (SNAC): split the weights as well
            cpad = -(-cin // 64) * 64
            w32 = w_mlx.float().permute(1, 0, 2)
            hi = w32.to(torch.bfloat16)
            lo = (w32 - hi.float()).to(torch.bfloat16)
            wt, wl = torch.zeros(k, cout, cpad, dtype=torch.bfloat16), torch.zeros(k, cout, cpad, dtype=torch.bfloat16)
            wt[:, :, :cin], wl[:, :, :cin] = hi, lo
            cwo.w_tc, cwo.w_tc_lo, cwo.cin_pad = wt.to(device).contiguous(), wl.to(device).contiguous(), cpad
    return cwo


def pack_linear(w: torch.Tensor, bias=None, device="cuda") -> ConvW:
    """nn.Linear weight [out, in] -> K=1 conv."""
    return pack_conv(w[:, None, :], bias, 1, device)


def conv1d(x: torch.Tensor, cw: ConvW, *, stride=1, dilation=1, pad_left=0, lout=None, pad_mode=0,
           pre: Optional[Pre] = None, post_act=0, post_p0=0.0, cscale=None, res=None, res_div=1,
           out_scale=1.0, out=None, accumulate=False, transpose=False, emit: Optional[Pre] = None):
    """b2a_conv1d_cl / b2a_convtr1d_cl.  For ``transpose`` ``pad_left`` is the left crop of the scatter output."""
    if isinstance(x, Planes):                      # operand already split by its producer (conv1d(..., emit=...)): tensor-core path only
        B, L, cin = x.shape
        if (cin != cw.cin or pre is not None or not _tc_eligible(cw, L, stride, transpose, pad_mode, dilation) or x.hi.shape[2] != cw.cin_pad
                or x.hi.dtype != (torch.float16 if cw.f16 else torch.bfloat16)):
            raise ValueError("conv1d: a Planes operand needs a tensor-core-eligible layer with matching channels, dtype and no prologue")
        if lout is None:
            lout = (L + 2 * pad_left - dilation * (cw.K - 1) - 1) // stride + 1
        return _conv1d_tc(x, cw, dilation, pad_left, lout, None, post_act, post_p0, cscale, res, res_div, out_scale, out, accumulate,
                          up_stride=stride if transpose else 0)
    _chk3(x, "conv1d x")
    B, L, cin = x.shape
    if cin != cw.cin:
        raise ValueError(f"conv1d: input has {cin} channels, weight expects {cw.cin}")
    if lout is None:
        if transpose:
            lout = (L - 1) * stride + cw.K - 2 * pad_left
        else:
            lout = (L + 2 * pad_left - dilation * (cw.K - 1) - 1) // stride + 1
    # Tiny GEMMs (a few rows: ALBERT at T = 130, decode-time prefills) are latency chains, not throughput problems: the fused kernel's
    # converter -> MMA -> split-K fix-up chain measured 30-40 us per launch there against ~14 us for the pre-split planes + TMA pipeline.
    small_gemm = cw.K == 1 and B * L <= 256 and _tc_eligible(cw, L, stride, transpose, pad_mode, dilation)
    if FUSED_DISPATCH[0] and emit is None and not small_gemm and fused_eligible(x, cw, stride, dilation, transpose, pad_mode, out, res):
        y = conv_fused(FusedProblem(x, cw, stride=stride, dilation=dilation, pad_left=pad_left, lout=lout, pre=pre, post_act=post_act,
                                    post_p0=post_p0, cscale=cscale, res=res, res_div=res_div, out_scale=out_scale, out=out,
                                    accumulate=accumulate, transpose=transpose))[0]
        return y
    if _tc_eligible(cw, L, stride, transpose, pad_mode, dilation):
        return _conv1d_tc(x, cw, dilation, pad_left, lout, pre, post_act, post_p0, cscale, res, res_div, out_scale, out, accumulate,
                          up_stride=stride if transpose else 0)
    planes = None
    if emit is not None:
        if not emit_eligible(cw, x, lout, stride, dilation, transpose) or res is not None or cscale is not None or accumulate or post_act or out is not None:
            raise ValueError("conv1d: emit= needs a stride-1 depthwise layer with Cout % 64 == 0 and no epilogue extras (see ops.emit_eligible)")
        planes = Planes(torch.empty(B, lout, cw.cout, device=x.device, dtype=torch.bfloat16),
                        torch.empty(B, lout, cw.cout, device=x.device, dtype=torch.bfloat16) if TC_MODE[0] == "x2" else None, cw.cout)
    elif out is None:
        out = torch.empty(B, lout, cw.cout, device=x.device, dtype=torch.float32)
    else:
        _chk3(out, "conv1d out")
        if out.shape != (B, lout, cw.cout):
            raise ValueError(f"conv1d: out has shape {tuple(out.shape)}, expected {(B, lout, cw.cout)}")
    p = Conv1dParams()
    p.x, p.x_bs, p.x_ld = x.data_ptr(), x.stride(0), x.stride(1)
    p.B, p.L, p.Cin = B, L, cin
    p.w, p.bias = cw.w.data_ptr(), _p(cw.bias)
    if planes is None:
        p.y, p.y_bs, p.y_ld = out.data_ptr(), out.stride(0), out.stride(1)
    else:
        p.emit_hi, p.emit_lo, p.emit_ld = planes.hi.data_ptr(), _p(planes.lo), cw.cout
        p.emit_act, p.emit_p0, p.emit_a, p.emit_b = emit.act, emit.p0, _p(emit.a), _p(emit.b)
    p.Lout, p.Cout = lout, cw.cout
    p.K, p.stride, p.dilation, p.pad_left, p.groups, p.pad_mode = cw.K, stride, dilation, pad_left, cw.groups, pad_mode
    if pre is not None:
        p.pre_scale, p.pre_shift = _p(pre.scale), _p(pre.shift)
        p.pre_act, p.pre_p0, p.pre_a, p.pre_b = pre.act, pre.p0, _p(pre.a), _p(pre.b)
    p.post_act, p.post_p0 = post_act, post_p0
    if cscale is not None:
        p.post_cscale = cscale.data_ptr()
        p.post_cscale_bs = cscale.stride(0) if cscale.dim() == 2 else 0
    if res is not None:
        _chk3(res, "conv1d res")
        p.res, p.res_bs, p.res_ld = res.data_ptr(), (res.stride(0) if res.shape[0] == B else 0), res.stride(1)
    p.res_div = res_div
    p.out_scale, p.accumulate = out_scale, int(accumulate)
    fn = _lib.lib().b2a_convtr1d_cl if transpose else _lib.lib().b2a_conv1d_cl
    if PROFILE_TAGS is not None:
        TAG[0] = f"cuda-core conv [{B}x{L}x{cw.cin}->{cw.cout} k{cw.K} s{stride} d{dilation} g{cw.groups}{' T' if transpose else ''}]"
    _call("conv" if cw.groups == 1 and cw.cin * cw.K >= 64 else "other", fn, 1, C.byref(p), _stream())
    if planes is not None:
        return planes
    return out


def emit_eligible(cw: "ConvW", x: torch.Tensor, lout: int, stride: int = 1, dilation: int = 1, transpose: bool = False) -> bool:
    """True when conv1d(x, cw, emit=...) can write the next layer's bf16 planes directly (the vectorised depthwise kernel)."""
    return (TC_MODE[0] != "off" and not transpose and stride == 1 and cw.groups == cw.cin == cw.cout and cw.cout % 64 == 0 and cw.K <= 16
            and lout >= 128 and x.stride(1) % 4 == 0 and x.stride(0) % 4 == 0 and x.data_ptr() % 16 == 0
            and (128 + (cw.K - 1) * dilation) * 128 * 4 <= 160 * 1024)


def emit_tc_eligible(cw: "ConvW", L: int) -> bool:
    """True when ``linear(x, cw, planes=True / qkv_heads=)`` can run: a tensor-core Linear at L rows whose Cout needs no pad
    channels in its consumer's bf16 planes."""
    return cw.K == 1 and not cw.f16 and cw.cout % 64 == 0 and _tc_eligible(cw, L, 1, False, 0)


def prep_bf16(x: torch.Tensor, pre: Optional[Pre], cpad: int, planes: int = 2, f16: bool = False):
    """Conv prologue -> (hi, lo) bf16 (or fp16) planes [B, L, cpad] (lo None when planes == 1)."""
    _chk3(x, "prep_bf16 x")
    B, L, Cc = x.shape
    dt = torch.float16 if f16 else torch.bfloat16
    hi = torch.empty(B, L, cpad, device=x.device, dtype=dt)
    lo = torch.empty(B, L, cpad, device=x.device, dtype=dt) if planes == 2 else None
    pre = pre or Pre()
    _call("prep", _lib.lib().b2a_prep_bf16, 1, x.data_ptr(), x.stride(0), x.stride(1), B, L, Cc, cpad, _p(pre.scale), _p(pre.shift),
          pre.act, pre.p0, _p(pre.a), _p(pre.b), hi.data_ptr(), _p(lo), int(f16), _stream())
    return hi, lo


def _new_planes(B: int, L: int, C: int, device) -> Planes:
    """Uninitialised bf16 planes [B, L, C] for a producer to fill (lo only in "x2" mode)."""
    return Planes(torch.empty(B, L, C, device=device, dtype=torch.bfloat16),
                  torch.empty(B, L, C, device=device, dtype=torch.bfloat16) if TC_MODE[0] == "x2" else None, C)


@dataclass
class AttnPlanes:
    """The q / k / v operands of the tensor-core attention, already split into its fp16 planes (q pre-scaled) inside its workspace
    ``ws`` by the fused qkv projection's epilogue: ``linear(x, cw, qkv_heads=H, qkv_scale=s)``."""
    ws: torch.Tensor
    B: int
    T: int
    H: int


def _conv1d_tc(x, cw, dilation, pad_left, lout, pre, post_act, post_p0, cscale, res, res_div, out_scale, out, accumulate,
               up_stride=0, emit: Optional[Planes] = None, attn: Optional[AttnPlanes] = None, attn_scale=0.0):
    if isinstance(x, Planes):
        B, L, _ = x.shape
        hi, lo = x.hi, x.lo
    else:
        B, L, _ = x.shape
        hi, lo = prep_bf16(x, pre, cw.cin_pad, 2 if TC_MODE[0] == "x2" else 1, cw.f16)
    if out is None:
        out = torch.empty(B, lout, cw.cout, device=hi.device, dtype=torch.float32)
    else:
        _chk3(out, "conv1d out")
        if out.shape != (B, lout, cw.cout):
            raise ValueError(f"conv1d: out has shape {tuple(out.shape)}, expected {(B, lout, cw.cout)}")
    if up_stride:
        taps, n_total = cw.K // up_stride, up_stride * cw.cout
        w_tc, w_lo = _tc_transposed_weights(cw, up_stride)
        shifts = (C.c_int32 * taps)(*[-j for j in range(taps)])
    else:
        taps, n_total, w_tc, w_lo = cw.K, cw.cout, cw.w_tc, cw.w_tc_lo
        shifts = (C.c_int32 * taps)(*[k * dilation - pad_left for k in range(taps)])
    cs, cs_bs = (None, 0) if cscale is None else (cscale.data_ptr(), cscale.stride(0) if cscale.dim() == 2 else 0)
    r, r_bs, r_ld = (None, 0, 0)
    if res is not None:
        _chk3(res, "conv1d res")
        r, r_bs, r_ld = res.data_ptr(), (res.stride(0) if res.shape[0] == B else 0), res.stride(1)
    _call("conv_tc", _lib.lib().b2a_conv1d_tc, 1, hi.data_ptr(), _p(lo), int(cw.f16), B, L, cw.cin_pad, w_tc.data_ptr(), _p(w_lo), taps, shifts, n_total, lout,
          _p(cw.bias), post_act, post_p0, cs, cs_bs, r, r_bs, r_ld, res_div, out_scale, int(accumulate), out.data_ptr(), out.stride(0),
          out.stride(1), up_stride, pad_left if up_stride else 0,
          None if emit is None else emit.hi.data_ptr(), None if emit is None else _p(emit.lo), 0 if emit is None else emit.hi.stride(1),
          None if attn is None else attn.ws.data_ptr(), 0 if attn is None else attn.H, float(attn_scale), _stream())
    return out


CL_PATHS = {1: "linear_rows", 2: "narrow", 3: "dense", 4: "dw_tiled4", 5: "dw_tiled", 6: "dw", 7: "convtr_dense", 8: "convtr_dw"}


def conv1d_cl_last_path() -> dict:
    """Kernel of this host thread's last b2a_conv1d_cl / b2a_convtr1d_cl launch: {"kernel": name (None before any launch),
    "variant": (v1, v2, v3)} as include/b200audio.h lists them per kernel (dense: (BN, CI, 0), dw_tiled4: (CW, KT, SNAKE), ...)."""
    out = (C.c_int32 * 4)()
    _lib.check(_lib.lib().b2a_conv1d_cl_last_path(out))
    return {"kernel": CL_PATHS.get(out[0]), "variant": (out[1], out[2], out[3])}


def conv1d_tc_last_config() -> dict:
    """Tiling of this host thread's last b2a_conv1d_tc launch: {"BN", "grid": (x, y, z), "stages"} (BN 0 before any launch)."""
    out = (C.c_int32 * 5)()
    _lib.check(_lib.lib().b2a_conv1d_tc_last_config(out))
    return {"BN": out[0], "grid": (out[1], out[2], out[3]), "stages": out[4]}


def conv1d_fused_last_config() -> dict:
    """Tiling of this host thread's last b2a_conv1d_fused launch: {"grid", "BN": [per problem], "ksplit": [per problem]}, problems in
    the order they were passed."""
    out = (C.c_int32 * 10)()
    _lib.check(_lib.lib().b2a_conv1d_fused_last_config(out))
    n = out[0]
    return {"grid": out[1], "BN": [out[2 + 2 * i] for i in range(n)], "ksplit": [out[3 + 2 * i] for i in range(n)]}


# ---------------------------------------------------------------------------------------------------------------- fused wgmma conv
# One launch per layer (or per GROUP of independent layers): InstanceNorm / AdaIN coefficients from the producer's (sum, sumsq), the
# input activation, the 16-bit hi/lo split, the tap-summed GEMM, the epilogue and the output's (sum, sumsq) -- csrc/conv_fused.cu.
FUSED = [os.environ.get("B2A_FUSED", "1") != "0"]
# conv1d() / linear() route single layers to the fused kernel only on request: its A operand is converted by the CTA's own warps, which
# pays off where it removes whole passes (Kokoro's AdaIN statistics + prologue, called explicitly through conv_fused) but loses to the
# pre-split planes + TMA pipeline on plain wide GEMMs (measured, round 2: Whisper encoder GEMMs 23 -> 89 ms, Mimi 34 -> 89 ms, SNAC 22 -> 33 ms
# with the fused kernel as the default route).
FUSED_DISPATCH = [os.environ.get("B2A_FUSED_DISPATCH", "0") == "1"]


@contextlib.contextmanager
def fused_dispatch(on: bool = True):
    """Route eligible conv1d() / linear() calls inside the block through the fused kernel (Kokoro: thin layers at L <= 780 where the
    prologue pass of the split path is a separate launch on the critical path)."""
    old = FUSED_DISPATCH[0]
    FUSED_DISPATCH[0] = bool(on) and FUSED[0]
    try:
        yield
    finally:
        FUSED_DISPATCH[0] = old
FUSED_WS_BYTES = 16 << 20
_FUSED_WS = {}


@dataclass
class PreStats:
    """Input transform whose scale/shift the kernel derives itself: InstanceNorm over L from ``stats`` [B, C, 2, 4] int64 (binned sum, sumsq:
    ``new_stats`` / ``stats_value``) as accumulated by the producing layer, folded with AdaIN's (1 + gamma) / beta rows ``gb`` [B, 2C] (None: plain InstanceNorm); then
    the activation."""
    stats: torch.Tensor
    gb: Optional[torch.Tensor] = None
    eps: float = 1e-5
    act: int = 0
    p0: float = 0.0
    a: Optional[torch.Tensor] = None
    b: Optional[torch.Tensor] = None


STAT_BINS, STAT_BIN0, STAT_BIN_BITS = 4, -100, 40          # csrc/common.cuh: B2A_NBIN, B2A_BIN0, B2A_BIN_BITS


def new_stats(B: int, Cc: int, device) -> torch.Tensor:
    """Zeroed (sum, sumsq) accumulator for ``FusedProblem(..., stats_out=)``: [B, C, 2, 4] int64 bins (multiples of 2^(-100 + 40 k)); integer
    atomics make the accumulation independent of the order in which CTAs arrive -> bit-reproducible statistics."""
    return torch.zeros(B, Cc, 2, STAT_BINS, device=device, dtype=torch.int64)


def stats_value(stats: torch.Tensor) -> torch.Tensor:
    """Binned accumulator [..., 4] int64 -> float64 values [...] (what repro_value computes on the device)."""
    w = torch.tensor([2.0 ** (STAT_BIN0 + STAT_BIN_BITS * k) for k in range(STAT_BINS)], dtype=torch.float64, device=stats.device)
    t = torch.zeros(stats.shape[:-1], dtype=torch.float64, device=stats.device)
    for k in range(STAT_BINS - 1, -1, -1):
        t = t + stats[..., k].double() * w[k]
    return t


def _al16(t: Optional[torch.Tensor]) -> bool:
    return t is None or (t.data_ptr() % 16 == 0 and t.stride(1) % 4 == 0 and t.stride(0) % 4 == 0)


def fused_eligible(x, cw: "ConvW", stride: int = 1, dilation: int = 1, transpose: bool = False, pad_mode: int = 0, out=None, res=None) -> bool:
    """Dense layers the fused kernel takes: tensor-core weights, stride 1 (or a polyphase transposed conv), taps spanning <= 64 rows,
    16-byte aligned fp32 rows, and room in shared memory for two weight stages (split fp32 weights at BN 128 in "x2" mode: a span of
    at most 24 rows; b2a_conv1d_fused_fits decides)."""
    if not FUSED[0] or TC_MODE[0] == "off" or cw.w_tc is None or pad_mode != 0 or cw.cout % 32 != 0 or cw.groups != 1 or isinstance(x, Planes):
        return False
    if x.dtype != torch.float32 or x.dim() != 3 or x.stride(2) != 1 or x.stride(1) % 4 or x.stride(0) % 4 or x.data_ptr() % 16:
        return False
    if x.stride(1) < -(-x.shape[2] // 4) * 4 or not _al16(out) or not _al16(res):
        return False
    if transpose:
        if not (dilation == 1 and cw.K % stride == 0 and cw.K // stride <= 32 and cw.cin * (cw.K // stride) >= TC_MIN_K):
            return False
        span, n_total = cw.K // stride - 1, stride * cw.cout
    else:
        if not (stride == 1 and cw.K <= 32 and cw.cin * cw.K >= TC_MIN_K):
            return False
        span, n_total = (cw.K - 1) * dilation, cw.cout
    return bool(_lib.lib().b2a_conv1d_fused_fits(span, n_total, cw.cout, 1 if cw.w_tc_lo is None else 2, 2 if TC_MODE[0] == "x2" else 1))


class FusedProblem:
    """One problem of a fused launch: the filled C struct, its output tensor and the tensors it points into (kept alive)."""

    def __init__(self, x, cw: "ConvW", *, stride=1, dilation=1, pad_left=0, lout=None, pre=None, x_add=(), in_scale=1.0, post_act=0, post_p0=0.0,
                 cscale=None, res=None, res_div=1, out_scale=1.0, out=None, accumulate=False, transpose=False, stats_out=None):
        _chk3(x, "conv_fused x")
        B, L, cin = x.shape
        if cin != cw.cin:
            raise ValueError(f"conv_fused: input has {cin} channels, weight expects {cw.cin}")
        if lout is None:
            lout = (L - 1) * stride + cw.K - 2 * pad_left if transpose else (L + 2 * pad_left - dilation * (cw.K - 1) - 1) + 1
        if out is None:
            out = torch.empty(B, lout, cw.cout, device=x.device, dtype=torch.float32)
        else:
            _chk3(out, "conv_fused out")
            if out.shape != (B, lout, cw.cout):
                raise ValueError(f"conv_fused: out has shape {tuple(out.shape)}, expected {(B, lout, cw.cout)}")
        p = ConvFParams()
        p.x, p.x_bs, p.x_ld, p.in_scale = x.data_ptr(), x.stride(0), x.stride(1), float(in_scale)
        keep = [x, out, cw]
        for i, xa in enumerate(x_add):
            if xa.shape != x.shape or xa.stride() != x.stride() or xa.dtype != torch.float32:
                raise ValueError("conv_fused: x_add tensors must have x's shape and strides")
            setattr(p, "x1" if i == 0 else "x2", xa.data_ptr())
            keep.append(xa)
        p.B, p.L, p.Cin = B, L, cin
        if isinstance(pre, PreStats):
            if pre.stats.dtype != torch.int64 or tuple(pre.stats.shape) != (B, cin, 2, STAT_BINS) or not pre.stats.is_contiguous():
                raise ValueError("conv_fused: stats must be a contiguous int64 [B, Cin, 2, 4] tensor (ops.new_stats)")
            p.pre_mode, p.pre_stats, p.pre_eps = 2, pre.stats.data_ptr(), float(pre.eps)
            if pre.gb is not None:
                if pre.gb.shape[-1] != 2 * cin or pre.gb.stride(-1) != 1:
                    raise ValueError("conv_fused: gb must be [B, 2*Cin] rows (gamma | beta)")
                p.pre_gb, p.pre_gb_bs = pre.gb.data_ptr(), (pre.gb.stride(0) if pre.gb.dim() == 2 and pre.gb.shape[0] == B and B > 1 else 0)
            keep += [pre.stats, pre.gb]
        elif pre is not None and pre.scale is not None:
            p.pre_mode, p.pre_scale, p.pre_shift = 1, pre.scale.data_ptr(), pre.shift.data_ptr()
            keep += [pre.scale, pre.shift]
        if pre is not None:
            p.pre_act, p.pre_p0, p.pre_a, p.pre_b = pre.act, float(pre.p0), _p(pre.a), _p(pre.b)
            keep += [pre.a, pre.b]
        if transpose:
            taps, n_total = cw.K // stride, stride * cw.cout
            w_tc, w_lo = _tc_transposed_weights(cw, stride)
            shifts = [-j for j in range(taps)]
            p.up_stride, p.up_crop = stride, pad_left
        else:
            taps, n_total, w_tc, w_lo = cw.K, cw.cout, cw.w_tc, cw.w_tc_lo
            shifts = [k * dilation - pad_left for k in range(taps)]
        p.w_hi, p.w_lo, p.cin_pad, p.taps, p.N = w_tc.data_ptr(), _p(w_lo), cw.cin_pad, taps, n_total
        for i, sft in enumerate(shifts):
            p.shifts[i] = sft
        p.Lout, p.bias, p.post_act, p.post_p0 = lout, _p(cw.bias), post_act, float(post_p0)
        if cscale is not None:
            p.cscale, p.cscale_bs = cscale.data_ptr(), (cscale.stride(0) if cscale.dim() == 2 else 0)
            keep.append(cscale)
        if res is not None:
            _chk3(res, "conv_fused res")
            p.res, p.res_bs, p.res_ld = res.data_ptr(), (res.stride(0) if res.shape[0] == B else 0), res.stride(1)
            keep.append(res)
        p.res_div, p.out_scale, p.accumulate = res_div, float(out_scale), int(accumulate)
        p.y, p.y_bs, p.y_ld = out.data_ptr(), out.stride(0), out.stride(1)
        if stats_out is not None:
            if stats_out.dtype != torch.int64 or tuple(stats_out.shape) != (B, cw.cout, 2, STAT_BINS) or not stats_out.is_contiguous():
                raise ValueError("conv_fused: stats_out must be a contiguous int64 [B, Cout, 2, 4] tensor (ops.new_stats)")
            p.stats_out = stats_out.data_ptr()
            keep.append(stats_out)
        self.p, self.out, self.keep, self.f16 = p, out, keep, cw.f16


def conv_fused(problems) -> list:
    """Launch 1..4 independent fused conv problems on one persistent grid; returns their outputs."""
    if isinstance(problems, FusedProblem):
        problems = [problems]
    n = len(problems)
    if not 1 <= n <= 4:
        raise ValueError("conv_fused: 1..4 problems per launch")
    f16 = problems[0].f16
    if any(pr.f16 != f16 for pr in problems):
        raise ValueError("conv_fused: all problems of a launch must use the same 16-bit operand type")
    arr = (ConvFParams * n)(*[pr.p for pr in problems])
    dev = problems[0].out.device
    key = (dev, torch.cuda.current_stream().cuda_stream)
    ws = _FUSED_WS.get(key)
    if ws is None:
        ws = _FUSED_WS[key] = torch.zeros(FUSED_WS_BYTES, device=dev, dtype=torch.uint8)      # split-K partial tiles + (self-resetting) counters
    if PROFILE_TAGS is not None:
        TAG[0] = "fused " + " + ".join(f"[{q.B}x{q.L}x{q.Cin}->{q.N} k{q.taps}{' up' + str(q.up_stride) if q.up_stride else ''}]" for q in (pr.p for pr in problems))
    _call("conv_tc", _lib.lib().b2a_conv1d_fused, 1, arr, n, 2 if TC_MODE[0] == "x2" else 1, int(f16), ws.data_ptr(), ws.numel(), _stream())
    return [pr.out for pr in problems]


def linear(x, cw: ConvW, *, planes=False, qkv_heads=0, qkv_scale=0.0, **kw):
    """nn.Linear on [..., in] via the K=1 conv; accepts [rows, in] or [B, L, in], or the ``Planes`` a producer emitted.

    ``planes=True`` returns (y, Planes): the epilogue also writes y's bf16 planes for the next GEMM.  ``qkv_heads=H`` returns
    (y, AttnPlanes): y is a fused [q | k | v] projection and the epilogue writes the operands of ``attention_planes`` (``qkv_scale``
    is the attention's softmax scale).  Both need the tensor-core path (``emit_tc_eligible``) and a 3-D operand."""
    if planes or qkv_heads:
        if isinstance(x, torch.Tensor) and x.dim() != 3:
            raise ValueError("linear: planes= / qkv_heads= need a 3-D operand")
        B, L, _ = x.shape
        if not emit_tc_eligible(cw, L):
            raise ValueError("linear: planes= / qkv_heads= need a tensor-core layer (ops.emit_tc_eligible)")
        for k in ("out", "res"):
            t = kw.get(k)
            if t is not None and t.dim() == 2:
                kw[k] = t[None]
        out, pre, res = kw.pop("out", None), kw.pop("pre", None), kw.pop("res", None)
        post_act, post_p0, cscale, out_scale = kw.pop("post_act", 0), kw.pop("post_p0", 0.0), kw.pop("cscale", None), kw.pop("out_scale", 1.0)
        if kw:
            raise TypeError(f"linear: unsupported arguments with planes= / qkv_heads=: {sorted(kw)}")
        if isinstance(x, Planes) and (pre is not None or x.C != cw.cin or x.hi.shape[2] != cw.cin_pad or x.hi.dtype != torch.bfloat16):
            raise ValueError("linear: a Planes operand needs matching channels and dtype and takes no prologue")
        if out is None:
            out = torch.empty(B, L, cw.cout, device=cw.w.device, dtype=torch.float32)
        em = at = None
        if qkv_heads:
            if cw.cout != 3 * 64 * qkv_heads:
                raise ValueError(f"linear: qkv_heads={qkv_heads} needs Cout = {3 * 64 * qkv_heads}, got {cw.cout}")
            at = AttnPlanes(torch.empty(_lib.lib().b2a_attention_tc_ws_bytes(B, qkv_heads, L, L), device=out.device, dtype=torch.uint8),
                            B, L, qkv_heads)
        else:
            em = _new_planes(B, L, cw.cout, out.device)
        y = _conv1d_tc(x, cw, 1, 0, L, pre, post_act, post_p0, cscale, res, 1, out_scale, out, False, emit=em, attn=at, attn_scale=qkv_scale)
        return y, (at if qkv_heads else em)
    if isinstance(x, torch.Tensor) and x.dim() == 2:
        o = kw.get("out")
        if o is not None and o.dim() == 2:
            kw["out"] = o[None]
        r = kw.get("res")
        if r is not None and r.dim() == 2:
            kw["res"] = r[None]
        return conv1d(x[None], cw, **kw)[0]
    return conv1d(x, cw, **kw)


def copy2d(src: torch.Tensor, dst: torch.Tensor) -> None:
    """dst[r, c] = src[r, c] for 2-D (row-strided) float32 views."""
    rows, cols = src.shape
    assert dst.shape == src.shape and src.stride(1) == 1 and dst.stride(1) == 1
    _call("other", _lib.lib().b2a_copy2d, 1, src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), rows, cols, _stream())


def stream_rows(entries) -> None:
    """One grouped launch of row-range moves: ``entries`` = [(src, dst, add)], src / dst float32 [B, rows, C] views of equal shape
    (row-strided), dst = src (``add`` False) or dst += src.  No entry may write rows another entry reads or writes (the C side checks)."""
    entries = [e for e in entries if e[0].numel()]
    if len(entries) > _lib.ROWOPS_MAX:
        raise ValueError(f"stream_rows: at most {_lib.ROWOPS_MAX} entries per launch, got {len(entries)}")
    if not entries:
        return
    arr = (_lib.RowOp * len(entries))()
    for i, (src, dst, add) in enumerate(entries):
        _chk3(src, "stream_rows src")
        _chk3(dst, "stream_rows dst")
        if src.shape != dst.shape:
            raise ValueError(f"stream_rows: source {tuple(src.shape)} and destination {tuple(dst.shape)} differ")
        B, rows, Cc = src.shape
        arr[i] = _lib.RowOp(src.data_ptr(), src.stride(0), src.stride(1), dst.data_ptr(), dst.stride(0), dst.stride(1), B, rows, Cc, int(bool(add)))
    _call("other", _lib.lib().b2a_stream_rows, 1, arr, len(entries), _stream())


def _stream_conv_params(x, cw: ConvW, B: int, L: int, lout: int, out, stride: int, dilation: int, pad_mode: int, pre: Optional[Pre],
                        post_act: int, res, res_div: int) -> Conv1dParams:
    p = Conv1dParams()
    if L:
        _chk3(x, "stream conv x")
        p.x, p.x_bs, p.x_ld = x.data_ptr(), x.stride(0), x.stride(1)
    p.B, p.L, p.Cin = B, L, cw.cin
    p.w, p.bias = cw.w.data_ptr(), _p(cw.bias)
    if lout:
        p.y, p.y_bs, p.y_ld = out.data_ptr(), out.stride(0), out.stride(1)
    p.Lout, p.Cout = lout, cw.cout
    p.K, p.stride, p.dilation, p.groups, p.pad_mode = cw.K, stride, dilation, cw.groups, pad_mode
    if pre is not None:
        if pre.scale is not None or pre.shift is not None or pre.a is not None or pre.b is not None:
            raise ValueError("stream conv: the prologue is an activation only")
        p.pre_act, p.pre_p0 = pre.act, pre.p0
    p.post_act = post_act
    if res is not None:
        _chk3(res, "stream conv res")
        p.res, p.res_bs, p.res_ld = res.data_ptr(), res.stride(0), res.stride(1)
    p.res_div, p.out_scale = res_div, 1.0
    return p


def conv1d_stream(x: Optional[torch.Tensor], cw: ConvW, hist: torch.Tensor, H: int, step: torch.Tensor, *, B=None, stride=1, dilation=1,
                  pad_mode=0, fresh=False, pre: Optional[Pre] = None, post_act=0, cscale=None, res=None, res_div=1, out=None) -> torch.Tensor:
    """b2a_conv1d_stream: the causal conv of [history (H rows) | x] -> its complete windows [B, Lout, Cout] (possibly 0 rows), the unconsumed
    rows carried into the other slot of ``hist`` float32 [2, B, keff - 1, Cin] (slot ``step[0] & 1`` is read).  ``x`` None = no new rows.
    ``cscale`` float32 [B, Cout] scales the output after post_act.  Returns the output; the caller's new history length is
    H + L - Lout * stride."""
    L = 0 if x is None else x.shape[1]
    B = x.shape[0] if x is not None else B
    keff = (cw.K - 1) * dilation + 1
    lout = (H + L - keff) // stride + 1 if H + L >= keff else 0
    if hist.dtype != torch.float32 or not hist.is_cuda or not hist.is_contiguous() or hist.shape != (2, B, max(keff - 1, 1), cw.cin):
        raise ValueError(f"conv1d_stream: history buffer must be float32 [2, {B}, {max(keff - 1, 1)}, {cw.cin}], got {tuple(hist.shape)}")
    if step.dtype != torch.int32 or not step.is_cuda or step.numel() < 1:
        raise ValueError(f"conv1d_stream: step must be an int32 CUDA tensor, got {step.dtype} {step.device}")
    if L and x.shape[2] != cw.cin:
        raise ValueError(f"conv1d_stream: input has {x.shape[2]} channels, weight expects {cw.cin}")
    if res is not None:
        _chk3(res, "conv1d_stream res")
        if res.shape[0] != B or res.shape[1] < -(-lout // max(res_div, 1)) or res.shape[2] != cw.cout:
            raise ValueError(f"conv1d_stream: res must be [{B}, >= ceil({lout} / {res_div}), {cw.cout}], got {tuple(res.shape)}")
    if out is None:
        out = torch.empty(B, lout, cw.cout, device=hist.device, dtype=torch.float32)
    else:
        _chk3(out, "conv1d_stream out")
        if out.shape != (B, lout, cw.cout):
            raise ValueError(f"conv1d_stream: out has shape {tuple(out.shape)}, expected {(B, lout, cw.cout)}")
    p = _stream_conv_params(x, cw, B, L, lout, out, stride, dilation, pad_mode, pre, post_act, res, res_div)
    if cscale is not None:
        if cscale.dtype != torch.float32 or not cscale.is_cuda or cscale.shape != (B, cw.cout) or cscale.stride(1) != 1:
            raise ValueError(f"conv1d_stream: cscale must be CUDA float32 [{B}, {cw.cout}], got {tuple(cscale.shape)} {cscale.dtype}")
        p.post_cscale, p.post_cscale_bs = cscale.data_ptr(), cscale.stride(0)
    _call("conv", _lib.lib().b2a_conv1d_stream, 1, C.byref(p), hist.data_ptr(), hist.stride(1), H, step.data_ptr(), int(fresh), _stream())
    return out


def convtr1d_stream(x: torch.Tensor, cw: ConvW, tail: torch.Tensor, *, stride: int, pre: Optional[Pre] = None, out=None) -> torch.Tensor:
    """b2a_convtr1d_stream: [B, L*stride, Cout] = bias + transposed conv of x + the held-back ``tail`` float32 [B, K - stride, Cout] on the
    first rows; ``tail`` then holds the next K - stride rows without the bias."""
    _chk3(x, "convtr1d_stream x")
    B, L, _ = x.shape
    if tail.dtype != torch.float32 or not tail.is_cuda or not tail.is_contiguous() or tail.shape != (B, cw.K - stride, cw.cout):
        raise ValueError(f"convtr1d_stream: tail must be contiguous float32 [{B}, {cw.K - stride}, {cw.cout}], got {tuple(tail.shape)}")
    if out is None:
        out = torch.empty(B, L * stride, cw.cout, device=x.device, dtype=torch.float32)
    else:
        _chk3(out, "convtr1d_stream out")
        if out.shape != (B, L * stride, cw.cout):
            raise ValueError(f"convtr1d_stream: out has shape {tuple(out.shape)}, expected {(B, L * stride, cw.cout)}")
    p = _stream_conv_params(x, cw, B, L, L * stride, out, stride, 1, 0, pre, 0, None, 1)
    _call("conv", _lib.lib().b2a_convtr1d_stream, 1, C.byref(p), tail.data_ptr(), tail.stride(0), _stream())
    return out


def _chk_rings(name: str, B: int, hd: int, k_ring: torch.Tensor, v_ring: torch.Tensor, pos: torch.Tensor) -> None:
    """The ring kernels read rows of exactly H*D floats at one batch stride and capacity, taken from k_ring, for both rings."""
    for r in (k_ring, v_ring):
        if r.dtype != torch.float32 or not r.is_cuda or r.dim() != 3 or not r.is_contiguous():
            raise ValueError(f"{name}: rings must be contiguous CUDA float32 [B, cap, H D] tensors, got {tuple(r.shape)} {r.dtype} {r.device}")
    if k_ring.shape != v_ring.shape or k_ring.shape[0] != B or k_ring.shape[2] != hd:
        raise ValueError(f"{name}: rings must both be [{B}, cap, {hd}], got {tuple(k_ring.shape)} and {tuple(v_ring.shape)}")
    if pos.dtype != torch.int32 or not pos.is_cuda or pos.numel() < 1:
        raise ValueError(f"{name}: pos must be an int32 CUDA tensor, got {pos.dtype} {pos.device}")


def ring_rope_kv(qkv: torch.Tensor, n_heads: int, k_ring: torch.Tensor, v_ring: torch.Tensor, pos: torch.Tensor, *, base: float) -> None:
    """b2a_ring_rope_kv: RoPE (interleaved pairs) of q in place and of k at positions pos[0] + t; k, v into ring rows (pos[0] + t) % cap."""
    _chk3(qkv, "ring_rope_kv qkv")
    B, T, w = qkv.shape
    if w % (3 * n_heads):
        raise ValueError(f"ring_rope_kv: qkv width {w} is not 3 x {n_heads} heads")
    D = w // (3 * n_heads)
    _chk_rings("ring_rope_kv", B, n_heads * D, k_ring, v_ring, pos)
    _call("rope", _lib.lib().b2a_ring_rope_kv, 1, qkv.data_ptr(), qkv.stride(0), qkv.stride(1), B, T, n_heads, D, base, k_ring.data_ptr(),
          v_ring.data_ptr(), k_ring.stride(0), k_ring.shape[1], pos.data_ptr(), _stream())


def ring_attn(q: torch.Tensor, k_ring: torch.Tensor, v_ring: torch.Tensor, pos: torch.Tensor, *, n_heads: int, scale: float, window: int,
              out=None) -> torch.Tensor:
    """b2a_ring_attn: q [B, T, H D] (row-strided view) at positions pos[0] + t against the ring caches [B, cap, H D] -> [B, T, H D]."""
    _chk3(q, "ring_attn q")
    B, T, hd = q.shape
    if hd % n_heads:
        raise ValueError(f"ring_attn: q width {hd} is not a multiple of {n_heads} heads")
    _chk_rings("ring_attn", B, hd, k_ring, v_ring, pos)
    if out is None:
        out = torch.empty(B, T, hd, device=q.device, dtype=torch.float32)
    else:
        _chk3(out, "ring_attn out")
        if out.shape != (B, T, hd):
            raise ValueError(f"ring_attn: out has shape {tuple(out.shape)}, expected {(B, T, hd)}")
    _call("attention", _lib.lib().b2a_ring_attn, 1, q.data_ptr(), q.stride(0), q.stride(1), k_ring.data_ptr(), v_ring.data_ptr(), k_ring.stride(0),
          k_ring.shape[1], out.data_ptr(), out.stride(0), out.stride(1), B, T, n_heads, hd // n_heads, scale, window, pos.data_ptr(), _stream())
    return out


def stream_advance(ctr: torch.Tensor, dpos: int) -> None:
    """ctr int32 [2]: ring position += dpos, history parity counter += 1 (the last launch of a streaming step)."""
    assert ctr.dtype == torch.int32 and ctr.numel() >= 2
    _call("other", _lib.lib().b2a_stream_advance, 1, ctr.data_ptr(), dpos, _stream())


def gather_rows(src: torch.Tensor, idx: torch.Tensor, out: Optional[torch.Tensor] = None, add: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[r, :] = src[idx[r], :] (+ add[r % add.shape[0], :]); src [N, C] float32, idx int64 [R]."""
    assert src.dim() == 2 and src.stride(1) == 1 and idx.dtype == torch.int64 and idx.is_contiguous()
    rows, cols = idx.shape[0], src.shape[1]
    if out is None:
        out = torch.empty(rows, cols, device=src.device, dtype=torch.float32)
    a, a_ld, a_per = (None, 0, 0) if add is None else (add.data_ptr(), add.stride(0), add.shape[0])
    _call("other", _lib.lib().b2a_gather_rows, 1, src.data_ptr(), src.stride(0), idx.data_ptr(), out.data_ptr(), out.stride(0),
          rows, cols, src.shape[0], a, a_ld, a_per, _stream())
    return out


def whisper_greedy_step(logits: torch.Tensor, tokens: torch.Tensor, cur_len: int, sample_begin: int, *, suppress_mask, blank_mask,
                        eot: int, no_timestamps: int, timestamp_begin: int, max_initial_ts: int, without_timestamps: bool,
                        sum_logprobs: torch.Tensor, not_done: torch.Tensor, temperature: float = 0.0, u: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Fused logit filters + greedy / categorical update (decoding.py:295-325,349-442).  logits [B,V] fp32, tokens [B, >=cur_len] int64;
    ``temperature`` > 0 draws from softmax(filtered / temperature) with one uniform per row ``u`` [B]."""
    B, V = logits.shape
    assert logits.stride(1) == 1 and tokens.dtype == torch.int64 and tokens.stride(1) == 1
    assert u is None or (u.dtype == torch.float32 and u.is_contiguous() and u.numel() == B)
    nxt = torch.empty(B, device=logits.device, dtype=torch.int64)
    _call("sampler", _lib.lib().b2a_whisper_greedy_step, 1, logits.data_ptr(), logits.stride(0), tokens.data_ptr(), tokens.stride(0), B, cur_len,
          sample_begin, V, _p(suppress_mask), _p(blank_mask), eot, no_timestamps, timestamp_begin, max_initial_ts, int(without_timestamps),
          nxt.data_ptr(), sum_logprobs.data_ptr(), not_done.data_ptr(), float(temperature), _p(u), _stream())
    return nxt


def durations_to_index(dur, max_frames: int, speed: float = 1.0):
    """Durations [T] (float32 pre-round sums, or int64 already-rounded) -> (pred_dur int64 [T], idx int64 [max_frames]
    whose first `total` entries are valid, total int64 [1] on device)."""
    assert dur.is_contiguous() and dur.dtype in (torch.float32, torch.int64)
    T = dur.shape[0]
    pred = torch.empty(T, device=dur.device, dtype=torch.int64)
    idx = torch.zeros(max_frames, device=dur.device, dtype=torch.int64)
    total = torch.zeros(1, device=dur.device, dtype=torch.int64)
    f, i = (dur.data_ptr(), None) if dur.dtype == torch.float32 else (None, dur.data_ptr())
    _call("other", _lib.lib().b2a_durations_to_index, 1, f, i, T, speed, pred.data_ptr(), idx.data_ptr(), max_frames, total.data_ptr(), _stream())
    return pred, idx, total


_WS = {}


def _workspace(nbytes: int, device) -> torch.Tensor:
    key = (device, torch.cuda.current_stream().cuda_stream)
    ws = _WS.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 1 << 20), device=device, dtype=torch.uint8)
        _WS[key] = ws
    return ws


def adain_coeffs(x: torch.Tensor, gb: Optional[torch.Tensor], eps=1e-5):
    """InstanceNorm stats of x [B,L,C] folded with AdaIN (gamma|beta) [B,2C] -> (scale, shift) [B,C]."""
    _chk3(x, "adain_coeffs x")
    B, L, Cc = x.shape
    scale = torch.empty(B, Cc, device=x.device, dtype=torch.float32)
    shift = torch.empty(B, Cc, device=x.device, dtype=torch.float32)
    ws = _workspace(_lib.lib().b2a_adain_ws_bytes(B, L, Cc), x.device)
    _call("adain_stats", _lib.lib().b2a_adain_coeffs, 2, x.data_ptr(), x.stride(0), x.stride(1), B, L, Cc, _p(gb), eps,
                                           scale.data_ptr(), shift.data_ptr(), ws.data_ptr(), _stream())
    return scale, shift


def channel_stats(x: torch.Tensor, dsts) -> None:
    """Add (sum, sumsq) over L of x [B, L, C] to each binned accumulator in ``dsts`` (views [B, C, 2, 4] of possibly wider [B, C', 2, 4] buffers)."""
    _chk3(x, "channel_stats x")
    B, L, Cc = x.shape
    if isinstance(dsts, torch.Tensor):
        dsts = [dsts]
    n = len(dsts)
    for d in dsts:
        assert d.dtype == torch.int64 and tuple(d.shape) == (B, Cc, 2, STAT_BINS) and d.stride(3) == 1 and d.stride(2) == STAT_BINS and d.stride(1) == 2 * STAT_BINS
    ptrs = (C.c_void_p * n)(*[d.data_ptr() for d in dsts])
    bss = (C.c_int64 * n)(*[d.stride(0) for d in dsts])
    _call("adain_stats", _lib.lib().b2a_channel_stats, 1, x.data_ptr(), x.stride(0), x.stride(1), B, L, Cc, ptrs, bss, n, _stream())


def coeffs_from_stats(stats: torch.Tensor, L: int, gb: Optional[torch.Tensor], eps=1e-5):
    """Binned (sum, sumsq) [B, C, 2, 4] -> AdaIN (scale, shift) [B, C] float32 for consumers outside the fused conv (depthwise layers)."""
    B, Cc = stats.shape[:2]
    assert stats.dtype == torch.int64 and stats.is_contiguous() and tuple(stats.shape[2:]) == (2, STAT_BINS)
    scale = torch.empty(B, Cc, device=stats.device, dtype=torch.float32)
    shift = torch.empty(B, Cc, device=stats.device, dtype=torch.float32)
    _call("adain_stats", _lib.lib().b2a_coeffs_from_stats, 1, stats.data_ptr(), B, L, Cc, _p(gb), eps, scale.data_ptr(), shift.data_ptr(), _stream())
    return scale, shift


def layernorm(x: torch.Tensor, w=None, b=None, *, eps=1e-5, res=None, ada=None, rms=False, post_act=0, post_p0=0.0,
              out=None, planes=False):
    """Row LayerNorm / RMSNorm over the last dim of a 2-D row-strided view.  ``planes=True`` returns (y, Planes [1, rows, C]): the
    kernel also writes y's bf16 planes for the next GEMM (C a multiple of 64, so that they need no pad channels)."""
    shp = x.shape
    x2 = x.reshape(-1, shp[-1]) if x.dim() != 2 else x
    assert x2.stride(1) == 1
    r2 = None
    if res is not None:
        r2 = res.reshape(-1, shp[-1]) if res.dim() != 2 else res
    if out is None:
        out = torch.empty(x2.shape, device=x.device, dtype=torch.float32)
    o2 = out.reshape(-1, shp[-1]) if out.dim() != 2 else out
    pl = None
    if planes:
        if shp[-1] % 64:
            raise ValueError(f"layernorm: planes=True needs C % 64 == 0, got {shp[-1]}")
        pl = _new_planes(1, x2.shape[0], shp[-1], x.device)
    _call("layernorm", _lib.lib().b2a_layernorm, 1, x2.data_ptr(), x2.stride(0), _p(r2), 0 if r2 is None else r2.stride(0), o2.data_ptr(),
                                        o2.stride(0), x2.shape[0], shp[-1], _p(w), _p(b), _p(ada), eps, int(rms), post_act,
                                        post_p0, None if pl is None else pl.hi.data_ptr(), None if pl is None else _p(pl.lo),
                                        shp[-1], _stream())
    y = out.reshape(shp) if out.dim() == 2 and len(shp) != 2 else out
    return (y, pl) if planes else y


def attention(q, k, v, *, n_heads, n_kv_heads=None, scale, causal=False, q_offset=0, window=0, k_len=None, out=None):
    """softmax(scale q k^T + mask) v.  q [B,Tq,H*D], k/v [B,Tk,Hkv*D] (row-strided views allowed).  ``window`` > 0 limits the causal
    mask to the last ``window`` positions, so it needs ``causal=True``."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _chk3(t, "attention " + n)
    if window > 0 and not causal:
        raise ValueError(f"attention: a sliding window ({window}) needs causal=True")
    B, Tq, hd = q.shape
    H = n_heads
    Hkv = n_kv_heads or H
    D = hd // H
    if out is None:
        out = torch.empty(B, Tq, hd, device=q.device, dtype=torch.float32)
    p = AttnParams()
    p.q, p.k, p.v, p.o = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    p.q_bs, p.q_ld, p.k_bs, p.k_ld = q.stride(0), q.stride(1), k.stride(0), k.stride(1)
    p.v_bs, p.v_ld, p.o_bs, p.o_ld = v.stride(0), v.stride(1), out.stride(0), out.stride(1)
    p.B, p.Tq, p.Tk, p.H, p.Hkv, p.D = B, Tq, k.shape[1], H, Hkv, D
    p.scale, p.causal, p.q_offset, p.window = scale, int(causal), q_offset, window
    p.k_len = _p(k_len)
    if ATTN_MODE[0] == "tc" and D == 64 and Hkv == H and k_len is None and k.shape[1] >= 64 and out.stride(1) % 4 == 0:
        ws = torch.empty(_lib.lib().b2a_attention_tc_ws_bytes(B, H, Tq, k.shape[1]), device=q.device, dtype=torch.uint8)
        _call("attention", _lib.lib().b2a_attention_tc, 4, C.byref(p), ws.data_ptr(), _stream())
        return out
    _call("attention", _lib.lib().b2a_attention, 1, C.byref(p), _stream())
    return out


_ALBERT_ERR = {}


def albert_error_word(device) -> torch.Tensor:
    """int32 [1] on ``device``: set to 1 by ``albert_encoder`` when one of its grid barriers saw no progress for 10 s (that call's
    output is then invalid).  Never cleared."""
    device = torch.device(device)
    w = _ALBERT_ERR.get(device)
    if w is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("albert_encoder: run it once outside graph capture first (its error word is allocated then)")
        w = _ALBERT_ERR[device] = torch.zeros(1, device=device, dtype=torch.int32)
    return w


def albert_encoder(h: torch.Tensor, hp: Planes, layers: int, qkv: ConvW, attn_out: ConvW, ffn: ConvW, ffn_out: ConvW, ln_attn, ln_full,
                   *, heads: int, scale: float, eps: float, timeline: Optional[torch.Tensor] = None) -> None:
    """``layers`` ALBERT layers on h [1, T, hidden] float32 and its bf16 planes ``hp``, both updated in place, in one persistent launch
    (b2a_albert_encoder); bit-identical to the ``linear(qkv_heads=)`` / ``attention_planes`` / ``linear`` / ``layernorm(planes=True)``
    sequence.  ``ln_attn`` / ``ln_full`` are (weight, bias) pairs; ``timeline`` int64 [layers * 7, SMs, 2] selects the profiling build."""
    if h.dtype != torch.float32 or not h.is_contiguous() or h.dim() != 3 or h.shape[0] != 1:
        raise ValueError(f"albert_encoder: h must be a contiguous float32 [1, T, hidden] tensor, got {tuple(h.shape)} {h.dtype}")
    T, hs = h.shape[1], h.shape[2]
    inter = ffn.cout
    for cw, (n, k) in ((qkv, (3 * hs, hs)), (attn_out, (hs, hs)), (ffn, (inter, hs)), (ffn_out, (hs, inter))):
        if cw.w_tc is None or cw.K != 1 or cw.f16 or cw.w_tc_lo is not None or (cw.cout, cw.cin_pad) != (n, k) or cw.bias is None:
            raise ValueError("albert_encoder: every projection needs bf16 tensor-core weights with a bias and matching shapes")
    two = TC_MODE[0] == "x2"
    if hp.hi.shape != (1, T, hs) or (hp.lo is not None) != two:
        raise ValueError("albert_encoder: hp must hold h's bf16 planes (hi, and lo in x2 mode)")
    a = _lib.AlbertParams()
    a.T, a.layers, a.heads, a.hidden, a.inter, a.planes = T, layers, heads, hs, inter, 2 if two else 1
    for i, cw in enumerate((qkv, attn_out, ffn, ffn_out)):
        a.w[i], a.bias[i] = cw.w_tc.data_ptr(), cw.bias.data_ptr()
    a.ln_w[0], a.ln_b[0] = ln_attn[0].data_ptr(), ln_attn[1].data_ptr()
    a.ln_w[1], a.ln_b[1] = ln_full[0].data_ptr(), ln_full[1].data_ptr()
    a.eps, a.scale = eps, scale
    a.h, a.h_hi, a.h_lo = h.data_ptr(), hp.hi.data_ptr(), _p(hp.lo)
    err = albert_error_word(h.device)
    ws = torch.empty(_lib.lib().b2a_albert_ws_bytes(T, heads, hs, inter), device=h.device, dtype=torch.uint8)
    _call("albert", _lib.lib().b2a_albert_encoder, 1, C.byref(a), ws.data_ptr(), err.data_ptr(), _p(timeline), _stream())


def attention_planes(ap: AttnPlanes, *, planes=False, out=None):
    """Non-causal tensor-core attention over the operands a fused qkv projection emitted (``linear(..., qkv_heads=)``): one launch.
    Returns ctx [B, T, H*64], or (ctx, Planes) with ``planes=True`` (ctx's bf16 planes for the output projection)."""
    B, T, H = ap.B, ap.T, ap.H
    if T < 64:
        raise ValueError("attention_planes: the tensor-core attention needs at least 64 keys")
    if out is None:
        out = torch.empty(B, T, H * 64, device=ap.ws.device, dtype=torch.float32)
    _chk3(out, "attention_planes out")
    pl = _new_planes(B, T, H * 64, out.device) if planes else None
    p = AttnParams()
    p.o, p.o_bs, p.o_ld = out.data_ptr(), out.stride(0), out.stride(1)
    p.B, p.Tq, p.Tk, p.H, p.Hkv, p.D = B, T, T, H, H, 64
    p.operands_ready = 1
    if pl is not None:
        p.emit_hi, p.emit_lo, p.emit_ld = pl.hi.data_ptr(), _p(pl.lo), H * 64
    _call("attention", _lib.lib().b2a_attention_tc, 1, C.byref(p), ap.ws.data_ptr(), _stream())
    return (out, pl) if planes else out


def rope_(x: torch.Tensor, n_heads: int, *, offset=0, base=10000.0, traditional=True) -> torch.Tensor:
    """In-place rotary embedding on x [B,T,H*D]."""
    _chk3(x, "rope x")
    B, T, hd = x.shape
    _call("rope", _lib.lib().b2a_rope, 1, x.data_ptr(), x.stride(0), x.stride(1), B, T, n_heads, hd // n_heads, offset, base,
                                   int(traditional), _stream())
    return x


def lstm_bidir(xproj: torch.Tensor, wh: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """xproj [B,T,2*4H] (forward|backward input projections incl. biases), wh [2,4H,H] -> [B,T,2H]."""
    B, T, g8 = xproj.shape
    H = g8 // 8
    assert xproj.is_contiguous() and wh.is_contiguous() and wh.shape == (2, 4 * H, H)
    if out is None:
        out = torch.empty(B, T, 2 * H, device=xproj.device, dtype=torch.float32)
    assert out.stride(2) == 1 and (B == 1 or out.stride(0) == T * out.stride(1))
    _call("lstm", _lib.lib().b2a_lstm_bidir, 1, xproj.data_ptr(), wh.data_ptr(), out.data_ptr(), out.stride(1), B, T, H, _stream())
    return out


def stft(x: torch.Tensor, window: torch.Tensor, n_fft: int, hop: int, pad_mode: int, frames: int):
    """x [B,n] -> (re, im) each [B, frames, n_fft//2+1]; pad_mode 0 none / 1 reflect / 2 constant."""
    B, n = x.shape
    assert x.stride(1) == 1 and window.shape[0] == n_fft
    nf = n_fft // 2 + 1
    re = torch.empty(B, frames, nf, device=x.device, dtype=torch.float32)
    im = torch.empty(B, frames, nf, device=x.device, dtype=torch.float32)
    _call("other", _lib.lib().b2a_stft, 1, x.data_ptr(), x.stride(0), B, n, window.data_ptr(), n_fft, hop, pad_mode, frames,
                                   re.data_ptr(), im.data_ptr(), _stream())
    return re, im


def whisper_logmel(x: torch.Tensor, padding: int, window: torch.Tensor, filters: torch.Tensor, frames: int) -> torch.Tensor:
    """x [B,n] float32 -> log-mel [B, frames, n_mels] (audio.py:41-82)."""
    B, n = x.shape
    assert x.stride(1) == 1 and filters.is_contiguous() and filters.shape[1] == 201
    out = torch.empty(B, frames, filters.shape[0], device=x.device, dtype=torch.float32)
    gmax = torch.empty(B, device=x.device, dtype=torch.float32)
    _call("logmel", _lib.lib().b2a_whisper_logmel, 2, x.data_ptr(), x.stride(0), B, n, padding, window.data_ptr(), filters.data_ptr(),
                                             filters.shape[0], frames, out.data_ptr(), gmax.data_ptr(), _stream())
    return out


def istft(re: torch.Tensor, im: torch.Tensor, n_fft: int, hop: int, window: torch.Tensor, *, norm_sq: bool, clamp_mode: int,
          trim: int, out_len: int) -> torch.Tensor:
    """re/im [B, n_freq, T] -> [B, out_len]."""
    B, nf, T = re.shape
    assert re.is_contiguous() and im.is_contiguous() and nf == n_fft // 2 + 1
    out = torch.empty(B, out_len, device=re.device, dtype=torch.float32)
    ws = torch.empty(B, T, n_fft, device=re.device, dtype=torch.float32)
    _call("other", _lib.lib().b2a_istft, 2, re.data_ptr(), im.data_ptr(), B, n_fft, T, hop, window.data_ptr(), int(norm_sq), clamp_mode,
                                    trim, out_len, out.data_ptr(), ws.data_ptr(), _stream())
    return out


def resample_poly(x: torch.Tensor, h: torch.Tensor, up: int, down: int, n_pre_pad: int, n_pre_remove: int, n_out: int) -> torch.Tensor:
    """x [B,n] float32, h float64 FIR (already * up) -> [B, n_out] (scipy.signal.resample_poly, padtype='edge')."""
    assert x.dim() == 2 and x.stride(1) == 1 and h.dtype == torch.float64 and h.is_contiguous()
    out = torch.empty(x.shape[0], n_out, device=x.device, dtype=torch.float32)
    _call("resample", _lib.lib().b2a_resample_poly, 1, x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], h.data_ptr(), h.shape[0], up, down,
          n_pre_pad, n_pre_remove, out.data_ptr(), n_out, _stream())
    return out


def kokoro_source(f0: torch.Tensor, noise: Optional[torch.Tensor], lin_w: torch.Tensor, lin_b: torch.Tensor) -> torch.Tensor:
    """F0 curve [B, nF] -> har [B, nF*60+1, 22] (magnitude | phase of the hn-NSF source STFT)."""
    B, nF = f0.shape
    assert f0.is_contiguous()
    har = torch.empty(B, nF * 60 + 1, 22, device=f0.device, dtype=torch.float32)
    src = torch.empty(B, nF * 300, device=f0.device, dtype=torch.float32)
    # length of the reference's down-sampled phase track: size = ceil(float(W) * float(scale)) with scale = 1/300
    # (tts/models/interpolate.py:43-50) -- nF or nF + 1 depending on floating-point rounding; evaluated the same way here.
    n_down = max(1, int(math.ceil(float(nF * 300) * float(1 / 300))))
    ph = torch.empty(B, n_down, 9, device=f0.device, dtype=torch.float64)
    if noise is not None:
        assert noise.is_contiguous() and noise.shape == (B, nF * 300, 9)
    _call("source", _lib.lib().b2a_kokoro_source, 3, f0.data_ptr(), B, nF, n_down, _p(noise), lin_w.data_ptr(), lin_b.data_ptr(), har.data_ptr(),
                                            src.data_ptr(), ph.data_ptr(), _stream())
    return har


def kokoro_source_conv(har: torch.Tensor, cw: ConvW, *, stride: int = 1, pad_left: int = 0) -> torch.Tensor:
    """A noise conv on the harmonic source: har [B, L, 22] -> [B, Lout, Cout], bit-identical to ``conv1d(har, cw, stride=, pad_left=)``
    (csrc/conv.cu, b2a_kokoro_source_conv: (K, stride) = (12, 6) or (1, 1))."""
    _chk3(har, "kokoro_source_conv har")
    B, L, cin = har.shape
    if cin != 22 or cw.cin != 22 or cw.groups != 1 or not har.is_contiguous():
        raise ValueError("kokoro_source_conv: expected a contiguous [B, L, 22] source and a dense 22-channel layer")
    lout = (L + 2 * pad_left - cw.K) // stride + 1
    out = torch.empty(B, lout, cw.cout, device=har.device, dtype=torch.float32)
    if PROFILE_TAGS is not None:
        TAG[0] = f"source conv [{B}x{L}x{cin}->{cw.cout} k{cw.K} s{stride}]"
    _call("conv" if cin * cw.K >= 64 else "other", _lib.lib().b2a_kokoro_source_conv, 1, har.data_ptr(), B, L, cw.w.data_ptr(), _p(cw.bias),
          out.data_ptr(), lout, cw.cout, cw.K, stride, pad_left, _stream())
    return out


def kokoro_istft_head(x: torch.Tensor) -> torch.Tensor:
    """conv_post output [B,T,22] -> waveform [B, (T-1)*5]."""
    _chk3(x, "kokoro_istft_head x")
    B, T, _ = x.shape
    audio = torch.empty(B, (T - 1) * 5, device=x.device, dtype=torch.float32)
    _call("istft_head", _lib.lib().b2a_kokoro_istft_head, 1, x.data_ptr(), x.stride(0), x.stride(1), B, T, audio.data_ptr(), _stream())
    return audio


def randn_(out: torch.Tensor, seed: int, offset: int = 0) -> torch.Tensor:
    """Fill a contiguous float32 tensor with N(0,1) draws from our Philox kernel."""
    assert out.is_contiguous() and out.dtype == torch.float32
    _call("other", _lib.lib().b2a_randn, 1, out.data_ptr(), out.numel(), seed, offset, _stream())
    return out


def randn_dev_(out: torch.Tensor, state: torch.Tensor) -> torch.Tensor:
    """N(0,1) fill keyed by a device-resident Philox state (int64 [2] = seed, counter offset) that the call advances: graph-replay safe."""
    assert out.is_contiguous() and out.dtype == torch.float32 and state.dtype == torch.int64 and state.numel() == 2 and state.is_contiguous()
    _call("other", _lib.lib().b2a_randn_dev, 2, out.data_ptr(), out.numel(), state.data_ptr(), _stream())
    return out


def sample_token(logits: torch.Tensor, *, temperature: float, top_k: int = 0, top_p: float = 1.0, min_p: float = 0.0, u=None,
                 suppress_mask=None, seen=None, repetition_penalty: float = 1.0, return_filtered: bool = False, mark_seen: bool = False,
                 out: Optional[torch.Tensor] = None, finished=None, eos: int = -1):
    """Fused sampler on logits [B,V] (V <= 4096) -> int64 tokens [B] (and the filtered logits when asked).  ``out`` may be a
    strided int64 view (e.g. a column of the [B,16] code matrix)."""
    B, V = logits.shape
    assert logits.stride(1) == 1 and (seen is None or (seen.dtype == torch.uint8 and seen.stride(1) == 1))
    if out is None:
        out = torch.empty(B, device=logits.device, dtype=torch.int64)
    assert out.dtype == torch.int64 and out.dim() == 1 and out.shape[0] == B
    filt = torch.empty(B, V, device=logits.device, dtype=torch.float32) if return_filtered else None
    _call("sampler", _lib.lib().b2a_sample_token, 1, logits.data_ptr(), logits.stride(0), B, V, _p(suppress_mask), _p(seen),
          0 if seen is None else seen.stride(0), int(mark_seen), repetition_penalty, temperature, top_k, top_p, min_p, _p(u),
          out.data_ptr(), out.stride(0) if B > 1 else 1, _p(filt), _p(finished), eos, _stream())
    return (out, filt) if return_filtered else out


def gemv_eligible(cw: "ConvW") -> bool:
    """The decode GEMV streams ONE bf16 plane of weights in 16-byte (8-element) loads: bf16-exact K=1 layers whose input width is a
    multiple of 8 only (fp16 / fp32 checkpoints, layers whose Cout is not a multiple of 32 and other input widths go through
    ``linear``)."""
    return cw.K == 1 and cw.w_tc is not None and not cw.f16 and cw.w_tc_lo is None and cw.cin % 8 == 0


def gemv(x: torch.Tensor, cw: "ConvW", *, norm_w=None, norm_eps: float = 1e-6, swiglu: bool = False, res=None, out=None,
         prefetch: Optional["ConvW"] = None) -> torch.Tensor:
    """Decode-time nn.Linear on x [M, K] (any M; looped in groups of 8) with the bf16 weight rows of ``cw`` ([N, cin_pad]):
    optional fused RMSNorm prologue, SwiGLU (interleaved gate/up rows) and residual.  ``prefetch``: the next projection, whose
    weights are pulled into L2 while this one runs."""
    if not (x.dim() == 2 and x.stride(1) == 1 and gemv_eligible(cw)):
        raise NotImplementedError("gemv needs a bf16-exact K=1 weight with Cout % 32 == 0 and Cin % 8 == 0 (see ops.gemv_eligible); "
                                  "use ops.linear")
    M, K = x.shape
    N = cw.cout
    n_out = N // 2 if swiglu else N
    if out is None:
        out = torch.empty(M, n_out, device=x.device, dtype=torch.float32)
    assert K == cw.cin and out.shape == (M, n_out) and out.stride(1) == 1
    pf, pf_bytes = (None, 0) if prefetch is None or prefetch.w_tc is None else (prefetch.w_tc.data_ptr(), prefetch.w_tc.numel() * 2)
    for m0 in range(0, M, 8):
        m = min(8, M - m0)
        r = None if res is None else res[m0:m0 + m]
        _call("gemv", _lib.lib().b2a_gemv_bf16, 1, x[m0:m0 + m].data_ptr(), x.stride(0), m, K, cw.w_tc.data_ptr(), cw.cin_pad, N,
              _p(cw.bias), _p(norm_w), norm_eps, int(swiglu), _p(r), 0 if r is None else r.stride(0), out[m0:m0 + m].data_ptr(),
              out.stride(0), pf if m0 == 0 else None, pf_bytes, _stream())
    return out


def qknorm_rope_cache(qkv: torch.Tensor, n_heads: int, n_kv: int, head_dim: int, k_cache: torch.Tensor, v_cache: torch.Tensor, *,
                      q_norm=None, k_norm=None, eps: float = 1e-6, pos3=None, base_dev=None, base: int = 0, mrope=(0, 0),
                      theta: float = 10000.0, q_out=None, pos_shift=None, base_rows=None, slot=None) -> torch.Tensor:
    """qkv [B,S,(Hq+2Hkv)D] -> q_out [B,S,Hq*D] (normed + rotated), k/v appended to caches [B,Smax,Hkv*D] at row base+s.
    ``base_rows`` int32 [B]: per-row base (a negative row position is left padding and writes nothing); ``slot`` int32 [B]: the
    cache batch index of each row."""
    _chk3(qkv, "qkv")
    B, S, _ = qkv.shape
    if q_out is None:
        q_out = torch.empty(B, S, n_heads * head_dim, device=qkv.device, dtype=torch.float32)
    assert k_cache.shape == v_cache.shape and k_cache.stride() == v_cache.stride() and k_cache.stride(2) == 1
    assert pos3 is None or (pos3.dtype == torch.int32 and pos3.is_contiguous() and pos3.shape == (3, B, S))
    _call("rope", _lib.lib().b2a_qknorm_rope_cache, 1, qkv.data_ptr(), qkv.stride(0), qkv.stride(1), B, S, n_heads, n_kv, head_dim,
          _p(q_norm), _p(k_norm), eps, _p(pos3), _p(base_dev), base, mrope[0], mrope[1], theta, q_out.data_ptr(), q_out.stride(0),
          q_out.stride(1), k_cache.data_ptr(), v_cache.data_ptr(), k_cache.stride(0), k_cache.stride(1), k_cache.shape[1], _p(pos_shift),
          _p(_rows_i32(base_rows, B)), _p(_rows_i32(slot, B)), _stream())
    return q_out


def attn_decode(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, n_heads: int, n_kv: int, head_dim: int, *, scale: float,
                base_dev=None, base: int = 0, kv_start=None, max_k: Optional[int] = None, out=None, base_rows=None, slot=None) -> torch.Tensor:
    """Causal GQA attention of q [B,S,Hq*D] against cache rows [kv_start, base+s]; out [B,S,Hq*D].  ``base_rows`` / ``slot`` as in
    ``qknorm_rope_cache`` (a negative query position gives a zero row)."""
    _chk3(q, "q")
    B, S, _ = q.shape
    if out is None:
        out = torch.empty(B, S, n_heads * head_dim, device=q.device, dtype=torch.float32)
    if max_k is None:
        max_k = k_cache.shape[1] if base_dev is not None or base_rows is not None else base + S
    _call("attention", _lib.lib().b2a_attn_decode, 1, q.data_ptr(), q.stride(0), q.stride(1), k_cache.data_ptr(), v_cache.data_ptr(),
          k_cache.stride(0), k_cache.stride(1), out.data_ptr(), out.stride(0), out.stride(1), B, S, n_heads, n_kv, head_dim, scale,
          _p(base_dev), base, _p(kv_start), max_k, _p(_rows_i32(base_rows, B)), _p(_rows_i32(slot, B)), _stream())
    return out


def attn_prefill(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, n_heads: int, n_kv: int, head_dim: int, *, scale: float,
                 base_dev=None, base: int = 0, kv_start=None, max_k: Optional[int] = None, out=None, base_rows=None, slot=None) -> torch.Tensor:
    """``attn_decode``'s contract on the tensor cores, for prefills of >= 64 rows with head_dim 128 and two query heads per KV head."""
    _chk3(q, "q")
    B, S, _ = q.shape
    if out is None:
        out = torch.empty(B, S, n_heads * head_dim, device=q.device, dtype=torch.float32)
    if max_k is None:
        max_k = k_cache.shape[1] if base_dev is not None or base_rows is not None else base + S
    _call("attention", _lib.lib().b2a_attn_prefill, 1, q.data_ptr(), q.stride(0), q.stride(1), k_cache.data_ptr(), v_cache.data_ptr(),
          k_cache.stride(0), k_cache.stride(1), out.data_ptr(), out.stride(0), out.stride(1), B, S, n_heads, n_kv, head_dim, scale,
          _p(base_dev), base, _p(kv_start), max_k, _p(_rows_i32(base_rows, B)), _p(_rows_i32(slot, B)), _stream())
    return out


def swiglu(x: torch.Tensor, out=None, interleaved: bool = False) -> torch.Tensor:
    """x [..., 2I] (gate | up halves, or interleaved pairs) -> silu(gate) * up [..., I]."""
    shp = x.shape
    I = shp[-1] // 2
    x2 = x.reshape(-1, shp[-1])
    assert x2.stride(1) == 1
    if out is None:
        out = torch.empty(*shp[:-1], I, device=x.device, dtype=torch.float32)
    o2 = out.reshape(-1, I)
    _call("other", _lib.lib().b2a_swiglu, 1, x2.data_ptr(), x2.stride(0), x2.shape[0], I, int(interleaved), o2.data_ptr(), o2.stride(0), _stream())
    return out


class EmbedTables:
    """Device arrays of table pointers / sizes for embed_sum (built once per model)."""

    def __init__(self, tables):
        self.tables = [t for t in tables]
        for t in self.tables:
            assert t.dim() == 2 and t.is_contiguous() and t.dtype == torch.float32 and t.shape[1] == self.tables[0].shape[1]
        dev = self.tables[0].device
        self.ptrs = torch.tensor([t.data_ptr() for t in self.tables], dtype=torch.int64, device=dev)
        self.bins = torch.tensor([t.shape[0] for t in self.tables], dtype=torch.int32, device=dev)
        self.dim = self.tables[0].shape[1]


def embed_sum(codes: torch.Tensor, tabs: EmbedTables, *, text=None, pad=None, out=None, err=None, tidx=None,
              finished=None) -> torch.Tensor:
    """out[b] = text-or-pad(b) + sum_g tables[g][codes[b,g]]; codes int64 [B,G] (G <= len(tables)).  ``text`` [B, n, H] is read at
    the per-row trailing indices ``tidx`` int32 [B] (clamp-pad rule; advanced for rows that are not ``finished``); without them
    every row reads ``pad`` [H] (None = 0)."""
    if (text is None) != (tidx is None):
        raise ValueError("embed_sum: text= and tidx= go together")
    assert codes.dtype == torch.int64 and codes.dim() == 2 and codes.stride(1) == 1
    B, G = codes.shape
    assert G <= len(tabs.tables)
    if out is None:
        out = torch.empty(B, tabs.dim, device=codes.device, dtype=torch.float32)
    tb, ts, nt = (0, 0, 0) if text is None else (text.stride(0), text.stride(1), text.shape[1])
    _call("other", _lib.lib().b2a_embed_sum, 1, codes.data_ptr(), codes.stride(0), B, G, tabs.dim, tabs.ptrs.data_ptr(), tabs.bins.data_ptr(),
          _p(text), tb, ts, nt, _p(pad), out.data_ptr(), out.stride(0), _p(err), _p(tidx), _p(finished), _stream())
    return out


def _rows_i32(t: Optional[torch.Tensor], B: int) -> Optional[torch.Tensor]:
    """A per-row device array (``base_rows`` / ``slot``): int32 [B], contiguous."""
    assert t is None or (t.dtype == torch.int32 and t.is_cuda and t.is_contiguous() and t.numel() == B), "per-row arrays are int32 [B] on the device"
    return t


def slot_advance(lengths: torch.Tensor, frames: torch.Tensor, finished: torch.Tensor, cap: torch.Tensor, codes: torch.Tensor,
                 out: torch.Tensor, u_tab: torch.Tensor, u: torch.Tensor) -> None:
    """End of a batch-session frame over B slots (include/b200audio.h: b2a_slot_advance): live slots record ``codes`` [B, G] into
    ``out`` [B, F, G] at their frame count, advance their cache length and frame count, finish at ``cap`` and load the next frame's
    uniforms ``u`` [G, B] from ``u_tab`` [B, F, G]."""
    B, G = codes.shape
    assert codes.dtype == torch.int64 and codes.is_contiguous() and out.dtype == torch.int64 and out.is_contiguous() and out.shape[0] == B
    assert finished.dtype == torch.uint8 and all(t.dtype == torch.int32 and t.numel() == B for t in (lengths, frames, cap))
    assert u_tab.is_contiguous() and u_tab.shape[0] == B and u.is_contiguous() and u.shape == (G, B)
    _call("other", _lib.lib().b2a_slot_advance, 1, lengths.data_ptr(), frames.data_ptr(), finished.data_ptr(), cap.data_ptr(), codes.data_ptr(),
          G, out.data_ptr(), out.stride(0), u_tab.data_ptr(), u_tab.stride(0), u.data_ptr(), B, _stream())


def incr_(p: torch.Tensor, v: int = 1) -> None:
    assert p.dtype == torch.int32
    _call("other", _lib.lib().b2a_incr_i32, 1, p.data_ptr(), v, _stream())


def rvq_decode(codes: torch.Tensor, codebooks: torch.Tensor, out: Optional[torch.Tensor] = None, check=True,
               err: Optional[torch.Tensor] = None) -> torch.Tensor:
    """codes int64 [B,nq,T], codebooks [nq,bins,dim] -> sum of gathers [B,T,dim].  ``err``: a zeroed int32 [1] flag to reuse (saves
    the fill kernel of a fresh one); it stays zero unless a code is out of range."""
    assert codes.dtype == torch.int64 and (codes.stride(2) == 1 or codes.shape[2] == 1) and codebooks.is_contiguous()
    B, nq, T = codes.shape
    _, bins, dim = codebooks.shape
    if out is None:
        out = torch.empty(B, T, dim, device=codes.device, dtype=torch.float32)
    if err is None:
        err = torch.zeros(1, device=codes.device, dtype=torch.int32)
    _call("rvq", _lib.lib().b2a_rvq_decode, 1, codes.data_ptr(), codes.stride(0), codes.stride(1), B, nq, T, codebooks.data_ptr(), bins,
                                         dim, out.data_ptr(), out.stride(1), err.data_ptr(), _stream())
    if check and int(err.item()) != 0:
        raise ValueError(f"rvq_decode: code index out of range [0, {bins})")
    return out


def rvq_encode(x: torch.Tensor, codebooks: torch.Tensor, c2: torch.Tensor, *, mode: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Nearest-code search with the residual loop: x [R, D] fp32 rows, codebooks [nq, bins, D], c2 [nq, bins] float64 (|e|^2 / 2, or |en|^2 for
    ``mode=1`` = SNAC's single-level cosine search on an L2-normalised table) -> int64 codes [R, nq] (or ``out``, any strides)."""
    assert x.dim() == 2 and x.stride(1) == 1 and x.dtype == torch.float32 and codebooks.is_contiguous() and c2.dtype == torch.float64 and c2.is_contiguous()
    R, D = x.shape
    nq, bins, _ = codebooks.shape
    if out is None:
        out = torch.empty(R, nq, device=x.device, dtype=torch.int64)
    assert out.shape == (R, nq) and out.dtype == torch.int64
    _call("rvq", _lib.lib().b2a_rvq_encode, 1, x.data_ptr(), x.stride(0), R, D, codebooks.data_ptr(), c2.data_ptr(), bins, nq, mode, out.data_ptr(),
          out.stride(0), out.stride(1), _stream())
    return out


def snac_from_codes(codes, strides, embs, ws, biases, dim: int, check=True) -> torch.Tensor:
    """SNAC quantizer.from_codes: codes[l] int64 [B, T/stride_l]; embs[l] [bins, cd]; ws[l] [cd, dim]; -> [B,T,dim]."""
    n = len(codes)
    B = codes[0].shape[0]
    T = codes[-1].shape[1] * strides[-1]
    bins, cd = embs[0].shape
    out = torch.empty(B, T, dim, device=codes[0].device, dtype=torch.float32)
    err = torch.zeros(1, device=out.device, dtype=torch.int32)
    arr = lambda ts: (C.c_void_p * n)(*[None if t is None else t.data_ptr() for t in ts])
    for c in codes:
        assert c.dtype == torch.int64 and c.is_contiguous()
    _call("rvq", _lib.lib().b2a_snac_from_codes, 1, arr(codes), (C.c_int32 * n)(*strides), n, arr(embs), arr(ws), arr(biases), B, T, bins,
                                              cd, dim, out.data_ptr(), err.data_ptr(), _stream())
    if check and int(err.item()) != 0:
        raise ValueError(f"snac_from_codes: code index out of range [0, {bins})")
    return out


def dac_levels(levels, device) -> torch.Tensor:
    """Device-side table of b2a_dac_level_t from ``levels``: dicts of CUDA tensors {w_in, b_in, cbn, c2, cb, w_out, b_out} (w_in / b_in /
    cbn / c2 None for a decode-only table).  The returned uint8 tensor keeps the table; the caller keeps the tensors it points to."""
    arr = (_lib.DacLevel * len(levels))()
    off = 0
    for a, lv in zip(arr, levels):
        for k in ("w_in", "b_in", "cbn", "c2", "cb", "w_out", "b_out"):
            t = lv.get(k)
            assert t is None or (t.is_cuda and t.is_contiguous() and t.dtype == (torch.float64 if k == "c2" else torch.float32))
            setattr(a, k, _p(t))
        a.cd, a.lat_off = lv["cb"].shape[1], off
        off += a.cd
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(device)


def dac_rvq_encode(z: Optional[torch.Tensor], table: torch.Tensor, n_levels: int, bins: int, lat_ch: int, dim: int, *,
                   latents: Optional[torch.Tensor] = None):
    """DAC residual quantiser, all ``n_levels`` in one launch: z [B, T, dim] fp32 -> (codes int64 [B, n_levels, T], latents [B, lat_ch, T],
    z_q [B, T, dim], loss_part float64 [CTAs] whose sum is the commitment (= codebook) loss).  ``z=None`` with ``latents`` given runs
    from_latents: the search and the out-projections on the given z_e, no residual."""
    if z is not None:
        _chk3(z, "dac_rvq_encode z")
        assert z.is_contiguous() and z.shape[2] == dim
        B, T, _ = z.shape
        latents = torch.empty(B, lat_ch, T, device=z.device, dtype=torch.float32)
    else:
        assert latents.dtype == torch.float32 and latents.is_cuda and latents.is_contiguous() and latents.shape[1] == lat_ch
        B, _, T = latents.shape
    dev = latents.device
    codes = torch.empty(B, n_levels, T, device=dev, dtype=torch.int64)
    zq = torch.empty(B, T, dim, device=dev, dtype=torch.float32)
    loss = torch.empty(-(-B * T // 8), device=dev, dtype=torch.float64)
    _call("rvq", _lib.lib().b2a_dac_rvq_encode, 1, _p(z), dim, B, T, dim, table.data_ptr(), n_levels, bins, lat_ch, codes.data_ptr(),
          latents.data_ptr(), zq.data_ptr(), loss.data_ptr(), _stream())
    return codes, latents, zq, loss


def dac_from_codes(codes: torch.Tensor, table: torch.Tensor, bins: int, lat_ch: int, dim: int, *, want_zp=False, check=True):
    """DAC quantizer.from_codes for the first codes.shape[1] code books: codes int64 [B, nq, T] -> (z_q [B, T, dim], z_p [B, lat_ch, T] or None)."""
    assert codes.dtype == torch.int64 and codes.is_cuda and codes.dim() == 3 and (codes.stride(2) == 1 or codes.shape[2] == 1)
    B, nq, T = codes.shape
    out = torch.empty(B, T, dim, device=codes.device, dtype=torch.float32)
    zp = torch.empty(B, lat_ch, T, device=codes.device, dtype=torch.float32) if want_zp else None
    err = torch.zeros(1, device=codes.device, dtype=torch.int32)
    _call("rvq", _lib.lib().b2a_dac_from_codes, 1, codes.data_ptr(), codes.stride(0), codes.stride(1), B, nq, T, table.data_ptr(), bins, lat_ch,
          dim, out.data_ptr(), _p(zp), err.data_ptr(), _stream())
    if check and int(err.item()) != 0:
        raise ValueError(f"dac_from_codes: code index out of range [0, {bins})")
    return out, zp


# ---------------------------------------------------------------------------------------------------------------- BigVGAN
def aa_snakebeta(x: torch.Tensor, a: torch.Tensor, inv_b: torch.Tensor, f_up: torch.Tensor, f_down: torch.Tensor, *,
                 planes_for: Optional[ConvW] = None):
    """BigVGAN's Activation1d(SnakeBeta) (resample.py:157-177) in one launch: x [B, L, C] -> fp32 [B, L, C], or with ``planes_for`` the
    bf16 ``Planes`` [B, L, planes_for.cin_pad] that ``conv1d(planes, planes_for, ...)`` takes with no prologue.  ``a`` / ``inv_b`` [C]:
    the SnakeBeta gains as the kernel applies them (exp(alpha), 1 / (exp(beta) + 1e-9) for snake_logscale); ``f_up`` / ``f_down``: the
    12 taps of the up- and down-sampling filters."""
    _chk3(x, "aa_snakebeta x")
    B, L, Cc = x.shape
    for name, t, n in (("a", a, Cc), ("inv_b", inv_b, Cc), ("f_up", f_up, f_up.numel()), ("f_down", f_down, f_down.numel())):
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or t.numel() != n:
            raise ValueError(f"aa_snakebeta: {name} must be a contiguous CUDA float32 tensor of {n} values")
    if f_up.numel() != f_down.numel():
        raise ValueError("aa_snakebeta: the up- and down-sampling filters must have the same number of taps")
    if planes_for is not None:
        if planes_for.cin != Cc or planes_for.w_tc is None or planes_for.f16:
            raise ValueError("aa_snakebeta: planes_for must be a bf16 tensor-core conv taking the activation's channels")
        out = _new_planes(B, L, planes_for.cin_pad, x.device)
        out.C = Cc
        _call("aa_act", _lib.lib().b2a_aa_snakebeta, 1, x.data_ptr(), x.stride(0), x.stride(1), B, L, Cc, a.data_ptr(), inv_b.data_ptr(),
              f_up.data_ptr(), f_down.data_ptr(), 2, f_up.numel(), None, 0, 0, out.hi.data_ptr(), _p(out.lo), planes_for.cin_pad, _stream())
        return out
    out = torch.empty(B, L, Cc, device=x.device, dtype=torch.float32)
    _call("aa_act", _lib.lib().b2a_aa_snakebeta, 1, x.data_ptr(), x.stride(0), x.stride(1), B, L, Cc, a.data_ptr(), inv_b.data_ptr(),
          f_up.data_ptr(), f_down.data_ptr(), 2, f_up.numel(), out.data_ptr(), out.stride(0), out.stride(1), None, None, 0, _stream())
    return out


# ---------------------------------------------------------------------------------------------------------------- speaker encoder
def spk_logmel(x: torch.Tensor, window: torch.Tensor, filters: torch.Tensor) -> torch.Tensor:
    """Qwen3-TTS speaker log-mel (qwen3_tts.py:64-121): x [B, n] float32 -> [B, frames, n_mels]; ``window`` [1024], ``filters`` [n_mels, 513]."""
    B, n = x.shape
    assert x.dtype == torch.float32 and x.stride(1) == 1 and window.numel() == 1024 and filters.is_contiguous() and filters.shape[1] == 513
    if n <= 384:
        raise ValueError(f"speaker log-mel: the reflect padding of 384 samples needs more than 384 samples, got {n}")
    frames = 1 + (n + 768 - 1024) // 256
    out = torch.empty(B, frames, filters.shape[0], device=x.device, dtype=torch.float32)
    _call("logmel", _lib.lib().b2a_spk_logmel, 1, x.data_ptr(), x.stride(0), B, n, window.data_ptr(), filters.data_ptr(), filters.shape[0],
          frames, out.data_ptr(), _stream())
    return out


def spk_reflect_pad(x: torch.Tensor, pad: int, cpad: int = 0, planes: int = 2):
    """Reflect "same" padding (speaker_encoder.py:11-26) written as the next conv's operand: ``cpad`` 0 -> fp32 [B, T+2pad, C];
    otherwise the bf16 ``Planes`` [B, T+2pad, cpad] of the tensor-core conv (``planes`` 1: hi only)."""
    _chk3(x, "spk_reflect_pad x")
    B, T, Cc = x.shape
    if pad >= T:
        raise ValueError(f"reflect padding of {pad} rows needs more than {pad} frames, got {T}")
    if cpad:
        pl = Planes(torch.empty(B, T + 2 * pad, cpad, device=x.device, dtype=torch.bfloat16),
                    torch.empty(B, T + 2 * pad, cpad, device=x.device, dtype=torch.bfloat16) if planes == 2 else None, Cc)
        _call("prep", _lib.lib().b2a_spk_reflect_pad, 1, x.data_ptr(), x.stride(0), x.stride(1), B, T, Cc, pad, None, pl.hi.data_ptr(),
              _p(pl.lo), cpad, _stream())
        return pl
    out = torch.empty(B, T + 2 * pad, Cc, device=x.device, dtype=torch.float32)
    _call("prep", _lib.lib().b2a_spk_reflect_pad, 1, x.data_ptr(), x.stride(0), x.stride(1), B, T, Cc, pad, out.data_ptr(), None, None, 0,
          _stream())
    return out


SPK_RES2NET_TILE = 32      # output rows per CTA of the Res2Net chain (halo (scale-1)*pad rows per side is recomputed)


def spk_res2net(y: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, scale: int, dilation: int, out=None, tile: int = 0) -> torch.Tensor:
    """Res2NetBlock (speaker_encoder.py:60-101) in one launch: y [B, T, scale*C] -> [B, T, scale*C]; ``w`` [scale-1, K, C, C]
    (stage, tap, in, out), ``bias`` [scale-1, C]."""
    _chk3(y, "spk_res2net y")
    B, T, CC = y.shape
    S1, K, Cc, _ = w.shape
    assert S1 == scale - 1 and CC == scale * Cc and w.is_contiguous() and bias.is_contiguous() and w.dtype == torch.float32
    pad = (K - 1) * dilation // 2
    if pad >= T:
        raise ValueError(f"Res2Net: reflect padding of {pad} rows needs more than {pad} frames, got {T}")
    if out is None:
        out = torch.empty(B, T, CC, device=y.device, dtype=torch.float32)
    _chk3(out, "spk_res2net out")
    _call("other", _lib.lib().b2a_spk_res2net, 1, y.data_ptr(), y.stride(0), y.stride(1), out.data_ptr(), out.stride(0), out.stride(1),
          w.data_ptr(), bias.data_ptr(), B, T, Cc, scale, K, dilation, tile or SPK_RES2NET_TILE, _stream())
    return out


def spk_channel_stats(x: torch.Tensor, with_std: bool, eps: float = 1e-12, out=None) -> torch.Tensor:
    """Per-channel mean over T of x [B, T, C] -> [B, C], or [B, 2C] = (mean | sqrt(var + eps)) with ``with_std``; fixed order."""
    _chk3(x, "spk_channel_stats x")
    B, T, Cc = x.shape
    if out is None:
        out = torch.empty(B, (2 if with_std else 1) * Cc, device=x.device, dtype=torch.float32)
    _call("other", _lib.lib().b2a_spk_channel_stats, 1, x.data_ptr(), x.stride(0), x.stride(1), B, T, Cc, int(with_std), eps,
          out.data_ptr(), out.stride(0), _stream())
    return out


def spk_se_gate(mean: torch.Tensor, w1, b1, w2, b2) -> torch.Tensor:
    """sigmoid(w2 relu(w1 mean + b1) + b2) per item: mean [B, C], w1 [S, C], w2 [C, S] -> gate [B, C]."""
    B, Cc = mean.shape
    S = w1.shape[0]
    assert mean.stride(1) == 1 and w1.is_contiguous() and w2.is_contiguous() and tuple(w2.shape) == (Cc, S)
    gate = torch.empty(B, Cc, device=mean.device, dtype=torch.float32)
    _call("other", _lib.lib().b2a_spk_se_gate, 1, mean.data_ptr(), mean.stride(0), B, Cc, S, w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
          b2.data_ptr(), gate.data_ptr(), _stream())
    return gate


def spk_se_apply(y: torch.Tensor, gate: torch.Tensor, res: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out = y * gate[b, c] + res (all [B, T, C] row-strided views)."""
    for t, n in ((y, "y"), (res, "res"), (out, "out")):
        _chk3(t, "spk_se_apply " + n)
    B, T, Cc = y.shape
    assert res.shape == y.shape and out.shape == y.shape and gate.is_contiguous() and tuple(gate.shape) == (B, Cc)
    _call("other", _lib.lib().b2a_spk_se_apply, 1, y.data_ptr(), y.stride(0), y.stride(1), gate.data_ptr(), res.data_ptr(), res.stride(0),
          res.stride(1), out.data_ptr(), out.stride(0), out.stride(1), B, T, Cc, _stream())
    return out


def spk_gemv(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: int = 0) -> torch.Tensor:
    """y[b] = act(w x[b] + bias): x [B, K] (unit column stride), w [N, K] fp32 (row-strided) -> [B, N]."""
    B, K = x.shape
    N = w.shape[0]
    assert x.stride(1) == 1 and w.stride(1) == 1 and w.shape[1] == K and x.dtype == w.dtype == torch.float32
    y = torch.empty(B, N, device=x.device, dtype=torch.float32)
    _call("gemv", _lib.lib().b2a_spk_gemv, 1, x.data_ptr(), x.stride(0), B, K, w.data_ptr(), w.stride(0), N, _p(bias), act, y.data_ptr(),
          y.stride(0), _stream())
    return y


def spk_asp_act(h: torch.Tensor, cb: torch.Tensor) -> torch.Tensor:
    """In place: h = tanh(relu(h + cb[b])), h [B, T, A], cb [B, A]."""
    _chk3(h, "spk_asp_act h")
    B, T, A = h.shape
    assert cb.is_contiguous() and tuple(cb.shape) == (B, A)
    _call("other", _lib.lib().b2a_spk_asp_act, 1, h.data_ptr(), h.stride(0), h.stride(1), cb.data_ptr(), B, T, A, _stream())
    return h


def spk_asp_pool(logits: torch.Tensor, x: torch.Tensor, eps: float = 1e-12) -> torch.Tensor:
    """Softmax over time per channel + weighted mean / std (speaker_encoder.py:208-216): logits, x [B, T, C] -> [B, 2C] (mean | std)."""
    _chk3(logits, "spk_asp_pool logits")
    _chk3(x, "spk_asp_pool x")
    B, T, Cc = x.shape
    assert logits.shape == x.shape
    out = torch.empty(B, 2 * Cc, device=x.device, dtype=torch.float32)
    _call("other", _lib.lib().b2a_spk_asp_pool, 1, logits.data_ptr(), logits.stride(0), logits.stride(1), x.data_ptr(), x.stride(0),
          x.stride(1), B, T, Cc, eps, out.data_ptr(), out.stride(0), _stream())
    return out


# ---------------------------------------------------------------------------------------------------------------- Vocos
def vocos_dwnorm(x: torch.Tensor, dw: Optional[ConvW], w: Optional[torch.Tensor], b: Optional[torch.Tensor], *, ada: Optional[torch.Tensor] = None,
                 eps: float = 1e-6, fp32: bool = True, planes: bool = False):
    """Vocos's ConvNeXt dwconv + LayerNorm / AdaLayerNorm (vocos.py:183-187) in one launch; ``dw`` None: the norm alone (the backbone's
    norm and final_layer_norm).  x [B, L, C]; ``dw`` a depthwise ``pack_conv`` (odd K <= 15); affine ``w`` / ``b`` (either may be None),
    or ``ada`` [B, 2C] rows (scale | shift, row stride free) applied as scale v + shift.  Returns fp32 [B, L, C] (``fp32``), the next
    GEMM's bf16 ``Planes`` [B, L, C] (``planes``, C % 64 == 0), or (y, planes) with both."""
    _chk3(x, "vocos_dwnorm x")
    B, L, Cc = x.shape
    if not (fp32 or planes):
        raise ValueError("vocos_dwnorm: ask for fp32 rows, planes or both")
    if dw is not None and (dw.groups != Cc or dw.cin != Cc or dw.K % 2 == 0 or dw.K > 15):
        raise ValueError("vocos_dwnorm: dw must be a depthwise conv over x's channels with an odd number of taps <= 15")
    if ada is not None and (ada.dim() != 2 or ada.shape[0] != B or ada.shape[1] != 2 * Cc or ada.stride(1) != 1 or ada.dtype != torch.float32):
        raise ValueError(f"vocos_dwnorm: ada must be float32 [B, 2C] = {(B, 2 * Cc)} rows with unit column stride")
    y = torch.empty(B, L, Cc, device=x.device, dtype=torch.float32) if fp32 else None
    pl = _new_planes(B, L, Cc, x.device) if planes else None
    _call("vocos_norm", _lib.lib().b2a_vocos_dwnorm, 1, x.data_ptr(), x.stride(0), x.stride(1), B, L, Cc,
          None if dw is None else dw.w.data_ptr(), None if dw is None else _p(dw.bias), 0 if dw is None else dw.K, _p(w), _p(b), _p(ada),
          0 if ada is None else ada.stride(0), float(eps), _p(y), 0 if y is None else y.stride(0), 0 if y is None else y.stride(1),
          None if pl is None else pl.hi.data_ptr(), None if pl is None else _p(pl.lo), _stream())
    if fp32 and planes:
        return y, pl
    return y if fp32 else pl


def vocos_istft_head(h: torch.Tensor, n_fft: int, hop: int, window: torch.Tensor) -> torch.Tensor:
    """ISTFTHead after its linear (vocos.py:126-140, dsp.py:436-513): h [B, T, ld >= n_fft + 2] (log-magnitude | phase columns; any
    columns beyond n_fft + 2 are ignored) -> waveform [B, (T - 1) * hop].  ``window``: the symmetric Hann window [n_fft]."""
    _chk3(h, "vocos_istft_head h")
    B, T, ld = h.shape
    if ld < n_fft + 2 or window.numel() != n_fft or window.dtype != torch.float32 or not window.is_contiguous():
        raise ValueError(f"vocos_istft_head: needs h rows of >= {n_fft + 2} columns and a contiguous float32 window of {n_fft}")
    out = torch.empty(B, (T - 1) * hop, device=h.device, dtype=torch.float32)
    if T > 1:
        _call("vocos_head", _lib.lib().b2a_vocos_istft_head, 1, h.data_ptr(), h.stride(0), h.stride(1), B, T, n_fft, hop, window.data_ptr(),
              out.data_ptr(), out.stride(0), _stream())
    return out


def vocos_logmel(x: torch.Tensor, window: torch.Tensor, filters: torch.Tensor) -> torch.Tensor:
    """Vocos's log-mel (mel.py:8-33) at n_fft 1024 / hop 256: x [B, n] float32 -> [B, n // 256, n_mels]; ``window`` the symmetric Hann
    window [1024], ``filters`` HTK mel filters [n_mels, 513]."""
    B, n = x.shape
    if x.dtype != torch.float32 or x.stride(1) != 1 or window.numel() != 1024 or not filters.is_contiguous() or filters.shape[1] != 513:
        raise ValueError("vocos_logmel: x [B, n] float32 with unit stride, a 1024-sample window and [n_mels, 513] filters")
    if n <= 512:
        raise ValueError(f"vocos log-mel: the reflect padding of 512 samples needs more than 512 samples, got {n}")
    frames = n // 256
    out = torch.empty(B, frames, filters.shape[0], device=x.device, dtype=torch.float32)
    _call("logmel", _lib.lib().b2a_vocos_logmel, 1, x.data_ptr(), x.stride(0), B, n, window.data_ptr(), filters.data_ptr(), filters.shape[0],
          frames, out.data_ptr(), _stream())
    return out


# ---------------------------------------------------------------------------------------------------------------- EnCodec
def encodec_lstm(xproj: torch.Tensor, wh: torch.Tensor, err: torch.Tensor, skip: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One unidirectional LSTM layer (encodec.py:89-169): xproj [R, T, 4H] (x Wx^T + bias), wh [4H, H] -> h [R, T, H] (+ ``skip``).
    ``err``: int32 [1] on the device, set to 1 by a step that waited more than 10 s (checked by the caller)."""
    R, T, g4 = xproj.shape
    H = g4 // 4
    for name, t in (("xproj", xproj), ("wh", wh)) + ((("skip", skip),) if skip is not None else ()):
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"encodec_lstm: {name} must be a contiguous CUDA float32 tensor")
    if tuple(wh.shape) != (4 * H, H) or (skip is not None and tuple(skip.shape) != (R, T, H)):
        raise ValueError(f"encodec_lstm: wh must be [{4 * H}, {H}] and skip [{R}, {T}, {H}]")
    out = torch.empty(R, T, H, device=xproj.device, dtype=torch.float32)
    _call("lstm", _lib.lib().b2a_encodec_lstm, 1, xproj.data_ptr(), wh.data_ptr(), _p(skip), out.data_ptr(), R, T, H, err.data_ptr(), _stream())
    return out


def encodec_pad(x: torch.Tensor, pad_left: int, pad_right: int, *, reflect: bool = True, coeffs=None, elu: bool = False,
                res: Optional[torch.Tensor] = None) -> torch.Tensor:
    """EncodecConv1d's input side: x [B, T, C] (row-strided views allowed) -> fp32 [B, pad_left + T + pad_right, C]; each source value
    gets the GroupNorm ``coeffs`` = (scale, shift) [B, C] and then ELU first; ``res`` [B, T, C] is added last (no padding then)."""
    _chk3(x, "encodec_pad x")
    B, T, Cc = x.shape
    if reflect and max(pad_left, pad_right) >= T:
        raise ValueError(f"EnCodec reflect padding ({pad_left}, {pad_right}) needs more than {max(pad_left, pad_right)} frames, got {T}")
    out = torch.empty(B, pad_left + T + pad_right, Cc, device=x.device, dtype=torch.float32)
    sc, sh = coeffs if coeffs is not None else (None, None)
    if res is not None:
        _chk3(res, "encodec_pad res")
    _call("prep", _lib.lib().b2a_encodec_pad, 1, x.data_ptr(), x.stride(0), x.stride(1), B, T, Cc, pad_left, pad_right, int(reflect), _p(sc),
          _p(sh), int(elu), _p(res), 0 if res is None else res.stride(0), 0 if res is None else res.stride(1), out.data_ptr(), out.stride(0),
          out.stride(1), _stream())
    return out


def encodec_gn_coeffs(x: torch.Tensor, gamma: Optional[torch.Tensor], beta: Optional[torch.Tensor], eps: float = 1e-5):
    """GroupNorm(1, C) of x [B, T, C] folded with its affine -> (scale, shift) [B, C] float32 for ``encodec_pad(coeffs=)``."""
    _chk3(x, "encodec_gn_coeffs x")
    B, T, Cc = x.shape
    scale = torch.empty(B, Cc, device=x.device, dtype=torch.float32)
    shift = torch.empty(B, Cc, device=x.device, dtype=torch.float32)
    ws = _workspace(_lib.lib().b2a_encodec_gn_ws_bytes(B), x.device)
    _call("norm", _lib.lib().b2a_encodec_gn_coeffs, 2, x.data_ptr(), x.stride(0), x.stride(1), B, T, Cc, _p(gamma), _p(beta), eps,
          scale.data_ptr(), shift.data_ptr(), ws.data_ptr(), _stream())
    return scale, shift


def encodec_normalize(x: torch.Tensor, mask: Optional[torch.Tensor]):
    """Per chunk row of x [R, L, C]: (x * mask / scale, scale [R]) with scale = RMS of the masked mono mix + 1e-8 (encodec.py:574-579)."""
    _chk3(x, "encodec_normalize x")
    R, L, Cc = x.shape
    if mask is not None:
        assert mask.dtype in (torch.bool, torch.uint8) and tuple(mask.shape) == (R, L) and mask.stride(1) == 1
    y = torch.empty(R, L, Cc, device=x.device, dtype=torch.float32)
    scale = torch.empty(R, device=x.device, dtype=torch.float32)
    _call("other", _lib.lib().b2a_encodec_normalize, 1, x.data_ptr(), x.stride(0), x.stride(1), R, L, Cc, _p(mask),
          0 if mask is None else mask.stride(0), y.data_ptr(), scale.data_ptr(), _stream())
    return y, scale


def encodec_ola(frames: torch.Tensor, B: int, scale: Optional[torch.Tensor], stride: int, t_out: int) -> torch.Tensor:
    """Encodec._linear_overlap_add (encodec.py:654-677) of chunk decodes frames [N * B, L, C] (chunk-major), each times scale [N * B]
    (or None), truncated to ``t_out`` samples -> [B, t_out, C]."""
    NB, L, Cc = frames.shape
    assert frames.dtype == torch.float32 and frames.is_contiguous() and NB % B == 0
    assert scale is None or (scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == NB)
    out = torch.empty(B, t_out, Cc, device=frames.device, dtype=torch.float32)
    _call("other", _lib.lib().b2a_encodec_ola, 1, frames.data_ptr(), NB // B, B, L, Cc, _p(scale), stride, t_out, out.data_ptr(), _stream())
    return out


# ---------------------------------------------------------------------------------------------------------------- Soprano
def lm_sample_mlx(logits: torch.Tensor, *, temperature: float, top_p: float, u: Optional[torch.Tensor] = None,
                  step_dev: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, hist: Optional[torch.Tensor] = None,
                  finished: Optional[torch.Tensor] = None, stop_ids=()) -> torch.Tensor:
    """mlx-lm's ``make_sampler(temperature, top_p)`` on raw logits [B, V] (row stride free, unit column stride) -> int64 tokens [B]
    (b2a_lm_sample_mlx).  ``u`` float32 [B, n]: the draw of row b at step s is u[b, s], s = ``step_dev`` (int32 [1]) or 0.  ``hist`` int64
    [B, n] receives the token at column s.  ``finished`` uint8 [B]: rows set there write nothing; a row drawing one of ``stop_ids`` (at most
    two) is set."""
    B, V = logits.shape
    if logits.dtype != torch.float32 or not logits.is_cuda or logits.stride(1) != 1:
        raise ValueError("lm_sample_mlx: logits must be a CUDA float32 [B, V] tensor with unit column stride")
    if temperature > 0 and (u is None or u.dtype != torch.float32 or u.dim() != 2 or u.shape[0] != B or u.stride(1) != 1):
        raise ValueError("lm_sample_mlx: temperature > 0 needs float32 uniforms u [B, steps]")
    stops = [int(s) for s in stop_ids if s is not None]
    if len(stops) > 2:
        raise ValueError("lm_sample_mlx: at most two stop ids")
    stops += [-1] * (2 - len(stops))
    if out is None:
        out = torch.empty(B, device=logits.device, dtype=torch.int64)
    assert out.dtype == torch.int64 and out.is_contiguous() and out.numel() == B
    assert step_dev is None or (step_dev.dtype == torch.int32 and step_dev.is_cuda)
    assert hist is None or (hist.dtype == torch.int64 and hist.dim() == 2 and hist.stride(1) == 1 and hist.shape[0] == B)
    assert finished is None or (finished.dtype == torch.uint8 and finished.is_contiguous() and finished.numel() == B)
    _call("sampler", _lib.lib().b2a_lm_sample_mlx, 1, logits.data_ptr(), logits.stride(0), B, V, float(temperature), float(top_p), _p(u),
          0 if u is None else u.stride(0), _p(step_dev), out.data_ptr(), _p(hist), 0 if hist is None else hist.stride(0), _p(finished),
          stops[0], stops[1], _stream())
    return out


def soprano_upsample(x: torch.Tensor, up: int, *, planes_for: Optional[ConvW] = None):
    """SopranoDecoder's align-corners linear up-sampling (decoder.py:102-112): x [B, L, H] -> fp32 [B, up (L - 1) + 1, H], or with
    ``planes_for`` the bf16 ``Planes`` of that tensor-core conv (``conv1d(planes, planes_for, ...)`` takes them with no prologue)."""
    _chk3(x, "soprano_upsample x")
    B, L, H = x.shape
    Lo = up * (L - 1) + 1
    if planes_for is not None:
        if planes_for.cin != H or planes_for.w_tc is None or planes_for.f16:
            raise ValueError("soprano_upsample: planes_for must be a bf16 tensor-core conv taking the hidden width")
        out = _new_planes(B, Lo, planes_for.cin_pad, x.device)
        out.C = H
        _call("other", _lib.lib().b2a_soprano_upsample, 1, x.data_ptr(), x.stride(0), x.stride(1), B, L, H, up, None, 0, 0,
              out.hi.data_ptr(), _p(out.lo), planes_for.cin_pad, _stream())
        return out
    out = torch.empty(B, Lo, H, device=x.device, dtype=torch.float32)
    _call("other", _lib.lib().b2a_soprano_upsample, 1, x.data_ptr(), x.stride(0), x.stride(1), B, L, H, up, out.data_ptr(), out.stride(0),
          out.stride(1), None, None, 0, _stream())
    return out


def store_rows_at(src: torch.Tensor, dst: torch.Tensor, idx_dev: torch.Tensor, add: int = 0) -> None:
    """dst[b, idx_dev[0] + add, :] = src[b, :] for src [B, H] and dst [B, T, H] float32 (rows outside [0, T) are skipped)."""
    B, H = src.shape
    assert src.dtype == dst.dtype == torch.float32 and src.stride(1) == 1 and dst.stride(2) == 1 and dst.shape[0] == B and dst.shape[2] == H
    assert idx_dev.dtype == torch.int32 and idx_dev.is_cuda
    _call("other", _lib.lib().b2a_soprano_store_rows, 1, src.data_ptr(), src.stride(0), B, H, dst.data_ptr(), dst.stride(0), dst.stride(1),
          idx_dev.data_ptr(), int(add), dst.shape[1], _stream())
