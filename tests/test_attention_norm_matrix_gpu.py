"""Transformer building blocks (csrc/attn.cu: b2a_attention, b2a_rope; csrc/attn_tc.cu: b2a_attention_tc; csrc/norm.cu: b2a_layernorm,
b2a_adain_coeffs, b2a_channel_stats, b2a_coeffs_from_stats) against float64 on every dispatch branch.  Every Whisper encoder and decoder
layer runs them, as do Kokoro's text side, the Mimi and SNAC transformers and the Qwen3 speech-tokenizer transformer.

Where each kernel and branch is run:
- ``ops.attention`` sends D = 64, H == Hkv, no ``k_len``, Tk >= 64 to the tensor-core path (``ATTN_MODE`` "tc": attn_tc_prep_qk_kernel
  twice, attn_tc_prep_vt_kernel, attn_tc_kernel; 4 launches) and everything else to attn_kernel<64> (1 launch).  Every attention test
  forces both modes; the ids say which kernel ran (``tc`` / ``cuda``), and ``test_attention_dispatch`` asserts it from ``ops.LAUNCHES``
  at Tk = 63 | 64 | 65 | 127 | 128 | 129 and Tq = 1 .. 129 (one and two 128-query CTAs).
- Masking: ``test_attention_masks[*-causal-qoff]`` (the Whisper decoder's prefill against a cache), ``[*-window-skip-tile]`` (the first
  key tiles of both query tiles are skipped: t_lo = 3 and 5), ``[*-window-ge-Tk]``, ``[*-window-mid-tile]`` (windows that start inside
  a key tile), ``[*-window-qoff]``.  GQA and ``k_len`` reach only attn_kernel (``test_attention_gqa``, ``test_attention_k_len``).
- attn_tc_kernel also in ``test_attention_strided_views[tc-*]`` and ``test_attention_operand_magnitude[tc-*]``; attn_kernel in the
  ``cuda`` ids of the same tests.
- rope_kernel: every ``test_rope_vs_float64`` case; ``[*-h16-d128-*]`` has more elements than one grid (132 x 16 CTAs of 256 threads)
  and takes the grid-stride loop.
- b2a_layernorm (norm.cu host rule: C % 4 == 0, C <= 1024 and 16-byte aligned rows -> layernorm_vec_kernel<4> for C <= 512, else <8>;
  anything else -> the scalar layernorm_kernel): the ids of ``test_layernorm_vs_float64`` name the kernel (``vec4-C4``, ``vec4-C128``,
  ``vec4-C508``, ``vec4-C512``, ``vec8-C516``, ``vec8-C768``, ``vec8-C1024``, ``scalar-C1028``, ``scalar-C1280``, ``scalar-C2048``,
  ``scalar-C130``, ``scalar-C6``, ``scalar-C512-ld514``); ``test_layernorm_dispatch_table_reaches_every_kernel`` checks the table.
  The emitted bf16 planes (vector kernels only): ``test_layernorm_planes``.  Zero rows: ``test_layernorm_zero_rows``.
- adain_partial_kernel + adain_final_kernel: ``test_adain_coeffs_vs_float64`` (L = 1 .. 1000: one to four 256-row chunks);
  channel_stats_kernel + coeffs_from_stats_kernel: ``test_channel_stats_and_coeffs`` (1 to 4 destinations).

Tolerances, all max |y - ref| / max |ref| against float64 on the CPU:
- Attention 2e-5.  attn_kernel is fp32 throughout (scores as two 32-term fma chains, expf, p v sums); attn_tc_kernel multiplies fp16
  hi / lo splits of Q, K, V and P with three products per MMA, fp32-grade while the operands stay inside fp16's range (the operand
  envelope below).  Scores are rounded to fp32 in both kernels, about |s| 2^-24 each, so the error grows with |q| |k|: with q or k
  at rms 2^8 (scores of std ~250, softmax near one-hot) both kernels sit at 1.5e-5 .. 1.9e-5 on an H100 80GB HBM3 (700 W), the
  largest use of a bound in this file.  Negative controls, on both kernels: the causal bound one key short and one key long, the
  window one key short and long, GQA's head map h % Hkv instead of h / (H / Hkv).
- Operand envelope of attn_tc_kernel: the lo plane of an fp16 split is rounded to fp16's subnormal spacing 2^-24 (6e-8).  For V of
  rms 1e-4 the lo parts (~2^-12 of an element, 2e-8) fall below it, so hi + lo keep little more than hi's 11 bits (1.4e-4 on an
  H100 80GB HBM3 at 700 W).  There the kernel must stay within 3x the error of ``tc_emulation`` (the same split emulated in
  float64); attn_kernel must still meet 2e-5.  ``test_tc_emulation_envelope`` (CPU) holds the emulation within the bound at rms
  2^-10, the envelope's edge.
  Negative control: the emulation with hi planes only (one product) is more than 5x the bound away from the kernel at rms 1.
- Rotary 1e-6.  The angles and their sin / cos are float64; the two products and the sum of the rotation are float64 rounded once to
  fp32 (2^-24 = 6e-8 of each element).  Negative control at offset 20000: angles computed in float32 (one ulp of 20000 rad is 2^-9).
- LayerNorm / RMSNorm 1e-5.  fp32 sums over C <= 2048 terms (mean, then the centred sum of squares) and rsqrtf: a few 2^-24 times
  sqrt(C) of the output scale, also with a row mean 50 and std 3.  Negative controls: the unbiased variance for LayerNorm (1 / 2C of
  the output) and LayerNorm instead of RMSNorm.  Emitted planes are bit-identical to ``ops.prep_bf16`` of the fp32 output.
- AdaIN coefficients 1e-5: float64 partial sums, one rounding to fp32 of scale and shift.  Negative control (mean 1e3, std 0.1):
  E[x^2] - mean^2 in float32.  The binned statistics path must agree with ``adain_coeffs`` within 1e-6 (both are float64 sums rounded
  to fp32 once; the bins keep 48 bits of every chunk sum) and be bit-reproducible.

Output columns and rows outside every written view hold a sentinel that must survive.
"""
import ctypes as C
import math

import pytest
import torch

from oracle import nn as ON

gpu = pytest.mark.gpu
DEV = "cuda:0"
TOL_ATTN = 2e-5
TOL_ROPE = 1e-6
TOL_LN = 1e-5
TOL_ADAIN = 1e-5
TOL_STATS_AGREE = 1e-6
NEG = 5                      # every negative control exceeds NEG x its bound
SENTINEL = -1234.5
LOG2E = 1.4426950408889634
MODES = ["tc", "cuda"]


def _rand(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_err(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


# ------------------------------------------------------------------------------------------------------------ float64 references
def attn_ref(q, k, v, H, Hkv, scale, causal=False, q_offset=0, window=0, k_len=None, bound_shift=0, head_map="group"):
    """softmax(scale q k^T + mask) v on q [B,Tq,H D], k / v [B,Tk,Hkv D].  Key j is visible to query i when j < min(k_len[b], Tk) and,
    with ``causal``, j <= i + q_offset + bound_shift and (window > 0) i + q_offset - j < window.  A query with no visible key gives
    zeros.  ``head_map`` "group" is the reference's head repeat (h / (H / Hkv)); "mod" (h % Hkv) and ``bound_shift`` are negative
    controls only."""
    B, Tq, _ = q.shape
    Tk = k.shape[1]
    D = q.shape[2] // H
    qh = q.double().reshape(B, Tq, H, D).transpose(1, 2)
    idx = torch.arange(H) // (H // Hkv) if head_map == "group" else torch.arange(H) % Hkv
    kh = k.double().reshape(B, Tk, Hkv, D).transpose(1, 2)[:, idx]
    vh = v.double().reshape(B, Tk, Hkv, D).transpose(1, 2)[:, idx]
    i, j = torch.arange(Tq)[:, None] + q_offset, torch.arange(Tk)[None, :]
    ok = torch.ones(B, Tq, Tk, dtype=torch.bool)
    if causal:
        ok = ok & (j <= i + bound_shift)
        if window > 0:
            ok = ok & (i - j < window)
    if k_len is not None:
        ok = ok & (j[None] < torch.tensor(k_len)[:, None, None])
    ok = ok[:, None]
    p = torch.softmax((qh @ kh.transpose(-1, -2) * scale).masked_fill(~ok, float("-inf")), dim=-1)
    p = torch.where(ok.any(-1, keepdim=True), p, torch.zeros_like(p))
    return (p @ vh).transpose(1, 2).reshape(B, Tq, H * D)


def tc_emulation(q, k, v, scale, planes=2):
    """attn_tc_kernel's arithmetic in float64 for non-causal attention with H == Hkv (q, k, v [B,T,H 64]): q * fp32(scale log2 e), k
    and v split in fp32 into fp16 hi + lo planes; S = Qh Kh + Ql Kh + Qh Kl summed exactly; P = exp2(S - row max) in fp32 split the
    same way; O = (Ph Vh + Pl Vh + Ph Vl) / sum P.  ``planes=1``: hi planes only, one product per MMA (a negative control).  The kernel
    rescales P by a running maximum per key tile, which moves no P across fp16's normal range at these sizes."""
    B, Tq, HD = q.shape
    Tk, H = k.shape[1], HD // 64

    def split(x):
        hi = x.half().float()
        lo = (x - hi).half().float() if planes == 2 else torch.zeros_like(hi)
        return hi.double(), lo.double()

    def heads(x, T):
        return x.reshape(B, T, H, 64).transpose(1, 2)
    mul = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    qh, ql = split(heads(q.float() * mul, Tq))
    kh, kl = split(heads(k.float(), Tk))
    vh, vl = split(heads(v.float(), Tk))
    s = qh @ kh.transpose(-1, -2) + ql @ kh.transpose(-1, -2) + qh @ kl.transpose(-1, -2)
    p = torch.exp2(s - s.amax(-1, keepdim=True)).float()
    ph, pl = split(p)
    o = (ph @ vh + pl @ vh + ph @ vl) / p.double().sum(-1, keepdim=True)
    return o.transpose(1, 2).reshape(B, Tq, HD)


def rope_ref(x, H, offset, base, traditional, angle_dtype=torch.float64):
    """``ops.rope_`` on x [B,T,H D]: rotate the pairs (2i, 2i+1) (traditional) or (i, i + D/2) by (t + offset) base^(-2i/D).  The angles
    are computed in ``angle_dtype`` (float32 for a negative control only), sin / cos and the rotation in float64."""
    B, T, HD = x.shape
    D, half = HD // H, HD // H // 2
    pos = torch.arange(offset, offset + T, dtype=angle_dtype)
    inv = torch.exp(-torch.arange(0, half, dtype=angle_dtype) * (math.log(base) / half))
    ang = (pos[:, None] * inv[None, :]).double()
    c, s = torch.cos(ang), torch.sin(ang)
    xh = x.double().reshape(B, T, H, D)
    a, b = (xh[..., 0::2], xh[..., 1::2]) if traditional else (xh[..., :half], xh[..., half:])
    c, s = c[None, :, None], s[None, :, None]
    ra, rb = a * c - b * s, a * s + b * c
    out = torch.stack([ra, rb], -1).reshape(B, T, H, D) if traditional else torch.cat([ra, rb], -1)
    return out.reshape(B, T, HD)


def ln_ref(x, w=None, b=None, eps=1e-5, res=None, ada=None, rms=False, slope=None, unbiased=False):
    """``ops.layernorm`` on rows x [R, C]: LayerNorm (or RMSNorm) of x + res, then (1 + ada[:C]) y + ada[C:] or y w + b, then LeakyReLU
    of ``slope``.  ``unbiased`` (n - 1 variance) is a negative control only."""
    v = x.double() + (0 if res is None else res.double())
    Cc = v.shape[-1]
    if rms:
        y = ON.rms_norm(v, torch.ones(Cc, dtype=torch.float64), eps)
    elif unbiased:
        y = (v - v.mean(-1, keepdim=True)) / torch.sqrt(v.var(-1, unbiased=True, keepdim=True) + eps)
    else:
        y = ON.layer_norm(v, eps=eps)
    if ada is not None:
        y = (1 + ada.double()[:Cc]) * y + ada.double()[Cc:]
    else:
        if w is not None:
            y = y * w.double()
        if b is not None:
            y = y + b.double()
    return y if slope is None else ON.leaky_relu(y, slope)


def adain_ref(x, gb, eps=1e-5, stats_dtype=torch.float64):
    """InstanceNorm statistics over L of x [B,L,C] folded with AdaIN (gamma | beta) [B,2C]: scale = (1 + gamma) / sqrt(var + eps),
    shift = beta - scale mean.  ``stats_dtype`` float32 computes var = E[x^2] - mean^2 in float32 (a negative control only)."""
    xs = x.to(stats_dtype)
    mean = xs.mean(1)
    var = ((xs * xs).mean(1) - mean * mean).clamp(min=0).double()
    mean = mean.double()
    Cc = x.shape[2]
    g, be = (1.0, 0.0) if gb is None else (1 + gb.double()[:, :Cc], gb.double()[:, Cc:])
    sc = g / torch.sqrt(var + eps)
    return sc, be - sc * mean


# ------------------------------------------------------------------------------------------------------------ CPU: the references
def test_attn_ref_equals_oracle_sdpa():
    """attn_ref is the oracle's SDPA with the reference's causal + sliding-window mask and its GQA head repeat; k_len masks the keys past
    it as an additive -inf does."""
    B, Tq, Tk, H, Hkv, D, off, win = 2, 7, 19, 4, 2, 16, 12, 9
    q, k, v = _rand(B, Tq, H * D, seed=1), _rand(B, Tk, Hkv * D, seed=2), _rand(B, Tk, Hkv * D, seed=3)
    i, j = torch.arange(Tq)[:, None] + off, torch.arange(Tk)[None, :]
    mask = torch.where((j <= i) & (i - j < win), 0.0, float("-inf")).double()
    sh = (lambda t, h: t.double().reshape(B, -1, h, D).transpose(1, 2))
    want = ON.sdpa(sh(q, H), sh(k, Hkv), sh(v, Hkv), 0.3, mask).transpose(1, 2).reshape(B, Tq, H * D)
    assert rel_err(attn_ref(q, k, v, H, Hkv, 0.3, True, off, win), want) < 1e-13
    kl = [15, 40]                                          # row 0: every query still sees a key
    m2 = mask[None, None].repeat(B, 1, 1, 1)
    m2[0, :, :, 15:] = float("-inf")
    want = ON.sdpa(sh(q, H), sh(k, Hkv), sh(v, Hkv), 0.3, m2).transpose(1, 2).reshape(B, Tq, H * D)
    got = attn_ref(q, k, v, H, Hkv, 0.3, True, off, win, k_len=kl)
    assert rel_err(got[:1], want[:1]) < 1e-13 and rel_err(got[1:], want[1:]) < 1e-13


def test_tc_emulation_envelope():
    """On the inputs of ``test_attention_small_v_envelope``: the emulated split meets the attention bound at rms 1 and with q, k or v
    at rms 2^-10 (the edge of the envelope the header documents); hi planes alone do not, and v of rms 1e-4 leaves the envelope."""
    q, k, v = _qkv(1, 300, 300, 2, 2, seed=80, scale=1.0)

    def err(q, k, v, planes=2):
        return rel_err(tc_emulation(q, k, v, 0.125, planes), attn_ref(q, k, v, 2, 2, 0.125))
    s = 2.0 ** -10
    assert err(q, k, v) < TOL_ATTN / 4
    assert max(err(q * s, k, v), err(q, k * s, v), err(q, k, v * s)) < TOL_ATTN
    assert err(q, k, v, planes=1) > NEG * TOL_ATTN and err(q, k, v * 1e-4) > NEG * TOL_ATTN


def test_rope_ref_equals_oracle():
    x = _rand(2, 9, 3 * 32, seed=7)
    for trad, fn in ((True, ON.rope_traditional), (False, ON.rope_half)):
        want = fn(x.double().reshape(2, 9, 3, 32).transpose(1, 2), 5, 1e4).transpose(1, 2).reshape(2, 9, 96)
        assert rel_err(rope_ref(x, 3, 5, 1e4, trad), want) < 1e-14


def test_ln_and_adain_refs_equal_the_oracle():
    x, r, w, b = _rand(5, 24, seed=8), _rand(5, 24, seed=9), _rand(24, seed=10), _rand(24, seed=11)
    assert rel_err(ln_ref(x, w, b, 1e-5, res=r), ON.layer_norm(x.double() + r.double(), w.double(), b.double(), 1e-5)) < 1e-14
    assert rel_err(ln_ref(x, w, None, 1e-6, rms=True), ON.rms_norm(x.double(), w.double(), 1e-6)) < 1e-14
    xb = _rand(2, 40, 6, seed=12) * 3 + 5
    sc, sh = adain_ref(xb, None)
    y = xb.double() * sc[:, None] + sh[:, None]
    assert y.mean(1).abs().max() < 1e-12 and (y.var(1, unbiased=False) - 1).abs().max() < 1e-5


# ------------------------------------------------------------------------------------------------------------ attention
def _attn(mode, q, k, v, **kw):
    """``ops.attention`` with ATTN_MODE forced to ``mode``; returns (out, kernel launches)."""
    from mlx_audio_b200 import ops
    old = ops.ATTN_MODE[0]
    ops.ATTN_MODE[0] = mode
    try:
        n0 = ops.LAUNCHES[0]
        y = ops.attention(q, k, v, **kw)
        return y, ops.LAUNCHES[0] - n0
    finally:
        ops.ATTN_MODE[0] = old


def attn_kernel_for(mode, Tk, H, Hkv, k_len=None):
    """The kernel ``ops.attention`` runs for head_dim 64: "tc" (attn_tc_kernel and its three prologue launches) or "cuda" (attn_kernel)."""
    return "tc" if mode == "tc" and Tk >= 64 and H == Hkv and k_len is None else "cuda"


LAUNCHES_OF = {"tc": 4, "cuda": 1}


def _qkv(B, Tq, Tk, H, Hkv, seed, scale=1.5):
    D = 64
    return _rand(B, Tq, H * D, seed=seed, scale=scale), _rand(B, Tk, Hkv * D, seed=seed + 1, scale=scale), \
        _rand(B, Tk, Hkv * D, seed=seed + 2, scale=scale)


DISPATCH = [(Tq, Tk) for Tk in (63, 64, 65, 127, 128, 129) for Tq in (1, 63, 127, 128, 129)]


@gpu
@pytest.mark.parametrize("Tq,Tk", DISPATCH, ids=[f"Tq{a}-Tk{b}" for a, b in DISPATCH])
@pytest.mark.parametrize("mode", MODES)
def test_attention_dispatch(mode, Tq, Tk):
    """Non-causal, and causal at q_offset max(Tk - Tq, 0): within the bound of float64, on the kernel the dispatch rule names."""
    B, H = 2, 3
    q, k, v = _qkv(B, Tq, Tk, H, H, seed=Tq + 7 * Tk)
    want_kernel = attn_kernel_for(mode, Tk, H, H)
    assert want_kernel == ("tc" if mode == "tc" and Tk >= 64 else "cuda")
    for causal in (False, True):
        off = max(Tk - Tq, 0) if causal else 0
        y, n = _attn(mode, q.to(DEV), k.to(DEV), v.to(DEV), n_heads=H, scale=0.125, causal=causal, q_offset=off)
        e = rel_err(y, attn_ref(q, k, v, H, H, 0.125, causal, off))
        assert n == LAUNCHES_OF[want_kernel] and e < TOL_ATTN, (causal, n, e)


# name: (Tq, Tk, q_offset, window).  All causal.
MASKS = {"causal-qoff": (100, 230, 130, 0),
         "causal-qoff-1row": (1, 200, 199, 0),
         "window-skip-tile": (165, 500, 335, 100),       # query tiles 0 / 1 start at keys 236 / 364: key tiles 3 / 5
         "window-ge-Tk": (150, 150, 0, 400),
         "window-mid-tile": (300, 300, 0, 37),
         "window-qoff": (140, 210, 70, 90)}


@gpu
@pytest.mark.parametrize("case", list(MASKS))
@pytest.mark.parametrize("mode", MODES)
def test_attention_masks(mode, case):
    Tq, Tk, off, win = MASKS[case]
    B, H = 2, 2
    q, k, v = _qkv(B, Tq, Tk, H, H, seed=len(case) + Tq)
    y, n = _attn(mode, q.to(DEV), k.to(DEV), v.to(DEV), n_heads=H, scale=0.125, causal=True, q_offset=off, window=win)
    e = rel_err(y, attn_ref(q, k, v, H, H, 0.125, True, off, win))
    print(f"\n[attn mask] {mode} {case}: {e:.1e}")
    assert n == LAUNCHES_OF[attn_kernel_for(mode, Tk, H, H)] and e < TOL_ATTN, (n, e)


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_attention_mask_bounds_discriminate(mode):
    """Negative controls: the causal bound one key short and one key long (Whisper's decoder shape), and the window one key short and
    one key long (a window that starts inside a key tile), each more than 5x the bound away from the kernel."""
    B, H = 2, 2
    e = {}
    for name, (Tq, Tk, off, win) in (("causal", MASKS["causal-qoff"]), ("window", MASKS["window-qoff"])):
        q, k, v = _qkv(B, Tq, Tk, H, H, seed=300 + Tq)
        y, _ = _attn(mode, q.to(DEV), k.to(DEV), v.to(DEV), n_heads=H, scale=0.125, causal=True, q_offset=off, window=win)
        e[name] = rel_err(y, attn_ref(q, k, v, H, H, 0.125, True, off, win))
        if name == "causal":
            e["short"] = rel_err(y, attn_ref(q, k, v, H, H, 0.125, True, off, win, bound_shift=-1))
            e["long"] = rel_err(y, attn_ref(q, k, v, H, H, 0.125, True, off, win, bound_shift=1))
        else:
            e["window-1"] = rel_err(y, attn_ref(q, k, v, H, H, 0.125, True, off, win - 1))
            e["window+1"] = rel_err(y, attn_ref(q, k, v, H, H, 0.125, True, off, win + 1))
    print(f"\n[attn controls] {mode}: {e}")
    assert e["causal"] < TOL_ATTN and e["window"] < TOL_ATTN, e
    assert min(e["short"], e["long"], e["window-1"], e["window+1"]) > NEG * TOL_ATTN, e


@gpu
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("G", [2, 4, 8], ids=lambda g: f"gqa{g}")
@pytest.mark.parametrize("mode", MODES)
def test_attention_gqa(mode, G, causal):
    """H = G Hkv query heads over Hkv = 2 key / value heads: attn_kernel in both modes (the tensor-core kernel needs H == Hkv).
    Negative control: the head map h % Hkv."""
    Hkv, Tq, Tk = 2, 150, 150
    H = G * Hkv
    q, k, v = _qkv(2, Tq, Tk, H, Hkv, seed=40 + G + int(causal))
    y, n = _attn(mode, q.to(DEV), k.to(DEV), v.to(DEV), n_heads=H, n_kv_heads=Hkv, scale=0.125, causal=causal)
    e = rel_err(y, attn_ref(q, k, v, H, Hkv, 0.125, causal))
    e_mod = rel_err(y, attn_ref(q, k, v, H, Hkv, 0.125, causal, head_map="mod"))
    assert n == 1 and e < TOL_ATTN and e_mod > NEG * TOL_ATTN, (n, e, e_mod)


@gpu
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("mode", MODES)
def test_attention_k_len(mode, causal):
    """Per-row key counts 0, 37, Tk and 500 > Tk (clamped to Tk): attn_kernel in both modes.  The row with no key is exactly zero."""
    B, H, Tq, Tk = 4, 2, 130, 150
    kl = [0, 37, Tk, 500]
    q, k, v = _qkv(B, Tq, Tk, H, H, seed=50 + int(causal))
    off = Tk - Tq if causal else 0
    y, n = _attn(mode, q.to(DEV), k.to(DEV), v.to(DEV), n_heads=H, scale=0.125, causal=causal, q_offset=off,
                 k_len=torch.tensor(kl, dtype=torch.int32, device=DEV))
    e = rel_err(y, attn_ref(q, k, v, H, H, 0.125, causal, off, k_len=[min(x, Tk) for x in kl]))
    e_full = rel_err(y[1:], attn_ref(q, k, v, H, H, 0.125, causal, off)[1:])            # k_len ignored
    assert n == 1 and e < TOL_ATTN and e_full > NEG * TOL_ATTN, (n, e, e_full)
    assert float(y[0].abs().max()) == 0.0


@gpu
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("mode", MODES)
def test_attention_strided_views(mode, causal):
    """q / k / v are column views of one [B, T + 6, 3 H 64 + 12] buffer (batch stride (T + 6) row, not T row; q at column 4), and
    ``out=`` is a view of a wider, taller buffer whose other elements hold a sentinel that must survive."""
    B, H, T = 3, 2, 130
    HD = 64 * H
    W = 3 * HD + 12
    buf = _rand(B, T + 6, W, seed=60 + int(causal), scale=1.5)
    g = buf.to(DEV)
    q, k, v = g[:, 2:2 + T, 4:4 + HD], g[:, 2:2 + T, 4 + HD:4 + 2 * HD], g[:, 2:2 + T, 4 + 2 * HD:4 + 3 * HD]
    obuf = torch.full((B, T + 3, HD + 24), SENTINEL, device=DEV)
    out = obuf[:, 1:1 + T, 8:8 + HD]
    _, n = _attn(mode, q, k, v, n_heads=H, scale=0.125, causal=causal, out=out)
    qc, kc, vc = (t.cpu() for t in (q, k, v))
    e = rel_err(out, attn_ref(qc, kc, vc, H, H, 0.125, causal))
    keep = torch.ones(obuf.shape, dtype=torch.bool)
    keep[:, 1:1 + T, 8:8 + HD] = False
    assert n == LAUNCHES_OF[attn_kernel_for(mode, T, H, H)] and e < TOL_ATTN, (n, e)
    assert bool((obuf.cpu()[keep] == SENTINEL).all())


RMS_EXP = [-6, -4, -2, 0, 2, 4, 6, 8]


@gpu
@pytest.mark.parametrize("which", ["q", "k", "v"])
@pytest.mark.parametrize("mode", MODES)
def test_attention_operand_magnitude(mode, which):
    """One of q, k, v at rms 2^-6 .. 2^8, the others at rms 1 (T = 300, scale 0.125): both kernels within the bound."""
    B, H, T = 1, 2, 300
    errs = {}
    for ex in RMS_EXP:
        q, k, v = _qkv(B, T, T, H, H, seed=70 + ex, scale=1.0)
        t = {"q": q, "k": k, "v": v}
        t[which] = t[which] * 2.0 ** ex
        y, n = _attn(mode, t["q"].to(DEV), t["k"].to(DEV), t["v"].to(DEV), n_heads=H, scale=0.125)
        errs[ex] = rel_err(y, attn_ref(t["q"], t["k"], t["v"], H, H, 0.125))
        assert n == LAUNCHES_OF[mode]
    print(f"\n[attn magnitude] {mode} {which}: " + " ".join(f"2^{x} {e:.1e}" for x, e in errs.items()))
    assert max(errs.values()) < TOL_ATTN, errs


@gpu
@pytest.mark.parametrize("mode", MODES)
def test_attention_small_v_envelope(mode):
    """V of rms 1e-4: attn_kernel within the bound; attn_tc_kernel within 3x the error of the float64 emulation of its fp16 hi / lo
    split (the envelope the header documents).  Negative control at rms 1: the emulation with hi planes only."""
    B, H, T = 1, 2, 300
    q, k, v = _qkv(B, T, T, H, H, seed=80, scale=1.0)
    vs = v * 1e-4
    y, n = _attn(mode, q.to(DEV), k.to(DEV), vs.to(DEV), n_heads=H, scale=0.125)
    e = rel_err(y, attn_ref(q, k, vs, H, H, 0.125))
    assert n == LAUNCHES_OF[mode]
    if mode == "cuda":
        assert e < TOL_ATTN, e
        print(f"\n[attn small v] cuda: {e:.1e}")
        return
    e_emu = rel_err(tc_emulation(q, k, vs, 0.125), attn_ref(q, k, vs, H, H, 0.125))
    y1, _ = _attn(mode, q.to(DEV), k.to(DEV), v.to(DEV), n_heads=H, scale=0.125)
    e1 = rel_err(y1, attn_ref(q, k, v, H, H, 0.125))
    e_hi = rel_err(y1, tc_emulation(q, k, v, 0.125, planes=1))
    print(f"\n[attn small v] tc: {e:.1e} (emulated {e_emu:.1e}); rms 1: {e1:.1e}, hi-only emulation {e_hi:.1e}")
    assert e < 3 * e_emu and e1 < TOL_ATTN and e_hi > NEG * TOL_ATTN, (e, e_emu, e1, e_hi)


def _params(q, k, v, o, H, **kw):
    from mlx_audio_b200 import _lib
    p = _lib.AttnParams()
    p.q, p.k, p.v, p.o = q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr()
    p.q_bs, p.q_ld, p.k_bs, p.k_ld = q.stride(0), q.stride(1), k.stride(0), k.stride(1)
    p.v_bs, p.v_ld, p.o_bs, p.o_ld = v.stride(0), v.stride(1), o.stride(0), o.stride(1)
    p.B, p.Tq, p.Tk, p.H, p.Hkv, p.D = q.shape[0], q.shape[1], k.shape[1], H, H, 64
    p.scale = 0.125
    for a, val in kw.items():
        setattr(p, a, val)
    return p


@gpu
@pytest.mark.parametrize("case", ["window-without-causal", "q-misaligned", "q-batch-stride", "o-misaligned"])
def test_attention_rejects_invalid_arguments(case):
    """A sliding window without causal masking, a q view one float off 16 bytes, a q batch stride that is not a multiple of 4 and a
    misaligned output: ``ops.attention`` in both modes and both C entry points raise ValueError before any launch."""
    from mlx_audio_b200 import _lib, ops
    B, H, T = 2, 2, 96
    HD = 64 * H
    q = torch.zeros(B, T, HD, device=DEV)
    k, v, o = torch.zeros_like(q), torch.zeros_like(q), torch.zeros_like(q)
    kw = {}
    if case == "window-without-causal":
        kw = dict(window=16)
    elif case == "q-misaligned":
        q = torch.zeros(B, T, HD + 4, device=DEV)[:, :, 1:1 + HD]
    elif case == "q-batch-stride":
        q = torch.zeros(B * T * HD + 4, device=DEV).as_strided((B, T, HD), (T * HD + 1, HD, 1))
    else:
        o = torch.zeros(B, T, HD + 4, device=DEV)[:, :, 1:1 + HD]
    for mode in MODES:
        n0 = ops.LAUNCHES[0]
        with pytest.raises(ValueError):
            _attn(mode, q, k, v, n_heads=H, scale=0.125, out=o, **kw)
        assert ops.LAUNCHES[0] == n0
    p = _params(q, k, v, o, H, **kw)
    ws = torch.empty(_lib.lib().b2a_attention_tc_ws_bytes(B, H, T, T), device=DEV, dtype=torch.uint8)
    s = torch.cuda.current_stream().cuda_stream
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().b2a_attention(C.byref(p), s))
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().b2a_attention_tc(C.byref(p), ws.data_ptr(), s))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------ rotary
ROPE = [(trad, D, H, off) for trad in (True, False) for D in (64, 128) for H in (1, 8, 16) for off in (0, 7, 20000)]
ROPE_GRID = 132 * 16 * 256             # attn.cu caps the grid at 132 x 16 CTAs of 256 threads: larger inputs take the grid-stride loop


@gpu
@pytest.mark.parametrize("trad,D,H,off", ROPE,
                         ids=[f"{'trad' if t else 'half'}-h{h}-d{d}-off{o}" for t, d, h, o in ROPE])
def test_rope_vs_float64(trad, D, H, off):
    """In place on the q and k column views of a [B = 2, T, 3 H D] buffer at bases 1e4 and 1e6; the v columns hold a sentinel that must
    survive.  Negative control at offset 20000: the angles in float32."""
    from mlx_audio_b200 import ops
    B, T = 2, 300
    d = H * D
    assert (B * T * H * D // 2 > ROPE_GRID) == (H == 16 and D == 128)
    for base in (1e4, 1e6):
        qk = _rand(B, T, 2 * d, seed=D + H + off + int(base) % 97 + int(trad))
        buf = torch.full((B, T, 3 * d), SENTINEL, device=DEV)
        buf[:, :, :2 * d] = qk.to(DEV)
        ops.rope_(buf[:, :, :d], H, offset=off, base=base, traditional=trad)
        ops.rope_(buf[:, :, d:2 * d], H, offset=off, base=base, traditional=trad)
        got = buf.cpu()
        want = torch.cat([rope_ref(qk[..., :d], H, off, base, trad), rope_ref(qk[..., d:], H, off, base, trad)], -1)
        e = rel_err(got[..., :2 * d], want)
        assert e < TOL_ROPE and bool((got[..., 2 * d:] == SENTINEL).all()), (base, e)
        if off == 20000:
            want32 = torch.cat([rope_ref(qk[..., :d], H, off, base, trad, torch.float32),
                                rope_ref(qk[..., d:], H, off, base, trad, torch.float32)], -1)
            e32 = rel_err(got[..., :2 * d], want32)
            assert e32 > NEG * TOL_ROPE, (base, e, e32)


# ------------------------------------------------------------------------------------------------------------ LayerNorm
def ln_kernel(C, x_ld, y_ld, res_ld=None, offsets_aligned=True):
    """The kernel b2a_layernorm launches (norm.cu host rule)."""
    al = C % 4 == 0 and C <= 1024 and x_ld % 4 == 0 and y_ld % 4 == 0 and (res_ld is None or res_ld % 4 == 0) and offsets_aligned
    return ("vec4" if C <= 512 else "vec8") if al else "scalar"


# (C, x row stride)
LN_SHAPES = [(4, 12), (128, 136), (508, 516), (512, 512), (516, 524), (768, 768), (1024, 1032), (1028, 1036), (1280, 1280),
             (2048, 2056), (130, 138), (6, 14), (512, 514)]
LN_VARIANTS = ["affine", "rms-w", "none", "res", "ada", "lrelu", "out-strided", "inplace", "mean50"]


def _ln_id(C, ld):
    return f"{ln_kernel(C, ld, ld)}-C{C}" + (f"-ld{ld}" if ld == C + 2 else "")


def test_layernorm_dispatch_table_reaches_every_kernel():
    kinds = [ln_kernel(C, ld, ld) for C, ld in LN_SHAPES]
    assert set(kinds) == {"vec4", "vec8", "scalar"}
    assert kinds.count("vec4") == 4 and kinds.count("vec8") == 3 and kinds.count("scalar") == 6
    assert _ln_id(512, 514) == "scalar-C512-ld514" and _ln_id(1024, 1032) == "vec8-C1024"


@gpu
@pytest.mark.parametrize("C,ld", LN_SHAPES, ids=[_ln_id(C, ld) for C, ld in LN_SHAPES])
def test_layernorm_vs_float64(C, ld):
    """Every LN_VARIANTS option on 37 rows (not a multiple of the 4 rows of a vector CTA or the 8 of a scalar one) of width C at row
    stride ``ld``: affine, RMSNorm with a weight (the talker's), no affine, a residual (row stride C + 4), AdaLN, LeakyReLU after the
    affine (Kokoro's duration LSTM), ``out=`` a column view of a wider buffer with sentinel columns, in place, rows of mean 50 and std 3.
    Negative controls: the unbiased variance (LayerNorm variants), LayerNorm for RMSNorm."""
    from mlx_audio_b200 import ops
    R = 37
    errs = {}
    for i, var in enumerate(LN_VARIANTS):
        s = 1000 + 10 * i + C
        xs = _rand(R, C, seed=s) * (3.0 if var == "mean50" else 1.0) + (50.0 if var == "mean50" else 0.0)
        w, b = 1 + 0.2 * _rand(C, seed=s + 1), 0.3 * _rand(C, seed=s + 2)
        xbuf = torch.full((R, ld), SENTINEL, device=DEV)
        x = xbuf[:, :C]
        x.copy_(xs)
        kw, ref = dict(eps=1e-5), dict(eps=1e-5)
        res = None
        if var in ("affine", "out-strided", "inplace", "mean50", "res", "lrelu"):
            kw.update(w=w.to(DEV), b=b.to(DEV))
            ref.update(w=w, b=b)
        if var == "rms-w":
            kw.update(w=w.to(DEV), rms=True, eps=1e-6)
            ref.update(w=w, rms=True, eps=1e-6)
        if var in ("res", "inplace"):
            rs = _rand(R, C, seed=s + 3)
            res = torch.zeros(R, C + 4, device=DEV)[:, :C]
            res.copy_(rs)
            kw.update(res=res)
            ref.update(res=rs)
        if var == "ada":
            ada = 0.3 * _rand(2 * C, seed=s + 4)
            kw.update(ada=ada.to(DEV))
            ref.update(ada=ada)
        if var == "lrelu":
            kw.update(post_act=ops.ACT["lrelu"], post_p0=0.2)
            ref.update(slope=0.2)
        obuf = None
        if var == "out-strided":
            obuf = torch.full((R, C + 12), SENTINEL, device=DEV)
            kw.update(out=obuf[:, 4:4 + C])
        elif var == "inplace":
            kw.update(out=x)
        y = ops.layernorm(x, **kw)
        want = ln_ref(xs, **ref)
        e = rel_err(y, want)
        ctl = rel_err(y, ln_ref(xs, **dict(ref, rms=False))) if ref.get("rms") else rel_err(y, ln_ref(xs, **ref, unbiased=True))
        errs[var] = (e, ctl)
        assert e < TOL_LN and ctl > NEG * TOL_LN, (var, e, ctl)
        assert bool((xbuf.cpu()[:, C:] == SENTINEL).all()), var
        if var == "inplace":
            assert y.data_ptr() == x.data_ptr() and torch.equal(xbuf.cpu()[:, :C], y.cpu())
        else:
            assert torch.equal(x.cpu(), xs), var                        # the input is left alone
        if obuf is not None:
            ob = obuf.cpu()
            assert bool((ob[:, :4] == SENTINEL).all()) and bool((ob[:, 4 + C:] == SENTINEL).all())
    print(f"\n[layernorm] {_ln_id(C, ld)}: " + " ".join(f"{k} {a:.1e} ({c:.0e})" for k, (a, c) in errs.items()))


@gpu
@pytest.mark.parametrize("tc_mode", ["x2", "x1"])
@pytest.mark.parametrize("C", [128, 512, 768, 1024], ids=lambda c: f"{'vec4' if c <= 512 else 'vec8'}-C{c}")
def test_layernorm_planes(C, tc_mode):
    """``planes=True`` (C % 64 == 0, vector kernels only): the bf16 planes are bit-identical to ``ops.prep_bf16`` of the fp32 output,
    which itself equals the output without planes.  In x1 mode ``Planes.lo`` is None and the kernel is given a null lo pointer."""
    from mlx_audio_b200 import ops
    R = 37
    x = _rand(R, C, seed=C, scale=2.0).to(DEV)
    w, b = (1 + 0.2 * _rand(C, seed=C + 1)).to(DEV), (0.3 * _rand(C, seed=C + 2)).to(DEV)
    old, old_call = ops.TC_MODE[0], ops._call
    seen = []

    def spy(kind, fn, n, *args):
        if kind == "layernorm":
            seen.append(args[16])                            # emit_lo
        return old_call(kind, fn, n, *args)
    ops.TC_MODE[0] = tc_mode
    ops._call = spy
    try:
        y, pl = ops.layernorm(x, w, b, eps=1e-5, planes=True)
        hi, lo = ops.prep_bf16(y[None], None, C, 2 if tc_mode == "x2" else 1)
    finally:
        ops.TC_MODE[0], ops._call = old, old_call
    assert torch.equal(y, ops.layernorm(x, w, b, eps=1e-5))
    assert pl.C == C and tuple(pl.hi.shape) == (1, R, C) and torch.equal(pl.hi, hi)
    if tc_mode == "x2":
        assert seen == [pl.lo.data_ptr()] and torch.equal(pl.lo, lo)
    else:
        assert pl.lo is None and lo is None and seen == [None]


@gpu
def test_layernorm_planes_need_the_vectorised_kernel():
    from mlx_audio_b200 import ops
    x = torch.zeros(5, 1280, device=DEV)
    with pytest.raises(ValueError):
        ops.layernorm(x, planes=True)
    with pytest.raises(ValueError):
        ops.layernorm(torch.zeros(5, 1000, device=DEV), planes=True)         # C % 64 != 0


@gpu
@pytest.mark.parametrize("C", [4, 768, 1280], ids=["vec4", "vec8", "scalar"])
def test_layernorm_zero_rows(C):
    """Zero rows launch nothing and return an empty result (an empty CUDA tensor's data pointer is null; the entry point used to reject
    it as a null pointer)."""
    from mlx_audio_b200 import ops
    x = torch.empty(0, C, device=DEV)
    y = ops.layernorm(x, torch.ones(C, device=DEV), torch.zeros(C, device=DEV))
    assert tuple(y.shape) == (0, C)
    if C % 64 == 0 and C <= 1024:
        y, pl = ops.layernorm(x, planes=True)
        assert tuple(y.shape) == (0, C) and tuple(pl.hi.shape) == (1, 0, C)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------ AdaIN / statistics
@gpu
@pytest.mark.parametrize("L", [1, 7, 255, 256, 257, 1000], ids=lambda v: f"L{v}")
def test_adain_coeffs_vs_float64(L):
    """B = 3, C = 70 (not a multiple of the 32-channel CTA), x a view of a [3, L + 3, 100] buffer (batch stride (L + 3) 100, row stride
    100, first channel 10); gb None and given; rows of mean 0 / std 2 and of mean 1e3 / std 0.1.  Negative control (L >= 7, mean 1e3):
    var = E[x^2] - mean^2 in float32."""
    from mlx_audio_b200 import ops
    B, Cc = 3, 70
    for big in (False, True):
        xs = _rand(B, L, Cc, seed=L + int(big)) * (0.1 if big else 2.0) + (1e3 if big else 0.0)
        buf = torch.full((B, L + 3, 100), SENTINEL, device=DEV)
        x = buf[:, 1:1 + L, 10:10 + Cc]
        x.copy_(xs)
        xs = x.cpu()
        gb = 0.3 * _rand(B, 2 * Cc, seed=L + 5)
        for g in (None, gb):
            sc, sh = ops.adain_coeffs(x, None if g is None else g.to(DEV))
            rsc, rsh = adain_ref(xs, g)
            e = max(rel_err(sc, rsc), rel_err(sh, rsh))
            assert e < TOL_ADAIN, (big, g is None, e)
            if big and L >= 7:
                fsc, fsh = adain_ref(xs, g, stats_dtype=torch.float32)
                e32 = max(rel_err(sc, fsc), rel_err(sh, fsh))
                assert e32 > NEG * TOL_ADAIN, (e, e32)


@gpu
@pytest.mark.parametrize("n_dst", [1, 2, 3, 4])
def test_channel_stats_and_coeffs(n_dst):
    """``channel_stats`` into n_dst destinations, each a channel-offset view of its own wider [B, C', 2, 4] buffer (different batch
    strides): x0 (L 300, mean 50 / std 3) onto zeroed bins, then x1 (L 37) onto those.  Every destination then holds bins(x0) + bins(x1)
    exactly and the channels outside the views keep their sentinel; ``coeffs_from_stats`` over L 337 agrees with ``adain_coeffs`` of the
    concatenated rows within 1e-6 and with float64 within 1e-5; a second run gives the same bits."""
    from mlx_audio_b200 import ops
    B, Cc, L0, L1 = 3, 70, 300, 37
    nb = ops.STAT_BINS
    x0 = (_rand(B, L0, Cc, seed=90 + n_dst) * 3 + 50)
    x1 = _rand(B, L1, Cc, seed=91 + n_dst)
    g0 = torch.zeros(B, L0 + 4, Cc + 6, device=DEV)
    x0d = g0[:, 2:2 + L0, 3:3 + Cc]
    x0d.copy_(x0)
    x1d = x1.to(DEV)
    gb = 0.3 * _rand(B, 2 * Cc, seed=92)
    sent = 0x5A5A5A5A

    def run():
        wides, views = [], []
        for i in range(n_dst):
            w = torch.full((B, Cc + 5 * (i + 1), 2, nb), sent, dtype=torch.int64, device=DEV)
            v = w[:, 3 * i + 1:3 * i + 1 + Cc]
            v.zero_()
            wides.append(w)
            views.append(v)
        ops.channel_stats(x0d, views)
        first = [v.clone() for v in views]
        ops.channel_stats(x1d, views)
        return wides, views, first
    wides, views, first = run()
    z1 = torch.zeros(B, Cc, 2, nb, dtype=torch.int64, device=DEV)
    ops.channel_stats(x1d, z1)
    for i, (w, v) in enumerate(zip(wides, views)):
        assert torch.equal(first[i], first[0]) and torch.equal(v, first[0] + z1), i
        keep = torch.ones(w.shape[:2], dtype=torch.bool)
        keep[:, 3 * i + 1:3 * i + 1 + Cc] = False
        assert bool((w.cpu()[keep] == sent).all()), i
    sc, sh = ops.coeffs_from_stats(views[-1].contiguous(), L0 + L1, gb.to(DEV))
    xcat = torch.cat([x0, x1], 1)
    asc, ash = ops.adain_coeffs(xcat.to(DEV), gb.to(DEV))
    rsc, rsh = adain_ref(xcat, gb)
    agree = max(rel_err(sc, asc), rel_err(sh, ash))
    e = max(rel_err(sc, rsc), rel_err(sh, rsh))
    assert agree < TOL_STATS_AGREE and e < TOL_ADAIN, (agree, e)
    wides2, views2, _ = run()
    assert all(torch.equal(a, b) for a, b in zip(wides, wides2))
    sc2, sh2 = ops.coeffs_from_stats(views2[-1].contiguous(), L0 + L1, gb.to(DEV))
    assert torch.equal(sc, sc2) and torch.equal(sh, sh2)
