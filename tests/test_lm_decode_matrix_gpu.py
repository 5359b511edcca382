"""Autoregressive-LM step kernels (csrc/lm.cu: b2a_gemv_bf16, b2a_qknorm_rope_cache, b2a_attn_decode, b2a_swiglu; csrc/attn_prefill.cu:
b2a_attn_prefill) against float64 on every dispatch branch.  These run every Qwen3-TTS frame (talker, code predictor, batch session,
in-context prefill) and Soprano's LM, through talker.py's ``_DecoderStack``.

Where each branch is run:
- GEMV instantiations (lm.cu host rule ``wide = M > 2 && (K/8) % 4 == 0``, rows launched in groups of 8): the ids of
  ``test_gemv_vs_float64`` name the kernels each case launches (``narrow1``, ``narrow2``, ``narrow4``, ``narrow8``, ``wide4``,
  ``wide8``); ``test_gemv_dispatch_table_reaches_every_instantiation`` checks that the cases reach all six.
- Head dims 32 / 64 / 128 of ``qknorm_rope_cache_kernel`` and ``attn_decode_kernel``: the ``d32`` / ``d64`` / ``d128`` ids.
- ``attn_decode``'s shared-memory opt-in (a score buffer of max_k floats past the function's default limit):
  ``test_attn_decode_long_cache[*-smem-opt-in]`` (12289 keys) and ``[*-smem-limit]`` (49152); ``[*-smem-default]`` (12288 keys,
  exactly 48 KB of scores) and ``[*-smem-47k]`` (12032) are just under 48 KB, where the opt-in used to be skipped.
- Prefill tile skips: key tiles before ``kv_start`` (``t_lo``) in ``test_attn_prefill_vs_float64[*-kv64-skip1]`` and
  ``[*-kv150-skip2]``; a 64-row query tile that is all left padding (no key tile at all) in every case of that test (row 1's first
  tile); ``max_k < base + S`` in every case.

Tolerances, all max |y - ref| / max |ref| against float64 on the CPU:
- GEMV 2e-5.  The weights are bf16-exact, so the only rounding is the fp32 of the activations, the norm and the K <= 3072 term sums
  (a few 2^-24 times sqrt(K) of the scale).  Negative control: the reference with the activations rounded to bf16 (what a kernel
  that converted x to bf16 would compute) must exceed 5x the bound, in every case.
- q/k RMSNorm + rotary 1e-5.  A handful of fp32 operations per element (the sum of squares, rsqrt, the two products of the rotation)
  with cos / sin evaluated in float64 and rounded to fp32.  Negative controls: the angles computed in float32 (one fp32 ulp of an
  angle near 40 000 rad is 2^-8) and MRoPE with sections (24, 20) instead of (20, 20) (at head_dim 128; at 32 and 64 both cover every
  frequency slot).  V rows are copied into the cache: bit-exact.
- Attention 2e-5.  Decode runs on the CUDA cores in fp32 (scores, exp, p v sums); prefill multiplies fp16 hi / lo splits with three
  products per MMA, fp32-grade.  Negative controls, on both kernels: the causal bound one key short (base + s) and one key long
  (base + s + 2), and kv_start ignored.
- SwiGLU 1e-6: elementwise, one expf, a division and two products in fp32: a few ulp (2^-24 = 6e-8) of each element.

Cache rows no query may see are NaN in the attention tests, so a kernel that read one would fail the bound; cache rows no query writes
hold a sentinel in the rotary tests and must keep it.
"""
import math

import pytest
import torch

from oracle import nn as ON
from oracle import qwen3 as Q

gpu = pytest.mark.gpu
DEV = "cuda:0"
TOL_GEMV = 2e-5
TOL_ATTN = 2e-5
TOL_ROPE = 1e-5
TOL_SWIGLU = 1e-6
NEG = 5                      # every negative control exceeds NEG x its bound
SENTINEL = -1234.5


def _rand(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _bf(x):
    return x.to(torch.bfloat16).float()


def rel_err(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _i32(v):
    return torch.tensor(v, dtype=torch.int32, device=DEV)


# ------------------------------------------------------------------------------------------------------------ float64 references
def gemv_ref(x, w, bias=None, norm_w=None, eps=1e-6, swiglu=False, res=None):
    """``ops.gemv``: RMSNorm prologue, x @ W^T + bias, SwiGLU on interleaved (gate, up) rows, + residual."""
    x = x.double()
    if norm_w is not None:
        x = ON.rms_norm(x, norm_w.double(), eps)
    y = x @ w.double().T
    if bias is not None:
        y = y + bias.double()
    if swiglu:
        y = torch.nn.functional.silu(y[:, 0::2]) * y[:, 1::2]
    if res is not None:
        y = y + res.double()
    return y


def rope_ref(qkv, Hq, Hkv, D, pos3, q_norm=None, k_norm=None, eps=1e-6, mrope=(0, 0), theta=1e6, angle_dtype=torch.float64):
    """``ops.qknorm_rope_cache`` without the cache: qkv [B,S,(Hq+2Hkv)D] and rotary positions pos3 [3,B,S] -> q [B,S,Hq D] and the
    k, v rows [B,S,Hkv D].  ``mrope=(a, b)`` is the kernel's argument, the oracle's section[1], section[2] (talker.py passes
    (sec[1], sec[2])).  ``angle_dtype`` is the type the angles are computed in (float32 for a negative control only)."""
    B, S, _ = qkv.shape
    x = qkv.double()
    q = x[..., :Hq * D].reshape(B, S, Hq, D)
    k = x[..., Hq * D:(Hq + Hkv) * D].reshape(B, S, Hkv, D)
    v = x[..., (Hq + Hkv) * D:]
    if q_norm is not None:
        q = ON.rms_norm(q, q_norm.double(), eps)
    if k_norm is not None:
        k = ON.rms_norm(k, k_norm.double(), eps)
    cos, sin = Q.mrope_cos_sin(pos3, D, theta, (0, mrope[0], mrope[1]), angle_dtype)
    qr, kr = Q.apply_rope(q.transpose(1, 2), k.transpose(1, 2), cos.double(), sin.double())
    return qr.transpose(1, 2).reshape(B, S, Hq * D), kr.transpose(1, 2).reshape(B, S, Hkv * D), v


def cache_attn_ref(q, kc, vc, Hq, Hkv, D, base_rows, slot, kv_start, max_k, scale, bound_shift=0):
    """Causal GQA attention against a KV cache: query s of row b sees cache rows [kv_start[b], min(base_rows[b] + s + 1, max_k)) of
    cache batch slot[b]; a query with no visible key (a negative position, or kv_start past its last key) gives zeros.
    q [B,S,Hq D], caches [batches, rows, Hkv D]; ``base_rows`` per-row ints, ``slot`` / ``kv_start`` per-row ints or None (identity /
    0).  ``bound_shift`` moves the causal bound by whole keys: negative controls only."""
    B, S, _ = q.shape
    G = Hq // Hkv
    out = torch.zeros(B, S, Hq * D, dtype=torch.float64)
    for b in range(B):
        cb = b if slot is None else int(slot[b])
        k0 = 0 if kv_start is None else int(kv_start[b])
        end = torch.clamp(int(base_rows[b]) + torch.arange(S) + 1 + bound_shift, max=max_k)     # exclusive, per query
        hi = int(end.max())
        if hi <= k0:
            continue
        k = kc[cb, k0:hi].double().view(-1, Hkv, D).repeat_interleave(G, dim=1)
        v = vc[cb, k0:hi].double().view(-1, Hkv, D).repeat_interleave(G, dim=1)
        sc = torch.einsum("shd,nhd->hsn", q[b].double().view(S, Hq, D), k) * scale
        vis = torch.arange(k0, hi)[None, :] < end[:, None]                                       # [S, keys]
        p = torch.softmax(sc.masked_fill(~vis, float("-inf")), dim=-1)
        p = torch.where(vis.any(-1)[None, :, None], p, torch.zeros_like(p))                   # no visible key: zeros
        out[b] = torch.einsum("hsn,nhd->shd", p, v).reshape(S, Hq * D)
    return out


# ------------------------------------------------------------------------------------------------------------ CPU: the references
def test_cache_attn_ref_equals_oracle_sdpa():
    """With one base, identity slots and no kv_start, cache_attn_ref is the oracle's SDPA with its causal mask over the first base + S
    cache rows (GQA 4, base 6, S 5)."""
    B, S, Hq, Hkv, D, base = 2, 5, 8, 2, 16, 6
    q, kc, vc = _rand(B, S, Hq * D, seed=1), _rand(B, 20, Hkv * D, seed=2), _rand(B, 20, Hkv * D, seed=3)
    got = cache_attn_ref(q, kc, vc, Hq, Hkv, D, [base] * B, None, None, base + S, 0.3)
    n = base + S
    k = kc[:, :n].double().view(B, n, Hkv, D).transpose(1, 2)
    v = vc[:, :n].double().view(B, n, Hkv, D).transpose(1, 2)
    want = ON.sdpa(q.double().view(B, S, Hq, D).transpose(1, 2), k, v, 0.3, Q.causal_mask(S, n, torch.float64))
    assert rel_err(got, want.transpose(1, 2).reshape(B, S, Hq * D)) < 1e-13
    # kv_start masks the keys before it, as an additive -inf on those columns does
    ks = [2, 0]
    got = cache_attn_ref(q, kc, vc, Hq, Hkv, D, [base] * B, None, ks, base + S, 0.3)
    mask = Q.causal_mask(S, n, torch.float64)[None, None].repeat(B, 1, 1, 1)
    for b, s0 in enumerate(ks):
        mask[b, :, :, :s0] = float("-inf")
    want = ON.sdpa(q.double().view(B, S, Hq, D).transpose(1, 2), k, v, 0.3, mask)
    assert rel_err(got, want.transpose(1, 2).reshape(B, S, Hq * D)) < 1e-13


def test_mrope_ref_with_equal_positions_is_plain_rope():
    """MRoPE with the same position on all three axes is plain RoPE, whatever the sections; with differing positions it is not."""
    B, S, Hq, Hkv, D = 2, 3, 2, 1, 128
    qkv = _rand(B, S, (Hq + 2 * Hkv) * D, seed=4)
    pos = torch.randint(0, 40000, (B, S), generator=torch.Generator().manual_seed(5))
    q1, k1, _ = rope_ref(qkv, Hq, Hkv, D, pos[None].expand(3, B, S), mrope=(20, 20))
    cos, sin = Q.rope_cos_sin(pos, D, 1e6)
    q2, k2 = Q.apply_rope(qkv[..., :Hq * D].double().view(B, S, Hq, D).transpose(1, 2),
                          qkv[..., Hq * D:(Hq + Hkv) * D].double().view(B, S, Hkv, D).transpose(1, 2), cos, sin)
    assert rel_err(q1, q2.transpose(1, 2).reshape(B, S, -1)) < 1e-14 and rel_err(k1, k2.transpose(1, 2).reshape(B, S, -1)) < 1e-14
    pos3 = torch.stack([pos, pos + 1000, pos + 2000])
    assert rel_err(rope_ref(qkv, Hq, Hkv, D, pos3, mrope=(20, 20))[0], q1) > 1e-3


# ------------------------------------------------------------------------------------------------------------ GEMV
GEMV_GROUP = 8               # ops.gemv launches at most 8 rows at a time
GEMV_M = [1, 2, 3, 4, 5, 8, 9, 16]
GEMV_K = [64, 1000, 1024, 3072]        # 1000: (K/8) % 4 != 0, the narrow kernels for M > 2
GEMV_KERNELS = {"narrow1", "narrow2", "narrow4", "narrow8", "wide4", "wide8"}


def gemv_kernels(M, K):
    """The instantiations b2a_gemv_bf16 launches for ``ops.gemv`` on M rows of width K (lm.cu: M == 1 -> <1>, M == 2 -> <2>, else
    the wide kernel when (K/8) % 4 == 0, <4> for M <= 4 and <8> above)."""
    out = []
    for m0 in range(0, M, GEMV_GROUP):
        m = min(GEMV_GROUP, M - m0)
        wide = m > 2 and (K // 8) % 4 == 0
        out.append(("wide" if wide else "narrow") + str(1 if m == 1 else 2 if m == 2 else 4 if m <= 4 else 8))
    return out


GEMV_CASES = [(M, K) for M in GEMV_M for K in GEMV_K]


def test_gemv_dispatch_table_reaches_every_instantiation():
    seen = {k for M, K in GEMV_CASES for k in gemv_kernels(M, K)}
    assert seen == GEMV_KERNELS, seen
    assert gemv_kernels(3, 1000) == ["narrow4"] and gemv_kernels(5, 1000) == ["narrow8"]
    assert gemv_kernels(3, 1024) == ["wide4"] and gemv_kernels(9, 64) == ["wide8", "narrow1"] and gemv_kernels(16, 3072) == ["wide8"] * 2


def test_gemv_eligible_needs_k_multiple_of_8():
    """The GEMV loads 8 bf16 weights and 8 activations at a time: a layer of another input width is not eligible, so
    ``_DecoderStack._proj`` sends it to ``linear``.  ``gemv_eligible`` used to accept it, and the C entry point then rejected the
    call, so ``_proj`` raised instead of falling back."""
    from mlx_audio_b200 import ops

    def cw(K):
        cpad = -(-K // 64) * 64
        c = ops.ConvW(torch.zeros(1, K, 64), None, 1, K, 64, 1)
        c.w_tc, c.cin_pad = torch.zeros(1, 64, cpad, dtype=torch.bfloat16), cpad
        return c
    assert ops.gemv_eligible(cw(1000)) and ops.gemv_eligible(cw(64))
    assert not any(ops.gemv_eligible(cw(K)) for K in (1001, 1004, 1006, 36))


def _gemv_weight(w, bias=None):
    """A ``ConvW`` with the bf16 rows [N, cin_pad] laid out as pack_conv lays them (input padded to a multiple of 64), for any N
    (pack_conv makes the bf16 plane only when N % 32 == 0)."""
    from mlx_audio_b200 import ops
    N, K = w.shape
    cpad = -(-K // 64) * 64
    wt = torch.zeros(1, N, cpad, dtype=torch.bfloat16)
    wt[0, :, :K] = w.to(torch.bfloat16)
    cw = ops.ConvW(w.t().contiguous()[None].to(DEV), None if bias is None else bias.to(DEV), 1, K, N, 1)
    cw.w_tc, cw.cin_pad = wt.to(DEV), cpad
    assert ops.gemv_eligible(cw)
    return cw


# (name, N, swiglu, norm, bias, residual, x row stride > K).  N tails: 101 = 8*12 + 5 and 70 = 8*8 + 6 leave part of the last CTA in
# both row tilings (4 rows narrow, 8 wide); the SwiGLU widths 98, 100, 102 (N % 8 = 2, 4, 6) leave 1..3 of a wide CTA's 4 pairs
# and, for 98 and 102, one of a narrow CTA's 2.
GEMV_VARIANTS = [("linear-norm-bias-res-xstride", 101, False, True, True, True, True),
                 ("linear-plain", 70, False, False, False, False, False),
                 ("swiglu-norm-res", 98, True, True, False, True, False),
                 ("swiglu-xstride", 100, True, False, False, False, True),
                 ("swiglu-norm-res-xstride", 102, True, True, False, True, True)]


@gpu
@pytest.mark.parametrize("M,K", GEMV_CASES, ids=[f"M{M}-K{K}-" + "+".join(gemv_kernels(M, K)) for M, K in GEMV_CASES])
def test_gemv_vs_float64(M, K):
    """Every variant of GEMV_VARIANTS at M rows of width K; the output with ``prefetch=`` equals the output without, and a second run
    equals the first, bit for bit."""
    from mlx_audio_b200 import ops
    errs = {}
    for i, (name, N, swiglu, norm, bias, res, xstride) in enumerate(GEMV_VARIANTS):
        seed = 100 * i + M + K
        w = _bf(_rand(N, K, seed=seed) / math.sqrt(K))
        b = _rand(N, seed=seed + 1, scale=0.5) if bias else None
        nw = 1 + 0.1 * _rand(K, seed=seed + 2) if norm else None
        x = _rand(M, K, seed=seed + 3)
        r = _rand(M, N // 2 if swiglu else N, seed=seed + 4) if res else None
        cw = _gemv_weight(w, b)
        if xstride:
            xd = torch.zeros(M, K + 12, device=DEV)[:, :K]          # rows 16-byte aligned, x_ld = K + 12
            xd.copy_(x)
        else:
            xd = x.to(DEV)
        kw = dict(norm_w=None if nw is None else nw.to(DEV), norm_eps=1e-6, swiglu=swiglu, res=None if r is None else r.to(DEV))
        y = ops.gemv(xd, cw, **kw)
        ref = gemv_ref(x, w, b, nw, 1e-6, swiglu, r)
        e, e_bf = rel_err(y, ref), rel_err(y, gemv_ref(_bf(x), w, b, nw, 1e-6, swiglu, r))
        errs[name] = (e, e_bf)
        assert e < TOL_GEMV and e_bf > NEG * TOL_GEMV, (name, e, e_bf)
        if i == 0:
            other = _gemv_weight(_bf(_rand(256, 512, seed=seed + 5)))
            assert torch.equal(ops.gemv(xd, cw, prefetch=other, **kw), y) and torch.equal(ops.gemv(xd, cw, **kw), y)
    print(f"\n[gemv] M {M} K {K} {gemv_kernels(M, K)}: " + " ".join(f"{n} {e:.1e} (bf16 x {c:.1e})" for n, (e, c) in errs.items()))


@gpu
def test_decoder_projection_with_k_not_multiple_of_8_uses_linear():
    """A bf16 layer of input width 1001 is not GEMV-eligible: ``ops.gemv`` refuses it and ``_DecoderStack._proj`` runs it through
    ``linear`` (RMSNorm + residual, and SwiGLU), within the GEMV bound of float64."""
    from mlx_audio_b200 import ops
    from mlx_audio_b200.tts.models.qwen3_tts.talker import _DecoderStack
    M, K = 3, 1001
    w, wg = _bf(_rand(64, K, seed=60) / math.sqrt(K)), _bf(_rand(128, K, seed=61) / math.sqrt(K))
    x, nw, r = _rand(M, K, seed=62), 1 + 0.1 * _rand(K, seed=63), _rand(M, 64, seed=64)
    cw, cg = ops.pack_linear(w, None, DEV), ops.pack_linear(wg, None, DEV)
    assert cw.w_tc is not None and not ops.gemv_eligible(cw)
    xd = x.to(DEV)
    with pytest.raises(NotImplementedError):
        ops.gemv(xd, cw)
    stack = object.__new__(_DecoderStack)          # _proj reads only eps
    stack.eps = 1e-6
    assert rel_err(stack._proj(xd, cw, norm_w=nw.to(DEV), res=r.to(DEV)), gemv_ref(x, w, None, nw, 1e-6, False, r)) < TOL_GEMV
    assert rel_err(stack._proj(xd, cg, norm_w=nw.to(DEV), swiglu=True), gemv_ref(x, wg, None, nw, 1e-6, True)) < TOL_GEMV


# ------------------------------------------------------------------------------------------------------------ q/k norm + rotary + cache
QK_CASES = ["host", "base_dev-no-norm", "pos3-mrope", "pos_shift-clamp", "base_rows-slot", "large-pos-past-smax"]


def _qk_case(name, D):
    """Inputs of one qknorm_rope_cache case: B rows of S, cache batches, rotary positions [3,B,S] (what the kernel must use),
    per-row base and slot, cache rows smax, and the ops keyword arguments."""
    B, S, nslots, smax, theta = 3, 5, 3, 64, 1e6
    base, slot, pos3, shift, norms, mrope, kw = [9] * 3, [0, 1, 2], None, None, True, (0, 0), {}
    if name == "host":
        kw = dict(base=9)
    elif name == "base_dev-no-norm":                        # code predictor / Soprano: no MRoPE, theta 1e4 (Soprano)
        norms, theta, kw = False, 1e4, dict(base_dev=_i32([9]))
    elif name == "pos3-mrope":                              # explicit T / H / W positions, all different, up to 40 000
        mrope, kw = (20, 20), dict(base=9)
        pos3 = torch.randint(0, 40000, (3, B, S), generator=torch.Generator().manual_seed(D), dtype=torch.int32)
    elif name == "pos_shift-clamp":                         # left-padded batch rows: position = max(row - pad, 0)
        base, shift = [12] * 3, [0, 4, 14]
        kw = dict(base=12, pos_shift=_i32(shift))
    elif name == "base_rows-slot":                          # continuous batching: ragged bases (one left-padded), slot map with gaps
        nslots, base, slot = 5, [20, -3, 0], [4, 0, 2]
        kw = dict(base_rows=_i32(base), slot=_i32(slot))
    elif name == "large-pos-past-smax":                     # rows base + s >= smax are not written
        B, S, smax, base, slot = 2, 8, 40000, [39995] * 2, [0, 1]
        nslots, kw = 2, dict(base=39995)
    rot = torch.tensor(base)[:, None] + torch.arange(S)[None]
    if shift is not None:
        rot = (rot - torch.tensor(shift)[:, None]).clamp(min=0)
    rot = rot[None].expand(3, B, S) if pos3 is None else pos3
    if pos3 is not None:
        kw["pos3"] = pos3.to(DEV)
    return B, S, nslots, smax, theta, base, slot, rot, norms, mrope, kw


def _check_cache(kc, vc, k, v, base, slot, smax):
    """Row base[b] + s of cache batch slot[b] holds k / v of (b, s) when 0 <= base[b] + s < smax (v bit-exact); every other element of
    the buffers (rows past smax included) still holds the sentinel.  Returns the error of the k rows."""
    kc, vc = kc.cpu(), vc.cpu()
    written = torch.zeros(kc.shape[:2], dtype=torch.bool)
    got, want = [], []
    for b in range(k.shape[0]):
        for s in range(k.shape[1]):
            r = base[b] + s
            if 0 <= r < smax:
                written[slot[b], r] = True
                got.append(kc[slot[b], r])
                want.append(k[b, s])
                assert torch.equal(vc[slot[b], r], v[b, s].float()), (b, s)
    assert got and bool((kc[~written] == SENTINEL).all()) and bool((vc[~written] == SENTINEL).all())
    return rel_err(torch.stack(got), torch.stack(want))


@gpu
@pytest.mark.parametrize("case", QK_CASES)
@pytest.mark.parametrize("D", [32, 64, 128], ids=lambda d: f"d{d}")
def test_qknorm_rope_cache_vs_float64(D, case):
    from mlx_audio_b200 import ops
    Hq, Hkv = 4, 2
    B, S, nslots, smax, theta, base, slot, rot, norms, mrope, kw = _qk_case(case, D)
    qkv = _rand(B, S, (Hq + 2 * Hkv) * D, seed=D + len(case))
    qn, kn = (1 + 0.1 * _rand(D, seed=D + 1), 1 + 0.1 * _rand(D, seed=D + 2)) if norms else (None, None)
    kbuf = torch.full((nslots, smax + 4, Hkv * D), SENTINEL, device=DEV)        # 4 rows past smax: must stay untouched
    vbuf = kbuf.clone()
    q = ops.qknorm_rope_cache(qkv.to(DEV), Hq, Hkv, D, kbuf[:, :smax], vbuf[:, :smax], q_norm=None if qn is None else qn.to(DEV),
                              k_norm=None if kn is None else kn.to(DEV), eps=1e-6, mrope=mrope, theta=theta, **kw)
    ref = dict(q_norm=qn, k_norm=kn, eps=1e-6, mrope=mrope, theta=theta)
    qr, kr, vr = rope_ref(qkv, Hq, Hkv, D, rot, **ref)
    live = [(b, s) for b in range(B) for s in range(S) if base[b] + s >= 0]        # left-padding rows: q unspecified, nothing cached
    eq = rel_err(torch.stack([q.cpu()[b, s] for b, s in live]), torch.stack([qr[b, s] for b, s in live]))
    ek = _check_cache(kbuf, vbuf, kr, vr, base, slot, smax)
    msg = f"\n[rope] d{D} {case}: q {eq:.1e} k {ek:.1e}"
    assert eq < TOL_ROPE and ek < TOL_ROPE, msg
    if case in ("pos3-mrope", "large-pos-past-smax"):      # negative control: float32 angles
        e32 = rel_err(q, rope_ref(qkv, Hq, Hkv, D, rot, **ref, angle_dtype=torch.float32)[0])
        msg += f" float32 angles {e32:.1e}"
        assert e32 > NEG * TOL_ROPE, msg
    if case == "pos3-mrope" and D == 128:                   # negative control: the sections of the wrong mrope_section entries
        ew = rel_err(q, rope_ref(qkv, Hq, Hkv, D, rot, **dict(ref, mrope=(24, 20)))[0])
        msg += f" sections (24, 20) {ew:.1e}"
        assert ew > NEG * TOL_ROPE, msg
    print(msg)


@gpu
@pytest.mark.parametrize("D", [32, 64, 128], ids=lambda d: f"d{d}")
def test_scalar_and_per_row_bases_are_bit_identical(D):
    """Host base, device base and every row at that base through ``base_rows`` / identity ``slot``: the same q, caches and decode
    attention bit for bit."""
    from mlx_audio_b200 import ops
    Hq, Hkv, B, S, base, rows = 4, 2, 3, 4, 21, 64
    qkv = _rand(B, S, (Hq + 2 * Hkv) * D, seed=70 + D).to(DEV)
    kc0, vc0 = _rand(B, rows, Hkv * D, seed=71).to(DEV), _rand(B, rows, Hkv * D, seed=72).to(DEV)
    kw = dict(q_norm=(1 + 0.1 * _rand(D, seed=73)).to(DEV), k_norm=(1 + 0.1 * _rand(D, seed=74)).to(DEV), eps=1e-6, theta=1e6,
              mrope=(20, 20))
    outs = []
    for rows_kw in (dict(base=base), dict(base_dev=_i32([base])), dict(base_rows=_i32([base] * B), slot=_i32(list(range(B))))):
        kc, vc = kc0.clone(), vc0.clone()
        q = ops.qknorm_rope_cache(qkv, Hq, Hkv, D, kc, vc, **kw, **rows_kw)
        a = ops.attn_decode(q, kc, vc, Hq, Hkv, D, scale=D ** -0.5, max_k=rows, **rows_kw)
        outs.append((q, kc, vc, a))
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(outs[0], o))


# ------------------------------------------------------------------------------------------------------------ attention
def _caches(nslots, rows, width, windows, seed):
    """Random K / V caches [nslots, rows, width], NaN outside the key windows {slot: (lo, hi)} (whole slots when absent)."""
    kc, vc = _rand(nslots, rows, width, seed=seed), _rand(nslots, rows, width, seed=seed + 1)
    for c in (kc, vc):
        for s in range(nslots):
            lo, hi = windows.get(s, (0, 0))
            c[s, :max(lo, 0)] = float("nan")
            c[s, max(hi, lo, 0):] = float("nan")
    return kc, vc


def _windows(base, slot, kv_start, S, max_k):
    """{slot: (first, end)} cache rows some query of the row may see."""
    return {slot[b]: (kv_start[b], min(base[b] + S, max_k)) for b in range(len(base))}


def _check_attn(got, want, label):
    e = rel_err(got, want)
    assert e < TOL_ATTN, (label, e)
    got = got.cpu()
    assert bool((got[want == 0] == 0).all()), label                 # queries with no visible key: exact zeros
    return e


DEC_D = [32, 64, 128]


@gpu
@pytest.mark.parametrize("S", [1, 5, 300], ids=lambda s: f"S{s}")
@pytest.mark.parametrize("G", [1, 2, 4, 8], ids=lambda g: f"gqa{g}")
@pytest.mark.parametrize("D", DEC_D, ids=lambda d: f"d{d}")
def test_attn_decode_vs_float64(D, G, S):
    """B = 4 rows at ragged ``base_rows`` (row 1 at -2: its first queries are left padding), a slot map with gaps over 6 cache batches,
    ``kv_start`` (row 0 from key 7, row 3 past its last key)."""
    from mlx_audio_b200 import ops
    Hkv = 2
    Hq = G * Hkv
    nslots, rows = 6, 512
    base, slot, ks = [40, -2, 17, 9], [5, 0, 3, 1], [7, 0, 0, 9 + S + 5]
    q = _rand(4, S, Hq * D, seed=D + G + S, scale=1.5)
    kc, vc = _caches(nslots, rows, Hkv * D, _windows(base, slot, ks, S, rows), seed=D * G + S)
    want = cache_attn_ref(q, kc, vc, Hq, Hkv, D, base, slot, ks, rows, D ** -0.5)
    got = ops.attn_decode(q.to(DEV), kc.to(DEV), vc.to(DEV), Hq, Hkv, D, scale=D ** -0.5, base_rows=_i32(base), slot=_i32(slot),
                          kv_start=_i32(ks))
    print(f"\n[attn_decode] d{D} gqa{G} S{S}: {_check_attn(got, want, 'decode'):.1e}")


@gpu
@pytest.mark.parametrize("D", DEC_D, ids=lambda d: f"d{d}")
def test_attn_decode_max_k_clamp_host_and_device_base(D):
    """Base 50, S = 6, max_k = 53: queries 3.. stop at key 52 (klen = min(base + s + 1, max_k)); B = 2 with kv_start [0, 20]; the host
    and the device base give the same bits."""
    from mlx_audio_b200 import ops
    Hq, Hkv, S, base, max_k = 4, 1, 6, 50, 53
    q = _rand(2, S, Hq * D, seed=80 + D, scale=1.5)
    ks = [0, 20]
    kc, vc = _caches(2, 64, Hkv * D, _windows([base] * 2, [0, 1], ks, S, max_k), seed=81 + D)
    want = cache_attn_ref(q, kc, vc, Hq, Hkv, D, [base] * 2, None, ks, max_k, D ** -0.5)
    args = (q.to(DEV), kc.to(DEV), vc.to(DEV), Hq, Hkv, D)
    host = ops.attn_decode(*args, scale=D ** -0.5, base=base, kv_start=_i32(ks), max_k=max_k)
    dev = ops.attn_decode(*args, scale=D ** -0.5, base_dev=_i32([base]), kv_start=_i32(ks), max_k=max_k)
    _check_attn(host, want, "host base")
    assert torch.equal(host, dev)


@gpu
@pytest.mark.parametrize("max_k", [12032, 12288, 12289, 49152], ids=["smem-47k", "smem-default", "smem-opt-in", "smem-limit"])
@pytest.mark.parametrize("D", DEC_D, ids=lambda d: f"d{d}")
def test_attn_decode_long_cache(D, max_k):
    """A cache of max_k keys: the scores take max_k floats of dynamic shared memory.  Base max_k - 2, S = 4: the last two queries are
    clamped to max_k keys; the rows past max_k are NaN.  At 12288 keys (48 KB of scores) the launch used to fail with an invalid
    argument: the host opted in only above 48 KB of dynamic memory, but without the opt-in the kernel's static shared memory comes
    out of the same 48 KB.  The host now reads the function's dynamic limit and opts in above it."""
    from mlx_audio_b200 import ops
    Hq, Hkv, S, base = 2, 1, 4, max_k - 2
    q = _rand(1, S, Hq * D, seed=90 + D, scale=1.5)
    kc, vc = _caches(1, max_k + 64, Hkv * D, {0: (0, max_k)}, seed=91 + D)
    want = cache_attn_ref(q, kc, vc, Hq, Hkv, D, [base], None, None, max_k, D ** -0.5)
    got = ops.attn_decode(q.to(DEV), kc.to(DEV), vc.to(DEV), Hq, Hkv, D, scale=D ** -0.5, base=base, max_k=max_k)
    print(f"\n[attn_decode long] d{D} max_k {max_k}: {_check_attn(got, want, 'long'):.1e}")


@gpu
def test_attn_decode_rejects_max_k_past_the_shared_memory_limit():
    from mlx_audio_b200 import ops
    q, kc = torch.zeros(1, 1, 128, device=DEV), torch.zeros(1, 8, 128, device=DEV)
    with pytest.raises(ValueError, match="max_k"):
        ops.attn_decode(q, kc, kc, 1, 1, 128, scale=0.1, base=0, max_k=48 * 1024 + 1)


PF_KV = [0, 37, 64, 150]


@gpu
@pytest.mark.parametrize("kv", PF_KV, ids=["kv0", "kv37-mask", "kv64-skip1", "kv150-skip2"])
@pytest.mark.parametrize("S", [64, 65, 127, 200], ids=lambda s: f"S{s}")
def test_attn_prefill_vs_float64(S, kv):
    """B = 2 through a slot map: row 0 at base 130 from key ``kv`` (64 and 150 skip whole key tiles before it; queries before key 150
    see nothing), row 1 at base -70 (its first 64-row query tile is all left padding: exact zeros without a key tile) from key kv / 3.
    Once with max_k the cache size and once with max_k = 130 + S - 10 < base + S; each time within the bound of float64 and of
    ``attn_decode`` on the same inputs."""
    from mlx_audio_b200 import ops
    Hq, Hkv, D, rows = 4, 2, 128, 512
    base, slot, ks = [130, -70], [2, 0], [kv, kv // 3]
    q = _rand(2, S, Hq * D, seed=S + kv, scale=1.5)
    for max_k in (rows, 130 + S - 10):
        kc, vc = _caches(3, rows, Hkv * D, _windows(base, slot, ks, S, max_k), seed=S * kv + max_k)
        want = cache_attn_ref(q, kc, vc, Hq, Hkv, D, base, slot, ks, max_k, D ** -0.5)
        args = (q.to(DEV), kc.to(DEV), vc.to(DEV), Hq, Hkv, D)
        kw = dict(scale=D ** -0.5, base_rows=_i32(base), slot=_i32(slot), kv_start=_i32(ks), max_k=max_k)
        got = ops.attn_prefill(*args, **kw)
        e = _check_attn(got, want, f"prefill max_k {max_k}")
        assert float(got[1, :64].abs().max()) == 0.0
        dec = ops.attn_decode(*args, **kw)
        ed = float((got - dec).abs().max()) / float(want.abs().max())
        assert ed < TOL_ATTN, (max_k, ed)
        print(f"\n[attn_prefill] S{S} kv{kv} max_k {max_k}: {e:.1e} (vs decode {ed:.1e})")


@gpu
def test_attn_prefill_host_and_device_base():
    """Base 100 from the host and from the device (S = 130, kv_start [64, 0]): float64 within the bound, the same bits."""
    from mlx_audio_b200 import ops
    Hq, Hkv, D, S, base, rows = 4, 2, 128, 130, 100, 256
    q = _rand(2, S, Hq * D, seed=110, scale=1.5)
    ks = [64, 0]
    kc, vc = _caches(2, rows, Hkv * D, _windows([base] * 2, [0, 1], ks, S, rows), seed=111)
    want = cache_attn_ref(q, kc, vc, Hq, Hkv, D, [base] * 2, None, ks, rows, D ** -0.5)
    args = (q.to(DEV), kc.to(DEV), vc.to(DEV), Hq, Hkv, D)
    host = ops.attn_prefill(*args, scale=D ** -0.5, base=base, kv_start=_i32(ks), max_k=rows)
    dev = ops.attn_prefill(*args, scale=D ** -0.5, base_dev=_i32([base]), kv_start=_i32(ks), max_k=rows)
    _check_attn(host, want, "prefill host base")
    assert torch.equal(host, dev)


@gpu
@pytest.mark.parametrize("kernel", ["decode", "prefill"])
def test_attention_bound_discriminates(kernel):
    """Negative controls on a cache with no NaN rows: references whose causal bound is one key short (base + s) or long (base + s + 2),
    or that ignore kv_start, are each more than 5x the bound away from the kernel."""
    from mlx_audio_b200 import ops
    Hq, Hkv, D, rows = 4, 2, 128, 256
    S = 5 if kernel == "decode" else 65
    base, ks = [30, 12], [5, 3]
    q = _rand(2, S, Hq * D, seed=120, scale=1.5)
    kc, vc = _rand(2, rows, Hkv * D, seed=121), _rand(2, rows, Hkv * D, seed=122)
    fn = ops.attn_decode if kernel == "decode" else ops.attn_prefill
    got = fn(q.to(DEV), kc.to(DEV), vc.to(DEV), Hq, Hkv, D, scale=D ** -0.5, base_rows=_i32(base), kv_start=_i32(ks), max_k=rows)

    def err(**over):
        a = dict(kv_start=ks, bound_shift=0)
        a.update(over)
        return rel_err(got, cache_attn_ref(q, kc, vc, Hq, Hkv, D, base, None, a["kv_start"], rows, D ** -0.5, a["bound_shift"]))
    e = {"ok": err(), "short": err(bound_shift=-1), "long": err(bound_shift=1), "no kv_start": err(kv_start=None)}
    print(f"\n[attn controls] {kernel}: {e}")
    assert e["ok"] < TOL_ATTN and min(e["short"], e["long"], e["no kv_start"]) > NEG * TOL_ATTN, e


# ------------------------------------------------------------------------------------------------------------ SwiGLU
SWIGLU_GRID = 132 * 16 * 256          # lm.cu caps the grid at 132 x 16 CTAs of 256 threads: larger inputs take the grid-stride loop


@gpu
@pytest.mark.parametrize("interleaved", [False, True], ids=["halves", "interleaved"])
@pytest.mark.parametrize("rows,I,pad,grid_stride", [(3, 1000, 0, False), (7, 300, 20, False), (300, 2000, 8, True)],
                         ids=["small", "strided", "grid-stride"])
def test_swiglu_vs_float64(rows, I, pad, grid_stride, interleaved):
    """Gate / up as halves or interleaved pairs; rows strided by ``pad`` extra columns (input and output); more than one grid of
    elements.  Negative control: the other layout."""
    from mlx_audio_b200 import ops
    assert (rows * I > SWIGLU_GRID) == grid_stride
    x = _rand(rows, 2 * I, seed=rows + I, scale=3.0)
    xd = torch.zeros(rows, 2 * I + pad, device=DEV)[:, :2 * I]
    xd.copy_(x)
    out = torch.zeros(rows, I + pad, device=DEV)[:, :I]
    ops.swiglu(xd, out=out, interleaved=interleaved)
    x = x.double()

    def ref(il):
        g, u = (x[:, 0::2], x[:, 1::2]) if il else (x[:, :I], x[:, I:])
        return torch.nn.functional.silu(g) * u
    e, e_other = rel_err(out, ref(interleaved)), rel_err(out, ref(not interleaved))
    assert e < TOL_SWIGLU and e_other > NEG * TOL_SWIGLU, (e, e_other)
