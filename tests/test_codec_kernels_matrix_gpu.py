"""Codec kernels (csrc/codec.cu, csrc/dac.cu, csrc/encodec.cu, csrc/bigvgan.cu, csrc/vocos.cu) against float64 on every dispatch
branch.  Mimi and the Qwen3-TTS speech tokenizer decode codes with ``rvq_decode`` and encode with ``rvq_encode`` (mode 0); SNAC
encodes with ``rvq_encode`` (mode 1) and decodes with ``snac_from_codes``; DAC runs ``dac_rvq_encode`` / ``dac_from_codes``; EnCodec
runs the pad / GroupNorm / normalise / overlap-add chunk ops and ``encodec_lstm``; BigVGAN runs ``aa_snakebeta``; Vocos runs
``vocos_dwnorm`` and ``vocos_istft_head``.

Where each kernel and branch is run:
- rvq_decode_kernel: ``test_rvq_decode_vs_float64[nq*-dim*]`` for nq 1, 2, 8, 32 and dim 4, 124, 128, 132, 512 (124 and 132 leave
  lanes past ``d < dim`` in the last 128-column pass), each through a codes view of a wider buffer (level stride T + 5, batch stride
  (nq + 2)(T + 5)) into an ``out=`` view with out_ld = dim + 8, whose pad columns must keep their NaN.  ``test_rvq_decode_rows``
  runs B T = 16 895, 16 896, 16 897 and 40 000 rows: the grid is capped at 132 * 16 CTAs of 8 warps = 16 896 rows, so the larger
  ones take the grid-stride loop.  ``test_rvq_decode_code_range`` puts ``code == bins`` and ``code == -1`` in and expects ValueError.
- rvq_encode_kernel: ``test_rvq_encode_vs_float64[mode*-R*-bins*-D*]``, mode 0 (Mimi residual, 3 levels) and mode 1 (SNAC cosine),
  R 1, 3, 4, 5 (partial VQ_ROWS = 4 tiles), bins 1, 255, 256, 257, 2048 (threads that own no code, one code per thread, a second
  code for thread 0, eight per thread), D 4, and D 6388 (4 x 6388 x 8 + 384 = 200 KiB exactly, the largest tile).  Half the code
  book's rows repeat earlier rows at shuffled indices, and half the inputs sit next to a repeated row: exact ties within a thread,
  across lanes and across warps must take the lower index, at every level.  Codes go to a transposed ``out`` (row stride 1).
- snac_from_codes_kernel: ``test_snac_from_codes_vs_float64[L*-cd*-dim*]``: 1 to 4 levels with strides (1), (1, 2), (1, 2, 4),
  (1, 2, 4, 8) at T 13, 14, 12 and 24 (the first three not multiples of the 8-frame CTA), cd 1, 8, 16, dim 1, 255, 768, B = 3, no
  bias on odd levels.  ``test_snac_from_codes_checks`` covers out-of-range codes and a T that a stride does not divide.
- dac_rvq_encode_kernel / dac_from_codes_kernel: ``test_dac_vs_float64[D*-L*-B*-T*]`` at D 4, 1024 and 2560 (2 x 8 x 2560 x 4 =
  160 KiB, the largest tile), 1, 9 and 32 levels whose codebook_dim alternates 16 and 1, B = 2 with T = 13 (CTA 1 holds frames of
  both items).  The same test runs the ``from_latents`` route on the encoder's latents and ``dac_from_codes`` on its codes (z_p
  bit-exact).  D = 2561 is rejected in ``test_argument_checks``.
- encodec_pad_kernel: ``test_encodec_pad[*]``: reflect and zero padding, pad T - 1 on both sides, asymmetric and one-sided pads,
  T = 1, no coeffs (bit-exact copy), coeffs, coeffs + ELU, and a residual add, on row-strided views of every other batch item.
- encodec_gn_partials_kernel + encodec_gn_coeffs_kernel: ``test_encodec_gn_coeffs[*]`` at T C 3, 3200 and 44 800 (past 64 x 256:
  the grid-stride loop), rows of mean 1e3 with std 1e-3, gamma / beta None or given; each row alone gives the same bits.
- encodec_normalize_kernel: ``test_encodec_normalize[*]`` at C 1, 2, L 7 and 3000 (past the 1024 threads), mask None, partial and
  all zero, and an all-zero chunk (scale exactly float32(1e-8), output 0).
- encodec_ola_kernel: ``test_encodec_ola[*]``: stride < L and = L, N = 1, t_out at and below the full length (the last frame cut),
  scale None or per frame.
- encodec_lstm_kernel<H, RB>: ``test_encodec_lstm[H*-R*-T*]`` at H 128 (cluster of 4, NC 8, Q 2), 256 (8, 16, 4) and 512 (16, 32,
  8), R = 1 (RB = 1), R = 5 (RB = 4: a second cluster with one live row), R = 2 at T = 1; skip None or given.  Every row must equal
  its R = 1 call bit for bit, and the error word must stay 0.
- aa_snakebeta_kernel: ``test_aa_snakebeta[C*]`` at C 1, 47, 48 (tile = C), 49, 50, 100 (32-channel tiles, the last one partial),
  each at L 1 to 7, 63, 64, 65 (a second 64-row tile of one row) and 130, B = 3 on strided views, each row bit-identical to a
  single-row call.  Every third channel has alpha ~ 1e4, so |alpha u| > 8192 (the ``sinf`` branch of b2a_sin) is asserted to occur.
  ``test_aa_snakebeta_planes[*]`` writes hi + lo (x2) and hi only (x1) planes with cpad = 64 ceil(C / 64) > C: pad channels
  exactly 0, hi and lo exactly the split of the fp32 result.
- vocos_dwnorm_kernel<4 | 8, ADA>: ``test_vocos_dwnorm[C*-K*-*]`` at C 4, 64 (idle lanes), 132, 512, 516 (NV = 8, partial lanes),
  K 0, 1, 3, 15, affine, w only, b only and ada, conv bias on and off, L 1, 15, 16, 17, on a row-strided x; planes next to fp32 where
  C % 64 == 0.  ``[C1024-K1-*]`` and ``[C1024-K15-*]``: K = 15 at C = 1024 fills exactly the 120 KiB tile.
- vocos_istft_head_kernel: ``test_vocos_istft_head[n*-hop*-T*]`` for n_fft / hop 16 / 4, 1024 / 128, 2048 / 256 (a 256-sample run
  overlaps 68, 10 and 9 frames: more than HD_FCH = 6, the second spectrum chunk), 2048 / 2048 and 1024 / 300 (a hop that does not
  divide n_fft), T 1, 2, 3, 937, log-magnitudes above ln 100 (clipped), h_ld > n_fft + 2 and B = 3, each row bit-identical.
- Host checks: ``test_argument_checks``: every B2A_CHECK_ARG / B2A_E_UNSUPPORTED of the five files that ``ops`` reaches raises
  with its message and launches nothing.

Tolerances (u = 2^-24).  Each assertion divides the error by its bound and requires a ratio <= 1; the largest ratio measured on an
H100 80GB HBM3 (700 W) is given with each bound.  Each family has a negative control that must fail by more than NEG = 5 times.
- rvq_decode: bit-exact against the float32 left-to-right sum over levels; against float64 within (nq - 1) u sum_q |e_q|.
  Measured: 0 at nq = 1, 1.0 at nq = 2 (one rounding, which reaches its half-ulp bound), 0.43 at nq = 8, 0.10 at nq = 32, 0.98
  on the long runs.  Negative control: level 0's codes shifted by one.
- rvq_encode / DAC search: scores are float64 fma chains; two scores differ from float64 by at most (D + 8) 2^-53 (sum |x e| + |c|)
  each, so codes must equal the float64 arg-min wherever the best-to-second margin exceeds twice that.  DAC's z_e carries the fp32
  error below; |dxn| <= 2 |dz_e| / |z_e| moves any score gap by at most 8 |dz_e| / |z_e|.  Negative control: the reference's ties
  resolved to the higher index.
- snac_from_codes: fp32 chain of sum_l (cd + 1) terms (bias then the cd fma per level): (sum_l (cd_l + 1)) u sum |terms|.
  Measured: 0.50.  Negative control: level 0's codes shifted by one.
- DAC encode: per level z_e = (D + 1) u (|r| |w_in| + |b_in|) plus |w_in|^T e_r, e_r / e_zq accumulating the out-projection chain
  (cd + 1) u (|e| |w_out| + |b_out|) and one rounding u |r| / u |zq| per level.  The reference follows the kernel's codes (ties
  inside the margin may pick either).  Loss: sum_q mean(2 |z_e - e| e_z + e_z^2).  from_codes: the snac chain bound.
  Measured: latents 0.39, z_q 0.12 (0.12 from latents), from_codes 0.23, loss 4e-5.  Negative control: z_q without the last level's bias.
- encodec_pad: bit-exact without coeffs; with them u |a| for the fma, ELU (expm1f within 2 ulp) carries it times e^a plus 2 u |y|,
  the residual add u |y|.  Measured: 1.0 (the fma's rounding
  reaches its half-ulp bound).  Negative control: the shift left out.
- encodec_gn_coeffs: the one-pass float64 variance moves by (3 k + 4) 2^-53 mean(x^2) (k = the summation depth); scale within
  (2 u + dvar / 2 (var + eps)) |scale| (two fp32 roundings), shift within u |shift| + 2 u |mean scale| + |mean| dscale.
  Measured: scale 0.85, shift 0.88.  Negative control: eps left out.
- encodec_normalize: the fp32 mono mix (exact at C = 1, u |x0 + x1| at C = 2), the cast and the + 1e-8: dscale <= u rms(|mono|)
  + 2 u scale; y within u |y| + |x| dscale / scale^2.  Measured: scale 0.53,
  y 0.61.  Negative control: the mono mix taken without the mask.
- encodec_ola: weights within 2 u, fma chain K u sum w |v| plus 2 u sum |v|, the weight sum K u sum w + 2 K u, carried through the
  division plus u |out|.  Measured: 0.20.  Negative control: the frames in reverse order.
- encodec_lstm: 2e-5 max |h| (test_encodec_gpu.py's bound at H = 512): the fast-math gates (__expf, __fdividef, about 2^-21
  relative) and the fp32 dot products give ~1e-6 per step, and the forget gate (< 1) keeps the recurrence from compounding it
  over the 40 steps here.  Measured: 0.015.  Negative control: the i and f gates swapped.
- aa_snakebeta: up-sampling 6 u sum |2 f x|; the argument a u adds |a| du + u |a u|; __sinf after the reduction is within 2^-21;
  sin^2 and the fma carry it with u |v|; the 12-tap down-sampling sums sum |f| dv + 12 u sum |f v|.  Measured: 0.14.
  Negative control: f_up reversed.
- vocos_dwnorm: the conv chain (K + 1) u (sum |w x| + |b|); the mean (NV + 8) u mean |v|; centred values those plus u |d|; the
  variance 2 |e_d| / |d| + (4 NV + 7) u relative; rsqrtf 2 ulp; products and affine one rounding each.  Doubled for second-order
  terms.  Measured: 0.44.  Negative control: the conv taps reversed.
- vocos_istft_head: per frame (4 sqrt(N) + 16) u S (S = sum_k wgt_k |X_k| / N: expf, sincosf and the rounded twiddle angle
  2 i / N within 12 u per term, the fma chain over N / 2 + 1 bins), through the overlap-add (K u sum w |y|), the window sum
  (K u sum w) and the division, plus u |out|.  Measured: 0.10 at n_fft 16,
  0.04 to 0.06 above.  Negative control: the phase sign flipped.
"""
import math

import pytest
import torch

from oracle import bigvgan as OB
from oracle import codec as OC
from oracle import dac as ODAC
from oracle import encodec as OE
from oracle import vocos as OV

gpu = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
U64 = 2.0 ** -53
NEG = 5


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _report(name, ratio):
    print(f"{name}: max error / bound = {ratio:.3g}")


def _ratio(err, bound):
    err, bound = torch.as_tensor(err, dtype=torch.float64), torch.as_tensor(bound, dtype=torch.float64)
    if err.numel() == 0:
        return 0.0
    return float((err / bound.clamp_min(1e-300)).max())


def _check(name, got, ref, bound):
    """got (device or CPU) against the float64 ref within bound, elementwise; returns the ratio."""
    err = (got.double().cpu() - ref).abs()
    r = _ratio(err, bound)
    _report(name, r)
    assert r <= 1.0, (name, r)
    return r


def _neg(name, got, bad_ref, bound):
    r = _ratio((got.double().cpu() - bad_ref).abs(), bound)
    _report(name + " (negative control)", r)
    assert r > NEG, (name, r)


def _wide(t, extra=7, off=3, every=2):
    """A [B, L, C] float32 tensor on the device as a view: channels offset inside wider rows, every other batch item."""
    B, L, C = t.shape
    buf = torch.full((every * B, L, C + extra), float("nan"))
    buf[::every, :, off:off + C] = t
    v = buf.to(DEV)[::every, :, off:off + C]
    assert not v.is_contiguous()
    return v


# ================================================================================================================== rvq_decode
def rvq_decode_ref(codes, cb):
    """codes int64 [B, nq, T], cb float32 [nq, bins, dim] -> (fp32 left-to-right sum, float64 sum, float64 sum of |e|) [B, T, dim]."""
    g = [cb[q][codes[:, q]] for q in range(cb.shape[0])]
    acc = g[0].clone()
    for e in g[1:]:
        acc = acc + e
    return acc, sum(e.double() for e in g), sum(e.double().abs() for e in g)


RVQD_CASES = [(nq, dim) for nq in (1, 2, 8, 32) for dim in (4, 124, 128, 132, 512)]


@gpu
@pytest.mark.parametrize("nq,dim", RVQD_CASES, ids=[f"nq{n}-dim{d}" for n, d in RVQD_CASES])
def test_rvq_decode_vs_float64(nq, dim):
    from mlx_audio_b200 import ops
    B, T, bins = 2, 37, 64
    g = _gen(nq * 1000 + dim)
    cb = torch.randn(nq, bins, dim, generator=g)
    codes = torch.randint(0, bins, (B, nq, T), generator=g)
    wide = torch.randint(0, bins, (B, nq + 2, T + 5), generator=g)
    wide[:, 1:nq + 1, 2:T + 2] = codes
    cv = wide.to(DEV)[:, 1:nq + 1, 2:T + 2]
    assert cv.stride(1) == T + 5 and cv.stride(0) == (nq + 2) * (T + 5)
    out = torch.full((B, T, dim + 8), float("nan"), device=DEV)
    cbd = cb.to(DEV)
    ops.rvq_decode(cv, cbd, out=out[..., :dim])
    y = out[..., :dim].cpu()
    assert torch.isnan(out[..., dim:]).all()
    assert torch.equal(ops.rvq_decode(codes.to(DEV), cbd).cpu(), y)
    acc, s64, a64 = rvq_decode_ref(codes, cb)
    assert torch.equal(y, acc)                                          # nq = 1: the gather itself
    bound = max(nq - 1, 1) * U * a64
    _check(f"rvq_decode nq{nq} dim{dim}", y, s64, bound)
    bad = codes.clone()
    bad[:, 0] = (bad[:, 0] + 1) % bins
    _neg(f"rvq_decode nq{nq} dim{dim}", y, rvq_decode_ref(bad, cb)[1], bound)


@gpu
@pytest.mark.parametrize("B,T", [(1, 16895), (1, 16896), (1, 16897), (2, 20000)])
def test_rvq_decode_rows(B, T):
    from mlx_audio_b200 import ops
    nq, bins, dim = 3, 32, 132
    g = _gen(T)
    cb = torch.randn(nq, bins, dim, generator=g)
    codes = torch.randint(0, bins, (B, nq, T), generator=g)
    y = ops.rvq_decode(codes.to(DEV), cb.to(DEV)).cpu()
    acc, s64, a64 = rvq_decode_ref(codes, cb)
    assert torch.equal(y, acc)
    _check(f"rvq_decode rows {B * T}", y, s64, (nq - 1) * U * a64)


@gpu
def test_rvq_decode_code_range():
    from mlx_audio_b200 import ops
    cb = torch.randn(2, 16, 8, device=DEV)
    for bad in (16, -1):
        codes = torch.zeros(1, 2, 5, dtype=torch.int64)
        codes[0, 1, 3] = bad
        with pytest.raises(ValueError, match="code index out of range"):
            ops.rvq_decode(codes.to(DEV), cb)
    ops.rvq_decode(torch.full((1, 2, 5), 15, dtype=torch.int64, device=DEV), cb)     # code == bins - 1 is legal


# ================================================================================================================== rvq_encode
def _tied_codebook(nq, bins, D, g, decay):
    """[nq, bins, D] float32 whose first nu = ceil(bins / 2) rows are distinct and whose other rows repeat them at shuffled indices
    (so the lowest index holding a row is the row's own index), with level q scaled by decay^q; returns (table, perm, nu)."""
    nu = (bins + 1) // 2
    base = torch.randn(nq, nu, D, generator=g) * torch.tensor([decay ** q for q in range(nq)])[:, None, None]
    perm = torch.cat([torch.arange(nu), torch.randperm(nu, generator=g)[:bins - nu]])
    return base[:, perm].contiguous(), perm, nu


def rvq_encode_ref(x, table, perm, nu, mode, follow=None, ties="low"):
    """Float64 nearest-code search on the distinct rows.  -> (codes [R, nq], margin [R, nq], bound [R, nq]).  ``follow``: codes
    [R, nq] whose rows update the residual (the kernel's), so that later levels are compared on the kernel's path."""
    nq = table.shape[0]
    r = x.double()
    if mode == 1:
        r = r / r.norm(dim=1, keepdim=True).clamp_min(1e-12)
    codes, margins, bounds = [], [], []
    for q in range(nq):
        e = table[q, :nu].double()
        if mode == 0:
            c2 = (e ** 2).sum(1) / 2
            s = c2[None] - r @ e.T
            sb = (r.abs() @ e.abs().T + c2[None]).amax(1)
        else:
            c2 = (e ** 2).sum(1)
            xn2 = (r ** 2).sum(1, keepdim=True)
            s = (xn2 - 2 * (r @ e.T)) + c2[None]
            sb = (2 * r.abs() @ e.abs().T + xn2 + c2[None]).amax(1)
        D = x.shape[1]
        if nu > 1:
            two = torch.topk(s, 2, dim=1, largest=False)
            best, margin = two.indices[:, 0], two.values[:, 1] - two.values[:, 0]
        else:
            best, margin = torch.zeros(x.shape[0], dtype=torch.int64), torch.full((x.shape[0],), math.inf, dtype=torch.float64)
        idx = best.clone()
        if ties == "high":                                              # negative control: the highest index holding the row
            for i in range(len(idx)):
                idx[i] = int(torch.nonzero(perm == best[i]).max())
        codes.append(idx)
        margins.append(margin)
        bounds.append(2 * (D + 8) * U64 * sb)
        k = idx if follow is None else follow[:, q]
        if mode == 0:
            r = r - table[q][k].double()
    return torch.stack(codes, 1), torch.stack(margins, 1), torch.stack(bounds, 1)


RVQE_CASES = ([(0, R, bins, 4) for R in (1, 3, 4, 5) for bins in (1, 255, 256, 257, 2048)]
              + [(1, R, bins, 4) for R in (1, 3, 4, 5) for bins in (1, 255, 256, 257, 2048)]
              + [(0, 5, 2048, 6388), (0, 3, 257, 6388), (1, 5, 2048, 6388)])


@gpu
@pytest.mark.parametrize("mode,R,bins,D", RVQE_CASES, ids=[f"mode{m}-R{r}-bins{b}-D{d}" for m, r, b, d in RVQE_CASES])
def test_rvq_encode_vs_float64(mode, R, bins, D):
    from mlx_audio_b200 import ops
    nq = 3 if mode == 0 else 1
    if D > 1000:
        nq = min(nq, 2)
    g = _gen(mode * 100000 + R * 10000 + bins + D)
    table, perm, nu = _tied_codebook(nq, bins, D, g, 0.05)
    if mode == 1:
        table = (table.double() / table.double().norm(dim=2, keepdim=True)).float()
    # half the rows sit next to a repeated row at every level, the rest are random
    dup = perm[nu:] if bins > nu else torch.arange(nu)
    x = torch.randn(R, D, generator=g, dtype=torch.float64)
    for i in range(0, R, 2):
        x[i] = sum(table[q, int(dup[torch.randint(0, len(dup), (1,), generator=g)])].double() for q in range(nq))
        x[i] += 1e-3 * (0.05 ** (nq - 1)) * torch.randn(D, generator=g, dtype=torch.float64)
    x = x.float()
    c2 = ((table.double() ** 2).sum(-1) / (2 if mode == 0 else 1)).to(DEV).contiguous()
    out = torch.full((nq, R), -7, dtype=torch.int64, device=DEV).t()
    ops.rvq_encode(x.to(DEV), table.to(DEV).contiguous(), c2, mode=mode, out=out)
    got = out.cpu()
    assert (got >= 0).all() and (got < bins).all()
    ref, margin, bound = rvq_encode_ref(x, table, perm, nu, mode, follow=got)
    ok = margin > bound
    assert ok.float().mean() >= 0.5, ok
    assert torch.equal(got[ok], ref[ok]), (got, ref, margin)
    assert (got < nu).all(), "a repeated row won over the lower index holding the same row"
    if bins > nu:
        hi, _, _ = rvq_encode_ref(x, table, perm, nu, mode, follow=got, ties="high")
        assert not torch.equal(got[ok], hi[ok])                         # negative control: ties resolved to the higher index


# ================================================================================================================== snac_from_codes
def snac_ref(codes, strides, embs, ws, biases, T):
    """float64 from_codes: (out [B, T, dim], bound) with the fp32 chain bound of the module docstring."""
    out, absum, n = 0.0, 0.0, 0
    for c, s, e, w, b in zip(codes, strides, embs, ws, biases):
        ee = e.double()[c]                                              # [B, Tl, cd]
        z = ee @ w.double() + (0.0 if b is None else b.double())
        a = ee.abs() @ w.double().abs() + (0.0 if b is None else b.double().abs())
        out = out + torch.repeat_interleave(z, s, dim=1)
        absum = absum + torch.repeat_interleave(a, s, dim=1)
        n += e.shape[1] + 1
    return out, n * U * absum


SNAC_STRIDES = {1: ((1,), 13), 2: ((1, 2), 14), 3: ((1, 2, 4), 12), 4: ((1, 2, 4, 8), 24)}
SNAC_CASES = [(L, cd, dim) for L in (1, 2, 3, 4) for cd in (1, 8, 16) for dim in (1, 255, 768)]


def _snac_case(L, cd, dim, g, B=3, bins=300):
    strides, T = SNAC_STRIDES[L]
    codes = [torch.randint(0, bins, (B, T // s), generator=g) for s in strides]
    embs = [torch.randn(bins, cd, generator=g) for _ in strides]
    ws = [torch.randn(cd, dim, generator=g) / math.sqrt(cd) for _ in strides]
    biases = [None if l % 2 else 0.1 * torch.randn(dim, generator=g) for l in range(L)]
    return strides, T, codes, embs, ws, biases


def _dev(ts):
    return [None if t is None else t.to(DEV).contiguous() for t in ts]


@gpu
@pytest.mark.parametrize("L,cd,dim", SNAC_CASES, ids=[f"L{l}-cd{c}-dim{d}" for l, c, d in SNAC_CASES])
def test_snac_from_codes_vs_float64(L, cd, dim):
    from mlx_audio_b200 import ops
    g = _gen(L * 1000 + cd * 10 + dim)
    strides, T, codes, embs, ws, biases = _snac_case(L, cd, dim, g)
    y = ops.snac_from_codes(_dev(codes), list(strides), _dev(embs), _dev(ws), _dev(biases), dim)
    assert y.shape == (3, T, dim)
    ref, bound = snac_ref(codes, strides, embs, ws, biases, T)
    _check(f"snac L{L} cd{cd} dim{dim}", y, ref, bound)
    bad = [codes[0].clone().add_(1).remainder_(300)] + codes[1:]
    _neg(f"snac L{L} cd{cd} dim{dim}", y, snac_ref(bad, strides, embs, ws, biases, T)[0], bound)


@gpu
def test_snac_from_codes_checks():
    from mlx_audio_b200 import ops
    g = _gen(5)
    strides, T, codes, embs, ws, biases = _snac_case(2, 8, 16, g)
    for bad in (300, -1):
        c = [codes[0], codes[1].clone()]
        c[1][1, 2] = bad
        with pytest.raises(ValueError, match="code index out of range"):
            ops.snac_from_codes(_dev(c), list(strides), _dev(embs), _dev(ws), _dev(biases), 16)
    # strides (2, 1): T = 13 from the last level, which 2 does not divide
    c = [torch.zeros(3, 6, dtype=torch.int64), torch.zeros(3, 13, dtype=torch.int64)]
    n0 = ops.LAUNCHES[0]
    with pytest.raises(ValueError, match="T must be a multiple of every vq stride"):
        ops.snac_from_codes(_dev(c), [2, 1], _dev(embs), _dev(ws), _dev(biases), 16)
    assert ops.LAUNCHES[0] == n0


# ================================================================================================================== DAC
def _dac_levels(D, cds, bins, g):
    lv = []
    for cd in cds:
        cb = torch.randn(bins, cd, generator=g)
        cn = (cb.double() / cb.double().norm(dim=1, keepdim=True).clamp_min(1e-12)).float()
        lv.append(dict(w_in=torch.randn(D, cd, generator=g) / math.sqrt(D), b_in=0.1 * torch.randn(cd, generator=g), cbn=cn,
                       c2=(cn.double() ** 2).sum(1), cb=cb, w_out=0.5 * torch.randn(cd, D, generator=g) / math.sqrt(cd),
                       b_out=0.01 * torch.randn(D, generator=g)))
    return lv


def dac_encode_ref(z, levels, follow, latents=None, cn64=None):
    """Float64 ResidualVectorQuantize on z [R, D] (or from_latents on ``latents`` [R, lat_ch]) following the kernel's codes
    ``follow`` [R, nq].  -> dict of codes / margin / score bound [R, nq], latents [R, lat_ch] with their bound, z_q with its bound,
    loss with its bound."""
    R = follow.shape[0]
    r = None if z is None else z.double()
    eR = None if z is None else torch.zeros_like(r)
    zq, eZ = 0.0, 0.0
    codes, margins, sbs, lats, elats = [], [], [], [], []
    loss, eloss, off = 0.0, 0.0, 0
    for q, lv in enumerate(levels):
        cd = lv["cb"].shape[1]
        if z is None:
            ze = latents[:, off:off + cd].double()
            eze = torch.zeros_like(ze)
        else:
            wi = lv["w_in"].double()
            ze = r @ wi + lv["b_in"].double()
            eze = eR @ wi.abs() + (r.shape[1] + 1) * U * (r.abs() @ wi.abs() + lv["b_in"].double().abs())
        off += cd
        nrm = ze.norm(dim=1, keepdim=True).clamp_min(1e-12)
        xn = ze / nrm
        cn = lv["cbn"].double() if cn64 is None else cn64[q]
        s = ((xn ** 2).sum(1, keepdim=True) - 2 * xn @ cn.T) + (cn ** 2).sum(1)[None]
        # exact ties (every code of one sign at codebook_dim 1) go to the lowest index; the margin is to the next distinct score
        best = torch.argmin(s, dim=1)
        bv = s.gather(1, best[:, None])
        codes.append(best)
        margins.append((s.masked_fill(s == bv, math.inf).amin(1) - bv[:, 0]))
        sbs.append(8 * eze.norm(dim=1) / nrm[:, 0] + 2 * (cd + 8) * U64 * 4)
        lats.append(ze); elats.append(eze)
        e = lv["cb"].double()[follow[:, q]]
        d = ze - e
        loss = loss + (d ** 2).mean()
        eloss = eloss + (2 * d.abs() * eze + eze ** 2).mean() + 1e-15 * (d ** 2).mean()
        wo, bo = lv["w_out"].double(), lv["b_out"].double()
        zqi = e @ wo + bo
        chain = (cd + 1) * U * (e.abs() @ wo.abs() + bo.abs())
        zq = zq + zqi
        eZ = eZ + chain + U * zq.abs()
        if z is not None:
            r = r - zqi
            eR = eR + chain + U * r.abs()
    return dict(codes=torch.stack(codes, 1), margin=torch.stack(margins, 1), sb=torch.stack(sbs, 1), lat=torch.cat(lats, 1),
                elat=torch.cat(elats, 1), zq=zq, ezq=eZ, loss=loss, eloss=eloss)


def dac_from_codes_ref(codes, levels):
    """codes [B, nq, T] -> (z_q [B, T, D], bound, z_p [B, sum cd, T])."""
    zq, a, n, zp = 0.0, 0.0, 0, []
    for q in range(codes.shape[1]):
        lv = levels[q]
        e = lv["cb"][codes[:, q]]                                       # [B, T, cd]
        zp.append(e.transpose(1, 2))
        zq = zq + e.double() @ lv["w_out"].double() + lv["b_out"].double()
        a = a + e.double().abs() @ lv["w_out"].double().abs() + lv["b_out"].double().abs()
        n += lv["cb"].shape[1] + 1
    return zq, n * U * a, torch.cat(zp, 1)


DAC_CASES = [(4, 1, 2, 13, 37), (4, 9, 2, 13, 1024), (1024, 9, 2, 13, 1024), (1024, 32, 1, 40, 1024), (2560, 9, 2, 13, 1024),
             (2560, 32, 2, 5, 256)]


@gpu
@pytest.mark.parametrize("D,L,B,T,bins", DAC_CASES, ids=[f"D{d}-L{l}-B{b}-T{t}" for d, l, b, t, _ in DAC_CASES])
def test_dac_vs_float64(D, L, B, T, bins):
    from mlx_audio_b200 import ops
    g = _gen(D * 100 + L * 10 + T)
    cds = [16 if q % 2 == 0 else 1 for q in range(L)]
    levels = _dac_levels(D, cds, bins, g)
    dlev = [{k: v.to(DEV).contiguous() for k, v in lv.items()} for lv in levels]
    table = ops.dac_levels(dlev, DEV)
    lat_ch = sum(cds)
    z = torch.randn(B, T, D, generator=g)
    codes, lat, zq, loss = ops.dac_rvq_encode(z.to(DEV), table, L, bins, lat_ch, D)
    torch.cuda.synchronize()
    codes, lat, zq = codes.cpu(), lat.cpu(), zq.cpu()
    R = B * T
    follow = codes.permute(0, 2, 1).reshape(R, L)
    ref = dac_encode_ref(z.reshape(R, D), levels, follow)
    ok = ref["margin"] > ref["sb"]
    assert ok.float().mean() >= 0.5
    assert torch.equal(follow[ok], ref["codes"][ok])
    lat_r = lat.permute(0, 2, 1).reshape(R, lat_ch)
    _check(f"dac latents D{D} L{L}", lat_r, ref["lat"], ref["elat"])
    _check(f"dac z_q D{D} L{L}", zq.reshape(R, D), ref["zq"], ref["ezq"])
    lsum = float(loss.sum())
    _check(f"dac loss D{D} L{L}", torch.tensor([lsum]), torch.tensor([float(ref["loss"])]), torch.tensor([float(ref["eloss"])]))
    _neg(f"dac z_q D{D} L{L}", zq.reshape(R, D), ref["zq"] - levels[-1]["b_out"].double(), ref["ezq"])

    # from_latents on the encoder's own latents: no residual, codes exact where the float64 margin allows
    codes2, _, zq2, _ = ops.dac_rvq_encode(None, table, L, bins, lat_ch, D, latents=lat.to(DEV).contiguous())
    f2 = codes2.cpu().permute(0, 2, 1).reshape(R, L)
    ref2 = dac_encode_ref(None, levels, f2, latents=lat_r)
    ok2 = ref2["margin"] > ref2["sb"]
    assert torch.equal(f2[ok2], ref2["codes"][ok2]) and ok2.float().mean() >= 0.9
    _check(f"dac from_latents z_q D{D} L{L}", zq2.cpu().reshape(R, D), ref2["zq"], ref2["ezq"])

    # from_codes: z_p is the code-book rows, bit for bit; z_q within the chain bound; the first nq levels only
    for nq in sorted({1, L}):
        y, zp = ops.dac_from_codes(codes[:, :nq].to(DEV).contiguous(), table, bins, sum(cds[:nq]), D, want_zp=True)
        zr, bd, zpr = dac_from_codes_ref(codes[:, :nq], levels)
        assert torch.equal(zp.cpu(), zpr)
        _check(f"dac from_codes D{D} nq{nq}", y, zr, bd)


# ================================================================================================================== EnCodec
def pad_ref(x, pl, pr, reflect, coeffs=None, elu=False, res=None):
    """float64 encodec_pad and its bound: x [B, T, C] float32."""
    v = x.double()
    e = torch.zeros_like(v)
    if coeffs is not None:
        sc, sh = (c.double()[:, None, :] for c in coeffs)
        v = v * sc + sh
        e = (U + 4 * U64) * v.abs()                                    # the fma's rounding, plus the reference's float64 ones
        if elu:
            y = OE.elu(v)
            e = e * torch.exp(v.clamp(max=0.0)) + 2 * U * y.abs()
            v = y
    mode = "reflect" if reflect else "zero"
    v, e = OE.pad1d(v, pl, pr, mode), OE.pad1d(e, pl, pr, mode)
    if res is not None:
        v = v + res.double()
        e = e + U * v.abs()
    return v, e


PAD_CASES = [(5, 3, 4, 4, True), (5, 3, 0, 4, True), (5, 3, 4, 0, True), (17, 8, 3, 7, True), (17, 8, 3, 7, False),
             (1, 4, 2, 5, False), (1, 4, 0, 0, True), (300, 64, 6, 1, True), (40, 16, 0, 0, False)]
PAD_IDS = [f"T{t}-C{c}-{pl}-{pr}-{'reflect' if r else 'zero'}" for t, c, pl, pr, r in PAD_CASES]


@gpu
@pytest.mark.parametrize("T,C,pl,pr,reflect", PAD_CASES, ids=PAD_IDS)
def test_encodec_pad(T, C, pl, pr, reflect):
    from mlx_audio_b200 import ops
    g = _gen(T * 100 + C + pl * 7 + pr)
    B = 3
    x = torch.randn(B, T, C, generator=g)
    xd = _wide(x)
    y = ops.encodec_pad(xd, pl, pr, reflect=reflect).cpu()
    assert torch.equal(y, OE.pad1d(x.double(), pl, pr, "reflect" if reflect else "zero").float())   # a copy: bit-exact
    if reflect and pl + pr > 0 and T > 2:
        assert not torch.equal(y, OB._edge(x, pl, pr))                  # negative control: edge padding
    sc, sh = 1 + 0.5 * torch.randn(B, C, generator=g), torch.randn(B, C, generator=g)
    cd = (sc.to(DEV), sh.to(DEV))
    for elu in (False, True):
        y = ops.encodec_pad(xd, pl, pr, reflect=reflect, coeffs=cd, elu=elu)
        ref, e = pad_ref(x, pl, pr, reflect, (sc, sh), elu)
        _check(f"encodec_pad {PAD_IDS[PAD_CASES.index((T, C, pl, pr, reflect))]} elu{int(elu)}", y, ref, e)
        _neg("encodec_pad", y, pad_ref(x, pl, pr, reflect, (sc, torch.zeros_like(sh)), elu)[0], e)
    if pl == pr == 0:
        res = torch.randn(B, T, C, generator=g)
        y = ops.encodec_pad(xd, 0, 0, reflect=reflect, res=_wide(res, extra=5, off=1)).cpu()
        assert torch.equal(y, x + res)
        y = ops.encodec_pad(xd, 0, 0, reflect=reflect, coeffs=cd, elu=True, res=res.to(DEV))
        ref, e = pad_ref(x, 0, 0, reflect, (sc, sh), True, res)
        _check("encodec_pad coeffs+elu+res", y, ref, e)


def gn_ref(x, gamma, beta, eps=1e-5):
    """float64 GroupNorm(1, C) folded: (scale, shift, bounds) [B, C] for x [B, T, C] float32."""
    v = x.double()
    B, T, C = v.shape
    n = T * C
    mean = v.mean(dim=(1, 2))
    var = ((v - mean[:, None, None]) ** 2).mean(dim=(1, 2))
    rstd = 1.0 / torch.sqrt(var + eps)
    gm = torch.ones(C, dtype=torch.float64) if gamma is None else gamma.double()
    bt = torch.zeros(C, dtype=torch.float64) if beta is None else beta.double()
    sc = rstd[:, None] * gm[None]
    sh = bt[None] - mean[:, None] * sc
    k = math.ceil(n / (64 * 256)) + 5 + 8 + 64
    dvar = (3 * k + 4) * U64 * (v ** 2).mean(dim=(1, 2))
    esc = (2 * U + dvar / (2 * (var + eps)) + 2 * U64)[:, None] * sc.abs()
    esh = U * sh.abs() + 2 * U * (mean[:, None] * sc).abs() + mean.abs()[:, None] * esc
    return sc, sh, esc, esh


GN_CASES = [(1, 3, True), (100, 32, True), (100, 32, False), (700, 64, True), (700, 64, False)]


@gpu
@pytest.mark.parametrize("T,C,affine", GN_CASES, ids=[f"T{t}-C{c}-{'affine' if a else 'none'}" for t, c, a in GN_CASES])
def test_encodec_gn_coeffs(T, C, affine):
    from mlx_audio_b200 import ops
    g = _gen(T * 10 + C)
    x = torch.stack([torch.randn(T, C, generator=g), 1e3 + 1e-3 * torch.randn(T, C, generator=g),
                     2 + 5 * torch.randn(T, C, generator=g)]).float()
    gamma = 1 + 0.3 * torch.randn(C, generator=g) if affine else None
    beta = 0.2 * torch.randn(C, generator=g) if affine else None
    xd = _wide(x)
    dv = lambda t: None if t is None else t.to(DEV)                     # noqa: E731
    sc, sh = ops.encodec_gn_coeffs(xd, dv(gamma), dv(beta))
    rs, rh, es, eh = gn_ref(x, gamma, beta)
    _check(f"gn scale T{T} C{C}", sc, rs, es)
    _check(f"gn shift T{T} C{C}", sh, rh, eh)
    bs, bh, _, _ = gn_ref(x, gamma, beta, eps=0.0)
    _neg(f"gn scale T{T} C{C}", sc, bs, es)
    for b in range(3):
        s1, h1 = ops.encodec_gn_coeffs(xd[b:b + 1], dv(gamma), dv(beta))
        assert torch.equal(s1[0], sc[b]) and torch.equal(h1[0], sh[b])


def normalize_ref(x, mask):
    """float64 encodec_normalize with its bounds: x [R, L, C] float32, mask [R, L] bool or None."""
    v = x.double()
    m = torch.ones(v.shape[:2], dtype=torch.float64) if mask is None else mask.double()
    y, scale = OE.normalize(v, m)
    scale = scale[:, 0, 0]
    C = v.shape[2]
    mono_abs = ((v * m[..., None]).sum(2).abs() / C) if C == 2 else torch.zeros(v.shape[:2], dtype=torch.float64)
    esc = U * torch.sqrt((mono_abs ** 2).mean(1)) + 2 * U * scale + U64 * scale * v.shape[1]
    ey = U * y.abs() + (v * m[..., None]).abs() * (esc / scale ** 2)[:, None, None]
    return y, scale, ey, esc


NORM_CASES = [(C, L, mk) for C in (1, 2) for L in (7, 3000) for mk in ("none", "partial", "zeros")]


@gpu
@pytest.mark.parametrize("C,L,mk", NORM_CASES, ids=[f"C{c}-L{l}-{m}" for c, l, m in NORM_CASES])
def test_encodec_normalize(C, L, mk):
    from mlx_audio_b200 import ops
    g = _gen(C * 10000 + L)
    R = 3
    x = torch.randn(R, L, C, generator=g) * torch.tensor([1.0, 1e-3, 30.0])[:, None, None]
    x[1, : L // 2] = 0.0
    mask = None if mk == "none" else (torch.rand(R, L, generator=g) > 0.3) if mk == "partial" else torch.zeros(R, L, dtype=torch.bool)
    md = None if mask is None else mask.to(DEV)
    y, sc = ops.encodec_normalize(_wide(x), md)
    ry, rs, ey, es = normalize_ref(x, mask)
    if mk == "zeros":
        assert torch.equal(sc.cpu(), torch.full((R,), 1e-8)) and not bool(y.any())
        return
    _check(f"normalize scale C{C} L{L} {mk}", sc, rs, es)
    _check(f"normalize y C{C} L{L} {mk}", y, ry, ey)
    if mk == "partial":
        _neg(f"normalize C{C} L{L}", sc, normalize_ref(x, None)[1], es)
    z = torch.zeros(1, L, C)
    y0, s0 = ops.encodec_normalize(z.to(DEV), None)                     # an all-zero chunk
    assert torch.equal(s0.cpu(), torch.full((1,), 1e-8)) and not bool(y0.any())


def ola_ref(frames, B, scale, stride, t_out):
    """float64 encodec_ola through the oracle (frames cut at t_out) and its bound."""
    NB, L, C = frames.shape
    N = NB // B
    f = frames.double().reshape(N, B, L, C)
    if scale is not None:
        f = f * scale.double().reshape(N, B)[..., None, None]
    fl = [f[k][:, :t_out - k * stride] for k in range(N)]              # every frame cut at t_out, the last one included
    out = OE.linear_overlap_add(fl, stride)
    w = torch.tensor([0.5 - abs((j + 1) / (L + 1) - 0.5) for j in range(L)], dtype=torch.float64)
    sw, aw, av = (torch.zeros(t_out, dtype=torch.float64), torch.zeros(B, t_out, C, dtype=torch.float64),
                  torch.zeros(B, t_out, C, dtype=torch.float64))
    kc = torch.zeros(t_out, dtype=torch.float64)
    for k in range(N):
        n = min(L, t_out - k * stride)
        sw[k * stride:k * stride + n] += w[:n]
        kc[k * stride:k * stride + n] += 1
        aw[:, k * stride:k * stride + n] += w[:n, None] * f[k][:, :n].abs()
        av[:, k * stride:k * stride + n] += f[k][:, :n].abs()
    eacc = (kc + 1)[None, :, None] * U * aw + 2 * U * av
    ews = kc * U * sw + 2 * U * kc
    return out, (eacc + out.abs() * ews[None, :, None]) / sw[None, :, None] + U * out.abs()


OLA_CASES = [(1, 16, 16, 1, 16), (1, 16, 16, 2, 7), (3, 16, 16, 2, 48), (4, 24, 10, 2, 54), (4, 24, 10, 2, 35), (5, 100, 37, 1, 200)]


@gpu
@pytest.mark.parametrize("N,L,stride,C,t_out", OLA_CASES, ids=[f"N{n}-L{l}-s{s}-C{c}-t{t}" for n, l, s, c, t in OLA_CASES])
def test_encodec_ola(N, L, stride, C, t_out):
    from mlx_audio_b200 import ops
    g = _gen(N * 1000 + L + t_out)
    B = 2
    frames = torch.randn(N * B, L, C, generator=g)
    for scale in (None, 0.5 + torch.rand(N * B, generator=g)):
        y = ops.encodec_ola(frames.to(DEV), B, None if scale is None else scale.to(DEV), stride, t_out)
        ref, bd = ola_ref(frames, B, scale, stride, t_out)
        _check(f"ola N{N} L{L} s{stride} t{t_out}", y, ref, bd)
        if N > 1:
            rev = frames.reshape(N, B, L, C).flip(0).reshape(N * B, L, C)
            rs = None if scale is None else scale.reshape(N, B).flip(0).reshape(-1)
            _neg(f"ola N{N}", y, ola_ref(rev, B, rs, stride, t_out)[0], bd)


def lstm_ref(xp, wh, swap=False):
    """float64 LSTM over the input projection xp [R, T, 4H] (gates i, f, g, o), h0 = c0 = 0."""
    xp, wh = xp.double(), wh.double()
    R, T, G = xp.shape
    H = G // 4
    h = torch.zeros(R, H, dtype=torch.float64)
    c = torch.zeros_like(h)
    out = []
    for t in range(T):
        a = xp[:, t] + h @ wh.T
        i, f = torch.sigmoid(a[:, :H]), torch.sigmoid(a[:, H:2 * H])
        if swap:
            i, f = f, i
        c = f * c + i * torch.tanh(a[:, 2 * H:3 * H])
        h = torch.sigmoid(a[:, 3 * H:]) * torch.tanh(c)
        out.append(h)
    return torch.stack(out, 1)


LSTM_TOL = 2e-5
LSTM_CASES = [(H, R, T, skip) for H in (128, 256, 512) for R, T, skip in ((1, 40, False), (5, 40, True), (5, 1, False), (2, 1, True))]


@gpu
@pytest.mark.parametrize("H,R,T,skip", LSTM_CASES, ids=[f"H{h}-R{r}-T{t}-{'skip' if s else 'noskip'}" for h, r, t, s in LSTM_CASES])
def test_encodec_lstm(H, R, T, skip):
    from mlx_audio_b200 import ops
    g = _gen(H * 100 + R * 10 + T)
    xp = torch.randn(R, T, 4 * H, generator=g)
    wh = 0.5 / math.sqrt(H) * torch.randn(4 * H, H, generator=g)
    sk = torch.randn(R, T, H, generator=g) if skip else None
    err = torch.zeros(1, device=DEV, dtype=torch.int32)
    whd = wh.to(DEV)
    y = ops.encodec_lstm(xp.to(DEV), whd, err, skip=None if sk is None else sk.to(DEV))
    ref = lstm_ref(xp, wh) + (0.0 if sk is None else sk.double())
    bound = LSTM_TOL * float(ref.abs().max())
    _check(f"lstm H{H} R{R} T{T}", y, ref, torch.full_like(ref, bound))
    _neg(f"lstm H{H} R{R} T{T}", y, lstm_ref(xp, wh, swap=True) + (0.0 if sk is None else sk.double()), torch.full_like(ref, bound))
    for r in range(R):
        one = ops.encodec_lstm(xp[r:r + 1].to(DEV), whd, err, skip=None if sk is None else sk[r:r + 1].to(DEV))
        assert torch.equal(one, y[r:r + 1]), r
    torch.cuda.synchronize()
    assert int(err.item()) == 0


# ================================================================================================================== aa_snakebeta
def aa_ref(x, a, ib, fu, fd):
    """float64 Activation1d(SnakeBeta) with ratio 2, 12 taps, edge clamps, and the bound of the module docstring; also the
    largest |a u| seen.  x [B, L, C] float32."""
    x, a, ib, fu, fd = (t.double() for t in (x, a, ib, fu, fd))
    B, L, C = x.shape
    n = torch.arange(2 * L)
    s, odd = n // 2, n % 2
    u = torch.zeros(B, 2 * L, C, dtype=torch.float64)
    au = torch.zeros_like(u)
    for q in range(6):
        idx = (s + 2 + odd - q).clamp(0, L - 1)
        f = 2 * fu[2 * q + 1 - odd]
        u += f[None, :, None] * x[:, idx]
        au += (f[None, :, None] * x[:, idx]).abs()
    eu = 6 * U * au
    arg = a * u
    sn = torch.sin(arg)
    v = u + ib * sn ** 2
    earg = a.abs() * eu + U * arg.abs()
    esin = earg + 2.0 ** -21
    ev = eu + ib.abs() * ((2 * sn.abs() + esin) * esin + U * sn ** 2) + U * v.abs()
    out = torch.zeros(B, L, C, dtype=torch.float64)
    eo = torch.zeros_like(out)
    ao = torch.zeros_like(out)
    t = torch.arange(L)
    for k in range(12):
        idx = (2 * t + k - 5).clamp(0, 2 * L - 1)
        out += fd[k] * v[:, idx]
        ao += (fd[k] * v[:, idx]).abs()
        eo += fd[k].abs() * ev[:, idx]
    return out, eo + 12 * U * ao, float(arg.abs().max())


def _aa_params(C, g, big=True):
    a = 0.5 + torch.rand(C, generator=g)
    if big:
        a[1::3] = 1e4 * (1 + torch.rand(len(a[1::3]), generator=g))
    ib = 1.0 / (torch.exp(0.3 * torch.randn(C, generator=g)) + 1e-9)
    fu, fd = torch.randn(12, generator=g) / 3, torch.randn(12, generator=g) / 3
    return a.float(), ib.float(), fu, fd


AA_LS = (1, 2, 3, 4, 5, 6, 7, 63, 64, 65, 130)


@gpu
@pytest.mark.parametrize("C", [1, 47, 48, 49, 50, 100])
def test_aa_snakebeta(C):
    from mlx_audio_b200 import ops
    g = _gen(C)
    a, ib, fu, fd = _aa_params(C, g)
    args = [t.to(DEV).contiguous() for t in (a, ib, fu, fd)]
    big = 0.0
    for L in AA_LS:
        x = 2.0 * torch.randn(3, L, C, generator=g)
        xd = _wide(x)
        y = ops.aa_snakebeta(xd, *args)
        for b in range(3):
            assert torch.equal(ops.aa_snakebeta(xd[b:b + 1], *args)[0], y[b]), (L, b)
        ref, bd, amax = aa_ref(x, a, ib, fu, fd)
        big = max(big, amax)
        _check(f"aa_snakebeta C{C} L{L}", y, ref, bd)
        _neg(f"aa_snakebeta C{C} L{L}", y, aa_ref(x, a, ib, fu.flip(0), fd)[0], bd)
    if C > 1:
        assert big > 8192                                              # the sinf branch of b2a_sin ran


class _TC:
    """Stand-in for a tensor-core conv's packing: only the channel count and the planes' width matter to aa_snakebeta."""
    def __init__(self, C, cpad=None):
        self.cin, self.cin_pad, self.w_tc, self.f16 = C, cpad or -(-C // 64) * 64, torch.empty(0), False


@gpu
@pytest.mark.parametrize("C", [1, 47, 49, 100])
@pytest.mark.parametrize("mode", ["x2", "x1"])
def test_aa_snakebeta_planes(C, mode, monkeypatch):
    from mlx_audio_b200 import ops
    monkeypatch.setattr(ops, "TC_MODE", [mode])
    g = _gen(C + 7)
    a, ib, fu, fd = _aa_params(C, g)
    args = [t.to(DEV).contiguous() for t in (a, ib, fu, fd)]
    x = _wide(torch.randn(2, 65, C, generator=g))
    y = ops.aa_snakebeta(x, *args)
    pl = ops.aa_snakebeta(x, *args, planes_for=_TC(C))
    cp = -(-C // 64) * 64
    assert pl.hi.shape == (2, 65, cp) and cp > C
    hi = y.to(torch.bfloat16)
    assert torch.equal(pl.hi[..., :C], hi) and not bool(pl.hi[..., C:].any())
    if mode == "x2":
        assert torch.equal(pl.lo[..., :C], (y - hi.float()).to(torch.bfloat16)) and not bool(pl.lo[..., C:].any())
    else:
        assert pl.lo is None


# ================================================================================================================== vocos_dwnorm
def dwnorm_ref(x, dw_w, dw_b, w, b, ada, NV, eps=1e-6, flip=False):
    """float64 depthwise conv + LayerNorm and the bound of the module docstring.  x [B, L, C] float32; dw_w [K, C]."""
    v = x.double()
    B, L, C = v.shape
    ec = torch.zeros_like(v)
    if dw_w is not None:
        K = dw_w.shape[0]
        wk = dw_w.double().flip(0) if flip else dw_w.double()
        xp = torch.nn.functional.pad(v, (0, 0, K // 2, K // 2))
        conv = sum(wk[k][None, None] * xp[:, k:k + L] for k in range(K))
        ac = sum((wk[k][None, None] * xp[:, k:k + L]).abs() for k in range(K))
        if dw_b is not None:
            conv, ac = conv + dw_b.double(), ac + dw_b.double().abs()
        v, ec = conv, (K + 1) * U * ac
    mean = v.mean(-1, keepdim=True)
    d = v - mean
    var = (d ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    o = d * rstd
    emean = ec.mean(-1, keepdim=True) + (NV + 8) * U * v.abs().mean(-1, keepdim=True)
    ed = ec + emean + U * d.abs()
    evar = 2 * torch.sqrt((ed ** 2).sum(-1, keepdim=True) / (d ** 2).sum(-1, keepdim=True).clamp_min(1e-300)) + (4 * NV + 7) * U
    er = 0.5 * evar * var / (var + eps) + 3 * U
    eo = ed * rstd + o.abs() * er + U * o.abs()
    if ada is not None:
        s, sh = ada[:, None, :C].double(), ada[:, None, C:].double()
        y = o * s + sh
        ey = s.abs() * eo + U * y.abs()
    else:
        y, ey = o, eo
        if w is not None:
            y = y * w.double()
            ey = ey * w.double().abs() + U * y.abs()
        if b is not None:
            y = y + b.double()
            ey = ey + U * y.abs()
    return y, 2 * ey


DN_MODES = ("affine", "w", "b", "ada")
DN_CASES = ([(C, K, m, True) for C in (4, 64, 132, 512, 516) for K in (0, 1, 3, 15) for m in DN_MODES]
            + [(C, K, "affine", False) for C in (4, 64, 132, 512, 516) for K in (1, 3, 15)]
            + [(1024, K, m, bias) for K in (1, 15) for m, bias in (("affine", True), ("ada", False))])
DN_IDS = [f"C{c}-K{k}-{m}-{'bias' if bi else 'nobias'}" for c, k, m, bi in DN_CASES]


@gpu
@pytest.mark.parametrize("C,K,mode,bias", DN_CASES, ids=DN_IDS)
def test_vocos_dwnorm(C, K, mode, bias):
    from mlx_audio_b200 import ops
    g = _gen(C * 100 + K * 10 + DN_MODES.index(mode))
    NV = 4 if C <= 512 else 8
    B = 2
    wk = torch.randn(K, C, generator=g) / math.sqrt(max(K, 1))
    bk = 0.1 * torch.randn(C, generator=g) if bias else None
    dw = ops.pack_conv(wk.t()[:, :, None].contiguous(), bk, C, DEV) if K else None
    w = (1 + 0.1 * torch.randn(C, generator=g)) if mode in ("affine", "w") else None
    b = 0.1 * torch.randn(C, generator=g) if mode in ("affine", "b") else None
    ada = torch.cat([1 + 0.3 * torch.randn(B, C, generator=g), 0.2 * torch.randn(B, C, generator=g)], 1) if mode == "ada" else None
    dv = lambda t: None if t is None else t.to(DEV).contiguous()       # noqa: E731
    for L in (1, 15, 16, 17):
        x = torch.randn(B, L, C, generator=g) + 0.5
        buf = torch.full((B, L, C + 12), float("nan"))
        buf[:, :, 4:4 + C] = x
        xd = buf.to(DEV)[:, :, 4:4 + C]
        planes = C % 64 == 0
        res = ops.vocos_dwnorm(xd, dw, dv(w), dv(b), ada=dv(ada), fp32=True, planes=planes)
        y, pl = res if planes else (res, None)
        ref, bd = dwnorm_ref(x, wk if K else None, bk, w, b, ada, NV)
        _check(f"dwnorm C{C} K{K} {mode} L{L}", y, ref, bd)
        if planes:
            hi = y.to(torch.bfloat16)
            assert torch.equal(pl.hi, hi)
            if pl.lo is not None:
                assert torch.equal(pl.lo, (y - hi.float()).to(torch.bfloat16))
        one = ops.vocos_dwnorm(xd[1:], dw, dv(w), dv(b), ada=None if ada is None else dv(ada[1:]))
        assert torch.equal(one[0], y[1])
        if K == 15 and L == 17:
            _neg(f"dwnorm C{C} K{K}", y, dwnorm_ref(x, wk, bk, w, b, ada, NV, flip=True)[0], bd)


# ================================================================================================================== vocos_istft_head
def head_ref(h, n_fft, hop, win, conj=False):
    """float64 ISTFTHead after the linear: h [B, T, ld] float32, win [n_fft] float32 -> (out [B, (T - 1) hop], bound)."""
    B, T, _ = h.shape
    nb = n_fft // 2 + 1
    mag = torch.exp(h[..., :nb].double()).clamp(max=100.0)
    ph = h[..., nb:2 * nb].double()
    X = mag * torch.exp((-1j if conj else 1j) * ph)                     # [B, T, nb]
    fr = torch.fft.irfft(X, n=n_fft, dim=-1)                            # [B, T, n_fft]
    wgt = torch.full((nb,), 2.0, dtype=torch.float64)
    wgt[0] = wgt[-1] = 1.0
    S = (mag * wgt).sum(-1) / n_fft                                     # [B, T]
    ef = (4 * math.sqrt(n_fft) + 16) * U * S
    w = win.double()
    total = (T - 1) * hop + n_fft
    num = torch.zeros(B, total, dtype=torch.float64)
    anum, enum_ = torch.zeros_like(num), torch.zeros_like(num)
    den, kc = torch.zeros(total, dtype=torch.float64), torch.zeros(total, dtype=torch.float64)
    for f in range(T):
        sl = slice(f * hop, f * hop + n_fft)
        num[:, sl] += fr[:, f] * w
        anum[:, sl] += (fr[:, f] * w).abs()
        enum_[:, sl] += w * ef[:, f:f + 1]
        den[sl] += w
        kc[sl] += 1
    cut = slice(n_fft // 2, n_fft // 2 + (T - 1) * hop)
    num, anum, enum_, den, kc = num[:, cut], anum[:, cut], enum_[:, cut], den[cut], kc[cut]
    big = den > 1e-10
    out = torch.where(big, num / torch.where(big, den, 1.0), num)
    en = enum_ + kc * U * anum
    e = torch.where(big, (en + out.abs() * kc * U * den) / torch.where(big, den, 1.0) + U * out.abs(), en)
    return out, e


HEAD_CASES = [(n, hp, T) for n, hp in ((16, 4), (1024, 128), (2048, 256), (2048, 2048), (1024, 300)) for T in (1, 2, 3, 937)]


@gpu
@pytest.mark.parametrize("n_fft,hop,T", HEAD_CASES, ids=[f"n{n}-hop{h}-T{t}" for n, h, t in HEAD_CASES])
def test_vocos_istft_head(n_fft, hop, T):
    from mlx_audio_b200 import ops
    from mlx_audio_b200.codec.models.vocos import hanning
    g = _gen(n_fft * 10 + hop + T)
    B, nb = 3, n_fft // 2 + 1
    ld = n_fft + 2 + 10
    h = torch.full((B, T, ld), 1e3)
    h[..., :nb] = torch.randn(B, T, nb, generator=g) - 0.5
    h[..., :nb][torch.rand(B, T, nb, generator=g) < 0.1] = 5.5        # e^5.5 = 245: clipped at 100
    h[..., nb:2 * nb] = 3.0 * torch.randn(B, T, nb, generator=g)
    buf = torch.full((2 * B, T, ld), float("nan"))
    buf[::2] = h
    hd = buf.to(DEV)[::2]
    assert hd.stride(1) == ld and hd.stride(0) == 2 * T * ld
    win = torch.from_numpy(hanning(n_fft)).float()
    wd = win.to(DEV)
    y = ops.vocos_istft_head(hd, n_fft, hop, wd)
    assert y.shape == (B, (T - 1) * hop)
    if T == 1:
        return
    for b in range(B):
        assert torch.equal(ops.vocos_istft_head(hd[b:b + 1], n_fft, hop, wd)[0], y[b])
    ref, bd = head_ref(h, n_fft, hop, win)
    _check(f"istft_head n{n_fft} hop{hop} T{T}", y, ref, bd)
    _neg(f"istft_head n{n_fft} hop{hop} T{T}", y, head_ref(h, n_fft, hop, win, conj=True)[0], bd)


# ================================================================================================================== CPU: reference pins
def _wn_params(P, pre, w_mlx, bias=None):
    """Weight-norm parameters whose g v / |v| is w_mlx [out, K, in] (float64)."""
    P[pre + ".weight_v"] = w_mlx
    P[pre + ".weight_g"] = torch.sqrt((w_mlx ** 2).sum(dim=(1, 2), keepdim=True))
    if bias is not None:
        P[pre + ".bias"] = bias


def test_codec_reference_pins():
    """rvq_decode_ref / rvq_encode_ref (mode 0) against the Mimi quantiser with identity projections, snac_ref against SNAC's
    from_codes."""
    g = _gen(1)
    B, T, nq, bins, D = 2, 9, 4, 32, 12
    cb = torch.randn(nq, bins, D, generator=g)
    codes = torch.randint(0, bins, (B, nq, T), generator=g)
    P = {}
    eye = torch.eye(D, dtype=torch.float64)[:, None, :]
    for name, qs in (("rvq_first", [0]), ("rvq_rest", list(range(1, nq)))):
        P[f"quantizer.{name}.output_proj.weight"] = eye
        P[f"quantizer.{name}.input_proj.weight"] = eye
        for li, qi in enumerate(qs):
            P[f"quantizer.{name}.vq.layers.{li}.codebook.embedding_sum"] = cb[qi].double()
            P[f"quantizer.{name}.vq.layers.{li}.codebook.cluster_usage"] = torch.ones(bins, dtype=torch.float64)
    want = OC.mimi_quantizer_decode(P, codes, {}).transpose(1, 2)
    assert torch.allclose(rvq_decode_ref(codes, cb)[1], want, rtol=1e-12, atol=1e-12)
    x = torch.randn(B, T, D, generator=g).float()
    enc = OC.mimi_quantizer_encode(P, x.double().transpose(1, 2), {"nq": nq})
    # the split quantiser: level 0 alone, then levels 1.. on a fresh residual
    parts = [rvq_encode_ref(x.reshape(B * T, D), t, torch.arange(bins), bins, 0) for t in (cb[:1], cb[1:])]
    ours, margin = torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1)
    ok = margin > 1e-9
    assert torch.equal(ours[ok], enc.permute(0, 2, 1).reshape(B * T, nq)[ok]) and ok.float().mean() > 0.9

    strides, Tt, sc, embs, ws, biases = _snac_case(3, 8, 20, g)
    Ps = {}
    for i in range(3):
        Ps[f"quantizer.quantizers.{i}.codebook.weight"] = embs[i].double()
        _wn_params(Ps, f"quantizer.quantizers.{i}.out_proj", ws[i].double().t()[:, None, :],
                   None if biases[i] is None else biases[i].double())
    want = OC.snac_from_codes(Ps, sc, {"vq_strides": list(strides)}).transpose(1, 2)
    assert torch.allclose(snac_ref(sc, strides, embs, ws, biases, Tt)[0], want, rtol=1e-12, atol=1e-12)


def test_dac_reference_pins():
    """dac_encode_ref against quantize / from_latents, dac_from_codes_ref against from_codes."""
    g = _gen(2)
    D, bins, B, T = 24, 64, 2, 7
    cds = [8, 1, 16]
    levels = _dac_levels(D, cds, bins, g)
    P = {}
    cn64 = []
    for i, lv in enumerate(levels):
        pre = f"quantizer.quantizers.{i}"
        _wn_params(P, pre + ".in_proj", lv["w_in"].double().t()[:, None, :], lv["b_in"].double())
        _wn_params(P, pre + ".out_proj", lv["w_out"].double().t()[:, None, :], lv["b_out"].double())
        P[pre + ".codebook.weight"] = lv["cb"].double()
        cn64.append(lv["cb"].double() / lv["cb"].double().norm(dim=1, keepdim=True))
    cfg = {"n_codebooks": len(cds), "codebook_dim": cds}
    z = torch.randn(B, T, D, generator=g)
    zq, codes, lat, closs, _ = ODAC.quantize(P, z.double().transpose(1, 2), cfg)
    R = B * T
    follow = codes.permute(0, 2, 1).reshape(R, -1)
    ref = dac_encode_ref(z.reshape(R, D), levels, follow, cn64=cn64)
    assert torch.equal(ref["codes"][ref["margin"] > 1e-9], follow[ref["margin"] > 1e-9])
    assert torch.allclose(ref["zq"], zq.transpose(1, 2).reshape(R, D), rtol=1e-10, atol=1e-10)
    assert torch.allclose(ref["lat"], lat.permute(0, 2, 1).reshape(R, -1), rtol=1e-10, atol=1e-10)
    assert abs(float(ref["loss"]) - float(closs)) <= 1e-10 * float(closs)
    zq2, _, codes2 = ODAC.from_latents(P, lat, cfg)
    ref2 = dac_encode_ref(None, levels, codes2.permute(0, 2, 1).reshape(R, -1), latents=lat.permute(0, 2, 1).reshape(R, -1), cn64=cn64)
    assert torch.allclose(ref2["zq"], zq2.transpose(1, 2).reshape(R, D), rtol=1e-10, atol=1e-10)
    zq3, zp3, _ = ODAC.from_codes(P, codes, cfg)
    ours, _, zp = dac_from_codes_ref(codes, levels)
    assert torch.allclose(ours, zq3.transpose(1, 2), rtol=1e-10, atol=1e-10) and torch.equal(zp.double(), zp3)


def test_encodec_reference_pins():
    """gn_ref against group_norm, normalize_ref (built on normalize), ola_ref (built on linear_overlap_add) against a direct
    weighted average, lstm_ref against lstm_layer, pad_ref against pad1d + elu."""
    g = _gen(3)
    x = torch.randn(2, 30, 6, generator=g)
    gamma, beta = torch.randn(6, generator=g), torch.randn(6, generator=g)
    sc, sh, _, _ = gn_ref(x, gamma, beta)
    P = {"c.norm.weight": gamma.double(), "c.norm.bias": beta.double()}
    assert torch.allclose(x.double() * sc[:, None] + sh[:, None], OE.group_norm(P, "c", x.double()), rtol=1e-12, atol=1e-12)
    y, s, _, _ = normalize_ref(x[..., :2], None)
    mono = x[..., :2].double().mean(2)
    assert torch.allclose(s, torch.sqrt((mono ** 2).mean(1)) + 1e-8, rtol=1e-14)
    frames = torch.randn(3 * 2, 8, 1, generator=g)
    out, _ = ola_ref(frames, 2, None, 5, 18)
    w = torch.tensor([0.5 - abs((j + 1) / 9 - 0.5) for j in range(8)], dtype=torch.float64)
    f = frames.double().reshape(3, 2, 8)
    t = 12                                                              # frames 1 (j = 7) and 2 (j = 2)
    assert abs(float(out[0, t, 0]) - float((w[7] * f[1, 0, 7] + w[2] * f[2, 0, 2]) / (w[7] + w[2]))) < 1e-12
    H = 8
    xin = torch.randn(2, 5, H, generator=g, dtype=torch.float64)
    Pl = {"l.Wx": torch.randn(4 * H, H, generator=g, dtype=torch.float64), "l.Wh": torch.randn(4 * H, H, generator=g, dtype=torch.float64),
          "l.bias": torch.randn(4 * H, generator=g, dtype=torch.float64)}
    assert torch.allclose(lstm_ref(xin @ Pl["l.Wx"].T + Pl["l.bias"], Pl["l.Wh"]), OE.lstm_layer(Pl, "l", xin), rtol=1e-12, atol=1e-12)
    scl, shf = torch.rand(2, 6, generator=g) + 0.5, torch.randn(2, 6, generator=g)
    v, _ = pad_ref(x, 3, 2, True, (scl, shf), True)
    want = OE.pad1d(OE.elu(x.double() * scl.double()[:, None] + shf.double()[:, None]), 3, 2, "reflect")
    assert torch.equal(v, want)


def test_bigvgan_reference_pins():
    g = _gen(4)
    x = torch.randn(2, 9, 5, generator=g)
    a, ib, fu, fd = _aa_params(5, g, big=False)
    beta = 1.0 / ib.double() - 1e-9
    P = {"p.act.alpha": a.double(), "p.act.beta": beta, "p.upsample.filter": fu.double(), "p.downsample.lowpass.filter": fd.double()}
    want = OB.activation1d(P, "p", x.double(), False)
    assert torch.allclose(aa_ref(x, a, ib, fu, fd)[0], want, rtol=1e-9, atol=1e-9)


def test_vocos_reference_pins():
    from mlx_audio_b200.codec.models.vocos import hanning
    g = _gen(5)
    x = torch.randn(2, 6, 8, generator=g)
    w, b = torch.randn(8, generator=g), torch.randn(8, generator=g)
    assert torch.allclose(dwnorm_ref(x, None, None, w, b, None, 4)[0], OV._layer_norm(x.double(), w.double(), b.double()), rtol=1e-12)
    n_fft, hop, T = 64, 16, 7
    h = torch.randn(2, T, n_fft + 2, generator=g)
    h[..., 3] = 5.5
    S, clipped = OV.spectrum(h, n_fft)
    assert clipped > 0
    want = OV.istft(S, n_fft, hop)
    ours, _ = head_ref(h, n_fft, hop, torch.from_numpy(hanning(n_fft)).float())
    # the oracle's window is float64; ours is the kernel's float32 window
    assert torch.allclose(ours, want, rtol=1e-6, atol=1e-6)
    ours64, _ = head_ref(h, n_fft, hop, torch.from_numpy(hanning(n_fft)))
    assert torch.allclose(ours64, want, rtol=1e-11, atol=1e-11)


# ================================================================================================================== GPU: host checks
@gpu
def test_argument_checks():
    from mlx_audio_b200 import _lib, ops
    from mlx_audio_b200.codec.models.vocos import hanning
    z = lambda *s: torch.zeros(*s, device=DEV)                          # noqa: E731

    def raises(exc, match, fn):
        n0 = ops.LAUNCHES[0]
        with pytest.raises(exc, match=match):
            fn()
        assert ops.LAUNCHES[0] == n0

    i64 = lambda *s: torch.zeros(*s, dtype=torch.int64, device=DEV)    # noqa: E731
    raises(ValueError, "dim and out_ld must be multiples of 4", lambda: ops.rvq_decode(i64(1, 1, 4), z(1, 8, 6)))
    raises(ValueError, "dim and out_ld must be multiples of 4", lambda: ops.rvq_decode(i64(1, 1, 4), z(1, 8, 4), out=z(1, 4, 6)[..., :4]))
    raises(ValueError, "bad pointers/shape", lambda: ops.rvq_decode(i64(0, 1, 4), z(1, 8, 4)))
    c2 = torch.zeros(2, 8, dtype=torch.float64, device=DEV)
    raises(ValueError, r"dim % 4 == 0; mode 1 = one level", lambda: ops.rvq_encode(z(3, 6), z(1, 8, 6), c2[:1]))
    raises(ValueError, r"dim % 4 == 0; mode 1 = one level", lambda: ops.rvq_encode(z(3, 4), z(2, 8, 4), c2, mode=1))
    raises(ValueError, "dim too large", lambda: ops.rvq_encode(z(3, 6392), z(1, 8, 6392), c2[:1]))
    ops.rvq_encode(z(3, 6388), z(1, 8, 6388), c2[:1])                   # the largest tile is legal

    one = [i64(1, 8)]
    raises(ValueError, r"bad shape \(levels<=4, codebook_dim<=16\)",
           lambda: ops.snac_from_codes(one * 5, [1] * 5, [z(4, 2)] * 5, [z(2, 4)] * 5, [None] * 5, 4))
    raises(ValueError, r"bad shape \(levels<=4, codebook_dim<=16\)", lambda: ops.snac_from_codes(one, [1], [z(4, 17)], [z(17, 4)], [None], 4))

    g = _gen(9)
    lv = [{k: v.to(DEV).contiguous() for k, v in d.items()} for d in _dac_levels(2564, [4], 8, g)]
    tab = ops.dac_levels(lv, DEV)
    raises(ValueError, "latent dimension too large for the frame tile", lambda: ops.dac_rvq_encode(z(1, 8, 2561), tab, 1, 8, 4, 2561))
    raises(ValueError, r"codebook_dim must be in \[1, 16\] at every level", lambda: ops.dac_rvq_encode(z(1, 8, 2560), tab, 1, 8, 17, 2560))
    raises(ValueError, r"codebook_dim must be in \[1, 16\] at every level", lambda: ops.dac_from_codes(i64(1, 2, 8), tab, 8, 1, 2560))
    many = ops.dac_levels([{"cb": z(8, 16), "w_out": z(16, 4), "b_out": z(4)}] * 97, DEV)
    raises(ValueError, "too many latent channels", lambda: ops.dac_from_codes(i64(1, 97, 8), many, 8, 97 * 16, 4))

    x = z(1, 16, 24)
    a, ib = torch.ones(24, device=DEV), torch.ones(24, device=DEV)
    raises(NotImplementedError, r"ratio 2 with 8 taps \(only ratio 2, 12 taps\)", lambda: ops.aa_snakebeta(x, a, ib, z(8), z(8)))
    raises(ValueError, "output row narrower than C", lambda: ops.aa_snakebeta(x, a, ib, z(12), z(12), planes_for=_TC(24, cpad=16)))
    raises(ValueError, r"exactly one of y \(fp32\) and hi \(bf16 planes\)", lambda: _lib.check(_lib.lib().b2a_aa_snakebeta(
        x.data_ptr(), 0, 24, 1, 16, 24, a.data_ptr(), ib.data_ptr(), z(12).data_ptr(), z(12).data_ptr(), 2, 12, None, 0, 0, None, None, 0,
        ops._stream())))

    raises(ValueError, r"C % 4 == 0, C <= 1024", lambda: ops.vocos_dwnorm(z(1, 4, 6), None, None, None))
    raises(ValueError, r"C % 4 == 0, C <= 1024", lambda: ops.vocos_dwnorm(z(1, 4, 1028), None, None, None))
    raises(ValueError, r"C % 4 == 0, C <= 1024", lambda: ops.vocos_dwnorm(z(1, 4, 70)[..., 2:66], None, None, None))
    raises(ValueError, r"bf16 planes need C % 64 == 0", lambda: ops.vocos_dwnorm(z(1, 4, 132), None, None, None, planes=True))
    raises(ValueError, "depthwise taps must be 0", lambda: _lib.check(_lib.lib().b2a_vocos_dwnorm(
        x.data_ptr(), 0, 24, 1, 16, 24, z(2, 24).data_ptr(), None, 2, None, None, None, 0, 1e-6, z(1, 16, 24).data_ptr(), 0, 24, None,
        None, ops._stream())))
    raises(ValueError, "no output", lambda: _lib.check(_lib.lib().b2a_vocos_dwnorm(
        x.data_ptr(), 0, 24, 1, 16, 24, None, None, 0, None, None, None, 0, 1e-6, None, 0, 24, None, None, ops._stream())))
    raises(ValueError, "AdaLN rows", lambda: _lib.check(_lib.lib().b2a_vocos_dwnorm(
        x.data_ptr(), 0, 24, 1, 16, 24, None, None, 0, None, None, z(1, 48).data_ptr(), 40, 1e-6, z(1, 16, 24).data_ptr(), 0, 24, None,
        None, ops._stream())))
    win = lambda n: torch.from_numpy(hanning(n)).float().to(DEV)        # noqa: E731
    unsup = r"even n_fft <= 2048 and hop > 0 only"
    raises(NotImplementedError, unsup, lambda: ops.vocos_istft_head(z(1, 3, 20), 17, 4, win(17)))
    raises(NotImplementedError, unsup, lambda: ops.vocos_istft_head(z(1, 3, 2052), 2050, 256, win(2050)))
    raises(NotImplementedError, unsup, lambda: ops.vocos_istft_head(z(1, 3, 20), 16, 0, win(16)))
    raises(ValueError, r"row stride >= n_fft \+ 2", lambda: _lib.check(_lib.lib().b2a_vocos_istft_head(
        z(1, 3, 20).data_ptr(), 60, 17, 1, 3, 16, 4, win(16).data_ptr(), z(1, 8).data_ptr(), 8, ops._stream())))
    raises(ValueError, r"output rows shorter than \(T - 1\) \* hop", lambda: _lib.check(_lib.lib().b2a_vocos_istft_head(
        z(1, 3, 20).data_ptr(), 60, 20, 1, 3, 16, 4, win(16).data_ptr(), z(1, 8).data_ptr(), 7, ops._stream())))

    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    raises(NotImplementedError, r"hidden size 64 not supported \(128, 256, 512\)", lambda: ops.encodec_lstm(z(1, 4, 256), z(256, 64), err))
    raises(ValueError, "reflect padding", lambda: ops.encodec_pad(z(1, 4, 3), 4, 0))
    raises(ValueError, "a residual add takes no padding", lambda: ops.encodec_pad(z(1, 4, 3), 1, 0, reflect=False, res=z(1, 5, 3)))
    raises(ValueError, "reflect padding", lambda: _lib.check(_lib.lib().b2a_encodec_pad(
        z(1, 4, 3).data_ptr(), 12, 3, 1, 4, 3, 0, 4, 1, None, None, 0, None, 0, 0, z(1, 8, 3).data_ptr(), 24, 3, ops._stream())))
    raises(ValueError, "bad pointers/shape", lambda: _lib.check(_lib.lib().b2a_encodec_pad(
        z(1, 4, 3).data_ptr(), 12, 3, 1, 4, 3, 0, 0, 1, z(3).data_ptr(), None, 0, None, 0, 0, z(1, 4, 3).data_ptr(), 12, 3, ops._stream())))
    raises(ValueError, "Tout beyond the frames, or a gap between frames", lambda: ops.encodec_ola(z(2, 8, 1), 1, None, 4, 13))
    raises(ValueError, "Tout beyond the frames, or a gap between frames", lambda: ops.encodec_ola(z(2, 8, 1), 1, None, 9, 10))
    raises(ValueError, "bad pointers/shape", lambda: ops.encodec_normalize(z(0, 8, 1), None))
    raises(ValueError, "bad pointers/shape", lambda: ops.encodec_gn_coeffs(z(1, 0, 4), None, None))
    torch.cuda.synchronize()
