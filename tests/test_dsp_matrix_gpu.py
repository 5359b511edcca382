"""Signal-processing kernels (csrc/dsp.cu; the direct-DFT log-mel of csrc/spk_logmel.cuh as csrc/speaker.cu and csrc/vocos.cu
instantiate it) against float64 on every dispatch branch.  Whisper reads its input through ``whisper_logmel``; Kokoro turns F0 into
its harmonic source with ``kokoro_source``, writes audio through ``kokoro_istft_head`` and draws its noise from ``randn_dev_``;
Qwen3-TTS voice cloning runs ``spk_logmel``, Vocos ``vocos_logmel``; ``mlx_audio.dsp`` runs ``stft`` / ``istft`` and
``utils.resample_audio`` runs ``resample_poly``.

Where each kernel and branch is run:
- stft_kernel / dft_frames<false>: ``test_stft_vs_float64[n*-pad*]`` for n_fft 2, 20, 64, 400, 1024, 2048, 4096 and pad_mode 0 (none),
  1 (reflect), 2 (constant), each at hop 1, n_fft / 4, a hop that does not divide n_fft and n_fft + 3, with 1, 8k and 8k +- 1 frames
  (a partial last CTA of 8 frames).  n_fft 2048 and 4096 need 80 / 160 KiB of dynamic shared memory: the 200 KiB opt-in.  The
  reflect ids include the minimum legal length n = n_fft / 2 + 1.  Every case runs B = 3 rows that are views of a wider buffer and
  checks each row bit for bit against a single-row call.
- whisper_logmel_kernel + whisper_logmel_finish: ``test_whisper_logmel_vs_float64``.  The all-zero shortcut is taken when a CTA's
  first frame starts at or after n (clause 1) and padding >= 400 (clause 2): ``[*-pad400-start-at-n]`` and ``[*-pad400-start-n+1]``
  take it, ``[*-pad400-start-n-1]`` fails clause 1 by one sample, ``[*-pad399-start-at-n]`` fails clause 2 by one sample, ``[*-pad0]``
  (reflection of real signal) and ``[*-pad250]`` (reflections land in the zero pad) never take it, ``[*-pad480000]`` takes it for
  every CTA past the signal.  ``test_whisper_shortcut_equals_transform`` checks that the shortcut and the transform write the same
  bits for the same zero frames.  n_mels 80 and 128 (large-v3).  Rows of rms 1, 1e-3 and silence check that the per-row maximum is
  per row, and a loud batch runs first to show that it does not carry over between calls.
- irfft_frames_kernel + ola_kernel: ``test_istft_vs_float64[n*-hop*]`` for n_fft 2, 16, 64, 400, 1024, 4096 (49 160 B: the opt-in) and
  hops n_fft / 4, n_fft / 2, n_fft, a non-divisor and n_fft + 3 (gaps where no frame reaches), each at T = 1, 2, 3, 937 with norm_sq
  True / False x clamp_mode 0 / 1 x trim 0 / n_fft / 2, out_len shorter than and equal to the full length, a periodic Hann window and a
  random one.  The clamp modes differ only where 0 < window sum <= 1e-10: sample 0 of the random window (w[0] = 3e-11) and sample 1
  of the periodic Hann at n_fft 1024 / 4096 with norm_sq (w[1]^2 = 8.8e-11 / 3.5e-13), both at trim 0.  Every case puts garbage in
  the imaginary parts of the DC and Nyquist bins; ``test_istft_ignores_dc_nyquist_imag`` requires bit-identical output with NaN
  there.  ``test_istft_reference_pins`` (CPU) pins the reference to ``OD.istft`` and ``OD.istft_cache``.
- ksrc_phase_kernel, ksrc_sample_kernel, ksrc_stft_kernel: ``test_kokoro_source_vs_float64``: nF 1, 2, 14 (n_down = nF + 1), 46 and
  600 (180 000 samples of float64 phase); ``noise`` given (``[*-noise]``) and ``None`` (``[*-silent]``: the ``noise ? .. : 0`` branch);
  B = 3 rows each bit-identical to a single-row call; f0 of exactly 10.0 and its float32 neighbours (the voiced threshold); f0 whose
  9th harmonic passes 12 kHz.  Exactly-real bins (DC, Nyquist, every bin of frame 0) with |X| > 1e-2 must have an angle of exactly 0
  or +pi: their imaginary part is float64 rounding noise of at most ~1e-16 sum_i |x_i w_i| <= 1e-15 (sin(pi) in the twiddle table
  is 1.2e-16), which the kernel's rule |im| <= 1e-12 |re| zeroes once |re| > 1e-3.
- kokoro_istft_head_kernel: ``test_kokoro_istft_head_vs_float64`` at T = 2, 3, 300, 4001 on a column slice of a wider [B, T, 64]
  buffer taken every other batch row, so x_ld = 64 and x_bs = 2 T 64, with log-magnitudes up to 8.
- randn_kernel + randn_advance_kernel: ``test_philox_known_answers`` (CPU) checks the reference generator against Random123's
  published philox4x32-10 vectors.  ``test_randn_vs_reference`` for n = 0 .. 5 (partial last group of 4), 1023 and 5 000 001 (more
  than one grid of 2112 x 256 threads x 4 values: the grid-stride loop), seeds with the high word set and counters that carry into
  the high word.  n = 0 on an empty tensor (null data pointer) draws nothing and raises nothing.  ``test_randn_stream_continuity`` covers split draws, ``randn_dev_`` (state read from device memory and advanced) and
  two replays of a captured CUDA graph.  ``test_randn_distribution`` checks 2^22 draws.
- resample_poly_kernel: ``test_resample_poly_vs_float64`` for 44100->24000, 48000->16000, 16000->24000, 24000->16000, 22050->24000 with
  n_in = 1 and 50 (the input-edge clamp acts at both ends of every output) and 48 000, on B = 2 strided rows.
  ``test_resample_reference_pins_scipy`` (CPU) pins the reference to ``scipy.signal.resample_poly(padtype="edge")``.
- spk_logmel_kernel<384, true> (``[spk-*]``) and <512, false> (``[vocos-*]``): ``test_mel_logmel_vs_float64`` at the minimum length
  (385 / 513, reflection reaches both ends of frame 0) and one above, frames = 1 (speaker only: Vocos drops the last of at least 3),
  8k + 1 frames (a partial CTA), B = 3 strided rows each bit-identical to a single-row call.  ``test_mel_reference_pins`` (CPU) pins
  the reference to ``OD.qwen3_mel_spectrogram`` and ``OV.log_mel_spectrogram``.
- Host checks: ``test_argument_checks`` (every B2A_CHECK_ARG of dsp.cu that ``ops`` can reach, the ``n_down`` check through the C entry
  point, and the length checks of ``spk_logmel`` / ``vocos_logmel``): each raises ValueError with its message and launches nothing.

Tolerances (u = 2^-24, the fp32 unit roundoff).  Each assertion divides the error by its bound and requires a ratio <= 1; the largest
ratio measured on an H100 80GB HBM3 (700 W) is given with each bound.  Every family has a negative control: the same assertion
against a perturbed reference must fail by more than NEG = 5 times its bound.
- Direct DFT (stft, and the spectra inside both log-mels): per frame max_k |X_k - ref_k| <= 4 sqrt(N) u sum_i |x_i w_i|.  Each term
  is an fp32 product x_i w_i times a table twiddle (sincospif, within an ulp), so the terms carry at most 2 u |x_i w_i| each: 2 u
  sum |x w| in all.  The fp32 fma chain of N terms rounds N partial sums, each at most sum |x w| in size and with errors of random
  sign: sqrt(N) u sum |x w| at one standard deviation.  c = 4 covers both with room (N = 2: 5.7 u sum |x w| >= the worst case of 4).
  Measured: 0.30 of the bound at N = 2, 0.11 at 20, 0.09 at 64 and 0.015 .. 0.04 from 400 up.  Negative controls: the window
  reversed; edge padding instead of reflect padding.
- Whisper log-mel: log10 of the mel energy, compared where the reference lies more than 0.05 above its row's max - 8 clamp.  The
  bound is derived per entry: |dP_k| <= 2 |X_k| E + E^2 with E the DFT bound above, plus 2 u P_k for the squares and 201 u mel for
  the fp32 sum of 201 positive terms, over mel ln 10, plus 4e-6 for log10f; divided by 4 by the final scaling.  Below the clamp by
  more than 0.05 every entry must be one value, the row's clamp, within the bound of the row's maximum.  A silent row is exactly
  (-10 + 4) / 4 = -1.5.  Measured: 0.054 of the bound.  Negative control: edge padding instead of reflect padding.
- iSTFT: per sample, from the per-frame scale S = sum_k wgt_k |X_k| / N (wgt 2, 1 at DC and Nyquist): each windowed frame value is
  within (4 sqrt(N / 2) + 2) u S |w_m| (the same fma-chain argument for the inverse DFT of N / 2 + 1 bins, then the / N and the window
  product); the overlap-add of K = ceil(N / hop) terms adds K u sum |ws|, and the window sum K u of itself.  Dividing by the window sum
  (clamped as each clamp_mode does) carries these over, plus 2 u |out|.  Measured: 0.29 of the bound at N = 2, 0.16 at 16, 0.10 at
  64 and 0.017 .. 0.054 from 400 up.  Negative controls: the other clamp_mode's rule, and the DC / Nyquist bins taken with their
  imaginary part (as |X| with the sign of the real part).
- Kokoro source: per sample, the merged source is within e = 13 u (|b| + sum_h |w_h s_h|) + 4 u |src| of float64 (the phase is float64
  in the kernel; the fp32 sine, noise mix and 9-term fma chain give the first term, tanhf's 2 ulp the second).  The float64 STFT
  moves that to each frame as sum_i hann_i e_i; magnitudes must lie within it plus 2 u |X|, and angles (modulo 2 pi, where |X| >
  1e-4) within 1.5 of it over |X| plus 4 pi u.  Measured: 0.16 of the bound.  Negative control: f0 = 10.0 counted as voiced.
- Kokoro head: per output sample, each frame's inverse DFT is within 32 u S (S = 0.05 sum_k wgt_k e^{x_k}: expf, sinf and sincosf
  within 2 ulp, rounded twiddles, the products and an 11-term fp32 sum), carried through the overlap-add and the division by the
  window sum, plus 2 u |out|.  Measured: 0.12 of the bound.  Negative control: the phase sign flipped.
- randn: |v - ref| <= 1e-5.  The uniforms are bit-exact (emulated in float32); r = sqrt(-2 logf(u)) <= 6.8 is within 2 ulp
  (logf 1 ulp, halved by the square root, sqrtf 1/2 ulp), sincospif within 1 ulp (2^-24 absolute), the product 1/2 ulp: at most
  6.8 x 4 u = 1.6e-6.  Measured: 6.1e-7.  Negative controls: the round multiplier M0 + 1; the key increment W0 + 1.  Split draws,
  ``randn_dev_`` and graph replays must be bit-identical to the single call they continue.  The distribution check requires the
  mean, the variance, the lag-1..4 correlations and the 4 sigma tail count within 5 standard deviations of N(0, 1), and the KS
  test's p-value above 5.7e-7 (5 sigma).
- resample_poly: |y - ref| <= u |ref| + 2^-40 sum_t |h_t x_i| + 2^-149.  The kernel accumulates in float64 and casts once (u |ref|);
  at most 385 float64 roundings in another order differ by far less than 2^-40 of the absolute sum; 2^-149 is the float32 denormal
  spacing.  Measured: 0.997 of the bound: the cast alone is within half an ulp, u |ref|, and the kernel reaches it, so the float64
  sums agree to far better than 2^-40.  Negative control: the filter phase t0 off by one.
- Speaker / Vocos log-mel: natural log of the mel energy where the reference mel >= 1e-3; |dmel| <= E sum_k f_mk + (2 + 513) u mel (E
  the DFT bound, 2 u for the magnitude, 513 u for the fp32 sum of positive terms), over mel, plus 2e-6 for logf.  Where the
  reference mel plus that bound stays below 1e-5 the output must be log(1e-5) within 1e-6.  Measured: 0.32 of the bound.  Negative
  control: edge padding instead of reflect padding at the minimum length.
"""
import math

import numpy as np
import pytest
import torch

from oracle import dsp as OD

gpu = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
C_DFT = 4.0
C_HEAD = 32.0
NEG = 5                      # every negative control exceeds NEG x its bound


def _rng(seed):
    return np.random.default_rng(seed)


def _report(name, ratio):
    print(f"{name}: max error / bound = {ratio:.3g}")


def _nondiv(N):
    """The smallest hop above N / 4 that does not divide N."""
    h = max(1, N // 4) + 1
    while N % h == 0:
        h += 1
    return h


def _rand_window(N, seed):
    """A positive, non-symmetric window: a reversed index changes every frame."""
    return (0.25 + _rng(seed).random(N)).astype(np.float32)


def _strided_rows(rows, extra=37, off=5):
    """float32 rows [B, n] as a view of a wider device buffer (stride(0) = n + extra > n)."""
    B, n = rows.shape
    buf = torch.full((B, n + extra), float("nan"))
    buf[:, off:off + n] = torch.as_tensor(rows)
    return buf.to(DEV)[:, off:off + n]


# ------------------------------------------------------------------------------------------------------------ float64 references
def pad_signal(x64, p, mode):
    """Centre padding of p samples: "reflect" (no repeated edge), "constant" (zeros), "edge" (a negative control only)."""
    if p == 0:
        return x64
    return np.pad(x64, (p, p), mode=mode) if mode != "constant" else np.pad(x64, (p, p))


def frame_spectra(x32, w32, N, hop, frames, p, mode):
    """Windowed frames of the padded float64 signal and their float64 rfft: (X [frames, N/2+1], sum_i |x_i w_i| [frames])."""
    xp = pad_signal(np.asarray(x32, dtype=np.float64), p, mode)
    need = (frames - 1) * hop + N
    if xp.shape[0] < need:
        xp = np.concatenate([xp, np.zeros(need - xp.shape[0])])
    idx = np.arange(frames)[:, None] * hop + np.arange(N)[None, :]
    fr = xp[idx] * np.asarray(w32, dtype=np.float64)[None, :]
    return np.fft.rfft(fr, axis=-1), np.abs(fr).sum(-1)


def dft_bound(N, absum):
    return C_DFT * math.sqrt(N) * U * absum


_PAD_NAMES = {0: None, 1: "reflect", 2: "constant"}


def stft_ref(x32, w32, N, hop, pad_mode, frames, reflect_as="reflect"):
    """``ops.stft`` in float64: [B, frames, N/2+1] complex and the per-frame bound [B, frames]."""
    mode = _PAD_NAMES[pad_mode]
    if mode == "reflect":
        mode = reflect_as
    p = N // 2 if pad_mode else 0
    out = [frame_spectra(r, w32, N, hop, frames, p, mode) for r in x32]
    return np.stack([o[0] for o in out]), np.stack([dft_bound(N, o[1]) for o in out])


def stft_ratio(re, im, ref, bound):
    err = np.abs(re.double().cpu().numpy() + 1j * im.double().cpu().numpy() - ref).max(-1)
    return float((err / (bound + 1e-30)).max())


WHISPER_N, WHISPER_HOP, WHISPER_NF = 400, 160, 201


def whisper_ref(x32, padding, filt32, frames, reflect_as="reflect"):
    """log10(max(mel, 1e-10)) [B, frames, n_mels] of the power spectrum of the zero-padded, reflect-centred signal, with the derived
    per-entry bound on it (see the module docstring)."""
    w = OD.hanning(WHISPER_N).astype(np.float32)
    f = np.asarray(filt32, dtype=np.float64)
    L, bL = [], []
    for r in x32:
        a = np.concatenate([np.asarray(r, dtype=np.float64), np.zeros(padding)])
        X, absum = frame_spectra(a, w, WHISPER_N, WHISPER_HOP, frames, WHISPER_N // 2, reflect_as)
        E = dft_bound(WHISPER_N, absum)[:, None]
        aX = np.abs(X)
        mel = (aX ** 2) @ f.T
        dmel = 2 * E * (aX @ f.T) + E ** 2 * f.sum(1)[None, :] + (WHISPER_NF + 2) * U * mel
        L.append(np.log10(np.maximum(mel, 1e-10)))
        bL.append(dmel / (np.maximum(mel, 1e-10) * math.log(10)) + 4e-6)
    return np.stack(L), np.stack(bL)


def whisper_ratio(y, L, bL, margin=0.05):
    """Largest error / bound of the Whisper log-mel y [B, frames, n_mels] against the unclamped float64 log10 L (see the docstring)."""
    y = y.cpu().numpy().astype(np.float64)
    worst = 0.0
    for b in range(L.shape[0]):
        Lmax = L[b].max()
        clamp = Lmax - 8.0
        loud, quiet = L[b] > clamp + margin, L[b] < clamp - margin
        assert float(bL[b][loud].max()) < margin / 2              # the margin separates the two regions in the kernel too
        err = np.abs(y[b] - (L[b] + 4.0) / 4.0)
        worst = max(worst, float((err[loud] / (bL[b][loud] / 4.0)).max()))
        if quiet.any():
            vals = np.unique(y[b][quiet])
            assert vals.size == 1, vals                            # one clamp value per row
            bmax = float(bL[b][L[b] > Lmax - 1.0].max())
            worst = max(worst, abs(float(vals[0]) - (clamp + 4.0) / 4.0) / (bmax / 4.0))
    return worst


def irfft_frames(re, im, N, w64, dc_nyq="ignore"):
    """Windowed inverse rFFTs [B, T, N] of re / im [B, N/2+1, T] and the per-frame scale S = sum_k wgt_k |X_k| / N [B, T].
    ``dc_nyq`` "abs" takes the DC and Nyquist bins as |X| with the sign of the real part (a negative control only)."""
    X = (np.asarray(re, dtype=np.float64) + 1j * np.asarray(im, dtype=np.float64)).transpose(0, 2, 1).copy()
    if dc_nyq == "abs":
        for k in (0, N // 2):
            X[..., k] = np.sign(X[..., k].real) * np.abs(X[..., k])
    else:
        X[..., 0] = X[..., 0].real
        X[..., N // 2] = X[..., N // 2].real
    wgt = np.full(N // 2 + 1, 2.0)
    wgt[0] = wgt[N // 2] = 1.0
    return np.fft.irfft(X, n=N, axis=-1) * w64, (np.abs(X) * wgt).sum(-1) / N


def ola(fr, hop):
    """Overlap-add of frames [B, T, N] at ``hop`` -> [B, (T - 1) hop + N]."""
    B, T, N = fr.shape
    out = np.zeros((B, (T - 1) * hop + N))
    for t in range(T):
        out[:, t * hop:t * hop + N] += fr[:, t]
    return out


def istft_ola(ws, S, N, hop, w64):
    """The overlap-adds istft_ref divides: the signal, its absolute sum, its error bound (see the docstring) and both window sums."""
    T = ws.shape[1]
    K = -(-N // hop)
    absA = ola(np.abs(ws), hop)
    Aerr = ola((C_DFT * math.sqrt(N / 2) + 2) * U * S[..., None] * np.abs(w64)[None, None, :], hop) + K * U * absA
    D = {sq: ola(np.broadcast_to((w64 * w64 if sq else w64)[None, None, :], (1, T, N)), hop)[0] for sq in (True, False)}
    return dict(A=ola(ws, hop), absA=absA, Aerr=Aerr, D=D, K=K)


def istft_ref(parts, norm_sq, clamp_mode, trim, out_len):
    """Overlap-add of the windowed frames divided by the window sum as ``clamp_mode`` says (0: divide only where the sum exceeds
    1e-10; 1: divide by max(sum, 1e-10)), samples [trim, trim + out_len); with the per-sample bound (see the docstring)."""
    sl = slice(trim, trim + out_len)
    A, absA, Aerr, D, K = parts["A"][:, sl], parts["absA"][:, sl], parts["Aerr"][:, sl], parts["D"][norm_sq][sl], parts["K"]
    if clamp_mode == 0:
        big = D > 1e-10
        Dd = np.where(big, D, 1.0)
        out = np.where(big, A / Dd, A)
        bound = np.where(big, (Aerr + absA * K * U) / Dd, Aerr)
    else:
        Dd = np.maximum(D, 1e-10)
        out = A / Dd
        bound = (Aerr + absA * np.where(D > 1e-10, K * U, 0.0)) / Dd
    return out, bound + 2 * U * np.abs(out)


def ratio(y, ref, bound):
    y = y.double().cpu().numpy() if isinstance(y, torch.Tensor) else np.asarray(y, dtype=np.float64)
    return float((np.abs(y - ref) / (bound + 1e-300)).max())


def source_ref(f0, noise, lw, lb, voiced_threshold=10.0):
    """float64 hn-NSF source (``OK.sinegen``, the 9 -> 1 linear layer, tanh) and its STFT magnitude / phase [B, T, 11], with the per-frame
    bound on the magnitudes [B, T] (see the docstring).  ``voiced_threshold`` below 10 is a negative control only."""
    from oracle import kokoro as OK
    f0s = torch.repeat_interleave(torch.as_tensor(f0).double()[:, :, None], 300, dim=1)
    sw, _, _ = OK.sinegen(f0s, noise=None if noise is None else torch.as_tensor(noise).double(), voiced_threshold=voiced_threshold)
    lw64, lb64 = np.asarray(lw, dtype=np.float64), float(lb)
    terms = sw.numpy() * lw64[None, None, :]
    src = np.tanh(terms.sum(-1) + lb64)
    e = 13 * U * (abs(lb64) + np.abs(terms).sum(-1)) + 4 * U * np.abs(src)
    mag, ph = OK.mlxstft_transform(src, 20, 5, 20)
    hann = OD.hanning(20, periodic=True)
    be = np.stack([frame_spectra(r, hann, 20, 5, mag.shape[2], 10, "reflect")[1] for r in e])   # sum_i hann_i e_i per frame
    return mag.transpose(0, 2, 1), ph.transpose(0, 2, 1), be


def head_ref(x, flip_phase=False):
    """``OK.mlxstft_inverse`` of exp(x[..., :11]) e^{j sin(x[..., 11:])} -> [B, (T - 1) 5], with the per-sample bound."""
    from oracle import kokoro as OK
    x = np.asarray(x, dtype=np.float64)
    mag = np.exp(x[..., :11])
    ph = np.sin(x[..., 11:]) * (-1.0 if flip_phase else 1.0)
    out = OK.mlxstft_inverse(mag.transpose(0, 2, 1), ph.transpose(0, 2, 1), 20, 5, 20)[:, 0]
    wgt = np.full(11, 2.0)
    wgt[0] = wgt[10] = 1.0
    S = 0.05 * (mag * wgt).sum(-1)                                      # [B, T]
    w = OD.hanning(20, periodic=True)
    err = ola(C_HEAD * U * S[..., None] * w[None, None, :], 5) + 4 * U * ola(S[..., None] * w[None, None, :], 5)
    D = ola(np.broadcast_to((w * w)[None, None, :], (1, x.shape[1], 20)), 5)[0]
    bound = (err / np.maximum(D, 1e-10))[:, 10:10 + out.shape[1]]
    return out, bound + 2 * U * np.abs(out)


# Philox4x32-10 with the kernel's layout (csrc/dsp.cu: randn_kernel)
PH_M0, PH_M1 = 0xD2511F53, 0xCD9E8D57
PH_W0, PH_W1 = 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32(c, key, rounds=10, m0=PH_M0, w0=PH_W0):
    """c: four uint64 arrays of 32-bit words, key: (k0, k1).  Each round: (c0, c1, c2, c3) <- (hi(M1 c2) ^ c1 ^ k0, lo(M1 c2),
    hi(M0 c0) ^ c3 ^ k1, lo(M0 c0)), then the key is bumped by (W0, W1)."""
    c0, c1, c2, c3 = (np.asarray(v, dtype=np.uint64) for v in c)
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    m0, m1 = np.uint64(m0), np.uint64(PH_M1)
    for _ in range(rounds):
        p0, p1 = m0 * c0, m1 * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK
        k0, k1 = (k0 + np.uint64(w0)) & _MASK, (k1 + np.uint64(PH_W1)) & _MASK
    return c0, c1, c2, c3


def randn_ref(n, seed, offset, **kw):
    """``ops.randn_(n, seed, offset)``: counter (c0, c1) = the 64-bit offset + i, (c2, c3) = (0x2545F491, 0x9E3779B9), key = the seed's
    (low, high) words; uniforms ((float)c + 0.5f) 2^-32 in float32; Box-Muller in float64 on them."""
    n4 = (n + 3) // 4
    ctr = (np.uint64(offset) + np.arange(n4, dtype=np.uint64))
    c = philox4x32((ctr & _MASK, ctr >> np.uint64(32), np.full(n4, 0x2545F491, np.uint64), np.full(n4, 0x9E3779B9, np.uint64)),
                   (seed & 0xFFFFFFFF, seed >> 32), **kw)
    u = [((v.astype(np.float32) + np.float32(0.5)) * np.float32(2.3283064365386963e-10)).astype(np.float64) for v in c]
    r0, r1 = np.sqrt(-2 * np.log(u[0])), np.sqrt(-2 * np.log(u[2]))
    v = np.stack([r0 * np.cos(2 * np.pi * u[1]), r0 * np.sin(2 * np.pi * u[1]), r1 * np.cos(2 * np.pi * u[3]), r1 * np.sin(2 * np.pi * u[3])], 1)
    return v.reshape(-1)[:n]


def resample_plan(orig, target, n_in):
    from mlx_audio_b200.resample import _poly_plan, _polyphase_filter
    up, down, fir = _polyphase_filter(orig, target)
    n_out, n_pre_pad, n_pre_remove = _poly_plan(n_in, up, down, len(fir))
    return up, down, fir * up, n_pre_pad, n_pre_remove, n_out


def resample_ref(x, h, up, down, n_pre_pad, n_pre_remove, n_out, t0_shift=0):
    """out[n] = sum over t = c(n) (mod up), 0 <= t < n_h of h[t] x[clamp((c(n) - t) / up)], c(n) = (n + n_pre_remove) down - n_pre_pad,
    in float64, with sum |h x| per output.  ``t0_shift`` != 0 moves the filter phase (a negative control only)."""
    x = np.asarray(x, dtype=np.float64)
    n_h = h.shape[0]
    taps = np.arange(-(-n_h // up))
    out, absum = np.empty(n_out), np.empty(n_out)
    for s in range(0, n_out, 2048):
        n = np.arange(s, min(n_out, s + 2048))
        c = (n + n_pre_remove) * down - n_pre_pad
        t = ((c + t0_shift) % up)[:, None] + taps[None, :] * up
        ok = t < n_h
        i = np.clip((c[:, None] - t) // up, 0, x.shape[0] - 1)
        v = np.where(ok, h[np.minimum(t, n_h - 1)] * x[i], 0.0)
        out[n], absum[n] = v.sum(1), np.abs(v).sum(1)
    return out, absum


MEL_N, MEL_HOP, MEL_NF = 1024, 256, 513
MEL_KINDS = {"spk": (384, True), "vocos": (512, False)}


def mel_frames(kind, n):
    return 1 + (n + 768 - MEL_N) // MEL_HOP if kind == "spk" else n // MEL_HOP


def mel_ref(kind, x32, w32, filt32, pad_as="reflect"):
    """log(max(mel, 1e-5)) [B, frames, n_mels] of the reflect-padded direct DFT (magnitude sqrt(|X|^2 + 1e-9) for the speaker
    variant, |X| for Vocos), the mel energy, and the derived bound on |dmel| (see the docstring)."""
    pad, eps = MEL_KINDS[kind]
    f = np.asarray(filt32, dtype=np.float64)
    logs, mels, dmels = [], [], []
    for r in x32:
        X, absum = frame_spectra(r, w32, MEL_N, MEL_HOP, mel_frames(kind, len(r)), pad, pad_as)
        mag = np.sqrt(np.abs(X) ** 2 + 1e-9) if eps else np.abs(X)
        mel = mag @ f.T
        mels.append(mel)
        dmels.append(dft_bound(MEL_N, absum)[:, None] * f.sum(1)[None, :] + (2 + MEL_NF) * U * mel)
        logs.append(np.log(np.maximum(mel, 1e-5)))
    return np.stack(logs), np.stack(mels), np.stack(dmels)


def mel_ratio(y, logs, mel, dmel):
    y = y.cpu().numpy().astype(np.float64)
    loud = mel >= 1e-3
    worst = float((np.abs(y - logs)[loud] / (dmel[loud] / mel[loud] + 2e-6)).max())
    clamped = mel + dmel < 1e-5
    if clamped.any():
        worst = max(worst, float(np.abs(y[clamped] - math.log(1e-5)).max()) / 1e-6)
    return worst


def _spk_filters():
    return OD.mel_filters(24000, 1024, 128, 0.0, 12000.0, norm="slaney", mel_scale="slaney")


def _vocos_filters():
    from oracle import vocos as OV
    return OV.mel_filters_htk(24000, 1024, 100).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------ CPU: the references
def test_philox_known_answers():
    """Random123's published philox4x32-10 known-answer vectors (kat_vectors): the reference generator is Philox4x32-10."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        got = philox4x32([[v] for v in ctr], key)
        assert tuple(int(v[0]) for v in got) == want
        assert tuple(int(v[0]) for v in philox4x32([[v] for v in ctr], key, m0=PH_M0 + 1)) != want


def test_stft_reference_pins():
    """stft_ref is the oracle's STFT (dsp.py) for a window array, in all three padding modes."""
    x = _rng(1).standard_normal((1, 301)).astype(np.float32)
    w = _rand_window(64, 2)
    for mode, kw in ((0, dict(center=False)), (1, dict(center=True, pad_mode="reflect")), (2, dict(center=True, pad_mode="constant"))):
        want = OD.stft(x[0], n_fft=64, hop_length=13, window=w.astype(np.float64), **kw)
        got, _ = stft_ref(x, w, 64, 13, mode, want.shape[0])
        assert np.abs(got[0] - want).max() < 1e-12 * np.abs(want).max()


def test_whisper_reference_pins():
    """whisper_ref, clamped and scaled per row, is the oracle's Whisper log-mel."""
    x = (0.3 * _rng(3).standard_normal((1, 4000))).astype(np.float32)
    filt = OD.mel_filters(16000, 400, 80, norm="slaney", mel_scale=None)
    for padding in (0, 480):
        want = OD.whisper_log_mel(x[0], 80, padding)
        L, _ = whisper_ref(x, padding, filt, (4000 + padding) // 160)
        got = (np.maximum(L[0], L[0].max() - 8) + 4) / 4
        assert np.abs(got - want).max() < 1e-6                            # the window rounded to float32 here


def test_istft_reference_pins():
    """istft_ref is ``OD.istft`` (clamp_mode 0, trim n_fft / 2, both norms) and ``OD.istft_cache`` (clamp_mode 1, norm_sq)."""
    N, hop, T = 64, 16, 9
    g = _rng(4)
    re, im = g.standard_normal((2, 33, T)), g.standard_normal((2, 33, T))
    w = OD.hanning(N, periodic=True)
    parts = istft_ola(*irfft_frames(re, im, N, w), N, hop, w)
    for norm_sq in (True, False):
        want = np.stack([OD.istft(re[b] + 1j * im[b], hop_length=hop, win_length=N, window=w, normalized=norm_sq) for b in range(2)])
        got, _ = istft_ref(parts, norm_sq, 0, N // 2, want.shape[1])
        assert np.abs(got - want).max() < 1e-12
    want = OD.istft_cache(re, im, N, hop, N, w, center=True)
    got, _ = istft_ref(parts, True, 1, N // 2, want.shape[1])
    assert np.abs(got - want).max() < 1e-12


def test_resample_reference_pins_scipy():
    """resample_ref (the kernel's documented formula) is ``scipy.signal.resample_poly(padtype="edge")`` on float64 input."""
    from scipy import signal
    for orig, target in ((44100, 24000), (48000, 16000), (16000, 24000), (24000, 16000), (22050, 24000)):
        for n_in in (50, 3001):
            x = _rng(n_in).standard_normal(n_in)
            up, down, h, pre, rem, n_out = resample_plan(orig, target, n_in)
            want = signal.resample_poly(x, up, down, window=h / up, padtype="edge")
            got, _ = resample_ref(x, h, up, down, pre, rem, n_out)
            assert got.shape == want.shape and np.abs(got - want).max() < 1e-12 * np.abs(want).max()


def test_mel_reference_pins():
    """mel_ref is the oracle's Qwen3-TTS speaker log-mel and Vocos's log-mel with their windows and filters."""
    from oracle import vocos as OV
    x = (0.2 * _rng(5).standard_normal((1, 3000))).astype(np.float32)
    w = OD.hanning(1024).astype(np.float32)
    logs, _, _ = mel_ref("spk", x, w, _spk_filters())
    want = OD.qwen3_mel_spectrogram(x.astype(np.float64))
    assert logs.shape == want.shape and np.abs(logs - want).max() < 1e-5      # window and filters rounded to float32 here
    logs, _, _ = mel_ref("vocos", x, w, _vocos_filters())
    want = OV.log_mel_spectrogram(x[0]).numpy()
    assert logs.shape == want.shape and np.abs(logs - want).max() < 1e-5


def test_source_and_head_reference_pins():
    """source_ref follows the test of ``ops.kokoro_source`` in tests/test_ops_gpu.py; head_ref is ``OK.mlxstft_inverse``.  The bounds
    are finite and positive."""
    f0 = np.array([[0.0, 120.0, 10.0, 300.0]], dtype=np.float32)
    mag, ph, be = source_ref(f0, None, np.full(9, 0.2), 0.05)
    assert mag.shape == (1, 4 * 60 + 1, 11) and be.shape == (1, 4 * 60 + 1) and (be > 0).all()
    x = 0.5 * _rng(6).standard_normal((1, 7, 22))
    out, bound = head_ref(x)
    assert out.shape == (1, 30) and (bound > 0).all()


# ------------------------------------------------------------------------------------------------------------ GPU: stft
STFT_NFFT = [2, 20, 64, 400, 1024, 2048, 4096]


def _stft_cases(N, pad_mode):
    """(hop, n) pairs: hop 1, N / 4, a non-divisor and N + 3 with 9, 16, 15 and 7 frames, plus reflect at the minimum length."""
    cases = []
    for hop, F in ((1, 9), (max(1, N // 4), 16), (_nondiv(N), 15), (N + 3, 7)):
        if pad_mode == 0:
            n = (F - 1) * hop + N
        else:
            n = (F - 1) * hop + hop // 2
            if pad_mode == 1 and n <= N // 2:
                if hop == 1 and N > 400:
                    continue                               # would be N / 2 + 2 frames of a large transform
                n = N // 2 + 1
        cases.append((hop, max(n, 1)))
    if pad_mode == 1:
        cases.append((max(1, N // 4), N // 2 + 1))
    return cases


def _stft_frames(n, N, hop, pad_mode):
    return 1 + ((n + (N if pad_mode else 0)) - N) // hop


@gpu
@pytest.mark.parametrize("pad_mode", [0, 1, 2], ids=["pad0", "pad1-reflect", "pad2-constant"])
@pytest.mark.parametrize("N", STFT_NFFT, ids=[f"n{n}" for n in STFT_NFFT])
def test_stft_vs_float64(N, pad_mode):
    from mlx_audio_b200 import ops
    w = _rand_window(N, N)
    wd = torch.as_tensor(w).to(DEV)
    worst, neg_rev, neg_edge = 0.0, np.inf, np.inf
    for j, (hop, n) in enumerate(_stft_cases(N, pad_mode)):
        frames = _stft_frames(n, N, hop, pad_mode)
        x = _rng(1000 * N + j).standard_normal((3, n)).astype(np.float32)
        xd = _strided_rows(x)
        re, im = ops.stft(xd, wd, N, hop, pad_mode, frames)
        ref, bound = stft_ref(x, w, N, hop, pad_mode, frames)
        worst = max(worst, stft_ratio(re, im, ref, bound))
        for b in range(3):                                             # batch rows are independent and bit-identical
            r1, i1 = ops.stft(xd[b:b + 1], wd, N, hop, pad_mode, frames)
            assert torch.equal(r1[0], re[b]) and torch.equal(i1[0], im[b])
        rr, _ = stft_ref(x, w[::-1].copy(), N, hop, pad_mode, frames)
        neg_rev = min(neg_rev, stft_ratio(re, im, rr, bound))
        if pad_mode == 1:
            re_, _ = stft_ref(x, w, N, hop, pad_mode, frames, reflect_as="edge")
            neg_edge = min(neg_edge, stft_ratio(re, im, re_, bound))
    _report(f"stft n{N} pad{pad_mode}", worst)
    assert worst <= 1.0
    assert neg_rev > NEG                                       # window reversed
    if pad_mode == 1:
        assert neg_edge > NEG                                  # edge padding instead of reflect padding


# ------------------------------------------------------------------------------------------------------------ GPU: whisper log-mel
WHISPER_CASES = [                                 # (n_mels, n, padding, id); CTA 3 starts its first frame at 24 * 160 - 200 = 3640
    (80, 16080, 0, "pad0"), (128, 16080, 0, "pad0"),
    (80, 4013, 250, "pad250"),
    (80, 3640, 400, "pad400-start-at-n"), (128, 3640, 400, "pad400-start-at-n"),
    (80, 3639, 400, "pad400-start-n+1"),
    (80, 3641, 400, "pad400-start-n-1"),
    (80, 3640, 399, "pad399-start-at-n"), (128, 3640, 399, "pad399-start-at-n"),
    (128, 16000, 480000, "pad480000"),
]


def _whisper_inputs(n, seed):
    """Rows of rms 1 (noise plus a 440 Hz tone), rms 1e-3, and silence."""
    g = _rng(seed)
    t = np.arange(n) / 16000.0
    loud = 0.7 * g.standard_normal(n) + np.sin(2 * np.pi * 440 * t)
    return np.stack([loud, 1e-3 * g.standard_normal(n), np.zeros(n)]).astype(np.float32)


def _whisper_consts(n_mels):
    filt = OD.mel_filters(16000, 400, n_mels, norm="slaney", mel_scale=None)
    return filt, torch.as_tensor(OD.hanning(400)).float().to(DEV), torch.as_tensor(filt).to(DEV)


@gpu
@pytest.mark.parametrize("n_mels,n,padding", [c[:3] for c in WHISPER_CASES], ids=[f"m{c[0]}-{c[3]}" for c in WHISPER_CASES])
def test_whisper_logmel_vs_float64(n_mels, n, padding):
    from mlx_audio_b200 import ops
    filt, wd, fd = _whisper_consts(n_mels)
    x = _whisper_inputs(n, n + padding)
    frames = (n + padding) // 160
    xd = _strided_rows(x)
    ops.whisper_logmel(1e3 * xd, padding, wd, fd, frames)                  # a loud batch first: its maxima must not carry over
    y = ops.whisper_logmel(xd, padding, wd, fd, frames)
    L, bL = whisper_ref(x, padding, filt, frames)
    worst = whisper_ratio(y, L, bL)
    _report(f"whisper m{n_mels} n{n} pad{padding}", worst)
    assert worst <= 1.0
    assert bool((y[2] == -1.5).all())                                      # the silent row: (-10 + 4) / 4 exactly
    Le, _ = whisper_ref(x, padding, filt, frames, reflect_as="edge")
    assert whisper_ratio(y, Le, bL) > NEG                                  # edge padding instead of reflect padding


@gpu
@pytest.mark.parametrize("n_mels", [80, 128])
def test_whisper_shortcut_equals_transform(n_mels):
    """Frame 24 (CTA 3) of n = 3640 sees only zero padding: with padding 400 the kernel writes it without a transform, with padding 399
    it runs the transform on the same zeros.  Frames 0..23 read the same samples in both, so both outputs are bit-identical."""
    from mlx_audio_b200 import ops
    _, wd, fd = _whisper_consts(n_mels)
    xd = _strided_rows(_whisper_inputs(3640, 7))
    a = ops.whisper_logmel(xd, 400, wd, fd, 25)
    b = ops.whisper_logmel(xd, 399, wd, fd, 25)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------ GPU: istft
ISTFT_NFFT = [2, 16, 64, 400, 1024, 4096]
HOP_KINDS = {"quarter": lambda N: max(1, N // 4), "half": lambda N: max(1, N // 2), "full": lambda N: N, "nondiv": _nondiv,
             "gap": lambda N: N + 3}


def _istft_windows(N):
    hann = OD.hanning(N, periodic=True).astype(np.float32)
    rnd = _rand_window(N, 3 * N)
    rnd[0] = 3e-11                                    # 0 < w[0], w[0]^2 < 1e-10: the clamp modes differ at sample 0 with trim 0
    return {"hann": hann, "rand": rnd}


@gpu
@pytest.mark.parametrize("hop_kind", list(HOP_KINDS))
@pytest.mark.parametrize("N", ISTFT_NFFT, ids=[f"n{n}" for n in ISTFT_NFFT])
def test_istft_vs_float64(N, hop_kind):
    from mlx_audio_b200 import ops
    hop = HOP_KINDS[hop_kind](N)
    nf = N // 2 + 1
    worst, neg_clamp, neg_dc = 0.0, np.inf, np.inf
    for T in (1, 2, 3, 937):
        g = _rng(N * 7 + T)
        re, im = g.standard_normal((2, nf, T)).astype(np.float32), g.standard_normal((2, nf, T)).astype(np.float32)
        im[:, 0], im[:, N // 2] = 10 * g.standard_normal((2, T)), 10 * g.standard_normal((2, T))   # ignored by the inverse rFFT
        red, imd = torch.as_tensor(re).to(DEV), torch.as_tensor(im).to(DEV)
        full = (T - 1) * hop + N
        for wname, w in _istft_windows(N).items():
            w64 = w.astype(np.float64)
            wd = torch.as_tensor(w).to(DEV)
            parts = istft_ola(*irfft_frames(re, im, N, w64), N, hop, w64)
            j = 0
            for norm_sq in (True, False):
                for clamp_mode in (0, 1):
                    for trim in (0, N // 2):
                        out_len = full - trim if j % 2 == 0 else max(1, full - trim - hop - 1)
                        j += 1
                        y = ops.istft(red, imd, N, hop, wd, norm_sq=norm_sq, clamp_mode=clamp_mode, trim=trim, out_len=out_len)
                        ref, bound = istft_ref(parts, norm_sq, clamp_mode, trim, out_len)
                        worst = max(worst, ratio(y, ref, bound))
                        if trim == 0 and wname == "rand" and T == 3:
                            other, _ = istft_ref(parts, norm_sq, 1 - clamp_mode, trim, out_len)
                            neg_clamp = min(neg_clamp, ratio(y, other, bound))
                        if T == 3 and trim == N // 2 and norm_sq and clamp_mode == 0 and wname == "hann":
                            alt, _ = istft_ref(istft_ola(*irfft_frames(re, im, N, w64, dc_nyq="abs"), N, hop, w64), norm_sq, clamp_mode, trim,
                                               out_len)
                            neg_dc = min(neg_dc, ratio(y, alt, bound))
    _report(f"istft n{N} {hop_kind}", worst)
    assert worst <= 1.0
    assert neg_clamp > NEG                                         # the other clamp_mode's rule
    assert neg_dc > NEG                                            # DC / Nyquist imaginary parts counted


@gpu
@pytest.mark.parametrize("N", [2, 64, 4096])
def test_istft_ignores_dc_nyquist_imag(N):
    from mlx_audio_b200 import ops
    g = _rng(N)
    T, hop = 5, max(1, N // 4)
    re, im = torch.as_tensor(g.standard_normal((2, N // 2 + 1, T)), dtype=torch.float32), torch.as_tensor(g.standard_normal((2, N // 2 + 1, T)), dtype=torch.float32)
    w = torch.as_tensor(_rand_window(N, 1)).to(DEV)
    im0, imn = im.clone(), im.clone()
    im0[:, 0], im0[:, N // 2] = 0.0, 0.0
    imn[:, 0], imn[:, N // 2] = float("nan"), float("nan")
    kw = dict(norm_sq=True, clamp_mode=1, trim=0, out_len=(T - 1) * hop + N)
    a = ops.istft(re.to(DEV), im0.to(DEV), N, hop, w, **kw)
    b = ops.istft(re.to(DEV), imn.to(DEV), N, hop, w, **kw)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------ GPU: Kokoro source + head
def _f0_curve(nF, seed, kind):
    g = _rng(seed)
    f0 = (80 + 300 * g.random(nF)).astype(np.float32)
    f0[: max(0, nF // 6)] = 0.0
    if kind == "threshold":                                        # the voiced test f0 > 10 at its edge, in float32
        edge = np.array([10.0, np.nextafter(np.float32(10), np.float32(11)), np.nextafter(np.float32(10), np.float32(9))], np.float32)
        f0[nF // 3: nF // 3 + 3] = edge[: max(0, min(3, nF - nF // 3))]
    elif kind == "high":                                           # the 9th harmonic passes 12 kHz
        f0[nF // 2:] = 1400.0 + 200 * g.random(nF - nF // 2)
    return f0


SOURCE_CASES = [  # (nF, B, noise, f0 kind)
    (1, 1, True, "plain"), (1, 3, False, "plain"),
    (2, 3, False, "plain"), (2, 1, True, "threshold"),
    (14, 3, True, "threshold"), (14, 3, False, "threshold"),
    (46, 3, False, "high"), (46, 2, True, "high"),
    (600, 2, True, "threshold"),
]


@gpu
@pytest.mark.parametrize("nF,B,with_noise,kind", SOURCE_CASES,
                         ids=[f"nF{c[0]}-B{c[1]}-{'noise' if c[2] else 'silent'}-{c[3]}" for c in SOURCE_CASES])
def test_kokoro_source_vs_float64(nF, B, with_noise, kind):
    from mlx_audio_b200 import ops
    f0 = np.stack([_f0_curve(nF, 10 * nF + b, kind if b != 1 else "plain") * (1.0 if b != 2 else 0.5) for b in range(B)])
    if kind == "threshold":
        f0[-1] = _f0_curve(nF, 99, kind)
    noise = _rng(nF).standard_normal((B, nF * 300, 9)).astype(np.float32) if with_noise else None
    g = _rng(5)
    lw, lb = (0.3 * g.standard_normal(9)).astype(np.float32), (0.1 * g.standard_normal(1)).astype(np.float32)
    lwd, lbd = torch.as_tensor(lw).to(DEV), torch.as_tensor(lb).to(DEV)
    nd = None if noise is None else torch.as_tensor(noise).to(DEV)
    har = ops.kokoro_source(torch.as_tensor(f0).to(DEV), nd, lwd, lbd)
    for b in range(B):                                              # rows are independent of their batch
        one = ops.kokoro_source(torch.as_tensor(f0[b:b + 1]).to(DEV), None if nd is None else nd[b:b + 1].contiguous(), lwd, lbd)
        assert torch.equal(one[0], har[b])
    har = har.cpu().numpy().astype(np.float64)
    mag, ph, be = source_ref(f0, noise, lw, lb[0])
    assert har.shape == (B, nF * 60 + 1, 22)
    bmag = be[..., None] + 2 * U * mag
    r_mag = float((np.abs(har[..., :11] - mag) / bmag).max())
    floor = mag > 1e-4
    dphi = np.abs(np.angle(np.exp(1j * (har[..., 11:] - ph))))
    r_ph = float((dphi / (1.5 * bmag / np.maximum(mag, 1e-300) + 4 * np.pi * U))[floor].max())
    _report(f"source nF{nF} B{B} noise={with_noise} {kind}", max(r_mag, r_ph))
    assert r_mag <= 1.0 and r_ph <= 1.0
    real = np.zeros_like(floor)                                     # exactly-real bins: DC, Nyquist, all of frame 0
    real[..., [0, 10]] = True
    real[:, 0, :] = True
    ang = har[..., 11:][real & (mag > 1e-2)]
    assert np.isin(ang.astype(np.float32), [np.float32(0.0), np.float32(np.pi)]).all()
    if kind == "threshold":
        mag_ge, _, _ = source_ref(f0, noise, lw, lb[0], voiced_threshold=float(np.nextafter(10.0, 0.0)))
        assert float((np.abs(har[..., :11] - mag_ge) / bmag).max()) > NEG          # f0 = 10.0 counted as voiced


@gpu
@pytest.mark.parametrize("T", [2, 3, 300, 4001])
def test_kokoro_istft_head_vs_float64(T):
    from mlx_audio_b200 import ops
    g = _rng(T)
    B = 2
    buf = torch.full((2 * B, T, 64), float("nan"))
    xv = np.concatenate([g.uniform(-4, 8, (B, T, 11)), g.uniform(-6, 6, (B, T, 11))], -1).astype(np.float32)
    buf[::2, :, 17:39] = torch.as_tensor(xv)
    x = buf.to(DEV)[::2, :, 17:39]
    assert x.stride() == (2 * T * 64, 64, 1)
    y = ops.kokoro_istft_head(x)
    ref, bound = head_ref(xv)
    assert y.shape == ref.shape
    worst = ratio(y, ref, bound)
    _report(f"head T{T}", worst)
    assert worst <= 1.0
    alt, _ = head_ref(xv, flip_phase=True)
    assert ratio(y, alt, bound) > NEG                                          # phase sign flipped


# ------------------------------------------------------------------------------------------------------------ GPU: randn
TOL_RANDN = 1e-5
SEED_HI = 0x9E3779B97F4A7C15 & 0x7FFFFFFFFFFFFFFF                  # high word set; fits the int64 device state


@gpu
@pytest.mark.parametrize("n", [0, 1, 2, 3, 4, 5, 1023, 5_000_001])
def test_randn_vs_reference(n):
    from mlx_audio_b200 import ops
    for seed, offset in ((0, 0), (SEED_HI, 0), (12345, (1 << 32) - 2), (SEED_HI, 0x1_2345_6789)):
        y = ops.randn_(torch.full((n,), float("nan"), device=DEV), seed, offset).double().cpu().numpy()
        ref = randn_ref(n, seed, offset)
        err = float(np.abs(y - ref).max()) if n else 0.0
        _report(f"randn n{n} seed{seed:x} off{offset:x}", err / TOL_RANDN)
        assert err <= TOL_RANDN
        if n >= 4 and seed == SEED_HI and offset == 0:
            assert float(np.abs(y - randn_ref(n, seed, offset, m0=PH_M0 + 1)).max()) > NEG * TOL_RANDN   # a round constant changed
            assert float(np.abs(y - randn_ref(n, seed, offset, w0=PH_W0 + 1)).max()) > NEG * TOL_RANDN   # the key increment changed


@gpu
def test_randn_stream_continuity():
    from mlx_audio_b200 import ops
    seed, off = SEED_HI, (1 << 32) - 3
    whole = ops.randn_(torch.empty(4000 + 1237, device=DEV), seed, off)
    a = ops.randn_(torch.empty(4000, device=DEV), seed, off)
    b = ops.randn_(torch.empty(1237, device=DEV), seed, off + 1000)
    assert torch.equal(torch.cat([a, b]), whole)
    state = torch.tensor([seed, off], dtype=torch.int64, device=DEV)
    expect = off
    for n in (7, 4, 1, 1025):                                          # advances by ceil(n / 4) each call
        y = ops.randn_dev_(torch.empty(n, device=DEV), state)
        assert torch.equal(y, ops.randn_(torch.empty(n, device=DEV), seed, expect))
        expect += -(-n // 4)
        assert int(state[1]) == expect and int(state[0]) == seed
    ops.randn_dev_(torch.empty(0, device=DEV), state)                  # an empty tensor draws nothing
    assert int(state[1]) == expect
    n = 901
    out = torch.empty(n, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.randn_dev_(out, torch.tensor([seed, 0], dtype=torch.int64, device=DEV))    # warm-up outside the capture
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.randn_dev_(out, state)
    s.synchronize()
    assert int(state[1]) == expect                                     # capturing runs nothing
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ops.randn_(torch.empty(n, device=DEV), seed, expect))
        expect += -(-n // 4)
        assert int(state[1]) == expect


@gpu
def test_randn_distribution():
    from scipy import stats
    from mlx_audio_b200 import ops
    n = 1 << 22
    x = ops.randn_(torch.empty(n, device=DEV), 20240601, 0).double().cpu().numpy()
    sd = 1 / math.sqrt(n)
    assert abs(x.mean()) < 5 * sd
    assert abs(x.var() - 1) < 5 * math.sqrt(2) * sd
    for lag in (1, 2, 3, 4):
        assert abs(float(np.mean(x[:-lag] * x[lag:]))) < 5 * sd
    p4 = 2 * stats.norm.sf(4)
    assert abs(int((np.abs(x) > 4).sum()) - n * p4) < 5 * math.sqrt(n * p4 * (1 - p4))
    assert stats.kstest(x, "norm").pvalue > 5.7e-7


# ------------------------------------------------------------------------------------------------------------ GPU: resample_poly
RATES = [(44100, 24000), (48000, 16000), (16000, 24000), (24000, 16000), (22050, 24000)]


@gpu
@pytest.mark.parametrize("n_in", [1, 50, 48000])
@pytest.mark.parametrize("orig,target", RATES, ids=[f"{a}to{b}" for a, b in RATES])
def test_resample_poly_vs_float64(orig, target, n_in):
    from mlx_audio_b200 import ops
    up, down, h, pre, rem, n_out = resample_plan(orig, target, n_in)
    x = _rng(n_in + orig).standard_normal((2, n_in)).astype(np.float32)
    xd = _strided_rows(x, extra=11, off=3)
    y = ops.resample_poly(xd, torch.as_tensor(h, dtype=torch.float64).to(DEV), up, down, pre, rem, n_out).double().cpu().numpy()
    worst, neg = 0.0, np.inf
    for b in range(2):
        ref, absum = resample_ref(x[b], h, up, down, pre, rem, n_out)
        bound = U * np.abs(ref) + 2.0 ** -40 * absum + 2.0 ** -149
        worst = max(worst, ratio(y[b], ref, bound))
        if up > 1 and n_in > 1:                                        # one input sample: every phase sums to about 1
            alt, _ = resample_ref(x[b], h, up, down, pre, rem, n_out, t0_shift=1)
            neg = min(neg, ratio(y[b], alt, bound))
    _report(f"resample {orig}->{target} n_in{n_in}", worst)
    assert worst <= 1.0
    if up > 1 and n_in > 1:
        assert neg > NEG                                               # filter phase t0 off by one


# ------------------------------------------------------------------------------------------------------------ GPU: speaker / Vocos log-mel
MEL_CASES = [("spk", 385), ("spk", 386), ("spk", 511), ("spk", 2304), ("spk", 4352 + 100),
             ("vocos", 513), ("vocos", 514), ("vocos", 2304), ("vocos", 4352 + 255)]


@gpu
@pytest.mark.parametrize("kind,n", MEL_CASES, ids=[f"{k}-n{n}" for k, n in MEL_CASES])
def test_mel_logmel_vs_float64(kind, n):
    from mlx_audio_b200 import ops
    fn = ops.spk_logmel if kind == "spk" else ops.vocos_logmel
    filt = _spk_filters() if kind == "spk" else _vocos_filters()
    w = _rand_window(MEL_N, 11)
    wd, fd = torch.as_tensor(w).to(DEV), torch.as_tensor(filt).to(DEV)
    g = _rng(n)
    x = np.stack([0.5 * g.standard_normal(n), 1e-3 * g.standard_normal(n), np.zeros(n)]).astype(np.float32)
    xd = _strided_rows(x)
    y = fn(xd, wd, fd)
    assert y.shape == (3, mel_frames(kind, n), filt.shape[0])
    for b in range(3):
        assert torch.equal(fn(xd[b:b + 1], wd, fd)[0], y[b])
    logs, mel, dmel = mel_ref(kind, x, w, filt)
    worst = mel_ratio(y, logs, mel, dmel)
    _report(f"{kind} logmel n{n}", worst)
    assert worst <= 1.0
    le, _, _ = mel_ref(kind, x, w, filt, pad_as="edge")
    assert mel_ratio(y, le, mel, dmel) > NEG                           # edge padding instead of reflect padding


# ------------------------------------------------------------------------------------------------------------ GPU: host checks
@gpu
def test_argument_checks():
    from mlx_audio_b200 import _lib, ops
    z = lambda *s: torch.zeros(*s, device=DEV)                          # noqa: E731

    def raises(match, fn):
        n0 = ops.LAUNCHES[0]
        with pytest.raises(ValueError, match=match):
            fn()
        assert ops.LAUNCHES[0] == n0

    even = "n_fft must be even and <= 4096"
    raises(even, lambda: ops.stft(z(1, 100), z(3), 3, 1, 0, 1))                         # odd
    raises(even, lambda: ops.stft(z(1, 100), z(1), 1, 1, 0, 1))                         # < 2
    raises(even, lambda: ops.stft(z(1, 5000), z(4098), 4098, 1, 0, 1))                  # > 4096
    raises(even, lambda: ops.istft(z(1, 1, 2), z(1, 1, 2), 1, 1, z(4), norm_sq=True, clamp_mode=0, trim=0, out_len=4))   # < 2, odd
    raises(even, lambda: ops.istft(z(1, 2050, 2), z(1, 2050, 2), 4098, 1, z(4098), norm_sq=True, clamp_mode=0, trim=0, out_len=4))
    raises("reflect padding needs n > n_fft/2", lambda: ops.stft(z(1, 32), z(64), 64, 16, 1, 3))
    ops.stft(z(1, 33), z(64), 64, 16, 1, 3)                                                # n = n_fft / 2 + 1 is legal
    raises("reflect padding needs more than 200 samples", lambda: ops.whisper_logmel(z(1, 100), 100, z(400), z(80, 201), 1))
    raises("bad pointers/shape", lambda: ops.kokoro_istft_head(z(1, 1, 22)))             # T = 1
    raises("384 samples", lambda: ops.spk_logmel(z(1, 384), z(1024), z(128, 513)))
    raises("512 samples", lambda: ops.vocos_logmel(z(1, 512), z(1024), z(100, 513)))
    f0, har, src, ph = z(1, 4), z(1, 241, 22), z(1, 1200), torch.zeros(1, 6, 9, dtype=torch.float64, device=DEV)
    lw, lb = z(9), z(1)
    for n_down in (3, 6):                                                                  # n_down must be nF or nF + 1
        raises("n_down must be", lambda: _lib.check(_lib.lib().b2a_kokoro_source(
            f0.data_ptr(), 1, 4, n_down, None, lw.data_ptr(), lb.data_ptr(), har.data_ptr(), src.data_ptr(), ph.data_ptr(), ops._stream())))
    torch.cuda.synchronize()
