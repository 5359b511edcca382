// DSP frontend / backend kernels (include/b200audio.h): STFT, Whisper log-mel, iSTFT, and the Kokoro
// hn-NSF source + iSTFT head.  All HBM-bound or latency-bound; the transforms are direct DFTs against
// an exact twiddle table in shared memory (index (k*n) mod N, so no angle accumulates error).
#include "common.cuh"

namespace {

constexpr int FT = 8;   // frames per CTA

__device__ __forceinline__ float load_padded(const float* __restrict__ x, int64_t n, int64_t n_total, int64_t i,
                                              int pad, int pad_mode) {
  // i indexes the (virtually) centre-padded signal; samples in [n, n_total) are the caller's zero padding
  int64_t s = i - pad;
  if (s < 0) { if (pad_mode == 1) s = -s; else return 0.f; }
  else if (s >= n_total) { if (pad_mode == 1) s = 2 * (n_total - 1) - s; else return 0.f; }
  return (s >= 0 && s < n) ? __ldg(x + s) : 0.f;
}

// Power or complex spectrum of FT frames per CTA. smem: tw_c[N], tw_s[N], fr[FT][N]
template <bool POWER>
__device__ void dft_frames(const float* __restrict__ x, int64_t n, int64_t n_total, const float* __restrict__ window,
                           int N, int hop, int pad, int pad_mode, int64_t f0, int64_t frames, float* sm,
                           float* out_a, float* out_b, int64_t out_stride /* per frame */) {
  float* tw_c = sm; float* tw_s = sm + N; float* fr = sm + 2 * N;
  const int nf = N / 2 + 1;
  for (int i = threadIdx.x; i < N; i += blockDim.x) { float s, c; sincospif(2.f * i / N, &s, &c); tw_c[i] = c; tw_s[i] = s; }
  for (int idx = threadIdx.x; idx < FT * N; idx += blockDim.x) {
    int f = idx / N, i = idx % N;
    int64_t fr_idx = f0 + f;
    fr[idx] = fr_idx < frames ? load_padded(x, n, n_total, fr_idx * hop + i, pad, pad_mode) * __ldg(window + i) : 0.f;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < FT * nf; idx += blockDim.x) {
    int f = idx / nf, k = idx % nf;
    if (f0 + f >= frames) continue;
    const float* xr = fr + f * N;
    float re = 0.f, im = 0.f;
    int ph = 0;
    for (int i = 0; i < N; i++) {
      re = fmaf(xr[i], tw_c[ph], re); im = fmaf(-xr[i], tw_s[ph], im);
      ph += k; if (ph >= N) ph -= N;
    }
    if (POWER) out_a[f * out_stride + k] = re * re + im * im;
    else { out_a[(f0 + f) * out_stride + k] = re; out_b[(f0 + f) * out_stride + k] = im; }
  }
}

__global__ void stft_kernel(const float* __restrict__ x, int64_t x_bs, int64_t n, const float* __restrict__ window, int N,
                            int hop, int pad_mode, int64_t frames, float* __restrict__ out_re, float* __restrict__ out_im) {
  extern __shared__ __align__(16) float sm[];
  const int b = blockIdx.y;
  const int nf = N / 2 + 1;
  dft_frames<false>(x + (int64_t)b * x_bs, n, n, window, N, hop, pad_mode ? N / 2 : 0, pad_mode, (int64_t)blockIdx.x * FT, frames,
                    sm, out_re + (int64_t)b * frames * nf, out_im + (int64_t)b * frames * nf, nf);
}

__device__ __forceinline__ void atomic_max_pos(float* addr, float v) { atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v)); }

// log10(max(mel,1e-10)) per frame + per-utterance max (stored with a +16 offset so the int atomicMax trick is valid)
__global__ void whisper_logmel_kernel(const float* __restrict__ x, int64_t x_bs, int64_t n, int64_t padding,
                                      const float* __restrict__ window, const float* __restrict__ filters, int n_mels,
                                      int64_t frames, float* __restrict__ out, float* __restrict__ gmax) {
  constexpr int N = 400, HOP = 160, NF = 201;
  extern __shared__ __align__(16) float sm[];
  float* pw = sm + 2 * N + FT * N;       // [FT][NF]
  __shared__ float bmax[8];
  const int b = blockIdx.y;
  const int64_t f0 = (int64_t)blockIdx.x * FT, n_total = n + padding;
  float* ob = out + (int64_t)b * frames * n_mels;
  float lmax = -16.f;
  // frames that only see the caller's zero padding: log10(1e-10) = -10 without doing the transform
  const bool all_zero = (f0 * HOP - N / 2 >= n) && ((f0 + FT - 1) * HOP - N / 2 + N <= n_total || padding >= N);
  if (all_zero) {
    for (int idx = threadIdx.x; idx < FT * n_mels; idx += blockDim.x) {
      int f = idx / n_mels; if (f0 + f < frames) ob[(f0 + f) * n_mels + idx % n_mels] = -10.f;
    }
    lmax = -10.f;
  } else {
    dft_frames<true>(x + (int64_t)b * x_bs, n, n_total, window, N, HOP, N / 2, 1, f0, frames, sm, pw, nullptr, NF);
    __syncthreads();
    for (int idx = threadIdx.x; idx < FT * n_mels; idx += blockDim.x) {
      int f = idx / n_mels, m = idx % n_mels;
      if (f0 + f >= frames) continue;
      const float* fl = filters + (int64_t)m * NF;
      const float* pr = pw + f * NF;
      float acc = 0.f;
      for (int k = 0; k < NF; k++) acc = fmaf(pr[k], __ldg(fl + k), acc);
      float lv = log10f(fmaxf(acc, 1e-10f));
      ob[(f0 + f) * n_mels + m] = lv;
      lmax = fmaxf(lmax, lv);
    }
  }
  lmax = warp_max(lmax);
  if ((threadIdx.x & 31) == 0) bmax[threadIdx.x >> 5] = lmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = bmax[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); i++) v = fmaxf(v, bmax[i]);
    atomic_max_pos(gmax + b, v + 16.f);
  }
}

__global__ void whisper_logmel_finish(float* __restrict__ out, const float* __restrict__ gmax, int64_t per_batch, int B) {
  int64_t total = per_batch * B;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float mx = gmax[i / per_batch] - 16.f;
    out[i] = (fmaxf(out[i], mx - 8.f) + 4.f) * 0.25f;
  }
}

// inverse rFFT of every frame times the synthesis window -> ws [B, T, N]
__global__ void irfft_frames_kernel(const float* __restrict__ re, const float* __restrict__ im, int N, int T,
                                    const float* __restrict__ window, float* __restrict__ ws) {
  extern __shared__ __align__(16) float sm[];
  float* tw_c = sm; float* tw_s = sm + N; float* sr = sm + 2 * N; float* si = sr + (N / 2 + 1);
  const int nf = N / 2 + 1, t = blockIdx.x, b = blockIdx.y;
  for (int i = threadIdx.x; i < N; i += blockDim.x) { float s, c; sincospif(2.f * i / N, &s, &c); tw_c[i] = c; tw_s[i] = s; }
  for (int k = threadIdx.x; k < nf; k += blockDim.x) {
    sr[k] = re[((int64_t)b * nf + k) * T + t]; si[k] = im[((int64_t)b * nf + k) * T + t];
  }
  __syncthreads();
  for (int m = threadIdx.x; m < N; m += blockDim.x) {
    float acc = sr[0];
    int ph = 0;
    for (int k = 1; k < nf; k++) {
      ph += m; if (ph >= N) ph -= N;
      float wgt = (2 * k == N) ? 1.f : 2.f;              // Nyquist bin counted once; its imaginary part is ignored
      float term = sr[k] * tw_c[ph] - ((2 * k == N) ? 0.f : si[k] * tw_s[ph]);
      acc = fmaf(wgt, term, acc);
    }
    ws[((int64_t)b * T + t) * N + m] = acc / N * __ldg(window + m);
  }
}

__global__ void ola_kernel(const float* __restrict__ ws, int N, int T, int hop, const float* __restrict__ window,
                           int norm_sq, int clamp_mode, int64_t trim, int64_t out_len, float* __restrict__ out, int B) {
  int64_t total = out_len * B;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int b = (int)(idx / out_len);
    int64_t pos = idx % out_len + trim;
    int64_t f_hi = pos / hop; if (f_hi > T - 1) f_hi = T - 1;
    int64_t f_lo = (pos - N + hop) / hop; if (pos - N + 1 <= 0) f_lo = 0; if (f_lo < 0) f_lo = 0;
    float acc = 0.f, wsum = 0.f;
    for (int64_t f = f_lo; f <= f_hi; f++) {
      int m = (int)(pos - f * hop);
      if (m < 0 || m >= N) continue;
      acc += ws[((int64_t)b * T + f) * N + m];
      float w = __ldg(window + m);
      wsum += norm_sq ? w * w : w;
    }
    if (clamp_mode == 0) out[idx] = wsum > 1e-10f ? acc / wsum : acc;
    else out[idx] = acc / fmaxf(wsum, 1e-10f);
  }
}

// ---------------------------------------------------------------- Kokoro hn-NSF source
constexpr int KH = 9;              // harmonics (fundamental + 8)
constexpr int KUP = 300;           // samples per F0 frame
constexpr double KSR = 24000.0;

// Frame-rate phase of the reference (istftnet.py:585-591): the sample-rate rad values (piecewise constant per F0 frame) are
// linearly DOWN-sampled to n_down points (interpolate1d, align_corners False), then cumulatively summed.  n_down =
// ceil(float(L) * float(1/300)) is computed by the host exactly as the reference does and is nF or nF+1 depending on
// floating-point rounding, so the positions are NOT frame-aligned in general.
__device__ __forceinline__ double ksrc_rad(const float* __restrict__ f0b, int64_t n, int h) {
  double r = (double)f0b[n / KUP] * (h + 1) / KSR;
  return r - floor(r);
}
__device__ __forceinline__ double ksrc_rad_down(const float* __restrict__ f0b, int64_t L, int n_down, int i, int h) {
  const double sc = (double)L / (double)n_down;
  double x = (double)i * sc + 0.5 * sc - 0.5; if (x < 0) x = 0;
  int64_t lo = (int64_t)floor(x); int64_t hi = lo + 1 < L ? lo + 1 : L - 1; double fr = x - (double)lo;
  return ksrc_rad(f0b, lo, h) * (1.0 - fr) + ksrc_rad(f0b, hi, h) * fr;
}
// C[b,i,h] = sum_{j<=i} rad_down[j,h]  (phase in cycles)
__global__ void ksrc_phase_kernel(const float* __restrict__ f0, int nF, int n_down, double* __restrict__ ph) {
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
  __shared__ double part[256];
  const float* f0b = f0 + (int64_t)b * nF;
  const int64_t L = (int64_t)nF * KUP;
  const int per = (n_down + nt - 1) / nt, beg = tid * per, end = min(n_down, beg + per);
  double s = 0;
  for (int i = beg; i < end; i++) s += ksrc_rad_down(f0b, L, n_down, i, h);
  part[tid] = s;
  __syncthreads();
  if (tid == 0) { double run = 0; for (int i = 0; i < nt; i++) { double v = part[i]; part[i] = run; run += v; } }
  __syncthreads();
  double run = part[tid];
  for (int i = beg; i < end; i++) {
    run += ksrc_rad_down(f0b, L, n_down, i, h);
    ph[((int64_t)b * n_down + i) * KH + h] = run;
  }
}

__global__ void ksrc_sample_kernel(const float* __restrict__ f0, int nF, int n_down, const double* __restrict__ ph,
                                   const float* __restrict__ noise, const float* __restrict__ lin_w,
                                   const float* __restrict__ lin_b, float* __restrict__ src, int B) {
  const int64_t n_s = (int64_t)nF * KUP, total = n_s * B;
  const double s2 = (double)n_down / (double)((int64_t)n_down * KUP);     // in_width / size of the x300 up-sampling
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int b = (int)(idx / n_s); int64_t n = idx % n_s;
    int fi = (int)(n / KUP);
    float f0v = f0[(int64_t)b * nF + fi];
    float uv = f0v > 10.f ? 1.f : 0.f;
    // linear x300 up-sampling of the frame-rate phase (interpolate.py:94-115, align_corners False, coords clamped at 0)
    double pos = (double)n * s2 + 0.5 * s2 - 0.5; if (pos < 0) pos = 0;
    int lo = (int)floor(pos); int hi = min(lo + 1, n_down - 1); double fr = pos - lo;
    const double* p_lo = ph + ((int64_t)b * n_down + lo) * KH; const double* p_hi = ph + ((int64_t)b * n_down + hi) * KH;
    float namp = uv * 0.003f + (1.f - uv) * (0.1f / 3.f);
    float accv = lin_b[0];
#pragma unroll
    for (int h = 0; h < KH; h++) {
      double cyc = (p_lo[h] * (1.0 - fr) + p_hi[h] * fr) * KUP;       // phase / 2pi
      cyc -= floor(cyc);
      float sv = (float)sinpi(2.0 * cyc) * 0.1f;
      float nz = noise ? noise[idx * KH + h] : 0.f;
      accv = fmaf(lin_w[h], sv * uv + namp * nz, accv);
    }
    src[idx] = tanhf(accv);
  }
}

__constant__ double c_tw20_c[20], c_tw20_s[20], c_hann20[20];

// STFT(n_fft 20, hop 5, periodic Hann, reflect centre) of the merged source -> |X| (11) | angle (11), float64 inside
__global__ void ksrc_stft_kernel(const float* __restrict__ src, int64_t n_s, float* __restrict__ har, int B) {
  const int64_t T = n_s / 5 + 1, total = T * B;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int b = (int)(idx / T); int64_t t = idx % T;
    const float* sp = src + (int64_t)b * n_s;
    double xw[20];
#pragma unroll
    for (int i = 0; i < 20; i++) {
      int64_t s = t * 5 + i - 10;
      if (s < 0) s = -s; else if (s >= n_s) s = 2 * (n_s - 1) - s;
      xw[i] = (double)sp[s] * c_hann20[i];
    }
    float* hp = har + idx * 22;
#pragma unroll
    for (int k = 0; k < 11; k++) {
      double re = 0, im = 0;
#pragma unroll
      for (int i = 0; i < 20; i++) { int p = (k * i) % 20; re += xw[i] * c_tw20_c[p]; im -= xw[i] * c_tw20_s[p]; }
      // Exactly-real bins (DC, Nyquist, and every bin of the reflect-symmetric frame 0) have an imaginary part that is pure
      // rounding noise; its sign would pick +pi or -pi at random (in the reference's FFT too).  Canonical choice on both
      // sides of the parity test: treat |im| <= 1e-12 |re| as +0, i.e. angle 0 or +pi.
      if (fabs(im) <= 1e-12 * fabs(re)) im = 0.0;
      hp[k] = (float)sqrt(re * re + im * im);
      hp[11 + k] = (float)atan2(im, re);
    }
  }
}

// conv_post output [T,22] -> waveform: spec = exp(x[:11]), phase = sin(x[11:]), X = spec*e^{j phase},
// 20-point inverse rFFT, periodic Hann, overlap-add (hop 5), / sum w^2, trim 10 each side.
__global__ void kokoro_istft_head_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int T,
                                         float* __restrict__ audio, int B) {
  const int64_t out_len = (int64_t)(T - 1) * 5, total = out_len * B;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int b = (int)(idx / out_len); int64_t pos = idx % out_len + 10;
    int64_t f_hi = pos / 5; if (f_hi > T - 1) f_hi = T - 1;
    int64_t f_lo = (pos - 19 + 4) / 5; if (f_lo < 0) f_lo = 0;
    float acc = 0.f, wsum = 0.f;
    for (int64_t f = f_lo; f <= f_hi; f++) {
      int m = (int)(pos - f * 5);
      if (m < 0 || m >= 20) continue;
      const float* xp = x + (int64_t)b * x_bs + f * x_ld;
      float tsum = 0.f;
#pragma unroll
      for (int k = 0; k < 11; k++) {
        float mag = expf(xp[k]);
        float phs = sinf(xp[11 + k]);
        float sn, cs; sincosf(phs, &sn, &cs);
        int p = (k * m) % 20;
        float c = (float)c_tw20_c[p], s = (float)c_tw20_s[p];
        if (k == 0) tsum += mag * cs;
        else if (k == 10) tsum += mag * cs * c;                      // Nyquist: real part only, cos(pi m)
        else tsum += 2.f * mag * (cs * c - sn * s);
      }
      float w = (float)c_hann20[m];
      acc = fmaf(tsum * 0.05f, w, acc);
      wsum = fmaf(w, w, wsum);
    }
    audio[idx] = wsum > 1e-10f ? acc / wsum : acc;
  }
}

bool g_tw20_init = false;
void init_tw20() {
  if (g_tw20_init) return;
  double c[20], s[20], w[20];
  for (int i = 0; i < 20; i++) {
    c[i] = cos(2.0 * M_PI * i / 20.0); s[i] = sin(2.0 * M_PI * i / 20.0);
    w[i] = 0.5 * (1.0 - cos(2.0 * M_PI * i / 20.0));                // periodic Hann(20), istftnet.py:469
  }
  cudaMemcpyToSymbol(c_tw20_c, c, sizeof(c)); cudaMemcpyToSymbol(c_tw20_s, s, sizeof(s)); cudaMemcpyToSymbol(c_hann20, w, sizeof(w));
  g_tw20_init = true;
}

int grid_for(int64_t total, int bs) { int64_t g = (total + bs - 1) / bs; return (int)(g > 132 * 16 ? 132 * 16 : (g < 1 ? 1 : g)); }

}  // namespace

extern "C" int32_t b2a_stft(const float* x, int64_t x_bs, int32_t B, int64_t n, const float* window, int32_t n_fft, int32_t hop,
                            int32_t pad_mode, int64_t frames, float* out_re, float* out_im, void* stream) {
  B2A_CHECK_ARG(x && window && out_re && out_im && B > 0 && n > 0 && hop > 0 && frames > 0, "bad pointers/shape");
  B2A_CHECK_ARG(n_fft >= 2 && n_fft <= 4096 && n_fft % 2 == 0, "n_fft must be even and <= 4096");
  if (pad_mode == 1) B2A_CHECK_ARG(n > n_fft / 2, "reflect padding needs n > n_fft/2");
  size_t smem = (size_t)(2 + FT) * n_fft * sizeof(float);
  B2A_SMEM_OPTIN(stft_kernel, 200 * 1024);
  dim3 grid(cdiv(frames, FT), B);
  stft_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(x, x_bs, n, window, n_fft, hop, pad_mode, frames, out_re, out_im);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_whisper_logmel(const float* x, int64_t x_bs, int32_t B, int64_t n, int64_t padding, const float* window,
                                      const float* filters, int32_t n_mels, int64_t frames, float* out, float* gmax, void* stream) {
  B2A_CHECK_ARG(x && window && filters && out && gmax && B > 0 && n > 0 && padding >= 0 && frames > 0 && n_mels > 0, "bad pointers/shape");
  B2A_CHECK_ARG(n + padding > 200, "reflect padding needs more than 200 samples");
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(gmax, 0, sizeof(float) * B, st);
  size_t smem = (size_t)((2 + FT) * 400 + FT * 201) * sizeof(float);
  B2A_SMEM_OPTIN(whisper_logmel_kernel, 64 * 1024);
  dim3 grid(cdiv(frames, FT), B);
  whisper_logmel_kernel<<<grid, 256, smem, st>>>(x, x_bs, n, padding, window, filters, n_mels, frames, out, gmax);
  int64_t per = frames * n_mels;
  whisper_logmel_finish<<<grid_for(per * B, 256), 256, 0, st>>>(out, gmax, per, B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_istft(const float* re, const float* im, int32_t B, int32_t n_fft, int32_t T, int32_t hop, const float* window,
                             int32_t norm_sq, int32_t clamp_mode, int64_t trim, int64_t out_len, float* out, float* ws, void* stream) {
  B2A_CHECK_ARG(re && im && window && out && ws && B > 0 && T > 0 && hop > 0 && out_len > 0 && trim >= 0, "bad pointers/shape");
  B2A_CHECK_ARG(n_fft >= 2 && n_fft <= 4096 && n_fft % 2 == 0, "n_fft must be even and <= 4096");
  cudaStream_t st = (cudaStream_t)stream;
  size_t smem = (size_t)(2 * n_fft + 2 * (n_fft / 2 + 1)) * sizeof(float);
  dim3 grid(T, B);
  B2A_SMEM_OPTIN(irfft_frames_kernel, 64 * 1024);      // n_fft = 4096 needs 49 160 B of dynamic shared memory, just above the 48 KB default
  irfft_frames_kernel<<<grid, 128, smem, st>>>(re, im, n_fft, T, window, ws);
  ola_kernel<<<grid_for(out_len * B, 256), 256, 0, st>>>(ws, n_fft, T, hop, window, norm_sq, clamp_mode, trim, out_len, out, B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_kokoro_source(const float* f0, int32_t B, int32_t n_frames, int32_t n_down, const float* noise, const float* lin_w,
                                     const float* lin_b, float* har, float* src_ws, double* ph_ws, void* stream) {
  B2A_CHECK_ARG(f0 && lin_w && lin_b && har && src_ws && ph_ws && B > 0 && n_frames > 0, "bad pointers/shape");
  B2A_CHECK_ARG(n_down >= n_frames && n_down <= n_frames + 1, "n_down must be ceil(float(300*n_frames) * float(1/300))");
  cudaStream_t st = (cudaStream_t)stream;
  init_tw20();
  ksrc_phase_kernel<<<dim3(KH, B), 256, 0, st>>>(f0, n_frames, n_down, ph_ws);
  int64_t n_s = (int64_t)n_frames * KUP;
  ksrc_sample_kernel<<<grid_for(n_s * B, 256), 256, 0, st>>>(f0, n_frames, n_down, ph_ws, noise, lin_w, lin_b, src_ws, B);
  ksrc_stft_kernel<<<grid_for((n_s / 5 + 1) * B, 128), 128, 0, st>>>(src_ws, n_s, har, B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_kokoro_istft_head(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, float* audio, void* stream) {
  B2A_CHECK_ARG(x && audio && B > 0 && T > 1, "bad pointers/shape");
  init_tw20();
  kokoro_istft_head_kernel<<<grid_for((int64_t)(T - 1) * 5 * B, 256), 256, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, T, audio, B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

// ---------------------------------------------------------------- counter-based Gaussian noise (Philox4x32-10 + Box-Muller)
// Replaces mx.random.normal for the SineGen / NoiseBlock draws (istftnet.py:649, snac/layers.py:263) in production runs.
namespace {
__device__ __forceinline__ void philox_round(uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3, uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0, hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
  uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
  c0 = n0; c1 = n1; c2 = n2; c3 = n3;
}
// seed / counter offset either as launch arguments (state == nullptr) or read from device memory {seed, offset}: a captured
// CUDA graph then draws FRESH noise on every replay (randn_advance_kernel moves the offset past the counters just used)
__global__ void randn_kernel(float* __restrict__ out, int64_t n, uint64_t seed, uint64_t offset, const uint64_t* __restrict__ state) {
  if (state) { seed = state[0]; offset = state[1]; }
  int64_t n4 = (n + 3) / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t ctr = offset + (uint64_t)i;
    uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0x2545F491u, c3 = 0x9E3779B9u;
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; r++) { philox_round(c0, c1, c2, c3, k0, k1); k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    float u0 = ((float)c0 + 0.5f) * 2.3283064365386963e-10f, u1 = ((float)c1 + 0.5f) * 2.3283064365386963e-10f;
    float u2 = ((float)c2 + 0.5f) * 2.3283064365386963e-10f, u3 = ((float)c3 + 0.5f) * 2.3283064365386963e-10f;
    float r0 = sqrtf(-2.f * logf(u0)), r1 = sqrtf(-2.f * logf(u2));
    float s0, cs0, s1, cs1; sincospif(2.f * u1, &s0, &cs0); sincospif(2.f * u3, &s1, &cs1);
    float v[4] = {r0 * cs0, r0 * s0, r1 * cs1, r1 * s1};
    for (int j = 0; j < 4; j++) { int64_t o = i * 4 + j; if (o < n) out[o] = v[j]; }
  }
}
__global__ void randn_advance_kernel(uint64_t* state, uint64_t by) { state[1] += by; }
}  // namespace

extern "C" int32_t b2a_randn(float* out, int64_t n, uint64_t seed, uint64_t offset, void* stream) {
  B2A_CHECK_ARG(n >= 0, "bad pointer/size");
  if (n == 0) return B2A_OK;                 // before the pointer check: an empty CUDA tensor has a null data pointer
  B2A_CHECK_ARG(out, "bad pointer/size");
  randn_kernel<<<grid_for((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(out, n, seed, offset, nullptr);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_randn_dev(float* out, int64_t n, uint64_t* state, void* stream) {
  B2A_CHECK_ARG(state && n >= 0, "bad pointer/size");
  if (n == 0) return B2A_OK;
  B2A_CHECK_ARG(out, "bad pointer/size");
  randn_kernel<<<grid_for((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(out, n, 0, 0, state);
  randn_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state, (uint64_t)((n + 3) / 4));
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

// ---------------------------------------------------------------- polyphase resampler (resample.py:10-47 -> scipy.signal.resample_poly)
// out[b, n] = sum_t h[t] * xu[c(n) - t],  c(n) = (n + n_pre_remove)*down - n_pre_pad,  xu[i] = x[clamp(i/up)] when up | i (edge
// padding of the input, padtype="edge"), else 0 -- i.e. only taps t == c (mod up) contribute.  h is the float64 Kaiser-sinc FIR
// already scaled by `up`; accumulation is float64 like SciPy's (float32 x, float64 h), result cast to float32.
namespace {
__global__ void resample_poly_kernel(const float* __restrict__ x, int64_t x_bs, int64_t n_in, const double* __restrict__ h, int n_h,
                                     int up, int down, int64_t n_pre_pad, int64_t n_pre_remove, float* __restrict__ out,
                                     int64_t n_out, int B) {
  const int64_t total = n_out * B;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(idx / n_out); const int64_t n = idx % n_out;
    const float* xb = x + (int64_t)b * x_bs;
    const int64_t c = (n + n_pre_remove) * down - n_pre_pad;
    int64_t t0 = c % up; if (t0 < 0) t0 += up;                       // smallest t >= 0 with t == c (mod up)
    double acc = 0.0;
    for (int64_t t = t0; t < n_h; t += up) {
      int64_t i = (c - t) / up;                                      // exact: up | (c - t)
      i = i < 0 ? 0 : (i >= n_in ? n_in - 1 : i);
      acc += h[t] * (double)__ldg(xb + i);
    }
    out[idx] = (float)acc;
  }
}
}  // namespace

extern "C" int32_t b2a_resample_poly(const float* x, int64_t x_bs, int32_t B, int64_t n_in, const double* h, int32_t n_h, int32_t up,
                                     int32_t down, int64_t n_pre_pad, int64_t n_pre_remove, float* out, int64_t n_out, void* stream) {
  B2A_CHECK_ARG(x && h && out && B > 0 && n_in > 0 && n_h > 0 && up > 0 && down > 0 && n_out > 0, "bad pointers/shape");
  resample_poly_kernel<<<grid_for(n_out * B, 256), 256, 0, (cudaStream_t)stream>>>(x, x_bs, n_in, h, n_h, up, down, n_pre_pad,
                                                                                   n_pre_remove, out, n_out, B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
