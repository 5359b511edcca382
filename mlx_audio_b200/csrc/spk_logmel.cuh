// Reflect-padded direct-DFT log-mel at n_fft 1024 / hop 256, shared by the Qwen3-TTS speaker front end (speaker.cu: centre pad 384,
// sqrt(|X|^2 + 1e-9)) and Vocos's MelSpectrogramFeatures (vocos.cu: centre pad 512, plain |X|).  Each file instantiates its own
// variant, so the speaker encoder's kernel compiles exactly as it did before Vocos shared it.
#pragma once
#include "common.cuh"

namespace {

constexpr int MEL_FT = 8;          // frames per CTA
constexpr int MEL_N = 1024, MEL_HOP = 256, MEL_NF = MEL_N / 2 + 1;

// One CTA = MEL_FT frames of one item: reflect-padded (by PAD samples, no repeated edge) windowed frames, direct DFT against an
// exact twiddle table (index (k*i) mod N, no accumulated angle), sqrt(|X|^2 + 1e-9) (MAG_EPS) or sqrt(|X|^2), mel projection from a
// table, log(max(., 1e-5)).
template <int PAD, bool MAG_EPS>
__global__ void spk_logmel_kernel(const float* __restrict__ x, int64_t x_bs, int64_t n, const float* __restrict__ window,
                                  const float* __restrict__ filters, int n_mels, int64_t frames, float* __restrict__ out) {
  extern __shared__ __align__(16) float sm[];
  float* tw_c = sm;
  float* tw_s = sm + MEL_N;
  float* fr = sm + 2 * MEL_N;                 // [MEL_FT][MEL_N]
  float* mag = fr + MEL_FT * MEL_N;           // [MEL_FT][MEL_NF]
  const int b = blockIdx.y;
  const int64_t f0 = (int64_t)blockIdx.x * MEL_FT;
  const float* xb = x + (int64_t)b * x_bs;
  for (int i = threadIdx.x; i < MEL_N; i += blockDim.x) { float s, c; sincospif(2.f * i / MEL_N, &s, &c); tw_c[i] = c; tw_s[i] = s; }
  for (int idx = threadIdx.x; idx < MEL_FT * MEL_N; idx += blockDim.x) {
    const int f = idx / MEL_N, i = idx % MEL_N;
    float v = 0.f;
    if (f0 + f < frames) {
      int64_t s = (f0 + f) * MEL_HOP + i - PAD;              // position in the unpadded signal
      if (s < 0) s = -s;
      else if (s >= n) s = 2 * (n - 1) - s;
      v = __ldg(xb + s) * __ldg(window + i);
    }
    fr[idx] = v;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < MEL_FT * MEL_NF; idx += blockDim.x) {
    const int f = idx / MEL_NF, k = idx % MEL_NF;
    const float* xr = fr + f * MEL_N;
    float re = 0.f, im = 0.f;
    int ph = 0;
    for (int i = 0; i < MEL_N; i++) {
      re = fmaf(xr[i], tw_c[ph], re);
      im = fmaf(-xr[i], tw_s[ph], im);
      ph = (ph + k) & (MEL_N - 1);
    }
    mag[idx] = MAG_EPS ? sqrtf(re * re + im * im + 1e-9f) : sqrtf(re * re + im * im);
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < MEL_FT * n_mels; idx += blockDim.x) {
    const int f = idx / n_mels, m = idx % n_mels;
    if (f0 + f >= frames) continue;
    const float* fl = filters + (int64_t)m * MEL_NF;
    const float* mr = mag + f * MEL_NF;
    float acc = 0.f;
    for (int k = 0; k < MEL_NF; k++) acc = fmaf(mr[k], __ldg(fl + k), acc);
    out[((int64_t)b * frames + f0 + f) * n_mels + m] = logf(fmaxf(acc, 1e-5f));
  }
}

constexpr size_t spk_logmel_smem_bytes() { return (size_t)(2 * MEL_N + MEL_FT * MEL_N + MEL_FT * MEL_NF) * sizeof(float); }

}  // namespace
