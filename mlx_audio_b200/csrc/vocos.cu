// Vocos (codec/models/vocos/{vocos,mel}.py): the ConvNeXt block's depthwise conv + LayerNorm / AdaLayerNorm in one pass
// (b2a_vocos_dwnorm), the ISTFTHead after its linear (b2a_vocos_istft_head), and the log-mel front end on the speaker encoder's
// direct-DFT kernel (b2a_vocos_logmel).  Every sum runs in a fixed order, so a batch row's result does not depend on B.
#include <cuda_bf16.h>
#include "common.cuh"
#include "tc_common.cuh"
#include "layernorm_row.cuh"
#include "spk_logmel.cuh"

namespace {

// ---------------------------------------------------------------- depthwise conv + LayerNorm
constexpr int DN_RT = 16;          // rows per CTA
constexpr int DN_THREADS = 256;    // 8 warps, one row at a time each

// One CTA = DN_RT rows of one item.  With a conv (K > 0) it stages rows t0 - K/2 .. t0 + DN_RT + K/2 - 1 (zero outside [0, L)) in
// shared memory once, so each x element comes from HBM once and the halo rows of neighbouring CTAs from L2; each warp then forms a row
// as bias + sum_k w[k] x[t + k - K/2] (taps ascending) in registers and hands it to layernorm_row_regs.  K == 0: the row is x itself.
template <int NV, bool ADA>
__global__ void __launch_bounds__(DN_THREADS) vocos_dwnorm_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int L, int C,
                                                                  const float* __restrict__ dw_w, const float* __restrict__ dw_b, int K,
                                                                  const float* __restrict__ w, const float* __restrict__ bb,
                                                                  const float* __restrict__ ada, int64_t ada_bs, float eps,
                                                                  float* __restrict__ y, int64_t y_bs, int64_t y_ld,
                                                                  __nv_bfloat16* __restrict__ e_hi, __nv_bfloat16* __restrict__ e_lo) {
  extern __shared__ __align__(16) float4 dn_xs[];       // [DN_RT + K - 1][C / 4]
  const int b = blockIdx.y, t0 = blockIdx.x * DN_RT, nv = C >> 2, h = K >> 1;
  const float* xb = x + (int64_t)b * x_bs;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  if (K > 0) {
    const int rows = DN_RT + K - 1;
    for (int i = threadIdx.x; i < rows * nv; i += DN_THREADS) {
      const int r = i / nv, c4 = i - r * nv, t = t0 - h + r;
      dn_xs[i] = (t >= 0 && t < L) ? __ldg(reinterpret_cast<const float4*>(xb + (int64_t)t * x_ld) + c4) : zero;
    }
    __syncthreads();
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < DN_RT; r += DN_THREADS / 32) {
    const int t = t0 + r;
    if (t >= L) break;
    float4 v[NV];
#pragma unroll
    for (int j = 0; j < NV; j++) {
      const int i = lane + 32 * j;
      v[j] = zero;
      if (i >= nv) continue;
      if (K == 0) { v[j] = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)t * x_ld) + i); continue; }
      float4 a = zero;
#pragma unroll 1
      for (int k = 0; k < K; k++) {
        const float4 wk = __ldg(reinterpret_cast<const float4*>(dw_w + (int64_t)k * C) + i);
        const float4 s = dn_xs[(r + k) * nv + i];
        a.x = fmaf(wk.x, s.x, a.x); a.y = fmaf(wk.y, s.y, a.y); a.z = fmaf(wk.z, s.z, a.z); a.w = fmaf(wk.w, s.w, a.w);
      }
      if (dw_b) { const float4 bv = __ldg(reinterpret_cast<const float4*>(dw_b) + i); a.x += bv.x; a.y += bv.y; a.z += bv.z; a.w += bv.w; }
      v[j] = a;
    }
    const int64_t e = ((int64_t)b * L + t) * C;
    layernorm_row_regs<NV, ADA, true>(v, y ? y + (int64_t)b * y_bs + (int64_t)t * y_ld : nullptr, C, w, bb,
                                      ADA ? ada + (int64_t)b * ada_bs : nullptr, eps, 0, 0, 0.f, e_hi ? e_hi + e : nullptr,
                                      e_lo ? e_lo + e : nullptr, lane);
  }
}

// ---------------------------------------------------------------- ISTFTHead after its linear
constexpr int HD_RUN = 256;        // output samples per CTA, one per thread
constexpr int HD_FCH = 6;          // frames whose spectra are held in shared memory at a time

__device__ __forceinline__ int tw_slot(int i) { return i + (i >> 4); }   // one pad float2 per 16: stride-k reads spread over the banks

// One CTA = HD_RUN consecutive output samples of one item (padded position p = j + N/2).  It forms the complex spectra of the frames
// that overlap its run -- exp, clip at 100, precise sincosf, the irfft's 1/N and 2/N weights folded in, DC / Nyquist imaginary parts
// dropped -- HD_FCH frames at a time, then each thread sums its sample's inverse-DFT terms bin by bin (ascending) for each frame
// (ascending) against an exact twiddle table indexed (k n) mod N, windows them and divides by the summed window where it is > 1e-10.
__global__ void __launch_bounds__(HD_RUN) vocos_istft_head_kernel(const float* __restrict__ hd, int64_t h_bs, int64_t h_ld, int T, int N, int H,
                                                                  const float* __restrict__ window, float* __restrict__ out, int64_t out_bs,
                                                                  int64_t nout) {
  extern __shared__ __align__(16) float2 hd_sm[];
  const int NB = N / 2 + 1;
  float2* tw = hd_sm;                                   // [tw_slot(N)]
  float2* S = hd_sm + tw_slot(N);                       // [HD_FCH][NB]
  const int b = blockIdx.y;
  const int64_t j0 = (int64_t)blockIdx.x * HD_RUN, j = j0 + threadIdx.x;
  const int64_t p0 = j0 + N / 2, p1 = min(j0 + HD_RUN, nout) - 1 + N / 2;
  const int64_t f_lo = p0 - N + 1 > 0 ? (p0 - N + 1 + H - 1) / H : 0;
  const int64_t f_hi = min((int64_t)T - 1, p1 / H);
  for (int i = threadIdx.x; i < N; i += HD_RUN) {
    float s, c;
    sincospif(2.f * i / N, &s, &c);
    tw[tw_slot(i)] = make_float2(c, s);
  }
  const float* hb = hd + (int64_t)b * h_bs;
  const bool valid = j < nout;
  const int64_t p = j + N / 2;
  const float inv_n = 1.f / N, inv_n2 = 2.f / N;
  float num = 0.f, den = 0.f;
  for (int64_t fa = f_lo; fa <= f_hi; fa += HD_FCH) {
    const int nf = (int)min((int64_t)HD_FCH, f_hi + 1 - fa);
    __syncthreads();                                    // twiddles written / the previous chunk's spectra read
    for (int i = threadIdx.x; i < nf * NB; i += HD_RUN) {
      const int f = i / NB, k = i - f * NB;
      const float* row = hb + (fa + f) * h_ld;
      const float mag = fminf(expf(__ldg(row + k)), 100.f);
      float sn, cs;
      sincosf(__ldg(row + NB + k), &sn, &cs);
      const bool edge = k == 0 || k == N / 2;
      const float sc = edge ? inv_n : inv_n2;
      S[i] = make_float2(mag * cs * sc, edge ? 0.f : -(mag * sn) * sc);
    }
    __syncthreads();
    if (!valid) continue;
    for (int f = 0; f < nf; f++) {
      const int64_t n64 = p - (fa + f) * H;
      if (n64 < 0 || n64 >= N) continue;
      const int n = (int)n64;
      const float2* Sf = S + f * NB;
      float acc = 0.f;
      int idx = 0;
#pragma unroll 4
      for (int k = 0; k < NB; k++) {
        const float2 t = tw[tw_slot(idx)], s = Sf[k];
        acc = fmaf(s.x, t.x, acc);
        acc = fmaf(s.y, t.y, acc);
        idx += n;
        if (idx >= N) idx -= N;
      }
      const float wn = __ldg(window + n);
      num = fmaf(wn, acc, num);
      den += wn;
    }
  }
  if (valid) out[(int64_t)b * out_bs + j] = den > 1e-10f ? num / den : num;
}

constexpr int VOCOS_MEL_PAD = MEL_N / 2;   // stft(center=True): reflect pad n_fft // 2

}  // namespace

extern "C" int32_t b2a_vocos_dwnorm(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C, const float* dw_w,
                                    const float* dw_b, int32_t K, const float* w, const float* b, const float* ada, int64_t ada_bs, float eps,
                                    float* y, int64_t y_bs, int64_t y_ld, void* hi, void* lo, void* stream) {
  B2A_CHECK_ARG(x && B > 0 && L > 0 && C > 0 && x_ld >= C, "bad pointers / shape");
  B2A_CHECK_ARG(y || hi, "no output (y and hi both NULL)");
  B2A_CHECK_ARG(K == 0 || (dw_w && K % 2 == 1 && K <= 15), "depthwise taps must be 0 (no conv) or odd and <= 15");
  B2A_CHECK_ARG(C % 4 == 0 && C <= 1024 && x_ld % 4 == 0 && ((uintptr_t)x & 15) == 0 && (!dw_w || ((uintptr_t)dw_w & 15) == 0) &&
                (!dw_b || ((uintptr_t)dw_b & 15) == 0), "C % 4 == 0, C <= 1024 and 16-byte aligned rows and conv weights");
  B2A_CHECK_ARG(!y || (y_ld >= C && y_ld % 4 == 0 && ((uintptr_t)y & 15) == 0), "fp32 output rows: y_ld >= C, 16-byte aligned");
  B2A_CHECK_ARG(!hi || (C % 64 == 0 && ((uintptr_t)hi & 7) == 0 && (!lo || ((uintptr_t)lo & 7) == 0)), "bf16 planes need C % 64 == 0");
  B2A_CHECK_ARG(!ada || ada_bs >= 2 * C, "AdaLN rows are (scale | shift) [2C]");
  const size_t smem = K ? (size_t)(DN_RT + K - 1) * C * sizeof(float) : 0;
  const dim3 grid(cdiv(L, DN_RT), B);
  cudaStream_t st = (cudaStream_t)stream;
  __nv_bfloat16 *eh = (__nv_bfloat16*)hi, *el = (__nv_bfloat16*)lo;
#define DN_LAUNCH(NV, ADA)                                                                                                      \
  do {                                                                                                                          \
    B2A_SMEM_OPTIN((vocos_dwnorm_kernel<NV, ADA>), 30 * 1024 * 4);                                                              \
    vocos_dwnorm_kernel<NV, ADA><<<grid, DN_THREADS, smem, st>>>(x, x_bs, x_ld, L, C, dw_w, dw_b, K, w, b, ada, ada_bs, eps, y, y_bs, y_ld, eh, el); \
  } while (0)
  if (C <= 512) { if (ada) DN_LAUNCH(4, true); else DN_LAUNCH(4, false); }
  else { if (ada) DN_LAUNCH(8, true); else DN_LAUNCH(8, false); }
#undef DN_LAUNCH
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_vocos_istft_head(const float* h, int64_t h_bs, int64_t h_ld, int32_t B, int32_t T, int32_t n_fft, int32_t hop,
                                        const float* window, float* out, int64_t out_bs, void* stream) {
  if (n_fft <= 0 || n_fft % 2 || n_fft > 2048 || hop <= 0) {
    b2a_set_error("%s: n_fft %d, hop %d (even n_fft <= 2048 and hop > 0 only)", __func__, n_fft, hop);
    return B2A_E_UNSUPPORTED;
  }
  B2A_CHECK_ARG(h && window && out && B > 0 && T >= 1 && h_ld >= n_fft + 2, "bad pointers / shape (row stride >= n_fft + 2)");
  const int64_t nout = (int64_t)(T - 1) * hop;
  B2A_CHECK_ARG(out_bs >= nout, "output rows shorter than (T - 1) * hop");
  if (nout == 0) return B2A_OK;
  const size_t smem = (size_t)(n_fft + (n_fft >> 4) + HD_FCH * (n_fft / 2 + 1)) * sizeof(float2);
  B2A_SMEM_OPTIN(vocos_istft_head_kernel, (2048 + 128 + HD_FCH * 1025) * sizeof(float2));
  const dim3 grid(cdiv(nout, HD_RUN), B);
  vocos_istft_head_kernel<<<grid, HD_RUN, smem, (cudaStream_t)stream>>>(h, h_bs, h_ld, T, n_fft, hop, window, out, out_bs, nout);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_vocos_logmel(const float* x, int64_t x_bs, int32_t B, int64_t n, const float* window, const float* filters,
                                    int32_t n_mels, int64_t frames, float* out, void* stream) {
  B2A_CHECK_ARG(x && window && filters && out && B > 0 && n_mels > 0, "bad pointers/shape");
  B2A_CHECK_ARG(n > VOCOS_MEL_PAD, "reflect padding needs more than 512 samples");
  B2A_CHECK_ARG(frames == n / MEL_HOP, "frames must be n // 256 (the stft's last frame is dropped)");
  const size_t smem = spk_logmel_smem_bytes();
  B2A_SMEM_OPTIN((spk_logmel_kernel<VOCOS_MEL_PAD, false>), smem);
  dim3 grid(cdiv(frames, MEL_FT), B);
  spk_logmel_kernel<VOCOS_MEL_PAD, false><<<grid, 256, smem, (cudaStream_t)stream>>>(x, x_bs, n, window, filters, n_mels, frames, out);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
