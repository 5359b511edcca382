// BigVGAN anti-aliased SnakeBeta (include/b200audio.h: b2a_aa_snakebeta): Activation1d(SnakeBeta) of
// codec/models/bigvgan/resample.py:157-177 -- 2x up-sampling, SnakeBeta, low-pass + 2x down-sampling -- in one pass over the input.
#include <cuda_bf16.h>
#include "common.cuh"

namespace {

constexpr int AA_TR = 64;            // output rows per CTA
constexpr int AA_THREADS = 256;
constexpr int AA_TAPS = 12;
constexpr int AA_XROWS = AA_TR + 12; // input rows t0-5 .. t0+TR+5 (edge-clamped), one spare
constexpr int AA_VROWS = 2 * AA_TR + 10;

// With ratio 2 and 12 taps the reference's index arithmetic reduces to (n: up-sampled row, t: output row, every index edge-clamped):
//   UpSample1d   (resample.py:122-136)  u[2s]   = 2 sum_q f_up[2q+1] x[s+2-q],   u[2s+1] = 2 sum_q f_up[2q] x[s+3-q],   q = 0..5
//                (edge pad 5, MLX conv_transpose1d scatter y[2i+k] += x[i] f[k] -- no kernel flip --, crop 15 rows each side)
//   SnakeBeta    (activation.py:42-51)  v = u + inv_b sin(a u)^2
//   DownSample1d (resample.py:79-98)    out[t] = sum_k f_down[k] v[clamp(2t + k - 5, 0, 2L-1)],   k = 0..11   (edge pad 5 | 6)
// A CTA = AA_TR output rows x tc channels of one item: it stages input rows t0-5 .. t0+TR+4 (clamped) in shared memory, computes the
// 2 TR + 10 activated up-sampled rows the tile reads once each (clamped positions included), then the outputs.  Every sum runs in
// ascending tap order: the result does not depend on the tiling.
__global__ void __launch_bounds__(AA_THREADS) aa_snakebeta_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int L, int C, int tc,
                                                                  const float* __restrict__ alpha, const float* __restrict__ inv_beta,
                                                                  const float* __restrict__ f_up, const float* __restrict__ f_down,
                                                                  float* __restrict__ y, int64_t y_bs, int64_t y_ld, __nv_bfloat16* __restrict__ hi,
                                                                  __nv_bfloat16* __restrict__ lo, int cols) {
  extern __shared__ __align__(16) float aa_sm[];
  float* xs = aa_sm;                                    // [AA_XROWS][tc]
  float* vs = xs + AA_XROWS * tc;                       // [AA_VROWS][tc]
  __shared__ float fu[AA_TAPS], fd[AA_TAPS], sa[48], sb[48];
  const int tid = threadIdx.x, b = blockIdx.z;
  const int t0 = blockIdx.x * AA_TR, c0 = blockIdx.y * tc;
  if (tid < AA_TAPS) { fu[tid] = 2.f * __ldg(f_up + tid); fd[tid] = __ldg(f_down + tid); }     // x ratio: exact
  if (tid < tc) {
    const int c = c0 + tid;
    sa[tid] = c < C ? __ldg(alpha + c) : 0.f;
    sb[tid] = c < C ? __ldg(inv_beta + c) : 0.f;
  }
  const float* xb = x + (int64_t)b * x_bs;
  for (int i = tid; i < AA_XROWS * tc; i += AA_THREADS) {
    const int j = i / tc, cc = i - j * tc, c = c0 + cc;
    const int r = min(max(t0 - 5 + j, 0), L - 1);
    xs[i] = c < C ? __ldg(xb + (int64_t)r * x_ld + c) : 0.f;
  }
  __syncthreads();
  const int n_last = 2 * L - 1;
  for (int i = tid; i < AA_VROWS * tc; i += AA_THREADS) {
    const int m = i / tc, cc = i - m * tc;
    const int n = min(max(2 * t0 - 5 + m, 0), n_last);
    const int s = n >> 1, odd = n & 1;
    const int j0 = s - t0 + 7 + odd;                    // local row of x[s + 2 + odd]
    float acc = 0.f;
#pragma unroll
    for (int q = 0; q < 6; q++) acc = fmaf(fu[2 * q + 1 - odd], xs[(j0 - q) * tc + cc], acc);
    const float sn = b2a_sin(sa[cc] * acc);
    vs[i] = fmaf(sb[cc], sn * sn, acc);
  }
  __syncthreads();
  for (int i = tid; i < AA_TR * tc; i += AA_THREADS) {
    const int r = i / tc, cc = i - r * tc, c = c0 + cc, t = t0 + r;
    if (t >= L || c >= cols) continue;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < AA_TAPS; k++) acc = fmaf(fd[k], vs[(2 * r + k) * tc + cc], acc);
    if (c >= C) acc = 0.f;                              // pad channels of the bf16 planes
    if (y) {
      y[(int64_t)b * y_bs + (int64_t)t * y_ld + c] = acc;
    } else {
      const int64_t o = ((int64_t)b * L + t) * cols + c;
      const __nv_bfloat16 h = __float2bfloat16_rn(acc);
      hi[o] = h;
      if (lo) lo[o] = __float2bfloat16_rn(acc - __bfloat162float(h));
    }
  }
}

}  // namespace

extern "C" int32_t b2a_aa_snakebeta(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C, const float* alpha,
                                    const float* inv_beta, const float* f_up, const float* f_down, int32_t ratio, int32_t taps, float* y,
                                    int64_t y_bs, int64_t y_ld, void* hi, void* lo, int32_t cpad, void* stream) {
  if (ratio != 2 || taps != AA_TAPS) {
    b2a_set_error("%s: ratio %d with %d taps (only ratio 2, 12 taps)", __func__, ratio, taps);
    return B2A_E_UNSUPPORTED;
  }
  B2A_CHECK_ARG(x && alpha && inv_beta && f_up && f_down && B > 0 && L > 0 && C > 0 && x_ld >= C, "bad pointers / shape");
  B2A_CHECK_ARG((y != nullptr) != (hi != nullptr), "exactly one of y (fp32) and hi (bf16 planes)");
  B2A_CHECK_ARG(y ? y_ld >= C : cpad >= C, "output row narrower than C");
  const int tc = C <= 48 ? C : 32;
  const int cols = y ? C : cpad;
  const size_t smem = (size_t)(AA_XROWS + AA_VROWS) * tc * sizeof(float);
  dim3 grid(cdiv(L, AA_TR), cdiv(cols, tc), B);
  aa_snakebeta_kernel<<<grid, AA_THREADS, smem, (cudaStream_t)stream>>>(x, x_bs, x_ld, L, C, tc, alpha, inv_beta, f_up, f_down, y, y_bs, y_ld,
                                                                      (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, cols);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
