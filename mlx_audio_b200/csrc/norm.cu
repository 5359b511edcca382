// Normalisation kernels: InstanceNorm/AdaIN coefficient folding and row LayerNorm / RMSNorm
// (include/b200audio.h: b2a_adain_coeffs, b2a_layernorm).  Statistics are accumulated in float64
// so that var = E[x^2] - mean^2 stays exact for long sequences; the normalisation itself is
// applied for free inside the consuming conv's prologue (conv.cu: Pre).
#include "common.cuh"
#include "tc_common.cuh"
#include "layernorm_row.cuh"

namespace {

constexpr int ROWS_PER_CHUNK = 256;

// grid (ceil(C/32), nchunk, B), block (32, 8): thread column c sums rows ty, ty+8, ...
__global__ void adain_partial_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int L, int C,
                                     double* __restrict__ ws, int nchunk) {
  __shared__ double s1[8][33], s2[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, chunk = blockIdx.y, b = blockIdx.z;
  const int r0 = chunk * ROWS_PER_CHUNK, r1 = min(L, r0 + ROWS_PER_CHUNK);
  double a1 = 0.0, a2 = 0.0;                      // float64 partials: exact var = E[x^2]-mean^2 even when |mean| >> std
  if (c < C) {
    const float* xp = x + (int64_t)b * x_bs + c;
    for (int r = r0 + threadIdx.y; r < r1; r += 8) { double v = (double)__ldg(xp + (int64_t)r * x_ld); a1 += v; a2 = fma(v, v, a2); }
  }
  s1[threadIdx.y][threadIdx.x] = a1; s2[threadIdx.y][threadIdx.x] = a2;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double t1 = 0, t2 = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { t1 += s1[i][threadIdx.x]; t2 += s2[i][threadIdx.x]; }
    double* w = ws + (((int64_t)b * nchunk + chunk) * C + c) * 2;
    w[0] = t1; w[1] = t2;
  }
}

// (sum, sumsq) of every channel ADDED to up to four binned accumulators [B][.][2][B2A_NBIN] (each pointer already offset to its first
// channel, `bs` int64 elements between batches): the statistics format the fused conv's epilogue produces and its prologue consumes.
__global__ void channel_stats_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int L, int C, long long* d0, long long* d1,
                                     long long* d2, long long* d3, int64_t bs0, int64_t bs1, int64_t bs2, int64_t bs3) {
  __shared__ double s1[8][33], s2[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x, chunk = blockIdx.y, b = blockIdx.z;
  const int r0 = chunk * ROWS_PER_CHUNK, r1 = min(L, r0 + ROWS_PER_CHUNK);
  double a1 = 0.0, a2 = 0.0;
  if (c < C) {
    const float* xp = x + (int64_t)b * x_bs + c;
    for (int r = r0 + threadIdx.y; r < r1; r += 8) { double v = (double)__ldg(xp + (int64_t)r * x_ld); a1 += v; a2 = fma(v, v, a2); }
  }
  s1[threadIdx.y][threadIdx.x] = a1; s2[threadIdx.y][threadIdx.x] = a2;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double t1 = 0, t2 = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { t1 += s1[i][threadIdx.x]; t2 += s2[i][threadIdx.x]; }
    long long* ds[4] = {d0, d1, d2, d3};
    const int64_t bss[4] = {bs0, bs1, bs2, bs3};
#pragma unroll
    for (int i = 0; i < 4; i++)
      if (ds[i]) { long long* w = ds[i] + (int64_t)b * bss[i] + (int64_t)c * 2 * B2A_NBIN; repro_add_d(w, t1); repro_add_d(w + B2A_NBIN, t2); }
  }
}

__global__ void coeffs_from_stats_kernel(const long long* __restrict__ st, int L, int C, const float* __restrict__ gb, float eps,
                                         float* __restrict__ scale, float* __restrict__ shift, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i % C;
  const long long* w = st + (int64_t)i * 2 * B2A_NBIN;
  double mean = repro_value(w) / L, var = repro_value(w + B2A_NBIN) / L - mean * mean;
  if (var < 0) var = 0;
  const double rstd = 1.0 / sqrt(var + (double)eps);
  double g = 1.0, be = 0.0;
  if (gb) { g = 1.0 + (double)gb[(int64_t)b * 2 * C + c]; be = (double)gb[(int64_t)b * 2 * C + C + c]; }
  const double sc = g * rstd;
  scale[i] = (float)sc;
  shift[i] = (float)(be - sc * mean);
}

// one warp per (b, c): lanes stride the chunk partials (a serial walk over ~200 chunks per thread cost 20 us per call)
__global__ void adain_final_kernel(const double* __restrict__ ws, int nchunk, int L, int C, const float* __restrict__ gb,
                                   float eps, float* __restrict__ scale, float* __restrict__ shift, int B) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= B * C) return;
  const int b = i / C, c = i % C;
  double t1 = 0, t2 = 0;
  for (int k = lane; k < nchunk; k += 32) { const double* w = ws + (((int64_t)b * nchunk + k) * C + c) * 2; t1 += w[0]; t2 += w[1]; }
  t1 = warp_sum_d(t1); t2 = warp_sum_d(t2);
  if (lane) return;
  double mean = t1 / L, var = t2 / L - mean * mean;
  if (var < 0) var = 0;
  double rstd = 1.0 / sqrt(var + (double)eps);
  double g = 1.0, be = 0.0;
  if (gb) { g = 1.0 + (double)gb[(int64_t)b * 2 * C + c]; be = (double)gb[(int64_t)b * 2 * C + C + c]; }
  double sc = g * rstd;
  scale[i] = (float)sc;
  shift[i] = (float)(be - sc * mean);
}

// one warp per row; C up to a few thousand
__global__ void layernorm_kernel(const float* __restrict__ x, int64_t x_ld, const float* __restrict__ res, int64_t res_ld,
                                 float* __restrict__ y, int64_t y_ld, int64_t rows, int C, const float* __restrict__ w,
                                 const float* __restrict__ bb, const float* __restrict__ ada, float eps, int rms,
                                 int post_act, float post_p0) {
  int64_t row = (int64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xp = x + row * x_ld;
  const float* rp = res ? res + row * res_ld : nullptr;
  float s1 = 0.f;
  for (int c = lane; c < C; c += 32) { float v = xp[c] + (rp ? rp[c] : 0.f); s1 += v; }
  s1 = warp_sum(s1);
  const float mean = rms ? 0.f : s1 / C;
  float s2 = 0.f;
  for (int c = lane; c < C; c += 32) { float v = xp[c] + (rp ? rp[c] : 0.f) - mean; s2 = fmaf(v, v, s2); }
  s2 = warp_sum(s2);
  const float rstd = rsqrtf(s2 / C + eps);
  float* yp = y + row * y_ld;
  for (int c = lane; c < C; c += 32) {
    float v = (xp[c] + (rp ? rp[c] : 0.f) - mean) * rstd;
    if (ada) v = fmaf(1.f + ada[c], v, ada[C + c]);
    else { if (w) v *= w[c]; if (bb) v += bb[c]; }
    if (post_act) v = b2a_act(v, post_act, post_p0, 1.f, 1.f);
    yp[c] = v;
  }
}

// Same operator with the row held in registers: one warp per row, float4 loads all issued before the first use (the three-pass scalar
// version above is three dependent chains of C/32 L2 round trips: 16 us per launch for ALBERT's 130 x 768 rows, 0.5 ms per utterance).
// NV = float4 slots per lane (C <= 128 * NV); rows and all row strides 16-byte aligned.
template <int NV>
__global__ void __launch_bounds__(128) layernorm_vec_kernel(const float* __restrict__ x, int64_t x_ld, const float* __restrict__ res, int64_t res_ld,
                                                            float* __restrict__ y, int64_t y_ld, int64_t rows, int C, const float* __restrict__ w,
                                                            const float* __restrict__ bb, const float* __restrict__ ada, float eps, int rms,
                                                            int post_act, float post_p0, __nv_bfloat16* __restrict__ e_hi,
                                                            __nv_bfloat16* __restrict__ e_lo, int64_t e_ld) {
  pdl_wait();                                              // x / res are the preceding kernel's output
  const int64_t row = (int64_t)blockIdx.x * 4 + threadIdx.x / 32;
  if (row >= rows) return;
  pdl_launch_dependents();
  layernorm_row_vec<NV>(x + row * x_ld, res ? res + row * res_ld : nullptr, y + row * y_ld, C, w, bb, ada, eps, rms, post_act, post_p0,
                        e_hi ? e_hi + row * e_ld : nullptr, e_lo ? e_lo + row * e_ld : nullptr, threadIdx.x & 31);
}

}  // namespace

extern "C" int64_t b2a_adain_ws_bytes(int32_t B, int32_t L, int32_t C) {
  int64_t nchunk = (L + ROWS_PER_CHUNK - 1) / ROWS_PER_CHUNK;
  return (int64_t)B * nchunk * C * 2 * (int64_t)sizeof(double);
}

extern "C" int32_t b2a_adain_coeffs(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C,
                                    const float* gb, float eps, float* scale, float* shift, void* ws, void* stream) {
  B2A_CHECK_ARG(x && scale && shift && ws && B > 0 && L > 0 && C > 0, "bad pointers/shape");
  cudaStream_t st = (cudaStream_t)stream;
  int nchunk = (L + ROWS_PER_CHUNK - 1) / ROWS_PER_CHUNK;
  dim3 grid(cdiv(C, 32), nchunk, B), block(32, 8);
  adain_partial_kernel<<<grid, block, 0, st>>>(x, x_bs, x_ld, L, C, (double*)ws, nchunk);
  adain_final_kernel<<<cdiv((int64_t)B * C, 8), 256, 0, st>>>((const double*)ws, nchunk, L, C, gb, eps, scale, shift, B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_channel_stats(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C, int64_t* const* dst,
                                     const int64_t* dst_bs, int32_t n_dst, void* stream) {
  B2A_CHECK_ARG(x && dst && dst_bs && B > 0 && L > 0 && C > 0 && n_dst >= 1 && n_dst <= 4, "bad pointers/shape (1..4 destinations)");
  long long* d[4] = {nullptr, nullptr, nullptr, nullptr};
  int64_t bs[4] = {0, 0, 0, 0};
  for (int i = 0; i < n_dst; i++) { B2A_CHECK_ARG(dst[i], "null destination"); d[i] = (long long*)dst[i]; bs[i] = dst_bs[i]; }
  dim3 grid(cdiv(C, 32), cdiv(L, ROWS_PER_CHUNK), B), block(32, 8);
  channel_stats_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, L, C, d[0], d[1], d[2], d[3], bs[0], bs[1], bs[2], bs[3]);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_coeffs_from_stats(const int64_t* stats, int32_t B, int32_t L, int32_t C, const float* gb, float eps, float* scale,
                                         float* shift, void* stream) {
  B2A_CHECK_ARG(stats && scale && shift && B > 0 && L > 0 && C > 0, "bad pointers/shape");
  coeffs_from_stats_kernel<<<cdiv((int64_t)B * C, 256), 256, 0, (cudaStream_t)stream>>>((const long long*)stats, L, C, gb, eps, scale, shift, B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_layernorm(const float* x, int64_t x_ld, const float* res, int64_t res_ld, float* y, int64_t y_ld,
                                 int64_t rows, int32_t C, const float* w, const float* b, const float* ada, float eps,
                                 int32_t rms, int32_t post_act, float post_p0, void* emit_hi, void* emit_lo, int64_t emit_ld,
                                 void* stream) {
  B2A_CHECK_ARG(rows >= 0 && C > 0, "bad shape");
  if (rows == 0) return B2A_OK;                            // before the pointer check: an empty torch tensor has a null data pointer
  B2A_CHECK_ARG(x && y, "null pointer");
  const bool al = C % 4 == 0 && C <= 1024 && x_ld % 4 == 0 && y_ld % 4 == 0 && (!res || res_ld % 4 == 0) && ((uintptr_t)x & 15) == 0 &&
                  ((uintptr_t)y & 15) == 0 && (!res || ((uintptr_t)res & 15) == 0);
  B2A_CHECK_ARG(!emit_hi || (al && emit_ld >= C && emit_ld % 4 == 0 && ((uintptr_t)emit_hi & 7) == 0 && ((uintptr_t)emit_lo & 7) == 0),
                "emitted planes need the vectorised kernel (C % 4 == 0, C <= 1024, 16-byte aligned rows), emit_ld >= C, a multiple of 4");
  cudaStream_t st = (cudaStream_t)stream;
  __nv_bfloat16 *eh = (__nv_bfloat16*)emit_hi, *el = (__nv_bfloat16*)emit_lo;
  cudaError_t e = cudaSuccess;
  if (al && C <= 512)
    e = b2a_launch_pdl(layernorm_vec_kernel<4>, dim3(cdiv(rows, 4)), dim3(128), 0, st, x, x_ld, res, res_ld, y, y_ld, rows, (int)C, w, b,
                       ada, eps, (int)rms, (int)post_act, post_p0, eh, el, emit_ld);
  else if (al)
    e = b2a_launch_pdl(layernorm_vec_kernel<8>, dim3(cdiv(rows, 4)), dim3(128), 0, st, x, x_ld, res, res_ld, y, y_ld, rows, (int)C, w, b,
                       ada, eps, (int)rms, (int)post_act, post_p0, eh, el, emit_ld);
  else
    layernorm_kernel<<<cdiv(rows, 8), 256, 0, st>>>(x, x_ld, res, res_ld, y, y_ld, rows, C, w, b, ada, eps, rms, post_act, post_p0);
  if (e != cudaSuccess) { b2a_set_error("b2a_layernorm: %s", cudaGetErrorString(e)); return B2A_E_CUDA; }
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
