// Codec token decode (include/b200audio.h: b2a_rvq_decode, b2a_snac_from_codes): residual-VQ codebook
// gathers summed in registers.  Index handling is exact integer work; out-of-range codes raise a flag.
#include "common.cuh"

namespace {

__global__ void rvq_decode_kernel(const int64_t* __restrict__ codes, int64_t codes_bs, int64_t codes_qs, int nq, int64_t T,
                                  const float* __restrict__ cb, int bins, int dim, float* __restrict__ out, int64_t out_ld,
                                  int* __restrict__ err, int B) {
  // one warp per (b,t): lanes stride the embedding dimension, the nq gathers accumulate in registers
  const int64_t total = (int64_t)B * T;
  const int lane = threadIdx.x & 31;
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < total;
       row += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    int b = (int)(row / T); int64_t t = row % T;
    for (int d0 = 0; d0 < dim; d0 += 128) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      int d = d0 + lane * 4;
      for (int q = 0; q < nq; q++) {
        int64_t code = codes[(int64_t)b * codes_bs + (int64_t)q * codes_qs + t];
        if (code < 0 || code >= bins) { if (lane == 0) atomicExch(err, 1); code = 0; }
        if (d < dim) {
          float4 e = *reinterpret_cast<const float4*>(cb + ((int64_t)q * bins + code) * dim + d);
          acc.x += e.x; acc.y += e.y; acc.z += e.z; acc.w += e.w;
        }
      }
      if (d < dim) *reinterpret_cast<float4*>(out + row * out_ld + d) = acc;
    }
  }
}

// ---- residual-VQ ENCODE: nearest code per row, level after level on the shrinking residual -------------------------------
// CTA = VQ_ROWS rows held in shared memory as float64; thread = code (lanes walk a code's row of the table, which L1 keeps: 128 B lines
// are reused 32 times); scores accumulate in float64 so that the arg-min is decided by the inputs, not by summation order:
//   mode 0 (Mimi, quantization.py:37-45):   score(c) = |e_c|^2 / 2 - x . e_c          on the residual, then x -= e_best
//   mode 1 (SNAC, snac/vq.py:56-73):        score(c) = |xn|^2 - 2 xn . en_c + |en_c|^2 with L2-normalised rows (single level)
// Ties: lowest index (argmin / argmax(-dist) semantics).
constexpr int VQ_ROWS = 4;

__global__ void __launch_bounds__(256) rvq_encode_kernel(const float* __restrict__ x, int64_t x_ld, int64_t R, int D, const float* __restrict__ emb,
                                                         const double* __restrict__ c2, int bins, int nq, int mode, int64_t* __restrict__ codes,
                                                         int64_t codes_rs, int64_t codes_qs) {
  extern __shared__ double vq_sm[];
  double* r = vq_sm;                                   // [VQ_ROWS][D]
  double* red_v = r + VQ_ROWS * D;                     // [VQ_ROWS][8 warps]
  int* red_i = reinterpret_cast<int*>(red_v + VQ_ROWS * 8);
  __shared__ int best[VQ_ROWS];
  __shared__ double xn2[VQ_ROWS];
  const int64_t row0 = (int64_t)blockIdx.x * VQ_ROWS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < VQ_ROWS * D; i += 256) {
    const int rr = i / D, d = i - rr * D;
    r[i] = row0 + rr < R ? (double)x[(row0 + rr) * x_ld + d] : 0.0;
  }
  __syncthreads();
  if (mode == 1) {                                     // normalise the rows (F.normalize: x / max(|x|, 1e-12))
    if (warp < VQ_ROWS) {
      double s = 0.0;
      for (int d = lane; d < D; d += 32) s += r[warp * D + d] * r[warp * D + d];
      s = warp_sum_d(s);
      const double nrm = fmax(sqrt(s), 1e-12);
      for (int d = lane; d < D; d += 32) r[warp * D + d] /= nrm;
      __syncwarp();
      double s2 = 0.0;
      for (int d = lane; d < D; d += 32) s2 += r[warp * D + d] * r[warp * D + d];
      s2 = warp_sum_d(s2);
      if (lane == 0) xn2[warp] = s2;
    }
    __syncthreads();
  }
  for (int q = 0; q < nq; q++) {
    const float* eq = emb + (int64_t)q * bins * D;
    double bv[VQ_ROWS]; int bi[VQ_ROWS];
#pragma unroll
    for (int k = 0; k < VQ_ROWS; k++) { bv[k] = INFINITY; bi[k] = 0x7fffffff; }
    for (int c = tid; c < bins; c += 256) {
      const float* e = eq + (int64_t)c * D;
      double dot[VQ_ROWS];
#pragma unroll
      for (int k = 0; k < VQ_ROWS; k++) dot[k] = 0.0;
      for (int d = 0; d < D; d += 4) {
        const float4 ev = *reinterpret_cast<const float4*>(e + d);
#pragma unroll
        for (int k = 0; k < VQ_ROWS; k++) {
          const double* rk = r + k * D + d;
          dot[k] = fma(rk[0], (double)ev.x, dot[k]); dot[k] = fma(rk[1], (double)ev.y, dot[k]);
          dot[k] = fma(rk[2], (double)ev.z, dot[k]); dot[k] = fma(rk[3], (double)ev.w, dot[k]);
        }
      }
      const double cc = c2[(int64_t)q * bins + c];
#pragma unroll
      for (int k = 0; k < VQ_ROWS; k++) {
        const double v = mode == 0 ? cc - dot[k] : (xn2[k] - 2.0 * dot[k]) + cc;
        if (v < bv[k]) { bv[k] = v; bi[k] = c; }        // c increases per thread: strict < keeps the lowest index
      }
    }
#pragma unroll
    for (int k = 0; k < VQ_ROWS; k++) {
      double v = bv[k]; int i = bi[k];
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o); const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
      }
      if (lane == 0) { red_v[k * 8 + warp] = v; red_i[k * 8 + warp] = i; }
    }
    __syncthreads();
    if (tid < VQ_ROWS) {
      double v = red_v[tid * 8]; int i = red_i[tid * 8];
      for (int w = 1; w < 8; w++) { const double ov = red_v[tid * 8 + w]; const int oi = red_i[tid * 8 + w]; if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; } }
      best[tid] = i;
      if (row0 + tid < R) codes[(row0 + tid) * codes_rs + (int64_t)q * codes_qs] = i;
    }
    __syncthreads();
    if (mode == 0 && q + 1 < nq)
      for (int i = tid; i < VQ_ROWS * D; i += 256) { const int rr = i / D, d = i - rr * D; r[i] -= (double)eq[(int64_t)best[rr] * D + d]; }
    __syncthreads();
  }
}

struct SnacLevels {
  const int64_t* codes[4]; const float* emb[4]; const float* w[4]; const float* bias[4]; int stride[4]; int n;
};

__global__ void snac_from_codes_kernel(SnacLevels lv, int B, int64_t T, int bins, int cd, int dim, float* __restrict__ out,
                                       int* __restrict__ err) {
  // CTA = 8 frames; thread = output channel(s).  e[level][cd] staged in shared memory.
  __shared__ float es[8][4][16];
  const int64_t t0 = (int64_t)blockIdx.x * 8; const int b = blockIdx.y;
  for (int idx = threadIdx.x; idx < 8 * lv.n * cd; idx += blockDim.x) {
    int j = idx % cd, l = (idx / cd) % lv.n, f = idx / (cd * lv.n);
    int64_t t = t0 + f;
    float v = 0.f;
    if (t < T) {
      int64_t Tl = T / lv.stride[l];
      int64_t code = lv.codes[l][(int64_t)b * Tl + t / lv.stride[l]];
      if (code < 0 || code >= bins) { atomicExch(err, 1); code = 0; }
      v = lv.emb[l][code * cd + j];
    }
    es[f][l][j] = v;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < dim; c += blockDim.x) {
    float acc[8];
#pragma unroll
    for (int f = 0; f < 8; f++) acc[f] = 0.f;
    for (int l = 0; l < lv.n; l++) {
      float bl = lv.bias[l] ? lv.bias[l][c] : 0.f;
#pragma unroll
      for (int f = 0; f < 8; f++) acc[f] += bl;
      for (int j = 0; j < cd; j++) {
        float wv = lv.w[l][(int64_t)j * dim + c];
#pragma unroll
        for (int f = 0; f < 8; f++) acc[f] = fmaf(wv, es[f][l][j], acc[f]);
      }
    }
#pragma unroll
    for (int f = 0; f < 8; f++) if (t0 + f < T) out[((int64_t)b * T + t0 + f) * dim + c] = acc[f];
  }
}

}  // namespace

extern "C" int32_t b2a_rvq_decode(const int64_t* codes, int64_t codes_bs, int64_t codes_qs, int32_t B, int32_t nq, int64_t T,
                                  const float* codebooks, int32_t bins, int32_t dim, float* out, int64_t out_ld,
                                  int32_t* err_flag_dev, void* stream) {
  B2A_CHECK_ARG(codes && codebooks && out && err_flag_dev && B > 0 && nq > 0 && T > 0 && bins > 0, "bad pointers/shape");
  B2A_CHECK_ARG(dim > 0 && dim % 4 == 0 && out_ld % 4 == 0, "dim and out_ld must be multiples of 4");
  int64_t rows = (int64_t)B * T;
  int blocks = (int)((rows + 7) / 8); if (blocks > 132 * 16) blocks = 132 * 16;
  rvq_decode_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(codes, codes_bs, codes_qs, nq, T, codebooks, bins, dim, out, out_ld,
                                                               err_flag_dev, B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_snac_from_codes(const int64_t* const* codes_host_ptrs, const int32_t* strides_host, int32_t n_levels,
                                       const float* const* emb_host_ptrs, const float* const* w_host_ptrs,
                                       const float* const* bias_host_ptrs, int32_t B, int64_t T, int32_t bins, int32_t cd,
                                       int32_t dim, float* out, int32_t* err_flag_dev, void* stream) {
  B2A_CHECK_ARG(codes_host_ptrs && strides_host && emb_host_ptrs && w_host_ptrs && bias_host_ptrs && out && err_flag_dev, "null pointer");
  B2A_CHECK_ARG(n_levels > 0 && n_levels <= 4 && cd > 0 && cd <= 16 && B > 0 && T > 0 && dim > 0, "bad shape (levels<=4, codebook_dim<=16)");
  SnacLevels lv; lv.n = n_levels;
  for (int i = 0; i < n_levels; i++) {
    B2A_CHECK_ARG(strides_host[i] > 0 && T % strides_host[i] == 0, "T must be a multiple of every vq stride");
    lv.codes[i] = codes_host_ptrs[i]; lv.emb[i] = emb_host_ptrs[i]; lv.w[i] = w_host_ptrs[i]; lv.bias[i] = bias_host_ptrs[i];
    lv.stride[i] = strides_host[i];
  }
  dim3 grid(cdiv(T, 8), B);
  snac_from_codes_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(lv, B, T, bins, cd, dim, out, err_flag_dev);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_rvq_encode(const float* x, int64_t x_ld, int64_t rows, int32_t dim, const float* codebooks, const double* c2, int32_t bins,
                                  int32_t nq, int32_t mode, int64_t* codes, int64_t codes_row_stride, int64_t codes_level_stride, void* stream) {
  B2A_CHECK_ARG(x && codebooks && c2 && codes && rows > 0 && dim > 0 && dim % 4 == 0 && bins > 0 && nq > 0 && (mode == 0 || (mode == 1 && nq == 1)),
                "bad pointers / shape (dim % 4 == 0; mode 1 = one level)");
  const size_t smem = (size_t)VQ_ROWS * dim * 8 + VQ_ROWS * 8 * 8 + VQ_ROWS * 8 * 4;
  B2A_CHECK_ARG(smem <= 200 * 1024, "dim too large");
  B2A_SMEM_OPTIN(rvq_encode_kernel, 200 * 1024);
  rvq_encode_kernel<<<(unsigned)((rows + VQ_ROWS - 1) / VQ_ROWS), 256, smem, (cudaStream_t)stream>>>(x, x_ld, rows, dim, codebooks, c2, bins, nq, mode, codes,
                                                                                                    codes_row_stride, codes_level_stride);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
