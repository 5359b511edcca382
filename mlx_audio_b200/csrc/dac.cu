// Descript Audio Codec quantiser (include/b200audio.h: b2a_dac_rvq_encode, b2a_dac_from_codes): the factorised residual vector
// quantiser of codec/models/descript/nn/quantize.py for any number of code books, levels described by a device-side table.
#include "common.cuh"

namespace {

constexpr int DQ_FRAMES = 8;       // frames per CTA (both kernels)
constexpr int DQ_THREADS = 256;
constexpr int DQ_MAX_CD = 16;

// ---- encode: all levels of the residual quantiser for a tile of frames, the residual never leaving shared memory ---------------
// Per level:  z_e = W_in r + b_in  ->  nearest row of the L2-normalised code book to z_e / |z_e|  ->  r -= W_out e + b_out.
// The arithmetic of every step is that of the kernel the level-by-level host route runs for it, so that both routes produce the
// same bits and therefore the same codes on every frame, near-ties included:
//   in_proj   one fp32 fma chain per (frame, j) over ascending channels, bias added last      (conv1d_dense_kernel, K = 1)
//   search    float64: rows normalised by a lane-strided sum + xor tree, (|xn|^2 - 2 xn.c) + |c|^2 by an fma chain over
//             ascending d, strict < with the lower index on ties                               (rvq_encode_kernel, mode 1)
//   out_proj  fp32 fma chain over ascending j starting from the bias                           (snac_from_codes_kernel)
// With `z == nullptr` the kernel runs quantizer.from_latents instead: z_e is read from `latents`, there is no residual.
__global__ void __launch_bounds__(DQ_THREADS) dac_rvq_encode_kernel(const float* __restrict__ z, int64_t z_ld, int64_t R, int64_t T, int D,
                                                                    const b2a_dac_level_t* __restrict__ levels, int nq, int bins, int lat_ch,
                                                                    int64_t* __restrict__ codes, float* __restrict__ latents,
                                                                    float* __restrict__ zq_out, double* __restrict__ loss_part) {
  extern __shared__ __align__(16) float dq_sm[];
  float* r = dq_sm;                                     // [DQ_FRAMES][D] residual
  float* zq = r + DQ_FRAMES * D;                        // [DQ_FRAMES][D] sum of the levels' projections
  __shared__ float ze[DQ_FRAMES][DQ_MAX_CD];            // un-normalised projection (what `latents` holds)
  __shared__ float es[DQ_FRAMES][DQ_MAX_CD];            // chosen (un-normalised) code-book row
  __shared__ double xn[DQ_FRAMES][DQ_MAX_CD];
  __shared__ double xn2[DQ_FRAMES];
  __shared__ double red_v[DQ_FRAMES][DQ_THREADS / 32];
  __shared__ int red_i[DQ_FRAMES][DQ_THREADS / 32];
  __shared__ int best[DQ_FRAMES];
  __shared__ double sq[DQ_FRAMES * DQ_MAX_CD];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t row0 = (int64_t)blockIdx.x * DQ_FRAMES;
  const bool from_latents = z == nullptr;
  for (int i = tid; i < DQ_FRAMES * D; i += DQ_THREADS) {
    const int f = i / D, c = i - f * D;
    r[i] = (!from_latents && row0 + f < R) ? z[(row0 + f) * z_ld + c] : 0.f;
    zq[i] = 0.f;
  }
  double loss = 0.0;
  __syncthreads();
  for (int q = 0; q < nq; q++) {
    const b2a_dac_level_t lv = levels[q];
    const int cd = lv.cd;
    if (tid < DQ_FRAMES * cd) {
      const int f = tid / cd, j = tid - f * cd;
      const int64_t row = row0 + f;
      const int64_t lat_i = row < R ? ((row / T) * lat_ch + lv.lat_off + j) * T + row % T : 0;
      float v;
      if (from_latents) {
        v = row < R ? latents[lat_i] : 0.f;
      } else {
        const float* rf = r + f * D;
        const float* w = lv.w_in + j;
        float acc = 0.f;
#pragma unroll 8
        for (int c = 0; c < D; c++) acc = fmaf(rf[c], __ldg(w + (int64_t)c * cd), acc);
        v = acc + __ldg(lv.b_in + j);
        if (row < R) latents[lat_i] = v;
      }
      ze[f][j] = v;
    }
    __syncthreads();
    if (warp < DQ_FRAMES) {                             // F.normalize: x / max(|x|, 1e-12)
      double s = 0.0;
      for (int d = lane; d < cd; d += 32) s += (double)ze[warp][d] * (double)ze[warp][d];
      s = warp_sum_d(s);
      const double nrm = fmax(sqrt(s), 1e-12);
      double s2 = 0.0;
      for (int d = lane; d < cd; d += 32) { const double v = (double)ze[warp][d] / nrm; xn[warp][d] = v; s2 += v * v; }
      s2 = warp_sum_d(s2);
      if (lane == 0) xn2[warp] = s2;
    }
    __syncthreads();
    double bv[DQ_FRAMES]; int bi[DQ_FRAMES];
#pragma unroll
    for (int k = 0; k < DQ_FRAMES; k++) { bv[k] = INFINITY; bi[k] = 0x7fffffff; }
    for (int c = tid; c < bins; c += DQ_THREADS) {
      const float* e = lv.cbn + (int64_t)c * cd;
      double dot[DQ_FRAMES];
#pragma unroll
      for (int k = 0; k < DQ_FRAMES; k++) dot[k] = 0.0;
      for (int d = 0; d < cd; d++) {
        const double ev = (double)__ldg(e + d);
#pragma unroll
        for (int k = 0; k < DQ_FRAMES; k++) dot[k] = fma(xn[k][d], ev, dot[k]);
      }
      const double cc = lv.c2[c];
#pragma unroll
      for (int k = 0; k < DQ_FRAMES; k++) {
        const double v = (xn2[k] - 2.0 * dot[k]) + cc;
        if (v < bv[k]) { bv[k] = v; bi[k] = c; }        // c increases per thread: strict < keeps the lowest index
      }
    }
#pragma unroll
    for (int k = 0; k < DQ_FRAMES; k++) {
      double v = bv[k]; int i = bi[k];
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o); const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
      }
      if (lane == 0) { red_v[k][warp] = v; red_i[k][warp] = i; }
    }
    __syncthreads();
    if (tid < DQ_FRAMES) {
      double v = red_v[tid][0]; int i = red_i[tid][0];
      for (int w = 1; w < DQ_THREADS / 32; w++) {
        const double ov = red_v[tid][w]; const int oi = red_i[tid][w];
        if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
      }
      best[tid] = i;
      const int64_t row = row0 + tid;
      if (row < R) codes[((row / T) * nq + q) * T + row % T] = i;
    }
    __syncthreads();
    if (tid < DQ_FRAMES * cd) {
      const int f = tid / cd, j = tid - f * cd;
      const float e = __ldg(lv.cb + (int64_t)best[f] * cd + j);
      es[f][j] = e;
      const double dlt = (double)ze[f][j] - (double)e;
      sq[tid] = row0 + f < R ? dlt * dlt : 0.0;
    }
    __syncthreads();
    if (tid == 0) {                                     // mean over (frames, cd) of (z_e - e)^2, summed over levels, in a fixed order
      double s = 0.0;
      for (int i = 0; i < DQ_FRAMES * cd; i++) s += sq[i];
      loss += s / ((double)R * cd);
    }
    for (int c = tid; c < D; c += DQ_THREADS) {
      const float bl = __ldg(lv.b_out + c);
      float acc[DQ_FRAMES];
#pragma unroll
      for (int f = 0; f < DQ_FRAMES; f++) acc[f] = bl;
      for (int j = 0; j < cd; j++) {
        const float wv = __ldg(lv.w_out + (int64_t)j * D + c);
#pragma unroll
        for (int f = 0; f < DQ_FRAMES; f++) acc[f] = fmaf(wv, es[f][j], acc[f]);
      }
#pragma unroll
      for (int f = 0; f < DQ_FRAMES; f++) { r[f * D + c] -= acc[f]; zq[f * D + c] += acc[f]; }
    }
    __syncthreads();
  }
  for (int i = tid; i < DQ_FRAMES * D; i += DQ_THREADS) {
    const int f = i / D, c = i - f * D;
    if (row0 + f < R) zq_out[(row0 + f) * D + c] = zq[i];
  }
  if (tid == 0) loss_part[blockIdx.x] = loss;
}

// ---- decode: gather, project and sum any number of levels -------------------------------------------------------------------
// CTA = DQ_FRAMES frames of one batch item; the frames' code-book rows of all levels are staged in shared memory (and written out
// as z_p when asked for), then thread = output channel(s) runs the nq x cd fma chain for the 8 frames at once.
__global__ void __launch_bounds__(DQ_THREADS) dac_from_codes_kernel(const int64_t* __restrict__ codes, int64_t codes_bs, int64_t codes_qs, int64_t T,
                                                                    const b2a_dac_level_t* __restrict__ levels, int nq, int bins, int lat_ch,
                                                                    int D, float* __restrict__ out, float* __restrict__ zp, int* __restrict__ err) {
  extern __shared__ __align__(16) float fc_es[];        // [DQ_FRAMES][lat_ch]
  const int64_t t0 = (int64_t)blockIdx.x * DQ_FRAMES; const int b = blockIdx.y;
  for (int idx = threadIdx.x; idx < DQ_FRAMES * nq; idx += DQ_THREADS) {
    const int q = idx % nq, f = idx / nq;
    const int64_t t = t0 + f;
    const b2a_dac_level_t lv = levels[q];
    int64_t code = t < T ? codes[(int64_t)b * codes_bs + (int64_t)q * codes_qs + t] : 0;
    if (code < 0 || code >= bins) { atomicExch(err, 1); code = 0; }
    for (int j = 0; j < lv.cd; j++) {
      const float v = t < T ? __ldg(lv.cb + code * lv.cd + j) : 0.f;
      fc_es[f * lat_ch + lv.lat_off + j] = v;
      if (zp && t < T) zp[((int64_t)b * lat_ch + lv.lat_off + j) * T + t] = v;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < D; c += DQ_THREADS) {
    float acc[DQ_FRAMES];
#pragma unroll
    for (int f = 0; f < DQ_FRAMES; f++) acc[f] = 0.f;
    for (int q = 0; q < nq; q++) {
      const b2a_dac_level_t lv = levels[q];
      const float bl = __ldg(lv.b_out + c);
#pragma unroll
      for (int f = 0; f < DQ_FRAMES; f++) acc[f] += bl;
      for (int j = 0; j < lv.cd; j++) {
        const float wv = __ldg(lv.w_out + (int64_t)j * D + c);
#pragma unroll
        for (int f = 0; f < DQ_FRAMES; f++) acc[f] = fmaf(wv, fc_es[f * lat_ch + lv.lat_off + j], acc[f]);
      }
    }
#pragma unroll
    for (int f = 0; f < DQ_FRAMES; f++) if (t0 + f < T) out[((int64_t)b * T + t0 + f) * D + c] = acc[f];
  }
}

}  // namespace

extern "C" int64_t b2a_dac_rvq_encode_smem_bytes(int32_t dim) { return (int64_t)2 * DQ_FRAMES * dim * sizeof(float); }

extern "C" int32_t b2a_dac_rvq_encode(const float* z, int64_t z_ld, int32_t B, int64_t T, int32_t dim, const b2a_dac_level_t* levels_dev,
                                      int32_t n_levels, int32_t bins, int32_t latent_channels, int64_t* codes, float* latents, float* z_q,
                                      double* loss_part, void* stream) {
  B2A_CHECK_ARG(levels_dev && codes && latents && z_q && loss_part && B > 0 && T > 0 && dim > 0 && n_levels > 0 && bins > 0, "bad pointers / shape");
  B2A_CHECK_ARG(latent_channels >= n_levels && latent_channels <= n_levels * DQ_MAX_CD, "codebook_dim must be in [1, 16] at every level");
  const size_t smem = (size_t)b2a_dac_rvq_encode_smem_bytes(dim);
  B2A_CHECK_ARG(smem <= 160 * 1024, "latent dimension too large for the frame tile");
  B2A_SMEM_OPTIN(dac_rvq_encode_kernel, 160 * 1024);
  const int64_t R = (int64_t)B * T;
  dac_rvq_encode_kernel<<<(unsigned)((R + DQ_FRAMES - 1) / DQ_FRAMES), DQ_THREADS, smem, (cudaStream_t)stream>>>(
      z, z_ld, R, T, dim, levels_dev, n_levels, bins, latent_channels, codes, latents, z_q, loss_part);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_dac_from_codes(const int64_t* codes, int64_t codes_bs, int64_t codes_qs, int32_t B, int32_t n_levels, int64_t T,
                                      const b2a_dac_level_t* levels_dev, int32_t bins, int32_t latent_channels, int32_t dim, float* out,
                                      float* z_p, int32_t* err_flag_dev, void* stream) {
  B2A_CHECK_ARG(codes && levels_dev && out && err_flag_dev && B > 0 && n_levels > 0 && T > 0 && bins > 0 && dim > 0, "bad pointers / shape");
  B2A_CHECK_ARG(latent_channels >= n_levels && latent_channels <= n_levels * DQ_MAX_CD, "codebook_dim must be in [1, 16] at every level");
  const size_t smem = (size_t)DQ_FRAMES * latent_channels * sizeof(float);
  B2A_CHECK_ARG(smem <= 48 * 1024, "too many latent channels");
  dim3 grid(cdiv(T, DQ_FRAMES), B);
  dac_from_codes_kernel<<<grid, DQ_THREADS, smem, (cudaStream_t)stream>>>(codes, codes_bs, codes_qs, T, levels_dev, n_levels, bins, latent_channels,
                                                                          dim, out, z_p, err_flag_dev);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
