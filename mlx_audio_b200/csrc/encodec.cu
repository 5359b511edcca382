// EnCodec (include/b200audio.h: b2a_encodec_*; reference codec/models/encodec/encodec.py).
//
// b2a_encodec_lstm: the unidirectional 2-layer LSTM of EncodecLSTM, one layer per launch, over a precomputed input projection
// xproj [R, T, 4H] (gates i, f, g, o; bias included).  The recurrent weight W_h [4H, H] is fp32, 4 MiB at H = 512: one thread-block
// CLUSTER of H / 32 CTAs (16 at H = 512, a non-portable size) holds it on chip -- each CTA owns 32 units, i.e. 128 gate rows x H columns,
// half of them in registers (H / 4 floats per thread, as lstm.cu) and half in shared memory (128 KiB at H = 512).  One cluster advances
// RB rows per step, so the weights are read once per step for all its rows; more rows take more clusters, which are independent.
//
// The step scheme is lstm.cu's, generalised to H / 16 columns per lane: lane (grp, half, k) = (lane >> 4, lane >> 3 & 1, lane & 7) of
// warp w holds 8 gate rows (i, f, g, o of the 2 units of row group grp) over the NC = H / 16 columns {half * H / 2 + 8 i + k}; a fixed-
// order reduce-scatter over lane bits 0-2 and an xor-8 shuffle sums a row, so a row's result does not depend on RB or on R.  h lives in
// slot order (slot (half * 8 + k) * NC + i holds column half * H / 2 + 8 i + k) with the float4 index swizzled per lane group; warp w of
// CTA rank owns slots rank * 32 + 4 w + 0..3 and pushes them to every CTA of the cluster as one st.async ... complete_tx per row.
// Every wait is bounded (TIMEOUT_NS on %globaltimer): on expiry the CTA sets the error word and stops waiting, then runs to its end.
//
// b2a_encodec_pad: the input side of an EncodecConv1d (asymmetric reflect / zero padding) with an optional per-(row, channel) affine
// (GroupNorm(1, C) applied from b2a_encodec_gn_coeffs) and ELU in front, and an optional residual add; fp32 rows out.
// b2a_encodec_gn_coeffs: GroupNorm(1, C) statistics in float64 in a fixed order, folded with the affine into scale / shift [B, C].
// b2a_encodec_normalize: Encodec._encode_frame's RMS normalisation of a chunk.  b2a_encodec_ola: Encodec._linear_overlap_add.
#include "common.cuh"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace {

constexpr long long TIMEOUT_NS = 10000000000LL;    // 10 s without progress
constexpr int UPC = 32;                            // units per CTA (8 warps x 4)

__device__ __forceinline__ long long globaltimer() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
  uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r;
}
__device__ __forceinline__ void st_async_v4(uint32_t raddr, float4 v, uint32_t rbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
               ::"r"(raddr), "r"(__float_as_uint(v.x)), "r"(__float_as_uint(v.y)), "r"(__float_as_uint(v.z)), "r"(__float_as_uint(v.w)),
                 "r"(rbar) : "memory");
}
__device__ __forceinline__ bool bar_try_cluster(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// true once the phase completed; false (error word set) after TIMEOUT_NS, or soon after another CTA has set the error word
__device__ bool bar_wait_bounded(uint32_t bar, uint32_t parity, unsigned* err) {
  long long t0 = 0;
  for (int it = 0;; it++) {
    if (bar_try_cluster(bar, parity)) return true;
    if ((it & 63) == 63) {
      if (*(volatile unsigned*)err) return false;
      const long long now = globaltimer();
      if (!t0) t0 = now;
      else if (now - t0 > TIMEOUT_NS) { atomicExch(err, 1u); return false; }
    }
  }
}

template <int H>
struct LstmGeom {
  static constexpr int NCTA = H / UPC;             // CTAs per cluster
  static constexpr int NC = H / 16;                // columns per lane
  static constexpr int NR = NC / 2;                // of which in registers
  static constexpr int Q = NC / 4;                 // float4s per lane group in h
  __device__ static int slot_column(int p) { const int i = p % NC, hk = p / NC; return (hk >> 3) * (H / 2) + 8 * i + (hk & 7); }
  __device__ static int swz(int q) { return q ^ ((q / Q) & (Q - 1)); }         // float4 index -> stored float4 index
};

template <int H>
size_t lstm_smem_bytes(int RB) { return (size_t)8 * 32 * 8 * (H / 32) * 4 + (size_t)2 * RB * H * 4 + 16; }

template <int H, int RB>
__global__ void __launch_bounds__(256, 1)
encodec_lstm_kernel(const float* __restrict__ xproj, const float* __restrict__ wh, const float* __restrict__ skip, float* __restrict__ out,
                    int R, int T, unsigned* err) {
  using G = LstmGeom<H>;
  constexpr int NC = G::NC, NR = G::NR, NCTA = G::NCTA;
  extern __shared__ __align__(16) float smem[];
  float4* wsm = reinterpret_cast<float4*>(smem);                           // [warp][NR/4][row 8][lane 32] float4
  float* hbuf = smem + 8 * 32 * 8 * NR;                                     // [2][RB][H] in swizzled slot order
  uint64_t* hbar = reinterpret_cast<uint64_t*>(hbuf + 2 * RB * H);         // hbar[i]: "hbuf[i] holds the complete h of a step"
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int row0 = (blockIdx.x / NCTA) * RB;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int k = lane & 7, half = (lane >> 3) & 1, grp = lane >> 4;
  const int p0 = rank * UPC + warp * 4;
  const int hk = half * 8 + k;
  const int gate = ((lane >> 1) & 1) * 2 + ((lane >> 2) & 1);
  const int unit = G::slot_column(p0 + grp * 2 + (lane & 1));

  float w[8][NR];                                                           // row u*4 + g: gate g of unit (grp, u), columns i < NR
#pragma unroll
  for (int u = 0; u < 2; u++) {
    const int ju = G::slot_column(p0 + grp * 2 + u);
#pragma unroll
    for (int g = 0; g < 4; g++) {
      const float* wp = wh + ((int64_t)g * H + ju) * H + half * (H / 2) + k;
#pragma unroll
      for (int i = 0; i < NR; i++) w[u * 4 + g][i] = __ldg(wp + 8 * i);
      wp += 8 * NR;                                                         // columns i >= NR: shared memory
      for (int m = 0; m < NR / 4; m++)
        wsm[((warp * (NR / 4) + m) * 8 + u * 4 + g) * 32 + lane] =
            make_float4(__ldg(wp + 8 * (4 * m)), __ldg(wp + 8 * (4 * m + 1)), __ldg(wp + 8 * (4 * m + 2)), __ldg(wp + 8 * (4 * m + 3)));
    }
  }
  for (int i = tid; i < 2 * RB * H; i += 256) hbuf[i] = 0.f;               // step 0 reads h = 0
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&hbar[0])) : "memory");
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&hbar[1])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  float c[RB], xp_cur[RB];
  const float* xp_base[RB];
  bool live[RB];
#pragma unroll
  for (int r = 0; r < RB; r++) {
    live[r] = row0 + r < R;
    c[r] = 0.f;
    xp_base[r] = xproj + (int64_t)(live[r] ? row0 + r : 0) * T * 4 * H + gate * H + unit;
    xp_cur[r] = live[r] ? __ldg(xp_base[r]) : 0.f;
  }
  uint32_t rh = 0, rb = 0;                                                  // lane q < NCTA pushes to CTA q: its hbuf / hbar
  if (lane < NCTA) { rh = mapa(smem_addr(hbuf), lane); rb = mapa(smem_addr(&hbar[0]), lane); }
  const uint32_t push_off = (uint32_t)G::swz(p0 / 4) * 16;
  bool ok = true;
  cluster.sync();                                                           // zeros, weights + barrier inits visible cluster-wide

  // As in lstm.cu: h is double-buffered, no warp can run more than one step ahead of another in the cluster, complete_tx may reach a
  // barrier before its arm, the last step pushes nothing, and cluster.sync() before exit keeps every CTA alive for remote stores.
  for (int t = 0; t < T; t++) {
    const int cur = t & 1, nxt = cur ^ 1;
    if (tid == 0 && t + 1 < T)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(&hbar[nxt])), "r"(RB * H * 4) : "memory");
    float xp_next[RB];
#pragma unroll
    for (int r = 0; r < RB; r++) xp_next[r] = (t + 1 < T && live[r]) ? __ldg(xp_base[r] + (int64_t)(t + 1) * 4 * H) : 0.f;
    if (t > 0 && ok) ok = bar_wait_bounded(smem_addr(&hbar[cur]), ((t - 1) >> 1) & 1, err);
    float s[RB][8];
#pragma unroll
    for (int r = 0; r < RB; r++)
#pragma unroll
      for (int j = 0; j < 8; j++) s[r][j] = 0.f;
    const float* hb = hbuf + cur * RB * H;
#pragma unroll
    for (int m = 0; m < NC / 4; m++) {
      float4 hv[RB];
#pragma unroll
      for (int r = 0; r < RB; r++) hv[r] = reinterpret_cast<const float4*>(hb + r * H)[G::swz(hk * G::Q + m)];
      if (m < NR / 4) {
#pragma unroll
        for (int j = 0; j < 8; j++)
#pragma unroll
          for (int r = 0; r < RB; r++) {
            s[r][j] = fmaf(w[j][4 * m], hv[r].x, s[r][j]);
            s[r][j] = fmaf(w[j][4 * m + 1], hv[r].y, s[r][j]);
            s[r][j] = fmaf(w[j][4 * m + 2], hv[r].z, s[r][j]);
            s[r][j] = fmaf(w[j][4 * m + 3], hv[r].w, s[r][j]);
          }
      } else {
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float4 wv = wsm[((warp * (NR / 4) + (m - NR / 4)) * 8 + j) * 32 + lane];
#pragma unroll
          for (int r = 0; r < RB; r++) {
            s[r][j] = fmaf(wv.x, hv[r].x, s[r][j]);
            s[r][j] = fmaf(wv.y, hv[r].y, s[r][j]);
            s[r][j] = fmaf(wv.z, hv[r].z, s[r][j]);
            s[r][j] = fmaf(wv.w, hv[r].w, s[r][j]);
          }
        }
      }
    }
    const bool b0 = lane & 1, b1 = lane & 2, b2 = lane & 4;
#pragma unroll
    for (int r = 0; r < RB; r++) {
      float s4[4], s2[2];
#pragma unroll
      for (int j = 0; j < 4; j++) s4[j] = (b0 ? s[r][4 + j] : s[r][j]) + __shfl_xor_sync(0xffffffffu, b0 ? s[r][j] : s[r][4 + j], 1);
#pragma unroll
      for (int j = 0; j < 2; j++) s2[j] = (b1 ? s4[2 + j] : s4[j]) + __shfl_xor_sync(0xffffffffu, b1 ? s4[j] : s4[2 + j], 2);
      const float sh = (b2 ? s2[1] : s2[0]) + __shfl_xor_sync(0xffffffffu, b2 ? s2[0] : s2[1], 4);
      const float v = (sh + __shfl_xor_sync(0xffffffffu, sh, 8)) + xp_cur[r];
      const float a = gate == 2 ? 1.f - __fdividef(2.f, 1.f + __expf(2.f * v)) : __fdividef(1.f, 1.f + __expf(-v));
      const int src = (lane & 0x19);
      const float gi = __shfl_sync(0xffffffffu, a, src), gf = __shfl_sync(0xffffffffu, a, src + 4);
      const float gg = __shfl_sync(0xffffffffu, a, src + 2), go = __shfl_sync(0xffffffffu, a, src + 6);
      c[r] = fmaf(gf, c[r], gi * gg);
      const float hval = go * (1.f - __fdividef(2.f, 1.f + __expf(2.f * c[r])));
      if ((lane & 0xe) == 0 && live[r]) {
        const int64_t o = ((int64_t)(row0 + r) * T + t) * H + unit;
        out[o] = skip ? hval + skip[o] : hval;
      }
      const float4 h4 = make_float4(__shfl_sync(0xffffffffu, hval, 0), __shfl_sync(0xffffffffu, hval, 1),
                                    __shfl_sync(0xffffffffu, hval, 16), __shfl_sync(0xffffffffu, hval, 17));
      if (lane < NCTA && t + 1 < T)
        st_async_v4(rh + (uint32_t)((nxt * RB + r) * H * 4) + push_off, h4, rb + (uint32_t)(nxt * 8));
      xp_cur[r] = xp_next[r];
    }
  }
  cluster.sync();
}

template <int H, int RB>
int32_t launch_lstm(const float* xproj, const float* wh, const float* skip, float* out, int R, int T, unsigned* err, cudaStream_t st) {
  auto kern = encodec_lstm_kernel<H, RB>;
  const size_t smem = lstm_smem_bytes<H>(RB);
  constexpr int NCTA = LstmGeom<H>::NCTA;
  cudaError_t e = b2a_smem_optin((const void*)kern, (int)smem);
  if (e == cudaSuccess && NCTA > 8) e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  if (e != cudaSuccess) { b2a_set_error("b2a_encodec_lstm: %s", cudaGetErrorString(e)); return B2A_E_CUDA; }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(NCTA * cdiv(R, RB)); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = NCTA; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  int n_clusters = 0;
  e = cudaOccupancyMaxActiveClusters(&n_clusters, kern, &cfg);
  if (e != cudaSuccess) { b2a_set_error("b2a_encodec_lstm: %s", cudaGetErrorString(e)); return B2A_E_CUDA; }
  if (n_clusters < 1) {
    b2a_set_error("b2a_encodec_lstm: a cluster of %d CTAs with %zu bytes of shared memory each cannot be scheduled on this device", NCTA, smem);
    return B2A_E_UNSUPPORTED;
  }
  e = cudaLaunchKernelEx(&cfg, kern, xproj, wh, skip, out, R, T, err);
  if (e != cudaSuccess) { b2a_set_error("b2a_encodec_lstm: %s", cudaGetErrorString(e)); return B2A_E_CUDA; }
  return B2A_OK;
}

template <int H>
int32_t lstm_rows(const float* xproj, const float* wh, const float* skip, float* out, int R, int T, unsigned* err, cudaStream_t st) {
  return R == 1 ? launch_lstm<H, 1>(xproj, wh, skip, out, R, T, err, st) : launch_lstm<H, 4>(xproj, wh, skip, out, R, T, err, st);
}

// ---------------------------------------------------------------------------------------------------------------- conv input side
__global__ void encodec_pad_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int B, int T, int C, int pl, int pr, int reflect,
                                   const float* __restrict__ scale, const float* __restrict__ shift, int elu, const float* __restrict__ res,
                                   int64_t r_bs, int64_t r_ld, float* __restrict__ y, int64_t y_bs, int64_t y_ld) {
  const int To = T + pl + pr;
  const int64_t n = (int64_t)B * To * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t bt = i / C;
    const int t = (int)(bt % To), b = (int)(bt / To);
    int ts = t - pl;
    float v = 0.f;
    const bool inside = ts >= 0 && ts < T;
    if (inside || reflect) {
      if (ts < 0) ts = -ts;
      else if (ts >= T) ts = 2 * (T - 1) - ts;
      v = x[b * x_bs + ts * x_ld + c];
      if (scale) v = fmaf(v, scale[(int64_t)b * C + c], shift[(int64_t)b * C + c]);
      if (elu) v = v > 0.f ? v : expm1f(v);
    }
    if (res) v += res[b * r_bs + t * r_ld + c];
    y[b * y_bs + t * y_ld + c] = v;
  }
}

constexpr int GN_BLOCKS = 64;     // partial sums per row: fixed, so a row's statistics do not depend on B

__global__ void encodec_gn_partials_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int T, int C, double* __restrict__ part) {
  const int b = blockIdx.y;
  const int64_t n = (int64_t)T * C;
  double s = 0.0, s2 = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)GN_BLOCKS * blockDim.x) {
    const double v = x[b * x_bs + (i / C) * x_ld + (i % C)];
    s += v;
    s2 += v * v;
  }
  s = warp_sum_d(s);
  s2 = warp_sum_d(s2);
  __shared__ double red[2][8];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][w] = s; red[1][w] = s2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, a2 = 0.0;
    for (int j = 0; j < 8; j++) { a += red[0][j]; a2 += red[1][j]; }
    part[((int64_t)b * GN_BLOCKS + blockIdx.x) * 2] = a;
    part[((int64_t)b * GN_BLOCKS + blockIdx.x) * 2 + 1] = a2;
  }
}

__global__ void encodec_gn_coeffs_kernel(const double* __restrict__ part, int T, int C, const float* __restrict__ gamma,
                                         const float* __restrict__ beta, float eps, float* __restrict__ scale, float* __restrict__ shift) {
  const int b = blockIdx.x;
  __shared__ float mr[2];
  if (threadIdx.x == 0) {
    double a = 0.0, a2 = 0.0;
    for (int j = 0; j < GN_BLOCKS; j++) { a += part[((int64_t)b * GN_BLOCKS + j) * 2]; a2 += part[((int64_t)b * GN_BLOCKS + j) * 2 + 1]; }
    const double n = (double)T * C, mean = a / n, var = fmax(a2 / n - mean * mean, 0.0);
    mr[0] = (float)mean;
    mr[1] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float g = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
    const float sc = mr[1] * g;
    scale[(int64_t)b * C + c] = sc;
    shift[(int64_t)b * C + c] = be - mr[0] * sc;
  }
}

// ---------------------------------------------------------------------------------------------------------------- chunk scaling / OLA
__global__ void encodec_normalize_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int L, int C, const uint8_t* __restrict__ mask,
                                         int64_t m_bs, float* __restrict__ y, float* __restrict__ scale) {
  const int r = blockIdx.x;
  double s = 0.0;
  for (int t = threadIdx.x; t < L; t += blockDim.x) {
    const float m = (!mask || mask[r * m_bs + t]) ? 1.f : 0.f;
    float mono = 0.f;
    for (int c = 0; c < C; c++) mono += x[r * x_bs + (int64_t)t * x_ld + c] * m;
    mono /= (float)C;
    s += (double)mono * mono;
  }
  s = warp_sum_d(s);
  __shared__ double red[32];
  __shared__ float sc;
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int j = 0; j < (int)(blockDim.x >> 5); j++) a += red[j];
    sc = (float)sqrt(a / L) + 1e-8f;
    scale[r] = sc;
  }
  __syncthreads();
  const float d = sc;
  for (int64_t i = threadIdx.x; i < (int64_t)L * C; i += blockDim.x) {
    const int t = (int)(i / C), c = (int)(i % C);
    const float m = (!mask || mask[r * m_bs + t]) ? 1.f : 0.f;
    y[(int64_t)r * L * C + i] = x[r * x_bs + (int64_t)t * x_ld + c] * m / d;
  }
}

__global__ void encodec_ola_kernel(const float* __restrict__ frames, int N, int B, int L, int C, const float* __restrict__ scale, int stride,
                                   int Tout, float* __restrict__ out) {
  const int64_t n = (int64_t)B * Tout * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t bt = i / C;
    const int t = (int)(bt % Tout), b = (int)(bt / Tout);
    const int k1 = min(N - 1, t / stride);
    const int k0 = t >= L ? (t - L) / stride + 1 : 0;
    float acc = 0.f, ws = 0.f;
    for (int kk = k0; kk <= k1; kk++) {
      const int j = t - kk * stride;
      const float wgt = 0.5f - fabsf((float)(j + 1) / (float)(L + 1) - 0.5f);
      float v = frames[(((int64_t)kk * B + b) * L + j) * C + c];
      if (scale) v *= scale[(int64_t)kk * B + b];
      acc = fmaf(wgt, v, acc);
      ws += wgt;
    }
    out[i] = acc / ws;
  }
}

}  // namespace

extern "C" int32_t b2a_encodec_lstm(const float* xproj, const float* wh, const float* skip, float* out, int32_t R, int32_t T, int32_t H,
                                    uint32_t* err, void* stream) {
  B2A_CHECK_ARG(xproj && wh && out && err && R > 0 && T > 0, "bad pointers/shape");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned* e = reinterpret_cast<unsigned*>(err);
  switch (H) {
    case 512: return lstm_rows<512>(xproj, wh, skip, out, R, T, e, st);
    case 256: return lstm_rows<256>(xproj, wh, skip, out, R, T, e, st);
    case 128: return lstm_rows<128>(xproj, wh, skip, out, R, T, e, st);
    default: b2a_set_error("b2a_encodec_lstm: hidden size %d not supported (128, 256, 512)", H); return B2A_E_UNSUPPORTED;
  }
}

extern "C" int32_t b2a_encodec_pad(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t C, int32_t pad_left,
                                   int32_t pad_right, int32_t reflect, const float* scale, const float* shift, int32_t elu, const float* res,
                                   int64_t res_bs, int64_t res_ld, float* y, int64_t y_bs, int64_t y_ld, void* stream) {
  B2A_CHECK_ARG(x && y && B > 0 && T > 0 && C > 0 && pad_left >= 0 && pad_right >= 0 && (!scale == !shift), "bad pointers/shape");
  B2A_CHECK_ARG(!res || (pad_left == 0 && pad_right == 0), "a residual add takes no padding");
  if (reflect && (pad_left >= T || pad_right >= T)) {
    b2a_set_error("b2a_encodec_pad: reflect padding (%d, %d) needs more than %d frames, got %d", pad_left, pad_right,
                  pad_left > pad_right ? pad_left : pad_right, T);
    return B2A_E_INVALID;
  }
  const int64_t n = (int64_t)B * (T + pad_left + pad_right) * C;
  const int grid = (int)(n / 256 + 1 < 132 * 16 ? n / 256 + 1 : 132 * 16);
  encodec_pad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, B, T, C, pad_left, pad_right, reflect, scale, shift, elu, res,
                                                             res_bs, res_ld, y, y_bs, y_ld);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int64_t b2a_encodec_gn_ws_bytes(int32_t B) { return (int64_t)B * GN_BLOCKS * 2 * sizeof(double); }

extern "C" int32_t b2a_encodec_gn_coeffs(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t C, const float* gamma,
                                         const float* beta, float eps, float* scale, float* shift, void* ws, void* stream) {
  B2A_CHECK_ARG(x && scale && shift && ws && B > 0 && T > 0 && C > 0, "bad pointers/shape");
  double* part = reinterpret_cast<double*>(ws);
  encodec_gn_partials_kernel<<<dim3(GN_BLOCKS, B), 256, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, T, C, part);
  B2A_CHECK_LAUNCH();
  encodec_gn_coeffs_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(part, T, C, gamma, beta, eps, scale, shift);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_encodec_normalize(const float* x, int64_t x_bs, int64_t x_ld, int32_t R, int32_t L, int32_t C, const uint8_t* mask,
                                         int64_t mask_bs, float* y, float* scale, void* stream) {
  B2A_CHECK_ARG(x && y && scale && R > 0 && L > 0 && C > 0, "bad pointers/shape");
  encodec_normalize_kernel<<<R, 1024, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, L, C, mask, mask_bs, y, scale);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_encodec_ola(const float* frames, int32_t N, int32_t B, int32_t L, int32_t C, const float* scale, int32_t stride,
                                   int32_t Tout, float* out, void* stream) {
  B2A_CHECK_ARG(frames && out && N > 0 && B > 0 && L > 0 && C > 0 && stride > 0 && Tout > 0, "bad pointers/shape");
  B2A_CHECK_ARG(Tout <= stride * (N - 1) + L && stride <= L, "Tout beyond the frames, or a gap between frames");
  const int64_t n = (int64_t)B * Tout * C;
  const int grid = (int)(n / 256 + 1 < 132 * 16 ? n / 256 + 1 : 132 * 16);
  encodec_ola_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(frames, N, B, L, C, scale, stride, Tout, out);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
