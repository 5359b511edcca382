// Autoregressive-LM step kernels for the Qwen3-TTS talker / code predictor (include/b200audio.h: b2a_gemv_bf16,
// b2a_qknorm_rope_cache, b2a_attn_decode, b2a_swiglu, b2a_embed_sum, b2a_incr_i32).  A decode step multiplies 1..8 activation
// rows by every weight of the model, so it is HBM-bound on the bf16 weights: the GEMV streams each weight row exactly once
// with 16-byte loads, fuses the RMSNorm that precedes the projection and the SwiGLU / residual that follows it, and all
// position-dependent scalars (KV length, trailing-text index) are read from device memory so one CUDA graph replays
// every frame.
#include "common.cuh"
#include <cuda_bf16.h>

namespace {

constexpr int GV_THREADS = 128;     // 4 warps split K
constexpr int GV_ROWS = 4;          // weight rows per CTA

struct GemvParams {
  const float* x; int64_t x_ld; int M, K;
  const __nv_bfloat16* w; int64_t w_ld; int N;     // N = weight rows
  const float* bias; const float* norm_w; float norm_eps; int mode;
  const float* res; int64_t res_ld; float* y; int64_t y_ld;
  const char* pf; int64_t pf_bytes;                // next kernel's weights: pulled into the 50 MB L2 while this kernel runs
};

__device__ __forceinline__ void bf16x8_to_float(const uint4& u, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; i++) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}

// y[m, n] = epilogue( sum_k W[n,k] * xn[m,k] ),  xn = x (plain) or x * rsqrt(mean(x^2)+eps) * norm_w (RMSNorm prologue).
// mode 1 (SwiGLU): weight rows are interleaved (gate_0, up_0, gate_1, up_1, ...) and y[m, n/2] = silu(gate) * up.
template <int MT>
__global__ void __launch_bounds__(GV_THREADS) gemv_bf16_kernel(const GemvParams p) {
  __shared__ float red[GV_THREADS / 32][MT][GV_ROWS];
  __shared__ float ssq[GV_THREADS / 32][MT];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = blockIdx.x * GV_ROWS;
  if (p.pf) {                                      // one 128-byte line per thread and stride: HBM -> L2 overlaps this kernel and the launch gap
    const int64_t stride = (int64_t)gridDim.x * GV_THREADS * 128;
    for (int64_t off = ((int64_t)blockIdx.x * GV_THREADS + tid) * 128; off < p.pf_bytes; off += stride)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(p.pf + off));
  }
  float acc[MT][GV_ROWS];
  float sq[MT];
#pragma unroll
  for (int m = 0; m < MT; m++) { sq[m] = 0.f;
#pragma unroll
    for (int r = 0; r < GV_ROWS; r++) acc[m][r] = 0.f; }
  const int chunks = p.K >> 3;
  uint4 wv[GV_ROWS];
  auto load_w = [&](int c) {
#pragma unroll
    for (int r = 0; r < GV_ROWS; r++)
      wv[r] = (n0 + r < p.N && c < chunks) ? __ldcs(reinterpret_cast<const uint4*>(p.w + (int64_t)(n0 + r) * p.w_ld + ((int64_t)c << 3))) : make_uint4(0, 0, 0, 0);
  };
  load_w(tid);                                     // weights do not depend on the previous kernel: in flight before the dependency wait
  pdl_launch_dependents();
  pdl_wait();
  for (int c = tid; c < chunks; c += GV_THREADS) {
    const int k = c << 3;
    if (c != tid) load_w(c);
    float g[8];
    if (p.norm_w) {
      float4 g0 = __ldg(reinterpret_cast<const float4*>(p.norm_w + k)), g1 = __ldg(reinterpret_cast<const float4*>(p.norm_w + k + 4));
      g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
    }
    float xv[MT][8];
#pragma unroll
    for (int m = 0; m < MT; m++) {
      if (m < p.M) {
        float4 a = __ldg(reinterpret_cast<const float4*>(p.x + (int64_t)m * p.x_ld + k));
        float4 b = __ldg(reinterpret_cast<const float4*>(p.x + (int64_t)m * p.x_ld + k + 4));
        xv[m][0] = a.x; xv[m][1] = a.y; xv[m][2] = a.z; xv[m][3] = a.w; xv[m][4] = b.x; xv[m][5] = b.y; xv[m][6] = b.z; xv[m][7] = b.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; j++) xv[m][j] = 0.f;
      }
      if (p.norm_w) {
#pragma unroll
        for (int j = 0; j < 8; j++) { sq[m] = fmaf(xv[m][j], xv[m][j], sq[m]); xv[m][j] *= g[j]; }
      }
    }
#pragma unroll
    for (int r = 0; r < GV_ROWS; r++) {
      float wf[8];
      bf16x8_to_float(wv[r], wf);
#pragma unroll
      for (int m = 0; m < MT; m++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[m][r] = fmaf(wf[j], xv[m][j], acc[m][r]);
    }
  }
#pragma unroll
  for (int m = 0; m < MT; m++) {
#pragma unroll
    for (int r = 0; r < GV_ROWS; r++) { float v = warp_sum(acc[m][r]); if (lane == 0) red[warp][m][r] = v; }
    if (p.norm_w) { float v = warp_sum(sq[m]); if (lane == 0) ssq[warp][m] = v; }
  }
  __syncthreads();
  if (tid < MT * GV_ROWS) {
    const int m = tid / GV_ROWS, r = tid % GV_ROWS, n = n0 + r;
    if (m < p.M && n < p.N) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < GV_THREADS / 32; w++) v += red[w][m][r];
      if (p.norm_w) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < GV_THREADS / 32; w++) s += ssq[w][m];
        v *= rsqrtf(s / (float)p.K + p.norm_eps);
      }
      if (p.bias) v += __ldg(p.bias + n);
      red[0][m][r] = v;                                   // own slot: (m, r) is written by this thread only
    }
  }
  __syncthreads();
  if (p.mode == 1) {
    if (tid < MT * (GV_ROWS / 2)) {
      const int m = tid / (GV_ROWS / 2), q = tid % (GV_ROWS / 2), n = n0 + 2 * q;
      if (m < p.M && n + 1 < p.N) {
        float gte = red[0][m][2 * q], up = red[0][m][2 * q + 1];
        float v = gte / (1.f + expf(-gte)) * up;
        const int no = n >> 1;
        if (p.res) v += __ldg(p.res + (int64_t)m * p.res_ld + no);
        p.y[(int64_t)m * p.y_ld + no] = v;
      }
    }
  } else if (tid < MT * GV_ROWS) {
    const int m = tid / GV_ROWS, r = tid % GV_ROWS, n = n0 + r;
    if (m < p.M && n < p.N) {
      float v = red[0][m][r];
      if (p.res) v += __ldg(p.res + (int64_t)m * p.res_ld + n);
      p.y[(int64_t)m * p.y_ld + n] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Wide variant for 3..8 activation rows (batched decode): the x values a lane needs are loaded ONCE per K chunk and reused for
// GW_ROWS = 8 weight rows (the narrow kernel re-loads them for every 4 rows, which makes it LSU-bound at M = 8), each warp owns
// a contiguous quarter of K, partial sums leave the warp through a 62-shuffle reduce-scatter instead of 64 full butterflies.
constexpr int GW_ROWS = 8;

template <int MT>
__global__ void __launch_bounds__(GV_THREADS) gemv_bf16_wide_kernel(const GemvParams p) {
  constexpr int NV = MT * GW_ROWS;                  // partial sums per lane (power of two, >= 32)
  __shared__ float red[GV_THREADS / 32][NV];
  __shared__ float ssq[GV_THREADS / 32][MT];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = blockIdx.x * GW_ROWS;
  if (p.pf) {
    const int64_t stride = (int64_t)gridDim.x * GV_THREADS * 128;
    for (int64_t off = ((int64_t)blockIdx.x * GV_THREADS + tid) * 128; off < p.pf_bytes; off += stride)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(p.pf + off));
  }
  float acc[NV];
#pragma unroll
  for (int i = 0; i < NV; i++) acc[i] = 0.f;
  float sq[MT];
#pragma unroll
  for (int m = 0; m < MT; m++) sq[m] = 0.f;
  const int chunks = p.K >> 3, cw = chunks / (GV_THREADS / 32);          // host guarantees chunks % 4 == 0
  const int c_begin = warp * cw, c_end = c_begin + cw;
  uint4 wv[GW_ROWS];
  auto load_w = [&](int c) {
#pragma unroll
    for (int r = 0; r < GW_ROWS; r++)
      wv[r] = (n0 + r < p.N && c < c_end) ? __ldcs(reinterpret_cast<const uint4*>(p.w + (int64_t)(n0 + r) * p.w_ld + ((int64_t)c << 3))) : make_uint4(0, 0, 0, 0);
  };
  load_w(c_begin + lane);
  pdl_launch_dependents();
  pdl_wait();
  for (int c = c_begin + lane; c < c_end; c += 32) {
    const int k = c << 3;
    if (c != c_begin + lane) load_w(c);
    float g[8];
    if (p.norm_w) {
      float4 g0 = __ldg(reinterpret_cast<const float4*>(p.norm_w + k)), g1 = __ldg(reinterpret_cast<const float4*>(p.norm_w + k + 4));
      g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
    }
    float xv[MT][8];
#pragma unroll
    for (int m = 0; m < MT; m++) {
      if (m < p.M) {
        float4 a = __ldg(reinterpret_cast<const float4*>(p.x + (int64_t)m * p.x_ld + k));
        float4 b = __ldg(reinterpret_cast<const float4*>(p.x + (int64_t)m * p.x_ld + k + 4));
        xv[m][0] = a.x; xv[m][1] = a.y; xv[m][2] = a.z; xv[m][3] = a.w; xv[m][4] = b.x; xv[m][5] = b.y; xv[m][6] = b.z; xv[m][7] = b.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; j++) xv[m][j] = 0.f;
      }
      if (p.norm_w) {
#pragma unroll
        for (int j = 0; j < 8; j++) { sq[m] = fmaf(xv[m][j], xv[m][j], sq[m]); xv[m][j] *= g[j]; }
      }
    }
#pragma unroll
    for (int r = 0; r < GW_ROWS; r++) {
      float wf[8];
      bf16x8_to_float(wv[r], wf);
#pragma unroll
      for (int m = 0; m < MT; m++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[m * GW_ROWS + r] = fmaf(wf[j], xv[m][j], acc[m * GW_ROWS + r]);
    }
  }
  // reduce-scatter across the warp: after the stage with xor-distance s a lane keeps half of its values (upper half iff lane & s)
  int base = 0;
  {
    int n = NV;
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
      const int half = n >> 1;
      const bool up = (lane & s) != 0;
#pragma unroll
      for (int i = 0; i < NV / 2; i++) {
        if (i < half) {
          const float send = up ? acc[i] : acc[i + half];
          const float keep = up ? acc[i + half] : acc[i];
          acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
        }
      }
      if (up) base += half;
      n = half;
    }
  }
  constexpr int PER = NV / 32;                      // values left per lane
#pragma unroll
  for (int i = 0; i < PER; i++) red[warp][base + i] = acc[i];
  if (p.norm_w) {
#pragma unroll
    for (int m = 0; m < MT; m++) { float v = warp_sum(sq[m]); if (lane == 0) ssq[warp][m] = v; }
  }
  __syncthreads();
  if (tid < NV) {
    const int m = tid / GW_ROWS, r = tid % GW_ROWS, n = n0 + r;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < GV_THREADS / 32; w++) v += red[w][tid];
    if (p.norm_w) {
      float sacc = 0.f;
#pragma unroll
      for (int w = 0; w < GV_THREADS / 32; w++) sacc += ssq[w][m];
      v *= rsqrtf(sacc / (float)p.K + p.norm_eps);
    }
    if (p.bias && n < p.N) v += __ldg(p.bias + n);
    red[0][tid] = v;
  }
  __syncthreads();
  if (p.mode == 1) {
    if (tid < MT * (GW_ROWS / 2)) {
      const int m = tid / (GW_ROWS / 2), q = tid % (GW_ROWS / 2), n = n0 + 2 * q;
      if (m < p.M && n + 1 < p.N) {
        const float gte = red[0][m * GW_ROWS + 2 * q], up = red[0][m * GW_ROWS + 2 * q + 1];
        float v = gte / (1.f + expf(-gte)) * up;
        const int no = n >> 1;
        if (p.res) v += __ldg(p.res + (int64_t)m * p.res_ld + no);
        p.y[(int64_t)m * p.y_ld + no] = v;
      }
    }
  } else if (tid < NV) {
    const int m = tid / GW_ROWS, r = tid % GW_ROWS, n = n0 + r;
    if (m < p.M && n < p.N) {
      float v = red[0][tid];
      if (p.res) v += __ldg(p.res + (int64_t)m * p.res_ld + n);
      p.y[(int64_t)m * p.y_ld + n] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Per-head RMSNorm of q and k + (multimodal) rotary embedding + KV-cache append.  One warp per (b, s, head); a lane
// owns elements lane + 32 j, so the rotate_half partner (i, i + D/2) sits in the same lane.
struct QkParams {
  const float* qkv; int64_t qkv_bs, qkv_ss;        // [B,S,(Hq+2Hkv) D]: q heads | k heads | v heads
  int B, S, Hq, Hkv, D;
  const float* qn; const float* kn; float eps;     // per-head RMSNorm weights [D] (NULL = no norm)
  const int* pos3; const int* base_dev; int base_host;
  int sec_h, sec_w; float theta;
  const int* pos_shift;                            // [B] left-padding count: rotary position = max(cache row - pos_shift[b], 0) (qwen3 batches)
  const int* base_rows; const int* slot;           // [B] per-row base (negative row = left padding: no write) and cache batch index
  float* q_out; int64_t qo_bs, qo_ss;              // [B,S,Hq,D]
  float* kc; float* vc; int64_t c_bs, c_ss;        // caches [B,Smax,Hkv,D]
  int smax;
};

template <int D>
__global__ void qknorm_rope_cache_kernel(const QkParams p) {
  constexpr int E = D / 32;
  const int lane = threadIdx.x & 31;
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int HT = p.Hq + 2 * p.Hkv;
  pdl_launch_dependents();
  pdl_wait();
  if (wid >= (int64_t)p.B * p.S * HT) return;
  const int h = (int)(wid % HT);
  const int s = (int)((wid / HT) % p.S), b = (int)(wid / ((int64_t)HT * p.S));
  const int base = p.base_rows ? p.base_rows[b] : (p.base_dev ? *p.base_dev : p.base_host);
  const int cpos = base + s;
  const int cb = p.slot ? p.slot[b] : b;
  const float* src = p.qkv + (int64_t)b * p.qkv_bs + (int64_t)s * p.qkv_ss + (int64_t)h * D;
  float v[E];
#pragma unroll
  for (int j = 0; j < E; j++) v[j] = src[lane + 32 * j];
  if (h >= p.Hq + p.Hkv) {                         // v head: straight into the cache
    if (cpos >= 0 && cpos < p.smax) {
      float* dst = p.vc + (int64_t)cb * p.c_bs + (int64_t)cpos * p.c_ss + (int64_t)(h - p.Hq - p.Hkv) * D;
#pragma unroll
      for (int j = 0; j < E; j++) dst[lane + 32 * j] = v[j];
    }
    return;
  }
  const bool is_q = h < p.Hq;
  const float* nw = is_q ? p.qn : p.kn;
  if (nw) {
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < E; j++) ss = fmaf(v[j], v[j], ss);
    ss = warp_sum(ss);
    const float rinv = rsqrtf(ss / (float)D + p.eps);
#pragma unroll
    for (int j = 0; j < E; j++) v[j] = v[j] * rinv * __ldg(nw + lane + 32 * j);
  }
  // rotary: frequency slot i = (lane + 32 j) mod D/2
  float o[E];
  auto cs_of = [&](int i, float& c, float& sf) {
    int axis = 0;
    if (i % 3 == 1 && i < 3 * p.sec_h) axis = 1; else if (i % 3 == 2 && i < 3 * p.sec_w) axis = 2;
    int pos = p.pos3 ? p.pos3[((int64_t)axis * p.B + b) * p.S + s] : cpos;
    if (!p.pos3 && p.pos_shift) { pos -= p.pos_shift[b]; if (pos < 0) pos = 0; }
    const double inv = exp2(-(double)(2 * i) / (double)D * log2((double)p.theta));
    double sn, cs;
    sincos((double)pos * inv, &sn, &cs);
    c = (float)cs; sf = (float)sn;
  };
  if constexpr (E == 1) {                          // D = 32: the partner (i, i + 16) lives in lane ^ 16
    float c, sf;
    cs_of(lane & 15, c, sf);
    const float other = __shfl_xor_sync(0xffffffffu, v[0], 16);
    o[0] = lane < 16 ? v[0] * c - other * sf : v[0] * c + other * sf;
  } else {
#pragma unroll
    for (int j = 0; j < E / 2; j++) {
      float c, sf;
      cs_of(lane + 32 * j, c, sf);
      const float x1 = v[j], x2 = v[j + E / 2];
      o[j] = x1 * c - x2 * sf;                      // q*cos + rotate_half(q)*sin, first half: -x2
      o[j + E / 2] = x2 * c + x1 * sf;
    }
  }
  if (is_q) {
    float* dst = p.q_out + (int64_t)b * p.qo_bs + (int64_t)s * p.qo_ss + (int64_t)h * D;
#pragma unroll
    for (int j = 0; j < E; j++) dst[lane + 32 * j] = o[j];
  } else if (cpos >= 0 && cpos < p.smax) {
    float* dst = p.kc + (int64_t)cb * p.c_bs + (int64_t)cpos * p.c_ss + (int64_t)(h - p.Hq) * D;
#pragma unroll
    for (int j = 0; j < E; j++) dst[lane + 32 * j] = o[j];
  }
}

// ------------------------------------------------------------------------------------------------
// Attention for decode / short prefill against the KV cache: one CTA per (head, query, batch).
// Phase 1: warps stride over keys, lanes over D (coalesced rows), scores to shared memory.  Phase 2: softmax.
// Phase 3: warps stride over keys again accumulating p * v (lane owns D/32 channels), cross-warp reduce.
struct AdParams {
  const float* q; int64_t q_bs, q_ss;
  const float* kc; const float* vc; int64_t c_bs, c_ss;
  float* o; int64_t o_bs, o_ss;
  int B, S, Hq, Hkv; float scale;
  const int* base_dev; int base_host; const int* kv_start; int max_k;
  const int* base_rows; const int* slot;           // [B] per-row base (base + s < 0: zero output) and cache batch index
};

constexpr int AD_THREADS = 256;

template <int D>
__global__ void __launch_bounds__(AD_THREADS) attn_decode_kernel(const AdParams p) {
  constexpr int E = D / 32, NW = AD_THREADS / 32;
  extern __shared__ __align__(16) float sc[];       // [max_k] scores, then [NW][D] partial outputs
  __shared__ float redm[NW], reds[NW];
  const int h = blockIdx.x, s = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  pdl_launch_dependents();
  pdl_wait();
  const int base = p.base_rows ? p.base_rows[b] : (p.base_dev ? *p.base_dev : p.base_host);
  const int cb = p.slot ? p.slot[b] : b;
  int klen = base + s + 1;
  if (klen > p.max_k) klen = p.max_k;
  const int k0 = p.kv_start ? p.kv_start[b] : 0;
  const int hk = h / (p.Hq / p.Hkv);
  const float* qp = p.q + (int64_t)b * p.q_bs + (int64_t)s * p.q_ss + (int64_t)h * D;
  float qv[E];
#pragma unroll
  for (int j = 0; j < E; j++) qv[j] = qp[lane * E + j] * p.scale;
  const float* kb = p.kc + (int64_t)cb * p.c_bs + (int64_t)hk * D;
  const float* vb = p.vc + (int64_t)cb * p.c_bs + (int64_t)hk * D;
  float mloc = -INFINITY;
  for (int j = k0 + warp; j < klen; j += NW) {
    const float* kr = kb + (int64_t)j * p.c_ss + lane * E;
    float d = 0.f;
    if constexpr (E == 4) { float4 t = *reinterpret_cast<const float4*>(kr); d = qv[0] * t.x + qv[1] * t.y + qv[2] * t.z + qv[3] * t.w; }
    else if constexpr (E == 2) { float2 t = *reinterpret_cast<const float2*>(kr); d = qv[0] * t.x + qv[1] * t.y; }
    else d = qv[0] * kr[0];
    d = warp_sum(d);
    if (lane == 0) sc[j] = d;
    mloc = fmaxf(mloc, d);
  }
  if (lane == 0) redm[warp] = mloc;
  __syncthreads();
  float gm = redm[0];
#pragma unroll
  for (int w = 1; w < NW; w++) gm = fmaxf(gm, redm[w]);
  float sl = 0.f;
  for (int j = k0 + threadIdx.x; j < klen; j += AD_THREADS) { float e = __expf(sc[j] - gm); sc[j] = e; sl += e; }
  sl = warp_sum(sl);
  if (lane == 0) reds[warp] = sl;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < NW; w++) tot += reds[w];
  float acc[E];
#pragma unroll
  for (int j = 0; j < E; j++) acc[j] = 0.f;
  for (int j = k0 + warp; j < klen; j += NW) {
    const float pj = sc[j];
    const float* vr = vb + (int64_t)j * p.c_ss + lane * E;
    if constexpr (E == 4) { float4 t = *reinterpret_cast<const float4*>(vr); acc[0] = fmaf(pj, t.x, acc[0]); acc[1] = fmaf(pj, t.y, acc[1]); acc[2] = fmaf(pj, t.z, acc[2]); acc[3] = fmaf(pj, t.w, acc[3]); }
    else if constexpr (E == 2) { float2 t = *reinterpret_cast<const float2*>(vr); acc[0] = fmaf(pj, t.x, acc[0]); acc[1] = fmaf(pj, t.y, acc[1]); }
    else acc[0] = fmaf(pj, vr[0], acc[0]);
  }
  __syncthreads();                                  // scores no longer needed: reuse the buffer for the partials
  float* part = sc;                                 // [NW][D]  (max_k >= NW*D/... guaranteed by the host: smem >= NW*D floats)
#pragma unroll
  for (int j = 0; j < E; j++) part[warp * D + lane * E + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < D) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < NW; w++) v += part[w * D + threadIdx.x];
    p.o[(int64_t)b * p.o_bs + (int64_t)s * p.o_ss + (int64_t)h * D + threadIdx.x] = tot > 0.f ? v / tot : 0.f;
  }
}

__global__ void swiglu_kernel(const float* x, int64_t x_ld, int64_t rows, int I, int interleaved, float* y, int64_t y_ld) {
  const int64_t total = rows * I;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / I; const int i = (int)(idx % I);
    const float g = interleaved ? x[r * x_ld + 2 * i] : x[r * x_ld + i], u = interleaved ? x[r * x_ld + 2 * i + 1] : x[r * x_ld + I + i];
    y[r * y_ld + i] = g / (1.f + expf(-g)) * u;
  }
}

struct EmbedSumParams {
  const int64_t* codes; int64_t codes_bs; int B, G, dim;
  const float* const* tables; const int* bins;
  const float* text; int64_t text_bs, text_ss; int n_text; const float* pad;
  float* out; int64_t out_bs; int* err;
  int* tidx; const uint8_t* finished;              // per-row trailing index (advanced for unfinished rows), clamp-pad rule
};
__global__ void embed_sum_kernel(const EmbedSumParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= p.dim) return;
  float v = 0.f;
  if (p.tidx) {
    // _next_batch_input_embeds(pad_when_index_clamped=True) (qwen3_tts.py:993-1015): clamp to n_text-1, and a clamped-or-last index
    // reads the pad embedding (the last trailing row is never used in batch mode -- reference behaviour, kept)
    const int idx = p.tidx[b];
    const int cl = idx < p.n_text - 1 ? idx : p.n_text - 1;
    if (cl >= p.n_text - 1) v = p.pad ? p.pad[d] : 0.f;
    else v = p.text[(int64_t)b * p.text_bs + (int64_t)cl * p.text_ss + d];
  } else if (p.pad) v = p.pad[d];
  for (int g = 0; g < p.G; g++) {
    const int64_t c = p.codes[(int64_t)b * p.codes_bs + g];
    if (c < 0 || c >= p.bins[g]) { if (p.err) *p.err = 1; continue; }
    v += p.tables[g][c * p.dim + d];
  }
  p.out[(int64_t)b * p.out_bs + d] = v;
  // one thread per row advances the trailing index after every reader of this CTA has used it (rows span several CTAs: the index
  // is read at the top of each; the increment happens in a separate tiny kernel to stay race-free)
}

__global__ void advance_tidx_kernel(int* tidx, const uint8_t* finished, int B) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B && !(finished && finished[b])) tidx[b] += 1;
}

__global__ void incr_kernel(int* p, int v) { pdl_launch_dependents(); pdl_wait(); *p += v; }

// End of a batch-session frame, one thread per slot.  A slot that is not finished after this frame's sample (EOS sets the flag in
// the sampler; empty slots are kept finished) records its codes at its frame count, advances its cache length and frame count,
// finishes at its frame cap, and loads its next frame's uniforms.  Finished and empty slots are left unchanged.
__global__ void slot_advance_kernel(int* lengths, int* frames, uint8_t* finished, const int* cap, const int64_t* codes, int G,
                                    int64_t* out, int64_t out_bs, const float* u_tab, int64_t u_bs, float* u, int B) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || finished[b]) return;
  const int f = frames[b];
  for (int g = 0; g < G; g++) out[(int64_t)b * out_bs + (int64_t)f * G + g] = codes[(int64_t)b * G + g];
  frames[b] = f + 1;
  lengths[b] += 1;
  if (f + 1 >= cap[b]) { finished[b] = 1; return; }
  for (int g = 0; g < G; g++) u[(int64_t)g * B + b] = u_tab[(int64_t)b * u_bs + (int64_t)(f + 1) * G + g];
}

}  // namespace

extern "C" int32_t b2a_gemv_bf16(const float* x, int64_t x_ld, int32_t M, int32_t K, const void* w_bf16, int64_t w_ld, int32_t N,
                                 const float* bias, const float* norm_w, float norm_eps, int32_t mode, const float* res,
                                 int64_t res_ld, float* y, int64_t y_ld, const void* prefetch, int64_t prefetch_bytes, void* stream) {
  B2A_CHECK_ARG(M >= 1 && M <= 8, "M must be 1..8 (loop larger batches on the host)");
  B2A_CHECK_ARG(K % 8 == 0 && w_ld % 8 == 0 && x_ld % 4 == 0, "K, w_ld must be multiples of 8 and x_ld of 4 (16-byte loads)");
  B2A_CHECK_ARG(((uintptr_t)x & 15) == 0 && ((uintptr_t)w_bf16 & 15) == 0, "x and w must be 16-byte aligned");
  B2A_CHECK_ARG(mode == 0 || (mode == 1 && N % 2 == 0 && bias == nullptr), "mode 1 (SwiGLU) needs interleaved gate/up rows and no bias");
  GemvParams p{x, x_ld, M, K, (const __nv_bfloat16*)w_bf16, w_ld, N, bias, norm_w, norm_eps, mode, res, res_ld, y, y_ld,
               (const char*)prefetch, prefetch ? prefetch_bytes : 0};
  const int grid = (N + GV_ROWS - 1) / GV_ROWS;
  cudaStream_t st = (cudaStream_t)stream;
  const bool wide = M > 2 && (K >> 3) % (GV_THREADS / 32) == 0;
  const int gridw = (N + GW_ROWS - 1) / GW_ROWS;
  if (M == 1) b2a_launch_pdl(gemv_bf16_kernel<1>, dim3(grid), dim3(GV_THREADS), 0, st, p);
  else if (M == 2) b2a_launch_pdl(gemv_bf16_kernel<2>, dim3(grid), dim3(GV_THREADS), 0, st, p);
  else if (wide && M <= 4) b2a_launch_pdl(gemv_bf16_wide_kernel<4>, dim3(gridw), dim3(GV_THREADS), 0, st, p);
  else if (wide) b2a_launch_pdl(gemv_bf16_wide_kernel<8>, dim3(gridw), dim3(GV_THREADS), 0, st, p);
  else if (M <= 4) b2a_launch_pdl(gemv_bf16_kernel<4>, dim3(grid), dim3(GV_THREADS), 0, st, p);
  else b2a_launch_pdl(gemv_bf16_kernel<8>, dim3(grid), dim3(GV_THREADS), 0, st, p);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_qknorm_rope_cache(const float* qkv, int64_t qkv_bs, int64_t qkv_ss, int32_t B, int32_t S, int32_t Hq,
                                         int32_t Hkv, int32_t D, const float* q_norm_w, const float* k_norm_w, float eps,
                                         const int32_t* pos3, const int32_t* base_dev, int32_t base_host, int32_t sec_h,
                                         int32_t sec_w, float theta, float* q_out, int64_t qo_bs, int64_t qo_ss, float* k_cache,
                                         float* v_cache, int64_t c_bs, int64_t c_ss, int32_t smax, const int32_t* pos_shift,
                                         const int32_t* base_rows, const int32_t* slot, void* stream) {
  B2A_CHECK_ARG(D == 32 || D == 64 || D == 128, "head_dim must be 32, 64 or 128");
  B2A_CHECK_ARG(B > 0 && S > 0 && Hq > 0 && Hkv > 0 && Hq % Hkv == 0, "bad shape");
  QkParams p{qkv, qkv_bs, qkv_ss, B, S, Hq, Hkv, D, q_norm_w, k_norm_w, eps, pos3, base_dev, base_host, sec_h, sec_w, theta, pos_shift,
             base_rows, slot, q_out, qo_bs, qo_ss, k_cache, v_cache, c_bs, c_ss, smax};
  const int64_t warps = (int64_t)B * S * (Hq + 2 * Hkv);
  const int grid = (int)((warps * 32 + 255) / 256);
  if (D == 128) b2a_launch_pdl(qknorm_rope_cache_kernel<128>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, p);
  else if (D == 64) b2a_launch_pdl(qknorm_rope_cache_kernel<64>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, p);
  else b2a_launch_pdl(qknorm_rope_cache_kernel<32>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, p);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_attn_decode(const float* q, int64_t q_bs, int64_t q_ss, const float* k_cache, const float* v_cache,
                                   int64_t c_bs, int64_t c_ss, float* out, int64_t o_bs, int64_t o_ss, int32_t B, int32_t S,
                                   int32_t Hq, int32_t Hkv, int32_t D, float scale, const int32_t* base_dev, int32_t base_host,
                                   const int32_t* kv_start, int32_t max_k, const int32_t* base_rows, const int32_t* slot, void* stream) {
  B2A_CHECK_ARG(D == 32 || D == 64 || D == 128, "head_dim must be 32, 64 or 128");
  B2A_CHECK_ARG(B > 0 && S > 0 && Hq % Hkv == 0 && max_k > 0 && max_k <= 48 * 1024, "bad shape (max_k <= 49152)");
  B2A_CHECK_ARG(c_ss % 4 == 0 && c_bs % 4 == 0 && ((uintptr_t)k_cache & 15) == 0 && ((uintptr_t)v_cache & 15) == 0, "cache rows must be 16-byte aligned");
  AdParams p{q, q_bs, q_ss, k_cache, v_cache, c_bs, c_ss, out, o_bs, o_ss, B, S, Hq, Hkv, scale, base_dev, base_host, kv_start, max_k,
              base_rows, slot};
  size_t floats = (size_t)max_k;
  if (floats < (size_t)(AD_THREADS / 32) * D) floats = (size_t)(AD_THREADS / 32) * D;
  const size_t sm = floats * sizeof(float);
  dim3 grid(Hq, S, B);
  const auto kern = D == 128 ? attn_decode_kernel<128> : D == 64 ? attn_decode_kernel<64> : attn_decode_kernel<32>;
  B2A_SMEM_OPTIN(kern, sm);
  b2a_launch_pdl(kern, grid, dim3(AD_THREADS), sm, (cudaStream_t)stream, p);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_swiglu(const float* x, int64_t x_ld, int64_t rows, int32_t I, int32_t interleaved, float* y, int64_t y_ld, void* stream) {
  B2A_CHECK_ARG(rows > 0 && I > 0, "bad shape");
  int64_t total = rows * I;
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 16) blocks = 132 * 16;
  swiglu_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, x_ld, rows, I, interleaved, y, y_ld);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_embed_sum(const int64_t* codes, int64_t codes_bs, int32_t B, int32_t G, int32_t dim,
                                 const float* const* tables_dev, const int32_t* bins_dev, const float* text, int64_t text_bs,
                                 int64_t text_ss, int32_t n_text, const float* pad, float* out, int64_t out_bs,
                                 int32_t* err_flag_dev, int32_t* tidx, const uint8_t* finished, void* stream) {
  B2A_CHECK_ARG(B > 0 && G >= 0 && dim > 0, "bad shape");
  B2A_CHECK_ARG((tidx == nullptr) == (text == nullptr) && (text == nullptr || n_text > 0),
                "trailing text rows and per-row trailing indices go together");
  EmbedSumParams p{codes, codes_bs, B, G, dim, tables_dev, bins_dev, text, text_bs, text_ss, n_text, pad, out, out_bs, err_flag_dev,
                   tidx, finished};
  dim3 grid((dim + 255) / 256, B);
  b2a_launch_pdl(embed_sum_kernel, grid, dim3(256), 0, (cudaStream_t)stream, p);
  if (tidx) b2a_launch_pdl(advance_tidx_kernel, dim3((B + 63) / 64), dim3(64), 0, (cudaStream_t)stream, tidx, finished, (int)B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_slot_advance(int32_t* lengths, int32_t* frames, uint8_t* finished, const int32_t* cap, const int64_t* codes,
                                    int32_t G, int64_t* out, int64_t out_bs, const float* u_tab, int64_t u_bs, float* u, int32_t B,
                                    void* stream) {
  B2A_CHECK_ARG(lengths && frames && finished && cap && codes && out && u_tab && u, "null pointer");
  B2A_CHECK_ARG(B > 0 && G > 0 && out_bs >= G && u_bs >= G, "bad shape");
  b2a_launch_pdl(slot_advance_kernel, dim3((B + 63) / 64), dim3(64), 0, (cudaStream_t)stream, (int*)lengths, (int*)frames, finished,
                 (const int*)cap, codes, (int)G, out, out_bs, u_tab, u_bs, u, (int)B);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_incr_i32(int32_t* p, int32_t v, void* stream) {
  b2a_launch_pdl(incr_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, p, v);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
