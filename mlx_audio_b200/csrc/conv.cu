// 1-D convolution family on channels-last fp32 activations (include/b200audio.h: b2a_conv1d_cl,
// b2a_convtr1d_cl).  CUDA-core path: shared-memory tiled implicit GEMM for dense layers, a
// coalesced gather kernel for depthwise layers.  Every layer fuses its input transform
// (InstanceNorm/AdaIN apply + Snake/LeakyReLU/ELU), bias, activation, LayerScale/noise gain,
// residual add, output scale and accumulation, so each conv reads x once and writes y once.
#include "common.cuh"
#include <cuda_bf16.h>

namespace {

constexpr int BM = 64;          // output positions per CTA
constexpr int DW_TL = 128;      // positions per CTA of the staged depthwise kernels
constexpr int NT = 256;         // threads per CTA

struct Pre {                    // input transform, evaluated while staging x into shared memory
  const float* scale; const float* shift; int act; float p0; const float* a; const float* b; int cin;
  __device__ __forceinline__ float operator()(float v, int bidx, int c) const {
    if (scale) v = fmaf(v, __ldg(scale + (int64_t)bidx * cin + c), __ldg(shift + (int64_t)bidx * cin + c));
    if (act) v = b2a_act(v, act, p0, a ? __ldg(a + c) : 1.f, b ? __ldg(b + c) : 1.f);
    return v;
  }
};

__device__ __forceinline__ void epilogue_store(const b2a_conv1d_t& p, int b, int l, int co, float v) {
  if (p.bias) v += __ldg(p.bias + co);
  if (p.post_act) v = b2a_act(v, p.post_act, p.post_p0, 1.f, 1.f);
  if (p.post_cscale) v *= __ldg(p.post_cscale + (int64_t)b * p.post_cscale_bs + co);
  if (p.res) v += __ldg(p.res + (int64_t)b * p.res_bs + (int64_t)(l / p.res_div) * p.res_ld + co);
  v *= p.out_scale;
  float* yp = p.y + (int64_t)b * p.y_bs + (int64_t)l * p.y_ld + co;
  if (p.accumulate) v += *yp;
  *yp = v;
}

__device__ __forceinline__ Pre make_pre(const b2a_conv1d_t& p) {
  return Pre{p.pre_scale, p.pre_shift, p.pre_act, p.pre_p0, p.pre_a, p.pre_b, p.Cin};
}

// ------------------------------------------------------------------------------------------------
// Dense conv1d: CTA tile = 64 positions x BN channels; K-loop over channel chunks of CI with all
// taps resident: xs[rows][CI+1] holds the transformed input span once (no per-tap re-reads),
// ws[K][CI][BN] the weights.  Thread (tm,tn) owns 4 positions x NJ channels.
template <int BN>
__global__ void __launch_bounds__(NT) conv1d_dense_kernel(const b2a_conv1d_t p, int CI, int rows) {
  constexpr int NJ = BN / 16;
  extern __shared__ __align__(16) float smem[];
  float* xs = smem;                                   // [rows][CI+1]
  float* ws = smem + (((size_t)rows * (CI + 1) + 3) & ~(size_t)3);   // [K][CI][BN], 16-byte aligned for float4 reads
  const int tid = threadIdx.x, tn = tid & 15, tm = tid >> 4;
  const int l0 = blockIdx.x * BM, n0 = blockIdx.y * BN, b = blockIdx.z;
  const Pre pre = make_pre(p);
  const float* xb = p.x + (int64_t)b * p.x_bs;
  const int64_t pos0 = (int64_t)l0 * p.stride - p.pad_left;
  float acc[4][NJ];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < NJ; j++) acc[i][j] = 0.f;

  for (int c0 = 0; c0 < p.Cin; c0 += CI) {
    for (int idx = tid; idx < rows * CI; idx += NT) {
      int ci = idx % CI, r = idx / CI;
      int64_t pos = pos0 + r;
      int c = c0 + ci;
      float v = 0.f;
      if (c < p.Cin) {
        if (pos >= 0 && pos < p.L) v = pre(__ldg(xb + pos * p.x_ld + c), b, c);
        else if (p.pad_mode == 1) { int64_t q = pos < 0 ? 0 : p.L - 1; v = pre(__ldg(xb + q * p.x_ld + c), b, c); }
      }
      xs[r * (CI + 1) + ci] = v;
    }
    for (int idx = tid; idx < p.K * CI * BN; idx += NT) {
      int n = idx % BN, ci = (idx / BN) % CI, k = idx / (BN * CI);
      int c = c0 + ci, co = n0 + n;
      ws[idx] = (c < p.Cin && co < p.Cout) ? __ldg(p.w + ((int64_t)k * p.Cin + c) * p.Cout + co) : 0.f;
    }
    __syncthreads();
    for (int k = 0; k < p.K; k++) {
      const float* xr = xs + (size_t)(tm * 4 * p.stride + k * p.dilation) * (CI + 1);
      const float* wr = ws + (size_t)k * CI * BN + tn * NJ;
#pragma unroll 4
      for (int ci = 0; ci < CI; ci++) {
        float a[4], w[NJ];
#pragma unroll
        for (int i = 0; i < 4; i++) a[i] = xr[(size_t)i * p.stride * (CI + 1) + ci];
        if constexpr (NJ == 4) {
          float4 t = *reinterpret_cast<const float4*>(wr + ci * BN);
          w[0] = t.x; w[1] = t.y; w[2] = t.z; w[3] = t.w;
        } else {
#pragma unroll
          for (int j = 0; j < NJ; j++) w[j] = wr[ci * BN + j];
        }
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < NJ; j++) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    int l = l0 + tm * 4 + i;
    if (l >= p.Lout) continue;
#pragma unroll
    for (int j = 0; j < NJ; j++) {
      int co = n0 + tn * NJ + j;
      if (co < p.Cout) epilogue_store(p, b, l, co, acc[i][j]);
    }
  }
}

// Depthwise conv1d (groups == C): one thread per (l, c); consecutive threads take consecutive
// channels so every tap is a coalesced row segment; taps hit L1/L2 (HBM sees x once).
__global__ void __launch_bounds__(NT) conv1d_dw_kernel(const b2a_conv1d_t p) {
  const Pre pre = make_pre(p);
  const int64_t total = (int64_t)p.B * p.Lout * p.Cout;
  for (int64_t idx = (int64_t)blockIdx.x * NT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * NT) {
    int c = (int)(idx % p.Cout);
    int64_t t = idx / p.Cout;
    int l = (int)(t % p.Lout), b = (int)(t / p.Lout);
    const float* xb = p.x + (int64_t)b * p.x_bs + c;
    float acc = 0.f;
    int64_t pos = (int64_t)l * p.stride - p.pad_left;
    for (int k = 0; k < p.K; k++, pos += p.dilation) {
      float v = 0.f;
      if (pos >= 0 && pos < p.L) v = pre(__ldg(xb + pos * p.x_ld), b, c);
      else if (p.pad_mode == 1) v = pre(__ldg(xb + (pos < 0 ? 0 : (int64_t)p.L - 1) * p.x_ld), b, c);
      acc = fmaf(v, __ldg(p.w + (int64_t)k * p.Cout + c), acc);
    }
    epilogue_store(p, b, l, c, acc);
  }
}

// Vectorised variant (C % 4 == 0, 16-byte aligned rows): a lane owns FOUR consecutive channels, so global loads / stores and the
// per-tap shared-memory reads are 16 bytes wide (4x fewer LSU instructions than the scalar tile; the SNAC decoder's twelve
// depthwise layers were LSU-bound at 22 % of HBM bandwidth).  CTA = DW_TL positions x CW channels (CW = 64 or 128).
template <int KT, int CW, bool SNAKE>     // SNAKE: prologue (and emitted) activation known to be Snake at compile time (no switch, 3x less code)
__global__ void __launch_bounds__(NT) conv1d_dw_tiled4_kernel(const b2a_conv1d_t p, int rows) {
  constexpr int LPR = CW / 4, RPW = 32 / LPR;        // lanes per row, rows per warp-wide access
  extern __shared__ __align__(16) float smem[];      // [rows][CW]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c4 = (lane % LPR) * 4, rsub = lane / LPR;
  const int l0 = blockIdx.x * DW_TL, c0 = blockIdx.y * CW, b = blockIdx.z;
  const int c = c0 + c4;
  const bool cok = c < p.Cout;                       // C % 4 == 0: the whole quad is in or out
  const Pre pre = make_pre(p);
  const int K = KT ? KT : p.K;
  const float* xb = p.x + (int64_t)b * p.x_bs + c;
  const int64_t pos0 = (int64_t)l0 - p.pad_left;
  // per-channel prologue constants in registers (the generic functor re-loads them for every element)
  float pa[4] = {1.f, 1.f, 1.f, 1.f}, pb[4] = {1.f, 1.f, 1.f, 1.f}, ps[4] = {1.f, 1.f, 1.f, 1.f}, ph[4] = {0.f, 0.f, 0.f, 0.f};
  if (cok) {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      if (p.pre_a) pa[q] = __ldg(p.pre_a + c + q);
      if (p.pre_b) pb[q] = __ldg(p.pre_b + c + q);
      if (p.pre_scale) { ps[q] = __ldg(p.pre_scale + (int64_t)b * p.Cin + c + q); ph[q] = __ldg(p.pre_shift + (int64_t)b * p.Cin + c + q); }
    }
  }
  auto tr = [&](float v, int q) -> float {
    if constexpr (SNAKE) { const float sn = b2a_sin(pa[q] * v); return fmaf(pb[q], sn * sn, v); }
    else {
      if (p.pre_scale) v = fmaf(v, ps[q], ph[q]);
      if (p.pre_act) v = b2a_act(v, p.pre_act, p.pre_p0, pa[q], pb[q]);
      return v;
    }
  };
  // staging: FOUR rows per thread and iteration, all four 16-byte loads in flight before the first is used (one load per
  // iteration left the CTA waiting a full memory latency twelve times per tile)
  constexpr int RSTEP = (NT / 32) * RPW;
  for (int r0 = warp * RPW + rsub; r0 < rows; r0 += 4 * RSTEP) {
    float4 t[4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int r = r0 + u * RSTEP;
      int64_t pos = pos0 + r;
      if (pos < 0 || pos >= p.L) pos = p.pad_mode == 1 ? (pos < 0 ? 0 : (int64_t)p.L - 1) : -1;
      ok[u] = cok && r < rows && pos >= 0;
      t[u] = ok[u] ? __ldg(reinterpret_cast<const float4*>(xb + pos * p.x_ld)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int r = r0 + u * RSTEP;
      if (r < rows) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok[u]) { v.x = tr(t[u].x, 0); v.y = tr(t[u].y, 1); v.z = tr(t[u].z, 2); v.w = tr(t[u].w, 3); }
        *reinterpret_cast<float4*>(smem + (size_t)r * CW + c4) = v;
      }
    }
  }
  float4 w[KT ? KT : 16];
#pragma unroll
  for (int k = 0; k < (KT ? KT : 16); k++)
    w[k] = (cok && k < K) ? __ldg(reinterpret_cast<const float4*>(p.w + (int64_t)k * p.Cout + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (cok && p.bias) bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + c));
  __syncthreads();
  if (!cok) return;
  const int d = p.dilation;
  float ea[4] = {1.f, 1.f, 1.f, 1.f}, eb[4] = {1.f, 1.f, 1.f, 1.f};
  if (p.emit_hi) {
#pragma unroll
    for (int q = 0; q < 4; q++) { if (p.emit_a) ea[q] = __ldg(p.emit_a + c + q); if (p.emit_b) eb[q] = __ldg(p.emit_b + c + q); }
  }
  const bool fast = !p.res && !p.post_cscale && !p.accumulate && !p.post_act && (p.y_ld % 4 == 0) && (p.y_bs % 4 == 0) &&
                    ((reinterpret_cast<uintptr_t>(p.y) & 15) == 0);
#pragma unroll 2
  for (int i = warp * RPW + rsub; i < DW_TL; i += (NT / 32) * RPW) {
    const int l = l0 + i;
    if (l >= p.Lout) break;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < (KT ? KT : 16); k++) {
      if (KT || k < K) {
        const float4 xv = *reinterpret_cast<const float4*>(smem + (size_t)(i + k * d) * CW + c4);
        acc.x = fmaf(xv.x, w[k].x, acc.x); acc.y = fmaf(xv.y, w[k].y, acc.y); acc.z = fmaf(xv.z, w[k].z, acc.z); acc.w = fmaf(xv.w, w[k].w, acc.w);
      }
    }
    if (p.emit_hi) {                                    // the consumer's prologue + bf16 split, straight from registers
      float o[4] = {(acc.x + bias4.x) * p.out_scale, (acc.y + bias4.y) * p.out_scale, (acc.z + bias4.z) * p.out_scale, (acc.w + bias4.w) * p.out_scale};
      __align__(8) __nv_bfloat16 h[4], lw[4];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        float t = o[q];
        if constexpr (SNAKE) { const float sn = b2a_sin(ea[q] * t); t = fmaf(eb[q], sn * sn, t); }
        else if (p.emit_act) t = b2a_act(t, p.emit_act, p.emit_p0, ea[q], eb[q]);
        h[q] = __float2bfloat16_rn(t);
        lw[q] = __float2bfloat16_rn(t - __bfloat162float(h[q]));
      }
      const int64_t row = (int64_t)b * p.Lout + l;
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.emit_hi) + row * p.emit_ld + c) = *reinterpret_cast<uint2*>(h);
      if (p.emit_lo) *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.emit_lo) + row * p.emit_ld + c) = *reinterpret_cast<uint2*>(lw);
    } else if (fast) {
      float4 o = make_float4((acc.x + bias4.x) * p.out_scale, (acc.y + bias4.y) * p.out_scale, (acc.z + bias4.z) * p.out_scale,
                             (acc.w + bias4.w) * p.out_scale);
      *reinterpret_cast<float4*>(p.y + (int64_t)b * p.y_bs + (int64_t)l * p.y_ld + c) = o;
    } else {
      epilogue_store(p, b, l, c, acc.x); epilogue_store(p, b, l, c + 1, acc.y);
      epilogue_store(p, b, l, c + 2, acc.z); epilogue_store(p, b, l, c + 3, acc.w);
    }
  }
}

// Dense stride-1 conv with a NARROW output (Cout <= 4: the 64->1 / 96->1 waveform heads of Mimi, SNAC and the Qwen3 vocoder).
// The 64 x BN implicit-GEMM tile wastes 15/16 of its threads there (Mimi head: 14 ms for 4.9 GB of input).  Here a CTA stages
// NW_TL + (K-1)*dilation transformed input rows once (coalesced, prologue applied once per element), and each thread owns one
// output position: K*Cin FMAs against shared memory (row stride Cin+1: conflict-free), weights broadcast from shared memory.
// HBM-bound by construction: x is read once, y is 1/Cin of it.
constexpr int NW_TL = 256;
template <int ACT>      // ACT >= 0: prologue activation fixed at compile time (no AdaIN scale/shift); -1: generic functor
__global__ void __launch_bounds__(NT) conv1d_narrow_kernel(const b2a_conv1d_t p, int rows, bool v4) {   // v4: 16-byte staging loads
  extern __shared__ __align__(16) float smem[];
  const int ldx = p.Cin + 1;
  float* xs = smem;                                   // [rows][Cin+1]
  float* ws = smem + (size_t)rows * ldx;              // [K][Cin][Cout]
  const int tid = threadIdx.x, b = blockIdx.y;
  const int l0 = blockIdx.x * NW_TL;
  const Pre pre_f = make_pre(p);
  auto pre = [&](float v, int bi, int c) -> float {
    if constexpr (ACT == B2A_ACT_SNAKE) { const float sn = b2a_sin(__ldg(p.pre_a + c) * v); return fmaf(__ldg(p.pre_b + c), sn * sn, v); }
    else if constexpr (ACT == B2A_ACT_ELU) return v > 0.f ? v : expm1f(v);
    else if constexpr (ACT == B2A_ACT_LRELU) return v > 0.f ? v : v * p.pre_p0;
    else if constexpr (ACT == 0) return v;
    else return pre_f(v, bi, c);
  };
  const float* xb = p.x + (int64_t)b * p.x_bs;
  const int64_t pos0 = (int64_t)l0 - p.pad_left;
  if (v4) {
    // 16-byte loads, four in flight per thread before the first is consumed (the scalar one-load-per-iteration loop left the CTA
    // waiting a full memory latency 64 times per tile: 9.7 ms for Mimi's 4.9 GB head instead of ~1 ms)
    const int q4 = p.Cin >> 2, n4 = rows * q4;
    for (int i0 = tid; i0 < n4; i0 += 4 * NT) {
      float4 t[4]; int rr[4], cc[4]; bool ok[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int i = i0 + u * NT;
        rr[u] = i / q4; cc[u] = (i - rr[u] * q4) << 2;
        int64_t pos = pos0 + rr[u];
        if (pos < 0 || pos >= p.L) pos = p.pad_mode == 1 ? (pos < 0 ? 0 : (int64_t)p.L - 1) : -1;
        ok[u] = i < n4 && pos >= 0;
        t[u] = ok[u] ? __ldg(reinterpret_cast<const float4*>(xb + pos * p.x_ld + cc[u])) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        if (i0 + u * NT < n4) {
          float* d = xs + rr[u] * ldx + cc[u];
          if (ok[u]) { d[0] = pre(t[u].x, b, cc[u]); d[1] = pre(t[u].y, b, cc[u] + 1); d[2] = pre(t[u].z, b, cc[u] + 2); d[3] = pre(t[u].w, b, cc[u] + 3); }
          else { d[0] = 0.f; d[1] = 0.f; d[2] = 0.f; d[3] = 0.f; }
        }
      }
    }
  } else {
    for (int idx = tid; idx < rows * p.Cin; idx += NT) {
      const int c = idx % p.Cin, r = idx / p.Cin;
      const int64_t pos = pos0 + r;
      float v = 0.f;
      if (pos >= 0 && pos < p.L) v = pre(__ldg(xb + pos * p.x_ld + c), b, c);
      else if (p.pad_mode == 1) v = pre(__ldg(xb + (pos < 0 ? 0 : (int64_t)p.L - 1) * p.x_ld + c), b, c);
      xs[r * ldx + c] = v;
    }
  }
  for (int idx = tid; idx < p.K * p.Cin * p.Cout; idx += NT) ws[idx] = __ldg(p.w + idx);
  __syncthreads();
  const int l = l0 + tid;
  if (tid >= NW_TL || l >= p.Lout) return;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k = 0; k < p.K; k++) {
    const float* xr = xs + (size_t)(tid + k * p.dilation) * ldx;
    const float* wk = ws + (size_t)k * p.Cin * p.Cout;
    if (p.Cout == 1) {
#pragma unroll 8
      for (int c = 0; c < p.Cin; c++) acc[0] = fmaf(xr[c], wk[c], acc[0]);
    } else {
      for (int c = 0; c < p.Cin; c++) {
        const float xv = xr[c];
        for (int co = 0; co < p.Cout; co++) acc[co] = fmaf(xv, wk[c * p.Cout + co], acc[co]);
      }
    }
  }
  for (int co = 0; co < p.Cout; co++) epilogue_store(p, b, l, co, acc[co]);
}

// Depthwise conv1d, stride 1, staged: a CTA owns DW_TL positions x 32 channels.  The input span
// (DW_TL + (K-1)*dilation rows) is transformed ONCE (AdaIN/Snake prologue) while it is staged in
// shared memory, so the transcendental is paid per input element rather than per tap, and every
// tap is a conflict-free shared-memory read (lane == channel).  Halo rows are shared with the
// neighbouring CTAs through L2, so HBM sees x once.
template <int KT>
__global__ void __launch_bounds__(NT) conv1d_dw_tiled_kernel(const b2a_conv1d_t p, int rows) {
  extern __shared__ __align__(16) float smem[];      // [rows][32]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int l0 = blockIdx.x * DW_TL, c = blockIdx.y * 32 + lane, b = blockIdx.z;
  const bool cok = c < p.Cout;
  const Pre pre = make_pre(p);
  const int K = KT ? KT : p.K;
  const float* xb = p.x + (int64_t)b * p.x_bs + c;
  const int64_t pos0 = (int64_t)l0 - p.pad_left;
  for (int r = warp; r < rows; r += NT / 32) {
    int64_t pos = pos0 + r;
    float v = 0.f;
    if (cok) {
      if (pos >= 0 && pos < p.L) v = pre(__ldg(xb + pos * p.x_ld), b, c);
      else if (p.pad_mode == 1) v = pre(__ldg(xb + (pos < 0 ? 0 : (int64_t)p.L - 1) * p.x_ld), b, c);
    }
    smem[r * 32 + lane] = v;
  }
  float w[KT ? KT : 16];
#pragma unroll
  for (int k = 0; k < (KT ? KT : 16); k++) w[k] = (cok && k < K) ? __ldg(p.w + (int64_t)k * p.Cout + c) : 0.f;
  __syncthreads();
  if (!cok) return;
  const int d = p.dilation;
#pragma unroll 4
  for (int i = warp; i < DW_TL; i += NT / 32) {
    int l = l0 + i;
    if (l >= p.Lout) break;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < (KT ? KT : 16); k++)
      if (KT || k < K) acc = fmaf(smem[(i + k * d) * 32 + lane], w[k], acc);
    epilogue_store(p, b, l, c, acc);
  }
}

// ------------------------------------------------------------------------------------------------
// Dense transposed conv, gather (polyphase) form: output l (q = l + pad_left) takes taps
// k = q%s + j*s from input rows q/s - j.  Tile = 64 positions x 64 channels.
__global__ void __launch_bounds__(NT) convtr1d_dense_kernel(const b2a_conv1d_t p, int CI, int rows, int J) {
  constexpr int BN = 64;
  extern __shared__ __align__(16) float smem[];
  float* xs = smem;                                   // [rows][CI+1]
  float* ws = smem + (((size_t)rows * (CI + 1) + 3) & ~(size_t)3);   // [K][CI][BN], 16-byte aligned for float4 reads
  const int tid = threadIdx.x, tn = tid & 15, tm = tid >> 4;
  const int l0 = blockIdx.x * BM, n0 = blockIdx.y * BN, b = blockIdx.z;
  const int s = p.stride;
  const Pre pre = make_pre(p);
  const float* xb = p.x + (int64_t)b * p.x_bs;
  const int ibase = (l0 + p.pad_left) / s - (J - 1);
  int r_[4], ih_[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    int q = l0 + tm * 4 + i + p.pad_left;
    r_[i] = q % s; ih_[i] = q / s - ibase;
  }
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

  for (int c0 = 0; c0 < p.Cin; c0 += CI) {
    for (int idx = tid; idx < rows * CI; idx += NT) {
      int ci = idx % CI, r = idx / CI;
      int64_t pos = (int64_t)ibase + r;
      int c = c0 + ci;
      float v = 0.f;
      if (c < p.Cin && pos >= 0 && pos < p.L) v = pre(__ldg(xb + pos * p.x_ld + c), b, c);
      xs[r * (CI + 1) + ci] = v;
    }
    for (int idx = tid; idx < p.K * CI * BN; idx += NT) {
      int n = idx % BN, ci = (idx / BN) % CI, k = idx / (BN * CI);
      int c = c0 + ci, co = n0 + n;
      ws[idx] = (c < p.Cin && co < p.Cout) ? __ldg(p.w + ((int64_t)k * p.Cin + c) * p.Cout + co) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; i++) {
      for (int j = 0; j < J; j++) {
        int k = r_[i] + j * s;
        if (k >= p.K) break;
        const float* xr = xs + (size_t)(ih_[i] - j) * (CI + 1);
        const float* wr = ws + (size_t)k * CI * BN + tn * 4;
#pragma unroll 4
        for (int ci = 0; ci < CI; ci++) {
          float a = xr[ci];
          float4 t = *reinterpret_cast<const float4*>(wr + ci * BN);
          acc[i][0] = fmaf(a, t.x, acc[i][0]); acc[i][1] = fmaf(a, t.y, acc[i][1]);
          acc[i][2] = fmaf(a, t.z, acc[i][2]); acc[i][3] = fmaf(a, t.w, acc[i][3]);
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    int l = l0 + tm * 4 + i;
    if (l >= p.Lout) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      int co = n0 + tn * 4 + j;
      if (co < p.Cout) epilogue_store(p, b, l, co, acc[i][j]);
    }
  }
}

// grid (row groups of 16, channel groups of 128, batch): no 64-bit index arithmetic per element (the flat-index version spent
// its time in four 64-bit divisions per output: 10.6 ms for Mimi's 20 000 x 512 up-sampler)
constexpr int TRDW_ROWS = 16;
__global__ void __launch_bounds__(128) convtr1d_dw_kernel(const b2a_conv1d_t p) {
  const Pre pre = make_pre(p);
  const int s = p.stride;
  const int c = blockIdx.y * 128 + threadIdx.x, b = blockIdx.z;
  if (c >= p.Cout) return;
  const float* xb = p.x + (int64_t)b * p.x_bs + c;
  const int l_end = min(p.Lout, (int)(blockIdx.x + 1) * TRDW_ROWS);
  for (int l = blockIdx.x * TRDW_ROWS; l < l_end; l++) {
    const int q = l + p.pad_left;
    const int r = q % s, ih = q / s;
    float acc = 0.f;
    for (int k = r, i = ih; k < p.K && i >= 0; k += s, i--) {
      if (i < p.L) acc = fmaf(pre(__ldg(xb + (int64_t)i * p.x_ld), b, c), __ldg(p.w + (int64_t)k * p.Cout + c), acc);
    }
    epilogue_store(p, b, l, c, acc);
  }
}

__global__ void copy2d_kernel(const float* __restrict__ src, int64_t src_ld, float* __restrict__ dst, int64_t dst_ld,
                              int64_t rows, int cols) {
  int64_t total = rows * cols;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = idx / cols; int c = (int)(idx % cols);
    dst[r * dst_ld + c] = src[r * src_ld + c];
  }
}

__global__ void gather_rows_kernel(const float* __restrict__ src, int64_t src_ld, const int64_t* __restrict__ idx_,
                                   float* __restrict__ dst, int64_t dst_ld, int64_t rows, int cols, int64_t n_src,
                                   const float* __restrict__ add, int64_t add_ld, int64_t add_period) {
  int64_t total = rows * cols;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = idx / cols; int c = (int)(idx % cols);
    int64_t s = idx_[r];
    s = s < 0 ? 0 : (s >= n_src ? n_src - 1 : s);
    float v = src[s * src_ld + c];
    if (add) v += add[(r % add_period) * add_ld + c];          // e.g. token embedding + positional embedding (whisper.py:483-486)
    dst[r * dst_ld + c] = v;
  }
}

// single-CTA duration head + exclusive scan, then each token writes its own run of frame indices
__global__ void durations_to_index_kernel(const float* __restrict__ dur_f, const int64_t* __restrict__ dur_i, int T, float speed,
                                          int64_t* __restrict__ pred, int64_t* __restrict__ out, int64_t max_frames,
                                          int64_t* __restrict__ total) {
  extern __shared__ long long sc[];
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    long long d;
    if (dur_f) {
      float v = dur_f[i] / speed;
      if (isnan(v)) v = 1.f; else if (isinf(v)) v = v > 0 ? 100.f : 1.f;
      v = fminf(fmaxf(rintf(v), 1.f), 100.f);          // rintf = round-half-to-even like mx.round
      d = (long long)v;
    } else {
      d = dur_i[i] < 0 ? 0 : dur_i[i];
    }
    sc[i] = d; pred[i] = d;
  }
  __syncthreads();
  if (threadIdx.x == 0) {               // T <= 512 tokens: a serial scan is a few hundred ns
    long long run = 0;
    for (int i = 0; i < T; i++) { long long d = sc[i]; sc[i] = run; run += d; }
    *total = run;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    long long beg = sc[i], n = pred[i];
    for (long long f = beg; f < beg + n && f < max_frames; f++) out[f] = i;
  }
}

int check_common(const b2a_conv1d_t* p) {
  if (!p || !p->x || !p->w || (!p->y && !p->emit_hi)) return 1;
  if (p->B <= 0 || p->L <= 0 || p->Cin <= 0 || p->Cout <= 0 || p->Lout <= 0) return 2;
  if (p->K <= 0 || p->stride <= 0 || p->dilation <= 0 || p->res_div <= 0) return 3;
  if ((p->pre_scale == nullptr) != (p->pre_shift == nullptr)) return 4;
  return 0;
}

}  // namespace

namespace {
// nn.Linear on a handful of rows (Kokoro: the 49 684-wide style projection of ONE style vector, twice per utterance): thread per output
// column, the rows' inputs in shared memory, the [Cin][Cout] weight streamed once with coalesced loads.  The 64 x 64 tile kernel spends
// 93 us on it (777 latency-bound CTAs); this is one pass over the weight at HBM speed.
constexpr int LR_MAX = 8;
__global__ void __launch_bounds__(128) linear_rows_kernel(const b2a_conv1d_t p, int rows) {
  extern __shared__ float lr_x[];                                  // [rows][Cin]
  for (int i = threadIdx.x; i < rows * p.Cin; i += blockDim.x) {
    const int r = i / p.Cin, c = i - r * p.Cin;
    const int b = r / p.L, l = r - b * p.L;
    lr_x[i] = p.x[(int64_t)b * p.x_bs + (int64_t)l * p.x_ld + c];
  }
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= p.Cout) return;
  float acc[LR_MAX];
#pragma unroll
  for (int r = 0; r < LR_MAX; r++) acc[r] = 0.f;
  const float* w = p.w + n;
#pragma unroll 8
  for (int c = 0; c < p.Cin; c++) {
    const float wv = __ldg(w + (int64_t)c * p.Cout);
#pragma unroll
    for (int r = 0; r < LR_MAX; r++)
      if (r < rows) acc[r] = fmaf(wv, lr_x[r * p.Cin + c], acc[r]);
  }
  const float bias = p.bias ? p.bias[n] : 0.f;
#pragma unroll
  for (int r = 0; r < LR_MAX; r++) {
    if (r < rows) {
      const int b = r / p.L, l = r - b * p.L;
      float v = acc[r] + bias;
      if (p.post_act) v = b2a_act(v, p.post_act, p.post_p0, 1.f, 1.f);
      p.y[(int64_t)b * p.y_bs + (int64_t)l * p.y_ld + n] = v * p.out_scale;
    }
  }
}

thread_local int32_t g_last_path[4] = {0, 0, 0, 0};     // kernel id + variant of this host thread's last launch (b2a_conv1d_cl_last_path)

void set_last_path(int32_t kernel, int32_t v1 = 0, int32_t v2 = 0, int32_t v3 = 0) {
  g_last_path[0] = kernel; g_last_path[1] = v1; g_last_path[2] = v2; g_last_path[3] = v3;
}
}  // namespace

/* which kernel instantiation the dispatch rules below chose, so that tests can assert the branch they exercised */
extern "C" int32_t b2a_conv1d_cl_last_path(int32_t* out4) {
  B2A_CHECK_ARG(out4, "null pointer");
  for (int i = 0; i < 4; i++) out4[i] = g_last_path[i];
  return B2A_OK;
}

extern "C" int32_t b2a_conv1d_cl(const b2a_conv1d_t* p, void* stream) {
  int bad = check_common(p);
  if (bad) { b2a_set_error("b2a_conv1d_cl: invalid argument (check %d)", bad); return B2A_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  if (p->emit_hi && !(p->groups == p->Cin && p->Cin == p->Cout)) {
    b2a_set_error("b2a_conv1d_cl: plane emission is implemented for depthwise layers");
    return B2A_E_UNSUPPORTED;
  }
  if (p->groups == 1 && p->K == 1 && p->stride == 1 && p->pad_left == 0 && p->Lout == p->L && (int64_t)p->B * p->L <= LR_MAX && p->Cout >= 256 &&
      !p->pre_scale && !p->pre_act && !p->post_cscale && !p->res && !p->accumulate && !p->emit_hi &&
      (size_t)p->B * p->L * p->Cin * sizeof(float) <= 48 * 1024) {
    const int rows = p->B * p->L;
    linear_rows_kernel<<<cdiv(p->Cout, 128), 128, (size_t)rows * p->Cin * sizeof(float), st>>>(*p, rows);
    B2A_CHECK_LAUNCH();
    set_last_path(B2A_CONV_PATH_LINEAR_ROWS);
    return B2A_OK;
  }
  int32_t kernel = 0, v1 = 0, v2 = 0, v3 = 0;          // the launch's b2a_conv1d_cl_last_path record
  if (p->groups == 1 && p->stride == 1 && p->Cout <= 4 && p->Lout >= NW_TL &&
      ((size_t)(NW_TL + (p->K - 1) * p->dilation) * (p->Cin + 1) + (size_t)p->K * p->Cin * p->Cout) * sizeof(float) <= 160 * 1024) {
    const int rows = NW_TL + (p->K - 1) * p->dilation;
    const size_t sm = ((size_t)rows * (p->Cin + 1) + (size_t)p->K * p->Cin * p->Cout) * sizeof(float);
    dim3 grid(cdiv(p->Lout, NW_TL), p->B);
    const bool v4 = (p->Cin % 4 == 0) && (p->x_ld % 4 == 0) && (p->x_bs % 4 == 0) && (((uintptr_t)p->x & 15) == 0);
    const int act = p->pre_scale ? -1
                  : (p->pre_act == 0 || p->pre_act == B2A_ACT_ELU || p->pre_act == B2A_ACT_LRELU ||
                     (p->pre_act == B2A_ACT_SNAKE && p->pre_a && p->pre_b)) ? p->pre_act : -1;
    const auto kern = act == 0 ? conv1d_narrow_kernel<0>
                    : act == B2A_ACT_SNAKE ? conv1d_narrow_kernel<B2A_ACT_SNAKE>
                    : act == B2A_ACT_ELU ? conv1d_narrow_kernel<B2A_ACT_ELU>
                    : act == B2A_ACT_LRELU ? conv1d_narrow_kernel<B2A_ACT_LRELU> : conv1d_narrow_kernel<-1>;
    B2A_SMEM_OPTIN(kern, 160 * 1024);
    kern<<<grid, NT, sm, st>>>(*p, rows, v4);
    kernel = B2A_CONV_PATH_NARROW; v1 = act; v3 = v4;
  } else if (p->groups == 1) {
    const int CI = p->K <= 4 ? 32 : (p->K <= 12 ? 16 : 8);
    const int rows = (BM - 1) * p->stride + (p->K - 1) * p->dilation + 1;
    const int BN = p->Cout > 16 ? 64 : 16;
    size_t smem = ((((size_t)rows * (CI + 1) + 3) & ~(size_t)3) + (size_t)p->K * CI * BN) * sizeof(float);
    if (smem > 200 * 1024) { b2a_set_error("b2a_conv1d_cl: tile needs %zu B of shared memory", smem); return B2A_E_UNSUPPORTED; }
    dim3 grid(cdiv(p->Lout, BM), cdiv(p->Cout, BN), p->B);
    const auto kern = BN == 64 ? conv1d_dense_kernel<64> : conv1d_dense_kernel<16>;
    B2A_SMEM_OPTIN(kern, 200 * 1024);
    kern<<<grid, NT, smem, st>>>(*p, CI, rows);
    kernel = B2A_CONV_PATH_DENSE; v1 = BN; v2 = CI;
  } else if (p->groups == p->Cin && p->Cin == p->Cout) {
    int rows = DW_TL + (p->K - 1) * p->dilation;
    const bool v4 = p->stride == 1 && p->K <= 16 && p->Lout >= DW_TL && p->Cout % 4 == 0 && p->x_ld % 4 == 0 && p->x_bs % 4 == 0 &&
                    ((uintptr_t)p->x & 15) == 0 && ((uintptr_t)p->w & 15) == 0 && (!p->bias || ((uintptr_t)p->bias & 15) == 0) &&
                    (size_t)rows * 128 * 4 <= 160 * 1024;
    if (p->emit_hi && !(v4 && p->Cout % 64 == 0 && p->emit_ld >= p->Cout && p->emit_ld % 4 == 0 && !p->res && !p->post_cscale && !p->accumulate &&
                        !p->post_act)) {
      b2a_set_error("b2a_conv1d_cl: plane emission needs the vectorised depthwise path (stride 1, Cout %% 64 == 0, no epilogue extras)");
      return B2A_E_UNSUPPORTED;
    }
    if (v4) {
      const int CW = p->Cout >= 128 ? 128 : 64;
      dim3 grid((p->Lout + DW_TL - 1) / DW_TL, (p->Cout + CW - 1) / CW, p->B);
      const size_t sm = (size_t)rows * CW * sizeof(float);
      const bool snake = p->pre_act == B2A_ACT_SNAKE && !p->pre_scale && (!p->emit_hi || p->emit_act == B2A_ACT_SNAKE);
      const auto kern = p->K == 7 && snake ? (CW == 128 ? conv1d_dw_tiled4_kernel<7, 128, true> : conv1d_dw_tiled4_kernel<7, 64, true>)
                      : p->K == 7 ? (CW == 128 ? conv1d_dw_tiled4_kernel<7, 128, false> : conv1d_dw_tiled4_kernel<7, 64, false>)
                      : (CW == 128 ? conv1d_dw_tiled4_kernel<0, 128, false> : conv1d_dw_tiled4_kernel<0, 64, false>);
      B2A_SMEM_OPTIN(kern, 160 * 1024);
      kern<<<grid, NT, sm, st>>>(*p, rows);
      kernel = B2A_CONV_PATH_DW_TILED4; v1 = CW; v2 = p->K == 7 ? 7 : 0; v3 = p->K == 7 && snake;
    } else if (p->stride == 1 && p->K <= 16 && rows * 32 * 4 <= 96 * 1024 && p->Lout >= DW_TL) {
      dim3 grid((p->Lout + DW_TL - 1) / DW_TL, (p->Cout + 31) / 32, p->B);
      size_t sm = (size_t)rows * 32 * sizeof(float);
      const auto kern = p->K == 7 ? conv1d_dw_tiled_kernel<7> : conv1d_dw_tiled_kernel<0>;
      B2A_SMEM_OPTIN(kern, 96 * 1024);
      kern<<<grid, NT, sm, st>>>(*p, rows);
      kernel = B2A_CONV_PATH_DW_TILED; v1 = p->K == 7 ? 7 : 0;
    } else {
      int64_t total = (int64_t)p->B * p->Lout * p->Cout;
      int blocks = (int)((total + NT - 1) / NT); if (blocks > 132 * 32) blocks = 132 * 32;
      conv1d_dw_kernel<<<blocks, NT, 0, st>>>(*p);
      kernel = B2A_CONV_PATH_DW;
    }
  } else {
    b2a_set_error("b2a_conv1d_cl: groups must be 1 or Cin==Cout==groups (got %d)", p->groups);
    return B2A_E_UNSUPPORTED;
  }
  B2A_CHECK_LAUNCH();
  set_last_path(kernel, v1, v2, v3);
  return B2A_OK;
}

extern "C" int32_t b2a_convtr1d_cl(const b2a_conv1d_t* p, void* stream) {
  int bad = check_common(p);
  if (bad) { b2a_set_error("b2a_convtr1d_cl: invalid argument (check %d)", bad); return B2A_E_INVALID; }
  B2A_CHECK_ARG(p->emit_hi == nullptr && p->y != nullptr, "plane emission is not available for transposed convs");
  B2A_CHECK_ARG(p->dilation == 1, "dilation must be 1");
  B2A_CHECK_ARG(p->pad_left >= 0, "pad_left (crop) must be >= 0");
  cudaStream_t st = (cudaStream_t)stream;
  if (p->groups == 1) {
    const int CI = p->K <= 12 ? 16 : 8;
    const int J = (p->K + p->stride - 1) / p->stride;
    const int rows = (BM - 1) / p->stride + J + 1;
    size_t smem = ((((size_t)rows * (CI + 1) + 3) & ~(size_t)3) + (size_t)p->K * CI * 64) * sizeof(float);
    if (smem > 200 * 1024) { b2a_set_error("b2a_convtr1d_cl: tile needs %zu B of shared memory", smem); return B2A_E_UNSUPPORTED; }
    B2A_SMEM_OPTIN(convtr1d_dense_kernel, 200 * 1024);
    dim3 grid(cdiv(p->Lout, BM), cdiv(p->Cout, 64), p->B);
    convtr1d_dense_kernel<<<grid, NT, smem, st>>>(*p, CI, rows, J);
    B2A_CHECK_LAUNCH();
    set_last_path(B2A_CONV_PATH_CONVTR_DENSE, 64, CI);
  } else if (p->groups == p->Cin && p->Cin == p->Cout) {
    dim3 grid(cdiv(p->Lout, TRDW_ROWS), cdiv(p->Cout, 128), p->B);
    convtr1d_dw_kernel<<<grid, 128, 0, st>>>(*p);
    B2A_CHECK_LAUNCH();
    set_last_path(B2A_CONV_PATH_CONVTR_DW);
  } else {
    b2a_set_error("b2a_convtr1d_cl: groups must be 1 or Cin==Cout==groups (got %d)", p->groups);
    return B2A_E_UNSUPPORTED;
  }
  return B2A_OK;
}

// ------------------------------------------------------------------------------------------------
// Kokoro's harmonic-source convs (istftnet.py:780-800 noise_convs): 22 input channels (the source STFT's magnitude | phase),
// (K, stride) = (12, 6) into 256 channels and (1, 1) into 128.  The generic dense tile pads the 22 channels to its chunk width and
// pays runtime divisions for every staged element; here Cin, K and the stride are compile-time constants.  A CTA owns
// SC_BM positions x SC_BN channels: its input span is ONE contiguous block of rows x 22 floats (staged with 8-byte loads, zero
// outside [0, L)) and its weight slice [K][22][SC_BN] is staged once.  Warp = 64 positions x 32 channels; lane (tm, tn) owns
// positions tm + 8i (i < 8: consecutive lanes read rows stride*22 floats apart, distinct banks) and channels tn*8 .. tn*8+7.
//
// Every output gets exactly the fmaf sequence of conv1d_dense_kernel, whose chunk width is CI = 16 for K = 12 and 32 for K = 1:
// chunks [0, SPLIT) then [SPLIT, 22), each taps ascending then channels ascending, then bias.  The dense tile's zero-padded
// channels 22 .. CI-1 run fmaf(0, 0, acc) after each tap of the last chunk; that equals acc + 0 (identity except -0 -> +0), and a
// run of them equals one, so each is replaced by a single add of +0.
namespace {
constexpr int SC_CIN = 22, SC_BM = 128, SC_BN = 128;

template <int K, int S>
__global__ void __launch_bounds__(NT, 2) kokoro_source_conv_kernel(const float* __restrict__ x, int L, const float* __restrict__ w,
                                                                   const float* __restrict__ bias, float* __restrict__ y, int Lout,
                                                                   int Cout, int pad_left) {
  constexpr int SPLIT = K == 1 ? SC_CIN : 16;                  // channel chunks of the dense tile: CI = 32 (K <= 4) or 16 (K <= 12)
  constexpr int ROWS = (SC_BM - 1) * S + K;
  constexpr int XS = ((ROWS * SC_CIN + 3) / 4) * 4;             // floats of the staged input span, 16-byte aligned end
  extern __shared__ __align__(16) float smem[];
  float* xs = smem;                                             // [ROWS][22]
  float* ws = smem + XS;                                        // [K][22][SC_BN]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tn = lane & 3, tm = lane >> 2;
  const int wn = warp & 3, wm = warp >> 2;
  const int l0 = blockIdx.x * SC_BM, n0 = blockIdx.y * SC_BN, b = blockIdx.z;
  const int64_t e0 = ((int64_t)l0 * S - pad_left) * SC_CIN;     // first staged element (even: 22 is)
  const int64_t ne = (int64_t)L * SC_CIN;
  const float* xb = x + (int64_t)b * ne;
  for (int e = 2 * tid; e < ROWS * SC_CIN; e += 2 * NT) {
    const int64_t g = e0 + e;
    float2 v = make_float2(0.f, 0.f);
    if (g >= 0 && g < ne) v = __ldg(reinterpret_cast<const float2*>(xb + g));
    *reinterpret_cast<float2*>(xs + e) = v;
  }
  for (int e = 4 * tid; e < K * SC_CIN * SC_BN; e += 4 * NT) {
    const int r = e / SC_BN, n = e - r * SC_BN;
    *reinterpret_cast<float4*>(ws + e) = __ldg(reinterpret_cast<const float4*>(w + (int64_t)r * Cout + n0 + n));
  }
  __syncthreads();
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) acc[i][j] = 0.f;
  const float* xr = xs + (wm * 64 + tm) * S * SC_CIN;
  const float* wr = ws + wn * 32 + tn * 8;
  auto step = [&](int k, int c) {
    float a[8];
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = xr[(8 * i * S + k) * SC_CIN + c];
    const float4 w0 = *reinterpret_cast<const float4*>(wr + (k * SC_CIN + c) * SC_BN);
    const float4 w1 = *reinterpret_cast<const float4*>(wr + (k * SC_CIN + c) * SC_BN + 4);
    const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j < 8; j++) acc[i][j] = fmaf(a[i], wv[j], acc[i][j]);
  };
  if constexpr (SPLIT < SC_CIN) {
#pragma unroll 1
    for (int k = 0; k < K; k++) {
#pragma unroll
      for (int c = 0; c < SPLIT; c++) step(k, c);
    }
  }
#pragma unroll 1
  for (int k = 0; k < K; k++) {
#pragma unroll
    for (int c = SPLIT < SC_CIN ? SPLIT : 0; c < SC_CIN; c++) step(k, c);
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j < 8; j++) acc[i][j] = __fadd_rn(acc[i][j], 0.f);     // the padded channels' fmaf(0, 0, acc)
  }
  const int co = n0 + wn * 32 + tn * 8;
  float bv[8];
#pragma unroll
  for (int j = 0; j < 8; j++) bv[j] = bias ? __ldg(bias + co + j) : 0.f;
  float* yb = y + (int64_t)b * Lout * Cout + co;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int l = l0 + wm * 64 + tm + 8 * i;
    if (l >= Lout) break;
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; j++) o[j] = bias ? acc[i][j] + bv[j] : acc[i][j];
    *reinterpret_cast<float4*>(yb + (int64_t)l * Cout) = make_float4(o[0], o[1], o[2], o[3]);
    *reinterpret_cast<float4*>(yb + (int64_t)l * Cout + 4) = make_float4(o[4], o[5], o[6], o[7]);
  }
}

template <int K, int S>
int32_t launch_kokoro_source_conv(const float* x, int32_t B, int32_t L, const float* w, const float* bias, float* y, int32_t Lout,
                                  int32_t Cout, int32_t pad_left, cudaStream_t st) {
  constexpr int ROWS = (SC_BM - 1) * S + K;
  const size_t sm = ((size_t)((ROWS * SC_CIN + 3) / 4) * 4 + (size_t)K * SC_CIN * SC_BN) * sizeof(float);
  B2A_SMEM_OPTIN((kokoro_source_conv_kernel<K, S>), sm);
  dim3 grid(cdiv(Lout, SC_BM), Cout / SC_BN, B);
  kokoro_source_conv_kernel<K, S><<<grid, NT, sm, st>>>(x, L, w, bias, y, Lout, Cout, pad_left);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
}  // namespace

/* Kokoro's noise_convs on the harmonic source har [B, L, 22] (contiguous) -> y [B, Lout, Cout] (contiguous); bit-identical to
 * b2a_conv1d_cl on the same layer */
extern "C" int32_t b2a_kokoro_source_conv(const float* x, int32_t B, int32_t L, const float* w, const float* bias, float* y, int32_t Lout,
                                          int32_t Cout, int32_t K, int32_t stride, int32_t pad_left, void* stream) {
  B2A_CHECK_ARG(x && w && y && B > 0 && L > 0 && Lout > 0, "bad pointers / shape");
  B2A_CHECK_ARG(Cout > 0 && Cout % SC_BN == 0, "Cout must be a multiple of 128");
  B2A_CHECK_ARG(((uintptr_t)x & 7) == 0 && ((uintptr_t)w & 15) == 0 && ((uintptr_t)y & 15) == 0, "x needs 8-byte, w and y 16-byte alignment");
  cudaStream_t st = (cudaStream_t)stream;
  if (K == 12 && stride == 6) return launch_kokoro_source_conv<12, 6>(x, B, L, w, bias, y, Lout, Cout, pad_left, st);
  if (K == 1 && stride == 1) return launch_kokoro_source_conv<1, 1>(x, B, L, w, bias, y, Lout, Cout, pad_left, st);
  b2a_set_error("b2a_kokoro_source_conv: (K, stride) must be (12, 6) or (1, 1), got (%d, %d)", K, stride);
  return B2A_E_UNSUPPORTED;
}

extern "C" int32_t b2a_copy2d(const float* src, int64_t src_ld, float* dst, int64_t dst_ld, int64_t rows, int32_t cols, void* stream) {
  B2A_CHECK_ARG(src && dst && rows >= 0 && cols > 0, "bad pointers/shape");
  if (rows == 0) return B2A_OK;
  int64_t total = rows * cols;
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 16) blocks = 132 * 16;
  copy2d_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, src_ld, dst, dst_ld, rows, cols);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_gather_rows(const float* src, int64_t src_ld, const int64_t* idx, float* dst, int64_t dst_ld,
                                   int64_t rows, int32_t cols, int64_t n_src_rows, const float* add, int64_t add_ld,
                                   int64_t add_period, void* stream) {
  B2A_CHECK_ARG(src && dst && idx && rows >= 0 && cols > 0 && n_src_rows > 0 && (!add || add_period > 0), "bad pointers/shape");
  if (rows == 0) return B2A_OK;
  int64_t total = rows * cols;
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 16) blocks = 132 * 16;
  gather_rows_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, src_ld, idx, dst, dst_ld, rows, cols, n_src_rows, add, add_ld,
                                                               add_period);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_durations_to_index(const float* dur_f, const int64_t* dur_i, int32_t T, float speed, int64_t* pred_dur_out,
                                          int64_t* idx_out, int64_t max_frames, int64_t* total_dev, void* stream) {
  B2A_CHECK_ARG((dur_f || dur_i) && pred_dur_out && idx_out && total_dev && T > 0 && T <= 4096 && speed > 0.f,
                "bad pointers / T out of range / speed <= 0");
  durations_to_index_kernel<<<1, 256, T * sizeof(long long), (cudaStream_t)stream>>>(dur_f, dur_i, T, speed, pred_dur_out, idx_out,
                                                                                     max_frames, total_dev);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
