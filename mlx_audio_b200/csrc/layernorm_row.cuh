// One row of the register-resident LayerNorm / RMSNorm, computed by one warp; shared by layernorm_vec_kernel (norm.cu), the
// persistent ALBERT kernel (albert.cu) and Vocos's depthwise-conv + LayerNorm kernel (vocos.cu).  NV = float4 slots per lane
// (C <= 128 * NV); row pointers 16-byte aligned; x and y may alias (every load of the row is issued before the first store).
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

// Statistics, affine and stores of a row already in registers: v[j] holds channels 4 (lane + 32 j) .. + 3, zero beyond C.
// ROW_AFFINE: ``ada`` is a per-row (scale | shift) pair [2C] applied as scale v + shift (Vocos's AdaLayerNorm) instead of the shared
// (1 + a) v + b form.  Y_OPT: y may be NULL (only the bf16 planes are written).
template <int NV, bool ROW_AFFINE = false, bool Y_OPT = false>
__device__ __forceinline__ void layernorm_row_regs(float4 (&v)[NV], float* y, int C, const float* w, const float* bb, const float* ada,
                                                   float eps, int rms, int post_act, float post_p0, __nv_bfloat16* e_hi,
                                                   __nv_bfloat16* e_lo, int lane) {
  const int nv = C >> 2;
  float s1 = 0.f;
#pragma unroll
  for (int j = 0; j < NV; j++) s1 += (v[j].x + v[j].y) + (v[j].z + v[j].w);
  s1 = warp_sum(s1);
  const float mean = rms ? 0.f : s1 / C;
  float s2 = 0.f;
#pragma unroll
  for (int j = 0; j < NV; j++) {
    if (lane + 32 * j < nv) {
      const float a = v[j].x - mean, b = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
      s2 = fmaf(a, a, s2); s2 = fmaf(b, b, s2); s2 = fmaf(c, c, s2); s2 = fmaf(d, d, s2);
    }
  }
  s2 = warp_sum(s2);
  const float rstd = rsqrtf(s2 / C + eps);
  float4* yp = reinterpret_cast<float4*>(y);
#pragma unroll
  for (int j = 0; j < NV; j++) {
    const int i = lane + 32 * j;
    if (i < nv) {
      float o[4] = {(v[j].x - mean) * rstd, (v[j].y - mean) * rstd, (v[j].z - mean) * rstd, (v[j].w - mean) * rstd};
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int c = 4 * i + q;
        if (ROW_AFFINE) o[q] = fmaf(ada[c], o[q], ada[C + c]);
        else if (ada) o[q] = fmaf(1.f + ada[c], o[q], ada[C + c]);
        else { if (w) o[q] *= w[c]; if (bb) o[q] += bb[c]; }
        if (post_act) o[q] = b2a_act(o[q], post_act, post_p0, 1.f, 1.f);
      }
      if (!Y_OPT || y) yp[i] = make_float4(o[0], o[1], o[2], o[3]);
      if (e_hi) {
        __align__(8) __nv_bfloat16 h[4], l[4];
#pragma unroll
        for (int q = 0; q < 4; q++) tc::split16(o[q], h[q], l[q]);
        *reinterpret_cast<uint2*>(e_hi + 4 * i) = *reinterpret_cast<const uint2*>(h);
        if (e_lo) *reinterpret_cast<uint2*>(e_lo + 4 * i) = *reinterpret_cast<const uint2*>(l);
      }
    }
  }
}

template <int NV>
__device__ __forceinline__ void layernorm_row_vec(const float* x, const float* res, float* y, int C, const float* w, const float* bb,
                                                  const float* ada, float eps, int rms, int post_act, float post_p0,
                                                  __nv_bfloat16* e_hi, __nv_bfloat16* e_lo, int lane) {
  const float4* xp = reinterpret_cast<const float4*>(x);
  const float4* rp = reinterpret_cast<const float4*>(res);
  const int nv = C >> 2;
  float4 v[NV];
#pragma unroll
  for (int j = 0; j < NV; j++) {
    const int i = lane + 32 * j;
    v[j] = i < nv ? xp[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (rp) {
#pragma unroll
    for (int j = 0; j < NV; j++) {
      const int i = lane + 32 * j;
      if (i < nv) { const float4 r = rp[i]; v[j].x += r.x; v[j].y += r.y; v[j].z += r.z; v[j].w += r.w; }
    }
  }
  layernorm_row_regs<NV>(v, y, C, w, bb, ada, eps, rms, post_act, post_p0, e_hi, e_lo, lane);
}
