// Attention + rotary embedding (include/b200audio.h: b2a_attention, b2a_rope).
// CUDA-core flash-style kernel: one thread owns one query row (q and the output accumulator live in
// registers), keys/values stream through shared memory in tiles of 64 and are read as warp
// broadcasts, the softmax is online in fp32 over chunks of 8 keys -- no cross-thread traffic at all.
#include "common.cuh"

namespace {

constexpr int QT = 128;   // queries (threads) per CTA
constexpr int KT = 64;    // keys per shared-memory tile

template <int D>
__global__ void __launch_bounds__(QT) attn_kernel(const b2a_attn_t p) {
  __shared__ __align__(16) float ks[KT][D];
  __shared__ __align__(16) float vs[KT][D];
  const int tid = threadIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * QT, qi = q0 + tid;
  const int hk = h / (p.H / p.Hkv);
  const bool active = qi < p.Tq;
  const int klen = p.k_len ? min(p.k_len[b], p.Tk) : p.Tk;
  float q[D], acc[D];
  float m = -INFINITY, l = 0.f;
#pragma unroll
  for (int d = 0; d < D; d++) { acc[d] = 0.f; q[d] = 0.f; }
  if (active) {
    const float* qp = p.q + (int64_t)b * p.q_bs + (int64_t)qi * p.q_ld + h * D;
#pragma unroll
    for (int d = 0; d < D; d += 4) {
      float4 t = *reinterpret_cast<const float4*>(qp + d);
      q[d] = t.x * p.scale; q[d + 1] = t.y * p.scale; q[d + 2] = t.z * p.scale; q[d + 3] = t.w * p.scale;
    }
  }
  // key range visible to this CTA's queries
  int j_lo = 0, j_hi = klen;
  if (p.causal) {
    j_hi = min(klen, min(p.Tq - 1, q0 + QT - 1) + p.q_offset + 1);
    if (p.window > 0) j_lo = max(0, q0 + p.q_offset - p.window + 1);
  }
  const int pos = qi + p.q_offset;
  const float* kb = p.k + (int64_t)b * p.k_bs + hk * D;
  const float* vb = p.v + (int64_t)b * p.v_bs + hk * D;
  for (int j0 = (j_lo / KT) * KT; j0 < j_hi; j0 += KT) {
    for (int idx = tid; idx < KT * (D / 4); idx += QT) {
      int r = idx / (D / 4), c4 = (idx % (D / 4)) * 4, j = j0 + r;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (j < klen) {
        kv = *reinterpret_cast<const float4*>(kb + (int64_t)j * p.k_ld + c4);
        vv = *reinterpret_cast<const float4*>(vb + (int64_t)j * p.v_ld + c4);
      }
      *reinterpret_cast<float4*>(&ks[r][c4]) = kv;
      *reinterpret_cast<float4*>(&vs[r][c4]) = vv;
    }
    __syncthreads();
    if (active) {
      for (int c = 0; c < KT; c += 8) {
        float s[8];
        float cmax = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 8; jj++) {
          const int j = j0 + c + jj;
          float d0 = 0.f, d1 = 0.f;
#pragma unroll
          for (int d = 0; d < D; d += 8) {
            float4 a = *reinterpret_cast<const float4*>(&ks[c + jj][d]);
            float4 e = *reinterpret_cast<const float4*>(&ks[c + jj][d + 4]);
            d0 = fmaf(q[d], a.x, d0); d0 = fmaf(q[d + 1], a.y, d0); d0 = fmaf(q[d + 2], a.z, d0); d0 = fmaf(q[d + 3], a.w, d0);
            d1 = fmaf(q[d + 4], e.x, d1); d1 = fmaf(q[d + 5], e.y, d1); d1 = fmaf(q[d + 6], e.z, d1); d1 = fmaf(q[d + 7], e.w, d1);
          }
          bool ok = j < klen;
          if (p.causal) { ok = ok && j <= pos; if (p.window > 0) ok = ok && (pos - j < p.window); }
          s[jj] = ok ? d0 + d1 : -INFINITY;
          cmax = fmaxf(cmax, s[jj]);
        }
        if (cmax == -INFINITY) continue;
        const float m_new = fmaxf(m, cmax);
        const float corr = expf(m - m_new);          // m = -inf -> 0
        l *= corr;
#pragma unroll
        for (int d = 0; d < D; d++) acc[d] *= corr;
#pragma unroll
        for (int jj = 0; jj < 8; jj++) {
          const float pj = expf(s[jj] - m_new);       // masked -> 0
          l += pj;
#pragma unroll
          for (int d = 0; d < D; d += 4) {
            float4 vv = *reinterpret_cast<const float4*>(&vs[c + jj][d]);
            acc[d] = fmaf(pj, vv.x, acc[d]); acc[d + 1] = fmaf(pj, vv.y, acc[d + 1]);
            acc[d + 2] = fmaf(pj, vv.z, acc[d + 2]); acc[d + 3] = fmaf(pj, vv.w, acc[d + 3]);
          }
        }
        m = m_new;
      }
    }
    __syncthreads();
  }
  if (active) {
    const float inv = l > 0.f ? 1.f / l : 0.f;
    float* op = p.o + (int64_t)b * p.o_bs + (int64_t)qi * p.o_ld + h * D;
#pragma unroll
    for (int d = 0; d < D; d += 4)
      *reinterpret_cast<float4*>(op + d) = make_float4(acc[d] * inv, acc[d + 1] * inv, acc[d + 2] * inv, acc[d + 3] * inv);
  }
}

__global__ void rope_kernel(float* __restrict__ x, int64_t x_bs, int64_t x_ld, int B, int T, int H, int D, int offset,
                            float base, int traditional) {
  const int half = D / 2;
  int64_t total = (int64_t)B * T * H * half;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int i = (int)(idx % half);
    int64_t r = idx / half;
    int h = (int)(r % H); r /= H;
    int t = (int)(r % T); int b = (int)(r / T);
    // angle in float64: positions reach 2e4 and fp32 would lose ~1e-3 rad
    double inv = exp(-(double)i * (log((double)base) / half));
    double ang = (double)(t + offset) * inv;
    double sn, cs; sincos(ang, &sn, &cs);
    float* xp = x + (int64_t)b * x_bs + (int64_t)t * x_ld + h * D;
    int i0 = traditional ? 2 * i : i, i1 = traditional ? 2 * i + 1 : i + half;
    float a = xp[i0], c = xp[i1];
    xp[i0] = (float)(a * cs - c * sn);
    xp[i1] = (float)(a * sn + c * cs);
  }
}

}  // namespace

extern "C" int32_t b2a_attention(const b2a_attn_t* p, void* stream) {
  B2A_CHECK_ARG(p && p->q && p->k && p->v && p->o, "null pointer");
  B2A_CHECK_ARG(p->B > 0 && p->Tq > 0 && p->Tk > 0 && p->H > 0 && p->Hkv > 0 && p->H % p->Hkv == 0, "bad shape");
  B2A_CHECK_ARG(p->window <= 0 || p->causal, "a sliding window needs causal masking");
  B2A_CHECK_ARG((p->q_ld % 4 == 0) && (p->k_ld % 4 == 0) && (p->v_ld % 4 == 0) && (p->o_ld % 4 == 0), "token strides must be multiples of 4");
  B2A_CHECK_ARG((p->q_bs % 4 == 0) && (p->k_bs % 4 == 0) && (p->v_bs % 4 == 0) && (p->o_bs % 4 == 0), "batch strides must be multiples of 4");
  B2A_CHECK_ARG((((uintptr_t)p->q | (uintptr_t)p->k | (uintptr_t)p->v | (uintptr_t)p->o) & 15) == 0, "q/k/v/o must be 16-byte aligned");
  dim3 grid(cdiv(p->Tq, QT), p->H, p->B);
  if (p->D == 64) attn_kernel<64><<<grid, QT, 0, (cudaStream_t)stream>>>(*p);
  else { b2a_set_error("b2a_attention: head dim %d not supported (64)", p->D); return B2A_E_UNSUPPORTED; }
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_rope(float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t H, int32_t D,
                            int32_t offset, float base, int32_t traditional, void* stream) {
  B2A_CHECK_ARG(x && B > 0 && T > 0 && H > 0 && D > 0 && D % 2 == 0, "bad pointers/shape");
  int64_t total = (int64_t)B * T * H * (D / 2);
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 16) blocks = 132 * 16;
  rope_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, B, T, H, D, offset, base, traditional);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
