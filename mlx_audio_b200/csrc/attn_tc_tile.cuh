// The online-softmax step of the tensor-core flash attention for one warpgroup's 64 query rows and one 64-key tile, shared by
// attn_tc_kernel (attn_tc.cu) and the persistent ALBERT kernel (albert.cu).  Operands are fp16 hi / lo planes in 128B-swizzled shared
// memory: Q (pre-scaled by scale * log2 e) and K K-major, V transposed (64 dims x 64 keys).
#pragma once
#include "tc_common.cuh"

namespace tc {

// D[64 x 64] (+)= A[64 x 16] (fp16, registers) * B[16 x 64] (fp16, shared memory, K-major)
__device__ __forceinline__ void wgmma_rs_n64(float* d, const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// Key tile [kt, kt + 64): S = Q K^T, mask keys outside [kmin[h], kmax[h]] of this thread's two rows h, fold the tile into the running
// row max m, partial row sum l (this thread's columns; reduced over the quad by attn_tc_row_inv) and output o.  Returns after the
// tile's MMAs have retired: the K / V stage may be released.
__device__ __forceinline__ void attn_tc_tile(float* o, float* m, float* l, uint64_t dqh, uint64_t dql, uint64_t dkh, uint64_t dkl,
                                             uint64_t dvh, uint64_t dvl, int kt, const int* kmax, const int* kmin, int lane) {
  float sc[32];
  wgmma_fence();
  wgmma_chunk<2, true>(sc, dqh, dkh, 0u);                      // S = Qh Kh^T + Ql Kh^T + Qh Kl^T
  wgmma_chunk<2, true>(sc, dql, dkh, 1u);
  wgmma_chunk<2, true>(sc, dqh, dkl, 1u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs<32>(sc);
  // mask + row max (element 4j + e: row h = e >> 1, key kt + 8j + 2 (lane % 4) + (e & 1))
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < 8; j++) {
#pragma unroll
    for (int e = 0; e < 4; e++) {
      const int h = e >> 1, kk = kt + 8 * j + 2 * (lane & 3) + (e & 1);
      if (kk > kmax[h] || kk < kmin[h]) sc[4 * j + e] = -INFINITY;
      mx[h] = fmaxf(mx[h], sc[4 * j + e]);
    }
  }
  float alpha[2], mn[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    mn[h] = fmaxf(m[h], mx[h]);
    alpha[h] = (mn[h] == -INFINITY) ? 1.f : exp2f(m[h] - mn[h]);     // m = -inf -> 0 (o is 0 anyway)
    m[h] = mn[h];
  }
  float rs[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 32; j++) {
    const int h = (j >> 1) & 1;
    const float pv = (mn[h] == -INFINITY) ? 0.f : exp2f(sc[j] - mn[h]);
    sc[j] = pv;
    rs[h] += pv;
  }
  l[0] = l[0] * alpha[0] + rs[0];
  l[1] = l[1] * alpha[1] + rs[1];
  // O_tile = Ph Vh + Pl Vh + Ph Vl   (A = P [64 x 64 keys] from registers, B = V^T tile [64 dims x 64 keys]) into a fresh accumulator,
  // folded into O by fp32 FMAs below: accumulating onto the running O inside the MMA would round each tile's contribution against
  // O's magnitude, and the result would then depend on where the key tiles start (a span decode vs the one-shot decode).
  uint32_t ph[4][4], pl[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; kk++) {
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const float a = sc[8 * kk + 2 * r], b = sc[8 * kk + 2 * r + 1];
      const __half2 hh = __floats2half2_rn(a, b);
      const float2 hf = __half22float2(hh);
      ph[kk][r] = *reinterpret_cast<const uint32_t*>(&hh);
      pl[kk][r] = pack_half2(a - hf.x, b - hf.y);
    }
  }
  float pv[32];
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; kk++) wgmma_rs_n64(pv, ph[kk], dvh + 2 * kk, kk ? 1u : 0u);
#pragma unroll
  for (int kk = 0; kk < 4; kk++) wgmma_rs_n64(pv, pl[kk], dvh + 2 * kk, 1u);
#pragma unroll
  for (int kk = 0; kk < 4; kk++) wgmma_rs_n64(pv, ph[kk], dvl + 2 * kk, 1u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs<32>(pv);
#pragma unroll
  for (int j = 0; j < 32; j++) o[j] = fmaf(o[j], alpha[(j >> 1) & 1], pv[j]);
}

// 1 / (row sum) of this thread's two rows after the last tile (0 for a row that saw no key)
__device__ __forceinline__ void attn_tc_row_inv(float* l, float* inv) {
#pragma unroll
  for (int h = 0; h < 2; h++) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    inv[h] = l[h] > 0.f ? 1.f / l[h] : 0.f;
  }
}

}  // namespace tc
