// Causal GQA prefill attention against the fp32 KV cache on the Hopper tensor cores (include/b200audio.h: b2a_attn_prefill):
// the talker's self-attention (talker.py:288-312) for prompts of 64 rows and more -- the in-context voice-cloning prompt holds one row
// per reference codec frame, so it runs to hundreds of rows, where b2a_attn_decode (one CTA per query row, each re-reading every
// earlier K / V row from the cache) moves ~Hq S^2 / 2 KB per layer.  Here each K / V row is read once per 64-query tile per KV head.
//
// One CTA = 64 query rows x one KV head x one batch row, 256 threads = two consumer warpgroups, one per query head of the GQA pair
// (Hq = 2 Hkv): both consume the same K / V tile in shared memory.  Per key tile of 64:
//   load     all threads read the tile's fp32 cache rows and write fp16 hi / lo planes (hi = fp16(v), lo = fp16(v - hi)) into
//            128B-swizzled shared memory: K as [keys][dims] (two 64-dim chunks), V transposed as [dims][keys]; the next tile is loaded
//            while the tensor cores compute this tile's scores (two stages)
//   S = Q K^T   wgmma M64 x N64 x K16, 3 products (hi*hi, lo*hi, hi*lo) for fp32-grade scores; Q is pre-scaled by scale * log2 e
//   softmax  online, on the accumulator fragments (exp2)
//   O += P V    wgmma M64 x N128 with A = P from registers (hi / lo), B = the V^T tile, 3 products, accumulated onto O after O *= alpha
// Keys are visited in ascending tile order with no split across CTAs, so the result is bit-reproducible.  Tiles entirely before
// kv_start[b] or after the CTA's last query are never loaded; keys outside [kv_start[b], base + s] are masked per element.
#include "common.cuh"
#include "tc_common.cuh"

using namespace tc;

namespace {

constexpr int BM = 64, BN = 64, HD = 128, THREADS = 256;

// smem (1024-aligned): Q [head 2][plane 2][dim chunk 2] x 8K | [stage 2] x { K [plane 2][dim chunk 2] x 8K | V^T [plane 2] x 16K }
constexpr int Q_TILE = 8192, OFF_KV = 8 * Q_TILE, OFF_V = 32768, KV_STAGE = 65536, SMEM_BYTES = OFF_KV + 2 * KV_STAGE + 1024;

struct PfParams {
  const float* q; int64_t q_bs, q_ss;              // [B, S, Hq*128], normed + rotated
  const float* kc; const float* vc; int64_t c_bs, c_ss;   // caches [B, rows, Hkv*128]
  float* o; int64_t o_bs, o_ss;                    // [B, S, Hq*128]
  int S, Hkv; float qmul;                          // qmul = scale * log2(e)
  const int* base_dev; int base_host; const int* kv_start; int max_k;
  const int* base_rows; const int* slot;           // [B] per-row base (negative query positions: zero output) and cache batch index
};

// D[64 x 128] (+)= A[64 x 16] (fp16, registers) * B[16 x 128] (fp16, shared memory, K-major)
__device__ __forceinline__ void wgmma_rs_n128(float* d, const uint32_t* a, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}

// byte offset of the 16-byte chunk holding columns [8c, 8c + 8) of `row` in a 128B-swizzled tile of 128-byte rows (TMA's SWIZZLE_128B rule)
__device__ __forceinline__ int sw_chunk(int row, int c) { return row * 128 + ((c ^ (row & 7)) << 4); }

// 8 consecutive fp32 values -> their fp16 hi / lo planes as two 16-byte chunks
__device__ __forceinline__ void split8(const float* src, float mul, uint4& hi, uint4& lo) {
  const float4 a = *reinterpret_cast<const float4*>(src), c = *reinterpret_cast<const float4*>(src + 4);
  const float v[8] = {a.x * mul, a.y * mul, a.z * mul, a.w * mul, c.x * mul, c.y * mul, c.z * mul, c.w * mul};
  __align__(16) __half hh[8], ll[8];
#pragma unroll
  for (int j = 0; j < 8; j++) split16(v[j], hh[j], ll[j]);
  hi = *reinterpret_cast<const uint4*>(hh);
  lo = *reinterpret_cast<const uint4*>(ll);
}

// K / V rows [kt, kt + 64) of KV head hk into one stage; rows outside [klo, khi) are zero (never read from the cache).
// Thread t owns key kt + (t & 63) and dim groups (t >> 6) + 4 i: a warp covers 32 keys of one dim group, so the transposed V stores of
// a warp hit 16 distinct words and the K stores fill whole 128-byte wavefronts.
__device__ __forceinline__ void load_kv(uint8_t* st, const PfParams& p, int cb, int hk, int kt, int klo, int khi) {
  const int j = threadIdx.x & 63, key = kt + j;
  const bool ok = key >= klo && key < khi;
  const int64_t row = (int64_t)cb * p.c_bs + (int64_t)key * p.c_ss + (int64_t)hk * HD;
#pragma unroll 2
  for (int i = 0; i < 4; i++) {
    const int c8 = (threadIdx.x >> 6) + 4 * i;                    // dims [8 c8, 8 c8 + 8)
    uint4 kh = make_uint4(0, 0, 0, 0), kl = kh, vh = kh, vl = kh;
    if (ok) {
      split8(p.kc + row + 8 * c8, 1.f, kh, kl);
      split8(p.vc + row + 8 * c8, 1.f, vh, vl);
    }
    const int ch = c8 >> 3, cc = c8 & 7;
    *reinterpret_cast<uint4*>(st + ch * Q_TILE + sw_chunk(j, cc)) = kh;
    *reinterpret_cast<uint4*>(st + 2 * Q_TILE + ch * Q_TILE + sw_chunk(j, cc)) = kl;
    const __half* h = reinterpret_cast<const __half*>(&vh);
    const __half* l = reinterpret_cast<const __half*>(&vl);
#pragma unroll
    for (int e = 0; e < 8; e++) {                                  // V^T: row = dim 8 c8 + e, column = key j
      const int off = sw_chunk(8 * c8 + e, j >> 3) + 2 * (j & 7);
      *reinterpret_cast<__half*>(st + OFF_V + off) = h[e];
      *reinterpret_cast<__half*>(st + OFF_V + 16384 + off) = l[e];
    }
  }
}

__global__ void __launch_bounds__(THREADS, 1) attn_prefill_kernel(const PfParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, w4 = warp & 3;
  const int q0 = blockIdx.x * BM, hk = blockIdx.y, b = blockIdx.z;
  pdl_wait();                                                    // q and the cache rows are the predecessor's output
  const int base = p.base_rows ? p.base_rows[b] : (p.base_dev ? *p.base_dev : p.base_host);
  const int cb = p.slot ? p.slot[b] : b;
  const int klo = p.kv_start ? p.kv_start[b] : 0;
  const int rows = p.S - q0 < BM ? p.S - q0 : BM;
  int khi = base + q0 + rows;                                    // keys [klo, khi) can be seen by some row of this tile (none when
                                                                 // every row is left padding: base + q0 + rows <= 0)
  if (khi > p.max_k) khi = p.max_k;
  const int t_lo = klo / BN, t_hi = (khi + BN - 1) / BN;
  const int nt = khi > klo ? t_hi - t_lo : 0;

  // ---- Q of both heads: [head][plane][chunk] tiles, rows past S zero
  for (int i = threadIdx.x; i < 2 * BM * (HD / 8); i += THREADS) {
    const int c8 = i & 15, r = (i >> 4) & 63, g = i >> 10;
    uint4 hi = make_uint4(0, 0, 0, 0), lo = hi;
    if (r < rows) split8(p.q + (int64_t)b * p.q_bs + (int64_t)(q0 + r) * p.q_ss + (int64_t)(2 * hk + g) * HD + 8 * c8, p.qmul, hi, lo);
    uint8_t* t = smem + (g * 4 + (c8 >> 3)) * Q_TILE + sw_chunk(r, c8 & 7);
    *reinterpret_cast<uint4*>(t) = hi;
    *reinterpret_cast<uint4*>(t + 2 * Q_TILE) = lo;
  }
  if (nt > 0) load_kv(smem + OFF_KV, p, cb, hk, t_lo * BN, klo, khi);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the wgmma operand reads
  __syncthreads();

  int kmax[2];                                                   // last key of this thread's two rows
#pragma unroll
  for (int h = 0; h < 2; h++) {
    kmax[h] = base + q0 + w4 * 16 + (lane >> 2) + 8 * h;
    if (kmax[h] > p.max_k - 1) kmax[h] = p.max_k - 1;
  }
  float o[64];
#pragma unroll
  for (int j = 0; j < 64; j++) o[j] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t sb = smem_u32(smem);
  const uint32_t qt = sb + wg * 4 * Q_TILE;                      // this warpgroup's head: hi c0 | hi c1 | lo c0 | lo c1
  for (int t = 0; t < nt; t++) {
    const int kt = (t_lo + t) * BN, s = t & 1;
    const uint32_t st = sb + OFF_KV + s * KV_STAGE;
    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 2; c++) {                                // S = Qh Kh^T + Ql Kh^T + Qh Kl^T over both 64-dim chunks
      const uint64_t dqh = gmma_desc_sw128(qt + c * Q_TILE), dql = gmma_desc_sw128(qt + (2 + c) * Q_TILE);
      const uint64_t dkh = gmma_desc_sw128(st + c * Q_TILE), dkl = gmma_desc_sw128(st + (2 + c) * Q_TILE);
      wgmma_chunk<2, true>(sc, dqh, dkh, c ? 1u : 0u);
      wgmma_chunk<2, true>(sc, dql, dkh, 1u);
      wgmma_chunk<2, true>(sc, dqh, dkl, 1u);
    }
    wgmma_commit();
    if (t + 1 < nt) load_kv(smem + OFF_KV + (s ^ 1) * KV_STAGE, p, cb, hk, kt + BN, klo, khi);   // overlaps the score MMAs
    wgmma_wait<0>();
    wgmma_fence_regs<32>(sc);
    // mask + row max (element 4j + e: row h = e >> 1, key kt + 8j + 2 (lane % 4) + (e & 1))
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; j++) {
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int h = e >> 1, kk = kt + 8 * j + 2 * (lane & 3) + (e & 1);
        if (kk > kmax[h] || kk < klo) sc[4 * j + e] = -INFINITY;
        mx[h] = fmaxf(mx[h], sc[4 * j + e]);
      }
    }
    float alpha[2], mn[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      mn[h] = fmaxf(m[h], mx[h]);
      alpha[h] = (mn[h] == -INFINITY) ? 1.f : exp2f(m[h] - mn[h]);
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
    l[0] = l[0] * alpha[0] + rs[0];                              // per-thread partial row sums: reduced over the quad at the end
    l[1] = l[1] * alpha[1] + rs[1];
    uint32_t ph[4][4], pl[4][4];                                 // P as the A operand of four K16 steps (the M64 x N64 accumulator layout)
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const float a = sc[8 * kk + 2 * r], c = sc[8 * kk + 2 * r + 1];
        const __half2 hh = __floats2half2_rn(a, c);
        const float2 hf = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(a - hf.x, c - hf.y);
        ph[kk][r] = *reinterpret_cast<const uint32_t*>(&hh);
        pl[kk][r] = *reinterpret_cast<const uint32_t*>(&ll);
      }
    }
#pragma unroll
    for (int j = 0; j < 64; j++) o[j] *= alpha[(j >> 1) & 1];
    const uint64_t dvh = gmma_desc_sw128(st + OFF_V), dvl = gmma_desc_sw128(st + OFF_V + 16384);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; kk++) wgmma_rs_n128(o, ph[kk], dvh + 2 * kk, 1u);
#pragma unroll
    for (int kk = 0; kk < 4; kk++) wgmma_rs_n128(o, pl[kk], dvh + 2 * kk, 1u);
#pragma unroll
    for (int kk = 0; kk < 4; kk++) wgmma_rs_n128(o, ph[kk], dvl + 2 * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<64>(o);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the next stage's stores -> visible to the next MMAs
    __syncthreads();                                             // ... and this stage is free for the load after next
  }
  pdl_launch_dependents();
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    inv[h] = l[h] > 0.f ? 1.f / l[h] : 0.f;
  }
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int r = w4 * 16 + (lane >> 2) + 8 * h;
    if (r < rows) {
      float* dst = p.o + (int64_t)b * p.o_bs + (int64_t)(q0 + r) * p.o_ss + (int64_t)(2 * hk + wg) * HD + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 16; j++)
        *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[4 * j + 2 * h] * inv[h], o[4 * j + 2 * h + 1] * inv[h]);
    }
  }
}

}  // namespace

extern "C" int32_t b2a_attn_prefill(const float* q, int64_t q_bs, int64_t q_ss, const float* k_cache, const float* v_cache,
                                    int64_t c_bs, int64_t c_ss, float* out, int64_t o_bs, int64_t o_ss, int32_t B, int32_t S,
                                    int32_t Hq, int32_t Hkv, int32_t D, float scale, const int32_t* base_dev, int32_t base_host,
                                    const int32_t* kv_start, int32_t max_k, const int32_t* base_rows, const int32_t* slot,
                                    void* stream) {
  B2A_CHECK_ARG(q && k_cache && v_cache && out, "null pointer");
  B2A_CHECK_ARG(D == HD && Hq == 2 * Hkv, "tensor-core prefill attention: head_dim 128, two query heads per KV head");
  B2A_CHECK_ARG(B > 0 && S > 0 && Hkv > 0 && max_k > 0 && c_ss >= (int64_t)Hkv * D, "bad shape");
  B2A_CHECK_ARG(q_ss % 4 == 0 && q_bs % 4 == 0 && ((uintptr_t)q & 15) == 0, "q rows must be 16-byte aligned");
  B2A_CHECK_ARG(c_ss % 4 == 0 && c_bs % 4 == 0 && ((uintptr_t)k_cache & 15) == 0 && ((uintptr_t)v_cache & 15) == 0,
                "cache rows must be 16-byte aligned");
  B2A_CHECK_ARG(o_ss % 2 == 0 && o_bs % 2 == 0 && ((uintptr_t)out & 7) == 0, "out rows must be 8-byte aligned");
  PfParams p{q, q_bs, q_ss, k_cache, v_cache, c_bs, c_ss, out, o_bs, o_ss, S, Hkv, scale * 1.4426950408889634f,
             base_dev, base_host, kv_start, max_k, base_rows, slot};
  B2A_SMEM_OPTIN(attn_prefill_kernel, SMEM_BYTES);
  dim3 grid((unsigned)((S + BM - 1) / BM), (unsigned)Hkv, (unsigned)B);
  b2a_launch_pdl(attn_prefill_kernel, grid, dim3(THREADS), SMEM_BYTES, (cudaStream_t)stream, p);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
