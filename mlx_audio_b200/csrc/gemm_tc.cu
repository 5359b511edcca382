// Tensor-core path for the genuinely dense layers (include/b200audio.h: b2a_prep_bf16, b2a_conv1d_tc).
//
// A stride-1 1-D convolution over channels-last activations is a sum of row-shifted GEMMs:
//     Y[l, n] = sum_tap sum_ci  A[l + shift_tap, ci] * W[tap][n][ci]
// so one wgmma kernel serves every dense conv (and every Linear: one tap, shift 0).  TMA fetches the shifted A tile for each tap
// straight from the activation matrix -- rows outside [0, L) are zero-filled by the TMA unit, which IS the convolution's zero
// padding -- and the weight tile, both into 128B-swizzled shared memory that wgmma consumes through shared-memory descriptors.
// Two consumer warpgroups each own 64 rows of the 128-row tile and keep their fp32 accumulator in registers; after the K loop the
// tile goes through shared memory to an epilogue in which each warp streams 32-row x 32-column chunks as whole row segments and
// fuses bias / activation / LayerScale / residual / scale / accumulate.
//
// Precision: activations are stored as TWO bf16 planes (hi = bf16(a), lo = bf16(a - hi)) written by the
// prologue kernel together with the AdaIN/Snake/LeakyReLU input transform; weights are bf16-exact
// (bf16 checkpoint), so  (hi + lo) * w  reproduces the fp32 product to ~2^-17 while running on the bf16
// tensor pipe (2 MMAs per tile instead of 1).  `planes = 1` drops the lo plane (pure bf16 activations).
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (MMA, then epilogue), warp 8 = TMA producer.  One 128 x BN output
// tile per CTA; BN <= 128 keeps the accumulator at <= 64 registers per thread.
#include "common.cuh"
#include "tc_common.cuh"
#include "tc_epilogue.cuh"
#include <stdlib.h>

using namespace tc;

namespace {

constexpr int TM = 128;            // rows (positions) per CTA tile = two wgmma M64 halves
constexpr int TK = 64;             // bf16 elements per 128-byte swizzle row == K extent of one stage
constexpr int THREADS = 288;
constexpr int BN_MAX = 128;

struct TcParams {
  int B, L, Lout, Cout, cin_pad, taps, planes, wplanes, BN, stages, f16;
  int Mrows, up_s, up_crop, C;     // transposed-conv mode: N = up_s * C, GEMM row m & column (r, co) -> output row m*up_s + r - up_crop
  int shift[32];
  const float* bias; int post_act; float post_p0;
  const float* cscale; int64_t cscale_bs;
  const float* res; int64_t res_bs, res_ld; int res_div;
  float out_scale; int accumulate;
  float* y; int64_t y_bs, y_ld;
  long long* dbg;                 // optional: clock64 stamps from CTA (0,0,0) (b2a_conv1d_tc_debug)
  // optional: the consumer's A operand, split16 of each final value y.  Either bf16 planes [B][Lout][e_ld] of the next GEMM, or (attn.qh
  // != null) the fp16 attention operands of a fused qkv projection: column n = part * a_hs + head * 64 + d, part 0 = Q (times a_qmul),
  // 1 = K, 2 = V (transposed, keys zero-padded to attn.tkp).
  __nv_bfloat16 *e_hi, *e_lo; int64_t e_ld;
  AttnOperands attn; int a_H, a_hs; float a_qmul;
};

// Where this lane's column of the output tile goes as split16 planes (tc::EmitCol).
__device__ __forceinline__ EmitCol emit_col(const TcParams& p, int b, int n) {
  if (p.attn.qh) return emit_col_attn(p.attn, (int64_t)b * p.a_H, p.Lout, p.a_hs, p.a_qmul, n);
  EmitCol c{nullptr, nullptr, 0, 1.f, false};
  if (p.e_hi) {
    const int64_t o = (int64_t)b * p.Lout * p.e_ld + n;
    c.hi = (uint16_t*)p.e_hi + o; c.lo = p.e_lo ? (uint16_t*)p.e_lo + o : nullptr; c.step = p.e_ld;
  }
  return c;
}

// smem: [stages] x { A_hi 16 KB | A_lo 16 KB (planes==2) | W BN*128 B (x wplanes) }, then barriers.  After the K loop the stage
// memory holds the 128 x (BN + 8) fp32 output tile (row stride = 8 mod 32 words: the fragment stores of a quarter-warp hit distinct banks).
template <int NB, bool F16>
__global__ void __launch_bounds__(THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
               const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo, const TcParams p) {
  constexpr int BN = NB * 32;
  constexpr int LD = BN + 8;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int a_bytes = TM * 128, w_bytes = BN * 128;
  const int stage_bytes = a_bytes * p.planes + w_bytes * p.wplanes;
  const size_t ring = (size_t)p.stages * stage_bytes;
  const size_t tile_bytes = (size_t)TM * LD * 4;
  uint64_t* full = (uint64_t*)(smem + (ring > tile_bytes ? ring : tile_bytes));
  uint64_t* empty = full + p.stages;

  const bool dbg = p.dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0;
  if (dbg && threadIdx.x == 0) p.dbg[0] = clock64();
  const int l0 = blockIdx.x * TM, n0 = blockIdx.y * BN, b = blockIdx.z;
  const int kchunks = p.cin_pad / TK;
  const int iters = p.taps * kchunks;

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_lo) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_wlo) : "memory");
    for (int s = 0; s < p.stages; s++) { mbar_init(full + s, 1); mbar_init(empty + s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) p.dbg[1] = clock64();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      // The weights never depend on the preceding kernel: the first ring's weight tiles are in flight before the programmatic
      // dependency wait, and each of those stages' A tiles joins the same transaction count after it.
      const int pre = iters < p.stages ? iters : p.stages;
      for (int it = 0; it < pre; it++) {
        const int tap = it / kchunks, kc = it % kchunks;
        uint8_t* st = smem + (size_t)it * stage_bytes;
        mbar_expect_tx(full + it, (uint32_t)stage_bytes);
        tma_load_2d(st + (size_t)a_bytes * p.planes, &map_w, full + it, kc * TK, tap * p.Cout + n0);
        if (p.wplanes == 2) tma_load_2d(st + (size_t)a_bytes * p.planes + w_bytes, &map_wlo, full + it, kc * TK, tap * p.Cout + n0);
      }
      pdl_wait();
      for (int it = 0; it < iters; it++) {
        const int s = it % p.stages, ph = (it / p.stages) & 1;
        const int tap = it / kchunks, kc = it % kchunks;
        uint8_t* st = smem + (size_t)s * stage_bytes;
        if (it >= pre) {
          mbar_wait(empty + s, ph ^ 1);
          mbar_expect_tx(full + s, (uint32_t)stage_bytes);
          tma_load_2d(st + (size_t)a_bytes * p.planes, &map_w, full + s, kc * TK, tap * p.Cout + n0);
          if (p.wplanes == 2) tma_load_2d(st + (size_t)a_bytes * p.planes + w_bytes, &map_wlo, full + s, kc * TK, tap * p.Cout + n0);
        }
        tma_load_3d(st, &map_hi, full + s, kc * TK, l0 + p.shift[tap], b);
        if (p.planes == 2) tma_load_3d(st + a_bytes, &map_lo, full + s, kc * TK, l0 + p.shift[tap], b);
      }
    }
    return;
  }
  pdl_wait();                                              // the epilogue reads res / y and writes y: after the predecessor

  // ===== consumer warpgroup wg: rows [64 wg, 64 wg + 64) of the tile =====
  const int wg = warp >> 2;
  float acc[NB * 16];
  {
    const bool two_a = p.planes == 2, two_w = p.wplanes == 2;
    int prev = -1;
    for (int it = 0; it < iters; it++) {
      const int s = it % p.stages;
      mbar_wait(full + s, (it / p.stages) & 1);
      if (dbg && threadIdx.x == 0 && it == 0) p.dbg[2] = clock64();
      if (dbg && threadIdx.x == 0 && it == iters - 1) p.dbg[3] = clock64();
      const uint32_t st = smem_u32(smem + (size_t)s * stage_bytes);
      // products kept: a_hi*w_hi, a_lo*w_hi, and (fp32 checkpoints: weights split too) a_hi*w_lo; a_lo*w_lo ~ 2^-17*2^-9 is dropped
      const uint64_t ad = gmma_desc_sw128(st + wg * 64 * 128), wd = gmma_desc_sw128(st + a_bytes * p.planes);
      wgmma_fence();
      wgmma_chunk<NB, F16>(acc, ad, wd, it != 0);
      if (two_a) wgmma_chunk<NB, F16>(acc, gmma_desc_sw128(st + a_bytes + wg * 64 * 128), wd, 1u);
      if (two_w) wgmma_chunk<NB, F16>(acc, ad, gmma_desc_sw128(st + a_bytes * p.planes + w_bytes), 1u);
      wgmma_commit();
      wgmma_wait<1>();                                      // the previous stage's MMAs have retired: hand it back to the producer
      wgmma_fence_regs<NB * 16>(acc);
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty + prev);
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_regs<NB * 16>(acc);
  }
  pdl_launch_dependents();
  // both warpgroups are done reading the operand ring (and every TMA write to it has landed): it becomes the output tile
  bar_sync(1, 256);
  float* tile = reinterpret_cast<float*>(smem);
  store_acc<NB>(acc, tile, LD, wg * 64);
  bar_sync(1, 256);
  if (dbg && threadIdx.x == 0) p.dbg[4] = clock64();

  // ===== epilogue: warp w streams (32-row quarter, 32-column chunk) pairs w, w + 8, ... =====
  const int mul = p.up_s ? p.up_s : 1;
  for (int pair = warp; pair < 4 * NB; pair += 8) {
    const int quarter = pair & 3, c0 = (pair >> 2) * 32;
    const float* stage = tile + (size_t)(quarter * 32) * LD + c0;
    const int mrow0 = l0 + quarter * 32;
    if (mrow0 >= p.Mrows) continue;
    const int n = n0 + c0 + lane;                          // GEMM column of this lane for every row below
    const int ph = p.up_s ? n / p.C : 0;                   // up-sampling phase (uniform over the 32-column chunk)
    const int co = n - ph * p.C;                           // output channel
    const int add = p.up_s ? ph - p.up_crop : 0;
    const float bias = p.bias ? __ldg(p.bias + co) : 0.f;
    const float cs = p.cscale ? __ldg(p.cscale + (int64_t)b * p.cscale_bs + co) : 1.f;
    float* ycol = p.y + (int64_t)b * p.y_bs + co;
    const float* rcol = p.res ? p.res + (int64_t)b * p.res_bs + co : nullptr;
    // Valid rows form a contiguous range [i_lo, i_hi) of the 32 (row = row0 + i*mul is monotonic); full chunks take the
    // predicate-free path with every residual / previous-output load of the chunk in flight together.
    const int row0 = mrow0 * mul + add;
    const int mvalid = min(32, p.Mrows - mrow0);
    int i_lo = 0, i_hi = mvalid;
    if (row0 < 0) i_lo = (-row0 + mul - 1) / mul;
    if (row0 + (mvalid - 1) * mul >= p.Lout) i_hi = p.Lout > row0 ? (p.Lout - row0 + mul - 1) / mul : 0;
    const int64_t ystride = (int64_t)mul * p.y_ld;
    float* yp = ycol + (int64_t)row0 * p.y_ld;
    const bool half_res = p.res_div == 2;                  // nearest x2 shortcut (istftnet.py:838-850); only with mul == 1
    const int odd = row0 & 1;
    const float* rp = rcol ? rcol + (int64_t)(half_res ? (row0 >> 1) : row0) * p.res_ld : nullptr;
    const int64_t rstride = (int64_t)mul * p.res_ld;
    const float osc = p.out_scale;
    const EmitCol ec = emit_col(p, b, n);                  // up-sampling mode never emits (host check), so row = row0 + i below
    if (i_lo == 0 && i_hi == 32) {
      float rr[32];
      if (rp) {
        if (!half_res) {
#pragma unroll
          for (int i = 0; i < 32; i++) rr[i] = __ldg(rp + i * rstride);
        } else {
#pragma unroll
          for (int i = 0; i < 32; i++) rr[i] = __ldg(rp + (int64_t)((i + odd) >> 1) * p.res_ld);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 32; i++) rr[i] = 0.f;
      }
      if (p.accumulate) {
        float oo[32];
#pragma unroll
        for (int i = 0; i < 32; i++) oo[i] = yp[i * ystride];
#pragma unroll
        for (int i = 0; i < 32; i++) rr[i] = rr[i] * osc + oo[i];
      } else {
#pragma unroll
        for (int i = 0; i < 32; i++) rr[i] *= osc;
      }
      const float cso = cs * osc;
      if (p.post_act) {
#pragma unroll
        for (int i = 0; i < 32; i++) {
          const float v = epilogue_value(stage[i * LD + lane], bias, p.post_act, p.post_p0, cso, rr[i]);
          yp[i * ystride] = v;
          if (ec.hi) emit_store(ec, row0 + i, v);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 32; i++) {
          const float v = epilogue_value(stage[i * LD + lane], bias, 0, 0.f, cso, rr[i]);
          yp[i * ystride] = v;
          if (ec.hi) emit_store(ec, row0 + i, v);
        }
      }
    } else {
      for (int i = i_lo; i < i_hi; i++) {                  // ragged edge tiles: plain loop
        const int row = row0 + i * mul;
        float t = stage[i * LD + lane] + bias;
        if (p.post_act) t = act_noinline(t, p.post_act, p.post_p0);
        float rv = rcol ? __ldg(rcol + (int64_t)(half_res ? (row >> 1) : row) * p.res_ld) : 0.f;
        float o = p.accumulate ? ycol[(int64_t)row * p.y_ld] : 0.f;
        const float v = (t * cs + rv) * osc + o;
        ycol[(int64_t)row * p.y_ld] = v;
        if (ec.hi) emit_store(ec, row, v);
      }
      // transposed V: the zero keys that pad Lout to attn.tkp (< 8 rows past the last valid one, so inside this ragged chunk)
      if (ec.hi && ec.step == 1)
        for (int64_t row = p.Lout; row < p.attn.tkp; row++) { ec.hi[row] = 0; ec.lo[row] = 0; }
    }
  }
  if (dbg && warp == 0 && lane == 0) p.dbg[5] = clock64();
}

// ---- prologue: fp32 activations -> (hi, lo) bf16 planes with the fused input transform; pad channels are zeroed
// 8 channels per thread: 2 x 16-byte reads, one 16-byte write per plane
// ACT >= 0: the activation is a compile-time constant (no per-element switch, a third of the code: the generic instantiation was
// instruction-cache- and branch-bound); ACT = -1: runtime `act`.
template <typename T16, int ACT>
__global__ void prep_bf16_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int B, int L, int C, int cpad,
                                 const float* __restrict__ scale, const float* __restrict__ shift, int act, float p0,
                                 const float* __restrict__ a, const float* __restrict__ bb, T16* __restrict__ hi,
                                 T16* __restrict__ lo) {
  const int cp8 = cpad / 8;
  const int64_t total = (int64_t)B * L * cp8;
  const bool vec = (x_ld % 4 == 0) && (x_bs % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  // Measured alternatives that were SLOWER than this plain grid-stride loop (kept out): a channel group pinned per thread with the
  // constants in registers and no divisions (Whisper prep 5.0 -> 7.7 ms), and two index slots per iteration with both loads in
  // flight (vocoder prep 24 -> 30 ms: the extra registers cost more occupancy than the second load buys).
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cp8) * 8;
    const int64_t r = idx / cp8;
    const int l = (int)(r % L), b = (int)(r / L);
    const float* xp = x + (int64_t)b * x_bs + (int64_t)l * x_ld + c;
    float v[8];
    if (vec && c + 8 <= C) {
      float4 t0 = __ldg(reinterpret_cast<const float4*>(xp)), t1 = __ldg(reinterpret_cast<const float4*>(xp) + 1);
      v[0] = t0.x; v[1] = t0.y; v[2] = t0.z; v[3] = t0.w; v[4] = t1.x; v[5] = t1.y; v[6] = t1.z; v[7] = t1.w;
    } else {
#pragma unroll
      for (int q = 0; q < 8; q++) v[q] = (c + q < C) ? __ldg(xp + q) : 0.f;
    }
    __align__(16) T16 h[8];
    __align__(16) T16 lw[8];
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int cc = c + q;
      float t = 0.f;
      if (cc < C) {
        t = v[q];
        if (scale) t = fmaf(t, __ldg(scale + (int64_t)b * C + cc), __ldg(shift + (int64_t)b * C + cc));
        if constexpr (ACT == B2A_ACT_SNAKE) { const float sn = b2a_sin(__ldg(a + cc) * t); t = fmaf(__ldg(bb + cc), sn * sn, t); }
        else if constexpr (ACT == B2A_ACT_ELU) t = t > 0.f ? t : expm1f(t);
        else if constexpr (ACT == B2A_ACT_LRELU) t = t > 0.f ? t : t * p0;
        else if constexpr (ACT == 0) { }
        else if (act) t = b2a_act(t, act, p0, a ? __ldg(a + cc) : 1.f, bb ? __ldg(bb + cc) : 1.f);
      }
      split16(t, h[q], lw[q]);
    }
    *reinterpret_cast<uint4*>(hi + r * cpad + c) = *reinterpret_cast<uint4*>(h);
    if (lo) *reinterpret_cast<uint4*>(lo + r * cpad + c) = *reinterpret_cast<uint4*>(lw);
  }
}

long long* g_dbg = nullptr;
thread_local int32_t g_last_cfg[5] = {0, 0, 0, 0, 0};   // BN, grid x / y / z, stages of this host thread's last launch

}  // namespace

/* debug aid: device buffer of 8 int64 that the next b2a_conv1d_tc launches stamp with clock64() at their phase boundaries */
extern "C" int32_t b2a_conv1d_tc_debug(void* dbg8) { g_dbg = (long long*)dbg8; return B2A_OK; }

/* the tile the dispatch rule chose for the last launch, so that tests can assert which kernel variant they exercised */
extern "C" int32_t b2a_conv1d_tc_last_config(int32_t* out5) {
  B2A_CHECK_ARG(out5, "null pointer");
  for (int i = 0; i < 5; i++) out5[i] = g_last_cfg[i];
  return B2A_OK;
}

extern "C" int32_t b2a_prep_bf16(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C, int32_t cpad,
                                 const float* scale, const float* shift, int32_t act, float p0, const float* a, const float* b,
                                 void* hi, void* lo, int32_t f16, void* stream) {
  B2A_CHECK_ARG(x && hi && B > 0 && L > 0 && C > 0 && cpad >= C && cpad % 64 == 0, "bad pointers/shape (cpad must be a multiple of 64)");
  B2A_CHECK_ARG((scale == nullptr) == (shift == nullptr), "scale and shift come together");
  int64_t total = (int64_t)B * L * (cpad / 8);
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 16) blocks = 132 * 16;
#define B2A_PREP_LAUNCH(T, A) prep_bf16_kernel<T, A><<<blocks, 256, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, B, L, C, cpad, scale, shift, act, p0, a, b, (T*)hi, (T*)lo)
  if (f16) {
    if (act == 0) B2A_PREP_LAUNCH(__half, 0); else B2A_PREP_LAUNCH(__half, -1);
  } else if (act == 0) B2A_PREP_LAUNCH(__nv_bfloat16, 0);
  else if (act == B2A_ACT_SNAKE && a && b) B2A_PREP_LAUNCH(__nv_bfloat16, B2A_ACT_SNAKE);
  else if (act == B2A_ACT_ELU) B2A_PREP_LAUNCH(__nv_bfloat16, B2A_ACT_ELU);
  else if (act == B2A_ACT_LRELU) B2A_PREP_LAUNCH(__nv_bfloat16, B2A_ACT_LRELU);
  else B2A_PREP_LAUNCH(__nv_bfloat16, -1);
#undef B2A_PREP_LAUNCH
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_conv1d_tc(const void* a_hi, const void* a_lo, int32_t f16, int32_t B, int32_t L, int32_t cin_pad, const void* w_bf16,
                                 const void* w_lo,
                                 int32_t taps, const int32_t* shifts_host, int32_t Cout, int32_t Lout, const float* bias,
                                 int32_t post_act, float post_p0, const float* cscale, int64_t cscale_bs, const float* res,
                                 int64_t res_bs, int64_t res_ld, int32_t res_div, float out_scale, int32_t accumulate, float* y,
                                 int64_t y_bs, int64_t y_ld, int32_t up_stride, int32_t up_crop,
                                 void* emit_hi, void* emit_lo, int64_t emit_ld, void* attn_ws, int32_t attn_heads, float attn_scale,
                                 void* stream) {
  B2A_CHECK_ARG(a_hi && w_bf16 && y && shifts_host, "null pointer");
  B2A_CHECK_ARG(!(emit_hi && attn_ws) && (!(emit_hi || attn_ws) || up_stride == 0), "one emitted operand at most, not in transposed mode");
  B2A_CHECK_ARG(!emit_hi || (emit_ld >= Cout && emit_ld % 8 == 0), "emitted planes: row stride >= Cout, a multiple of 8");
  B2A_CHECK_ARG(!attn_ws || (attn_heads > 0 && Cout == 3 * 64 * attn_heads), "attention operands: Cout = 3 * 64 * heads (q | k | v)");
  B2A_CHECK_ARG(up_stride >= 0 && up_crop >= 0 && (up_stride == 0 || (Cout % up_stride == 0 && (Cout / up_stride) % 32 == 0)),
                "transposed mode: Cout = up_stride * C with C a multiple of 32");
  B2A_CHECK_ARG(B > 0 && L > 0 && Lout > 0 && taps > 0 && taps <= 32 && cin_pad % 64 == 0 && (res_div == 1 || res_div == 2), "bad shape (res_div must be 1 or 2)");
  B2A_CHECK_ARG(Cout % 32 == 0 && y_ld % 4 == 0 && (res == nullptr || res_ld % 4 == 0), "Cout must be a multiple of 32; row strides multiples of 4");
  TcParams p;
  p.f16 = f16 ? 1 : 0;
  p.wplanes = w_lo ? 2 : 1;
  p.up_s = up_stride; p.up_crop = up_crop; p.C = up_stride ? Cout / up_stride : Cout;
  // GEMM rows: in polyphase mode every row m whose phases m * up_stride + r - up_crop reach an output row below Lout.  Rows past
  // L + taps - 1 read only the zero padding (TMA fills rows past L with zeros), so output rows past the scatter get the epilogue alone.
  p.Mrows = up_stride ? (L + taps - 1 > cdiv(Lout + up_crop, up_stride) ? L + taps - 1 : cdiv(Lout + up_crop, up_stride)) : Lout;
  p.B = B; p.L = L; p.Lout = Lout; p.Cout = Cout; p.cin_pad = cin_pad; p.taps = taps; p.planes = a_lo ? 2 : 1;
  // N tile = the widest divisor of Cout that is a multiple of 32 (the epilogue's chunk) and <= 128 (the register accumulator).  96 matters:
  // the Qwen3 vocoder's 96-, 192- and 384-channel blocks would otherwise run as 32-/64-wide tiles and re-read A three times.
  p.BN = 32;
  for (int bn = BN_MAX; bn >= 32; bn -= 32) if (Cout % bn == 0) { p.BN = bn; break; }
  // Few-row GEMMs (ALBERT at T = 130: 2 row tiles) leave most SMs idle at that width and every CTA runs the whole K loop alone:
  // when the grid covers under half the SMs, take the widest tile whose grid still reaches the SM count, else the narrowest (32).
  // Each output element still accumulates its whole K range in the same order inside one CTA.
  static const int nsm = [] { const int n = b2a_device_sm_count(); return n > 0 ? n : 132; }();
  const int64_t row_tiles = (int64_t)cdiv(p.Mrows, TM) * B;
  if (row_tiles * (Cout / p.BN) * 2 < nsm) {
    int bn = 32;
    for (int c = p.BN; c > 32; c -= 32) if (Cout % c == 0 && row_tiles * (Cout / c) >= nsm) { bn = c; break; }
    p.BN = bn;
  }
  for (int i = 0; i < taps; i++) p.shift[i] = shifts_host[i];
  p.e_hi = (__nv_bfloat16*)emit_hi; p.e_lo = (__nv_bfloat16*)emit_lo; p.e_ld = emit_ld;
  p.attn = attn_ws ? attn_operands(attn_ws, (int64_t)B * attn_heads, Lout, Lout) : AttnOperands{};
  p.a_H = attn_heads; p.a_hs = attn_heads * 64;
  p.a_qmul = attn_scale * 1.4426950408889634f;            // as b2a_attention_tc pre-scales Q: exp2 is its only transcendental
  p.bias = bias; p.post_act = post_act; p.post_p0 = post_p0; p.cscale = cscale; p.cscale_bs = cscale_bs;
  p.res = res; p.res_bs = res_bs; p.res_ld = res_ld; p.res_div = res_div; p.out_scale = out_scale; p.accumulate = accumulate;
  p.y = y; p.y_bs = y_bs; p.y_ld = y_ld;
  p.dbg = g_dbg;
  const int stage_bytes = TM * 128 * p.planes + p.BN * 128 * p.wplanes;
  const size_t tile_bytes = (size_t)TM * (p.BN + 8) * 4;
  // One CTA per SM (the epilogue's register arrays put a CTA at ~125 registers per thread): as many operand stages as fit.
  p.stages = (200 * 1024) / stage_bytes; if (p.stages > 6) p.stages = 6; if (p.stages < 2) p.stages = 2;
  const size_t ring = (size_t)p.stages * stage_bytes;
  const size_t smem = (ring > tile_bytes ? ring : tile_bytes) + 1024 /*align slack*/ + 2 * p.stages * 8 + 64;

  CUtensorMap mh, ml, mw, mwl;
  uint64_t adims[3] = {(uint64_t)cin_pad, (uint64_t)L, (uint64_t)B};
  uint64_t astr[2] = {(uint64_t)cin_pad * 2, (uint64_t)cin_pad * 2 * (uint64_t)L};
  uint32_t abox[3] = {TK, TM, 1};
  int e = b2a_tmap16(&mh, a_hi, 3, adims, astr, abox, p.f16);
  if (!e) e = b2a_tmap16(&ml, a_lo ? a_lo : a_hi, 3, adims, astr, abox, p.f16);
  uint64_t wdims[2] = {(uint64_t)cin_pad, (uint64_t)taps * Cout};
  uint64_t wstr[1] = {(uint64_t)cin_pad * 2};
  uint32_t wbox[2] = {TK, (uint32_t)p.BN};
  if (!e) e = b2a_tmap16(&mw, w_bf16, 2, wdims, wstr, wbox, p.f16);
  if (!e) e = b2a_tmap16(&mwl, w_lo ? w_lo : w_bf16, 2, wdims, wstr, wbox, p.f16);
  if (e) { b2a_set_error("b2a_conv1d_tc: cuTensorMapEncodeTiled failed (%d)", e); return B2A_E_CUDA; }

  typedef void (*KernelFn)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const TcParams);
  static const KernelFn kernels[2][4] = {
      {conv_tc_kernel<1, false>, conv_tc_kernel<2, false>, conv_tc_kernel<3, false>, conv_tc_kernel<4, false>},
      {conv_tc_kernel<1, true>, conv_tc_kernel<2, true>, conv_tc_kernel<3, true>, conv_tc_kernel<4, true>}};
  const KernelFn kern = kernels[p.f16][p.BN / 32 - 1];
  B2A_SMEM_OPTIN(kern, 227 * 1024);
  dim3 grid(cdiv(p.Mrows, TM), Cout / p.BN, B);
  if (b2a_launch_pdl(kern, grid, dim3(THREADS), smem, (cudaStream_t)stream, mh, ml, mw, mwl, p) != cudaSuccess) {
    b2a_set_error("b2a_conv1d_tc: %s", cudaGetErrorString(cudaGetLastError()));
    return B2A_E_CUDA;
  }
  g_last_cfg[0] = p.BN; g_last_cfg[1] = (int32_t)grid.x; g_last_cfg[2] = (int32_t)grid.y; g_last_cfg[3] = (int32_t)grid.z; g_last_cfg[4] = p.stages;
  return B2A_OK;
}
