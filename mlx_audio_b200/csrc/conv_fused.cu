// Fused dense conv1d / linear / polyphase transposed conv for sm_90a (include/b200audio.h: b2a_conv1d_fused).
//
// Round 1 ran every tensor-core layer as FOUR launches: InstanceNorm statistics (2 kernels), a prologue pass that re-read the fp32
// activations, applied AdaIN / Snake / LeakyReLU and wrote them back to HBM as bf16 (hi, lo) planes, and the tensor-core GEMM that
// read those planes once per tap.  This kernel does all of it in ONE launch and reads the activations ONCE:
//
//   worker warps (8)     (2 warpgroups; also run the epilogue below)
//                        fp32 activations (global, coalesced float4) -> [AdaIN scale/shift from the producer's (sum, sumsq)] ->
//                        Snake / LeakyReLU / ELU -> bf16 (or fp16) hi + lo planes written straight into the 128B-swizzled shared-memory
//                        tile the MMA consumes.  One (128 + span)-row tile per 64-channel K chunk serves EVERY tap: tap t multiplies
//                        rows [shift_t - shift_min, +128) of it through a row-shifted wgmma descriptor.  Rows outside [0, L) are
//                        written as zeros = the convolution's zero padding.  Double-buffered.
//   TMA warp             (alone in its warpgroup) weight tiles [BN x 64] per (K chunk, tap) through a ring of mbarrier stages.
//   MMA warpgroups (2)   wgmma M64 x BN x K16 each (the two 64-row halves of the tile), fp32 accumulator in registers, one
//                        asynchronous wgmma group per tap step; a finished tile is stored to a shared-memory output tile while the
//                        registers already take the next one.
//   epilogue             output tile rows -> coalesced rows; bias / activation / channel scale / residual /
//                        out_scale / accumulate / polyphase scatter fused; per-channel (sum, sumsq) of what was written is reduced in
//                        shared memory and added to a float64 accumulator in global memory -- the NEXT layer's AdaIN statistics.
//
// Grouped launches: up to 4 independent problems (e.g. the three parallel AdaINResBlock1 branches of a generator stage, kernel sizes
// 3 / 7 / 11) share one persistent grid; tiles are ordered heaviest problem first.  Small-M problems can split K across CTAs
// (partial accumulators in a global workspace, the last CTA to arrive reduces and runs the epilogue).
#include "common.cuh"
#include "tc_common.cuh"
#include <stdlib.h>

using namespace tc;

namespace {

constexpr int TM = 128;
constexpr int TK = 64;

constexpr int MAXG = B2A_CONVF_MAX_PROBLEMS;
// Roles sit on warpgroup boundaries because setmaxnreg re-allocates registers per warpgroup:
//   warpgroups 0, 1  MMA            96 registers (the launch allocation: 64 accumulator + issue state)
//   warpgroup 2      weight producer (warp 8, one lane; warps 9..11 idle)   32 registers (setmaxnreg.dec)
//   warpgroups 3, 4  workers        128 registers (setmaxnreg.inc): A-chunk conversion AND epilogues (see the kernel's worker section)
// 640 threads launch at 96 registers each (61 440 of the SM's 64 K); the producer's release of 64 x 128 covers the workers' 2 x 32 x 128.
constexpr int NWORK = 8;
constexpr int NSUB = NWORK / 4;                // workers per 32-row quarter: each takes every NSUB-th 32-column chunk
constexpr int WG_PROD = 2;
constexpr int W_PROD = WG_PROD * 4;            // the producer warp
constexpr int W_WORK0 = 12;                    // first worker warp (warpgroup 3)
constexpr int THREADS = (W_WORK0 + NWORK) * 32;           // 640
constexpr int REG_LAUNCH = 96;                 // 65536 / THREADS, rounded down to the allocation granule of 8
constexpr int REG_MMA = 96, REG_PROD = 32, REG_WORK = 128;    // per-thread registers after re-allocation
static_assert(THREADS % 128 == 0 && W_WORK0 % 4 == 0, "roles must sit on warpgroup boundaries");
static_assert(2 * REG_MMA + REG_PROD + 2 * REG_WORK <= 5 * REG_LAUNCH, "the re-allocated registers must fit in the launch allocation");

// Re-allocate this warpgroup's registers to R per thread (all 128 threads execute it).
template <int R> __device__ __forceinline__ void set_regs() {
  if constexpr (R < REG_LAUNCH) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
  else if constexpr (R > REG_LAUNCH) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
constexpr int RSTRIDE = NWORK * 32 / 16;                  // rows between a worker thread's consecutive A-tile rows (16 float4 slots per 64-channel row)
constexpr int SACC = 4 * 2 * 128 * 4;                     // per-tile (sum, sumsq) partials: [32-row quarter][which][column <= 128]
constexpr int CT_MAX = 1280;                              // channels of the per-CTA (scale, shift) table of the input transform
constexpr int CTAB = 2 * CT_MAX * 4;

struct FProb {
  const float* x; const float* x1; const float* x2; int64_t x_bs, x_ld; float in_scale;
  int B, L, Cin, cin_pad;
  int pre_mode;                                // 0 none, 1 scale/shift [B,Cin], 2 statistics (sum, sumsq) [B,Cin,2] (+ gamma|beta [B,2Cin])
  const float* pre_scale; const float* pre_shift;
  const long long* pre_stats; const float* pre_gb; int64_t pre_gb_bs; float pre_eps, pre_invL;
  int pre_act; float pre_p0; const float* pre_a; const float* pre_b;
  int taps, wplanes, BN, ntn, ntm, Ntot, R, shift_min, ksplit, kper;
  int shift[32];
  int Lout, Mrows, up_s, up_crop, C;
  const float* bias; int post_act; float post_p0; const float* cscale; int64_t cscale_bs;
  const float* res; int64_t res_bs, res_ld; int res_div; float out_scale; int accumulate;
  float* y; int64_t y_bs, y_ld;
  long long* stats_out;
  float* ws; int* counters;                    // split-K workspace [tile][ksplit][128*BN] and arrival counters [tile]
  int tile_begin;
};

struct FParams {
  int G, ntiles, planes, f16, wst, w_stage, a_plane, acc_ld;     // acc_ld: floats per row of the shared-memory output tile
  unsigned long long* dbg;                     // optional [gridDim][32] globaltimer stamps (b2a_conv1d_fused_debug)
  int dbg_flags;                               // experiments (env B2A_FUSED_DBGFLAGS): 1 = converter skips the global loads, 2 = skips the smem stores,
                                               // 4 = skips fence.proxy.async, 16 = workers skip the conversion, 32 = skip the epilogue body;
                                               // results are then garbage -- timing only
  FProb pr[MAXG];
};
// dynamic shared memory a launch may take: the kernel keeps a static shared copy of FParams beside it
constexpr size_t DYN_SMEM_MAX = (size_t)227 * 1024 - ((sizeof(FParams) + 1023) & ~(size_t)1023);

struct TileRef { int g, b, mt, nt, ks; };

// Tile order: the tiles of the heaviest problem first.
__device__ __forceinline__ TileRef decode_tile(const FParams& p, int tile) {
  int g = 0;
#pragma unroll
  for (int i = 1; i < MAXG; i++) if (i < p.G && tile >= p.pr[i].tile_begin) g = i;
  int local = tile - p.pr[g].tile_begin;
  const FProb& P = p.pr[g];
  TileRef t;
  t.g = g;
  t.ks = local % P.ksplit; local /= P.ksplit;
  t.nt = local % P.ntn; local /= P.ntn;
  t.mt = local % P.ntm; t.b = local / P.ntm;
  return t;
}

// tc::split16 of two adjacent channels a (low half) and b (high half) with packed conversions: bit-identical to two scalar calls
template <typename T16> __device__ __forceinline__ void split16x2(float a, float b, uint32_t& hi, uint32_t& lo);
template <> __device__ __forceinline__ void split16x2<__nv_bfloat16>(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - __low2float(h), b - __high2float(h));
  hi = *reinterpret_cast<const uint32_t*>(&h); lo = *reinterpret_cast<const uint32_t*>(&l);
}
template <> __device__ __forceinline__ void split16x2<__half>(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const __half2 l = __floats2half2_rn(a - __low2float(h), b - __high2float(h));
  hi = *reinterpret_cast<const uint32_t*>(&h); lo = *reinterpret_cast<const uint32_t*>(&l);
}

__device__ __noinline__ float act_slow(float v, int act, float p0) { return b2a_act(v, act, p0, 1.f, 1.f); }
__device__ __noinline__ float act_slow2(float v, int act, float p0, float a, float b) { return b2a_act(v, act, p0, a, b); }

// accumulate the SM cycles a role spends inside a wait (debug runs only): slots 16.. of the CTA's row.  clock64, not %globaltimer: the
// global timer read costs ~1 us on this part and, placed around every wait, it WAS the timeline (measured: same kernel 2x slower).
#define TIMED_WAIT(p, acc, stmt) do { if (DBG && (p).dbg) { const long long t0_ = clock64(); stmt; acc += (unsigned long long)(clock64() - t0_); } else { stmt; } } while (0)
__device__ __forceinline__ void stamp(const FParams& p, int slot) {
  if (p.dbg) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); p.dbg[(size_t)blockIdx.x * 32 + slot] = t; }
}

// One float4 (4 channels of one row) -> transformed hi / lo 16-bit quads at the swizzled position of row r, 8-byte slot c4.
// ACT >= 0: the activation is a compile-time constant (round 1 measured the inlined runtime switch instruction-cache- and branch-bound); -1: runtime.
template <typename T16, int ACT>
__device__ __forceinline__ void convert_store(float4 v, bool valid, const float sc[4], const float sh[4], const float aa[4], const float bb[4],
                                              const bool chok[4], int act, float p0, uint8_t* hi, uint8_t* lo, int r, int c4, bool do_store = true) {
  const float t[4] = {v.x, v.y, v.z, v.w};
  float u[4];
  // Every element is transformed and the padding / out-of-range ones are replaced by zero afterwards: a branch per element around the
  // transform cost a BSSY / BSYNC pair each, and the worker warps' instruction issue bounds the generator-stage launches (DESIGN.md §5).
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const bool ok = valid && chok[q];
    float w = fmaf(t[q], sc[q], sh[q]);
    if constexpr (ACT == B2A_ACT_SNAKE) { const float s = b2a_sin_fast(aa[q] * w); w = fmaf(bb[q], s * s, w); }
    else if constexpr (ACT == B2A_ACT_LRELU) w = w > 0.f ? w : w * p0;
    else if constexpr (ACT == B2A_ACT_ELU) w = w > 0.f ? w : expm1f(w);
    else if constexpr (ACT == 0) { }
    else if (ok && act) w = act_slow2(w, act, p0, aa[q], bb[q]);
    u[q] = ok ? w : 0.f;
  }
  // hi = rn(u), lo = rn(u - hi), two channels per conversion instruction (the same round-to-nearest as the scalar conversions)
  uint2 h, l;
  split16x2<T16>(u[0], u[1], h.x, l.x);
  split16x2<T16>(u[2], u[3], h.y, l.y);
  const uint32_t off = (uint32_t)r * 128u + ((((uint32_t)c4 >> 1) ^ ((uint32_t)r & 7u)) << 4) + (((uint32_t)c4 & 1u) << 3);
  if (do_store) {
    *reinterpret_cast<uint2*>(hi + off) = h;
    if (lo) *reinterpret_cast<uint2*>(lo + off) = l;
  } else if (h.x == 0x12345678u && l.y == 0x9abcdef0u) {
    hi[0] = 1;                                                             // timing experiment: keep the conversion alive without the stores
  }
}

// One K chunk of the A tile: rows r0, r0 + RSTRIDE, ... of 4 channels.  ALL loads of a batch are issued before anything consumes them: a
// consumer placed between two loads -- even a predicated-off one, e.g. the optional x1 / x2 adds -- waits on the scoreboard of the
// load in front of it and serialises the batch into one L2 round trip per row (measured: 2-10 us per K chunk instead of < 1 us).
// NADD = number of extra input tensors summed into x (0, 1 or 2); U = rows in flight per thread.
template <typename T16, int ACT, int NADD, int U>
__device__ __forceinline__ void convert_chunk(const float* __restrict__ xb, const float* __restrict__ xb1, const float* __restrict__ xb2, int64_t x_ld,
                                              int L, int lbase, int ch, int c4, int r0, int R, bool anych, const float sc[4], const float sh[4],
                                              const float aa[4], const float bb[4], const bool chok[4], int act, float p0, uint8_t* hi, uint8_t* lo,
                                              int flags = 0) {
  for (int r = r0; r < R; r += RSTRIDE * U) {
    float4 v[U], w1[NADD > 0 ? U : 1], w2[NADD > 1 ? U : 1];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int rr = r + u * RSTRIDE;
      const int l = lbase + rr;
      ok[u] = rr < R && l >= 0 && l < L && anych;
      const int64_t off = ok[u] ? (int64_t)l * x_ld + ch : 0;     // masked rows read row 0 of the chunk (always valid memory), result discarded
      if (flags & 1) v[u] = make_float4((float)rr, 1.f, 2.f, 3.f); else
      v[u] = __ldg(reinterpret_cast<const float4*>(xb + off));
      if constexpr (NADD > 0) w1[u] = __ldg(reinterpret_cast<const float4*>(xb1 + off));
      if constexpr (NADD > 1) w2[u] = __ldg(reinterpret_cast<const float4*>(xb2 + off));
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int rr = r + u * RSTRIDE;
      if constexpr (NADD > 0) { v[u].x += w1[u].x; v[u].y += w1[u].y; v[u].z += w1[u].z; v[u].w += w1[u].w; }
      if constexpr (NADD > 1) { v[u].x += w2[u].x; v[u].y += w2[u].y; v[u].z += w2[u].z; v[u].w += w2[u].w; }
      if (rr < R) convert_store<T16, ACT>(v[u], ok[u], sc, sh, aa, bb, chok, act, p0, hi, lo, rr, c4, !(flags & 2));
    }
  }
}

// AdaIN coefficients of one channel from the binned (sum, sumsq) of the producer (float64, as norm.cu's adain_final_kernel)
__device__ __forceinline__ void stats_coeffs(const FProb& P, int b, int c, float& sc, float& sh) {
  const long long* w = P.pre_stats + ((int64_t)b * P.Cin + c) * (2 * B2A_NBIN);
  const double invL = 1.0 / (double)P.L;
  const double mean = repro_value(w) * invL;
  double var = repro_value(w + B2A_NBIN) * invL - mean * mean;
  if (var < 0) var = 0;
  const double rstd = 1.0 / sqrt(var + (double)P.pre_eps);
  double g_ = 1.0, be = 0.0;
  if (P.pre_gb) { g_ = 1.0 + (double)__ldg(P.pre_gb + (int64_t)b * P.pre_gb_bs + c); be = (double)__ldg(P.pre_gb + (int64_t)b * P.pre_gb_bs + P.Cin + c); }
  const double s_ = g_ * rstd;
  sc = (float)s_ * P.in_scale;
  sh = (float)(be - s_ * mean);
}

// Per-tile control values of the MMA warpgroups.  The problem table lives in shared memory, and ptxas treats a shared-memory load as
// possibly different per thread: a wgmma under a branch or loop bound taken from it sits on a "divergent path", and ptxas then
// serialises every wgmma (warning C7520: each HGMMA waits for the one before it).  A shuffle from lane 0 is provably warp-uniform.
struct MmaCtl { int kc0, kc1, taps, nb, two_w; };
__device__ __forceinline__ MmaCtl mma_ctl(const FProb& P, const TileRef& t) {
  const int kchunks = P.cin_pad / TK;
  const int kc0 = t.ks * P.kper;
  MmaCtl c;
  c.kc0 = __shfl_sync(0xffffffffu, kc0, 0);
  c.kc1 = __shfl_sync(0xffffffffu, min(kchunks, kc0 + P.kper), 0);
  c.taps = __shfl_sync(0xffffffffu, P.taps, 0);
  c.nb = __shfl_sync(0xffffffffu, P.BN >> 5, 0);
  c.two_w = __shfl_sync(0xffffffffu, P.wplanes == 2, 0);
  return c;
}

// One output tile on MMA warpgroup wg (threads 0..255): rows [64 wg, 64 wg + 64) of every K chunk x tap, accumulated in registers, then
// stored to the shared-memory output tile once the workers have drained the previous one.  Each tap step issues its products
// (hi*hi, lo*hi, hi*lo), commits them as one group and waits only for the PREVIOUS step's group (wgmma.wait_group 1), whose ring slot /
// A buffer is then handed back.  two_a comes from the kernel parameters (uniform), the rest from MmaCtl.  acc is the caller's one
// 64-register accumulator, live across the tile loop, of which an NB variant uses the first NB * 16: with a separate array per variant
// ptxas gives each its own register range (16 + 32 + 48 + 64 = 160 registers) and serialises the wgmmas for want of registers (C7512).
// DBG: mwait (shared memory, this warpgroup's leader writes) accumulates the SM cycles spent waiting on full / a_full / tempty and in
// wgmma.wait_group (MW_* below).  The wait itself is emitted once either way: a second copy of each wgmma.wait_group would double the
// WARPGROUP.DEPBARs that tests/test_conv_fused_compile.py bounds.
enum { MW_FULL, MW_AFULL, MW_TEMPTY, MW_WGMMA, MW_N };
#define MMA_TIMED(slot, stmt) do { if constexpr (DBG) { const long long t0_ = clock64(); stmt; if (leader) mwait[slot] += (unsigned long long)(clock64() - t0_); } else { stmt; } } while (0)
template <int NB, bool F16, bool DBG>
__device__ __forceinline__ void mma_tile(const FParams& p, const FProb& P, const MmaCtl& c, bool two_a, float* acc, uint32_t a0, uint32_t w0,
                                         uint64_t* full, uint64_t* empty, uint64_t* a_full, uint64_t* a_empty, uint64_t* tfull, uint64_t* tempty,
                                         float* acct, uint32_t lt, uint32_t& s, uint32_t& ph, uint32_t& cg, unsigned long long* mwait) {
  const int wg = threadIdx.x >> 7;
  const bool leader = (threadIdx.x & 127) == 0;
  const int kc0 = c.kc0, kc1 = c.kc1;
  const uint32_t wb = (uint32_t)NB * 32u * 128u, a_plane = (uint32_t)p.a_plane, a_buf = a_plane * (two_a ? 2u : 1u);
  const bool two_w = c.two_w != 0;
  const int taps = c.taps, smin = P.shift_min;
  int pend_s = -1, pend_a = -1;
  uint32_t accum = 0;                                            // the tile's first MMA overwrites the accumulator
  for (int kc = kc0; kc < kc1; kc++, cg++) {
    const uint32_t ab = cg & 1;
    MMA_TIMED(MW_AFULL, mbar_wait(a_full + ab, (cg >> 1) & 1));
    const uint32_t abase = a0 + ab * a_buf + (uint32_t)wg * 64u * 128u;
    for (int tap = 0; tap < taps; tap++) {
      MMA_TIMED(MW_FULL, mbar_wait(full + s, ph));
      const uint32_t wa = w0 + s * (uint32_t)p.w_stage;
      const uint32_t aa = abase + (uint32_t)(P.shift[tap] - smin) * 128u;
      const uint64_t wd = gmma_desc_sw128(wa), ad = gmma_desc_sw128(aa);
      wgmma_fence();
      wgmma_chunk<NB, F16>(acc, ad, wd, accum);                                             // a_hi * w_hi
      accum = 1;
      if (two_a) wgmma_chunk<NB, F16>(acc, gmma_desc_sw128(aa + a_plane), wd, 1u);         // a_lo * w_hi
      if (two_w) wgmma_chunk<NB, F16>(acc, ad, gmma_desc_sw128(wa + wb), 1u);              // a_hi * w_lo
      wgmma_commit();
      MMA_TIMED(MW_WGMMA, wgmma_wait<1>());
      wgmma_fence_regs<NB * 16>(acc);
      if (leader) {
        if (pend_s >= 0) mbar_arrive(empty + pend_s);
        if (pend_a >= 0) mbar_arrive(a_empty + pend_a);
      }
      pend_s = (int)s;
      pend_a = tap == taps - 1 ? (int)ab : -1;
      if (++s == (uint32_t)p.wst) { s = 0; ph ^= 1; }
    }
  }
  MMA_TIMED(MW_WGMMA, wgmma_wait<0>());
  wgmma_fence_regs<NB * 16>(acc);
  if (leader) {
    if (pend_s >= 0) mbar_arrive(empty + pend_s);
    if (pend_a >= 0) mbar_arrive(a_empty + pend_a);
  }
  MMA_TIMED(MW_TEMPTY, mbar_wait(tempty, (lt & 1) ^ 1));         // the workers have drained the previous tile
  store_acc<NB>(acc, acct, p.acc_ld, wg * 64);
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(tfull);               // 8 arrivals: the tile is complete
}

// Shared memory: [2] x A buffer (planes x a_plane bytes) | [wst] x W stage | output tile [128][acc_ld] | sacc | coefficient table | barriers.
// Each role builds this after its setmaxnreg: pointers computed above the role split would be live into every role, and the 32-register
// producer would spill them.
struct SmemLayout {
  int a_buf;
  uint8_t* wbase;
  float *acct, *sacc, *ctab;                 // ctab: [2][CT_MAX] scale | shift of the input transform
  uint64_t *full, *empty, *tfull, *tempty, *a_full, *a_empty;   // a_full / a_empty: [2]
  int* flag_slot;
  __device__ __forceinline__ SmemLayout(uint8_t* smem, const FParams& p) {
    a_buf = p.a_plane * p.planes;
    wbase = smem + (size_t)2 * a_buf;
    acct = reinterpret_cast<float*>(wbase + (size_t)p.wst * p.w_stage);
    sacc = acct + TM * p.acc_ld;
    ctab = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(sacc) + SACC);
    full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(ctab) + CTAB);
    empty = full + p.wst;
    tfull = empty + p.wst;
    tempty = tfull + 1;
    a_full = tempty + 1;
    a_empty = a_full + 2;
    flag_slot = reinterpret_cast<int*>(a_empty + 2);
  }
};

// DBG = false compiles every timing stamp, wait accumulator and ablation flag out of the production kernel.
template <bool DBG>
__global__ void __launch_bounds__(THREADS, 1)
conv_fused_kernel(const __grid_constant__ FParams gp, const __grid_constant__ CUtensorMap mw0, const __grid_constant__ CUtensorMap mw1,
                  const __grid_constant__ CUtensorMap mw2, const __grid_constant__ CUtensorMap mw3,
                  const __grid_constant__ CUtensorMap ml0, const __grid_constant__ CUtensorMap ml1,
                  const __grid_constant__ CUtensorMap ml2, const __grid_constant__ CUtensorMap ml3) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // The problem table is indexed by the tile's problem id at run time.  Reading it from the kernel-parameter (constant) bank costs a
  // dependent, dynamically indexed LDC per field -- hundreds of cycles each once 18 warps thrash the constant cache -- and those loads sat
  // inside every role's inner loop (measured: the MMA issuer spent ~1.5 us per K chunk issuing 8 MMAs).  One cooperative copy into shared
  // memory at kernel start makes every later access a ~30-cycle LDS.
  __shared__ __align__(16) FParams sparams;
  __shared__ unsigned long long mwait_all[DBG ? 2 * MW_N : 1];     // DBG: the MMA warpgroups' wait cycles (see mma_tile)
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&gp);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sparams);
    for (int i = threadIdx.x; i < (int)(sizeof(FParams) / 4); i += THREADS) dst[i] = src[i];
    if (DBG && threadIdx.x < 2 * MW_N) mwait_all[threadIdx.x] = 0;
  }
  __syncthreads();
  const FParams& p = sparams;
  if (threadIdx.x == 0) if (DBG) stamp(p, 0);

  if (warp == W_PROD && lane == 0) {
    const SmemLayout sl(smem, p);
    for (int s = 0; s < p.wst; s++) { mbar_init(sl.full + s, 1); mbar_init(sl.empty + s, 2); }
    mbar_init(sl.tfull, 8); mbar_init(sl.tempty, NWORK);
    mbar_init(sl.a_full, NWORK); mbar_init(sl.a_full + 1, NWORK); mbar_init(sl.a_empty, 2); mbar_init(sl.a_empty + 1, 2);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) if (DBG) stamp(p, 1);
  pdl_launch_dependents();        // the next kernel may start its own prologue / weight loads as SMs free up; it waits for us before reading

  // warpgroup index through a shuffle: provably uniform, so ptxas sees each role (and the wgmmas inside it) on a non-divergent path
  const int wgi = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  if (wgi == WG_PROD) {
    // ===== weight producer: independent of the previous kernel's output, so it starts before the programmatic-dependency wait =====
    set_regs<REG_PROD>();
    if (warp == W_PROD && lane == 0) {
      const SmemLayout sl(smem, p);
      uint8_t* const wbase = sl.wbase;
      uint64_t* const full = sl.full;
      uint64_t* const empty = sl.empty;
      const CUtensorMap* mws[MAXG] = {&mw0, &mw1, &mw2, &mw3};
      const CUtensorMap* mls[MAXG] = {&ml0, &ml1, &ml2, &ml3};
      for (int g = 0; g < p.G; g++) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(mws[g]) : "memory");
        if (p.pr[g].wplanes == 2) asm volatile("prefetch.tensormap [%0];" ::"l"(mls[g]) : "memory");
      }
      int s = 0; uint32_t ph = 0;
      unsigned long long w_pempty = 0;
      const long long pt0 = DBG ? clock64() : 0;
      for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        const TileRef t = decode_tile(p, tile);
        const FProb& P = p.pr[t.g];
        const int n0 = t.nt * P.BN;
        const int kchunks = P.cin_pad / TK;
        const int kc0 = t.ks * P.kper, kc1 = min(kchunks, kc0 + P.kper);
        const uint32_t wb = (uint32_t)P.BN * 128u;
        for (int kc = kc0; kc < kc1; kc++) {
          for (int tap = 0; tap < P.taps; tap++) {
            TIMED_WAIT(p, w_pempty, mbar_wait(empty + s, ph ^ 1));
            uint8_t* st = wbase + (size_t)s * p.w_stage;
            mbar_expect_tx(full + s, wb * (uint32_t)P.wplanes);
            tma_load_2d(st, mws[t.g], full + s, kc * TK, tap * P.Ntot + n0);
            if (P.wplanes == 2) tma_load_2d(st + wb, mls[t.g], full + s, kc * TK, tap * P.Ntot + n0);
            if (++s == p.wst) { s = 0; ph ^= 1; }
          }
        }
      }
      if (DBG && p.dbg) { p.dbg[(size_t)blockIdx.x * 32 + 21] = (unsigned long long)(clock64() - pt0); p.dbg[(size_t)blockIdx.x * 32 + 22] = w_pempty; }
    }
  } else if (wgi < WG_PROD) {
    // ===== MMA warpgroups =====
    set_regs<REG_MMA>();
    const SmemLayout sl(smem, p);
    uint64_t *const full = sl.full, *const empty = sl.empty, *const a_full = sl.a_full, *const a_empty = sl.a_empty;
    uint64_t *const tfull = sl.tfull, *const tempty = sl.tempty;
    float* const acct = sl.acct;
    const uint32_t a0 = smem_u32(smem), w0 = smem_u32(sl.wbase);
    const bool f16 = gp.f16 != 0, two_a = gp.planes == 2;       // kernel parameters: uniform
    uint32_t s = 0, ph = 0, lt = 0, cg = 0;
    float acc[4 * 16];                                          // shared by every NB variant (see mma_tile)
#pragma unroll
    for (int i = 0; i < 4 * 16; i++) acc[i] = 0.f;
    unsigned long long* const mwait = mwait_all + (DBG ? wgi * MW_N : 0);
    for (int tile = blockIdx.x; tile < gp.ntiles; tile += gridDim.x, lt++) {
      const TileRef t = decode_tile(p, tile);
      const FProb& P = p.pr[t.g];
      const MmaCtl c = mma_ctl(P, t);
#define B2A_MMA_TILE(NB) (f16 ? mma_tile<NB, true, DBG>(p, P, c, two_a, acc, a0, w0, full, empty, a_full, a_empty, tfull, tempty, acct, lt, s, ph, cg, mwait) \
                              : mma_tile<NB, false, DBG>(p, P, c, two_a, acc, a0, w0, full, empty, a_full, a_empty, tfull, tempty, acct, lt, s, ph, cg, mwait))
      switch (c.nb) {
        case 1: B2A_MMA_TILE(1); break;
        case 2: B2A_MMA_TILE(2); break;
        case 3: B2A_MMA_TILE(3); break;
        default: B2A_MMA_TILE(4); break;
      }
#undef B2A_MMA_TILE
    }
  } else {
    // ===== worker warps: A-tile conversion AND epilogue =====
    set_regs<REG_WORK>();
    const SmemLayout sl(smem, p);
    const int a_buf = sl.a_buf;
    float *const acct = sl.acct, *const sacc = sl.sacc, *const ctab = sl.ctab;
    uint64_t *const a_full = sl.a_full, *const a_empty = sl.a_empty, *const tfull = sl.tfull, *const tempty = sl.tempty;
    int* const flag_slot = sl.flag_slot;
    // The first version of this kernel split the roles (8 converter + 8 epilogue warps).  Its profile on the Kokoro layers: the converter
    // was the bottleneck everywhere (~5 us per K chunk, issue-latency bound with two warps per scheduler) while the epilogue warps
    // idled ~70 % of the time, and the two big loops evicted each other from the instruction caches (a third of the stall samples
    // were no_inst).  Now every worker runs the same loop at the same time, at twice the width:
    //     C(0) C(1) E(0) C(2) E(1) ... E(last)        C = convert all K chunks of a tile, E = epilogue of a tile
    // MMA(t) stores its tile once E(t-1) has freed the output tile, and E(t-1) precedes C(t+1) in this order: no deadlock.  E(t) runs after C(t+1), by when
    // the MMAs of tile t have normally retired, so the workers rarely wait on tfull.
    pdl_wait();
    if (warp == W_WORK0 && lane == 0) if (DBG) stamp(p, 3);
    const int ww = warp - W_WORK0;                   // 0..NWORK-1
    const int wt = ww * 32 + lane;                   // 0..32 NWORK - 1
    const int c4 = wt & 15;                          // float4 slot inside the 64-channel chunk (fixed per thread: constants stay in registers)
    const int r0 = wt >> 4;                          // first A-tile row of this thread (stride RSTRIDE)
    const int quarter = ww & 3, sub = ww >> 2;       // quarter = 32-row group of the output tile; sub picks the 32-column chunk
    const int et = wt;
    uint32_t cg = 0;
    int cur_key = -1;                                // (problem, batch) whose coefficients the table holds
    unsigned long long w_aempty = 0, w_tfull = 0;

    auto convert_tile = [&](const int tile) {
      {
        const TileRef t = decode_tile(p, tile);
        const FProb& P = p.pr[t.g];
        const int l0 = t.mt * TM, n0 = t.nt * P.BN, b = t.b;
        if (!P.up_s && P.ksplit == 1) {                           // pull this warp's residual / previous-output rows towards L2 while the MMAs run
          const int prow = l0 + quarter * 32 + lane;
          if (prow < P.Lout) {
            if (P.res) {
              const float* q = P.res + (int64_t)b * P.res_bs + (int64_t)(P.res_div == 2 ? (prow >> 1) : prow) * P.res_ld + n0;
              for (int c = sub * 32; c < P.BN; c += NSUB * 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(q + c));
            }
            if (P.accumulate) {
              const float* q = P.y + (int64_t)b * P.y_bs + (int64_t)prow * P.y_ld + n0;
              for (int c = sub * 32; c < P.BN; c += NSUB * 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(q + c));
            }
          }
        }
      }
      const TileRef t = decode_tile(p, tile);
      const FProb& P = p.pr[t.g];
      const int kchunks = P.cin_pad / TK;
      const int kc0 = t.ks * P.kper, kc1 = min(kchunks, kc0 + P.kper);
      const int lbase = t.mt * TM + P.shift_min;
      const float* xb = P.x + (int64_t)t.b * P.x_bs;
      const float* xb1 = P.x1 ? P.x1 + (int64_t)t.b * P.x_bs : nullptr;
      const float* xb2 = P.x2 ? P.x2 + (int64_t)t.b * P.x_bs : nullptr;
      const int R = P.R;
      // (scale, shift) of every input channel: computed once per (problem, batch) by the worker threads -- the float64 statistics
      // arithmetic costs ~150 double-precision operations per channel, far too much to repeat in every K chunk of every tile
      const bool tabled = P.pre_mode != 0 && P.Cin <= CT_MAX;
      const int key = (t.g << 16) | t.b;
      if (tabled && key != cur_key) {
        bar_sync(3, NWORK * 32);                       // nobody still reads the previous table
        for (int c = wt; c < P.Cin; c += NWORK * 32) {
          float sc_ = P.in_scale, sh_ = 0.f;
          if (P.pre_mode == 1) { sc_ = __ldg(P.pre_scale + (int64_t)t.b * P.Cin + c) * P.in_scale; sh_ = __ldg(P.pre_shift + (int64_t)t.b * P.Cin + c); }
          else stats_coeffs(P, t.b, c, sc_, sh_);
          ctab[c] = sc_; ctab[CT_MAX + c] = sh_;
        }
        bar_sync(3, NWORK * 32);
        cur_key = key;
      }
      for (int kc = kc0; kc < kc1; kc++, cg++) {
        const uint32_t ab = cg & 1;
        const int ch = kc * TK + c4 * 4;
        float sc[4], sh[4], aa[4], bb[4];
        bool chok[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int c = ch + q;
          chok[q] = c < P.Cin;
          sc[q] = P.in_scale; sh[q] = 0.f; aa[q] = 1.f; bb[q] = 1.f;
          if (chok[q]) {
            if (tabled) { sc[q] = ctab[c]; sh[q] = ctab[CT_MAX + c]; }
            else if (P.pre_mode == 1) { sc[q] = __ldg(P.pre_scale + (int64_t)t.b * P.Cin + c) * P.in_scale; sh[q] = __ldg(P.pre_shift + (int64_t)t.b * P.Cin + c); }
            else if (P.pre_mode == 2) stats_coeffs(P, t.b, c, sc[q], sh[q]);
            if (P.pre_a) aa[q] = __ldg(P.pre_a + c);
            if (P.pre_b) bb[q] = __ldg(P.pre_b + c);
          }
        }
        const bool anych = ch < P.Cin;
        TIMED_WAIT(p, w_aempty, mbar_wait(a_empty + ab, ((cg >> 1) & 1) ^ 1));
        uint8_t* hi = smem + (size_t)ab * a_buf;
        uint8_t* lo = p.planes == 2 ? hi + p.a_plane : nullptr;
#define B2A_CONVERT(T, A, N, UU) convert_chunk<T, A, N, UU>(xb, xb1, xb2, P.x_ld, P.L, lbase, chs, c4, r0, R, anych, sc, sh, aa, bb, chok, P.pre_act, P.pre_p0, hi, lo, (DBG ? p.dbg_flags : 0))
        const int chs = anych ? ch : 0;                    // chunks wholly past Cin (never with a valid weight column) still index valid memory
        // specialised bodies for the hot cases only (each instantiation is ~1-2 K instructions): single input x {none, Snake, LeakyReLU, ELU};
        // summed inputs (the folded branch average) and fp16 operands with an activation take the runtime-switch body
        if ((DBG ? p.dbg_flags : 0) & 16) { }
        else if (p.f16) { if (xb1 == nullptr && P.pre_act == 0) B2A_CONVERT(__half, 0, 0, 5); else if (xb2) B2A_CONVERT(__half, -1, 2, 2);
                     else if (xb1) B2A_CONVERT(__half, -1, 1, 3); else B2A_CONVERT(__half, -1, 0, 3); }
        else if (xb2) B2A_CONVERT(__nv_bfloat16, -1, 2, 2);
        else if (xb1) B2A_CONVERT(__nv_bfloat16, -1, 1, 3);
        else if (P.pre_act == 0) B2A_CONVERT(__nv_bfloat16, 0, 0, 5);
        else if (P.pre_act == B2A_ACT_SNAKE) B2A_CONVERT(__nv_bfloat16, B2A_ACT_SNAKE, 0, 5);
        else if (P.pre_act == B2A_ACT_LRELU) B2A_CONVERT(__nv_bfloat16, B2A_ACT_LRELU, 0, 5);
        else if (P.pre_act == B2A_ACT_ELU) B2A_CONVERT(__nv_bfloat16, B2A_ACT_ELU, 0, 3);
        else B2A_CONVERT(__nv_bfloat16, -1, 0, 3);
#undef B2A_CONVERT
        if (!((DBG ? p.dbg_flags : 0) & 4)) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the MMA's async-proxy reads
        __syncwarp();
        if (lane == 0) mbar_arrive(a_full + ab);
        if (warp == W_WORK0 && lane == 0) { if (cg == 0) if (DBG) stamp(p, 6); if (DBG) stamp(p, 7); }
      }
    };

    auto epilogue_tile = [&](const int tile, const uint32_t lt) {
      const TileRef t = decode_tile(p, tile);
      const FProb& P = p.pr[t.g];
      const int mul = P.up_s ? P.up_s : 1;
      const int l0 = t.mt * TM, n0 = t.nt * P.BN, b = t.b;
      const bool do_stats = P.stats_out != nullptr;
      TIMED_WAIT(p, w_tfull, mbar_wait(tfull, lt & 1));
      if (et == 0 && lt == 0) if (DBG) stamp(p, 8);
      const int mrow0 = l0 + quarter * 32;
      float* tq = acct + (size_t)(quarter * 32) * p.acc_ld;        // this warp's 32 rows of the output tile
      const int ALD = p.acc_ld;
      bool last_split = !((DBG ? p.dbg_flags : 0) & 32);
      if (P.ksplit > 1) {
        // ---- split-K: park this CTA's partial accumulator (through the transpose tile: whole 128-byte row segments), then only the
        // last CTA to arrive for the tile carries on
        const int tid = ((b * P.ntm + t.mt) * P.ntn + t.nt);
        float* mine = P.ws + ((int64_t)tid * P.ksplit + t.ks) * (TM * P.BN) + (int64_t)(quarter * 32) * P.BN;
        for (int c0 = sub * 32; c0 < P.BN; c0 += NSUB * 32) {
          const float* stage = tq + c0;
#pragma unroll 8
          for (int i = 0; i < 32; i++) mine[(int64_t)i * P.BN + c0 + lane] = stage[i * ALD + lane];
        }
        __threadfence();
        bar_sync(2, NWORK * 32);
        if (et == 0) {
          const int prev = atomicAdd(P.counters + tid, 1);
          const int last = prev == P.ksplit - 1;
          if (last) P.counters[tid] = 0;              // re-arm for the next launch that reuses this workspace
          *flag_slot = last;
        }
        bar_sync(2, NWORK * 32);
        last_split = *flag_slot != 0;
        if (last_split) __threadfence();
        if (et == 0 && lt == 0) if (DBG) stamp(p, 9);
      }
      if (last_split) {
        for (int c0 = sub * 32; c0 < P.BN; c0 += NSUB * 32) {
          float* stage = tq + c0;
          if (P.ksplit > 1) {
            // fixed-order sum of the partial tiles, read row by row (lane = column: coalesced, and already the layout the stores below want)
            const int tid = ((b * P.ntm + t.mt) * P.ntn + t.nt);
            const float* base = P.ws + (int64_t)tid * P.ksplit * (TM * P.BN) + (int64_t)(quarter * 32) * P.BN + c0 + lane;
            for (int i0 = 0; i0 < 32; i0 += 8) {
              float acc[8];
#pragma unroll
              for (int i = 0; i < 8; i++) acc[i] = 0.f;
              for (int s = 0; s < P.ksplit; s++) {
                const float* q = base + (int64_t)s * (TM * P.BN) + (int64_t)i0 * P.BN;
#pragma unroll
                for (int i = 0; i < 8; i++) acc[i] += __ldcg(q + (int64_t)i * P.BN);
              }
#pragma unroll
              for (int i = 0; i < 8; i++) stage[(i0 + i) * ALD + lane] = acc[i];
            }
            __syncwarp();
          }
          // Vectorised write-out: lane = (row sub-index rsub = lane / 8, four consecutive columns c4 = 4 (lane % 8)); one instruction moves
          // four output rows x 128 bytes, and all eight residual / previous-output loads of the chunk are in flight together (the scalar
          // version needed four dependent 16-load batches per warp and tile: ~10 us per tile, the kernel's bottleneck).
          const int rsub = lane >> 3, c4 = (lane & 7) * 4;
          const int n = n0 + c0 + c4;
          const int ph = P.up_s ? n / P.C : 0;
          const int co = n - ph * P.C;
          float st1[4] = {0.f, 0.f, 0.f, 0.f}, st2[4] = {0.f, 0.f, 0.f, 0.f};
          if (mrow0 < P.Mrows) {
            const int add = P.up_s ? ph - P.up_crop : 0;
            float bias[4], cso[4];
#pragma unroll
            for (int q = 0; q < 4; q++) {
              bias[q] = P.bias ? __ldg(P.bias + co + q) : 0.f;
              cso[q] = (P.cscale ? __ldg(P.cscale + (int64_t)b * P.cscale_bs + co + q) : 1.f) * P.out_scale;
            }
            float* ycol = P.y + (int64_t)b * P.y_bs + co;
            const float* rcol = P.res ? P.res + (int64_t)b * P.res_bs + co : nullptr;
            const int row0 = mrow0 * mul + add;
            const int mvalid = min(32, P.Mrows - mrow0);
            int i_lo = 0, i_hi = mvalid;
            if (row0 < 0) i_lo = (-row0 + mul - 1) / mul;
            if (row0 + (mvalid - 1) * mul >= P.Lout) i_hi = P.Lout > row0 ? (P.Lout - row0 + mul - 1) / mul : 0;
            const bool half_res = P.res_div == 2;
            const float osc = P.out_scale;
            float4 rr[8];
            bool okr[8];
#pragma unroll
            for (int i = 0; i < 8; i++) {                                  // the chunk's residual (+ previous output) rows: one batch of loads
              const int ti = 4 * i + rsub;                                 // tile row 0..31
              const int row = row0 + ti * mul;
              okr[i] = ti >= i_lo && ti < i_hi;
              rr[i] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (okr[i]) {
                if (rcol) rr[i] = __ldg(reinterpret_cast<const float4*>(rcol + (int64_t)(half_res ? (row >> 1) : row) * P.res_ld));
              }
            }
            if (P.accumulate) {
#pragma unroll
              for (int i = 0; i < 8; i++) {
                if (okr[i]) {
                  const float4 o = *reinterpret_cast<const float4*>(ycol + (int64_t)(row0 + (4 * i + rsub) * mul) * P.y_ld);
                  rr[i].x = fmaf(rr[i].x, osc, o.x); rr[i].y = fmaf(rr[i].y, osc, o.y); rr[i].z = fmaf(rr[i].z, osc, o.z); rr[i].w = fmaf(rr[i].w, osc, o.w);
                }
              }
            } else {
#pragma unroll
              for (int i = 0; i < 8; i++) { rr[i].x *= osc; rr[i].y *= osc; rr[i].z *= osc; rr[i].w *= osc; }
            }
#pragma unroll
            for (int i = 0; i < 8; i++) {
              const int ti = 4 * i + rsub;
              if (okr[i]) {
                const float4 sp = *reinterpret_cast<const float4*>(stage + ti * ALD + c4);   // a quarter-warp reads one 128-byte row segment
                float a[4] = {sp.x + bias[0], sp.y + bias[1], sp.z + bias[2], sp.w + bias[3]};
                if (P.post_act) {
#pragma unroll
                  for (int q = 0; q < 4; q++) a[q] = act_slow(a[q], P.post_act, P.post_p0);
                }
                float4 v;
                v.x = fmaf(a[0], cso[0], rr[i].x); v.y = fmaf(a[1], cso[1], rr[i].y); v.z = fmaf(a[2], cso[2], rr[i].z); v.w = fmaf(a[3], cso[3], rr[i].w);
                *reinterpret_cast<float4*>(ycol + (int64_t)(row0 + ti * mul) * P.y_ld) = v;
                st1[0] += v.x; st1[1] += v.y; st1[2] += v.z; st1[3] += v.w;
                st2[0] = fmaf(v.x, v.x, st2[0]); st2[1] = fmaf(v.y, v.y, st2[1]); st2[2] = fmaf(v.z, v.z, st2[2]); st2[3] = fmaf(v.w, v.w, st2[3]);
              }
            }
            __syncwarp();
          }
          if (do_stats) {                                                  // fixed-order reduction over the four row sub-indices, then one writer per slot
#pragma unroll
            for (int q = 0; q < 4; q++) {
              st1[q] += __shfl_xor_sync(0xffffffffu, st1[q], 8); st1[q] += __shfl_xor_sync(0xffffffffu, st1[q], 16);
              st2[q] += __shfl_xor_sync(0xffffffffu, st2[q], 8); st2[q] += __shfl_xor_sync(0xffffffffu, st2[q], 16);
            }
            if (rsub == 0) {
#pragma unroll
              for (int q = 0; q < 4; q++) { sacc[(quarter * 2 + 0) * 128 + c0 + c4 + q] = st1[q]; sacc[(quarter * 2 + 1) * 128 + c0 + c4 + q] = st2[q]; }
            }
          }
        }
      }
      __syncwarp();
      if (et == 0) { if (lt == 0) if (DBG) stamp(p, 10); if (DBG) stamp(p, 11); }
      if (lane == 0) mbar_arrive(tempty);                      // NWORK arrivals free the output tile for tile lt + 1
      if (do_stats) {
        bar_sync(1, NWORK * 32);
        if (last_split) {
          const int co0 = P.up_s ? (n0 % P.C) : n0;
          for (int i = et; i < 2 * P.BN; i += NWORK * 32) {
            const int which = i >= P.BN, col = i - which * P.BN;
            const float v = ((sacc[(0 * 2 + which) * 128 + col] + sacc[(1 * 2 + which) * 128 + col]) + sacc[(2 * 2 + which) * 128 + col]) +
                            sacc[(3 * 2 + which) * 128 + col];                      // fixed order over the four lane quarters
            repro_add(P.stats_out + (((int64_t)b * P.C + co0 + col) * 2 + which) * B2A_NBIN, v);
          }
        }
        bar_sync(1, NWORK * 32);
      }
    };

    int prev = -1;
    uint32_t nt_done = 0;
    long long cyc_c = 0, cyc_e = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      const long long c0_ = DBG ? clock64() : 0;
      convert_tile(tile);
      const long long c1_ = DBG ? clock64() : 0;
      if (prev >= 0) { epilogue_tile(prev, nt_done); nt_done++; }
      if (DBG) { cyc_c += c1_ - c0_; cyc_e += clock64() - c1_; }
      prev = tile;
    }
    { const long long c1_ = DBG ? clock64() : 0; if (prev >= 0) epilogue_tile(prev, nt_done); if (DBG) cyc_e += clock64() - c1_; }
    if (DBG && p.dbg && warp == W_WORK0 && lane == 0) { p.dbg[(size_t)blockIdx.x * 32 + 24] = (unsigned long long)cyc_c; p.dbg[(size_t)blockIdx.x * 32 + 25] = (unsigned long long)cyc_e; }
    if (DBG && p.dbg && warp == W_WORK0 && lane == 0) { p.dbg[(size_t)blockIdx.x * 32 + 19] = w_aempty; p.dbg[(size_t)blockIdx.x * 32 + 20] = w_tfull; }
  }
  if (threadIdx.x == 0) if (DBG) stamp(p, 12);
  __syncthreads();
  if (threadIdx.x == 0) if (DBG) stamp(p, 13);
  if (DBG && p.dbg && threadIdx.x < MW_N)                          // slots 26..29: both MMA warpgroups' wait cycles, summed
    p.dbg[(size_t)blockIdx.x * 32 + 26 + threadIdx.x] = mwait_all[threadIdx.x] + mwait_all[MW_N + threadIdx.x];
}

unsigned long long* g_fdbg = nullptr;
thread_local int32_t g_last_cfg[2 + 2 * MAXG] = {};    // problems, grid, then (BN, ksplit) per problem: this host thread's last launch

// N tile: the widest divisor of N (multiple of 32, <= 128) -- in polyphase mode also a divisor of C so that a tile stays inside one phase
int n_tile(int N, int C) {
  for (int c = 128; c >= 32; c -= 32) if (N % c == 0 && C % c == 0) return c;
  return 0;
}
int a_rows(int span) { return (TM + span + 7) / 8 * 8; }     // rows of one K chunk's A tile: 128 output rows + the taps' span, to 8
int acc_tile_ld(int bn) { return bn + 8; }                    // 8 mod 32 words: the accumulator fragment stores of a quarter-warp hit distinct banks
// GEMM rows: the output rows, or in polyphase mode every row m whose phases m * s + r - crop reach an output row below Lout.  Rows past
// L + taps - 1 read only the zero padding, so output rows past the scatter (output padding wider than the crop) get the epilogue alone.
int gemm_rows(const b2a_convf_t& q) {
  if (q.up_stride <= 0) return q.Lout;
  const int tail = cdiv(q.Lout + q.up_crop, q.up_stride);
  return q.L + q.taps - 1 > tail ? q.L + q.taps - 1 : tail;
}
// Weight stages (at most 8) that fit beside the two A buffers, the output tile and the fixed regions; *smem: the launch's dynamic
// shared memory with that many stages.  A launch needs two.
int weight_stages(int a_plane, int planes, int acc_ld, int w_stage, size_t* smem) {
  const size_t fixed = (size_t)2 * a_plane * planes + (size_t)TM * acc_ld * 4 + SACC + CTAB + 1024 /*align*/ + 512 /*barriers*/;
  int wst = fixed < DYN_SMEM_MAX ? (int)((DYN_SMEM_MAX - fixed) / w_stage) : 0;
  if (wst > 8) wst = 8;
  if (smem) *smem = fixed + (size_t)wst * w_stage;
  return wst;
}

}  // namespace

/* debug aid: device buffer of [gridDim][32] uint64 that the next launches stamp with %globaltimer at their phase boundaries (NULL: off) */
extern "C" int32_t b2a_conv1d_fused_debug(void* buf) { g_fdbg = (unsigned long long*)buf; return B2A_OK; }

/* the tiles and K splits the last launch chose, so that tests can assert which variant they exercised */
extern "C" int32_t b2a_conv1d_fused_last_config(int32_t* out10) {
  B2A_CHECK_ARG(out10, "null pointer");
  for (int i = 0; i < 2 + 2 * MAXG; i++) out10[i] = g_last_cfg[i];
  return B2A_OK;
}

/* whether one problem of this geometry fits a launch's shared memory (see include/b200audio.h) */
extern "C" int32_t b2a_conv1d_fused_fits(int32_t span, int32_t N, int32_t C, int32_t wplanes, int32_t planes) {
  if (span < 0 || span > 64 || N <= 0 || C <= 0 || N % C || (wplanes != 1 && wplanes != 2) || (planes != 1 && planes != 2)) return 0;
  const int bn = n_tile(N, C);
  return bn && weight_stages(a_rows(span) * 128, planes, acc_tile_ld(bn), bn * 128 * wplanes, nullptr) >= 2;
}

extern "C" int32_t b2a_conv1d_fused(const b2a_convf_t* pr, int32_t n, int32_t planes, int32_t f16, void* ws, int64_t ws_bytes, void* stream) {
  B2A_CHECK_ARG(pr && n >= 1 && n <= MAXG && (planes == 1 || planes == 2), "1..4 problems, planes 1 or 2");
  static const int nsm = [] { const int n = b2a_device_sm_count(); return n > 0 ? n : 132; }();
  FParams p;
  p.G = n; p.planes = planes; p.f16 = f16 ? 1 : 0; p.dbg = g_fdbg;
  { static int flags = -1; if (flags < 0) { const char* e = getenv("B2A_FUSED_DBGFLAGS"); flags = e ? atoi(e) : 0; } p.dbg_flags = flags; }
  // heaviest problem first (cost per tile ~ taps * K chunks): sort indices
  int order[MAXG];
  double cost[MAXG];
  for (int i = 0; i < n; i++) { order[i] = i; cost[i] = (double)pr[i].taps * pr[i].cin_pad; }
  for (int i = 0; i < n; i++) for (int j = i + 1; j < n; j++) if (cost[order[j]] > cost[order[i]]) { int t = order[i]; order[i] = order[j]; order[j] = t; }
  int maxR = 0, maxBN = 0, maxWst = 0, tiles_total = 0;
  int64_t base_tiles = 0, sum_base = 0, cnt_used = 0, ws_used = 0;
  for (int gi = 0; gi < n; gi++) {                         // output tiles of the whole launch before any split (same tile rule as below)
    const b2a_convf_t& q = pr[gi];
    if (q.N <= 0 || q.N % 32) continue;                    // rejected by the argument checks below
    const int bn = n_tile(q.N, q.up_stride > 0 ? q.N / q.up_stride : q.N);
    if (!bn) continue;
    sum_base += (int64_t)cdiv(gemm_rows(q), TM) * (q.N / bn) * q.B;
  }
  for (int gi = 0; gi < n; gi++) {
    const b2a_convf_t& q = pr[order[gi]];
    B2A_CHECK_ARG(q.x && q.w_hi && q.y && q.B > 0 && q.L > 0 && q.Lout > 0 && q.Cin > 0 && q.taps > 0 && q.taps <= 32 && q.cin_pad % 64 == 0 && q.cin_pad >= q.Cin,
                  "bad pointers / shape");
    B2A_CHECK_ARG(q.N % 32 == 0 && q.y_ld % 4 == 0 && (q.res == nullptr || q.res_ld % 4 == 0) && (q.res_div == 1 || q.res_div == 2), "N % 32, row strides % 4, res_div 1|2");
    B2A_CHECK_ARG(((uintptr_t)q.y & 15) == 0 && q.y_bs % 4 == 0 && (q.res == nullptr || (((uintptr_t)q.res & 15) == 0 && q.res_bs % 4 == 0)), "y / res must be 16-byte aligned");
    B2A_CHECK_ARG(q.x_ld % 4 == 0 && q.x_bs % 4 == 0 && ((uintptr_t)q.x & 15) == 0 && q.x_ld >= ((q.Cin + 3) & ~3), "x must be 16-byte aligned with row stride % 4 == 0 and >= ceil4(Cin)");
    B2A_CHECK_ARG((q.x1 == nullptr || ((uintptr_t)q.x1 & 15) == 0) && (q.x2 == nullptr || ((uintptr_t)q.x2 & 15) == 0), "x1 / x2 alignment");
    B2A_CHECK_ARG(q.up_stride >= 0 && (q.up_stride == 0 || (q.N % q.up_stride == 0 && (q.N / q.up_stride) % 32 == 0)), "transposed mode: N = up_stride * C, C % 32 == 0");
    B2A_CHECK_ARG(q.pre_mode >= 0 && q.pre_mode <= 2 && (q.pre_mode != 1 || (q.pre_scale && q.pre_shift)) && (q.pre_mode != 2 || q.pre_stats), "prologue mode / pointers");
    FProb& P = p.pr[gi];
    P.x = q.x; P.x1 = q.x1; P.x2 = q.x2; P.x_bs = q.x_bs; P.x_ld = q.x_ld; P.in_scale = q.in_scale;
    P.B = q.B; P.L = q.L; P.Cin = q.Cin; P.cin_pad = q.cin_pad;
    P.pre_mode = q.pre_mode; P.pre_scale = q.pre_scale; P.pre_shift = q.pre_shift; P.pre_stats = (const long long*)q.pre_stats; P.pre_gb = q.pre_gb;
    P.pre_gb_bs = q.pre_gb_bs; P.pre_eps = q.pre_eps; P.pre_invL = 1.0f / (float)q.L;
    P.pre_act = q.pre_act; P.pre_p0 = q.pre_p0; P.pre_a = q.pre_a; P.pre_b = q.pre_b;
    P.taps = q.taps; P.wplanes = q.w_lo ? 2 : 1; P.Ntot = q.N;
    int smin = q.shifts[0], smax = q.shifts[0];
    for (int i = 0; i < q.taps; i++) { P.shift[i] = q.shifts[i]; smin = q.shifts[i] < smin ? q.shifts[i] : smin; smax = q.shifts[i] > smax ? q.shifts[i] : smax; }
    if (smax - smin > 64) { b2a_set_error("b2a_conv1d_fused: taps span %d rows (> 64)", smax - smin); return B2A_E_UNSUPPORTED; }
    P.shift_min = smin; P.R = a_rows(smax - smin);
    P.up_s = q.up_stride; P.up_crop = q.up_crop; P.C = q.up_stride ? q.N / q.up_stride : q.N;
    P.Lout = q.Lout; P.Mrows = gemm_rows(q);
    P.ntm = cdiv(P.Mrows, TM);
    P.BN = n_tile(q.N, P.C); P.ntn = q.N / P.BN;
    base_tiles = (int64_t)P.ntm * P.ntn * q.B;
    // split K across CTAs when the whole launch cannot give every SM a tile (every problem of a group by the same rule: the decoder
    // blocks -- a k=3 conv over 390 rows grouped with its 1x1 shortcut -- are 48 tiles with 54 tap steps each)
    const int kchunks = q.cin_pad / TK;
    P.ksplit = 1;
    if (sum_base * 2 <= nsm && kchunks >= 4 && ws) {
      int ks = (int)(nsm / sum_base);
      if (ks > 8) ks = 8;
      if (ks > kchunks / 2) ks = kchunks / 2;
      if (ks >= 2) P.ksplit = ks;
    }
    P.kper = cdiv(kchunks, P.ksplit);
    P.ksplit = cdiv(kchunks, P.kper);                     // no empty splits
    P.bias = q.bias; P.post_act = q.post_act; P.post_p0 = q.post_p0; P.cscale = q.cscale; P.cscale_bs = q.cscale_bs;
    P.res = q.res; P.res_bs = q.res_bs; P.res_ld = q.res_ld; P.res_div = q.res_div; P.out_scale = q.out_scale; P.accumulate = q.accumulate;
    P.y = q.y; P.y_bs = q.y_bs; P.y_ld = q.y_ld; P.stats_out = (long long*)q.stats_out;
    P.ws = nullptr; P.counters = nullptr;
    if (P.ksplit > 1) {
      // workspace layout: [4 KB of arrival counters (one per output tile; a split launch has fewer than one per SM)] [partial tiles].  The counter region
      // has a FIXED size: were it sized per launch, the partial tiles of a launch with fewer tiles would overwrite counters that a later launch
      // with more tiles expects to be zero (they are self-resetting, never re-zeroed).
      const int64_t bytes = base_tiles * P.ksplit * (TM * P.BN) * 4;
      if (4096 + ws_used + bytes > ws_bytes || cnt_used + base_tiles > 1024) { P.ksplit = 1; P.kper = kchunks; }
      else {
        P.counters = (int*)ws + cnt_used; P.ws = (float*)((uint8_t*)ws + 4096 + ws_used);       // each problem of a group: its own counters and partial tiles
        cnt_used += base_tiles; ws_used += bytes;
      }
    }
    P.tile_begin = tiles_total;
    tiles_total += (int)(base_tiles * P.ksplit);
    maxR = P.R > maxR ? P.R : maxR; maxBN = P.BN > maxBN ? P.BN : maxBN;
    const int wsz = P.BN * 128 * P.wplanes;
    maxWst = wsz > maxWst ? wsz : maxWst;
  }
  p.ntiles = tiles_total;
  p.a_plane = maxR * 128;
  p.w_stage = maxWst;
  p.acc_ld = acc_tile_ld(maxBN);
  size_t smem = 0;
  const int wst = weight_stages(p.a_plane, planes, p.acc_ld, p.w_stage, &smem);
  if (wst < 2) { b2a_set_error("b2a_conv1d_fused: shared memory cannot hold two weight stages (R %d, BN %d)", maxR, maxBN); return B2A_E_UNSUPPORTED; }
  p.wst = wst;

  CUtensorMap mw[MAXG], ml[MAXG];
  for (int gi = 0; gi < MAXG; gi++) {
    const b2a_convf_t& q = pr[order[gi < n ? gi : 0]];
    const FProb& P = p.pr[gi < n ? gi : 0];
    const uint64_t wdims[2] = {(uint64_t)q.cin_pad, (uint64_t)q.taps * q.N}, wstr[1] = {(uint64_t)q.cin_pad * 2};
    const uint32_t wbox[2] = {TK, (uint32_t)P.BN};
    int e = b2a_tmap16(&mw[gi], q.w_hi, 2, wdims, wstr, wbox, p.f16);
    if (!e) e = b2a_tmap16(&ml[gi], q.w_lo ? q.w_lo : q.w_hi, 2, wdims, wstr, wbox, p.f16);
    if (e) { b2a_set_error("b2a_conv1d_fused: cuTensorMapEncodeTiled failed (%d)", e); return B2A_E_CUDA; }
  }
  const bool dbg = p.dbg != nullptr || p.dbg_flags != 0;
  const auto kern = dbg ? conv_fused_kernel<true> : conv_fused_kernel<false>;
  B2A_SMEM_OPTIN(kern, DYN_SMEM_MAX);
  const int grid = tiles_total < nsm ? tiles_total : nsm;
  cudaError_t err = b2a_launch_pdl(kern, dim3(grid), dim3(THREADS), smem, (cudaStream_t)stream, p, mw[0], mw[1], mw[2], mw[3], ml[0], ml[1],
                                   ml[2], ml[3]);
  if (err != cudaSuccess) { b2a_set_error("b2a_conv1d_fused: launch failed: %s", cudaGetErrorString(err)); return B2A_E_CUDA; }
  B2A_CHECK_LAUNCH();
  for (int i = 0; i < 2 + 2 * MAXG; i++) g_last_cfg[i] = 0;
  g_last_cfg[0] = n; g_last_cfg[1] = grid;
  for (int gi = 0; gi < n; gi++) { g_last_cfg[2 + 2 * order[gi]] = p.pr[gi].BN; g_last_cfg[3 + 2 * order[gi]] = p.pr[gi].ksplit; }
  return B2A_OK;
}
