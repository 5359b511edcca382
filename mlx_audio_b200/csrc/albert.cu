// Kokoro's ALBERT encoder layers as one persistent, cooperative tensor-core kernel (include/b200audio.h: b2a_albert_encoder).
//
// ALBERT shares one layer's weights across all of its layers, and at an utterance's T (~130 tokens) every GEMM of a layer is a few
// row blocks by a few thousand columns: a launch per GEMM spends most of its time in fill, drain and the gap to the next launch.  Here
// one grid of one CTA per SM runs every layer; per layer seven stages separated by grid-wide barriers:
//   0 qkv GEMM          epilogue writes the attention's fp16 Q (pre-scaled) / K / transposed, zero-padded V planes
//   1 attention         work unit = (head, 64-query block)
//   2 attn_out GEMM     + residual h                              -> t (fp32)
//   3 LayerNorm         t in place, and its bf16 planes (ffn's A)
//   4 ffn GEMM + GELU   bf16 planes only (ffn_out's A)
//   5 ffn_out GEMM      + residual t                              -> u (fp32)
//   6 LayerNorm         u -> h, and its bf16 planes (the next layer's qkv A)
// A GEMM work unit is 64 rows x 64 columns, warpgroup w owning columns [32 w, 32 w + 32); units are dealt round-robin over the grid.
// Every output element goes through the arithmetic of the separate kernels (conv_tc_kernel, attn_tc_kernel, layernorm_vec_kernel):
// the same wgmma m64nNk16 sequence over K (64-wide chunks in order, hi plane then lo plane), tc::epilogue_value, tc::attn_tc_tile and
// layernorm_row_vec, so the encoder's output equals the separate-op path bit for bit.
//
// Operand traffic (L2 -> SM, per layer, x2 planes, M = ceil(T / 64) row blocks): a GEMM with N columns and K channels reads its A
// rows N / 64 times and its weights M times: (N / 64) * M * 64 * K * 2 B * 2 planes + M * N * K * 2 B.  At T = 130 (M = 3): qkv
// 10.6 + 10.6, attn_out 3.5 + 3.5, ffn 9.4 + 9.4, ffn_out 9.4 + 9.4 MB, 66 MB per layer against the 110 MB of the 128-row, 32-column
// tiles of the launch chain.
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (MMA, epilogue, attention, LayerNorm rows), warp 8 = TMA producer.
// The producer runs ahead through a ring of SLOTS operand stages shared by all stages of all layers; weight tiles do not depend on the
// previous stage, so it issues the first ring's weight loads of a GEMM stage before it waits at the grid barrier.
//
// Grid barrier: a counter reset by a memset node in front of every launch; a CTA arrives with a gpu-scope release once all its
// consumer threads have written the stage, and waits with a gpu-scope acquire for (stage index) x (grid size) arrivals.  The
// epilogues write operand planes through the generic proxy that the next stage reads through TMA (the async proxy): the writers fence
// the proxies before arriving and the producer after its acquire.  The launch is cooperative, so a grid that cannot be co-resident fails
// at launch.  The wait is bounded: after TIMEOUT_NS without progress a CTA sets the error word and stops waiting at barriers (it then
// runs to its end on whatever data it finds, in bounded time: every other wait is on work the same CTA issues).
#include "common.cuh"
#include "tc_common.cuh"
#include "tc_epilogue.cuh"
#include "attn_tc_tile.cuh"
#include "layernorm_row.cuh"

using namespace tc;

namespace {

constexpr int THREADS = 288;
constexpr int SLOTS = 6;
constexpr int SLOT_BYTES = 32768;                  // GEMM: A hi 8K | A lo 8K | W 8K;  attention: K hi | K lo | V^T hi | V^T lo, 8K each
constexpr int PLANE = 64 * 128;                    // one 64-row x 64-channel 16-bit tile (128B-swizzled rows)
constexpr int OFF_Q = SLOTS * SLOT_BYTES;          // Q hi 8K | Q lo 8K
constexpr int OFF_BAR = OFF_Q + 2 * PLANE;
constexpr int SMEM_BYTES = OFF_BAR + (2 * SLOTS + 2) * 8 + 16 + 1024;
constexpr int STAGES = 7;                          // per layer
constexpr long long TIMEOUT_NS = 10000000000LL;    // 10 s

struct AlbertMaps {                                // GEMM g = qkv, attn_out, ffn, ffn_out
  CUtensorMap a_hi[4], a_lo[4], w[4];
  CUtensorMap qh, ql, kh, kl, vh, vl;
};

struct AlbertParams {
  int T, layers, planes, mb, H, hs, inter, nkt;
  int N[4], K[4];
  const float* bias[4];
  const float *ln_w[2], *ln_b[2]; float eps;
  float qmul;
  float *h, *t, *u;                                // fp32 [T][hs]
  __nv_bfloat16 *hp_hi, *hp_lo, *ap_hi, *ap_lo, *fp_hi, *fp_lo;    // bf16 planes (cp: written by the attention, read by TMA only)
  __nv_bfloat16 *cp_hi, *cp_lo;
  AttnOperands attn;
  unsigned* bar; unsigned* err;
  long long* tl;                                   // timeline build: [layers * STAGES][grid][2] globaltimer at stage start / end
};

// the GEMM (qkv, attn_out, ffn, ffn_out) a stage runs, -1 for the attention and the LayerNorms
__device__ __forceinline__ int gemm_of_stage(int s) { return s == 0 ? 0 : s == 2 ? 1 : s == 4 ? 2 : s == 5 ? 3 : -1; }

__device__ __forceinline__ long long globaltimer() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// true when `target` arrivals have been seen; false (and the error word set) after TIMEOUT_NS, or at once when it is already set
__device__ bool grid_wait(const AlbertParams& p, unsigned target) {
  long long t0 = 0;
  for (int it = 0;; it++) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p.bar) : "memory");
    if ((int)(v - target) >= 0) return true;
    if ((it & 63) == 63) {
      if (*(volatile unsigned*)p.err) return false;
      const long long now = globaltimer();
      if (!t0) t0 = now;
      else if (now - t0 > TIMEOUT_NS) { atomicExch(p.err, 1u); return false; }
    }
    __nanosleep(64);
  }
}

__device__ __forceinline__ void grid_arrive(unsigned* bar) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
}

__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

template <bool TL>
__global__ void __launch_bounds__(THREADS, 1) albert_kernel(const __grid_constant__ AlbertMaps maps, const AlbertParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + OFF_BAR);
  uint64_t* empty = full + SLOTS;
  uint64_t* q_full = empty + SLOTS;
  uint64_t* q_empty = q_full + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bid = blockIdx.x, grid = gridDim.x;
  const int total = p.layers * STAGES;

  if (warp == 8 && lane == 0) {
    for (int g = 0; g < 4; g++) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.a_hi[g]) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.w[g]) : "memory");
    }
    for (int s = 0; s < SLOTS; s++) { mbar_init(full + s, 1); mbar_init(empty + s, 2); }
    mbar_init(q_full, 1); mbar_init(q_empty, 2);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane != 0) return;
    uint32_t g = 0, qn = 0;
    for (int k = 0; k < total; k++) {
      const int stage = k % STAGES, gi = gemm_of_stage(stage);
      if (stage == 1) {
        const int units = p.H * p.mb;
        if (bid >= units) continue;
        grid_wait(p, (unsigned)k * grid);
        fence_proxy_async_global();
        for (int u = bid; u < units; u += grid) {
          const int head = u / p.mb, q0 = (u % p.mb) * 64;
          mbar_wait(q_empty, (qn & 1) ^ 1);
          mbar_expect_tx(q_full, 2 * PLANE);
          tma_load_3d(smem + OFF_Q, &maps.qh, q_full, 0, q0, head);
          tma_load_3d(smem + OFF_Q + PLANE, &maps.ql, q_full, 0, q0, head);
          qn++;
          for (int t = 0; t < p.nkt; t++, g++) {
            const int s = g % SLOTS;
            uint8_t* st = smem + (size_t)s * SLOT_BYTES;
            mbar_wait(empty + s, ((g / SLOTS) & 1) ^ 1);
            mbar_expect_tx(full + s, 4 * PLANE);
            tma_load_3d(st, &maps.kh, full + s, 0, t * 64, head);
            tma_load_3d(st + PLANE, &maps.kl, full + s, 0, t * 64, head);
            tma_load_3d(st + 2 * PLANE, &maps.vh, full + s, t * 64, 0, head);
            tma_load_3d(st + 3 * PLANE, &maps.vl, full + s, t * 64, 0, head);
          }
        }
        continue;
      }
      if (gi < 0) continue;
      const int units = p.mb * (p.N[gi] / 64), kc = p.K[gi] / 64;
      const uint32_t bytes = (uint32_t)(PLANE * p.planes + PLANE);
      bool waited = k == 0;
      for (int u = bid; u < units; u += grid) {
        const int m0 = (u % p.mb) * 64, n0 = (u / p.mb) * 64;
        int pre = 0;
        if (!waited) {
          pre = kc < SLOTS ? kc : SLOTS;
          for (int c = 0; c < pre; c++) {
            const uint32_t gc = g + c;
            const int s = gc % SLOTS;
            mbar_wait(empty + s, ((gc / SLOTS) & 1) ^ 1);
            mbar_expect_tx(full + s, bytes);
            tma_load_2d(smem + (size_t)s * SLOT_BYTES + 2 * PLANE, &maps.w[gi], full + s, c * 64, n0);
          }
          grid_wait(p, (unsigned)k * grid);
          fence_proxy_async_global();
          waited = true;
          for (int c = 0; c < pre; c++) {
            const int s = (g + c) % SLOTS;
            uint8_t* st = smem + (size_t)s * SLOT_BYTES;
            tma_load_2d(st, &maps.a_hi[gi], full + s, c * 64, m0);
            if (p.planes == 2) tma_load_2d(st + PLANE, &maps.a_lo[gi], full + s, c * 64, m0);
          }
        }
        for (int c = pre; c < kc; c++) {
          const uint32_t gc = g + c;
          const int s = gc % SLOTS;
          uint8_t* st = smem + (size_t)s * SLOT_BYTES;
          mbar_wait(empty + s, ((gc / SLOTS) & 1) ^ 1);
          mbar_expect_tx(full + s, bytes);
          tma_load_2d(st + 2 * PLANE, &maps.w[gi], full + s, c * 64, n0);
          tma_load_2d(st, &maps.a_hi[gi], full + s, c * 64, m0);
          if (p.planes == 2) tma_load_2d(st + PLANE, &maps.a_lo[gi], full + s, c * 64, m0);
        }
        g += kc;
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg, thread ct of 256 =====
  const int ct = threadIdx.x, wg = warp >> 2, w4 = warp & 3;
  const uint32_t sb = smem_u32(smem);
  uint32_t g = 0, qn = 0;
  for (int k = 0; k < total; k++) {
    const int stage = k % STAGES, gi = gemm_of_stage(stage);
    if (k > 0) {
      if (ct == 0) grid_wait(p, (unsigned)k * grid);
      bar_sync(1, 256);
    }
    if constexpr (TL) { if (ct == 0) p.tl[((int64_t)k * grid + bid) * 2] = globaltimer(); }
    if (gi >= 0) {
      // ---- GEMM: unit = rows [m0, m0 + 64) x columns [n0, n0 + 64)
      const int units = p.mb * (p.N[gi] / 64), kc = p.K[gi] / 64, N = p.N[gi];
      const float* bias = p.bias[gi];
      for (int u = bid; u < units; u += grid) {
        const int m0 = (u % p.mb) * 64, n0 = (u / p.mb) * 64;
        float acc[16];
        int prev = -1;
        for (int c = 0; c < kc; c++, g++) {
          const int s = g % SLOTS;
          mbar_wait(full + s, (g / SLOTS) & 1);
          const uint32_t st = sb + s * SLOT_BYTES;
          const uint64_t ad = gmma_desc_sw128(st), wd = gmma_desc_sw128(st + 2 * PLANE + wg * 32 * 128);
          wgmma_fence();
          wgmma_chunk<1, false>(acc, ad, wd, c != 0);
          if (p.planes == 2) wgmma_chunk<1, false>(acc, gmma_desc_sw128(st + PLANE), wd, 1u);
          wgmma_commit();
          wgmma_wait<1>();
          wgmma_fence_regs<16>(acc);
          if (prev >= 0 && (ct & 127) == 0) mbar_arrive(empty + prev);
          prev = s;
        }
        wgmma_wait<0>();
        wgmma_fence_regs<16>(acc);
        if ((ct & 127) == 0) mbar_arrive(empty + prev);
        // epilogue straight from the accumulator: element 4j + 2hh + e = row m0 + 16 w4 + lane / 4 + 8 hh, column 8j + 2 (lane % 4) + e
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int n = n0 + wg * 32 + 8 * j + 2 * (lane & 3);
          const float b0 = __ldg(bias + n), b1 = __ldg(bias + n + 1);
          EmitCol e0{}, e1{};
          if (gi == 0) { e0 = emit_col_attn(p.attn, 0, p.T, p.hs, p.qmul, n); e1 = emit_col_attn(p.attn, 0, p.T, p.hs, p.qmul, n + 1); }
#pragma unroll
          for (int hh = 0; hh < 2; hh++) {
            const int row = m0 + 16 * w4 + (lane >> 2) + 8 * hh;
            const float a0 = acc[4 * j + 2 * hh], a1 = acc[4 * j + 2 * hh + 1];
            if (row >= p.T) {
              if (gi == 0 && e0.step == 1 && row < p.attn.tkp) { e0.hi[row] = 0; e0.lo[row] = 0; e1.hi[row] = 0; e1.lo[row] = 0; }
              continue;
            }
            const int64_t o = (int64_t)row * N + n;
            if (gi == 0) {
              emit_store(e0, row, epilogue_value(a0, b0, 0, 0.f, 1.f, 0.f));
              emit_store(e1, row, epilogue_value(a1, b1, 0, 0.f, 1.f, 0.f));
            } else if (gi == 2) {
              const float y0 = epilogue_value(a0, b0, B2A_ACT_GELU, 0.f, 1.f, 0.f), y1 = epilogue_value(a1, b1, B2A_ACT_GELU, 0.f, 1.f, 0.f);
              __nv_bfloat162 h2, l2;
              split16(y0, h2.x, l2.x);
              split16(y1, h2.y, l2.y);
              *reinterpret_cast<__nv_bfloat162*>(p.fp_hi + o) = h2;
              if (p.planes == 2) *reinterpret_cast<__nv_bfloat162*>(p.fp_lo + o) = l2;
            } else {
              const float* res = gi == 1 ? p.h : p.t;
              float* out = gi == 1 ? p.t : p.u;
              const float2 r = *reinterpret_cast<const float2*>(res + o);
              *reinterpret_cast<float2*>(out + o) = make_float2(epilogue_value(a0, b0, 0, 0.f, 1.f, r.x), epilogue_value(a1, b1, 0, 0.f, 1.f, r.y));
            }
          }
        }
      }
    } else if (stage == 1) {
      // ---- attention: unit = (head, 64-query block), computed by warpgroup 0; warpgroup 1 only keeps the ring's count
      const int units = p.H * p.mb;
      for (int u = bid; u < units; u += grid, qn++) {
        const int head = u / p.mb, q0 = (u % p.mb) * 64;
        float o[32], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 32; j++) o[j] = 0.f;
        const int kmax[2] = {p.T - 1, p.T - 1}, kmin[2] = {0, 0};
        const uint64_t dqh = gmma_desc_sw128(sb + OFF_Q), dql = gmma_desc_sw128(sb + OFF_Q + PLANE);
        mbar_wait(q_full, qn & 1);
        for (int t = 0; t < p.nkt; t++, g++) {
          const int s = g % SLOTS;
          const uint32_t st = sb + s * SLOT_BYTES;
          mbar_wait(full + s, (g / SLOTS) & 1);
          if (wg == 0)
            attn_tc_tile(o, m, l, dqh, dql, gmma_desc_sw128(st), gmma_desc_sw128(st + PLANE), gmma_desc_sw128(st + 2 * PLANE),
                         gmma_desc_sw128(st + 3 * PLANE), t * 64, kmax, kmin, lane);
          if ((ct & 127) == 0) mbar_arrive(empty + s);
        }
        if ((ct & 127) == 0) mbar_arrive(q_empty);
        if (wg == 0) {
          float inv[2];
          attn_tc_row_inv(l, inv);
#pragma unroll
          for (int hh = 0; hh < 2; hh++) {
            const int q = q0 + w4 * 16 + (lane >> 2) + 8 * hh;
            if (q < p.T) {
              const int64_t e = (int64_t)q * p.hs + head * 64 + 2 * (lane & 3);
#pragma unroll
              for (int j = 0; j < 8; j++) {
                __nv_bfloat162 eh, el;
                split16(o[4 * j + 2 * hh] * inv[hh], eh.x, el.x);
                split16(o[4 * j + 2 * hh + 1] * inv[hh], eh.y, el.y);
                *reinterpret_cast<__nv_bfloat162*>(p.cp_hi + e + 8 * j) = eh;
                if (p.planes == 2) *reinterpret_cast<__nv_bfloat162*>(p.cp_lo + e + 8 * j) = el;
              }
            }
          }
        }
      }
    } else {
      // ---- LayerNorm: one warp per row
      const int which = stage == 3 ? 0 : 1;
      const float* x = which ? p.u : p.t;
      float* y = which ? p.h : p.t;
      __nv_bfloat16* eh = which ? p.hp_hi : p.ap_hi;
      __nv_bfloat16* el = p.planes == 2 ? (which ? p.hp_lo : p.ap_lo) : nullptr;
      for (int row = bid * 8 + warp; row < p.T; row += grid * 8) {
        const int64_t o = (int64_t)row * p.hs;
        layernorm_row_vec<8>(x + o, nullptr, y + o, p.hs, p.ln_w[which], p.ln_b[which], nullptr, p.eps, 0, 0, 0.f, eh + o,
                             el ? el + o : nullptr, lane);
      }
    }
    if constexpr (TL) { if (ct == 0) p.tl[((int64_t)k * grid + bid) * 2 + 1] = globaltimer(); }
    if (k + 1 < total) {
      fence_proxy_async_global();                          // this thread's generic writes, before the next stage's TMA reads
      bar_sync(1, 256);
      if (ct == 0) { __threadfence(); grid_arrive(p.bar); }
    }
  }
}

// workspace: barrier counter | t | u (fp32 [T][hs]) | cp, ap (bf16 hi, lo [T][hs]) | fp (bf16 hi, lo [T][inter]) | attention operands
struct WsLayout { int64_t t, u, cp_hi, cp_lo, ap_hi, ap_lo, fp_hi, fp_lo, attn, total; };
WsLayout ws_layout(int64_t T, int64_t H, int64_t hs, int64_t inter) {
  auto up = [](int64_t x) { return (x + 255) / 256 * 256; };
  WsLayout w;
  int64_t o = 256;
  w.t = o; o += up(T * hs * 4);
  w.u = o; o += up(T * hs * 4);
  w.cp_hi = o; o += up(T * hs * 2);
  w.cp_lo = o; o += up(T * hs * 2);
  w.ap_hi = o; o += up(T * hs * 2);
  w.ap_lo = o; o += up(T * hs * 2);
  w.fp_hi = o; o += up(T * inter * 2);
  w.fp_lo = o; o += up(T * inter * 2);
  w.attn = o; o += b2a_attention_tc_ws_bytes(1, (int32_t)H, (int32_t)T, (int32_t)T);
  w.total = o;
  return w;
}

}  // namespace

extern "C" int64_t b2a_albert_ws_bytes(int32_t T, int32_t heads, int32_t hidden, int32_t inter) {
  return ws_layout(T, heads, hidden, inter).total;
}

extern "C" int32_t b2a_albert_encoder(const b2a_albert_t* a, void* ws, uint32_t* err, int64_t* timeline, void* stream) {
  B2A_CHECK_ARG(a && ws && err && a->h && a->h_hi && (a->planes == 1 || (a->planes == 2 && a->h_lo)), "null pointer");
  for (int i = 0; i < 4; i++) B2A_CHECK_ARG(a->w[i] && a->bias[i], "null weight or bias");
  for (int i = 0; i < 2; i++) B2A_CHECK_ARG(a->ln_w[i] && a->ln_b[i], "null LayerNorm parameter");
  B2A_CHECK_ARG(a->T >= 64 && a->T <= 512 && a->layers > 0 && a->heads > 0 && a->hidden == 64 * a->heads && a->hidden <= 1024 &&
                a->inter % 64 == 0 && a->inter > 0, "shape: 64 <= T <= 512, hidden = 64 * heads <= 1024, inter a multiple of 64");
  const int T = a->T, H = a->heads, hs = a->hidden, inter = a->inter;
  uint8_t* base = (uint8_t*)ws;
  B2A_CHECK_ARG(((uintptr_t)base & 255) == 0, "workspace must be 256-byte aligned");
  const WsLayout L = ws_layout(T, H, hs, inter);
  cudaStream_t st = (cudaStream_t)stream;

  AlbertParams p{};
  p.T = T; p.layers = a->layers; p.planes = a->planes; p.mb = cdiv(T, 64); p.H = H; p.hs = hs; p.inter = inter; p.nkt = cdiv(T, 64);
  const int N[4] = {3 * hs, hs, inter, hs}, K[4] = {hs, hs, hs, inter};
  for (int i = 0; i < 4; i++) { p.N[i] = N[i]; p.K[i] = K[i]; p.bias[i] = a->bias[i]; }
  for (int i = 0; i < 2; i++) { p.ln_w[i] = a->ln_w[i]; p.ln_b[i] = a->ln_b[i]; }
  p.eps = a->eps;
  p.qmul = a->scale * 1.4426950408889634f;          // as b2a_conv1d_tc pre-scales Q for b2a_attention_tc
  p.h = a->h; p.t = (float*)(base + L.t); p.u = (float*)(base + L.u);
  p.hp_hi = (__nv_bfloat16*)a->h_hi; p.hp_lo = (__nv_bfloat16*)a->h_lo;
  p.cp_hi = (__nv_bfloat16*)(base + L.cp_hi); p.cp_lo = (__nv_bfloat16*)(base + L.cp_lo);
  p.ap_hi = (__nv_bfloat16*)(base + L.ap_hi); p.ap_lo = (__nv_bfloat16*)(base + L.ap_lo);
  p.fp_hi = (__nv_bfloat16*)(base + L.fp_hi); p.fp_lo = (__nv_bfloat16*)(base + L.fp_lo);
  p.attn = attn_operands(base + L.attn, H, T, T);
  p.bar = (unsigned*)base; p.err = err;
  p.tl = (long long*)timeline;

  AlbertMaps m;
  const void* a_hi[4] = {p.hp_hi, p.cp_hi, p.ap_hi, p.fp_hi};
  const void* a_lo[4] = {p.hp_lo, p.cp_lo, p.ap_lo, p.fp_lo};
  const uint32_t box[3] = {64, 64, 1};              // every operand map: 64 x 64 (x 1) tiles
  int e = 0;
  for (int i = 0; i < 4 && !e; i++) {
    const uint64_t ad[2] = {(uint64_t)K[i], (uint64_t)T}, as[1] = {(uint64_t)K[i] * 2};
    const uint64_t wd[2] = {(uint64_t)K[i], (uint64_t)N[i]};
    e = b2a_tmap16(&m.a_hi[i], a_hi[i], 2, ad, as, box, false);
    if (!e) e = b2a_tmap16(&m.a_lo[i], a->planes == 2 ? a_lo[i] : a_hi[i], 2, ad, as, box, false);
    if (!e) e = b2a_tmap16(&m.w[i], a->w[i], 2, wd, as, box, false);
  }
  const uint64_t qd[3] = {64, (uint64_t)T, (uint64_t)H}, qs[2] = {128, (uint64_t)T * 128};
  const uint64_t vd[3] = {(uint64_t)p.attn.tkp, 64, (uint64_t)H}, vs[2] = {(uint64_t)p.attn.tkp * 2, (uint64_t)p.attn.tkp * 128};
  if (!e) e = b2a_tmap16(&m.qh, p.attn.qh, 3, qd, qs, box, true);
  if (!e) e = b2a_tmap16(&m.ql, p.attn.ql, 3, qd, qs, box, true);
  if (!e) e = b2a_tmap16(&m.kh, p.attn.kh, 3, qd, qs, box, true);
  if (!e) e = b2a_tmap16(&m.kl, p.attn.kl, 3, qd, qs, box, true);
  if (!e) e = b2a_tmap16(&m.vh, p.attn.vh, 3, vd, vs, box, true);
  if (!e) e = b2a_tmap16(&m.vl, p.attn.vl, 3, vd, vs, box, true);
  if (e) { b2a_set_error("b2a_albert_encoder: cuTensorMapEncodeTiled failed (%d)", e); return B2A_E_CUDA; }

  void (*kern)(const AlbertMaps, const AlbertParams) = timeline ? albert_kernel<true> : albert_kernel<false>;
  B2A_SMEM_OPTIN(kern, SMEM_BYTES);
  // one CTA per SM, as many as can be co-resident (the cooperative launch refuses a grid that cannot)
  const int nsm = b2a_device_sm_count();
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, THREADS, SMEM_BYTES) != cudaSuccess || per_sm < 1 || nsm < 1) {
    b2a_set_error("b2a_albert_encoder: the kernel cannot be resident (%s)", cudaGetErrorString(cudaGetLastError()));
    return B2A_E_CUDA;
  }
  if (cudaMemsetAsync(p.bar, 0, 4, st) != cudaSuccess) { b2a_set_error("b2a_albert_encoder: %s", cudaGetErrorString(cudaGetLastError())); return B2A_E_CUDA; }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(nsm); cfg.blockDim = dim3(THREADS); cfg.dynamicSmemBytes = SMEM_BYTES; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  if (cudaLaunchKernelEx(&cfg, kern, m, p) != cudaSuccess) {
    b2a_set_error("b2a_albert_encoder: %s", cudaGetErrorString(cudaGetLastError()));
    return B2A_E_CUDA;
  }
  return B2A_OK;
}
