// Bidirectional LSTM recurrence (include/b200audio.h: b2a_lstm_bidir; reference modules.py:93-285).
// The recurrence is latency-bound: T sequential steps of a 1024x256 mat-vec.  One thread-block CLUSTER of 8 CTAs serves one
// (direction, batch) pair: each CTA owns 32 hidden units, i.e. 128 gate rows whose 128x256 slice of W_h lives entirely in REGISTERS
// (128 per thread, 256 threads) and is read from HBM once.  A step runs inside each warp with no CTA-wide barrier: the warp reads the
// previous h from shared memory, computes its 4 units' 16 gate rows, applies the gates and pushes its 4 new h values into all 8 CTAs'
// shared memory as one 16-byte `st.async ... mbarrier::complete_tx::bytes` per CTA, which delivers the data and signals the destination
// CTA's step barrier in one DSMEM transaction.  Each CTA arms that barrier with expect_tx(1 KiB) and every warp waits on its phase.
//
// Partition.  Lane (grp, half, k) = (lane >> 4, lane >> 3 & 1, lane & 7) holds 8 gate rows (i, f, g, o of the 2 units of row group grp)
// over the 16 columns {half*128 + 8i + k : i = 0..15}: 8 independent 16-long FMA chains per step.  A row's pre-activation is summed in
// a fixed order -- per half ((s0 + s1) + (s2 + s3)) + ((s4 + s5) + (s6 + s7)) over the k chains, then the two halves, then xproj -- by a
// reduce-scatter over lane bits 0, 1, 2 and an xor-8 shuffle, so every addition takes the same two operands whichever lane does it.
//
// h layout.  Column j = half*128 + 8i + k sits in slot p = (half*8 + k)*16 + i, so a lane's 16 columns are 4 aligned float4s; slot p is
// stored at hslot(p), which XORs the float4 index with p's bits 5-6 so that the 16 distinct float4s a warp reads at once fall in distinct
// bank groups.  Warp w of CTA rank owns the 4 units of slots rank*32 + w*4 + 0..3: one float4, pushed whole.
#include "common.cuh"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace {

constexpr int LH = 256, NCTA = 8, UPC = LH / NCTA;   // 32 units per CTA, 4 per warp

__device__ __forceinline__ int hslot(int p) { return p ^ (((p >> 5) & 3) << 2); }
__device__ __forceinline__ int slot_column(int p) { return ((p >> 7) << 7) | ((p & 15) << 3) | ((p >> 4) & 7); }

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
  uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r;
}
__device__ __forceinline__ void st_async_v4(uint32_t raddr, float4 v, uint32_t rbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
               ::"r"(raddr), "r"(__float_as_uint(v.x)), "r"(__float_as_uint(v.y)), "r"(__float_as_uint(v.z)), "r"(__float_as_uint(v.w)),
                 "r"(rbar) : "memory");
}
__device__ __forceinline__ void bar_wait_cluster(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok)
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
}

__global__ void __cluster_dims__(NCTA, 1, 1) __launch_bounds__(256, 1)
lstm_bidir_kernel(const float* __restrict__ xproj, const float* __restrict__ wh, float* __restrict__ out, int64_t out_ld, int T) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int k = lane & 7, half = (lane >> 3) & 1, grp = lane >> 4;
  const int p0 = rank * UPC + warp * 4;                             // slot of the warp's unit 0
  const int hk = half * 8 + k;                                      // this lane reads slots hk*16 + 0..15
  // after the reduce-scatter this lane holds gate `gate` of its unit (grp, lane & 1)
  const int gate = ((lane >> 1) & 1) * 2 + ((lane >> 2) & 1);
  const int unit = slot_column(p0 + grp * 2 + (lane & 1));
  __shared__ __align__(16) float hbuf[2][LH];
  __shared__ __align__(8) uint64_t hbar[2];                         // hbar[i]: "hbuf[i] holds the complete h of a step"

  float w[8][16];                                                   // row u*4 + g: gate g of unit (grp, u), columns half*128 + 8i + k
#pragma unroll
  for (int u = 0; u < 2; u++) {
    const int ju = slot_column(p0 + grp * 2 + u);
#pragma unroll
    for (int g = 0; g < 4; g++) {
      const float* wp = wh + ((int64_t)dir * 4 * LH + g * LH + ju) * LH + half * 128 + k;
#pragma unroll
      for (int i = 0; i < 16; i++) w[u * 4 + g][i] = __ldg(wp + 8 * i);
    }
  }
  for (int i = tid; i < 2 * LH; i += 256) (&hbuf[0][0])[i] = 0.f;   // step 0 reads h = 0
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&hbar[0])) : "memory");
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&hbar[1])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  float c = 0.f;
  const float* xp_base = xproj + (int64_t)b * T * 2 * 4 * LH + (int64_t)dir * 4 * LH + gate * LH + unit;
  float xp_cur = __ldg(xp_base + (int64_t)(dir == 0 ? 0 : T - 1) * 2 * 4 * LH);
  uint32_t rh = 0, rb = 0;                                          // lane q < 8 pushes to CTA q: its hbuf / hbar
  if (lane < NCTA) { rh = mapa(smem_addr(&hbuf[0][0]), lane); rb = mapa(smem_addr(&hbar[0]), lane); }
  const uint32_t push_off = (uint32_t)hslot(p0) * 4;
  cluster.sync();                                                   // zeros + barrier inits visible cluster-wide

  // No CTA-wide barrier in the loop; correctness rests on these invariants:
  //  - h is double-buffered.  A fast CTA cannot overwrite the buffer a slow warp is still reading: its next write there is the h of
  //    the following step, which needs this warp's own output of the current step, sent only after the warp's reads.  For the same
  //    reason no warp is ever more than one step ahead of another in the cluster.
  //  - complete_tx may reach a barrier before its arm (the phase cannot complete without the arm's arrival); thread 0 arms the next
  //    buffer at the start of each step, after it has itself waited on that buffer's previous phase.
  //  - the last step pushes nothing, and cluster.sync() before exit keeps every CTA alive while remote stores may target it.
  for (int step = 0; step < T; step++) {
    const int t = dir == 0 ? step : T - 1 - step;
    const int cur = step & 1, nxt = cur ^ 1;
    // arm the barrier that will collect THIS step's outputs (8 CTAs x 32 units x 4 bytes land in hbuf[nxt])
    if (tid == 0 && step + 1 < T)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(&hbar[nxt])), "r"(NCTA * UPC * 4) : "memory");
    float xp_next = 0.f;                                            // prefetch next step's input projection
    if (step + 1 < T) xp_next = __ldg(xp_base + (int64_t)(dir == 0 ? t + 1 : t - 1) * 2 * 4 * LH);
    if (step > 0) bar_wait_cluster(smem_addr(&hbar[cur]), ((step - 1) >> 1) & 1);     // h of step-1 complete in hbuf[cur]
    float hv[16];
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const float4 a = *reinterpret_cast<const float4*>(&hbuf[cur][hslot(hk * 16 + 4 * m)]);
      hv[4 * m] = a.x; hv[4 * m + 1] = a.y; hv[4 * m + 2] = a.z; hv[4 * m + 3] = a.w;
    }
    float s[8];
#pragma unroll
    for (int r = 0; r < 8; r++) s[r] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; i++) {
#pragma unroll
      for (int r = 0; r < 8; r++) s[r] = fmaf(w[r][i], hv[i], s[r]);
    }
    // reduce-scatter: lane bit 0 keeps the rows of unit (lane & 1), bit 1 gate bit 1, bit 2 gate bit 0
    const bool b0 = lane & 1, b1 = lane & 2, b2 = lane & 4;
    float s4[4], s2[2];
#pragma unroll
    for (int j = 0; j < 4; j++) s4[j] = (b0 ? s[4 + j] : s[j]) + __shfl_xor_sync(0xffffffffu, b0 ? s[j] : s[4 + j], 1);
#pragma unroll
    for (int j = 0; j < 2; j++) s2[j] = (b1 ? s4[2 + j] : s4[j]) + __shfl_xor_sync(0xffffffffu, b1 ? s4[j] : s4[2 + j], 2);
    float sh = (b2 ? s2[1] : s2[0]) + __shfl_xor_sync(0xffffffffu, b2 ? s2[0] : s2[1], 4);
    float v = sh + __shfl_xor_sync(0xffffffffu, sh, 8);             // the two halves
    v = v + xp_cur;
    // sigmoid / tanh through the SFU exponential and approximate division (abs error ~2e-7; libm's expf / tanhf cost ~150 cycles each)
    const float a = gate == 2 ? 1.f - __fdividef(2.f, 1.f + __expf(2.f * v)) : __fdividef(1.f, 1.f + __expf(-v));
    const int src = (lane & 0x19);                                  // lane of gate 0 of this lane's unit; gate g adds (g>>1)*2 + (g&1)*4
    const float gi = __shfl_sync(0xffffffffu, a, src), gf = __shfl_sync(0xffffffffu, a, src + 4);
    const float gg = __shfl_sync(0xffffffffu, a, src + 2), go = __shfl_sync(0xffffffffu, a, src + 6);
    c = fmaf(gf, c, gi * gg);
    const float hval = go * (1.f - __fdividef(2.f, 1.f + __expf(2.f * c)));
    if ((lane & 0xe) == 0) out[((int64_t)b * T + t) * out_ld + dir * LH + unit] = hval;     // lanes 0, 1, 16, 17: units 0..3
    const float4 h4 = make_float4(__shfl_sync(0xffffffffu, hval, 0), __shfl_sync(0xffffffffu, hval, 1),
                                  __shfl_sync(0xffffffffu, hval, 16), __shfl_sync(0xffffffffu, hval, 17));
    if (lane < NCTA && step + 1 < T)                                // the last step has no consumer: no store may outlive the CTA
      st_async_v4(rh + (uint32_t)(nxt * LH * 4) + push_off, h4, rb + (uint32_t)(nxt * 8));
    xp_cur = xp_next;
  }
  cluster.sync();                                                   // nobody exits while remote stores may still target it
}

}  // namespace

extern "C" int32_t b2a_lstm_bidir(const float* xproj, const float* wh, float* out, int64_t out_ld, int32_t B, int32_t T,
                                  int32_t H, void* stream) {
  B2A_CHECK_ARG(xproj && wh && out && B > 0 && T > 0, "bad pointers/shape");
  if (H != LH) { b2a_set_error("b2a_lstm_bidir: hidden size %d not supported (256)", H); return B2A_E_UNSUPPORTED; }
  lstm_bidir_kernel<<<dim3(NCTA, 2, B), 256, 0, (cudaStream_t)stream>>>(xproj, wh, out, out_ld, T);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
