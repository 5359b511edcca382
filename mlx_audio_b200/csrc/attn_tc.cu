// Flash attention on the Hopper tensor cores (include/b200audio.h: b2a_attention_tc) for head_dim 64:
// replaces mx.fast.scaled_dot_product_attention in the Whisper encoder / decoder prefill, Kokoro's ALBERT, Mimi and the
// Qwen3 vocoder transformer (whisper.py:369-385, modules.py:519-560, mimi/modules/transformer.py:79-112,
// speech_tokenizer.py:265-303).
//
// One CTA = 128 queries of one (batch, head), two consumer warpgroups of 64 query rows each; key tiles of 64.  Per key tile:
//   S = Q K^T        wgmma M64 x N64 x K16 from shared memory, operands fp16 hi/lo planes (3 products: hi*hi, lo*hi, hi*lo ->
//                    fp32-grade scores), fp32 accumulator in registers
//   softmax          on the accumulator fragments: a thread holds two rows x 16 columns; row max / sum over the four lanes of a quad
//   O_tile = P V     wgmma with A = P from registers (fp16 hi/lo, converted in place from the score fragments: the accumulator layout
//                    of M64 x N64 is the A-operand layout of four K16 steps) against V^T tiles (K-major, prepared by the prologue kernel);
//                    O = alpha O + O_tile in fp32 registers
// Q (pre-scaled by scale*log2 e so that exp2 is the only transcendental), K and V^T are converted once per call by
// attn_tc_prep_kernel; K/V tiles arrive by TMA into a two-stage ring (out-of-range keys zero-filled by the TMA unit and masked in the
// softmax).  Warp roles (288 threads): warps 0..7 = consumers, warp 8 = TMA producer.
#include "common.cuh"
#include "tc_common.cuh"
#include "attn_tc_tile.cuh"

using namespace tc;

namespace {

constexpr int BM = 128, BN = 64, HD = 64;
constexpr int THREADS = 288;

struct AtcParams {
  int B, H, Tq, Tk;
  int causal, q_offset, window;
  float* o; int64_t o_bs, o_ld;          // [B, Tq, H*64] fp32
  __nv_bfloat16 *e_hi, *e_lo; int64_t e_ld;   // optional bf16 hi / lo planes of o, [B, Tq, e_ld] (the next GEMM's A operand)
};

// ---- prologue: fp32 [B,T,H*64] -> fp16 hi/lo planes.  q,k: [B*H, T, 64];  v: transposed [B*H, 64, Tkp] (zero-padded keys)
__global__ void attn_tc_prep_qk_kernel(const float* x, int64_t x_bs, int64_t x_ld, int B, int H, int T, float mul, __half* hi, __half* lo) {
  const int64_t total = (int64_t)B * H * T * (HD / 8);
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % (HD / 8));
    const int64_t r = idx / (HD / 8);
    const int t = (int)(r % T);
    const int h = (int)((r / T) % H), b = (int)(r / ((int64_t)T * H));
    const float* src = x + (int64_t)b * x_bs + (int64_t)t * x_ld + h * HD + c8 * 8;
    float4 a = *reinterpret_cast<const float4*>(src), c = *reinterpret_cast<const float4*>(src + 4);
    float v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
    __align__(16) __half hh[8], ll[8];
#pragma unroll
    for (int j = 0; j < 8; j++) split16(v[j] * mul, hh[j], ll[j]);
    const int64_t dst = (((int64_t)b * H + h) * T + t) * HD + c8 * 8;
    *reinterpret_cast<uint4*>(hi + dst) = *reinterpret_cast<uint4*>(hh);
    *reinterpret_cast<uint4*>(lo + dst) = *reinterpret_cast<uint4*>(ll);
  }
}
// tile 64 keys x 64 dims through shared memory: out[bh][d][t]
__global__ void attn_tc_prep_vt_kernel(const float* v, int64_t v_bs, int64_t v_ld, int B, int H, int T, int Tp, __half* hi, __half* lo) {
  __shared__ float tile[64][65];
  const int t0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z;
  for (int i = threadIdx.x; i < 64 * 64; i += blockDim.x) {
    const int d = i & 63, tt = i >> 6;
    const int t = t0 + tt;
    tile[tt][d] = t < T ? v[(int64_t)b * v_bs + (int64_t)t * v_ld + h * HD + d] : 0.f;
  }
  __syncthreads();
  const int64_t base = ((int64_t)b * H + h) * HD;
  for (int i = threadIdx.x; i < 64 * 64; i += blockDim.x) {
    const int tt = i & 63, d = i >> 6;
    const int t = t0 + tt;
    if (t < Tp) {
      __half hh, ll;
      split16(tile[tt][d], hh, ll);
      hi[(base + d) * Tp + t] = hh;
      lo[(base + d) * Tp + t] = ll;
    }
  }
}

// smem (1024-aligned): Qh 16K | Ql 16K | [2] x { Kh 8K | Kl 8K | Vh 8K | Vl 8K } | barriers
constexpr int OFF_QH = 0, OFF_QL = 16384, OFF_KV = 32768, KV_STAGE = 32768, OFF_KH = 0, OFF_KL = 8192, OFF_VH = 16384, OFF_VL = 24576,
              OFF_BAR = OFF_KV + 2 * KV_STAGE, SMEM_BYTES = OFF_BAR + 128 + 1024;

__global__ void __launch_bounds__(THREADS, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap map_qh, const __grid_constant__ CUtensorMap map_ql,
               const __grid_constant__ CUtensorMap map_kh, const __grid_constant__ CUtensorMap map_kl,
               const __grid_constant__ CUtensorMap map_vh, const __grid_constant__ CUtensorMap map_vl, const AtcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = (uint64_t*)(smem + OFF_BAR);
  uint64_t *q_full = bars, *kv_full = bars + 1 /* [2] */, *kv_empty = bars + 3 /* [2] */;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BM, bh = blockIdx.y;

  // key-tile range of this query tile (uniform over its rows: conservative superset, exact mask applied per element)
  int k_hi = p.Tk;                                               // exclusive
  if (p.causal) { const int last = q0 + BM - 1 + p.q_offset + 1; if (last < k_hi) k_hi = last; }
  int k_lo = 0;
  if (p.window > 0) { const int first = q0 + p.q_offset - p.window + 1; if (first > 0) k_lo = first; }
  const int t_lo = k_lo / BN, t_hi = k_hi > 0 ? (k_hi + BN - 1) / BN : 0;
  const int nt = t_hi > t_lo ? t_hi - t_lo : 0;

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_qh) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_kh) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_vh) : "memory");
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; s++) { mbar_init(kv_full + s, 1); mbar_init(kv_empty + s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                                                    // the operand planes are the predecessor's output

  if (warp == 8) {
    if (lane == 0 && nt > 0) {
      mbar_expect_tx(q_full, 32768);
      tma_load_3d(smem + OFF_QH, &map_qh, q_full, 0, q0, bh);
      tma_load_3d(smem + OFF_QL, &map_ql, q_full, 0, q0, bh);
      for (int t = 0; t < nt; t++) {
        const int kt = (t_lo + t) * BN, s = t & 1;
        uint8_t* st = smem + OFF_KV + s * KV_STAGE;
        mbar_wait(kv_empty + s, ((t >> 1) & 1) ^ 1);
        mbar_expect_tx(kv_full + s, 32768);
        tma_load_3d(st + OFF_KH, &map_kh, kv_full + s, 0, kt, bh);
        tma_load_3d(st + OFF_KL, &map_kl, kv_full + s, 0, kt, bh);
        tma_load_3d(st + OFF_VH, &map_vh, kv_full + s, kt, 0, bh);
        tma_load_3d(st + OFF_VL, &map_vl, kv_full + s, kt, 0, bh);
      }
    }
    return;
  }

  // ===== consumer warpgroup wg: query rows [64 wg, 64 wg + 64) of the tile; this thread holds rows r[0], r[1] =====
  const int wg = warp >> 2, w4 = warp & 3;
  int qpos[2], kmax[2], kmin[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int row = wg * 64 + w4 * 16 + (lane >> 2) + 8 * h;
    qpos[h] = q0 + row + p.q_offset;                             // its position on the key axis (causal / window)
    kmax[h] = p.Tk - 1;                                          // last allowed key
    if (p.causal && qpos[h] < kmax[h]) kmax[h] = qpos[h];
    kmin[h] = p.window > 0 ? qpos[h] - p.window + 1 : 0;
  }
  float o[32];
#pragma unroll
  for (int j = 0; j < 32; j++) o[j] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t sb = smem_u32(smem);
  const uint64_t dqh = gmma_desc_sw128(sb + OFF_QH + wg * 8192), dql = gmma_desc_sw128(sb + OFF_QL + wg * 8192);
  if (nt > 0) mbar_wait(q_full, 0);
  for (int t = 0; t < nt; t++) {
    const int kt = (t_lo + t) * BN, s = t & 1;
    const uint32_t st = sb + OFF_KV + s * KV_STAGE;
    const uint64_t dkh = gmma_desc_sw128(st + OFF_KH), dkl = gmma_desc_sw128(st + OFF_KL);
    const uint64_t dvh = gmma_desc_sw128(st + OFF_VH), dvl = gmma_desc_sw128(st + OFF_VL);
    mbar_wait(kv_full + s, (t >> 1) & 1);
    attn_tc_tile(o, m, l, dqh, dql, dkh, dkl, dvh, dvl, kt, kmax, kmin, lane);
    if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty + s);     // both warpgroups release the stage
  }
  pdl_launch_dependents();
  // ---- write out: a quad of lanes covers 8 consecutive columns (32 B) of a row
  float inv[2];
  attn_tc_row_inv(l, inv);
  const int b = bh / p.H, hh = bh % p.H;
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int q = q0 + wg * 64 + w4 * 16 + (lane >> 2) + 8 * h;
    if (q < p.Tq) {
      float* dst = p.o + (int64_t)b * p.o_bs + (int64_t)q * p.o_ld + hh * HD + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 8; j++)
        *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[4 * j + 2 * h] * inv[h], o[4 * j + 2 * h + 1] * inv[h]);
      if (p.e_hi) {
        const int64_t e = ((int64_t)b * p.Tq + q) * p.e_ld + hh * HD + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 8; j++) {
          __nv_bfloat162 eh, el;
          split16(o[4 * j + 2 * h] * inv[h], eh.x, el.x);
          split16(o[4 * j + 2 * h + 1] * inv[h], eh.y, el.y);
          *reinterpret_cast<__nv_bfloat162*>(p.e_hi + e + 8 * j) = eh;
          if (p.e_lo) *reinterpret_cast<__nv_bfloat162*>(p.e_lo + e + 8 * j) = el;
        }
      }
    }
  }
}

}  // namespace

extern "C" int64_t b2a_attention_tc_ws_bytes(int32_t B, int32_t H, int32_t Tq, int32_t Tk) {
  const int64_t bh = (int64_t)B * H;
  return 2 * 2 * (bh * Tq * HD + bh * Tk * HD + bh * HD * (((int64_t)Tk + 7) / 8 * 8)) + 1024;
}

extern "C" int32_t b2a_attention_tc(const b2a_attn_t* a, void* ws, void* stream) {
  B2A_CHECK_ARG(a && ws && a->o && (a->operands_ready || (a->q && a->k && a->v)), "null pointer");
  B2A_CHECK_ARG(a->D == 64 && a->H == a->Hkv && a->k_len == nullptr, "tensor-core attention: head_dim 64, no GQA, no per-row key length");
  B2A_CHECK_ARG(a->B > 0 && a->Tq > 0 && a->Tk > 0 && a->H > 0, "bad shape");
  B2A_CHECK_ARG(a->window <= 0 || a->causal, "a sliding window needs causal masking");
  B2A_CHECK_ARG(a->operands_ready ||
                (a->q_ld % 4 == 0 && a->k_ld % 4 == 0 && a->q_bs % 4 == 0 && a->k_bs % 4 == 0 && ((uintptr_t)a->q & 15) == 0 && ((uintptr_t)a->k & 15) == 0),
                "q/k rows must be 16-byte aligned");
  B2A_CHECK_ARG(a->o_ld % 4 == 0 && a->o_bs % 4 == 0 && ((uintptr_t)a->o & 15) == 0, "o rows must be 16-byte aligned");
  B2A_CHECK_ARG(!a->emit_hi || (a->emit_ld >= a->H * HD && a->emit_ld % 8 == 0), "emitted planes: row stride >= H*64, a multiple of 8");
  cudaStream_t st = (cudaStream_t)stream;
  const int B = a->B, H = a->H, Tq = a->Tq, Tk = a->Tk;
  const int64_t bh = (int64_t)B * H;
  const AttnOperands op = attn_operands(ws, bh, Tq, Tk);
  __half *qh = op.qh, *ql = op.ql, *kh = op.kh, *kl = op.kl, *vh = op.vh, *vl = op.vl;
  const int64_t Tkp = op.tkp;
  if (!a->operands_ready) {
    int64_t tq = bh * Tq * (HD / 8), tk = bh * Tk * (HD / 8);
    int gq = (int)((tq + 255) / 256); if (gq > 132 * 16) gq = 132 * 16;
    int gk = (int)((tk + 255) / 256); if (gk > 132 * 16) gk = 132 * 16;
    attn_tc_prep_qk_kernel<<<gq, 256, 0, st>>>(a->q, a->q_bs, a->q_ld, B, H, Tq, a->scale * 1.4426950408889634f, qh, ql);
    attn_tc_prep_qk_kernel<<<gk, 256, 0, st>>>(a->k, a->k_bs, a->k_ld, B, H, Tk, 1.f, kh, kl);
    dim3 gv((unsigned)((Tkp + 63) / 64), H, B);
    attn_tc_prep_vt_kernel<<<gv, 256, 0, st>>>(a->v, a->v_bs, a->v_ld, B, H, Tk, (int)Tkp, vh, vl);
  }
  CUtensorMap mqh, mql, mkh, mkl, mvh, mvl;
  const uint64_t qd[3] = {HD, (uint64_t)Tq, (uint64_t)bh}, qs[2] = {HD * 2, (uint64_t)Tq * HD * 2};
  const uint64_t kd[3] = {HD, (uint64_t)Tk, (uint64_t)bh}, ks[2] = {HD * 2, (uint64_t)Tk * HD * 2};
  const uint64_t vd[3] = {(uint64_t)Tkp, HD, (uint64_t)bh}, vs[2] = {(uint64_t)Tkp * 2, (uint64_t)HD * Tkp * 2};
  const uint32_t qb[3] = {HD, BM, 1}, kb[3] = {HD, BN, 1}, vb[3] = {BN, HD, 1};
  int e = b2a_tmap16(&mqh, qh, 3, qd, qs, qb, true);
  if (!e) e = b2a_tmap16(&mql, ql, 3, qd, qs, qb, true);
  if (!e) e = b2a_tmap16(&mkh, kh, 3, kd, ks, kb, true);
  if (!e) e = b2a_tmap16(&mkl, kl, 3, kd, ks, kb, true);
  if (!e) e = b2a_tmap16(&mvh, vh, 3, vd, vs, vb, true);
  if (!e) e = b2a_tmap16(&mvl, vl, 3, vd, vs, vb, true);
  if (e) { b2a_set_error("b2a_attention_tc: cuTensorMapEncodeTiled failed (%d)", e); return B2A_E_CUDA; }
  AtcParams p{B, H, Tq, Tk, a->causal, a->q_offset, a->window, a->o, a->o_bs, a->o_ld,
              (__nv_bfloat16*)a->emit_hi, (__nv_bfloat16*)a->emit_lo, a->emit_ld};
  B2A_SMEM_OPTIN(attn_tc_kernel, SMEM_BYTES);
  dim3 grid((Tq + BM - 1) / BM, (unsigned)bh);
  if (b2a_launch_pdl(attn_tc_kernel, grid, dim3(THREADS), SMEM_BYTES, st, mqh, mql, mkh, mkl, mvh, mvl, p) != cudaSuccess) {
    b2a_set_error("b2a_attention_tc: %s", cudaGetErrorString(cudaGetLastError()));
    return B2A_E_CUDA;
  }
  return B2A_OK;
}
