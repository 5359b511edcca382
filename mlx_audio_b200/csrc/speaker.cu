// Qwen3-TTS speaker encoder (ECAPA-TDNN, tts/models/qwen3_tts/speaker_encoder.py) and its 24 kHz log-mel front end
// (qwen3_tts.py:64-121).  The encoder is tiny for an H100 (~10 MFLOP per mel frame, activations <= [T, 1536]), so these kernels are
// written for few launches and fixed-order reductions (bit-reproducible embeddings), not for throughput; the dense 1x1 / k5 layers
// run on the tensor-core conv, everything between them is here.
#include <cuda_bf16.h>
#include "common.cuh"
#include "spk_logmel.cuh"

namespace {

// ---------------------------------------------------------------- log-mel front end (spk_logmel.cuh): centre pad 384, |X| with 1e-9
constexpr int MEL_PAD = (MEL_N - MEL_HOP) / 2;

// ---------------------------------------------------------------- reflect "same" padding as the operand of the next conv
__device__ __forceinline__ int reflect_idx(int q, int T) {
  if (q < 0) q = -q;
  if (q >= T) q = 2 * (T - 1) - q;
  return q;
}

// y[b, r, c] = x[b, reflect(r - pad), c] for r in [0, T + 2 pad): fp32 rows [B, T+2pad, C] (f32 != NULL), or the bf16 (hi, lo) planes
// [B, T+2pad, cpad] of the tensor-core conv (lo may be NULL; pad channels zero), split as prep_bf16 splits them.
__global__ void spk_reflect_pad_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int B, int T, int C, int pad,
                                       float* __restrict__ f32, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int cpad) {
  const int Tp = T + 2 * pad, cw = f32 ? C : cpad;
  const int64_t total = (int64_t)B * Tp * cw;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cw);
    const int64_t r = idx / cw;
    const int row = (int)(r % Tp), b = (int)(r / Tp);
    const float v = c < C ? __ldg(x + (int64_t)b * x_bs + (int64_t)reflect_idx(row - pad, T) * x_ld + c) : 0.f;
    if (f32) { f32[idx] = v; continue; }
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[idx] = h;
    if (lo) lo[idx] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

// ---------------------------------------------------------------- Res2Net chain (speaker_encoder.py:60-101), one launch per block
// One CTA = one (item, tile of TT output rows).  Stage i (1 <= i < scale) is relu(conv_k,d(reflect_pad(chunk_i + out_{i-1}))) with
// out_0 = 0 on stage 1; the CTA recomputes each stage on its tile plus the halo the later stages need ((scale-1-i)*pad rows per side,
// clamped to the sequence -- reflected positions of a clamped window stay inside it, so every stage only reads rows it computed).
// Shared memory: two activation buffers [W][C+1] (odd row stride: no bank conflicts across rows) and one stage's weights [K][C][C]
// (ci-major, co fastest) + bias.  Each thread owns RB consecutive rows x CQ consecutive output channels; the summation order of every
// output is fixed (k, then ci), so the result does not depend on the tiling.
template <int CQ>
__global__ void __launch_bounds__(256) spk_res2net_kernel(const float* __restrict__ y, int64_t y_bs, int64_t y_ld, float* __restrict__ z,
                                                          int64_t z_bs, int64_t z_ld, const float* __restrict__ w, const float* __restrict__ bias,
                                                          int T, int C, int scale, int K, int dil, int pad, int TT) {
  constexpr int RB = 4;
  extern __shared__ __align__(16) float sm[];
  const int b = blockIdx.y, t0 = blockIdx.x * TT, t1 = min(T, t0 + TT);
  const int H = (scale - 1) * pad, W = TT + 2 * H, XS = C + 1, WB = (W * XS + 3) & ~3;
  const int base = t0 - H;                                   // buffer row 0 <-> sequence row `base`
  float* bufA = sm;
  float* bufB = bufA + WB;
  float* ws = bufB + WB;                                     // [K][C][C], 16-byte aligned
  float* bs = ws + K * C * C;                                // [C]
  const float* yb = y + (int64_t)b * y_bs;
  float* zb = z + (int64_t)b * z_bs;
  // chunk 0 passes through
  for (int idx = threadIdx.x; idx < (t1 - t0) * C; idx += blockDim.x) {
    const int r = t0 + idx / C, c = idx % C;
    zb[(int64_t)r * z_ld + c] = __ldg(yb + (int64_t)r * y_ld + c);
  }
  // stage 1 input: chunk 1 over the widest window
  int lo = max(0, t0 - H), hi = min(T, t1 + H);
  for (int idx = threadIdx.x; idx < (hi - lo) * C; idx += blockDim.x) {
    const int r = lo + idx / C, c = idx % C;
    bufA[(r - base) * XS + c] = __ldg(yb + (int64_t)r * y_ld + C + c);
  }
  float* xin = bufA;
  float* xout = bufB;
  const int nq = C / CQ;
  for (int i = 1; i < scale; i++) {
    const float* wi = w + (int64_t)(i - 1) * K * C * C;
    for (int idx = threadIdx.x; idx < K * C * C; idx += blockDim.x) ws[idx] = __ldg(wi + idx);
    for (int idx = threadIdx.x; idx < C; idx += blockDim.x) bs[idx] = __ldg(bias + (int64_t)(i - 1) * C + idx);
    if (i > 1) {                                             // stage input = chunk_i + out_{i-1} over out_{i-1}'s window [lo, hi)
      for (int idx = threadIdx.x; idx < (hi - lo) * C; idx += blockDim.x) {
        const int r = lo + idx / C, c = idx % C;
        xin[(r - base) * XS + c] += __ldg(yb + (int64_t)r * y_ld + (int64_t)i * C + c);
      }
    }
    __syncthreads();
    const int olo = max(0, t0 - (scale - 1 - i) * pad), ohi = min(T, t1 + (scale - 1 - i) * pad);
    const int ngr = (ohi - olo + RB - 1) / RB;
    for (int item = threadIdx.x; item < ngr * nq; item += blockDim.x) {
      const int co0 = (item % nq) * CQ, r0 = olo + (item / nq) * RB;
      float acc[RB][CQ];
#pragma unroll
      for (int r = 0; r < RB; r++)
#pragma unroll
        for (int q = 0; q < CQ; q++) acc[r][q] = bs[co0 + q];
      for (int k = 0; k < K; k++) {
        const float* xr[RB];
#pragma unroll
        for (int r = 0; r < RB; r++) {
          const int t = min(r0 + r, ohi - 1);
          xr[r] = xin + (reflect_idx(t + k * dil - pad, T) - base) * XS;
        }
        const float* wk = ws + k * C * C + co0;
        for (int ci = 0; ci < C; ci++) {
          float wv[CQ];
          if constexpr (CQ == 4) {
            const float4 w4 = *reinterpret_cast<const float4*>(wk + ci * C);
            wv[0] = w4.x; wv[1] = w4.y; wv[2] = w4.z; wv[3] = w4.w;
          } else {
#pragma unroll
            for (int q = 0; q < CQ; q++) wv[q] = wk[ci * C + q];
          }
#pragma unroll
          for (int r = 0; r < RB; r++) {
            const float xv = xr[r][ci];
#pragma unroll
            for (int q = 0; q < CQ; q++) acc[r][q] = fmaf(xv, wv[q], acc[r][q]);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < RB; r++) {
        const int t = r0 + r;
        if (t >= ohi) break;
#pragma unroll
        for (int q = 0; q < CQ; q++) {
          const float v = fmaxf(acc[r][q], 0.f);
          xout[(t - base) * XS + co0 + q] = v;
          if (t >= t0 && t < t1) zb[(int64_t)t * z_ld + (int64_t)i * C + co0 + q] = v;
        }
      }
    }
    __syncthreads();
    float* tmp = xin; xin = xout; xout = tmp;
    lo = olo; hi = ohi;
  }
}

// ---------------------------------------------------------------- per-channel statistics over time, fixed order
// CTA = (item, 32 channels); 8 row lanes per channel, each summing rows t = lane (mod 8) in order, combined in lane order.
// out[b*o_bs + c] = mean; with_std: out[b*o_bs + C + c] = sqrt(var + eps), var = mean((x - mean)^2).
constexpr int ST_CH = 32, ST_LANES = 8;

__global__ void spk_channel_stats_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int T, int C, int with_std, float eps,
                                         float* __restrict__ out, int64_t o_bs) {
  __shared__ float part[ST_LANES][ST_CH];
  __shared__ float mean_s[ST_CH];
  const int b = blockIdx.y, cl = threadIdx.x % ST_CH, lane = threadIdx.x / ST_CH, c = blockIdx.x * ST_CH + cl;
  const float* xb = x + (int64_t)b * x_bs + c;
  float s = 0.f;
  if (c < C)
    for (int t = lane; t < T; t += ST_LANES) s += __ldg(xb + (int64_t)t * x_ld);
  part[lane][cl] = s;
  __syncthreads();
  if (lane == 0) {
    float a = 0.f;
    for (int l = 0; l < ST_LANES; l++) a += part[l][cl];
    mean_s[cl] = a / (float)T;
    if (c < C) out[(int64_t)b * o_bs + c] = a / (float)T;
  }
  if (!with_std) return;
  __syncthreads();
  const float m = mean_s[cl];
  float v = 0.f;
  if (c < C)
    for (int t = lane; t < T; t += ST_LANES) { const float d = __ldg(xb + (int64_t)t * x_ld) - m; v = fmaf(d, d, v); }
  part[lane][cl] = v;
  __syncthreads();
  if (lane == 0 && c < C) {
    float a = 0.f;
    for (int l = 0; l < ST_LANES; l++) a += part[l][cl];
    out[(int64_t)b * o_bs + C + c] = sqrtf(a / (float)T + eps);
  }
}

// ---------------------------------------------------------------- squeeze-excitation (speaker_encoder.py:104-133)
// One CTA per item: h = relu(W1 mean + b1) [S], gate = sigmoid(W2 h + b2) [C]; one warp per output row, lane-strided partial sums
// reduced by the (fixed) butterfly.
__global__ void spk_se_gate_kernel(const float* __restrict__ mean, int64_t m_bs, int C, int S, const float* __restrict__ w1,
                                   const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                                   float* __restrict__ gate) {
  extern __shared__ __align__(16) float sm[];
  float* ms = sm;          // [C]
  float* hs = sm + C;      // [S]
  const int b = blockIdx.x, warp = threadIdx.x / 32, lane = threadIdx.x % 32, nw = blockDim.x / 32;
  for (int c = threadIdx.x; c < C; c += blockDim.x) ms[c] = mean[(int64_t)b * m_bs + c];
  __syncthreads();
  for (int j = warp; j < S; j += nw) {
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a = fmaf(__ldg(w1 + (int64_t)j * C + c), ms[c], a);
    a = warp_sum(a);
    if (lane == 0) hs[j] = fmaxf(a + __ldg(b1 + j), 0.f);
  }
  __syncthreads();
  for (int j = warp; j < C; j += nw) {
    float a = 0.f;
    for (int s = lane; s < S; s += 32) a = fmaf(__ldg(w2 + (int64_t)j * S + s), hs[s], a);
    a = warp_sum(a);
    if (lane == 0) gate[(int64_t)b * C + j] = 1.f / (1.f + expf(-(a + __ldg(b2 + j))));
  }
}

// out[b,t,c] = y[b,t,c] * gate[b,c] + res[b,t,c]  (the block's output, written into its channel slice of the MFA buffer)
__global__ void spk_se_apply_kernel(const float* __restrict__ y, int64_t y_bs, int64_t y_ld, const float* __restrict__ gate,
                                    const float* __restrict__ res, int64_t r_bs, int64_t r_ld, float* __restrict__ out, int64_t o_bs,
                                    int64_t o_ld, int B, int T, int C) {
  const int64_t total = (int64_t)B * T * C;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const int64_t r = idx / C;
    const int t = (int)(r % T), b = (int)(r / T);
    const float v = __ldg(y + (int64_t)b * y_bs + (int64_t)t * y_ld + c);
    out[(int64_t)b * o_bs + (int64_t)t * o_ld + c] = fmaf(v, __ldg(gate + (int64_t)b * C + c), __ldg(res + (int64_t)b * r_bs + (int64_t)t * r_ld + c));
  }
}

// ---------------------------------------------------------------- small row GEMV: y[b, j] = act(bias[j] + W[j, :] . x[b, :])
// One warp per output; used for the statistics half of the pooling TDNN and for the final projection (one row per item).
__global__ void spk_gemv_kernel(const float* __restrict__ x, int64_t x_bs, int K, const float* __restrict__ w, int64_t w_ld, int N,
                                const float* __restrict__ bias, int act, float* __restrict__ y, int64_t y_bs) {
  const int b = blockIdx.y, lane = threadIdx.x % 32;
  const int j = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (j >= N) return;
  const float* xb = x + (int64_t)b * x_bs;
  const float* wj = w + (int64_t)j * w_ld;
  float a = 0.f;
  for (int k = lane; k < K; k += 32) a = fmaf(__ldg(wj + k), __ldg(xb + k), a);
  a = warp_sum(a);
  if (lane == 0) {
    a += bias ? __ldg(bias + j) : 0.f;
    y[(int64_t)b * y_bs + j] = b2a_act(a, act, 0.f, 1.f, 1.f);
  }
}

// ---------------------------------------------------------------- attentive statistics pooling (speaker_encoder.py:171-217)
// h[b,t,j] = tanh(relu(h[b,t,j] + cb[b,j])): cb carries W_m.mean + W_s.std + bias, so the [T, 3C] concatenation is never built.
__global__ void spk_asp_act_kernel(float* __restrict__ h, int64_t h_bs, int64_t h_ld, const float* __restrict__ cb, int B, int T, int A) {
  const int64_t total = (int64_t)B * T * A;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx % A);
    const int64_t r = idx / A;
    const int t = (int)(r % T), b = (int)(r / T);
    float* p = h + (int64_t)b * h_bs + (int64_t)t * h_ld + j;
    *p = tanhf(fmaxf(*p + __ldg(cb + (int64_t)b * A + j), 0.f));
  }
}

// softmax over TIME of the logits per (item, channel), max-subtracted, then the weighted mean and sqrt(max(weighted var, eps)):
// pooled[b, c] = mean, pooled[b, C + c] = std.  Same fixed-order lane layout as spk_channel_stats_kernel; three passes over T.
__global__ void spk_asp_pool_kernel(const float* __restrict__ lg, int64_t l_bs, int64_t l_ld, const float* __restrict__ x, int64_t x_bs,
                                    int64_t x_ld, int T, int C, float eps, float* __restrict__ pooled, int64_t p_bs) {
  __shared__ float part[ST_LANES][ST_CH];
  __shared__ float part2[ST_LANES][ST_CH];
  __shared__ float bc[2][ST_CH];
  const int b = blockIdx.y, cl = threadIdx.x % ST_CH, lane = threadIdx.x / ST_CH, c = blockIdx.x * ST_CH + cl;
  const bool ok = c < C;
  const float* lb = lg + (int64_t)b * l_bs + c;
  const float* xb = x + (int64_t)b * x_bs + c;
  float m = -INFINITY;
  if (ok)
    for (int t = lane; t < T; t += ST_LANES) m = fmaxf(m, __ldg(lb + (int64_t)t * l_ld));
  part[lane][cl] = m;
  __syncthreads();
  if (lane == 0) {
    float a = part[0][cl];
    for (int l = 1; l < ST_LANES; l++) a = fmaxf(a, part[l][cl]);
    bc[0][cl] = a;
  }
  __syncthreads();
  m = bc[0][cl];
  float se = 0.f, sx = 0.f;
  if (ok)
    for (int t = lane; t < T; t += ST_LANES) {
      const float e = expf(__ldg(lb + (int64_t)t * l_ld) - m);
      se += e;
      sx = fmaf(e, __ldg(xb + (int64_t)t * x_ld), sx);
    }
  __syncthreads();
  part[lane][cl] = se;
  part2[lane][cl] = sx;
  __syncthreads();
  if (lane == 0) {
    float a = 0.f, s = 0.f;
    for (int l = 0; l < ST_LANES; l++) { a += part[l][cl]; s += part2[l][cl]; }
    bc[0][cl] = 1.f / a;                                     // 1 / sum of the shifted exponentials (>= 1: the max term is exp(0))
    bc[1][cl] = s / a;                                       // weighted mean
  }
  __syncthreads();
  const float inv = bc[0][cl], mu = bc[1][cl];
  float sv = 0.f;
  if (ok)
    for (int t = lane; t < T; t += ST_LANES) {
      const float d = __ldg(xb + (int64_t)t * x_ld) - mu;
      sv = fmaf(expf(__ldg(lb + (int64_t)t * l_ld) - m) * inv, d * d, sv);
    }
  __syncthreads();
  part[lane][cl] = sv;
  __syncthreads();
  if (lane == 0 && ok) {
    float a = 0.f;
    for (int l = 0; l < ST_LANES; l++) a += part[l][cl];
    pooled[(int64_t)b * p_bs + c] = mu;
    pooled[(int64_t)b * p_bs + C + c] = sqrtf(fmaxf(a, eps));
  }
}

int grid_1d(int64_t total) { int64_t g = (total + 255) / 256; return (int)(g < 4096 ? (g > 0 ? g : 1) : 4096); }

}  // namespace

// ---------------------------------------------------------------- C ABI
extern "C" int32_t b2a_spk_logmel(const float* x, int64_t x_bs, int32_t B, int64_t n, const float* window, const float* filters,
                                  int32_t n_mels, int64_t frames, float* out, void* stream) {
  B2A_CHECK_ARG(x && window && filters && out && B > 0 && n_mels > 0 && frames > 0, "bad pointers/shape");
  B2A_CHECK_ARG(n > MEL_PAD, "reflect padding needs more than 384 samples");
  B2A_CHECK_ARG(frames == 1 + (n + 2 * MEL_PAD - MEL_N) / MEL_HOP, "frames must be 1 + (n + 768 - 1024) / 256");
  const size_t smem = spk_logmel_smem_bytes();
  B2A_SMEM_OPTIN((spk_logmel_kernel<MEL_PAD, true>), smem);
  dim3 grid(cdiv(frames, MEL_FT), B);
  spk_logmel_kernel<MEL_PAD, true><<<grid, 256, smem, (cudaStream_t)stream>>>(x, x_bs, n, window, filters, n_mels, frames, out);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_spk_reflect_pad(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t C, int32_t pad,
                                       float* out_f32, void* hi, void* lo, int32_t cpad, void* stream) {
  B2A_CHECK_ARG(x && B > 0 && T > 0 && C > 0 && pad >= 0, "bad pointers/shape");
  B2A_CHECK_ARG(pad < T, "reflect padding needs pad < T");
  B2A_CHECK_ARG((out_f32 != nullptr) != (hi != nullptr), "exactly one of out_f32 / hi");
  B2A_CHECK_ARG(out_f32 || cpad >= C, "cpad < C");
  const int64_t total = (int64_t)B * (T + 2 * pad) * (out_f32 ? C : cpad);
  spk_reflect_pad_kernel<<<grid_1d(total), 256, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, B, T, C, pad, out_f32, (__nv_bfloat16*)hi,
                                                                           (__nv_bfloat16*)lo, cpad);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int64_t b2a_spk_res2net_smem_bytes(int32_t C, int32_t scale, int32_t K, int32_t pad, int32_t tile) {
  const int64_t W = tile + 2 * (int64_t)(scale - 1) * pad, WB = (W * (C + 1) + 3) & ~3;
  return (2 * WB + (int64_t)K * C * C + C) * (int64_t)sizeof(float);
}

extern "C" int32_t b2a_spk_res2net(const float* y, int64_t y_bs, int64_t y_ld, float* z, int64_t z_bs, int64_t z_ld, const float* w,
                                   const float* bias, int32_t B, int32_t T, int32_t C, int32_t scale, int32_t K, int32_t dilation,
                                   int32_t tile, void* stream) {
  B2A_CHECK_ARG(y && z && w && bias && B > 0 && T > 0 && C > 0 && scale >= 2 && K >= 1 && dilation >= 1 && tile > 0, "bad pointers/shape");
  B2A_CHECK_ARG(((K - 1) * dilation) % 2 == 0, "\"same\" reflect padding needs an even (K-1)*dilation");
  const int pad = (K - 1) * dilation / 2;
  B2A_CHECK_ARG(pad < T, "reflect padding needs pad < T");
  const int64_t smem = b2a_spk_res2net_smem_bytes(C, scale, K, pad, tile);
  if (smem > 227 * 1024) { b2a_set_error("%s: %lld bytes of shared memory", __func__, (long long)smem); return B2A_E_UNSUPPORTED; }
  dim3 grid(cdiv(T, tile), B);
  cudaStream_t st = (cudaStream_t)stream;
  const auto kern = C % 4 == 0 ? spk_res2net_kernel<4> : spk_res2net_kernel<1>;
  B2A_SMEM_OPTIN(kern, smem);
  kern<<<grid, 256, smem, st>>>(y, y_bs, y_ld, z, z_bs, z_ld, w, bias, T, C, scale, K, dilation, pad, tile);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_spk_channel_stats(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t C, int32_t with_std,
                                         float eps, float* out, int64_t o_bs, void* stream) {
  B2A_CHECK_ARG(x && out && B > 0 && T > 0 && C > 0, "bad pointers/shape");
  dim3 grid(cdiv(C, ST_CH), B);
  spk_channel_stats_kernel<<<grid, ST_CH * ST_LANES, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, T, C, with_std, eps, out, o_bs);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_spk_se_gate(const float* mean, int64_t m_bs, int32_t B, int32_t C, int32_t S, const float* w1, const float* b1,
                                   const float* w2, const float* b2, float* gate, void* stream) {
  B2A_CHECK_ARG(mean && w1 && b1 && w2 && b2 && gate && B > 0 && C > 0 && S > 0, "bad pointers/shape");
  const size_t smem = (size_t)(C + S) * sizeof(float);
  B2A_CHECK_ARG(smem <= 48 * 1024, "C + S too large");
  spk_se_gate_kernel<<<B, 512, smem, (cudaStream_t)stream>>>(mean, m_bs, C, S, w1, b1, w2, b2, gate);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_spk_se_apply(const float* y, int64_t y_bs, int64_t y_ld, const float* gate, const float* res, int64_t r_bs,
                                    int64_t r_ld, float* out, int64_t o_bs, int64_t o_ld, int32_t B, int32_t T, int32_t C, void* stream) {
  B2A_CHECK_ARG(y && gate && res && out && B > 0 && T > 0 && C > 0, "bad pointers/shape");
  spk_se_apply_kernel<<<grid_1d((int64_t)B * T * C), 256, 0, (cudaStream_t)stream>>>(y, y_bs, y_ld, gate, res, r_bs, r_ld, out, o_bs, o_ld,
                                                                                       B, T, C);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_spk_gemv(const float* x, int64_t x_bs, int32_t B, int32_t K, const float* w, int64_t w_ld, int32_t N,
                                const float* bias, int32_t act, float* y, int64_t y_bs, void* stream) {
  B2A_CHECK_ARG(x && w && y && B > 0 && K > 0 && N > 0 && w_ld >= K, "bad pointers/shape");
  dim3 grid(cdiv(N, 8), B);
  spk_gemv_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, x_bs, K, w, w_ld, N, bias, act, y, y_bs);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_spk_asp_act(float* h, int64_t h_bs, int64_t h_ld, const float* cb, int32_t B, int32_t T, int32_t A, void* stream) {
  B2A_CHECK_ARG(h && cb && B > 0 && T > 0 && A > 0, "bad pointers/shape");
  spk_asp_act_kernel<<<grid_1d((int64_t)B * T * A), 256, 0, (cudaStream_t)stream>>>(h, h_bs, h_ld, cb, B, T, A);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_spk_asp_pool(const float* logits, int64_t l_bs, int64_t l_ld, const float* x, int64_t x_bs, int64_t x_ld,
                                    int32_t B, int32_t T, int32_t C, float eps, float* pooled, int64_t p_bs, void* stream) {
  B2A_CHECK_ARG(logits && x && pooled && B > 0 && T > 0 && C > 0, "bad pointers/shape");
  dim3 grid(cdiv(C, ST_CH), B);
  spk_asp_pool_kernel<<<grid, ST_CH * ST_LANES, 0, (cudaStream_t)stream>>>(logits, l_bs, l_ld, x, x_bs, x_ld, T, C, eps, pooled, p_bs);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
