// Incremental (streaming) Mimi codec: carried-state causal convs, transposed convs with a held-back tail, and windowed attention over a
// per-layer ring KV cache (include/b200audio.h: b2a_conv1d_stream, b2a_convtr1d_stream, b2a_ring_rope_kv, b2a_ring_attn,
// b2a_stream_advance).  Replaces the reference's StreamableConv1d.step / StreamableConvTranspose1d.step (mimi/modules/conv.py:245-331),
// StreamingAdd (seanet.py:30-52: with every conv returning exactly its new rows the residual operands are always aligned) and the growing
// KVCache + context mask of the transformer (transformer.py:79-112).
//
// Every state read / write is hazard-free without grid-wide synchronisation:
//   - a conv's carried input rows live in two slots; the launch reads slot (*step & 1) and writes the other, and the step's last launch
//     (b2a_stream_advance) flips the parity -- all on the device, so a captured step replays with no host scalar;
//   - a transposed conv's tail row (l, co) is read (added into output row l) and rewritten (the new tail, output row L*stride + l) by the
//     same thread;
//   - the ring is written at positions *pos .. *pos + T - 1 and read over [p - window + 1, p]; capacity >= window + T keeps the two apart.
// Reductions run in a fixed order (no atomics): results are bit-reproducible, eager or replayed.
#include "common.cuh"

namespace {

constexpr int CO_T = 32;   // output channels per CTA (one per lane)
constexpr int RED_W = 8;   // warps splitting the reduction
constexpr int ROW_T = 4;   // output rows per CTA

struct ConvStreamArgs {
  b2a_conv1d_t p;
  float* hist;             // [2][B][keff - 1][Cin]: slot (*step & 1) holds the H carried rows, the other receives the new ones
  int64_t hist_bs;
  int H, fresh;
  const int32_t* step;
};

// virtual input row r of [history | new rows] for batch b, channel ci, before the prologue
__device__ __forceinline__ float vin(const ConvStreamArgs& a, const float* hist, int b, int r, int ci) {
  if (r >= a.H) return a.p.x[(int64_t)b * a.p.x_bs + (int64_t)(r - a.H) * a.p.x_ld + ci];
  if (a.fresh) return a.p.pad_mode == 1 ? a.p.x[(int64_t)b * a.p.x_bs + ci] : 0.f;
  return hist[(int64_t)b * a.hist_bs + (int64_t)r * a.p.Cin + ci];
}

__global__ void __launch_bounds__(CO_T * RED_W) conv_stream_kernel(const ConvStreamArgs a, int row_tiles) {
  const b2a_conv1d_t& p = a.p;
  const int64_t slot = (int64_t)p.B * a.hist_bs;
  const int par = *a.step & 1;
  const float* hist = a.hist + (par ? slot : 0);
  float* hist_out = a.hist + (par ? 0 : slot);
  const int b = blockIdx.z;
  if ((int)blockIdx.y >= row_tiles) {                 // history carry: rows [Lout*stride, H + L) of the virtual input
    if (a.fresh && p.L == 0) return;
    const int first = p.Lout * p.stride, n = a.H + p.L - first;
    const int64_t total = (int64_t)n * p.Cin;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int r = (int)(i / p.Cin), ci = (int)(i % p.Cin);
      hist_out[(int64_t)b * a.hist_bs + (int64_t)r * p.Cin + ci] = vin(a, hist, b, first + r, ci);
    }
    return;
  }
  __shared__ float red[RED_W][ROW_T][CO_T];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int co = blockIdx.x * CO_T + lane;
  const int l0 = blockIdx.y * ROW_T;
  float acc[ROW_T];
#pragma unroll
  for (int j = 0; j < ROW_T; j++) acc[j] = 0.f;
  if (co < p.Cout) {
    for (int k = 0; k < p.K; k++) {
      const float* wk = p.w + (int64_t)k * p.Cin * p.Cout + co;
      for (int ci = w; ci < p.Cin; ci += RED_W) {
        const float wv = wk[(int64_t)ci * p.Cout];
#pragma unroll
        for (int j = 0; j < ROW_T; j++) {
          const int l = l0 + j;
          if (l < p.Lout) {
            const float v = b2a_act(vin(a, hist, b, l * p.stride + k * p.dilation, ci), p.pre_act, p.pre_p0, 0.f, 0.f);
            acc[j] = fmaf(wv, v, acc[j]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < ROW_T; j++) red[w][j][lane] = acc[j];
  __syncthreads();
  if (w < ROW_T) {
    const int j = w, l = l0 + j;
    if (co < p.Cout && l < p.Lout) {
      float s = red[0][j][lane];
#pragma unroll
      for (int u = 1; u < RED_W; u++) s += red[u][j][lane];
      if (p.bias) s += p.bias[co];
      s = b2a_act(s, p.post_act, p.post_p0, 0.f, 0.f);
      if (p.post_cscale) s *= p.post_cscale[(int64_t)b * p.post_cscale_bs + co];
      if (p.res) s += p.res[(int64_t)b * p.res_bs + (int64_t)(l / p.res_div) * p.res_ld + co];
      p.y[(int64_t)b * p.y_bs + (int64_t)l * p.y_ld + co] = s * p.out_scale;
    }
  }
}

// Dense transposed conv: output rows [0, L*s) plus, for the CTAs whose rows l < K - s, the new tail rows L*s + l -- computed by the
// thread that reads tail row l for its output.
__global__ void __launch_bounds__(CO_T * RED_W) convtr_stream_kernel(const b2a_conv1d_t p, float* tail, int64_t tail_bs) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int co = blockIdx.x * CO_T + lane;
  const int l0 = blockIdx.y * ROW_T, b = blockIdx.z;
  const int s = p.stride, nt = p.K - s, Lo = p.L * s;
  __shared__ float red[RED_W][2 * ROW_T][CO_T];
  float acc[2 * ROW_T];
#pragma unroll
  for (int j = 0; j < 2 * ROW_T; j++) acc[j] = 0.f;
  const bool has_tail = l0 < nt;
  if (co < p.Cout) {
    for (int ci = w; ci < p.Cin; ci += RED_W) {
      const float* xb = p.x + (int64_t)b * p.x_bs + ci;
#pragma unroll
      for (int j = 0; j < 2 * ROW_T; j++) {
        if (j >= ROW_T && !has_tail) break;
        const int m = j < ROW_T ? l0 + j : Lo + l0 + j - ROW_T;
        if (j < ROW_T ? m >= Lo : (l0 + j - ROW_T) >= nt) continue;
        float sacc = acc[j];
        for (int k = m % s; k < p.K; k += s) {
          const int i = (m - k) / s;
          if (i < 0) break;
          if (i >= p.L) continue;
          const float v = b2a_act(xb[(int64_t)i * p.x_ld], p.pre_act, p.pre_p0, 0.f, 0.f);
          sacc = fmaf(p.w[((int64_t)k * p.Cin + ci) * p.Cout + co], v, sacc);
        }
        acc[j] = sacc;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 2 * ROW_T; j++) red[w][j][lane] = acc[j];
  __syncthreads();
  if (w < ROW_T && co < p.Cout) {
    const int l = l0 + w;
    if (l < Lo) {
      float sum = red[0][w][lane], st = red[0][w + ROW_T][lane];
#pragma unroll
      for (int u = 1; u < RED_W; u++) { sum += red[u][w][lane]; st += red[u][w + ROW_T][lane]; }
      float o = sum + (p.bias ? p.bias[co] : 0.f);
      if (l < nt) {
        float* tp = tail + (int64_t)b * tail_bs + (int64_t)l * p.Cout + co;
        o += *tp;
        *tp = st;                                        // same thread: read before write
      }
      p.y[(int64_t)b * p.y_bs + (int64_t)l * p.y_ld + co] = o * p.out_scale;
    }
  }
}

// Depthwise transposed conv (groups == C): one thread per (b, output row, c), the same tail rule.
__global__ void convtr_stream_dw_kernel(const b2a_conv1d_t p, float* tail, int64_t tail_bs) {
  const int s = p.stride, nt = p.K - s, Lo = p.L * s, C = p.Cout;
  const int64_t total = (int64_t)p.B * Lo * C;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const int64_t r = idx / C;
    const int l = (int)(r % Lo), b = (int)(r / Lo);
    const float* xb = p.x + (int64_t)b * p.x_bs + c;
    auto row = [&](int m) {
      float acc = 0.f;
      for (int k = m % s; k < p.K; k += s) {
        const int i = (m - k) / s;
        if (i < 0) break;
        if (i >= p.L) continue;
        acc = fmaf(p.w[(int64_t)k * C + c], b2a_act(xb[(int64_t)i * p.x_ld], p.pre_act, p.pre_p0, 0.f, 0.f), acc);
      }
      return acc;
    };
    float o = row(l) + (p.bias ? p.bias[c] : 0.f);
    if (l < nt) {
      float* tp = tail + (int64_t)b * tail_bs + (int64_t)l * C + c;
      o += *tp;
      *tp = row(Lo + l);
    }
    p.y[(int64_t)b * p.y_bs + (int64_t)l * p.y_ld + c] = o * p.out_scale;
  }
}

// Interleaved-pair RoPE of q (in place) and k at absolute positions *pos + t; k and v stored into ring row (*pos + t) % cap.
__global__ void ring_rope_kv_kernel(float* qkv, int64_t qkv_bs, int64_t qkv_ld, int B, int T, int H, int D, float base, float* k_ring,
                                    float* v_ring, int64_t ring_bs, int cap, const int32_t* pos) {
  const int half = D / 2, HD = H * D;
  const int p0 = *pos;
  const int64_t total = (int64_t)B * T * H * half;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx % half);
    int64_t r = idx / half;
    const int h = (int)(r % H); r /= H;
    const int t = (int)(r % T), b = (int)(r / T);
    // angle in float64, as b2a_rope: the one-shot decode rotates with the same arithmetic
    const double inv = exp(-(double)i * (log((double)base) / half));
    const double ang = (double)(p0 + t) * inv;
    double sn, cs;
    sincos(ang, &sn, &cs);
    float* row = qkv + (int64_t)b * qkv_bs + (int64_t)t * qkv_ld + h * D + 2 * i;
    const int64_t ro = (int64_t)b * ring_bs + (int64_t)((p0 + t) % cap) * HD + h * D + 2 * i;
    float a = row[0], c = row[1];
    row[0] = (float)(a * cs - c * sn);
    row[1] = (float)(a * sn + c * cs);
    a = row[HD]; c = row[HD + 1];
    k_ring[ro] = (float)(a * cs - c * sn);
    k_ring[ro + 1] = (float)(a * sn + c * cs);
    v_ring[ro] = row[2 * HD];
    v_ring[ro + 1] = row[2 * HD + 1];
  }
}

constexpr int AT = 128;         // threads per (query, head, batch) CTA
constexpr int WIN_MAX = 1024;

// One CTA per (query t, head h, batch b); D == 64.  Query at position p = *pos + t attends ring positions [max(0, p - window + 1), p] in
// ascending order: scores one key per thread, block max / sum as fixed trees, P V with two key halves per output dimension.
__global__ void __launch_bounds__(AT) ring_attn_kernel(const float* q, int64_t q_bs, int64_t q_ld, const float* k_ring, const float* v_ring,
                                                       int64_t ring_bs, int cap, float* out, int64_t o_bs, int64_t o_ld, int H, float scale,
                                                       int window, const int32_t* pos) {
  constexpr int D = 64;
  const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const int HD = H * D;
  const int p = *pos + t;
  const int lo = max(0, p - window + 1), n = p - lo + 1;
  __shared__ float qs[D];
  __shared__ float sc[WIN_MAX];
  __shared__ float red[AT / 32];
  __shared__ float pv[AT];
  if (tid < D) qs[tid] = q[(int64_t)b * q_bs + (int64_t)t * q_ld + h * D + tid] * scale;
  __syncthreads();
  const float* kb = k_ring + (int64_t)b * ring_bs + h * D;
  const float* vb = v_ring + (int64_t)b * ring_bs + h * D;
  float mx = -INFINITY;
  for (int j = tid; j < n; j += AT) {
    const float4* kr = reinterpret_cast<const float4*>(kb + (int64_t)((lo + j) % cap) * HD);
    float s = 0.f;
#pragma unroll
    for (int d4 = 0; d4 < D / 4; d4++) {
      const float4 kv = kr[d4];
      s = fmaf(qs[4 * d4], kv.x, s);
      s = fmaf(qs[4 * d4 + 1], kv.y, s);
      s = fmaf(qs[4 * d4 + 2], kv.z, s);
      s = fmaf(qs[4 * d4 + 3], kv.w, s);
    }
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int u = 1; u < AT / 32; u++) mx = fmaxf(mx, red[u]);
  __syncthreads();
  float sum = 0.f;
  for (int j = tid; j < n; j += AT) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  sum = red[0];
#pragma unroll
  for (int u = 1; u < AT / 32; u++) sum += red[u];
  const int d = tid & (D - 1), half = tid / D;
  float acc = 0.f;
  for (int j = half; j < n; j += AT / D) acc = fmaf(sc[j], vb[(int64_t)((lo + j) % cap) * HD + d], acc);
  pv[tid] = acc;
  __syncthreads();
  if (tid < D) out[(int64_t)b * o_bs + (int64_t)t * o_ld + h * D + d] = (pv[tid] + pv[tid + D]) / sum;
}

__global__ void stream_advance_kernel(int32_t* ctr, int32_t dpos) {
  ctr[0] += dpos;
  ctr[1] += 1;
}

bool conv_extras_ok(const b2a_conv1d_t* p) {
  return !p->pre_scale && !p->pre_shift && !p->pre_a && !p->pre_b && p->pre_act != B2A_ACT_SNAKE && !p->emit_hi && !p->emit_lo &&
         !p->accumulate;
}

}  // namespace

extern "C" int32_t b2a_conv1d_stream(const b2a_conv1d_t* p, float* hist, int64_t hist_bs, int32_t H, const int32_t* step_dev, int32_t fresh,
                                     void* stream) {
  B2A_CHECK_ARG(p && p->w && hist && step_dev && (p->y || p->Lout == 0), "null pointer");
  B2A_CHECK_ARG(p->x || p->L == 0, "null input with rows");
  B2A_CHECK_ARG(p->B > 0 && p->L >= 0 && p->Cin > 0 && p->Cout > 0 && p->K > 0 && p->stride > 0 && p->dilation > 0 && H >= 0,
                "bad shape");
  B2A_CHECK_ARG(p->groups == 1, "dense convolutions only");
  B2A_CHECK_ARG(p->pad_mode == 0 || p->pad_mode == 1, "pad_mode must be 0 (zeros) or 1 (edge)");
  B2A_CHECK_ARG(conv_extras_ok(p), "unsupported prologue / epilogue field (pre_scale/shift, snake, emit, accumulate)");
  B2A_CHECK_ARG(!p->res || p->res_div >= 1, "res_div must be >= 1");
  // Padded rows are zeros of the activated input: a prologue with act(0) != 0 would turn them into act(0) (the carry stores raw rows).
  B2A_CHECK_ARG(p->pad_mode == 1 || p->pre_act != B2A_ACT_SIGMOID, "a sigmoid prologue needs pad_mode 1 (act(0) != 0)");
  const int keff = (p->K - 1) * p->dilation + 1, V = H + p->L;
  B2A_CHECK_ARG(p->stride <= keff, "stride longer than the window (keff): the carry would go negative");
  const int lout = V >= keff ? (V - keff) / p->stride + 1 : 0;
  B2A_CHECK_ARG(p->Lout == lout, "Lout must be the number of complete windows of [history | new rows]");
  B2A_CHECK_ARG(V - lout * p->stride <= keff - 1, "history slot too small");
  B2A_CHECK_ARG(hist_bs >= (int64_t)(keff - 1) * p->Cin, "history batch stride shorter than keff - 1 rows");
  B2A_CHECK_ARG(!fresh || p->L > 0 || p->Lout == 0, "bad fresh call");
  ConvStreamArgs a;
  a.p = *p;
  a.hist = hist;
  a.hist_bs = hist_bs;
  a.H = H;
  a.fresh = fresh;
  a.step = step_dev;
  const int row_tiles = cdiv(lout, ROW_T);
  dim3 grid(cdiv(p->Cout, CO_T), row_tiles + 1, p->B);
  conv_stream_kernel<<<grid, CO_T * RED_W, 0, (cudaStream_t)stream>>>(a, row_tiles);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_convtr1d_stream(const b2a_conv1d_t* p, float* tail, int64_t tail_bs, void* stream) {
  B2A_CHECK_ARG(p && p->x && p->w && p->y && (tail || p->K == p->stride), "null pointer");     // K == stride: no tail, never touched
  B2A_CHECK_ARG(p->B > 0 && p->L > 0 && p->Cin > 0 && p->Cout > 0 && p->stride > 0 && p->K >= p->stride, "bad shape");
  B2A_CHECK_ARG(p->Lout == p->L * p->stride, "Lout must be L * stride");
  B2A_CHECK_ARG(p->K - p->stride <= p->Lout, "tail longer than the output");
  B2A_CHECK_ARG(p->dilation == 1 && p->pad_left == 0 && p->pad_mode == 0, "dilation 1, no crop, zero padding only");
  B2A_CHECK_ARG(conv_extras_ok(p) && !p->res && !p->post_cscale && p->post_act == 0, "prologue activation and bias only");
  B2A_CHECK_ARG(tail_bs >= (int64_t)(p->K - p->stride) * p->Cout, "tail batch stride shorter than K - stride rows");
  if (p->groups == 1) {
    dim3 grid(cdiv(p->Cout, CO_T), cdiv(p->Lout, ROW_T), p->B);
    convtr_stream_kernel<<<grid, CO_T * RED_W, 0, (cudaStream_t)stream>>>(*p, tail, tail_bs);
  } else {
    B2A_CHECK_ARG(p->groups == p->Cin && p->Cin == p->Cout, "groups must be 1 or == Cin == Cout");
    const int64_t total = (int64_t)p->B * p->Lout * p->Cout;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    convtr_stream_dw_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(*p, tail, tail_bs);
  }
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_ring_rope_kv(float* qkv, int64_t qkv_bs, int64_t qkv_ld, int32_t B, int32_t T, int32_t H, int32_t D, float base,
                                    float* k_ring, float* v_ring, int64_t ring_bs, int32_t cap, const int32_t* pos_dev, void* stream) {
  B2A_CHECK_ARG(qkv && k_ring && v_ring && pos_dev, "null pointer");
  B2A_CHECK_ARG(B > 0 && T > 0 && H > 0 && D > 0 && D % 2 == 0 && cap >= T, "bad shape");
  B2A_CHECK_ARG(qkv_ld >= 3 * H * D && ring_bs >= (int64_t)cap * H * D, "bad strides");
  const int64_t total = (int64_t)B * T * H * (D / 2);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  ring_rope_kv_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(qkv, qkv_bs, qkv_ld, B, T, H, D, base, k_ring, v_ring, ring_bs, cap, pos_dev);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_ring_attn(const float* q, int64_t q_bs, int64_t q_ld, const float* k_ring, const float* v_ring, int64_t ring_bs,
                                 int32_t cap, float* out, int64_t o_bs, int64_t o_ld, int32_t B, int32_t T, int32_t H, int32_t D, float scale,
                                 int32_t window, const int32_t* pos_dev, void* stream) {
  B2A_CHECK_ARG(q && k_ring && v_ring && out && pos_dev, "null pointer");
  B2A_CHECK_ARG(B > 0 && T > 0 && H > 0 && window > 0, "bad shape");
  if (D != 64) { b2a_set_error("b2a_ring_attn: head dim %d not supported (64)", D); return B2A_E_UNSUPPORTED; }
  B2A_CHECK_ARG(window <= WIN_MAX, "window longer than 1024 positions");
  B2A_CHECK_ARG(cap >= window + T - 1, "ring capacity below window + T - 1: new rows would overwrite keys still in a window");
  B2A_CHECK_ARG(((uintptr_t)k_ring & 15) == 0 && ((uintptr_t)v_ring & 15) == 0 && ring_bs % 4 == 0 && (H * D) % 4 == 0,
                "ring rows must be 16-byte aligned");
  ring_attn_kernel<<<dim3(T, H, B), AT, 0, (cudaStream_t)stream>>>(q, q_bs, q_ld, k_ring, v_ring, ring_bs, cap, out, o_bs, o_ld, H, scale,
                                                                   window, pos_dev);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_stream_advance(int32_t* ctr, int32_t dpos, void* stream) {
  B2A_CHECK_ARG(ctr && dpos >= 0, "bad arguments");
  stream_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(ctr, dpos);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
