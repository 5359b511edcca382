// Soprano TTS (include/b200audio.h: b2a_lm_sample_mlx, b2a_soprano_upsample, b2a_soprano_store_rows).
//
// b2a_lm_sample_mlx is mlx-lm's make_sampler(temp, top_p) (lm/sample_utils.py:11-70, 206-238, 279) on RAW logits, the way
// tts/models/soprano/soprano.py:336-346 calls it: apply_top_p exponentiates the logits without normalising them, so a token is kept
// iff the ascending-order inclusive cumulative sum of exp(logit) up to it exceeds 1 - top_p.  The kept set is a suffix of the ascending
// order; its first element is found by an 8-pass radix select (4-bit digits) on order-preserving keys, each pass building per-digit
// exp-sum histograms in fixed order (one shared-memory column per thread, no atomics), so a row's result never depends on B.
#include <cuda_bf16.h>
#include "common.cuh"

namespace {

constexpr int LS_THREADS = 512;
constexpr int LS_BINS = 16;
constexpr int LS_CACHE_MAX = 36864;             // rows of at most this many logits are staged in shared memory (147 KB)

struct LmSampleParams {
  const float* logits; int64_t logits_bs; int V;
  float inv_temp;                               // float32(1 / temp): categorical_sampling multiplies by it (sample_utils.py:279)
  double thr;                                   // 1 - top_p; < 0 disables the filter
  int greedy;                                   // temp == 0: argmax
  const float* u; int64_t u_bs; const int32_t* step;
  int64_t* out; int64_t* hist; int64_t hist_bs;
  uint8_t* finished; int stop0, stop1;
  int cache;
};

// ascending order-preserving key; -0.0 takes the key of +0.0 (they compare equal, so they tie and the lower index comes first)
__device__ __forceinline__ unsigned asc_key(float x) {
  unsigned u = __float_as_uint(x);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// exp(t) for t <= 0 in float64 to a few ulp (Cody-Waite reduction by ln 2, degree-12 Taylor on |r| <= ln 2 / 2): libm's exp carries a
// slow path whose stack frame would spill here.  Below -745 (and for -inf) the result is 0, as exp's.
__device__ __forceinline__ double exp_nonpos(double t) {
  if (!(t > -745.0)) return 0.0;
  const double n = rint(t * 1.4426950408889634);
  const double r = fma(-n, 1.9082149292705877e-10, fma(-n, 0.6931471803691238, t));
  double q = 1.0 / 479001600.0;
  q = fma(q, r, 1.0 / 39916800.0); q = fma(q, r, 1.0 / 3628800.0); q = fma(q, r, 1.0 / 362880.0); q = fma(q, r, 1.0 / 40320.0);
  q = fma(q, r, 1.0 / 5040.0); q = fma(q, r, 1.0 / 720.0); q = fma(q, r, 1.0 / 120.0); q = fma(q, r, 1.0 / 24.0);
  q = fma(q, r, 1.0 / 6.0); q = fma(q, r, 0.5); q = fma(q, r, 1.0); q = fma(q, r, 1.0);
  const int k = (int)n;                                                  // 2^k in two steps so that subnormal results stay exact
  const int k1 = k / 2, k2 = k - k1;
  return q * __longlong_as_double((long long)(1023 + k1) << 52) * __longlong_as_double((long long)(1023 + k2) << 52);
}

__global__ void __launch_bounds__(LS_THREADS) lm_sample_mlx_kernel(const LmSampleParams p) {
  extern __shared__ __align__(16) unsigned char ls_smem[];
  double* hs = reinterpret_cast<double*>(ls_smem);                       // [LS_BINS][LS_THREADS] per-thread digit sums
  float* lgs = reinterpret_cast<float*>(hs + LS_BINS * LS_THREADS);     // [V] staged row (p.cache)
  __shared__ double s_scan[LS_THREADS];
  __shared__ double s_bins[LS_BINS];
  __shared__ int s_cnt[LS_THREADS];
  __shared__ float s_bv[LS_THREADS / 32];
  __shared__ int s_bi[LS_THREADS / 32];
  __shared__ unsigned s_prefix;
  __shared__ double s_below;
  __shared__ int s_state, s_skip, s_pick, s_lastlive;
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, V = p.V;
  const int step = p.step ? *p.step : 0;
  if (p.finished && p.finished[b]) return;                               // a finished row writes nothing
  const float* lg = p.logits + (int64_t)b * p.logits_bs;
  if (p.cache) {
    for (int v = tid; v < V; v += nt) lgs[v] = lg[v];
    __syncthreads();
    lg = lgs;
  }
  int tok = 0;
  if (p.greedy) {                                                       // mx.argmax: the first index of the maximum
    float best = -INFINITY; int bi = 0x7fffffff;
    for (int v = tid; v < V; v += nt) { const float x = lg[v]; if (x > best) { best = x; bi = v; } }
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if ((tid & 31) == 0) { s_bv[tid >> 5] = best; s_bi[tid >> 5] = bi; }
    __syncthreads();
    if (tid == 0) {
      float bv = s_bv[0]; int bix = s_bi[0];
      for (int w = 1; w < nt / 32; w++) if (s_bv[w] > bv || (s_bv[w] == bv && s_bi[w] < bix)) { bv = s_bv[w]; bix = s_bi[w]; }
      tok = bix == 0x7fffffff ? 0 : bix;
    }
  } else {
    // ---- keep set: every key above T, and the key-T elements from the s_skip-th (index order) on.  state: 0 all kept, 1 filtered,
    // 2 nothing kept (the total exp-sum does not exceed 1 - top_p).
    if (tid == 0) { s_state = 0; s_prefix = 0u; s_below = 0.0; s_skip = 0; }
    __syncthreads();
    if (p.thr >= 0.0) {
      unsigned prefix = 0u, mask = 0u;
      for (int pass = 0; pass < 8; pass++) {
        const int shift = 28 - 4 * pass;
#pragma unroll
        for (int d = 0; d < LS_BINS; d++) hs[d * nt + tid] = 0.0;
        for (int v = tid; v < V; v += nt) {
          const float x = lg[v];
          const unsigned k = asc_key(x);
          if ((k & mask) == prefix) hs[((k >> shift) & 15u) * nt + tid] += (double)expf(x);
        }
        __syncthreads();
        {                                                                // bin d = warp d: its 512 columns, 16 per lane, then a butterfly
          const int d = tid >> 5, lane = tid & 31;
          if (d < LS_BINS) {
            double s = 0.0;
            for (int j = 0; j < nt / 32; j++) s += hs[d * nt + lane * (nt / 32) + j];
            s = warp_sum_d(s);
            if (lane == 0) s_bins[d] = s;
          }
        }
        __syncthreads();
        if (tid == 0) {
          double run = s_below, run_last = 0.0; int sel = -1, last = -1;
          for (int d = 0; d < LS_BINS; d++) {
            if (s_bins[d] > 0.0) { last = d; run_last = run; }
            if (run + s_bins[d] > p.thr) { sel = d; break; }
            run += s_bins[d];
          }
          // past pass 0 the parent bin crossed 1 - top_p, but its children, summed in another order, can fall a rounding step short:
          // the crossing is then in the last non-empty child
          if (sel < 0 && pass > 0 && last >= 0) { sel = last; run = run_last; }
          if (sel < 0) s_state = 2;
          else { s_prefix = prefix | ((unsigned)sel << shift); s_below = run; }
        }
        __syncthreads();
        if (s_state == 2) break;
        prefix = s_prefix; mask |= 15u << shift;
      }
    }
    const int state = s_state == 2 ? 2 : (p.thr >= 0.0 ? 1 : 0);
    const unsigned T = s_prefix;
    // each thread owns a contiguous index range: the key-T elements before it (index order) and, below, its share of the draw
    const int per = (V + nt - 1) / nt, lo = min(V, tid * per), hi = min(V, lo + per);
    int neq = 0;
    if (state == 1) for (int v = lo; v < hi; v++) neq += asc_key(lg[v]) == T;
    s_cnt[tid] = neq;
    __syncthreads();
    if (tid == 0) {
      int run = 0;
      for (int t = 0; t < nt; t++) { const int c = s_cnt[t]; s_cnt[t] = run; run += c; }
      if (state == 1) {
        // the boundary among the n_T elements of key T (all equal to x_T): the first j with below + (j + 1) e_T > thr, summed in
        // order; at least the last of them is kept (the bin crossed, so only rounding can leave the running sum short)
        const float xt = __uint_as_float((T & 0x80000000u) ? (T & 0x7fffffffu) : ~T);
        const double et = (double)expf(xt);
        double acc = s_below; int j = 0;
        while (j < run - 1) { acc += et; if (acc > p.thr) break; j++; }
        s_skip = j;
      }
    }
    __syncthreads();
    if (state == 2) {
      tok = 0;                                                           // every logit -inf: categorical = argmax(-inf + gumbel) = 0
    } else {
      // ---- categorical draw: inverse CDF in index order of softmax(kept * inv_temp)
      const int skip = s_skip;
      const int rank0 = s_cnt[tid];
      auto kept = [&](float x, int& rank) -> bool {
        if (state == 0) return true;
        const unsigned k = asc_key(x);
        if (k > T) return true;
        if (k < T) return false;
        return rank++ >= skip;
      };
      float m = -INFINITY;
      { int rank = rank0; for (int v = lo; v < hi; v++) { const float x = lg[v]; if (kept(x, rank)) m = fmaxf(m, __fmul_rn(x, p.inv_temp)); } }
      m = warp_max(m);
      if ((tid & 31) == 0) s_bv[tid >> 5] = m;
      __syncthreads();
      float gm = s_bv[0];
      for (int w = 1; w < nt / 32; w++) gm = fmaxf(gm, s_bv[w]);
      double mine = 0.0; int lastlive = -1;
      { int rank = rank0;
        for (int v = lo; v < hi; v++) { const float x = lg[v]; if (kept(x, rank)) { mine += exp_nonpos((double)__fmul_rn(x, p.inv_temp) - (double)gm); lastlive = v; } } }
      if (tid == 0) { s_pick = -1; s_lastlive = -1; }
      s_scan[tid] = mine;
      __syncthreads();
      for (int o = 1; o < nt; o <<= 1) {                                 // Hillis-Steele inclusive scan: fixed order
        const double t = tid >= o ? s_scan[tid - o] : 0.0;
        __syncthreads();
        s_scan[tid] += t;
        __syncthreads();
      }
      const double z = s_scan[nt - 1], target = (double)p.u[(int64_t)b * p.u_bs + step] * z;
      atomicMax(&s_lastlive, lastlive);
      // the exclusive bound is the previous thread's inclusive sum, bit for bit, so exactly one range (or none: fallback below) matches
      const double incl = s_scan[tid], excl = tid ? s_scan[tid - 1] : 0.0;
      if (incl > target && !(excl > target)) {
        double run = excl; int pick = lastlive, rank = rank0;
        for (int v = lo; v < hi; v++) {
          const float x = lg[v];
          if (kept(x, rank)) { run += exp_nonpos((double)__fmul_rn(x, p.inv_temp) - (double)gm); if (run > target) { pick = v; break; } }
        }
        s_pick = pick;
      }
      __syncthreads();
      if (tid == 0) tok = s_pick >= 0 ? s_pick : max(s_lastlive, 0);
    }
  }
  if (tid == 0) {
    p.out[b] = tok;
    if (p.hist) p.hist[(int64_t)b * p.hist_bs + step] = tok;
    if (p.finished && (tok == p.stop0 || tok == p.stop1)) p.finished[b] = 1;
  }
}

// align-corners linear up-sampling (tts/models/interpolate.py:86-117): output row i of Lo reads rows floor(pos), min(floor(pos)+1, L-1)
// with pos = float(i) * scale in fp32, exactly the reference's arithmetic (no contraction)
__global__ void soprano_upsample_kernel(const float* __restrict__ x, int64_t x_bs, int64_t x_ld, int L, int H, int Lo, float scale,
                                        float* y, int64_t y_bs, int64_t y_ld, __nv_bfloat16* hi, __nv_bfloat16* lo, int cols) {
  const int i = blockIdx.x, b = blockIdx.y;
  int l0 = 0, l1 = 0; float f = 0.f;
  if (L > 1) {
    const float pos = __fmul_rn((float)i, scale);
    const float fl = floorf(pos);
    l0 = (int)fl; l1 = min(l0 + 1, L - 1); f = __fsub_rn(pos, fl);
  }
  const float* r0 = x + (int64_t)b * x_bs + (int64_t)l0 * x_ld;
  const float* r1 = x + (int64_t)b * x_bs + (int64_t)l1 * x_ld;
  const float g = __fsub_rn(1.f, f);
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    float v = 0.f;
    if (c < H) v = L > 1 ? __fadd_rn(__fmul_rn(r0[c], g), __fmul_rn(r1[c], f)) : r0[c];
    if (y) {
      y[(int64_t)b * y_bs + (int64_t)i * y_ld + c] = v;
    } else {
      const int64_t o = ((int64_t)b * Lo + i) * cols + c;
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      hi[o] = h;
      if (lo) lo[o] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
  }
}

__global__ void soprano_store_rows_kernel(const float* __restrict__ src, int64_t src_bs, int H, float* dst, int64_t dst_bs, int64_t dst_ld,
                                          const int32_t* idx, int add, int cap) {
  const int b = blockIdx.x;
  const int r = *idx + add;
  if (r < 0 || r >= cap) return;
  for (int c = threadIdx.x; c < H; c += blockDim.x) dst[(int64_t)b * dst_bs + (int64_t)r * dst_ld + c] = src[(int64_t)b * src_bs + c];
}

}  // namespace

extern "C" int32_t b2a_lm_sample_mlx(const float* logits, int64_t logits_bs, int32_t B, int32_t V, float temperature, double top_p,
                                     const float* u, int64_t u_bs, const int32_t* step_dev, int64_t* out, int64_t* hist, int64_t hist_bs,
                                     uint8_t* finished, int32_t stop0, int32_t stop1, void* stream) {
  B2A_CHECK_ARG(logits && out && B > 0 && V > 0 && logits_bs >= V, "bad pointers / shape");
  B2A_CHECK_ARG(temperature >= 0.f, "temperature must be >= 0");
  B2A_CHECK_ARG(temperature == 0.f || u, "a uniform per row and step is required when temperature > 0");
  LmSampleParams p{};
  p.logits = logits; p.logits_bs = logits_bs; p.V = V;
  p.greedy = temperature == 0.f;
  p.inv_temp = p.greedy ? 1.f : (float)(1.0 / (double)temperature);
  p.thr = (top_p > 0.0 && top_p < 1.0) ? 1.0 - top_p : -1.0;
  p.u = u; p.u_bs = u_bs; p.step = step_dev; p.out = out; p.hist = hist; p.hist_bs = hist_bs;
  p.finished = finished; p.stop0 = stop0; p.stop1 = stop1;
  p.cache = V <= LS_CACHE_MAX;
  const size_t smem = (size_t)LS_BINS * LS_THREADS * sizeof(double) + (p.cache ? (size_t)V * sizeof(float) : 0);
  B2A_SMEM_OPTIN(lm_sample_mlx_kernel, LS_BINS * LS_THREADS * sizeof(double) + LS_CACHE_MAX * sizeof(float));
  lm_sample_mlx_kernel<<<B, LS_THREADS, smem, (cudaStream_t)stream>>>(p);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_soprano_upsample(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t H, int32_t up, float* y,
                                        int64_t y_bs, int64_t y_ld, void* hi, void* lo, int32_t cpad, void* stream) {
  B2A_CHECK_ARG(x && B > 0 && L > 0 && H > 0 && up > 0 && x_ld >= H, "bad pointers / shape");
  B2A_CHECK_ARG((y != nullptr) != (hi != nullptr), "exactly one of y (fp32) and hi (bf16 planes)");
  B2A_CHECK_ARG(y ? y_ld >= H : cpad >= H, "output row narrower than H");
  const int Lo = up * (L - 1) + 1;
  const float scale = Lo > 1 ? (float)((double)(L - 1) / (double)(Lo - 1)) : 0.f;   // python float, then float32 (interpolate.py:87)
  dim3 grid(Lo, B);
  soprano_upsample_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(x, x_bs, x_ld, L, H, Lo, scale, y, y_bs, y_ld, (__nv_bfloat16*)hi,
                                                                  (__nv_bfloat16*)lo, y ? H : cpad);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

extern "C" int32_t b2a_soprano_store_rows(const float* src, int64_t src_bs, int32_t B, int32_t H, float* dst, int64_t dst_bs, int64_t dst_ld,
                                          const int32_t* idx_dev, int32_t add, int32_t cap, void* stream) {
  B2A_CHECK_ARG(src && dst && idx_dev && B > 0 && H > 0 && dst_ld >= H, "bad pointers / shape");
  soprano_store_rows_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(src, src_bs, H, dst, dst_bs, dst_ld, idx_dev, add, cap);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
