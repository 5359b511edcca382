// Fused Whisper decode step (include/b200audio.h: b2a_whisper_greedy_step): SuppressBlank + SuppressTokens +
// ApplyTimestampRules + GreedyDecoder.update (stt/models/whisper/decoding.py:307-325,349-442) in one launch, token
// history read on the device -- the reference builds the timestamp mask on the host from tokens.tolist() every step.
#include "common.cuh"

namespace {

struct GreedyParams {
  const float* logits; int64_t logits_bs;       // [B, V] (last position)
  const int64_t* tokens; int64_t tokens_bs;     // [B, >= cur_len] history incl. the sot sequence
  int cur_len, sample_begin, V;
  const float* suppress;                        // [V] additive mask (0 / -inf) or NULL
  const float* blank;                           // [V] additive mask for the first sampled position or NULL
  int eot, no_timestamps, timestamp_begin, max_initial_ts, without_timestamps;
  int64_t* next_out;                            // [B]
  float* sum_logprobs;                          // [B] in/out
  int* not_done;                                // [1] incremented when a row's next token is not eot
  float temperature; const float* u;            // temperature > 0: categorical draw from softmax(filtered / temperature) by inverse CDF in
                                                // index order, driven by u[b] in [0,1) (decoding.py:295-316)
};

__device__ __forceinline__ float block_max(float v, float* sh) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = sh[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); i++) r = fmaxf(r, sh[i]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); i++) r += sh[i];
  __syncthreads();
  return r;
}

// one CTA per batch row
__global__ void whisper_greedy_kernel(const GreedyParams p) {
  __shared__ float sh[32];
  __shared__ int s_flags[4];                    // last_ts, pen_ts, ts_limit (exclusive upper end of the forbidden timestamp range), first
  __shared__ unsigned long long s_best;
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const float* lg = p.logits + (int64_t)b * p.logits_bs;
  const int64_t* tk = p.tokens + (int64_t)b * p.tokens_bs;
  const int tb = p.timestamp_begin;
  const bool first = p.cur_len == p.sample_begin;
  if (tid == 0) {
    const int n = p.cur_len - p.sample_begin;
    const int64_t* seq = tk + p.sample_begin;
    const int last_ts = n >= 1 && seq[n - 1] >= tb;
    const int pen_ts = n < 2 || seq[n - 2] >= tb;
    // The reference's "timestamps must not decrease" mask is `mask[k, timestamp_begin : last_timestamp]` where
    // last_timestamp is the POSITION of the last timestamp token in the sampled sequence (decoding.py:400-408), i.e. a slice
    // [50364 : small index) that is always empty.  Reproduced as the no-op it is: limit = timestamp_begin.
    const int limit = tb;
    s_flags[0] = last_ts; s_flags[1] = pen_ts; s_flags[2] = limit; s_best = 0ull;
  }
  __syncthreads();
  const int last_ts = s_flags[0], pen_ts = s_flags[1], limit = s_flags[2];
  const float NEG = -INFINITY;
  // filtered logit BEFORE the timestamp-rule mask (what ApplyTimestampRules sees), and the rule mask without the probability test
  auto pre = [&](int v) -> float {
    float x = lg[v];
    if (first && p.blank) x += p.blank[v];
    if (p.suppress) x += p.suppress[v];
    return x;
  };
  auto rule_masked = [&](int v) -> bool {
    if (p.without_timestamps) return false;
    if (v == p.no_timestamps) return true;
    if (last_ts) { if (pen_ts) { if (v >= tb) return true; } else { if (v < p.eot) return true; } }
    if (v >= tb && v < limit) return true;
    if (first) { if (v < tb) return true; if (p.max_initial_ts >= 0 && v > tb + p.max_initial_ts) return true; }
    return false;
  };
  bool text_masked = false;
  if (!p.without_timestamps) {
    // logsumexp over timestamps vs max over text of the pre-mask logits (the normaliser cancels in the comparison)
    float mt = NEG, mx_ts = NEG;
    for (int v = tid; v < p.V; v += nt) { float x = pre(v); if (v < tb) mt = fmaxf(mt, x); else mx_ts = fmaxf(mx_ts, x); }
    mt = block_max(mt, sh); mx_ts = block_max(mx_ts, sh);
    float se = 0.f;
    if (mx_ts > NEG) for (int v = tb + tid; v < p.V; v += nt) se += expf(pre(v) - mx_ts);
    se = block_sum(se, sh);
    const float ts_lse = mx_ts > NEG ? mx_ts + logf(se) : NEG;
    text_masked = ts_lse > mt;
  }
  // final logits: argmax (lowest index on ties) and logsumexp
  float best = NEG; int besti = 0x7fffffff;
  for (int v = tid; v < p.V; v += nt) {
    float x = (rule_masked(v) || (text_masked && v < tb)) ? NEG : pre(v);
    if (x > best) { best = x; besti = v; }
  }
  const float gmax = block_max(best, sh);
  if (tid == 0) s_best = gmax > NEG ? 0xffffffffull : 0ull;        // everything masked: argmax of all -inf is index 0 (mx.argmax)
  __syncthreads();
  if (gmax > NEG && best == gmax) atomicMin(&s_best, (unsigned long long)(unsigned)besti);   // lowest index on ties
  __syncthreads();
  float se = 0.f;
  if (gmax > NEG)
    for (int v = tid; v < p.V; v += nt) {
      float x = (rule_masked(v) || (text_masked && v < tb)) ? NEG : pre(v);
      se += expf(x - gmax);
    }
  se = block_sum(se, sh);
  __syncthreads();
  __shared__ double s_scan[512];
  __shared__ int s_pick, s_lastlive;
  float picked_logit = gmax;
  if (p.temperature > 0.f && gmax > NEG) {
    // categorical draw: every thread owns a contiguous index range; float64 range sums, block scan, then the owning thread walks its range
    auto fin = [&](int v) -> float { return (rule_masked(v) || (text_masked && v < tb)) ? NEG : pre(v); };
    const int per = (p.V + nt - 1) / nt, lo = tid * per, hi = min(p.V, lo + per);
    const double inv_t = 1.0 / (double)p.temperature;
    double mine = 0.0; int lastlive = -1;
    for (int v = lo; v < hi; v++) { const float x = fin(v); if (x > NEG) { mine += exp((double)(x - gmax) * inv_t); lastlive = v; } }
    if (tid == 0) { s_pick = -1; s_lastlive = -1; }
    s_scan[tid] = mine;
    __syncthreads();
    for (int o = 1; o < nt; o <<= 1) {                     // Hillis-Steele inclusive scan over the nt range sums
      const double t = tid >= o ? s_scan[tid - o] : 0.0;
      __syncthreads();
      s_scan[tid] += t;
      __syncthreads();
    }
    const double z = s_scan[nt - 1], target = (double)p.u[b] * z;
    atomicMax(&s_lastlive, lastlive);
    const double incl = s_scan[tid], excl = incl - mine;
    if (incl > target && !(excl > target)) {               // the first range whose inclusive sum passes the target
      double run = excl; int pick = lastlive;
      for (int v = lo; v < hi; v++) { const float x = fin(v); if (x > NEG) { run += exp((double)(x - gmax) * inv_t); if (run > target) { pick = v; break; } } }
      s_pick = pick;
    }
    __syncthreads();
    if (tid == 0) {
      const int pick = s_pick >= 0 ? s_pick : max(s_lastlive, 0);
      s_best = (unsigned long long)(unsigned)pick;
      s_scan[0] = (double)fin(pick);
    }
    __syncthreads();
    picked_logit = (float)s_scan[0];
  }
  if (tid == 0) {
    int nxt = (int)s_best;
    const float cur_lp = gmax > NEG ? (picked_logit - gmax) - logf(se) : NAN;   // logit[nxt] - logsumexp (argmax: logit[nxt] = gmax)
    const bool was_eot = tk[p.cur_len - 1] == p.eot;
    if (!was_eot) p.sum_logprobs[b] += cur_lp;
    if (was_eot) nxt = p.eot;
    p.next_out[b] = nxt;
    if (nxt != p.eot) atomicAdd(p.not_done, 1);
  }
}

}  // namespace

extern "C" int32_t b2a_whisper_greedy_step(const float* logits, int64_t logits_bs, const int64_t* tokens, int64_t tokens_bs,
                                           int32_t B, int32_t cur_len, int32_t sample_begin, int32_t V, const float* suppress_mask,
                                           const float* blank_mask, int32_t eot, int32_t no_timestamps, int32_t timestamp_begin,
                                           int32_t max_initial_ts, int32_t without_timestamps, int64_t* next_out,
                                           float* sum_logprobs, int32_t* not_done, float temperature, const float* u, void* stream) {
  B2A_CHECK_ARG(logits && tokens && next_out && sum_logprobs && not_done, "null pointer");
  B2A_CHECK_ARG(temperature >= 0.f && (temperature == 0.f || u), "temperature > 0 needs one uniform per row");
  B2A_CHECK_ARG(B > 0 && V > 0 && cur_len >= sample_begin && cur_len >= 1 && timestamp_begin > 0 && timestamp_begin <= V, "bad shape");
  GreedyParams p{logits, logits_bs, tokens, tokens_bs, cur_len, sample_begin, V, suppress_mask, blank_mask, eot, no_timestamps,
                 timestamp_begin, max_initial_ts, without_timestamps, next_out, sum_logprobs, not_done, temperature, u};
  whisper_greedy_kernel<<<B, 512, 0, (cudaStream_t)stream>>>(p);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}

// ------------------------------------------------------------------------------------------------------------------------
// Fused LM sampler (include/b200audio.h: b2a_sample_token): suppress -> repetition penalty -> temperature -> top-k -> top-p
// -> min-p -> categorical draw, the chain of tts/models/qwen3_tts/qwen3_tts.py:805-860 over lm/sample_utils.py:131-239,279.
// One CTA per row; the row (V <= 4096) is bitonic-sorted once in shared memory (value desc, index asc) and every filter is a
// rank / prefix test on that order.  The categorical draw is an inverse-CDF lookup in INDEX order driven by a caller-supplied
// uniform (MLX's PRNG cannot be reproduced, so parity tests inject u; production draws it with b2a_randn's Philox stream).
namespace {

constexpr int SV = 4096;

struct SampleParams {
  const float* logits; int64_t logits_bs; int V;
  const float* suppress;                  // [V] additive 0/-inf or NULL
  uint8_t* seen; int64_t seen_bs;         // [B,V] 1 = token already generated (repetition penalty set) or NULL
  int mark_seen; int64_t out_stride;      // mark_seen: set seen[b][token] after the draw; out[b * out_stride]
  uint8_t* finished; int eos;             // batch loop (qwen3_tts.py:1880-1887): finished rows emit eos; finished |= (token == eos)
  float rep_penalty, temperature; int top_k; float top_p, min_p;
  const float* u;                         // [B] uniforms in [0,1)
  int64_t* out;                           // [B]
  float* filtered;                        // [B,V] optional: the filtered logits the draw is made from (tests)
};

// categorical draw from the filtered logits lg[0..V) (index order, -inf = removed): inverse CDF with the supplied uniform, done by
// warp 0 in float64 over 32 contiguous chunks.  gm = max of lg.
__device__ __forceinline__ void draw_inverse_cdf(const SampleParams& p, const float* lg, int V, int b, float gm) {
  const float NEG = -INFINITY;
  const int tid = threadIdx.x;
  const float* s_scan = lg;
  if (tid < 32) {
    const int lane = tid, per = (V + 31) / 32, lo = lane * per, hi = min(V, lo + per);
    double sum = 0.0; int lastlive = -1;
    for (int v = lo; v < hi; v++) if (s_scan[v] > NEG) { sum += exp((double)(s_scan[v] - gm)); lastlive = v; }
    double inc = sum;
    for (int o = 1; o < 32; o <<= 1) { double t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    const double z = __shfl_sync(0xffffffffu, inc, 31);
    const double target = (double)p.u[b] * z;
    int glast = lastlive;
    for (int o = 16; o > 0; o >>= 1) glast = max(glast, __shfl_xor_sync(0xffffffffu, glast, o));
    const unsigned ball = __ballot_sync(0xffffffffu, inc > target);
    int pick = -1;
    if (ball) {
      const int L = __ffs(ball) - 1;
      if (lane == L) {
        double run = inc - sum;
        pick = lastlive;
        for (int v = lo; v < hi; v++) if (s_scan[v] > NEG) { run += exp((double)(s_scan[v] - gm)); if (run > target) { pick = v; break; } }
      }
      pick = __shfl_sync(0xffffffffu, pick, L);
    } else pick = glast;
    if (lane == 0) {
      if (pick < 0) pick = 0;
      bool live = true;
      if (p.finished) { if (p.finished[b]) { pick = p.eos; live = false; } else if (pick == p.eos) { p.finished[b] = 1; live = false; } }
      p.out[(int64_t)b * p.out_stride] = pick;
      if (p.mark_seen && p.seen && live) p.seen[(int64_t)b * p.seen_bs + pick] = 1;
    }
  }
}

__global__ void __launch_bounds__(1024) sample_kernel(const SampleParams p) {
  __shared__ float sv[SV];
  __shared__ unsigned short si[SV];               // indices < 4096 fit 16 bits (keeps static shared memory under 48 KB)
  __shared__ float red[32];
  __shared__ float s_scan[SV];
  const int b = blockIdx.x, tid = threadIdx.x, V = p.V;
  const float NEG = -INFINITY;
  const float* lg = p.logits + (int64_t)b * p.logits_bs;
  pdl_launch_dependents();
  pdl_wait();
  auto base = [&](int v) -> float {
    float x = lg[v];
    if (p.suppress) x += p.suppress[v];
    if (p.seen && p.seen[(int64_t)b * p.seen_bs + v] && p.rep_penalty != 1.f) x = x < 0.f ? x * p.rep_penalty : x / p.rep_penalty;
    return x;
  };
  if (p.temperature <= 0.f) {                                       // greedy (qwen3_tts.py:845-846): argmax, lowest index on ties
    float best = NEG; int bi = 0x7fffffff;
    for (int v = tid; v < V; v += blockDim.x) { float x = base(v); if (x > best) { best = x; bi = v; } }
    int* gi = reinterpret_cast<int*>(s_scan);
    sv[tid] = best; gi[tid] = bi;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
      if (tid < s) { if (sv[tid + s] > sv[tid] || (sv[tid + s] == sv[tid] && gi[tid + s] < gi[tid])) { sv[tid] = sv[tid + s]; gi[tid] = gi[tid + s]; } }
      __syncthreads();
    }
    if (tid == 0) {
      int pick = gi[0] == 0x7fffffff ? 0 : gi[0];
      bool live = true;
      if (p.finished) { if (p.finished[b]) { pick = p.eos; live = false; } else if (pick == p.eos) { p.finished[b] = 1; live = false; } }
      p.out[(int64_t)b * p.out_stride] = pick;
      if (p.mark_seen && p.seen && live) p.seen[(int64_t)b * p.seen_bs + pick] = 1;
    }
    return;
  }
  // logits / temperature as the reference divides: a multiply by 1 / t rounds differently for many float32 inputs (about a
  // quarter at t = 0.9) and can split two logits that tie after the division, which moves the top-k cut
  for (int v = tid; v < SV; v += blockDim.x) { sv[v] = v < V ? base(v) / p.temperature : NEG; si[v] = v; }
  __syncthreads();
  const bool filters_p = (p.top_p > 0.f && p.top_p < 1.f) || p.min_p > 0.f;
  if (!filters_p) {
    // ---- fast path (the Qwen3 defaults: top-k only): k-th largest by a 4-pass radix select on order-preserving keys, ties by
    // lowest index, instead of sorting all V logits.
    __shared__ unsigned hist[256];
    __shared__ unsigned sel_prefix, sel_remaining;
    __shared__ unsigned wcnt[32];
    // -0.0 takes the key of +0.0: the two compare equal, so they tie and the lower index wins, as on the sorted path
    auto keyof = [](float x) -> unsigned {
      unsigned u = __float_as_uint(x);
      if (u == 0x80000000u) u = 0u;
      return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    };
    const bool use_k = p.top_k > 0 && p.top_k < V;
    if (use_k) {
      if (tid == 0) { sel_prefix = 0u; sel_remaining = (unsigned)p.top_k; }
      for (int pass = 0; pass < 4; pass++) {
        const int shift = 24 - 8 * pass;
        if (tid < 256) hist[tid] = 0u;
        __syncthreads();
        const unsigned pref = sel_prefix, mask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
        for (int v = tid; v < V; v += blockDim.x) {
          const unsigned k = keyof(sv[v]);
          if ((k & mask) == pref) atomicAdd(&hist[(k >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid < 32) {                                              // lane owns bins [255 - 8*lane - 7, 255 - 8*lane] (descending)
          unsigned c[8], sum = 0u;
#pragma unroll
          for (int j = 0; j < 8; j++) { c[j] = hist[255 - (tid * 8 + j)]; sum += c[j]; }
          unsigned inc = sum;
          for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, inc, o); if (tid >= o) inc += t; }
          const unsigned rem = sel_remaining;
          const unsigned ball = __ballot_sync(0xffffffffu, inc >= rem);
          const int L = __ffs(ball) - 1;                             // first lane whose cumulative count reaches the remaining rank
          if (tid == L) {
            unsigned before = inc - sum;
            for (int j = 0; j < 8; j++) {
              if (before + c[j] >= rem) { sel_prefix = pref | ((unsigned)(255 - (tid * 8 + j)) << shift); sel_remaining = rem - before; break; }
              before += c[j];
            }
          }
        }
        __syncthreads();
      }
    }
    // survivors: key > T, plus the first sel_remaining (by index) of the elements with key == T
    const unsigned T = use_k ? sel_prefix : 0u;
    const unsigned need_eq = use_k ? sel_remaining : 0xFFFFFFFFu;
    const int per = (V + (int)blockDim.x - 1) / (int)blockDim.x, lo = tid * per, hi = min(V, lo + per);
    unsigned eq = 0u;
    for (int v = lo; v < hi; v++) eq += (use_k && keyof(sv[v]) == T) ? 1u : 0u;
    unsigned inc = eq;
    for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(0xffffffffu, inc, o); if ((tid & 31) >= o) inc += t; }
    if ((tid & 31) == 31) wcnt[tid >> 5] = inc;
    __syncthreads();
    unsigned woff = 0u;
    for (int w = 0; w < (tid >> 5); w++) woff += wcnt[w];
    unsigned rank = woff + inc - eq;                                 // equal-key elements before this thread's chunk
    float m2 = NEG;
    for (int v = lo; v < hi; v++) {
      float x = sv[v];
      if (use_k) {
        const unsigned k = keyof(x);
        bool keep = k > T;
        if (k == T) { keep = rank < need_eq; rank++; }
        if (!keep) x = NEG;
      }
      s_scan[v] = x;
      m2 = fmaxf(m2, x);
    }
    m2 = warp_max(m2);
    if ((tid & 31) == 0) red[tid >> 5] = m2;
    __syncthreads();
    float gm = red[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); i++) gm = fmaxf(gm, red[i]);
    if (p.filtered) for (int v = tid; v < V; v += blockDim.x) p.filtered[(int64_t)b * V + v] = s_scan[v];
    __syncthreads();
    draw_inverse_cdf(p, s_scan, V, b, gm);
    return;
  }
  // bitonic sort: descending value, ascending index among equals
  for (int k = 2; k <= SV; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < SV; i += blockDim.x) {
        int l = i ^ j;
        if (l > i) {
          bool desc = (i & k) == 0;
          float a = sv[i], c = sv[l]; unsigned short ai = si[i], ci = si[l];
          bool a_first = a > c || (a == c && ai < ci);              // a should come before c in the final order
          if (a_first != desc) { sv[i] = c; sv[l] = a; si[i] = ci; si[l] = ai; }
        }
      }
      __syncthreads();
    }
  // top-k: ranks >= k are removed
  const bool use_k = p.top_k > 0 && p.top_k < V;
  const int kcut = use_k ? p.top_k : V;
  const float vmax = sv[0];
  // softmax over the survivors (log_softmax of the top-k-masked logits)
  float se = 0.f;
  for (int r = tid; r < kcut; r += blockDim.x) se += sv[r] > NEG ? expf(sv[r] - vmax) : 0.f;
  se = warp_sum(se);
  if ((tid & 31) == 0) red[tid >> 5] = se;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); i++) tot += red[i];
  __syncthreads();
  const float lse = vmax + logf(tot);
  // top-p (ascending inclusive cumulative probability > 1 - top_p survives) and min-p on the sorted order
  const bool use_p = p.top_p > 0.f && p.top_p < 1.f;
  // inclusive prefix over DESCENDING ranks; ascending-inclusive cum of rank r = 1 - (prefix_desc_incl(r) - prob_r)
  for (int r = tid; r < SV; r += blockDim.x) s_scan[r] = (r < kcut && sv[r] > NEG) ? expf(sv[r] - lse) : 0.f;
  __syncthreads();
  for (int off = 1; off < SV; off <<= 1) {                          // Hillis-Steele scan (4096 elements, 1024 threads)
    float t[4];
    for (int q = 0; q < 4; q++) { int r = tid + q * blockDim.x; t[q] = (r >= off && r < SV) ? s_scan[r - off] : 0.f; }
    __syncthreads();
    for (int q = 0; q < 4; q++) { int r = tid + q * blockDim.x; if (r < SV) s_scan[r] += t[q]; }
    __syncthreads();
  }
  const float logminp = p.min_p > 0.f ? logf(p.min_p) : NEG;
  for (int r = tid; r < SV; r += blockDim.x) {
    bool keep = r < kcut && sv[r] > NEG;
    if (keep && use_p) {
      float pr = expf(sv[r] - lse);
      float cum_asc = 1.f - (s_scan[r] - pr);                       // sum of this and all smaller probabilities
      keep = cum_asc > 1.f - p.top_p;
    }
    if (keep && p.min_p > 0.f) keep = !((sv[r] - lse) < (vmax - lse) + logminp);     // remove logprob < max logprob + log(min_p)
    if (!keep) sv[r] = NEG;
  }
  __syncthreads();
  // scatter the filtered logits back to index order (s_scan reused as [V] buffer)
  for (int r = tid; r < SV; r += blockDim.x) if (si[r] < V) s_scan[si[r]] = sv[r];
  __syncthreads();
  if (p.filtered) for (int v = tid; v < V; v += blockDim.x) p.filtered[(int64_t)b * V + v] = s_scan[v];
  // categorical draw: inverse CDF in index order with the supplied uniform
  float m2 = NEG;
  for (int v = tid; v < V; v += blockDim.x) m2 = fmaxf(m2, s_scan[v]);
  m2 = warp_max(m2);
  if ((tid & 31) == 0) red[tid >> 5] = m2;
  __syncthreads();
  float gm = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); i++) gm = fmaxf(gm, red[i]);
  __syncthreads();
  draw_inverse_cdf(p, s_scan, V, b, gm);
}

}  // namespace

extern "C" int32_t b2a_sample_token(const float* logits, int64_t logits_bs, int32_t B, int32_t V, const float* suppress_mask,
                                    uint8_t* seen, int64_t seen_bs, int32_t mark_seen, float repetition_penalty, float temperature,
                                    int32_t top_k, float top_p, float min_p, const float* u, int64_t* out, int64_t out_stride,
                                    float* filtered_out, uint8_t* finished, int32_t eos, void* stream) {
  B2A_CHECK_ARG(logits && out && B > 0 && V > 0, "bad pointers/shape");
  B2A_CHECK_ARG(temperature <= 0.f || u != nullptr, "a uniform draw per row is required when temperature > 0");
  if (V > SV) { b2a_set_error("b2a_sample_token: vocab %d > %d not supported", V, SV); return B2A_E_UNSUPPORTED; }
  B2A_CHECK_ARG(min_p >= 0.f && min_p <= 1.f, "`min_p` has to be a float in the [0, 1] interval");
  SampleParams p{logits, logits_bs, V, suppress_mask, seen, seen_bs, mark_seen, out_stride < 1 ? 1 : out_stride, finished, eos, repetition_penalty, temperature, top_k, top_p, min_p, u, out, filtered_out};
  b2a_launch_pdl(sample_kernel, dim3(B), dim3(1024), 0, (cudaStream_t)stream, p);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
