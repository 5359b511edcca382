// State of the incremental (streaming) Qwen3-TTS speech-tokenizer decoder: one grouped launch of row-range copies / adds
// (b2a_stream_rows).  Replaces the reference's per-layer concatenations:
//   CausalConv1d.step / DecoderInitialConv.step / DecoderOutputConv.step (speech_tokenizer.py:71-83, 719-728, 771-780):
//     the last H = (K-1)*dilation input rows become the history head of the next call's input buffer   -> copy entries;
//   ConvNeXtBlock.step (:151-159): the depthwise conv's history, the same copy;
//   DecoderBlockUpsample.step (:645-656): the transposed conv's r-row overflow (bias included) is added into the head of the next
//     call's output                                                                                    -> add entries;
//   DecoderTransformer's KVCache growth (:610-617 calls the cache; growth in 256-frame steps): old rows into the larger buffer -> copy.
// Every entry moves a [B, rows, C] fp32 row range between two views with explicit batch / row strides.  Entries of one launch run
// concurrently, so the host keeps the ranges disjoint (ping-pong buffers: a history longer than the new rows reads rows of the buffer
// that the same carry would otherwise overwrite); b2a_stream_rows rejects overlapping ranges.
#include "common.cuh"

struct RowOpTable {
  b2a_rowop_t e[B2A_ROWOPS_MAX];
};

// blockIdx.y = entry; the x-blocks stride over its B * rows * C elements (float4 when every row start is 16-byte aligned).
__global__ void __launch_bounds__(256) stream_rows_kernel(const RowOpTable t) {
  const b2a_rowop_t& e = t.e[blockIdx.y];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool vec = ((e.C | e.src_bs | e.src_ld | e.dst_bs | e.dst_ld) & 3) == 0 && (((uintptr_t)e.src | (uintptr_t)e.dst) & 15) == 0;
  if (vec) {
    const int c4 = e.C >> 2;
    const int64_t total = (int64_t)e.B * e.rows * c4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
      const int c = (int)(i % c4) * 4;
      const int64_t br = i / c4;
      const int b = (int)(br / e.rows), r = (int)(br % e.rows);
      const float4 s = *reinterpret_cast<const float4*>(e.src + b * e.src_bs + r * e.src_ld + c);
      float4* d = reinterpret_cast<float4*>(e.dst + b * e.dst_bs + r * e.dst_ld + c);
      if (e.op == B2A_ROWOP_ADD) {
        const float4 o = *d;
        *d = make_float4(o.x + s.x, o.y + s.y, o.z + s.z, o.w + s.w);
      } else {
        *d = s;
      }
    }
  } else {
    const int64_t total = (int64_t)e.B * e.rows * e.C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
      const int c = (int)(i % e.C);
      const int64_t br = i / e.C;
      const int b = (int)(br / e.rows), r = (int)(br % e.rows);
      const float s = e.src[b * e.src_bs + r * e.src_ld + c];
      float* d = e.dst + b * e.dst_bs + r * e.dst_ld + c;
      *d = e.op == B2A_ROWOP_ADD ? *d + s : s;
    }
  }
}

// Byte span [lo, hi) an entry's view touches (conservative for strided views: first to last element).
static void span(const float* p, int64_t bs, int64_t ld, const b2a_rowop_t& e, uintptr_t* lo, uintptr_t* hi) {
  const int64_t last = (int64_t)(e.B - 1) * bs + (int64_t)(e.rows - 1) * ld + (e.C - 1);
  *lo = (uintptr_t)p;
  *hi = (uintptr_t)(p + last + 1);
}

static bool overlap(uintptr_t a0, uintptr_t a1, uintptr_t b0, uintptr_t b1) { return a0 < b1 && b0 < a1; }

extern "C" int32_t b2a_stream_rows(const b2a_rowop_t* ops, int32_t n, void* stream) {
  B2A_CHECK_ARG(ops && n >= 0 && n <= B2A_ROWOPS_MAX, "bad table / too many entries");
  RowOpTable t;
  int m = 0;
  int64_t most = 0;
  for (int i = 0; i < n; i++) {
    const b2a_rowop_t& e = ops[i];
    B2A_CHECK_ARG(e.src && e.dst && e.B >= 0 && e.rows >= 0 && e.C >= 0 && (e.op == B2A_ROWOP_COPY || e.op == B2A_ROWOP_ADD),
                  "bad entry");
    B2A_CHECK_ARG(e.src_ld >= e.C && e.dst_ld >= e.C, "row stride shorter than a row");
    if ((int64_t)e.B * e.rows * e.C == 0) continue;
    t.e[m++] = e;
    const int64_t sz = (int64_t)e.B * e.rows * e.C;
    if (sz > most) most = sz;
  }
  if (m == 0) return B2A_OK;
  for (int i = 0; i < m; i++) {
    uintptr_t d0, d1, s0, s1;
    span(t.e[i].dst, t.e[i].dst_bs, t.e[i].dst_ld, t.e[i], &d0, &d1);
    span(t.e[i].src, t.e[i].src_bs, t.e[i].src_ld, t.e[i], &s0, &s1);
    B2A_CHECK_ARG(!overlap(d0, d1, s0, s1), "an entry's source and destination overlap");
    for (int j = 0; j < m; j++) {
      if (j == i) continue;
      uintptr_t a0, a1, b0, b1;
      span(t.e[j].src, t.e[j].src_bs, t.e[j].src_ld, t.e[j], &a0, &a1);
      span(t.e[j].dst, t.e[j].dst_bs, t.e[j].dst_ld, t.e[j], &b0, &b1);
      B2A_CHECK_ARG(!overlap(d0, d1, a0, a1) && !overlap(d0, d1, b0, b1), "an entry writes rows another entry of the launch reads or writes");
    }
  }
  for (int i = m; i < B2A_ROWOPS_MAX; i++) t.e[i] = t.e[0];     // never read (grid.y = m); keeps the parameter block initialised
  int bx = (int)((most / 4 + 255) / 256);
  if (bx < 1) bx = 1;
  if (bx > 132 * 4) bx = 132 * 4;
  stream_rows_kernel<<<dim3(bx, m), 256, 0, (cudaStream_t)stream>>>(t);
  B2A_CHECK_LAUNCH();
  return B2A_OK;
}
