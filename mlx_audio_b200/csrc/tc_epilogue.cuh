// Per-element arithmetic of the tensor-core GEMM epilogue and of the operand planes it emits, shared by conv_tc_kernel (gemm_tc.cu)
// and the persistent ALBERT kernel (albert.cu), so that an output element goes through the same instructions whichever kernel
// computes it.
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace tc {

// Not inlined: the activation's result is rounded to fp32 before the scale / residual FMA, whatever the surrounding code.
static __device__ __noinline__ float act_noinline(float v, int act, float p0) { return b2a_act(v, act, p0, 1.f, 1.f); }

// y = act(acc + bias) * cso + rr, where cso = cscale * out_scale and rr = residual * out_scale (+ the previous output)
__device__ __forceinline__ float epilogue_value(float acc, float bias, int act, float p0, float cso, float rr) {
  if (act) return act_noinline(acc + bias, act, p0) * cso + rr;
  return (acc + bias) * cso + rr;
}

// Where one output column goes as split16 planes: hi / lo pointers at row 0, and the element step per row.
struct EmitCol { uint16_t *hi, *lo; int64_t step; float mul; bool f16; };

// Column n of a fused [q | k | v] projection (n = part * hs + head * 64 + d) in b2a_attention_tc's operand layout: fp16 Q (times
// qmul) and K [bh][T][64], V transposed [bh][64][tkp]; bh0 = batch * heads.
__device__ __forceinline__ EmitCol emit_col_attn(const AttnOperands& at, int64_t bh0, int T, int hs, float qmul, int n) {
  EmitCol c{nullptr, nullptr, 0, 1.f, true};
  const int part = n / hs, head = (n - part * hs) >> 6, d = n & 63;
  const int64_t bh = bh0 + head;
  if (part < 2) {
    const int64_t o = bh * T * 64 + d;
    c.hi = (uint16_t*)(part ? at.kh : at.qh) + o; c.lo = (uint16_t*)(part ? at.kl : at.ql) + o;
    c.step = 64; c.mul = part ? 1.f : qmul;
  } else {
    const int64_t o = (bh * 64 + d) * at.tkp;
    c.hi = (uint16_t*)at.vh + o; c.lo = (uint16_t*)at.vl + o; c.step = 1;
  }
  return c;
}

__device__ __forceinline__ void emit_store(const EmitCol& c, int64_t row, float v) {
  uint16_t h, l;
  if (c.f16) { __half a, b; split16(v * c.mul, a, b); h = __half_as_ushort(a); l = __half_as_ushort(b); }
  else { __nv_bfloat16 a, b; split16(v, a, b); h = __bfloat16_as_ushort(a); l = __bfloat16_as_ushort(b); }
  c.hi[row * c.step] = h;
  if (c.lo) c.lo[row * c.step] = l;
}

}  // namespace tc
