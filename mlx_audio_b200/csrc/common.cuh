// Shared device helpers for the b200audio kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <stdio.h>
#include "../../include/b200audio.h"

void b2a_set_error(const char* fmt, ...);

#define B2A_CHECK_ARG(cond, msg)                                   \
  do { if (!(cond)) { b2a_set_error("%s: %s", __func__, msg); return B2A_E_INVALID; } } while (0)

#define B2A_CHECK_LAUNCH()                                         \
  do { cudaError_t e_ = cudaGetLastError();                        \
       if (e_ != cudaSuccess) { b2a_set_error("%s: %s", __func__, cudaGetErrorString(e_)); return B2A_E_CUDA; } } while (0)

// Raise `kernel`'s dynamic shared-memory limit to at least `bytes` (api.cu).  Thread-safe; a limit never goes down, and the runtime is
// called only when it has to grow, so launch paths call this before every launch.
cudaError_t b2a_smem_optin(const void* kernel, int bytes);

// The same, returning B2A_E_CUDA from the calling function when the opt-in fails.  A template id with a comma goes in parentheses.
#define B2A_SMEM_OPTIN(kernel, bytes)                                                                                         \
  do { cudaError_t e_ = b2a_smem_optin((const void*)(kernel), (int)(bytes));                                                   \
       if (e_ != cudaSuccess) {                                                                                                 \
         b2a_set_error("%s: cannot raise the dynamic shared-memory limit to %d bytes: %s", __func__, (int)(bytes), cudaGetErrorString(e_)); \
         return B2A_E_CUDA; } } while (0)

// sin for the Snake activations: two-constant Cody-Waite reduction to [-pi, pi] + the SFU sine (abs error < 5e-7 there), ~6
// instructions instead of libm's ~40 -- the prologue kernels that apply Snake are otherwise instruction-bound, not HBM-bound.
__device__ __forceinline__ float b2a_sin(float x) {
  if (fabsf(x) > 8192.f) return sinf(x);
  const float k = rintf(x * 0.15915494309189535f);
  float r = fmaf(-k, 6.2831854820251465f, x);
  r = fmaf(-k, -1.7484555314695172e-07f, r);
  return __sinf(r);
}

// The same without the libm fall-back for huge arguments (its Payne-Hanek slow path is ~500 instructions of code per call site, which
// made the fused conv's converter loop instruction-cache-bound): three-constant Cody-Waite, accurate to ~1e-6 for |x| < 1e5 -- the Snake
// argument is alpha x a normalised activation, orders of magnitude below that; beyond it the result degrades gracefully (stays in [-1, 1]).
__device__ __forceinline__ float b2a_sin_fast(float x) {
  const float k = rintf(x * 0.15915494309189535f);
  float r = fmaf(-k, 6.28125f, x);                                   // 2 pi = 6.28125 + 1.9353071795864769e-3 (split so that k * C1 is exact)
  r = fmaf(-k, 1.9353071693331003e-3f, r);
  r = fmaf(-k, 1.0253331169063645e-11f, r);
  return __sinf(r);
}

__device__ __forceinline__ float b2a_act(float v, int act, float p0, float a, float b) {
  switch (act) {
    case B2A_ACT_LRELU: return v > 0.f ? v : v * p0;
    case B2A_ACT_SNAKE: { float s = b2a_sin(a * v); return fmaf(b, s * s, v); }
    case B2A_ACT_ELU: return v > 0.f ? v : expm1f(v);
    case B2A_ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
    case B2A_ACT_GELU_TANH: { float u = 0.7978845608028654f * (v + 0.044715f * v * v * v); return 0.5f * v * (1.f + tanhf(u)); }
    case B2A_ACT_TANH: return tanhf(v);
    case B2A_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case B2A_ACT_SILU: return v / (1.f + expf(-v));
    case B2A_ACT_CLIP1: return fminf(fmaxf(v, -1.f), 1.f);
    default: return v;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- reproducible (order-independent) accumulation of statistics --------------------------------------------------------------
// InstanceNorm (sum, sumsq) accumulators are added to by many CTAs in whatever order they finish.  Floating-point atomics would make
// the result depend on that order (graph replay != eager launch, run != run); so an accumulator is B2A_NBIN int64 bins, bin k counting
// multiples of 2^(B2A_BIN0 + 40 k).  An fp32 addend (24 significant bits) is split EXACTLY over the two bins it straddles and added with
// integer atomics -- associative, hence bit-reproducible -- and 23 bits of headroom per bin allow ~8 M addends.  Range 2^-100 .. 2^83;
// smaller parts are dropped, non-finite addends are ignored.
#define B2A_NBIN 4
#define B2A_BIN0 (-100)
#define B2A_BIN_BITS 40
__device__ __forceinline__ void repro_add(long long* bins, float v) {
  if (v == 0.f || !isfinite(v)) return;
  int e;
  frexpf(v, &e);                                       // |v| in [2^(e-1), 2^e)
  int k = (e - 1 - B2A_BIN0) / B2A_BIN_BITS;
  k = (e - 1) < B2A_BIN0 ? 0 : (k > B2A_NBIN - 1 ? B2A_NBIN - 1 : k);
  const double d = ldexp((double)v, -(B2A_BIN0 + B2A_BIN_BITS * k));
  const long long hi = (long long)d;                   // truncation; |d| < 2^63 inside the supported range
  atomicAdd(reinterpret_cast<unsigned long long*>(bins + k), (unsigned long long)hi);
  if (k > 0) {
    const long long lo = (long long)rint((d - (double)hi) * 1099511627776.0);     // exact: the addend's LSB is >= one unit of bin k-1
    if (lo) atomicAdd(reinterpret_cast<unsigned long long*>(bins + k - 1), (unsigned long long)lo);
  }
}
__device__ __forceinline__ void repro_add_d(long long* bins, double v) {   // float64 addend as two fp32 pieces (48 significant bits)
  const float h = (float)v;
  repro_add(bins, h);
  repro_add(bins, (float)(v - (double)h));
}
__device__ __forceinline__ double repro_value(const long long* bins) {
  double t = 0.0;
#pragma unroll
  for (int k = B2A_NBIN - 1; k >= 0; k--) t += (double)bins[k] * ldexp(1.0, B2A_BIN0 + B2A_BIN_BITS * k);
  return t;
}

// ---- programmatic dependent launch (PDL): a kernel launched with the attribute may start while its predecessor drains; it must
// not touch the predecessor's outputs (or write anything) before pdl_wait().  Everything independent of the predecessor --
// weight loads, L2 prefetches, address math -- goes before it.  Inside a CUDA graph the edges become programmatic dependencies.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool b2a_pdl_enabled();      // env B2A_PDL != "0" (api.cu)

template <typename... KArgs, typename... Args>
static inline cudaError_t b2a_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = b2a_pdl_enabled() ? 1 : 0;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}
