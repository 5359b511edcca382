// Error plumbing, device queries and the host-side launch helpers shared by every kernel family (include/b200audio.h, common.cuh).
#include "common.cuh"
#include "tc_common.cuh"
#include <stdlib.h>
#include <stdarg.h>
#include <mutex>
#include <unordered_map>

static thread_local char g_err[512] = "";

void b2a_set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}

extern "C" const char* b2a_last_error(void) { return g_err; }
extern "C" int32_t b2a_version(void) { return 100; }
extern "C" int32_t b2a_device_sm_count(void) {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  return n;
}

bool b2a_pdl_enabled() {
  static const bool on = [] { const char* e = getenv("B2A_PDL"); return !(e && e[0] == '0'); }();
  return on;
}

// A kernel's limit starts where the runtime puts it without an opt-in: 48 KB less the kernel's static shared memory, read once.  So a
// launch that fits under it makes no runtime call, and one that needs more is raised even when its size is just under 48 KB.
cudaError_t b2a_smem_optin(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::unordered_map<const void*, int> limit;
  std::lock_guard<std::mutex> lock(mu);
  auto it = limit.find(kernel);
  if (it == limit.end()) {
    cudaFuncAttributes fa;
    const cudaError_t e = cudaFuncGetAttributes(&fa, kernel);
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    it = limit.emplace(kernel, fa.maxDynamicSharedSizeBytes).first;
  }
  if (bytes <= it->second) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) { cudaGetLastError(); return e; }
  it->second = bytes;
  return cudaSuccess;
}

int b2a_tmap16(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box, bool f16) {
  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static const EncodeTiledFn encode = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    return cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess ? (EncodeTiledFn)fn : nullptr;
  }();
  if (!encode) return -1;
  cuuint64_t gd[3], gs[2]; cuuint32_t bx[3]; const cuuint32_t es[3] = {1, 1, 1};
  for (int i = 0; i < rank; i++) { gd[i] = dims[i]; bx[i] = box[i]; }
  for (int i = 0; i < rank - 1; i++) gs[i] = strides_bytes[i];
  const CUresult r = encode(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base),
                            gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}
