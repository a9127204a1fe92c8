// Library-level plumbing: version, thread-local error text, tensor-map encoding
// through a run-time resolved driver entry point (no link-time libcuda
// dependency, so the .so loads on a CPU-only box for the symbol tests).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "common.cuh"

namespace osvos {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, int elem_bytes, int rank, const void* base,
                      const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled is not available (no CUDA driver?)");
    return OSVOS_ERR_CUDA;
  }
  cuuint64_t gdims[5];
  cuuint64_t gstrides[4];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstrides[i - 1] = strides_bytes[i - 1];
  }
  (void)elem_bytes;
  CUresult r = fn(map, dtype, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdims, gstrides, gbox, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dims %llu %llu %llu %llu, box %u %u %u %u)",
                   (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
                   (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
                   box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return OSVOS_ERR_CUDA;
  }
  return OSVOS_OK;
}

int device_sm_count() {
  static int sms[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (sms[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    sms[dev] = v;
  }
  return sms[dev];
}

// Programmatic dependent launch: process default from OSVOS_PDL (read once), overridden per call sequence by
// osvos_set_pdl() - the engine switches it on around the inference pass.  A captured graph keeps the attribute its launches were captured with.
static int g_pdl_override = -1;   // -1: environment default
bool pdl_enabled() {
  if (g_pdl_override >= 0) return g_pdl_override == 1;
  static int state = -1;
  if (state < 0) {
    const char* e = getenv("OSVOS_PDL");
    state = (e != nullptr && atoi(e) != 0) ? 1 : 0;
  }
  return state == 1;
}

}  // namespace osvos

extern "C" int osvos_version(void) { return OSVOS_B200_VERSION; }
extern "C" int osvos_set_pdl(int mode) {
  const int prev = osvos::g_pdl_override;
  osvos::g_pdl_override = mode < 0 ? -1 : (mode != 0 ? 1 : 0);
  return prev;
}
extern "C" const char* osvos_last_error(void) { return osvos::g_err; }
