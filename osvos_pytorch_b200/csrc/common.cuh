// Shared host/device helpers for libosvos_b200: status codes, the driver entry
// point for cuTensorMapEncodeTiled (resolved at run time so the library loads on
// a box without libcuda), split-bf16 arithmetic.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/osvos_b200.h"

namespace osvos {

#define OSVOS_CHECK_ARG(cond)                                                              \
  do {                                                                                     \
    if (!(cond)) {                                                                         \
      set_last_error("%s:%d: invalid argument: %s", __FILE__, __LINE__, #cond);            \
      return OSVOS_ERR_INVALID_ARGUMENT;                                                   \
    }                                                                                      \
  } while (0)

#define OSVOS_CHECK_CUDA(expr)                                                             \
  do {                                                                                     \
    cudaError_t e__ = (expr);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__)); \
      return OSVOS_ERR_CUDA;                                                               \
    }                                                                                      \
  } while (0)

void set_last_error(const char* fmt, ...);

// Encodes a tiled tensor map over a bf16 / fp32 tensor. dims/strides innermost first;
// strides[0] is implied by the element size. Returns an OSVOS_* status.
int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, int elem_bytes, int rank, const void* base,
                      const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      CUtensorMapSwizzle swizzle);

int device_sm_count();

// Programmatic dependent launch: opt-in with OSVOS_PDL=1 (read once per process); otherwise plain stream-ordered
// launches.
bool pdl_enabled();

// Launches `kern` on `stream`; with PDL enabled the launch carries the programmatic-stream-serialization attribute,
// so the kernel's prologue (barrier init, descriptor prefetch) overlaps the previous kernel's tail.
// ONLY for kernels that execute pdl_wait() (ptx.cuh) before their first dependent global access.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// Opt-in to > 48 KiB of dynamic shared memory, once per (kernel instantiation, DEVICE): the attribute is per device, and
// the engine supports modules on any GPU of the process.  `done_mask` is the call site's static bit mask of devices.
template <typename K>
static inline cudaError_t ensure_dynamic_smem(K kern, int bytes, uint64_t* done_mask) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 64 && ((*done_mask >> dev) & 1ull)) return cudaSuccess;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && dev < 64) *done_mask |= 1ull << dev;
  return e;
}

// ---- split-bf16 ("bf16x2") representation of an fp32 value: v ~= hi + lo ------
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
}
// Grid-wide "last block finalizes" pattern: true in exactly one block, the last one to arrive, after every other
// block's prior global writes / atomics have become visible.  `counter` must be zero at launch.
__device__ __forceinline__ bool last_block_arrives(unsigned int* counter) {
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(counter, 1u) == gridDim.x * gridDim.y - 1;
  __syncthreads();
  if (is_last) __threadfence();
  return is_last;
}

// Fixed-order sum of rows[0..nrows)[col] * stride by one whole block (blockDim.x a multiple of 32, <= 1024): thread t
// adds rows t, t + blockDim.x, ... in order, the block's partials are then added in thread order by thread 0.  The order
// depends on nrows and blockDim.x only.  Every thread must call it; the result is valid in thread 0.
template <typename T>
__device__ __forceinline__ T block_ordered_sum(const T* rows, int nrows, size_t stride, T* red /* [blockDim.x] shared */) {
  T t = T(0);
  for (int r = threadIdx.x; r < nrows; r += blockDim.x) t += __ldcg(rows + static_cast<size_t>(r) * stride);
  __syncthreads();   // `red` may still be read by a previous call
  red[threadIdx.x] = t;
  __syncthreads();
  T s = T(0);
  if (threadIdx.x == 0)
    for (int i = 0; i < static_cast<int>(blockDim.x); ++i) s += red[i];
  return s;
}

__device__ __forceinline__ float bf16_lo_to_float(uint32_t packed) { return __uint_as_float(packed << 16); }
__device__ __forceinline__ float bf16_hi_to_float(uint32_t packed) { return __uint_as_float(packed & 0xFFFF0000u); }

}  // namespace osvos
