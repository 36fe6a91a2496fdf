// Host-side helpers shared by the C-ABI translation units: error convention, TMA descriptor encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace b200 {

// Thread-local last-error text, read through b200_last_error().
void set_error(const char* fmt, ...);
const char* get_error();

// Error codes of the C ABI (negative = failure).
enum : int { OK = 0, EINVAL_ = -1, EUNSUPPORTED_ = -2, ECUDA_ = -3 };

#define B200_CHECK_CUDA(expr)                                                                      \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      ::b200::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return ::b200::ECUDA_;                                                                       \
    }                                                                                              \
  } while (0)

#define B200_REQUIRE(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      ::b200::set_error(__VA_ARGS__);      \
      return ::b200::EINVAL_;              \
    }                                      \
  } while (0)

// Encode a bf16 tiled tensor map of rank 2..4 with 128B swizzle. dims/strides are in elements
// (innermost first, stride[0] == 1 implied); box in elements. Returns 0 on success.
int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                     const uint32_t* box);
// Same for fp32 tensors (4-byte elements; a 128B-swizzled box holds at most 32 of them in the innermost dimension).
int encode_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                    const uint32_t* box);

int device_sm_count();

// Number of kernels this library has launched (process-wide); see b200_launch_count().
extern unsigned long long g_launch_count;

#define B200_LAUNCHED()                                   \
  do {                                                    \
    ++::b200::g_launch_count;                             \
    B200_CHECK_CUDA(cudaPeekAtLastError());               \
  } while (0)

// Launch with programmatic stream serialization (see common.cuh pdl_wait): the kernel may be scheduled while its
// predecessor in the stream drains; every kernel of the library waits for that predecessor (griddepcontrol.wait) before it
// touches global memory.
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace b200
