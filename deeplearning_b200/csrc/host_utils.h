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

// Blocks of a grid-stride pass over `items` work items: ceil(items / per_block), at least 1 and at most cap_mult blocks
// per SM. The fixed-order reductions sum per block, so their results depend on this count.
inline int capped_grid(long long items, int per_block = 256, int cap_mult = 16) {
  long long blocks = (items + per_block - 1) / per_block;
  const long long cap = static_cast<long long>(device_sm_count()) * cap_mult;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

inline bool aligned16(const void* p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline bool opt16(const void* p) { return p == nullptr || aligned16(p); }   // optional operand: NULL or 16-byte aligned
inline cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }

// B, H, W, C of an NHWC bf16 map that the row passes read 8 channels at a time (C <= kRvMaxC of row_passes.cuh);
// returns a message or nullptr
inline const char* nhwc_bad_shape(int B, int H, int W, int C) {
  if (B < 1 || B > 65535) return "B must be in [1, 65535]";
  if (H < 1 || W < 1) return "H and W must be >= 1";
  if (C < 8 || C % 8 != 0 || C > 8192) return "C must be a multiple of 8 in [8, 8192]";
  return nullptr;
}

// Number of kernels this library has launched (process-wide); see b200_launch_count().
extern unsigned long long g_launch_count;

// Launch with programmatic stream serialization (see common.cuh pdl_wait): the kernel may be scheduled while its
// predecessor in the stream drains; every kernel of the library waits for that predecessor (griddepcontrol.wait) before it
// touches global memory. Called only through B200_LAUNCH.
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

// B200_LAUNCH(kernel, grid, block, smem, stream, args...): every kernel launch of the library. Launches with launch_pdl,
// counts the kernel in g_launch_count and checks the launch; on failure the enclosing entry returns ECUDA_. (Variadic, so
// that a kernel's template argument list needs no parentheses.)
#define B200_LAUNCH(...)                                   \
  do {                                                     \
    B200_CHECK_CUDA(::b200::launch_pdl(__VA_ARGS__));      \
    ++::b200::g_launch_count;                              \
    B200_CHECK_CUDA(cudaPeekAtLastError());                \
  } while (0)

}  // namespace b200
