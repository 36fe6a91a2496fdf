#include "host_utils.h"

#include <stdarg.h>
#include <string.h>

#include <mutex>

namespace b200 {

static thread_local char g_err[1024] = {0};
unsigned long long g_launch_count = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

static int encode_tmap_any(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                           const uint64_t* strides_elems, const uint32_t* box, int elem_bytes, CUtensorMapDataType dt);

int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                     const uint32_t* box) {
  return encode_tmap_any(out, base, rank, dims, strides_elems, box, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
}
int encode_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                    const uint32_t* box) {
  return encode_tmap_any(out, base, rank, dims, strides_elems, box, 4, CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
}

static int encode_tmap_any(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                           const uint64_t* strides_elems, const uint32_t* box, int elem_bytes, CUtensorMapDataType dt) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return ECUDA_;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_elems[i] * elem_bytes;  // bytes
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("tensor map base %p not 16-byte aligned", base);
    return EINVAL_;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (gstr[i] % 16 != 0) {
      set_error("tensor map stride[%d]=%llu bytes not a multiple of 16", i + 1, (unsigned long long)gstr[i]);
      return EINVAL_;
    }
  }
  CUresult r = fn(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u]", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
              rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return ECUDA_;
  }
  return OK;
}

int device_sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

}  // namespace b200
