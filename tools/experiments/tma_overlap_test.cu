// Does cuTensorMapEncodeTiled accept OVERLAPPING rows (stride[1] < dim[0] * elemsize) and does the TMA load them correctly?
// (Needed for a space-to-depth ResNet stem: 4 x-taps x 16 ch = 64 contiguous elements per pixel, pixel stride 16 elements.)
// nvcc -gencode arch=compute_90a,code=sm_90a -o tma_overlap_test tma_overlap_test.cu -lcuda
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>

__global__ void k(const __grid_constant__ CUtensorMap map, __nv_bfloat16* out, int x0, int y0) {
  __shared__ __align__(1024) __nv_bfloat16 tile[8 * 64];   // box: 64 elems x 8 rows (x) x 1 (y)
  __shared__ uint64_t bar;
  if (threadIdx.x == 0) {
    uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b));
    asm volatile("fence.mbarrier_init.release.cluster;");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(8 * 64 * 2));
    uint32_t d = (uint32_t)__cvta_generic_to_shared(tile);
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(d),
                 "l"(&map), "r"(b), "r"(0), "r"(x0), "r"(y0)
                 : "memory");
    uint32_t ok = 0;
    while (!ok) asm volatile("{.reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p;}" : "=r"(ok) : "r"(b));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 8 * 64; i += blockDim.x) out[i] = tile[i];
}

int main() {
  const int W = 40, H = 6, C = 16;   // pixels of 16 channels; a "row" = 4 pixels = 64 elements, rows start every pixel
  std::vector<__nv_bfloat16> h(W * H * C);
  for (int i = 0; i < W * H * C; ++i) h[i] = __float2bfloat16((float)(i % 2039));
  __nv_bfloat16 *d, *o;
  cudaMalloc(&d, h.size() * 2);
  cudaMalloc(&o, 8 * 64 * 2);
  cudaMemcpy(d, h.data(), h.size() * 2, cudaMemcpyHostToDevice);
  typedef CUresult (*Fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                         const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fp = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q);
  CUtensorMap map;
  cuuint64_t dims[3] = {64, (cuuint64_t)(W - 3), (cuuint64_t)H};
  cuuint64_t strides[2] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2};   // 32 B between overlapping rows, image row pitch
  cuuint32_t box[3] = {64, 8, 1}, es[3] = {1, 1, 1};
  CUresult r = ((Fn)fp)(&map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  printf("encode (overlapping stride 32 B < 128 B row): CUresult = %d\n", (int)r);
  if (r != CUDA_SUCCESS) return 0;
  k<<<1, 128>>>(map, o, 5, 2);
  cudaError_t e = cudaDeviceSynchronize();
  printf("kernel: %s\n", cudaGetErrorString(e));
  std::vector<__nv_bfloat16> got(8 * 64);
  cudaMemcpy(got.data(), o, got.size() * 2, cudaMemcpyDeviceToHost);
  int bad = 0;
  for (int r8 = 0; r8 < 8; ++r8)
    for (int c = 0; c < 64; ++c) {
      const int src = (2 * W + (5 + r8)) * C + c;   // y = 2, x = 5 + r8, then 64 contiguous elements
      if (__bfloat162float(got[r8 * 64 + c]) != __bfloat162float(h[src])) ++bad;
    }
  printf("mismatches: %d of 512\n", bad);
  return 0;
}
