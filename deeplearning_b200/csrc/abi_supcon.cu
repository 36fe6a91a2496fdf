// C-ABI entry points of the supervised contrastive learning passes (see supcon.cuh).  Every entry validates its shapes and
// pointers before it launches anything.
#include <math.h>
#include <stdint.h>

#include "../../include/b200cls.h"
#include "host_utils.h"
#include "supcon.cuh"

using namespace b200;

namespace {
int row_blocks(int N, int rows_per_block) { return (N + rows_per_block - 1) / rows_per_block; }
}  // namespace

#define SUPCON_REQUIRE_ROWS(what, N, D, maxD)                                                                     \
  B200_REQUIRE((N) >= 1 && (D) >= 4 && (D) <= (maxD) && (D) % 4 == 0 && static_cast<long long>(N) * (D) < (1ll << 31),     \
               what ": N must be >= 1 and D a multiple of 4 in [4, %d], N * D below 2^31 (N=%d D=%d)", maxD, N, D)

extern "C" {

int b200_supcon_max_dim(void) { return kSupconMaxD; }

int b200_supcon_normalize_fwd(const float* z, float* e, float* nrm, int N, int D, void* stream) {
  SUPCON_REQUIRE_ROWS("supcon_normalize_fwd", N, D, 1 << 16);
  B200_REQUIRE(z != nullptr && e != nullptr && nrm != nullptr, "supcon_normalize_fwd: z, e, nrm must be non-null");
  B200_LAUNCH(supcon_normalize_fwd_kernel, dim3(row_blocks(N, 8)), dim3(256), 0, as_stream(stream), z, N, D,
              e, nrm);
  return OK;
}

int b200_supcon_normalize_bwd(const float* de, const float* e, const float* nrm, void* dz, int N, int D, void* stream) {
  SUPCON_REQUIRE_ROWS("supcon_normalize_bwd", N, D, 1 << 16);
  B200_REQUIRE(de != nullptr && e != nullptr && nrm != nullptr && dz != nullptr,
               "supcon_normalize_bwd: de, e, nrm, dz must be non-null");
  B200_LAUNCH(supcon_normalize_bwd_kernel, dim3(row_blocks(N, 8)), dim3(256), 0, as_stream(stream), de, e,
              nrm, N, D, static_cast<__nv_bfloat16*>(dz));
  return OK;
}

int b200_supcon_loss_fwd(const float* e, const int* labels, int N, int D, float temperature, float base_temperature,
                         float* L, float* npos, float* row_loss, float* loss, void* stream) {
  SUPCON_REQUIRE_ROWS("supcon_loss_fwd", N, D, kSupconMaxD);
  B200_REQUIRE(temperature > 0.f && isfinite(temperature) && base_temperature > 0.f && isfinite(base_temperature),
               "supcon_loss_fwd: temperature and base_temperature must be finite and > 0 (%g, %g)", temperature,
               base_temperature);
  B200_REQUIRE(e != nullptr && labels != nullptr && L != nullptr && npos != nullptr && row_loss != nullptr && loss != nullptr,
               "supcon_loss_fwd: e, labels, L, npos, row_loss, loss must be non-null");
  B200_LAUNCH(supcon_loss_fwd_kernel, dim3(row_blocks(N, kSupconBM)), dim3(256), 0, as_stream(stream), e,
              labels, N, D, 1.0f / temperature, temperature / base_temperature, L, npos, row_loss);
  B200_LAUNCH(supcon_mean_kernel, dim3(1), dim3(256), 0, as_stream(stream), static_cast<const float*>(row_loss),
              N, loss);
  return OK;
}

int b200_supcon_loss_bwd(const float* e, const int* labels, const float* L, const float* npos, const float* grad_out,
                         float grad_scale, int N, int D, float temperature, float base_temperature, float* de, void* stream) {
  SUPCON_REQUIRE_ROWS("supcon_loss_bwd", N, D, kSupconMaxD);
  B200_REQUIRE(temperature > 0.f && isfinite(temperature) && base_temperature > 0.f && isfinite(base_temperature),
               "supcon_loss_bwd: temperature and base_temperature must be finite and > 0 (%g, %g)", temperature,
               base_temperature);
  B200_REQUIRE(isfinite(grad_scale), "supcon_loss_bwd: grad_scale must be finite (%g)", grad_scale);
  B200_REQUIRE(e != nullptr && labels != nullptr && L != nullptr && npos != nullptr && grad_out != nullptr && de != nullptr,
               "supcon_loss_bwd: e, labels, L, npos, grad_out, de must be non-null");
  static bool configured = false;
  if (!configured) {   // the widest accumulator, once: attribute calls stay out of graph captures
    B200_CHECK_CUDA(cudaFuncSetAttribute(supcon_loss_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kSupconBM * kSupconMaxD * static_cast<int>(sizeof(float))));
    configured = true;
  }
  const size_t smem = static_cast<size_t>(kSupconBM) * D * sizeof(float);
  // dloss / de_i = (1 / tau) sum_j (G_ij + G_ji) e_j with G_ij = g (tau / base_tau) / N (softmax_ij - [j in P_i] / |P_i|)
  const float c = grad_scale * (temperature / base_temperature) / static_cast<float>(N) / temperature;
  B200_LAUNCH(supcon_loss_bwd_kernel, dim3(row_blocks(N, kSupconBM)), dim3(256), smem, as_stream(stream), e,
              labels, L, npos, grad_out, c, N, D, 1.0f / temperature, de);
  return OK;
}

int b200_supcon_relu_bwd(const void* dy, const void* y, void* dx, long long n, void* stream) {
  B200_REQUIRE(n >= 1 && n <= (1ll << 40), "supcon_relu_bwd: n must be in [1, 2^40] (n=%lld)", n);
  B200_REQUIRE(dy != nullptr && y != nullptr && dx != nullptr, "supcon_relu_bwd: dy, y, dx must be non-null");
  B200_LAUNCH(supcon_relu_bwd_kernel, dim3(capped_grid(n)), dim3(256), 0, as_stream(stream),
              static_cast<const __nv_bfloat16*>(dy), static_cast<const __nv_bfloat16*>(y), n,
              static_cast<__nv_bfloat16*>(dx));
  return OK;
}

}  // extern "C"
