// C-ABI entry points of the squeeze-and-excitation tail (see se.cuh).  Every entry validates its shapes and pointers
// before it launches anything.
#include <stdint.h>

#include "../../include/b200cls.h"
#include "se.cuh"
#include "host_utils.h"

using namespace b200;

namespace {
constexpr int kSeMaxCr = 256;
constexpr int kSeMaxB = 65535;   // images travel in gridDim.y / gridDim.z

bool aligned16(const void* p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// B, HW, C of the streaming passes; returns a message or nullptr
const char* se_bad_shape(int B, int HW, int C) {
  if (B < 1 || B > kSeMaxB) return "B must be in [1, 65535]";
  if (HW < 1) return "HW must be >= 1";
  if (C < 64 || C % 64 != 0) return "C must be a positive multiple of 64";
  return nullptr;
}
const char* se_bad_width(int Cr) { return (Cr < 1 || Cr > kSeMaxCr) ? "Cr must be in [1, 256]" : nullptr; }
}  // namespace

#define SE_REQUIRE_SHAPE(what, msg, ...)                                                                      \
  B200_REQUIRE((msg) == nullptr, what ": %s (B=%d HW=%d C=%d Cr=%d)", (msg) ? (msg) : "", __VA_ARGS__)

extern "C" {

int b200_se_squeeze(const void* c, const float* scale, const float* shift, float* csum, float* pool, int B, int HW, int C,
                    void* stream) {
  const char* bad = se_bad_shape(B, HW, C);
  SE_REQUIRE_SHAPE("se_squeeze", bad, B, HW, C, 0);
  B200_REQUIRE(aligned16(c) && aligned16(scale) && aligned16(shift) && csum != nullptr && pool != nullptr,
               "se_squeeze: c, scale, shift must be 16-byte aligned and csum, pool non-null");
  B200_CHECK_CUDA(launch_pdl(se_squeeze_kernel, dim3(C / 64, B), dim3(256), 0, static_cast<cudaStream_t>(stream),
      static_cast<const uint4*>(c), scale, shift, csum, pool, HW, C / 8));
  B200_LAUNCHED();
  return OK;
}

int b200_se_excite(const float* pool, const float* w1, const float* w2, float* h, float* gate, int B, int C, int Cr,
                   void* stream) {
  const char* bad = se_bad_shape(B, 1, C);
  if (bad == nullptr) bad = se_bad_width(Cr);
  SE_REQUIRE_SHAPE("se_excite", bad, B, 1, C, Cr);
  B200_REQUIRE(aligned16(pool) && aligned16(w1) && w2 != nullptr && h != nullptr && gate != nullptr,
               "se_excite: pool, w1 must be 16-byte aligned and w2, h, gate non-null");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  B200_CHECK_CUDA(launch_pdl(se_fc1_kernel, dim3((Cr + 7) / 8, (B + 7) / 8), dim3(256), 0, st, pool, w1, h, B, C, Cr));
  B200_LAUNCHED();
  const size_t smem = static_cast<size_t>(32 * (Cr + 1) + 8 * Cr) * sizeof(float);   // <= 41 KB at Cr = 256
  B200_CHECK_CUDA(launch_pdl(se_fc2_kernel, dim3(C / 32, (B + 7) / 8), dim3(256), smem, st, static_cast<const float*>(h), w2,
      gate, B, C, Cr));
  B200_LAUNCHED();
  return OK;
}

int b200_se_apply(const void* c, const void* identity, void* y, const float* scale, const float* shift, const float* gate,
                  int B, int HW, int C, void* stream) {
  const char* bad = se_bad_shape(B, HW, C);
  SE_REQUIRE_SHAPE("se_apply", bad, B, HW, C, 0);
  B200_REQUIRE(aligned16(c) && aligned16(identity) && aligned16(y) && aligned16(scale) && aligned16(shift) && aligned16(gate),
               "se_apply: c, identity, y, scale, shift, gate must be non-null and 16-byte aligned");
  B200_CHECK_CUDA(launch_pdl(se_apply_kernel, dim3((HW + kSeApplyRows - 1) / kSeApplyRows, C / 64, B), dim3(256), 0,
      static_cast<cudaStream_t>(stream), static_cast<const uint4*>(c), static_cast<const uint4*>(identity),
      static_cast<uint4*>(y), scale, shift, gate, HW, C / 8));
  B200_LAUNCHED();
  return OK;
}

int b200_se_bwd_reduce(const void* g, const void* y, const void* c, void* dz, float* A, float* R, int B, int HW, int C,
                       void* stream) {
  const char* bad = se_bad_shape(B, HW, C);
  SE_REQUIRE_SHAPE("se_bwd_reduce", bad, B, HW, C, 0);
  B200_REQUIRE(aligned16(g) && aligned16(y) && aligned16(c) && aligned16(dz) && A != nullptr && R != nullptr,
               "se_bwd_reduce: g, y, c, dz must be 16-byte aligned and A, R non-null");
  B200_CHECK_CUDA(launch_pdl(se_bwd_reduce_kernel, dim3(C / 64, B), dim3(256), 0, static_cast<cudaStream_t>(stream),
      static_cast<const uint4*>(g), static_cast<const uint4*>(y), static_cast<const uint4*>(c), static_cast<uint4*>(dz), A, R,
      HW, C / 8));
  B200_LAUNCHED();
  return OK;
}

int b200_se_bwd_coeffs(const float* A, const float* R, const float* csum, const float* pool, const float* h,
                       const float* gate, const float* w1, const float* w2, const float* scale, const float* shift,
                       const float* mean, const float* invstd, int B, int HW, int C, int Cr, float* dh, float* dp,
                       float* dw1, float* dw2, float* dgamma, float* dbeta, float* m1, float* m2, void* stream) {
  const char* bad = se_bad_shape(B, HW, C);
  if (bad == nullptr) bad = se_bad_width(Cr);
  SE_REQUIRE_SHAPE("se_bwd_coeffs", bad, B, HW, C, Cr);
  const void* need[] = {A, R, csum, pool, h, gate, w1, w2, scale, shift, mean, invstd, dh, dp, dw1, dw2, dgamma, dbeta, m1, m2};
  for (const void* p : need) B200_REQUIRE(p != nullptr, "se_bwd_coeffs: every pointer argument is required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nj = (Cr + 31) / 32;
  const int blocks = nj * ((B + 7) / 8) + nj * (C / 32);
  B200_CHECK_CUDA(launch_pdl(se_bwd_gate_kernel, dim3(blocks), dim3(256), 0, st, A, R, gate, h, w2, scale, shift, dh, dw2, B, C,
      Cr));
  B200_LAUNCHED();
  static bool configured = false;   // w1 columns + a chunk of dh rows: up to 64 KB at Cr = 256
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(se_bwd_bn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (32 + kSeDhRows) * kSeMaxCr * static_cast<int>(sizeof(float))));
    configured = true;
  }
  B200_CHECK_CUDA(launch_pdl(se_bwd_bn_kernel, dim3(C / 32, 1 + (Cr + 7) / 8), dim3(256),
      static_cast<size_t>(32 + kSeDhRows) * Cr * sizeof(float), st, A, R, csum, pool, gate, static_cast<const float*>(dh), w1,
      mean, invstd, dp, dw1, dgamma, dbeta, m1, m2, B, HW, C, Cr));
  B200_LAUNCHED();
  return OK;
}

int b200_se_bwd_apply(const void* dz, const void* c, void* dc, const float* gate, const float* dp, const float* scale,
                      const float* mean, const float* invstd, const float* m1, const float* m2, int B, int HW, int C,
                      void* stream) {
  const char* bad = se_bad_shape(B, HW, C);
  SE_REQUIRE_SHAPE("se_bwd_apply", bad, B, HW, C, 0);
  B200_REQUIRE(aligned16(dz) && aligned16(c) && aligned16(dc) && aligned16(gate) && aligned16(dp) && aligned16(scale) &&
                   aligned16(mean) && aligned16(invstd) && aligned16(m1) && aligned16(m2),
               "se_bwd_apply: every pointer must be non-null and 16-byte aligned");
  B200_CHECK_CUDA(launch_pdl(se_bwd_apply_kernel, dim3((HW + kSeApplyRows - 1) / kSeApplyRows, C / 64, B), dim3(256), 0,
      static_cast<cudaStream_t>(stream), static_cast<const uint4*>(dz), static_cast<const uint4*>(c), static_cast<uint4*>(dc),
      gate, dp, scale, mean, invstd, m1, m2, HW, C / 8));
  B200_LAUNCHED();
  return OK;
}

}  // extern "C"
