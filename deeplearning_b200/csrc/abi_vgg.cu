// C-ABI entry points of the VGG passes and the Adam update (see vgg.cuh).  Every entry validates its shapes and pointers
// before it launches anything.
#include <stdint.h>

#include "../../include/b200cls.h"
#include "vgg.cuh"
#include "host_utils.h"

using namespace b200;

namespace {
bool aligned16(const void* p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
bool opt16(const void* p) { return p == nullptr || aligned16(p); }
cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }

int ew_blocks(long long items) {
  long long blocks = (items + 255) / 256;
  const long long cap = static_cast<long long>(device_sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  return blocks < 1 ? 1 : static_cast<int>(blocks);
}

const char* pool_bad_shape(int B, int H, int W, int C) {
  if (B < 1 || B > 65535) return "B must be in [1, 65535]";
  if (H < 1 || W < 1) return "H and W must be >= 1";
  if (C < 8 || C % 8 != 0 || C > kRvMaxC) return "C must be a multiple of 8 in [8, 8192]";
  return nullptr;
}

long long pool_blocks(int B, int H, int W) { return static_cast<long long>(B) * ((H + 1) / 2) * ((W + 1) / 2); }
}  // namespace

#define VGG_REQUIRE_SHAPE(what, msg, B, H, W, C) \
  B200_REQUIRE((msg) == nullptr, what ": %s (B=%d H=%d W=%d C=%d)", (msg) ? (msg) : "", B, H, W, C)

extern "C" {

int b200_vgg_pool_partial_rows(int B, int H, int W, int C) {
  if (pool_bad_shape(B, H, W, C) != nullptr) return -1;
  return repvgg_geom(pool_blocks(B, H, W), C).blocks;
}

int b200_vgg_pool_fwd(const void* x, const float* scale, const float* shift, void* y, void* idx, int B, int H, int W, int C,
                      void* stream) {
  const char* bad = pool_bad_shape(B, H, W, C);
  if (bad == nullptr && (H < 2 || W < 2)) bad = "a 2x2 pool needs H, W >= 2";
  VGG_REQUIRE_SHAPE("vgg_pool_fwd", bad, B, H, W, C);
  B200_REQUIRE(aligned16(x) && aligned16(y) && (reinterpret_cast<uintptr_t>(idx) & 7) == 0,
               "vgg_pool_fwd: x and y must be non-null and 16-byte aligned, idx 8-byte aligned or NULL");
  B200_REQUIRE((scale == nullptr) == (shift == nullptr) && opt16(scale) && opt16(shift),
               "vgg_pool_fwd: scale and shift go together (16-byte aligned)");
  const int cvec = C / 8;
  const long long n = static_cast<long long>(B) * (H / 2) * (W / 2) * cvec;
  const auto* px = static_cast<const uint4*>(x);
  auto* py = static_cast<uint4*>(y);
  auto* pi = static_cast<uint2*>(idx);
  if (scale != nullptr)
    B200_CHECK_CUDA(launch_pdl(vgg_pool_fwd_kernel<true>, dim3(ew_blocks(n)), dim3(256), 0, as_stream(stream), px, scale,
                               shift, py, pi, B, H, W, cvec));
  else
    B200_CHECK_CUDA(launch_pdl(vgg_pool_fwd_kernel<false>, dim3(ew_blocks(n)), dim3(256), 0, as_stream(stream), px, scale,
                               shift, py, pi, B, H, W, cvec));
  B200_LAUNCHED();
  return OK;
}

int b200_vgg_pool_bwd(const void* g, const void* idx, const void* y, const void* c, const float* scale, const float* shift,
                      void* dx, float* partial, int B, int H, int W, int C, void* stream) {
  const char* bad = pool_bad_shape(B, H, W, C);
  if (bad == nullptr && (H < 2 || W < 2)) bad = "a 2x2 pool needs H, W >= 2";
  VGG_REQUIRE_SHAPE("vgg_pool_bwd", bad, B, H, W, C);
  B200_REQUIRE(aligned16(g) && aligned16(idx) && aligned16(dx), "vgg_pool_bwd: g, idx, dx must be non-null and 16-byte aligned");
  const bool bn = c != nullptr;
  B200_REQUIRE(bn ? (y == nullptr && aligned16(scale) && aligned16(shift) && partial != nullptr)
                  : (aligned16(y) && scale == nullptr && shift == nullptr && partial == nullptr),
               "vgg_pool_bwd: give either the pooled output y (plain) or c, scale, shift and partial (BatchNorm)");
  const RvGeom gm = repvgg_geom(pool_blocks(B, H, W), C);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* pg = static_cast<const uint4*>(g);
  const auto* pi = static_cast<const uint2*>(idx);
  const auto* py = static_cast<const uint4*>(y);
  const auto* pc = static_cast<const uint4*>(c);
  auto* pd = static_cast<uint4*>(dx);
  if (bn)
    B200_CHECK_CUDA(launch_pdl(vgg_pool_bwd_kernel<true>, grid, dim3(256), 0, as_stream(stream), pg, pi, py, pc, scale, shift,
                               pd, partial, B, H, W, C, gm.rows_per_block, gm.gpc));
  else
    B200_CHECK_CUDA(launch_pdl(vgg_pool_bwd_kernel<false>, grid, dim3(256), 0, as_stream(stream), pg, pi, py, pc, scale,
                               shift, pd, partial, B, H, W, C, gm.rows_per_block, gm.gpc));
  B200_LAUNCHED();
  return OK;
}

int b200_vgg_avgpool7_fwd(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  VGG_REQUIRE_SHAPE("vgg_avgpool7_fwd", pool_bad_shape(B, H, W, C), B, H, W, C);
  B200_REQUIRE(C % kVggPoolChans == 0, "vgg_avgpool7_fwd: C=%d must be a multiple of %d", C, kVggPoolChans);
  B200_REQUIRE(aligned16(x) && aligned16(y), "vgg_avgpool7_fwd: x and y must be non-null and 16-byte aligned");
  B200_CHECK_CUDA(launch_pdl(vgg_avgpool7_fwd_kernel, dim3(B, C / kVggPoolChans), dim3(256), 0, as_stream(stream),
                             static_cast<const uint4*>(x), static_cast<uint32_t*>(y), H, W, C));
  B200_LAUNCHED();
  return OK;
}

int b200_vgg_avgpool7_bwd(const void* gy, void* gx, int B, int H, int W, int C, void* stream) {
  VGG_REQUIRE_SHAPE("vgg_avgpool7_bwd", pool_bad_shape(B, H, W, C), B, H, W, C);
  B200_REQUIRE(C % kVggPoolChans == 0, "vgg_avgpool7_bwd: C=%d must be a multiple of %d", C, kVggPoolChans);
  B200_REQUIRE(aligned16(gy) && aligned16(gx), "vgg_avgpool7_bwd: gy and gx must be non-null and 16-byte aligned");
  B200_CHECK_CUDA(launch_pdl(vgg_avgpool7_bwd_kernel, dim3(B, C / kVggPoolChans), dim3(256), 0, as_stream(stream),
                             static_cast<const uint32_t*>(gy), static_cast<uint4*>(gx), H, W, C));
  B200_LAUNCHED();
  return OK;
}

int b200_vgg_dropout_fwd(const void* x, const float* mask, void* y, long long n, void* stream) {
  B200_REQUIRE(n >= 8 && n % 8 == 0, "vgg_dropout_fwd: n=%lld must be a positive multiple of 8", n);
  B200_REQUIRE(aligned16(x) && aligned16(mask) && aligned16(y), "vgg_dropout_fwd: x, mask, y must be non-null and 16-byte aligned");
  B200_CHECK_CUDA(launch_pdl(vgg_dropout_fwd_kernel, dim3(ew_blocks(n / 8)), dim3(256), 0, as_stream(stream),
                             static_cast<const uint4*>(x), mask, static_cast<uint4*>(y), n / 8));
  B200_LAUNCHED();
  return OK;
}

int b200_vgg_dropout_bwd(const void* g, const void* h, float scale, void* dx, long long n, void* stream) {
  B200_REQUIRE(n >= 8 && n % 8 == 0, "vgg_dropout_bwd: n=%lld must be a positive multiple of 8", n);
  B200_REQUIRE(aligned16(g) && aligned16(h) && aligned16(dx), "vgg_dropout_bwd: g, h, dx must be non-null and 16-byte aligned");
  B200_CHECK_CUDA(launch_pdl(vgg_dropout_bwd_kernel, dim3(ew_blocks(n / 8)), dim3(256), 0, as_stream(stream),
                             static_cast<const uint4*>(g), static_cast<const uint4*>(h), scale, static_cast<uint4*>(dx), n / 8));
  B200_LAUNCHED();
  return OK;
}

int b200_adam(float* p, const float* g, float* m, float* v, long long n, const float* hyper, float beta1, float beta2,
              float eps, float weight_decay, float gscale, const float* clip_coef, void* stream) {
  B200_REQUIRE(n >= 1 && p != nullptr && g != nullptr && m != nullptr && v != nullptr && hyper != nullptr,
               "adam: n must be >= 1 and p, g, m, v, hyper non-null");
  B200_CHECK_CUDA(launch_pdl(adam_kernel, dim3(ew_blocks(n)), dim3(256), 0, as_stream(stream), p, g, m, v, n, hyper, beta1,
                             beta2, eps, weight_decay, gscale, clip_coef));
  B200_LAUNCHED();
  return OK;
}

}  // extern "C"
