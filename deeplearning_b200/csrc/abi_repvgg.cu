// C-ABI entry points of the RepVGG block passes (see repvgg.cuh).  Every entry validates its shapes and pointers before it
// launches anything.
#include <stdint.h>

#include "../../include/b200cls.h"
#include "repvgg.cuh"
#include "host_utils.h"

using namespace b200;

namespace {
// rows, C and the row pitches (in elements) of the pitched operands; returns a message or nullptr
const char* rv_bad_shape(long long rows, int C) {
  if (rows < 1) return "rows must be >= 1";
  if (C < 8 || C % 8 != 0 || C > kRvMaxC) return "C must be a multiple of 8 in [8, 8192]";
  return nullptr;
}
const char* rv_bad_pitch(long long ld, int C) {
  return (ld < C || ld % 8 != 0) ? "row pitches must be multiples of 8 and >= C" : nullptr;
}
}  // namespace

#define RV_REQUIRE_SHAPE(what, msg, rows, C)                                                                   \
  B200_REQUIRE((msg) == nullptr, what ": %s (rows=%lld C=%d)", (msg) ? (msg) : "", static_cast<long long>(rows), C)

extern "C" {

int b200_repvgg_partial_rows(long long rows, int C) {
  const char* bad = rv_bad_shape(rows, C);
  if (bad != nullptr) {
    set_error("repvgg_partial_rows: %s (rows=%lld C=%d)", bad, rows, C);
    return -1;
  }
  return repvgg_geom(rows, C).blocks;
}

int b200_repvgg_apply(const void* c3, long long ld3, const void* c1, long long ld1, const void* x, long long ldx,
                      const float* co3, const float* co1, const float* co_id, void* y, long long rows, int C, float* stats,
                      void* stream) {
  const char* bad = rv_bad_shape(rows, C);
  if (bad == nullptr) bad = rv_bad_pitch(ld3, C);
  if (bad == nullptr) bad = rv_bad_pitch(ld1, C);
  if (bad == nullptr && x != nullptr) bad = rv_bad_pitch(ldx, C);
  RV_REQUIRE_SHAPE("repvgg_apply", bad, rows, C);
  const bool id = x != nullptr;
  B200_REQUIRE(aligned16(c3) && aligned16(c1) && aligned16(co3) && aligned16(co1) && aligned16(y),
               "repvgg_apply: c3, c1, co3, co1, y must be non-null and 16-byte aligned");
  B200_REQUIRE(id == (co_id != nullptr) && (!id || (aligned16(x) && aligned16(co_id))),
               "repvgg_apply: the identity branch needs both x and co_id, 16-byte aligned");
  const RvGeom gm = repvgg_geom(rows, C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* p3 = static_cast<const __nv_bfloat16*>(c3);
  const auto* p1 = static_cast<const __nv_bfloat16*>(c1);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  uint4* py = static_cast<uint4*>(y);
  if (id && stats)
    B200_LAUNCH(repvgg_apply_kernel<true, true>, grid, dim3(256), 0, st, p3, ld3, p1, ld1, px, ldx, co3, co1,
                co_id, py, rows, C, gm.rows_per_block, gm.gpc, stats);
  else if (id)
    B200_LAUNCH(repvgg_apply_kernel<true, false>, grid, dim3(256), 0, st, p3, ld3, p1, ld1, px, ldx, co3, co1,
                co_id, py, rows, C, gm.rows_per_block, gm.gpc, stats);
  else if (stats)
    B200_LAUNCH(repvgg_apply_kernel<false, true>, grid, dim3(256), 0, st, p3, ld3, p1, ld1, px, ldx, co3, co1,
                co_id, py, rows, C, gm.rows_per_block, gm.gpc, stats);
  else
    B200_LAUNCH(repvgg_apply_kernel<false, false>, grid, dim3(256), 0, st, p3, ld3, p1, ld1, px, ldx, co3,
                co1, co_id, py, rows, C, gm.rows_per_block, gm.gpc, stats);
  return OK;
}

int b200_repvgg_bwd_reduce(const void* g, const void* y, const void* c3, long long ld3, const void* c1, long long ld1,
                           const void* x, long long ldx, long long rows, int C, float* partial, void* stream) {
  const char* bad = rv_bad_shape(rows, C);
  if (bad == nullptr) bad = rv_bad_pitch(ld3, C);
  if (bad == nullptr) bad = rv_bad_pitch(ld1, C);
  if (bad == nullptr && x != nullptr) bad = rv_bad_pitch(ldx, C);
  RV_REQUIRE_SHAPE("repvgg_bwd_reduce", bad, rows, C);
  B200_REQUIRE(aligned16(g) && aligned16(y) && aligned16(c3) && aligned16(c1) && partial != nullptr &&
                   (x == nullptr || aligned16(x)),
               "repvgg_bwd_reduce: g, y, c3, c1 (and x) must be non-null and 16-byte aligned, partial non-null");
  const RvGeom gm = repvgg_geom(rows, C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* pg = static_cast<const uint4*>(g);
  const auto* py = static_cast<const uint4*>(y);
  const auto* p3 = static_cast<const __nv_bfloat16*>(c3);
  const auto* p1 = static_cast<const __nv_bfloat16*>(c1);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  if (x != nullptr)
    B200_LAUNCH(repvgg_bwd_reduce_kernel<true>, grid, dim3(256), 0, st, pg, py, p3, ld3, p1, ld1, px, ldx, rows,
                C, gm.rows_per_block, gm.gpc, partial);
  else
    B200_LAUNCH(repvgg_bwd_reduce_kernel<false>, grid, dim3(256), 0, st, pg, py, p3, ld3, p1, ld1, px, ldx,
                rows, C, gm.rows_per_block, gm.gpc, partial);
  return OK;
}

int b200_repvgg_bwd_apply(const void* g, const void* y, const void* c3, long long ld3, const void* c1, long long ld1,
                          const void* x, long long ldx, const float* co3, const float* m3, const float* co1, const float* m1,
                          const float* co_id, const float* m_id, void* dc3, void* dc1, void* dx, long long rows, int C,
                          void* stream) {
  const char* bad = rv_bad_shape(rows, C);
  if (bad == nullptr) bad = rv_bad_pitch(ld3, C);
  if (bad == nullptr) bad = rv_bad_pitch(ld1, C);
  if (bad == nullptr && x != nullptr) bad = rv_bad_pitch(ldx, C);
  RV_REQUIRE_SHAPE("repvgg_bwd_apply", bad, rows, C);
  const bool id = x != nullptr;
  B200_REQUIRE(aligned16(g) && aligned16(y) && aligned16(c3) && aligned16(c1) && aligned16(co3) && aligned16(m3) &&
                   aligned16(co1) && aligned16(m1) && aligned16(dc3) && aligned16(dc1),
               "repvgg_bwd_apply: g, y, c3, c1, co3, m3, co1, m1, dc3, dc1 must be non-null and 16-byte aligned");
  B200_REQUIRE(!id || (aligned16(x) && aligned16(co_id) && aligned16(m_id) && aligned16(dx)),
               "repvgg_bwd_apply: the identity branch needs x, co_id, m_id and dx, 16-byte aligned");
  const RvGeom gm = repvgg_geom(rows, C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* pg = static_cast<const uint4*>(g);
  const auto* py = static_cast<const uint4*>(y);
  const auto* p3 = static_cast<const __nv_bfloat16*>(c3);
  const auto* p1 = static_cast<const __nv_bfloat16*>(c1);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  auto* d3 = static_cast<__nv_bfloat16*>(dc3);
  auto* d1 = static_cast<__nv_bfloat16*>(dc1);
  auto* dd = static_cast<__nv_bfloat16*>(dx);
  if (id)
    B200_LAUNCH(repvgg_bwd_apply_kernel<true>, grid, dim3(256), 0, st, pg, py, p3, ld3, p1, ld1, px, ldx, co3,
                m3, co1, m1, co_id, m_id, d3, d1, dd, rows, C, gm.rows_per_block, gm.gpc);
  else
    B200_LAUNCH(repvgg_bwd_apply_kernel<false>, grid, dim3(256), 0, st, pg, py, p3, ld3, p1, ld1, px, ldx, co3,
                m3, co1, m1, co_id, m_id, d3, d1, dd, rows, C, gm.rows_per_block, gm.gpc);
  return OK;
}

int b200_repvgg_fold(const float* w3, const float* w1, const float* gamma3, const float* beta3, const float* mean3,
                     const float* var3, float eps3, const float* gamma1, const float* beta1, const float* mean1,
                     const float* var1, float eps1, const float* gamma_id, const float* beta_id, const float* mean_id,
                     const float* var_id, float eps_id, int O, int I, int ldk, void* wp, float* bias, void* stream) {
  B200_REQUIRE(O >= 8 && O % 8 == 0 && O <= kRvMaxC && I >= 1 && ldk % 8 == 0 && ldk >= 9 * I,
               "repvgg_fold: need O a multiple of 8 in [8, 8192], I >= 1, ldk a multiple of 8 and >= 9*I (O=%d I=%d ldk=%d)",
               O, I, ldk);
  const void* need[] = {w3, w1, gamma3, beta3, mean3, var3, gamma1, beta1, mean1, var1, wp, bias};
  for (const void* p : need) B200_REQUIRE(p != nullptr, "repvgg_fold: w3, w1, both branch BatchNorms, wp and bias are required");
  const bool id = gamma_id != nullptr;
  B200_REQUIRE(id == (beta_id != nullptr) && id == (mean_id != nullptr) && id == (var_id != nullptr),
               "repvgg_fold: the identity BatchNorm needs all of gamma, beta, mean, var, or none");
  B200_REQUIRE(!id || O == I, "repvgg_fold: an identity branch needs O == I (O=%d I=%d)", O, I);
  const RvFoldBn b3{gamma3, beta3, mean3, var3, eps3}, b1{gamma1, beta1, mean1, var1, eps1};
  const RvFoldBn bi{gamma_id, beta_id, mean_id, var_id, eps_id};
  long long blocks = (static_cast<long long>(O) * ldk + 255) / 256;
  if (blocks > 4 * kNumSMs * 8) blocks = 4 * kNumSMs * 8;
  B200_LAUNCH(repvgg_fold_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0,
              static_cast<cudaStream_t>(stream), w3, w1, b3, b1, bi, O, I, ldk,
              static_cast<__nv_bfloat16*>(wp), bias);
  return OK;
}

}  // extern "C"
