// C-ABI entry points of the ShuffleNet v1 and v2 block tails (see shufflenet.cuh; the ReLU-on-load depthwise entries live
// with the other depthwise entries in abi_mbconv.cu).  Every entry validates its shapes and pointers before it launches anything.
#include <stdint.h>

#include "../../include/b200cls.h"
#include "shufflenet.cuh"
#include "host_utils.h"

using namespace b200;

namespace {
int pool_out(int n) { return (n - 1) / 2 + 1; }   // output extent of a 3x3 / stride 2 / pad 1 window

int pad8(int n) { return (n + 7) / 8 * 8; }

// ShuffleNet v2 tails: branch width b (even), half pitch bp, joined pitch pad8(2 b)
const char* v2_bad_widths(long long rows, int b, int bp) {
  if (rows < 1 || rows > (1ll << 40)) return "rows must be in [1, 2^40]";
  if (b < 2 || b % 2 != 0) return "b must be even and >= 2";
  if (bp < b || bp % 8 != 0) return "bp must be a multiple of 8 >= b";
  if (pad8(2 * b) > kRvMaxC || bp > kRvMaxC) return "2 b and bp must be at most 8192";
  return nullptr;
}
}  // namespace

#define SH_REQUIRE_SHAPE(what, msg, B, H, W, C) \
  B200_REQUIRE((msg) == nullptr, what ": %s (B=%d H=%d W=%d C=%d)", (msg) ? (msg) : "", B, H, W, C)

extern "C" {

int b200_shuffle_tail_s2_fwd(const void* x, const void* c3, const float* scale, const float* shift, void* y, int B, int H,
                             int W, int Cin, int Cc, void* stream) {
  SH_REQUIRE_SHAPE("shuffle_tail_s2_fwd", nhwc_bad_shape(B, H, W, Cin), B, H, W, Cin);
  B200_REQUIRE(Cc >= 8 && Cc % 8 == 0 && Cin + Cc <= kRvMaxC,
               "shuffle_tail_s2_fwd: Cc must be a multiple of 8 with Cin + Cc <= 8192 (Cin=%d Cc=%d)", Cin, Cc);
  B200_REQUIRE(aligned16(x) && aligned16(c3) && aligned16(scale) && aligned16(shift) && aligned16(y),
               "shuffle_tail_s2_fwd: x, c3, scale, shift, y must be non-null and 16-byte aligned");
  const int Ho = pool_out(H), Wo = pool_out(W);
  const long long n = static_cast<long long>(B) * Ho * Wo * ((Cin + Cc) / 8);
  B200_LAUNCH(shuffle_tail_s2_fwd_kernel, dim3(capped_grid(n)), dim3(256), 0, as_stream(stream),
              static_cast<const uint4*>(x), static_cast<const uint4*>(c3), scale, shift,
              static_cast<uint4*>(y), B, H, W, Ho, Wo, Cin, Cc);
  return OK;
}

int b200_shuffle_relu_bwd(const void* g, const void* y, const void* c, const float* scale, const float* shift, void* dz,
                          float* partial, void* gx, int B, int Ho, int Wo, int Cin, int Cc, int H, int W, void* stream) {
  SH_REQUIRE_SHAPE("shuffle_relu_bwd", nhwc_bad_shape(B, Ho, Wo, Cc), B, Ho, Wo, Cc);
  B200_REQUIRE(Cin >= 0 && Cin % 8 == 0 && Cin + Cc <= kRvMaxC,
               "shuffle_relu_bwd: Cin must be a multiple of 8 >= 0 with Cin + Cc <= 8192 (Cin=%d Cc=%d)", Cin, Cc);
  B200_REQUIRE(aligned16(g) && aligned16(c) && aligned16(dz) && partial != nullptr,
               "shuffle_relu_bwd: g, c, dz must be non-null and 16-byte aligned, partial non-null");
  const bool mask_y = y != nullptr;
  B200_REQUIRE(mask_y ? (scale == nullptr && shift == nullptr && aligned16(y))
                      : (aligned16(scale) && aligned16(shift) && Cin == 0 && gx == nullptr),
               "shuffle_relu_bwd: give y (16-byte aligned) or, for a mask from c scale + shift, scale and shift with "
               "Cin == 0 and no gx");
  const bool pool = gx != nullptr;
  B200_REQUIRE(pool == (Cin > 0), "shuffle_relu_bwd: gx is written exactly when Cin > 0 (the pool half)");
  B200_REQUIRE(!pool || (aligned16(gx) && H >= 1 && W >= 1 && pool_out(H) == Ho && pool_out(W) == Wo),
               "shuffle_relu_bwd: the pool half needs a 16-byte aligned gx and H, W with (H - 1) / 2 + 1 == Ho, "
               "(W - 1) / 2 + 1 == Wo (H=%d W=%d Ho=%d Wo=%d)", H, W, Ho, Wo);
  const long long rows = static_cast<long long>(B) * Ho * Wo;
  const RvGeom gm = repvgg_geom(rows, Cc);
  const dim3 grid(gm.blocks, gm.nchunk, pool ? 2 : 1);
  const auto* pg = static_cast<const uint4*>(g);
  const auto* py = static_cast<const uint4*>(y);
  const auto* pc = static_cast<const uint4*>(c);
  auto* pdz = static_cast<uint4*>(dz);
  auto* pgx = static_cast<uint4*>(gx);
  cudaStream_t st = as_stream(stream);
  if (pool)
    B200_LAUNCH(shuffle_relu_bwd_kernel<true, true>, grid, dim3(256), 0, st, pg, py, pc, scale, shift, pdz,
                partial, pgx, B, H, W, Ho, Wo, Cin, Cc, gm.rows_per_block, gm.gpc);
  else if (mask_y)
    B200_LAUNCH(shuffle_relu_bwd_kernel<true, false>, grid, dim3(256), 0, st, pg, py, pc, scale, shift, pdz,
                partial, pgx, B, H, W, Ho, Wo, Cin, Cc, gm.rows_per_block, gm.gpc);
  else
    B200_LAUNCH(shuffle_relu_bwd_kernel<false, false>, grid, dim3(256), 0, st, pg, py, pc, scale, shift,
                pdz, partial, pgx, B, H, W, Ho, Wo, Cin, Cc, gm.rows_per_block, gm.gpc);
  return OK;
}

int b200_shufflev2_tail_fwd(const void* u, const float* u_scale, const float* u_shift, const void* c3, const float* scale,
                            const float* shift, void* y0, void* y1, long long rows, int b, int bp, void* stream) {
  const char* bad = v2_bad_widths(rows, b, bp);
  B200_REQUIRE(bad == nullptr, "shufflev2_tail_fwd: %s (rows=%lld b=%d bp=%d)", bad ? bad : "", rows, b, bp);
  B200_REQUIRE(aligned16(u) && aligned16(c3) && aligned16(scale) && aligned16(shift) && aligned16(y0),
               "shufflev2_tail_fwd: u, c3, scale, shift, y0 must be non-null and 16-byte aligned");
  const bool bn_u = u_scale != nullptr || u_shift != nullptr;
  B200_REQUIRE(!bn_u || (aligned16(u_scale) && aligned16(u_shift)),
               "shufflev2_tail_fwd: u_scale and u_shift must be given together, 16-byte aligned");
  const bool split = y1 != nullptr;
  B200_REQUIRE(!split || aligned16(y1), "shufflev2_tail_fwd: y1 must be 16-byte aligned");
  const int jp = pad8(2 * b);
  const long long n = rows * (split ? 2 * (bp / 8) : jp / 8);
  const auto* pu = static_cast<const __nv_bfloat16*>(u);
  const auto* pc = static_cast<const __nv_bfloat16*>(c3);
  auto* p0 = static_cast<uint4*>(y0);
  auto* p1 = static_cast<uint4*>(y1);
  const dim3 grid(capped_grid(n));
  cudaStream_t st = as_stream(stream);
  if (bn_u && split)
    B200_LAUNCH(shufflev2_tail_fwd_kernel<true, true>, grid, dim3(256), 0, st, pu, u_scale, u_shift, pc, scale,
                shift, p0, p1, rows, b, bp, jp);
  else if (bn_u)
    B200_LAUNCH(shufflev2_tail_fwd_kernel<true, false>, grid, dim3(256), 0, st, pu, u_scale, u_shift, pc,
                scale, shift, p0, p1, rows, b, bp, jp);
  else if (split)
    B200_LAUNCH(shufflev2_tail_fwd_kernel<false, true>, grid, dim3(256), 0, st, pu, u_scale, u_shift, pc,
                scale, shift, p0, p1, rows, b, bp, jp);
  else
    B200_LAUNCH(shufflev2_tail_fwd_kernel<false, false>, grid, dim3(256), 0, st, pu, u_scale, u_shift, pc,
                scale, shift, p0, p1, rows, b, bp, jp);
  return OK;
}

int b200_shufflev2_tail_bwd(const void* g0, const void* g1, const void* c3, const float* scale, const float* shift,
                            void* dz3, float* partial3, const void* cu, const float* u_scale, const float* u_shift,
                            void* du, float* partial_u, long long rows, int b, int bp, void* stream) {
  const char* bad = v2_bad_widths(rows, b, bp);
  B200_REQUIRE(bad == nullptr, "shufflev2_tail_bwd: %s (rows=%lld b=%d bp=%d)", bad ? bad : "", rows, b, bp);
  B200_REQUIRE(aligned16(g0) && aligned16(c3) && aligned16(scale) && aligned16(shift) && aligned16(dz3) &&
                   aligned16(du) && partial3 != nullptr,
               "shufflev2_tail_bwd: g0, c3, scale, shift, dz3, du must be non-null and 16-byte aligned, partial3 non-null");
  const bool bn_u = cu != nullptr || u_scale != nullptr || u_shift != nullptr || partial_u != nullptr;
  B200_REQUIRE(!bn_u || (aligned16(cu) && aligned16(u_scale) && aligned16(u_shift) && partial_u != nullptr),
               "shufflev2_tail_bwd: cu, u_scale, u_shift (16-byte aligned) and partial_u must be given together");
  const bool split = g1 != nullptr;
  B200_REQUIRE(!split || aligned16(g1), "shufflev2_tail_bwd: g1 must be 16-byte aligned");
  const int jp = pad8(2 * b);
  const RvGeom gm = repvgg_geom(rows, bp);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* p0 = static_cast<const __nv_bfloat16*>(g0);
  const auto* p1 = static_cast<const __nv_bfloat16*>(g1);
  const auto* pc = static_cast<const uint4*>(c3);
  const auto* pu = static_cast<const uint4*>(cu);
  auto* pz = static_cast<uint4*>(dz3);
  auto* pd = static_cast<uint4*>(du);
  cudaStream_t st = as_stream(stream);
  if (bn_u && split)
    B200_LAUNCH(shufflev2_tail_bwd_kernel<true, true>, grid, dim3(256), 0, st, p0, p1, pc, scale, shift, pz,
                partial3, pu, u_scale, u_shift, pd, partial_u, rows, b, bp, jp, gm.rows_per_block, gm.gpc);
  else if (bn_u)
    B200_LAUNCH(shufflev2_tail_bwd_kernel<true, false>, grid, dim3(256), 0, st, p0, p1, pc, scale, shift, pz,
                partial3, pu, u_scale, u_shift, pd, partial_u, rows, b, bp, jp, gm.rows_per_block, gm.gpc);
  else if (split)
    B200_LAUNCH(shufflev2_tail_bwd_kernel<false, true>, grid, dim3(256), 0, st, p0, p1, pc, scale, shift, pz,
                partial3, pu, u_scale, u_shift, pd, partial_u, rows, b, bp, jp, gm.rows_per_block, gm.gpc);
  else
    B200_LAUNCH(shufflev2_tail_bwd_kernel<false, false>, grid, dim3(256), 0, st, p0, p1, pc, scale, shift,
                pz, partial3, pu, u_scale, u_shift, pd, partial_u, rows, b, bp, jp, gm.rows_per_block,
                gm.gpc);
  return OK;
}

}  // extern "C"
