// C-ABI entry points of the ShuffleNet v1 block tails (see shufflenet.cuh; the ReLU-on-load depthwise entries live with the
// other depthwise entries in abi_mbconv.cu).  Every entry validates its shapes and pointers before it launches anything.
#include <stdint.h>

#include "../../include/b200cls.h"
#include "shufflenet.cuh"
#include "host_utils.h"

using namespace b200;

namespace {
bool aligned16(const void* p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }

const char* sh_bad_shape(int B, int H, int W, int C) {
  if (B < 1 || B > 65535) return "B must be in [1, 65535]";
  if (H < 1 || W < 1) return "H and W must be >= 1";
  if (C < 8 || C % 8 != 0 || C > kRvMaxC) return "C must be a multiple of 8 in [8, 8192]";
  return nullptr;
}

int pool_out(int n) { return (n - 1) / 2 + 1; }   // output extent of a 3x3 / stride 2 / pad 1 window

int ew_blocks(long long items) {
  long long blocks = (items + 255) / 256;
  const long long cap = static_cast<long long>(device_sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  return blocks < 1 ? 1 : static_cast<int>(blocks);
}
}  // namespace

#define SH_REQUIRE_SHAPE(what, msg, B, H, W, C) \
  B200_REQUIRE((msg) == nullptr, what ": %s (B=%d H=%d W=%d C=%d)", (msg) ? (msg) : "", B, H, W, C)

extern "C" {

int b200_shuffle_tail_s2_fwd(const void* x, const void* c3, const float* scale, const float* shift, void* y, int B, int H,
                             int W, int Cin, int Cc, void* stream) {
  SH_REQUIRE_SHAPE("shuffle_tail_s2_fwd", sh_bad_shape(B, H, W, Cin), B, H, W, Cin);
  B200_REQUIRE(Cc >= 8 && Cc % 8 == 0 && Cin + Cc <= kRvMaxC,
               "shuffle_tail_s2_fwd: Cc must be a multiple of 8 with Cin + Cc <= 8192 (Cin=%d Cc=%d)", Cin, Cc);
  B200_REQUIRE(aligned16(x) && aligned16(c3) && aligned16(scale) && aligned16(shift) && aligned16(y),
               "shuffle_tail_s2_fwd: x, c3, scale, shift, y must be non-null and 16-byte aligned");
  const int Ho = pool_out(H), Wo = pool_out(W);
  const long long n = static_cast<long long>(B) * Ho * Wo * ((Cin + Cc) / 8);
  B200_CHECK_CUDA(launch_pdl(shuffle_tail_s2_fwd_kernel, dim3(ew_blocks(n)), dim3(256), 0, as_stream(stream),
                             static_cast<const uint4*>(x), static_cast<const uint4*>(c3), scale, shift,
                             static_cast<uint4*>(y), B, H, W, Ho, Wo, Cin, Cc));
  B200_LAUNCHED();
  return OK;
}

int b200_shuffle_relu_bwd(const void* g, const void* y, const void* c, const float* scale, const float* shift, void* dz,
                          float* partial, void* gx, int B, int Ho, int Wo, int Cin, int Cc, int H, int W, void* stream) {
  SH_REQUIRE_SHAPE("shuffle_relu_bwd", sh_bad_shape(B, Ho, Wo, Cc), B, Ho, Wo, Cc);
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
    B200_CHECK_CUDA(launch_pdl(shuffle_relu_bwd_kernel<true, true>, grid, dim3(256), 0, st, pg, py, pc, scale, shift, pdz,
                               partial, pgx, B, H, W, Ho, Wo, Cin, Cc, gm.rows_per_block, gm.gpc));
  else if (mask_y)
    B200_CHECK_CUDA(launch_pdl(shuffle_relu_bwd_kernel<true, false>, grid, dim3(256), 0, st, pg, py, pc, scale, shift, pdz,
                               partial, pgx, B, H, W, Ho, Wo, Cin, Cc, gm.rows_per_block, gm.gpc));
  else
    B200_CHECK_CUDA(launch_pdl(shuffle_relu_bwd_kernel<false, false>, grid, dim3(256), 0, st, pg, py, pc, scale, shift,
                               pdz, partial, pgx, B, H, W, Ho, Wo, Cin, Cc, gm.rows_per_block, gm.gpc));
  B200_LAUNCHED();
  return OK;
}

}  // extern "C"
