// C-ABI entry points of the EfficientNet MBConv passes (see mbconv.cuh).  Every entry validates its shapes and pointers
// before it launches anything.
#include <stdint.h>

#include "../../include/b200cls.h"
#include "mbconv.cuh"
#include "host_utils.h"

using namespace b200;

namespace {
const char* mb_bad_shape(long long B, long long HW, int C) {
  if (B < 1 || B > 65535) return "B must be in [1, 65535]";
  if (HW < 1) return "HW must be >= 1";
  if (C < 8 || C % 8 != 0 || C > kRvMaxC) return "C must be a multiple of 8 in [8, 8192]";
  return nullptr;
}

const char* dw_bad_shape(int B, int H, int W, int C, int k, int stride) {
  if (k != 3 && k != 5) return "k must be 3 or 5";
  if (stride != 1 && stride != 2) return "stride must be 1 or 2";
  if (H < 1 || W < 1) return "H and W must be >= 1";
  return mb_bad_shape(B, static_cast<long long>(H) * W, C);
}

int out_size(int n, int stride) { return (n - 1) / stride + 1; }   // pad k/2, odd k
}  // namespace

#define MB_REQUIRE_SHAPE(what, msg)                                                 \
  B200_REQUIRE((msg) == nullptr, what ": %s", (msg) ? (msg) : "")

// CALL(K, S) with the compile-time kernel size and stride of the runtime k / stride
#define DW_DISPATCH(k, stride, CALL)                  \
  do {                                                \
    if ((k) == 3 && (stride) == 1) { CALL(3, 1); }    \
    else if ((k) == 3) { CALL(3, 2); }                \
    else if ((stride) == 1) { CALL(5, 1); }           \
    else { CALL(5, 2); }                              \
  } while (0)

// CALL(S) with the compile-time stride of the runtime stride (3x3 kernels)
#define DW_STRIDE_DISPATCH(stride, CALL) \
  do {                                   \
    if ((stride) == 1) { CALL(1); }      \
    else { CALL(2); }                    \
  } while (0)

extern "C" {

int b200_dw_partial_rows(long long rows, int C) {
  if (rows < 1 || C < 8 || C % 8 != 0 || C > kRvMaxC) {
    set_error("dw_partial_rows: rows must be >= 1 and C a multiple of 8 in [8, 8192] (rows=%lld C=%d)", rows, C);
    return -1;
  }
  return dw_geom(rows, C).blocks;
}

int b200_dw_fwd(const void* x, const float* w, const float* scale, const float* shift, void* d, float* stats, int B, int H,
                int W, int C, int k, int stride, void* stream) {
  MB_REQUIRE_SHAPE("dw_fwd", dw_bad_shape(B, H, W, C, k, stride));
  B200_REQUIRE(aligned16(x) && w != nullptr && aligned16(d),
               "dw_fwd: x and d must be non-null and 16-byte aligned, w non-null");
  B200_REQUIRE((scale == nullptr) == (shift == nullptr) && opt16(scale) && opt16(shift),
               "dw_fwd: the on-load BatchNorm needs both scale and shift, 16-byte aligned");
  const int Ho = out_size(H, stride), Wo = out_size(W, stride);
  const DwGeom gm = dw_geom(static_cast<long long>(B) * Ho * Wo, C);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  auto* pd = static_cast<__nv_bfloat16*>(d);
  const bool pre = scale != nullptr, st = stats != nullptr;
#define DW_FWD(K, S)                                                                                                      \
  if (pre && st)                                                                                                          \
    B200_LAUNCH(dw_fwd_kernel<K, S, true, true>, grid, dim3(256), 0, as_stream(stream), px, w, scale,                    \
                shift, pd, stats, B, H, W, Ho, Wo, C, gm.rows_per_block);                                                 \
  else if (pre)                                                                                                           \
    B200_LAUNCH(dw_fwd_kernel<K, S, true, false>, grid, dim3(256), 0, as_stream(stream), px, w, scale,                   \
                shift, pd, stats, B, H, W, Ho, Wo, C, gm.rows_per_block);                                                 \
  else if (st)                                                                                                            \
    B200_LAUNCH(dw_fwd_kernel<K, S, false, true>, grid, dim3(256), 0, as_stream(stream), px, w, scale,                   \
                shift, pd, stats, B, H, W, Ho, Wo, C, gm.rows_per_block);                                                 \
  else                                                                                                                    \
    B200_LAUNCH(dw_fwd_kernel<K, S, false, false>, grid, dim3(256), 0, as_stream(stream), px, w, scale,                  \
                shift, pd, stats, B, H, W, Ho, Wo, C, gm.rows_per_block)
  DW_DISPATCH(k, stride, DW_FWD);
#undef DW_FWD
  return OK;
}

int b200_dw_dgrad(const void* dd, const float* w, const void* x, const float* scale, const float* shift,
                  const void* residual, void* dx, float* partial, int B, int H, int W, int C, int k, int stride,
                  void* stream) {
  MB_REQUIRE_SHAPE("dw_dgrad", dw_bad_shape(B, H, W, C, k, stride));
  B200_REQUIRE(aligned16(dd) && w != nullptr && aligned16(dx), "dw_dgrad: dd and dx must be non-null and 16-byte aligned, "
               "w non-null");
  const bool pre = scale != nullptr;
  B200_REQUIRE(!pre || (aligned16(x) && aligned16(scale) && aligned16(shift) && partial != nullptr),
               "dw_dgrad: the on-load BatchNorm needs x, scale, shift (16-byte aligned) and partial");
  B200_REQUIRE(pre || (shift == nullptr && partial == nullptr), "dw_dgrad: shift / partial given without scale");
  B200_REQUIRE(opt16(residual) && !(pre && residual != nullptr),
               "dw_dgrad: residual must be 16-byte aligned and cannot be combined with the on-load BatchNorm");
  const int Ho = out_size(H, stride), Wo = out_size(W, stride);
  const DwGeom gm = dw_geom(static_cast<long long>(B) * H * W, C);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* pdd = static_cast<const __nv_bfloat16*>(dd);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  const auto* pr = static_cast<const __nv_bfloat16*>(residual);
  auto* pdx = static_cast<__nv_bfloat16*>(dx);
  const bool res = residual != nullptr;
#define DW_DGRAD(K, S)                                                                                                    \
  if (pre)                                                                                                                \
    B200_LAUNCH(dw_dgrad_kernel<K, S, true, false>, grid, dim3(256), 0, as_stream(stream), pdd, w, px,                   \
                scale, shift, pr, pdx, partial, B, H, W, Ho, Wo, C, gm.rows_per_block);                                   \
  else if (res)                                                                                                           \
    B200_LAUNCH(dw_dgrad_kernel<K, S, false, true>, grid, dim3(256), 0, as_stream(stream), pdd, w, px,                   \
                scale, shift, pr, pdx, partial, B, H, W, Ho, Wo, C, gm.rows_per_block);                                   \
  else                                                                                                                    \
    B200_LAUNCH(dw_dgrad_kernel<K, S, false, false>, grid, dim3(256), 0, as_stream(stream), pdd, w, px,                  \
                scale, shift, pr, pdx, partial, B, H, W, Ho, Wo, C, gm.rows_per_block)
  DW_DISPATCH(k, stride, DW_DGRAD);
#undef DW_DGRAD
  return OK;
}

size_t b200_dw_wgrad_workspace_bytes(int B, int H, int W, int C, int k, int stride) {
  if (dw_bad_shape(B, H, W, C, k, stride) != nullptr) return 0;
  const long long rows = static_cast<long long>(B) * out_size(H, stride) * out_size(W, stride);
  return static_cast<size_t>(dw_geom(rows, C).blocks) * k * k * C * sizeof(float);
}

int b200_dw_wgrad(const void* dd, const void* x, const float* scale, const float* shift, float* dw, void* ws,
                  size_t ws_bytes, int B, int H, int W, int C, int k, int stride, void* stream) {
  MB_REQUIRE_SHAPE("dw_wgrad", dw_bad_shape(B, H, W, C, k, stride));
  B200_REQUIRE(aligned16(dd) && aligned16(x) && dw != nullptr && ws != nullptr,
               "dw_wgrad: dd and x must be non-null and 16-byte aligned, dw and ws non-null");
  B200_REQUIRE((scale == nullptr) == (shift == nullptr) && opt16(scale) && opt16(shift),
               "dw_wgrad: the on-load BatchNorm needs both scale and shift, 16-byte aligned");
  const size_t need = b200_dw_wgrad_workspace_bytes(B, H, W, C, k, stride);
  B200_REQUIRE(ws_bytes >= need, "dw_wgrad: workspace of %zu bytes, need %zu", ws_bytes, need);
  const int Ho = out_size(H, stride), Wo = out_size(W, stride);
  const DwGeom gm = dw_geom(static_cast<long long>(B) * Ho * Wo, C);
  const dim3 grid(gm.blocks, gm.nchunk, k);
  const auto* pdd = static_cast<const __nv_bfloat16*>(dd);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  float* pws = static_cast<float*>(ws);
  const bool pre = scale != nullptr;
#define DW_WGRAD(K, S)                                                                                                    \
  if (pre)                                                                                                                \
    B200_LAUNCH(dw_wgrad_kernel<K, S, true>, grid, dim3(256), 0, as_stream(stream), pdd, px, scale, shift,               \
                pws, B, H, W, Ho, Wo, C, gm.rows_per_block);                                                              \
  else                                                                                                                    \
    B200_LAUNCH(dw_wgrad_kernel<K, S, false>, grid, dim3(256), 0, as_stream(stream), pdd, px, scale,                     \
                shift, pws, B, H, W, Ho, Wo, C, gm.rows_per_block)
  DW_DISPATCH(k, stride, DW_WGRAD);
#undef DW_WGRAD
  const long long n = static_cast<long long>(k) * k * C;
  B200_LAUNCH(dw_wgrad_reduce_kernel, dim3(static_cast<unsigned>((n + 31) / 32)), dim3(256), 0,
              as_stream(stream), static_cast<const float*>(pws), dw, gm.blocks, k * k, C);
  return OK;
}

// ShuffleNet's depthwise convolution: the kDwRelu mode of the same kernels, k = 3
int b200_dw_relu_fwd(const void* x, const float* w, const float* scale, const float* shift, void* d, float* stats, int B,
                     int H, int W, int C, int stride, void* stream) {
  MB_REQUIRE_SHAPE("dw_relu_fwd", dw_bad_shape(B, H, W, C, 3, stride));
  B200_REQUIRE(aligned16(x) && w != nullptr && aligned16(d) && aligned16(scale) && aligned16(shift),
               "dw_relu_fwd: x, d, scale, shift must be non-null and 16-byte aligned, w non-null");
  const int Ho = out_size(H, stride), Wo = out_size(W, stride);
  const DwGeom gm = dw_geom(static_cast<long long>(B) * Ho * Wo, C);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  auto* pd = static_cast<__nv_bfloat16*>(d);
#define DWR_FWD(S)                                                                                                        \
  if (stats != nullptr)                                                                                                   \
    B200_LAUNCH(dw_fwd_kernel<3, S, kDwRelu, true>, grid, dim3(256), 0, as_stream(stream), px, w, scale,                 \
                shift, pd, stats, B, H, W, Ho, Wo, C, gm.rows_per_block);                                                 \
  else                                                                                                                    \
    B200_LAUNCH(dw_fwd_kernel<3, S, kDwRelu, false>, grid, dim3(256), 0, as_stream(stream), px, w, scale,                \
                shift, pd, stats, B, H, W, Ho, Wo, C, gm.rows_per_block)
  DW_STRIDE_DISPATCH(stride, DWR_FWD);
#undef DWR_FWD
  return OK;
}

int b200_dw_relu_dgrad(const void* dd, const float* w, const void* x, const float* scale, const float* shift, void* dx,
                       float* partial, int B, int H, int W, int C, int stride, void* stream) {
  MB_REQUIRE_SHAPE("dw_relu_dgrad", dw_bad_shape(B, H, W, C, 3, stride));
  B200_REQUIRE(aligned16(dd) && w != nullptr && aligned16(x) && aligned16(scale) && aligned16(shift) && aligned16(dx) &&
                   partial != nullptr,
               "dw_relu_dgrad: dd, x, scale, shift, dx must be non-null and 16-byte aligned, w and partial non-null");
  const int Ho = out_size(H, stride), Wo = out_size(W, stride);
  const DwGeom gm = dw_geom(static_cast<long long>(B) * H * W, C);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* pdd = static_cast<const __nv_bfloat16*>(dd);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* none = nullptr;
  auto* pdx = static_cast<__nv_bfloat16*>(dx);
#define DWR_DGRAD(S)                                                                                                      \
  B200_LAUNCH(dw_dgrad_kernel<3, S, kDwRelu, false>, grid, dim3(256), 0, as_stream(stream), pdd, w, px,                  \
              scale, shift, none, pdx, partial, B, H, W, Ho, Wo, C, gm.rows_per_block)
  DW_STRIDE_DISPATCH(stride, DWR_DGRAD);
#undef DWR_DGRAD
  return OK;
}

int b200_dw_relu_wgrad(const void* dd, const void* x, const float* scale, const float* shift, float* dw, void* ws,
                       size_t ws_bytes, int B, int H, int W, int C, int stride, void* stream) {
  MB_REQUIRE_SHAPE("dw_relu_wgrad", dw_bad_shape(B, H, W, C, 3, stride));
  B200_REQUIRE(aligned16(dd) && aligned16(x) && aligned16(scale) && aligned16(shift) && dw != nullptr && ws != nullptr,
               "dw_relu_wgrad: dd, x, scale, shift must be non-null and 16-byte aligned, dw and ws non-null");
  const size_t need = b200_dw_wgrad_workspace_bytes(B, H, W, C, 3, stride);
  B200_REQUIRE(ws_bytes >= need, "dw_relu_wgrad: workspace of %zu bytes, need %zu", ws_bytes, need);
  const int Ho = out_size(H, stride), Wo = out_size(W, stride);
  const DwGeom gm = dw_geom(static_cast<long long>(B) * Ho * Wo, C);
  const dim3 grid(gm.blocks, gm.nchunk, 3);
  const auto* pdd = static_cast<const __nv_bfloat16*>(dd);
  const auto* px = static_cast<const __nv_bfloat16*>(x);
  float* pws = static_cast<float*>(ws);
#define DWR_WGRAD(S)                                                                                                      \
  B200_LAUNCH(dw_wgrad_kernel<3, S, kDwRelu>, grid, dim3(256), 0, as_stream(stream), pdd, px, scale, shift,               \
              pws, B, H, W, Ho, Wo, C, gm.rows_per_block)
  DW_STRIDE_DISPATCH(stride, DWR_WGRAD);
#undef DWR_WGRAD
  const long long n = 9ll * C;
  B200_LAUNCH(dw_wgrad_reduce_kernel, dim3(static_cast<unsigned>((n + 31) / 32)), dim3(256), 0,
              as_stream(stream), static_cast<const float*>(pws), dw, gm.blocks, 9, C);
  return OK;
}

int b200_silu_bn_squeeze(const void* d, const float* scale, const float* shift, const float* mask, float* pool,
                         void* out16, int B, int HW, int C, void* stream) {
  MB_REQUIRE_SHAPE("silu_bn_squeeze", mb_bad_shape(B, HW, C));
  B200_REQUIRE(aligned16(d) && aligned16(scale) && aligned16(shift) && pool != nullptr,
               "silu_bn_squeeze: d, scale, shift must be non-null and 16-byte aligned, pool non-null");
  B200_REQUIRE((mask == nullptr) == (out16 == nullptr), "silu_bn_squeeze: the masked bf16 copy needs both mask and out16");
  const RvGeom gm = repvgg_geom(HW, C);
  const dim3 grid(B, gm.nchunk);
  const auto* pd = static_cast<const uint4*>(d);
  auto* po = static_cast<__nv_bfloat16*>(out16);
  if (mask != nullptr)
    B200_LAUNCH(mb_image_sum_kernel<false, true>, grid, dim3(256), 0, as_stream(stream),
                static_cast<const uint4*>(nullptr), pd, scale, shift, mask, pool, po, HW, C, gm.gpc);
  else
    B200_LAUNCH(mb_image_sum_kernel<false, false>, grid, dim3(256), 0, as_stream(stream),
                static_cast<const uint4*>(nullptr), pd, scale, shift, mask, pool, po, HW, C, gm.gpc);
  return OK;
}

int b200_excite_fwd(const float* pool, const float* w1, const float* b1, const float* w2, const float* b2, float* hpre,
                    float* gate, int B, int C, int Cr, void* stream) {
  MB_REQUIRE_SHAPE("excite_fwd", mb_bad_shape(B, 1, C));
  B200_REQUIRE(Cr >= 1 && Cr <= 256, "excite_fwd: Cr must be in [1, 256] (Cr=%d)", Cr);
  const void* need[] = {pool, w1, b1, w2, b2, hpre, gate};
  for (const void* p : need) B200_REQUIRE(p != nullptr, "excite_fwd: pool, w1, b1, w2, b2, hpre, gate are required");
  B200_LAUNCH(mb_excite_fwd_kernel, dim3(B), dim3(256), (C + Cr) * sizeof(float), as_stream(stream), pool,
              w1, b1, w2, b2, hpre, gate, C, Cr);
  return OK;
}

int b200_excite_bwd(const float* s, const float* pool, const float* hpre, const float* gate, const float* w1,
                    const float* w2, float* dgp, float* dhp, float* dw1, float* db1, float* dw2, float* db2, float* dpool,
                    int B, int C, int Cr, void* stream) {
  MB_REQUIRE_SHAPE("excite_bwd", mb_bad_shape(B, 1, C));
  B200_REQUIRE(Cr >= 1 && Cr <= 256, "excite_bwd: Cr must be in [1, 256] (Cr=%d)", Cr);
  const void* need[] = {s, pool, hpre, gate, w1, w2, dgp, dhp, dw1, db1, dw2, db2, dpool};
  for (const void* p : need) B200_REQUIRE(p != nullptr, "excite_bwd: every pointer is required");
  B200_LAUNCH(mb_excite_bwd_image_kernel, dim3(B), dim3(256), C * sizeof(float), as_stream(stream), s, gate,
              hpre, w2, dgp, dhp, C, Cr);
  const long long total = 2ll * C * Cr + C + Cr + static_cast<long long>(B) * C;
  long long blocks = (total + 255) / 256;
  if (blocks > 4 * kNumSMs * 8) blocks = 4 * kNumSMs * 8;
  B200_LAUNCH(mb_excite_bwd_params_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0,
              as_stream(stream), static_cast<const float*>(dgp), static_cast<const float*>(dhp), hpre, pool,
              w1, dw1, db1, dw2, db2, dpool, B, C, Cr);
  return OK;
}

int b200_gate_apply(const void* d, const float* scale, const float* shift, const float* gate, void* a, int B, int HW, int C,
                    void* stream) {
  MB_REQUIRE_SHAPE("gate_apply", mb_bad_shape(B, HW, C));
  B200_REQUIRE(aligned16(d) && aligned16(scale) && aligned16(shift) && aligned16(gate) && aligned16(a),
               "gate_apply: d, scale, shift, gate, a must be non-null and 16-byte aligned");
  const long long rows = static_cast<long long>(B) * HW;
  const RvGeom gm = repvgg_geom(rows, C);
  B200_LAUNCH(mb_apply_kernel<true, false, false>, dim3(gm.blocks, gm.nchunk), dim3(256), 0,
              as_stream(stream), static_cast<const uint4*>(d), scale, shift, gate,
              static_cast<const uint4*>(nullptr), static_cast<uint4*>(a), rows, HW, C, gm.rows_per_block,
              gm.gpc);
  return OK;
}

int b200_gate_reduce(const void* da, const void* d, const float* scale, const float* shift, float* s, int B, int HW, int C,
                     void* stream) {
  MB_REQUIRE_SHAPE("gate_reduce", mb_bad_shape(B, HW, C));
  B200_REQUIRE(aligned16(da) && aligned16(d) && aligned16(scale) && aligned16(shift) && s != nullptr,
               "gate_reduce: da, d, scale, shift must be non-null and 16-byte aligned, s non-null");
  const RvGeom gm = repvgg_geom(HW, C);
  B200_LAUNCH(mb_image_sum_kernel<true, false>, dim3(B, gm.nchunk), dim3(256), 0, as_stream(stream),
              static_cast<const uint4*>(da), static_cast<const uint4*>(d), scale, shift,
              static_cast<const float*>(nullptr), s, static_cast<__nv_bfloat16*>(nullptr), HW, C, gm.gpc);
  return OK;
}

int b200_silu_bn_bwd_reduce(const void* da, const float* gate, const float* dpool, const void* d, const float* scale,
                            const float* shift, void* dz, float* partial, int B, int HW, int C, void* stream) {
  MB_REQUIRE_SHAPE("silu_bn_bwd_reduce", mb_bad_shape(B, HW, C));
  B200_REQUIRE(aligned16(dpool) && aligned16(d) && aligned16(scale) && aligned16(shift) && aligned16(dz) &&
                   partial != nullptr,
               "silu_bn_bwd_reduce: dpool, d, scale, shift, dz must be non-null and 16-byte aligned, partial non-null");
  B200_REQUIRE((da == nullptr) == (gate == nullptr) && opt16(da) && opt16(gate),
               "silu_bn_bwd_reduce: da and gate come together, 16-byte aligned");
  const long long rows = static_cast<long long>(B) * HW;
  const RvGeom gm = repvgg_geom(rows, C);
  const dim3 grid(gm.blocks, gm.nchunk);
  if (da != nullptr)
    B200_LAUNCH(mb_bwd_reduce_kernel<true, true>, grid, dim3(256), 0, as_stream(stream),
                static_cast<const uint4*>(da), gate, dpool, static_cast<const uint4*>(d), scale, shift,
                static_cast<uint4*>(dz), partial, rows, HW, C, gm.rows_per_block, gm.gpc);
  else
    B200_LAUNCH(mb_bwd_reduce_kernel<true, false>, grid, dim3(256), 0, as_stream(stream),
                static_cast<const uint4*>(da), gate, dpool, static_cast<const uint4*>(d), scale, shift,
                static_cast<uint4*>(dz), partial, rows, HW, C, gm.rows_per_block, gm.gpc);
  return OK;
}

int b200_tail_apply(const void* c, const float* scale, const float* shift, const float* rs, const void* residual, void* y,
                    int B, int HW, int C, void* stream) {
  MB_REQUIRE_SHAPE("tail_apply", mb_bad_shape(B, HW, C));
  B200_REQUIRE(aligned16(c) && aligned16(scale) && aligned16(shift) && aligned16(y) && opt16(residual),
               "tail_apply: c, scale, shift, y (and residual) must be non-null and 16-byte aligned");
  const long long rows = static_cast<long long>(B) * HW;
  const RvGeom gm = repvgg_geom(rows, C);
  const dim3 grid(gm.blocks, gm.nchunk);
  const auto* pc = static_cast<const uint4*>(c);
  const auto* pr = static_cast<const uint4*>(residual);
  auto* py = static_cast<uint4*>(y);
  cudaStream_t st = as_stream(stream);
  if (rs != nullptr && residual != nullptr)
    B200_LAUNCH(mb_apply_kernel<false, true, true>, grid, dim3(256), 0, st, pc, scale, shift, rs, pr, py,
                rows, HW, C, gm.rows_per_block, gm.gpc);
  else if (rs != nullptr)
    B200_LAUNCH(mb_apply_kernel<false, true, false>, grid, dim3(256), 0, st, pc, scale, shift, rs, pr, py,
                rows, HW, C, gm.rows_per_block, gm.gpc);
  else if (residual != nullptr)
    B200_LAUNCH(mb_apply_kernel<false, false, true>, grid, dim3(256), 0, st, pc, scale, shift, rs, pr, py,
                rows, HW, C, gm.rows_per_block, gm.gpc);
  else
    B200_LAUNCH(mb_apply_kernel<false, false, false>, grid, dim3(256), 0, st, pc, scale, shift, rs, pr, py,
                rows, HW, C, gm.rows_per_block, gm.gpc);
  return OK;
}

int b200_tail_bwd_reduce(const void* g, const float* rs, const void* c, void* dz, float* partial, int B, int HW, int C,
                         void* stream) {
  MB_REQUIRE_SHAPE("tail_bwd_reduce", mb_bad_shape(B, HW, C));
  B200_REQUIRE(aligned16(g) && aligned16(c) && partial != nullptr,
               "tail_bwd_reduce: g and c must be non-null and 16-byte aligned, partial non-null");
  B200_REQUIRE((rs == nullptr) == (dz == nullptr) && opt16(dz),
               "tail_bwd_reduce: dz is stored exactly when rs is given (16-byte aligned)");
  const long long rows = static_cast<long long>(B) * HW;
  const RvGeom gm = repvgg_geom(rows, C);
  const dim3 grid(gm.blocks, gm.nchunk);
  const float* none = nullptr;
  if (rs != nullptr)
    B200_LAUNCH(mb_bwd_reduce_kernel<false, true>, grid, dim3(256), 0, as_stream(stream),
                static_cast<const uint4*>(g), rs, none, static_cast<const uint4*>(c), none, none,
                static_cast<uint4*>(dz), partial, rows, HW, C, gm.rows_per_block, gm.gpc);
  else
    B200_LAUNCH(mb_bwd_reduce_kernel<false, false>, grid, dim3(256), 0, as_stream(stream),
                static_cast<const uint4*>(g), rs, none, static_cast<const uint4*>(c), none, none,
                static_cast<uint4*>(dz), partial, rows, HW, C, gm.rows_per_block, gm.gpc);
  return OK;
}

}  // extern "C"
