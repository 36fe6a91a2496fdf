// C-ABI entry points of the transformer-side kernels: LayerNorm, patch extraction, attention (wgmma) forward/backward.
#include <string.h>

#include "../../include/b200cls.h"
#include "attention.cuh"
#include "attention_bwd.cuh"
#include "attention_fwd2.cuh"
#include "host_utils.h"
#include "convnext.cuh"
#include "transformer.cuh"
#include "window_attention.cuh"

using namespace b200;

namespace {
int ln_bwd_blocks(long long rows) {
  long long b = static_cast<long long>(device_sm_count()) * 3;
  if (b > (rows + 7) / 8) b = (rows + 7) / 8;
  return static_cast<int>(b < 1 ? 1 : b);
}
int encode3(CUtensorMap* m, const void* base, long long cols, long long T, long long B, int box_rows) {
  uint64_t dims[3] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(T), static_cast<uint64_t>(B)};
  uint64_t strides[3] = {1, static_cast<uint64_t>(cols), static_cast<uint64_t>(cols) * T};
  uint32_t box[3] = {64, static_cast<uint32_t>(box_rows), 1};
  return encode_tmap_bf16(m, base, 3, dims, strides, box);
}
}  // namespace

extern "C" {

int b200_layernorm_fwd(const void* x, int x_f32, const float* gamma, const float* beta, void* y, int y_f32, float* mean,
                       float* rstd, long long rows, int C, float eps, void* stream) {
  B200_REQUIRE(C % 8 == 0 && C <= 3072, "layernorm_fwd: C=%d must be a multiple of 8 and <= 3072", C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define LN_FWD(TI, TY, MV, LPR)                                                                                      \
  B200_LAUNCH(layernorm_fwd_kernel<TI, TY, MV, LPR>, dim3(capped_grid((rows + 32 / LPR - 1) / (32 / LPR), 8)), dim3(256), 0, st,                            \
      static_cast<const TI*>(x), gamma, beta, static_cast<TY*>(y), mean, rstd, rows, C, eps)
#define LN_FWD_T(MV, LPR)                              \
  do {                                                 \
    if (x_f32 && y_f32)                                \
      LN_FWD(float, float, MV, LPR);                   \
    else if (x_f32)                                    \
      LN_FWD(float, __nv_bfloat16, MV, LPR);           \
    else if (y_f32)                                    \
      LN_FWD(__nv_bfloat16, float, MV, LPR);           \
    else                                               \
      LN_FWD(__nv_bfloat16, __nv_bfloat16, MV, LPR);   \
  } while (0)
  if (C <= 128)
    LN_FWD_T(2, 8);     // 4 rows per warp (ConvNeXt / Swin stage 1: C = 96)
  else if (C <= 256)
    LN_FWD_T(2, 16);    // 2 rows per warp (C = 192)
  else if (C <= 1024)
    LN_FWD_T(4, 32);
  else
    LN_FWD_T(12, 32);
#undef LN_FWD_T
#undef LN_FWD
  return OK;
}

int b200_layernorm_bwd_blocks(long long rows, int C) {
  if (C % 8 != 0 || C > 1024) {
    set_error("layernorm_bwd_blocks: C=%d must be a multiple of 8 and <= 1024", C);
    return -1;
  }
  return ln_bwd_blocks(rows);
}

int b200_layernorm_bwd(const void* dy, const void* x, int x_f32, const float* mean, const float* rstd, const float* gamma,
                       const void* add, void* dx, int dx_f32, float* partial, long long rows, int C, void* stream) {
  B200_REQUIRE(C % 8 == 0 && C <= 1024, "layernorm_bwd: C=%d must be a multiple of 8 and <= 1024", C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = ln_bwd_blocks(rows);
  const __nv_bfloat16* dyp = static_cast<const __nv_bfloat16*>(dy);
#define LN_BWD_V(TI, TO, MV, LPR)                                                                                   \
  do {                                                                                                              \
    static bool cfg = false;                                                                                        \
    if (!cfg) {                                                                                                     \
      B200_CHECK_CUDA(cudaFuncSetAttribute(layernorm_bwd_kernel<TI, TO, MV, LPR>,                                   \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize,                             \
                                           8 * 2 * 1024 * (int)sizeof(float)));                                     \
      cfg = true;                                                                                                   \
    }                                                                                                               \
    const size_t smem = static_cast<size_t>(8) * (32 / LPR) * 2 * C * sizeof(float);                                \
    B200_LAUNCH(layernorm_bwd_kernel<TI, TO, MV, LPR>, dim3(grid), dim3(256), smem, st, dyp,                        \
                static_cast<const TI*>(x), mean, rstd, gamma, static_cast<const TO*>(add),                         \
                static_cast<TO*>(dx), partial, rows, C);                                                            \
  } while (0)
#define LN_BWD(TI, TO)                  \
  do {                                  \
    if (C <= 128)                       \
      LN_BWD_V(TI, TO, 2, 8);           \
    else if (C <= 256)                  \
      LN_BWD_V(TI, TO, 2, 16);          \
    else if (C <= 512)                  \
      LN_BWD_V(TI, TO, 2, 32);          \
    else if (C <= 768)                  \
      LN_BWD_V(TI, TO, 3, 32);          \
    else                                \
      LN_BWD_V(TI, TO, 4, 32);          \
  } while (0)
  if (x_f32 && dx_f32)
    LN_BWD(float, float);
  else if (x_f32 && !dx_f32)
    LN_BWD(float, __nv_bfloat16);
  else if (!x_f32 && dx_f32)
    LN_BWD(__nv_bfloat16, float);
  else
    LN_BWD(__nv_bfloat16, __nv_bfloat16);
#undef LN_BWD
#undef LN_BWD_V
  return OK;
}

int b200_patchify_nchw(const float* x, void* a, int B, int Cin, int H, int W, int ps, void* stream) {
  B200_REQUIRE(ps % 4 == 0 && H % ps == 0 && W % ps == 0 && W % 4 == 0, "patchify: patch %d must divide %dx%d (multiples of 4)", ps, H, W);
  const long long total = static_cast<long long>(B) * (H / ps) * (W / ps) * (Cin * ps * ps / 4);
  B200_LAUNCH(patchify_nchw_kernel, dim3(capped_grid(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      x, static_cast<__nv_bfloat16*>(a), B, Cin, H, W, ps);
  return OK;
}

int b200_cls_row(const float* cls, const float* pos, float* tokens, int B, int T, int D, void* stream) {
  B200_LAUNCH(cls_row_kernel, dim3(capped_grid(static_cast<long long>(B) * D, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), cls, pos, tokens, B, T, D);
  return OK;
}

int b200_batch_rowsum(const void* g, int g_f32, long long stride_b, int B, int D, float* out, int accumulate,
                      void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (g_f32)
    B200_LAUNCH(batch_rowsum_kernel<float>, dim3((D + 255) / 256), dim3(256), 0, st, static_cast<const float*>(g), stride_b, B, D, out, accumulate);
  else
    B200_LAUNCH(batch_rowsum_kernel<__nv_bfloat16>, dim3((D + 255) / 256), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(g), stride_b, B, D, out, accumulate);
  return OK;
}

int b200_copy_rows(const void* src, long long src_pitch_bytes, void* dst, long long dst_pitch_bytes, long long rows,
                   long long row_bytes, void* stream) {
  B200_REQUIRE(row_bytes % 16 == 0 && src_pitch_bytes % 16 == 0 && dst_pitch_bytes % 16 == 0,
               "copy_rows: sizes must be multiples of 16 bytes");
  B200_LAUNCH(copy_rows_kernel, dim3(capped_grid(rows * (row_bytes / 16), 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint8_t*>(src), src_pitch_bytes, static_cast<uint8_t*>(dst), dst_pitch_bytes, rows, row_bytes);
  return OK;
}

int b200_colsum_partial_slices(long long rows) {
  long long s = rows / 64;    // >= 64 rows per slice, up to 4 blocks per SM
  if (s < 1) s = 1;
  if (s > 592) s = 592;
  return static_cast<int>(s);
}

int b200_colsum_partial(const void* m, long long rows, long long ld, int cols, float* partial, void* stream) {
  B200_REQUIRE(cols % 8 == 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(m) & 15) == 0,
               "colsum_partial: cols=%d / ld=%lld must be multiples of 8 and the matrix 16-byte aligned", cols, ld);
  const int S = b200_colsum_partial_slices(rows);
  B200_LAUNCH(colsum_partial_kernel, dim3(dim3((cols / 8 + 255) / 256, S)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(m), rows, ld, cols, partial);
  return OK;
}

int b200_dwconv7_pack(const float* w, float* wt, int C, void* stream) {
  B200_LAUNCH(dwconv7_pack_kernel, dim3((49 * C + 255) / 256), dim3(256), 0, static_cast<cudaStream_t>(stream), w, wt, C);
  return OK;
}

static bool dw_tiled(int H, int W, int C) { return H % kDwTile == 0 && W % kDwTile == 0 && C % kDwCh == 0; }

int b200_dwconv7(const void* in, int in_f32, const float* wt, const float* bias, const void* add, void* out, int out_f32,
                 int flip, int B, int H, int W, int C, void* stream) {
  B200_REQUIRE(C % 4 == 0, "dwconv7: C=%d must be a multiple of 4", C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total = static_cast<long long>(B) * H * ((W + 3) / 4) * (C / 4);
  const int grid = capped_grid(total, 128, 32);
  const bool tiled = dw_tiled(H, W, C);
  const long long tgrid = tiled ? static_cast<long long>(B) * (H / kDwTile) * (W / kDwTile) * (C / kDwCh) : 0;
  B200_REQUIRE(tgrid < (1ll << 31), "dwconv7: tensor too large");
  constexpr int kTileSmem = kDwHalo * kDwHalo * kDwCh * sizeof(float);
#define DW(TI, TO, F)                                                                                                     \
  if (tiled) {                                                                                                            \
    static bool cfg = false;                                                                                              \
    if (!cfg) {                                                                                                           \
      B200_CHECK_CUDA(cudaFuncSetAttribute(dwconv7_tile_kernel<TI, TO, F>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                           kTileSmem));                                                                   \
      cfg = true;                                                                                                         \
    }                                                                                                                     \
    B200_LAUNCH(dwconv7_tile_kernel<TI, TO, F>, dim3(static_cast<unsigned>(tgrid)), dim3(128), kTileSmem, st,                                                 \
        static_cast<const TI*>(in), wt, bias, static_cast<const TO*>(add), static_cast<TO*>(out), B, H, W, C);             \
  } else                                                                                                                  \
    B200_LAUNCH(dwconv7_kernel<TI, TO, F>, dim3(grid), dim3(128), 0, st, static_cast<const TI*>(in), wt, bias, static_cast<const TO*>(add), static_cast<TO*>(out), B, H, W, C)
  if (in_f32 && !out_f32 && !flip)
    DW(float, __nv_bfloat16, false);
  else if (!in_f32 && !out_f32 && flip)
    DW(__nv_bfloat16, __nv_bfloat16, true);
  else if (!in_f32 && out_f32 && flip)
    DW(__nv_bfloat16, float, true);
  else if (in_f32 && out_f32 && !flip)
    DW(float, float, false);
  else {
    set_error("dwconv7: unsupported type combination in_f32=%d out_f32=%d flip=%d", in_f32, out_f32, flip);
    return EUNSUPPORTED_;
  }
#undef DW
  return OK;
}

static int dw_wgrad_blocks_y(int B, int H) {
  long long rows = static_cast<long long>(B) * H;
  long long by = device_sm_count() * 2;
  if (by > rows) by = rows;
  return static_cast<int>(by < 1 ? 1 : by);
}

struct DwWgradPlan {
  int blocks_y, tiles_per_cta;
};
static DwWgradPlan dw_wgrad_tile_plan(int B, int H, int W, int C) {
  const long long tiles = static_cast<long long>(B) * (H / kDwTile) * (W / kDwTile);
  long long by = (6ll * device_sm_count() + C / kDwCh - 1) / (C / kDwCh);  // two waves of 3 CTAs per SM over all channel groups
  if (by > tiles) by = tiles;
  if (by < 1) by = 1;
  const int tpc = static_cast<int>((tiles + by - 1) / by);
  return DwWgradPlan{static_cast<int>((tiles + tpc - 1) / tpc), tpc};
}

size_t b200_dwconv7_wgrad_workspace_bytes(int B, int H, int W, int C) {
  const int by = dw_tiled(H, W, C) ? dw_wgrad_tile_plan(B, H, W, C).blocks_y : dw_wgrad_blocks_y(B, H);
  return static_cast<size_t>(by) * 49 * C * sizeof(float);
}

int b200_dwconv7_wgrad(const void* du, const float* x, float* dw, void* workspace, size_t workspace_bytes, int B, int H,
                       int W, int C, int accumulate, void* stream) {
  B200_REQUIRE(C % 4 == 0, "dwconv7_wgrad: C=%d must be a multiple of 4", C);
  if (dw_tiled(H, W, C)) {
    const DwWgradPlan pl = dw_wgrad_tile_plan(B, H, W, C);
    B200_REQUIRE(workspace != nullptr && workspace_bytes >= static_cast<size_t>(pl.blocks_y) * 49 * C * sizeof(float),
                 "dwconv7_wgrad: workspace too small");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    constexpr int kSmem = (kDwHalo * kDwHalo * 4 + kDwTile * kDwTile * 2) * kDwCh;  // fp32 x halo + bf16 du tile
    static bool cfg = false;
    if (!cfg) {
      B200_CHECK_CUDA(cudaFuncSetAttribute(dwconv7_wgrad_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
      cfg = true;
    }
    B200_LAUNCH(dwconv7_wgrad_tile_kernel, dim3(dim3(C / kDwCh, pl.blocks_y)), dim3(128), kSmem, st, 
        static_cast<const __nv_bfloat16*>(du), x, static_cast<float*>(workspace), B, H, W, C, pl.tiles_per_cta);
    B200_LAUNCH(dwconv7_wgrad_finalize_kernel, dim3((49 * C + 255) / 256), dim3(256), 0, st, static_cast<const float*>(workspace), pl.blocks_y, C,
                                                                        dw, accumulate);
    return OK;
  }
  const int by = dw_wgrad_blocks_y(B, H);
  B200_REQUIRE(workspace != nullptr && workspace_bytes >= static_cast<size_t>(by) * 49 * C * sizeof(float),
               "dwconv7_wgrad: workspace too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long rows = static_cast<long long>(B) * H;
  const int rpb = static_cast<int>((rows + by - 1) / by);
  B200_LAUNCH(dwconv7_wgrad_kernel, dim3(dim3((C / 4 + 31) / 32, by)), dim3(224), 0, st, static_cast<const __nv_bfloat16*>(du), x,
                                                                    static_cast<float*>(workspace), B, H, W, C, rpb);
  B200_LAUNCH(dwconv7_wgrad_finalize_kernel, dim3((49 * C + 255) / 256), dim3(256), 0, st, static_cast<const float*>(workspace), by, C, dw, accumulate);
  return OK;
}

int b200_avgpool_any(const void* x, int x_f32, float* y, int B, int HW, int C, void* stream) {
  B200_REQUIRE(C % 4 == 0, "avgpool_any: C=%d must be a multiple of 4", C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = capped_grid(static_cast<long long>(B) * (C / 4), 128);
  if (x_f32)
    B200_LAUNCH(avgpool_any_fwd_kernel<float>, dim3(grid), dim3(128), 0, st, static_cast<const float*>(x), y, B, HW, C);
  else
    B200_LAUNCH(avgpool_any_fwd_kernel<__nv_bfloat16>, dim3(grid), dim3(128), 0, st, static_cast<const __nv_bfloat16*>(x), y, B, HW, C);
  return OK;
}

int b200_colsum_prod_partial(const void* a, const void* b, long long rows, long long ld, int cols, float* partial,
                             void* stream) {
  const int S = b200_colsum_partial_slices(rows);
  B200_LAUNCH(colsum_prod_partial_kernel, dim3(dim3((cols + 63) / 64, S)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(a), static_cast<const __nv_bfloat16*>(b), rows, ld, cols, partial);
  return OK;
}

int b200_layerscale_grads(const float* G, const float* W2, const float* b2, const float* gsum, const float* gamma,
                          float* dW2, float* db2, float* dgamma, int C, int K, void* stream) {
  B200_LAUNCH(layerscale_grads_kernel, dim3(C), dim3(256), 0, static_cast<cudaStream_t>(stream), G, W2, b2, gsum, gamma, dW2, db2, dgamma, C, K);
  return OK;
}

int b200_adamw_tick(float* hyper, float beta1, float beta2, void* stream) {
  B200_LAUNCH(adamw_tick_kernel, dim3(1), dim3(32), 0, static_cast<cudaStream_t>(stream), hyper, beta1, beta2);
  return OK;
}

int b200_adamw(float* p, const float* g, float* m, float* v, const float* wd, long long n, const float* hyper,
               float beta1, float beta2, float eps, float gscale, const float* clip_coef, void* stream) {
  B200_LAUNCH(adamw_kernel, dim3(capped_grid(n, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), p, g, m, v, wd, n, hyper, beta1, beta2,
                                                                               eps, gscale, clip_coef);
  return OK;
}

int b200_grad_clip_blocks(void) { return device_sm_count() * 4; }

int b200_grad_clip_coef(const float* g, long long n, float gscale, float max_norm, float* partial, float* clip,
                        void* stream) {
  B200_REQUIRE(n > 0 && max_norm > 0.f, "grad_clip_coef: bad arguments n=%lld max_norm=%f", n, max_norm);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "grad_clip_coef: the gradient arena must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = b200_grad_clip_blocks();
  B200_LAUNCH(grad_sumsq_partial_kernel, dim3(blocks), dim3(256), 0, st, g, n, partial);
  B200_LAUNCH(grad_clip_coef_kernel, dim3(1), dim3(256), 0, st, partial, blocks, gscale, max_norm, clip);
  return OK;
}

// ---------------------------------------------------------------------------------------------------- Swin
static int wattn_check(int B, int H, int W, int nH, int shift) {
  B200_REQUIRE(B > 0 && nH > 0 && H % 7 == 0 && W % 7 == 0, "window attention: H=%d W=%d must be multiples of the 7x7 window", H, W);
  B200_REQUIRE(shift >= 0 && shift < 7, "window attention: shift %d out of range", shift);
  return OK;
}

int b200_window_attention_fwd(const void* qkv, void* out, const float* bias_tab, int masked, float* lse, int B, int H,
                              int W, int nH, int shift, float scale, void* stream) {
  int rc = wattn_check(B, H, W, nH, shift);
  if (rc) return rc;
  WAttnParams p;
  memset(&p, 0, sizeof(p));
  p.qkv = static_cast<const __nv_bfloat16*>(qkv);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.bias = bias_tab, p.masked = masked, p.lse = lse;
  p.B = B, p.H = H, p.W = W, p.nH = nH, p.shift = shift, p.scale = scale;
  static bool cfg = false;
  if (!cfg) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(wattn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWAttnFwdSmem));
    cfg = true;
  }
  // one persistent, internally pipelined CTA per SM; CTAs of a head share its window pairs round-robin
  int grid = device_sm_count() / nH * nH;
  if (grid < nH) grid = nH;
  const int total = B * (H / 7) * (W / 7);
  if (grid > (total + 1) / 2 * nH) grid = (total + 1) / 2 * nH;
  B200_LAUNCH(wattn_fwd_kernel, dim3(grid), dim3(kWAttnFwdThreads), kWAttnFwdSmem, static_cast<cudaStream_t>(stream), p);
  return OK;
}

int b200_window_attention_bwd(const void* qkv, const void* out, const void* dout, const float* bias_tab, int masked,
                              const float* lse, void* dqkv, float* dbias, int B, int H, int W, int nH, int shift,
                              float scale, void* stream) {
  int rc = wattn_check(B, H, W, nH, shift);
  if (rc) return rc;
  WAttnParams p;
  memset(&p, 0, sizeof(p));
  p.qkv = static_cast<const __nv_bfloat16*>(qkv);
  p.o = static_cast<const __nv_bfloat16*>(out);
  p.dout = static_cast<const __nv_bfloat16*>(dout);
  p.dqkv = static_cast<__nv_bfloat16*>(dqkv);
  p.bias = bias_tab, p.masked = masked, p.lse = const_cast<float*>(lse), p.dbias = dbias;
  p.B = B, p.H = H, p.W = W, p.nH = nH, p.shift = shift, p.scale = scale;
  static bool cfg = false;
  if (!cfg) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(wattn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWAttnBwdSmem));
    cfg = true;
  }
  int grid = device_sm_count() / nH * nH;
  if (grid < nH) grid = nH;
  const int total = B * (H / 7) * (W / 7);
  if (grid > (total + 1) / 2 * nH) grid = (total + 1) / 2 * nH;
  B200_LAUNCH(wattn_bwd_kernel, dim3(grid), dim3(kWAttnFwdThreads), kWAttnBwdSmem, static_cast<cudaStream_t>(stream), p);
  return OK;
}

int b200_window_bias_gather(const float* table, const long long* index, const float* mask, int nW, float* bias_tab, int nH,
                            void* stream) {
  const int nWm = mask != nullptr ? nW : 1;
  B200_REQUIRE(nH > 0 && nWm > 0, "window_bias_gather: bad sizes nH=%d nW=%d", nH, nW);
  const long long n = static_cast<long long>(nH) * nWm * 49 * 64;
  B200_LAUNCH(wattn_bias_gather_kernel, dim3(capped_grid(n, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), table, index, mask, nWm, bias_tab,
                                                                                           nH);
  return OK;
}
int b200_window_bias_scatter(const float* dbias, const long long* index, float* dtable, int nH, void* stream) {
  B200_LAUNCH(wattn_bias_scatter_kernel, dim3((nH * 49 * 49 + 255) / 256), dim3(256), 0, static_cast<cudaStream_t>(stream), dbias, index, dtable, nH);
  return OK;
}

int b200_window_partition(const void* in, void* out, int B, int H, int W, int C, int shift, int ws, int elem_bytes,
                          void* stream) {
  B200_REQUIRE(ws > 0 && H % ws == 0 && W % ws == 0, "window_partition: %dx%d not divisible by window %d", H, W, ws);
  B200_REQUIRE((static_cast<long long>(C) * elem_bytes) % 16 == 0, "window_partition: C*elem_bytes must be a multiple of 16");
  const int cvec = C * elem_bytes / 16;
  const long long nvec = static_cast<long long>(B) * H * W * cvec;
  B200_REQUIRE(nvec < (1LL << 31), "window_partition: tensor too large (%lld 16-byte vectors)", nvec);
  B200_LAUNCH(window_permute_kernel<false>, dim3(capped_grid((nvec + 3) / 4, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(in), static_cast<uint4*>(out), B, H, W, cvec, shift, ws);
  return OK;
}
int b200_window_merge(const void* in, void* out, int B, int H, int W, int C, int shift, int ws, int elem_bytes,
                      void* stream) {
  B200_REQUIRE(ws > 0 && H % ws == 0 && W % ws == 0, "window_merge: %dx%d not divisible by window %d", H, W, ws);
  B200_REQUIRE((static_cast<long long>(C) * elem_bytes) % 16 == 0, "window_merge: C*elem_bytes must be a multiple of 16");
  const int cvec = C * elem_bytes / 16;
  const long long nvec = static_cast<long long>(B) * H * W * cvec;
  B200_REQUIRE(nvec < (1LL << 31), "window_merge: tensor too large (%lld 16-byte vectors)", nvec);
  B200_LAUNCH(window_permute_kernel<true>, dim3(capped_grid((nvec + 3) / 4, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(in), static_cast<uint4*>(out), B, H, W, cvec, shift, ws);
  return OK;
}

int b200_patch_merge_ln_fwd(const float* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd,
                            int B, int H, int W, int C, float eps, void* stream) {
  B200_REQUIRE(C % 8 == 0 && 4 * C <= 2048 && H % 2 == 0 && W % 2 == 0, "patch_merge_ln: C=%d H=%d W=%d unsupported", C, H, W);
  const long long rows = static_cast<long long>(B) * (H / 2) * (W / 2);
  B200_LAUNCH(patch_merge_ln_fwd_kernel<8>, dim3(capped_grid(rows, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      x, gamma, beta, static_cast<__nv_bfloat16*>(y), mean, rstd, B, H, W, C, eps);
  return OK;
}
int b200_patch_merge_ln_bwd_blocks(long long rows) { return ln_bwd_blocks(rows); }
int b200_patch_merge_ln_bwd(const void* dy, const float* x, const float* mean, const float* rstd, const float* gamma,
                            void* dx, float* partial, int B, int H, int W, int C, void* stream) {
  B200_REQUIRE(C % 8 == 0 && 4 * C <= 2048 && H % 2 == 0 && W % 2 == 0, "patch_merge_ln_bwd: C=%d H=%d W=%d unsupported", C, H, W);
  const long long rows = static_cast<long long>(B) * (H / 2) * (W / 2);
  const size_t smem = static_cast<size_t>(8) * 2 * 4 * C * sizeof(float);
  static bool cfg = false;
  if (!cfg) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(patch_merge_ln_bwd_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 2048 * 4));
    cfg = true;
  }
  B200_LAUNCH(patch_merge_ln_bwd_kernel<8>, dim3(ln_bwd_blocks(rows)), dim3(256), smem, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dy), x, mean, rstd, gamma, static_cast<__nv_bfloat16*>(dx), partial, B, H, W, C);
  return OK;
}

}  // extern "C"

namespace {
template <int NT>
int launch_attn_fwd(const AttnFwdParams& p, int grid, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd2_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttn2SmemBytes));
    configured = true;
  }
  B200_LAUNCH(attn_fwd2_kernel<NT>, dim3(grid), dim3(kAttn2Threads), kAttn2SmemBytes, st, p);
  return OK;
}
}  // namespace

extern "C" {

int b200_attention_fwd(const void* qkv, void* out, float* lse, int B, int T, int H, float scale, void* stream) {
  B200_REQUIRE(T >= 1 && T <= 256, "attention_fwd: T=%d unsupported (1..256 tokens)", T);
  B200_REQUIRE(B > 0 && H > 0, "attention_fwd: empty problem");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AttnFwdParams p;
  memset(&p, 0, sizeof(p));
  p.B = B, p.H = H, p.T = T;
  p.Tpad = (T + 63) / 64 * 64;
  p.mblocks = (T + 127) / 128;
  p.scale = scale;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.lse = lse;
  const long long HD = static_cast<long long>(H) * 64;
  int rc;
  if ((rc = encode3(&p.q_map, qkv, 3 * HD, T, B, 128))) return rc;
  if ((rc = encode3(&p.kv_map, qkv, 3 * HD, T, B, p.Tpad))) return rc;
  if ((rc = encode3(&p.o_map, out, HD, T, B, 128))) return rc;
  const int items = B * H;
  const int grid = items < device_sm_count() ? items : device_sm_count();
  switch (p.Tpad) {
    case 64: rc = launch_attn_fwd<64>(p, grid, st); break;
    case 128: rc = launch_attn_fwd<128>(p, grid, st); break;
    case 192: rc = launch_attn_fwd<192>(p, grid, st); break;
    default: rc = launch_attn_fwd<256>(p, grid, st); break;
  }
  if (rc) return rc;
  return OK;
}

int b200_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta, void* dqkv,
                       int B, int T, int H, float scale, void* stream) {
  B200_REQUIRE(T >= 1 && T <= 256, "attention_bwd: T=%d unsupported (1..256 tokens)", T);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  {
    const long long rows = static_cast<long long>(B) * T * H;
    B200_LAUNCH(attn_delta_kernel, dim3(capped_grid(rows, 128)), dim3(256), 0, st, 
        static_cast<const __nv_bfloat16*>(dout), static_cast<const __nv_bfloat16*>(out), delta, B, T, H);
  }
  AttnBwdParams p;
  memset(&p, 0, sizeof(p));
  p.B = B, p.H = H, p.T = T;
  p.nblk = (T + 127) / 128;
  p.scale = scale;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.lse = lse;
  p.delta = delta;
  const long long HD = static_cast<long long>(H) * 64;
  int rc;
  if ((rc = encode3(&p.qkv_map, qkv, 3 * HD, T, B, 128))) return rc;
  if ((rc = encode3(&p.do_map, dout, HD, T, B, 128))) return rc;
  if ((rc = encode3(&p.dqkv_map, dqkv, 3 * HD, T, B, 128))) return rc;
  static bool cfg = false;
  if (!cfg) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnBwdSmemBytes));
    cfg = true;
  }
  B200_LAUNCH(attn_bwd_kernel, dim3(B * H), dim3(kAttnBwdThreads), kAttnBwdSmemBytes, st, p);
  return OK;
}

}  // extern "C"
