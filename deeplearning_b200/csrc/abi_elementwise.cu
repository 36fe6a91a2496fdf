// C-ABI entry points for the HBM-bound passes (see elementwise.cuh).
#include <stdint.h>
#include <string.h>

#include "../../include/b200cls.h"
#include "elementwise.cuh"
#include "bn_algebra.cuh"
#include "host_utils.h"

using namespace b200;

namespace {
inline bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }
inline int reduce_slices(int T) {
  int s = T / 64;
  if (s < 1) s = 1;
  if (s > 64) s = 64;
  return s;
}

struct BnBwdPlan {
  int blocks, rows_per_block;
};
BnBwdPlan plan_bn_bwd(long long rows, int C) {
  const int cvec = C / 8;
  const int rpi = 256 / cvec;
  long long blocks = static_cast<long long>(device_sm_count()) * 8;
  long long rpb = (rows + blocks - 1) / blocks;
  rpb = ((rpb + rpi - 1) / rpi) * rpi;
  if (rpb < rpi) rpb = rpi;
  blocks = (rows + rpb - 1) / rpb;
  return BnBwdPlan{static_cast<int>(blocks), static_cast<int>(rpb)};
}
}  // namespace

extern "C" {

const char* b200_last_error(void) { return get_error(); }
int b200_abi_version(void) { return 3; }
int b200_sm_count(void) { return device_sm_count(); }
unsigned long long b200_launch_count(void) { return g_launch_count; }

size_t b200_reduce_scratch_bytes(int T, int C) {
  return 1024 + static_cast<size_t>(reduce_slices(T)) * 2 * C * sizeof(double);
}

int b200_bn_finalize(const float* partial, int T, int C, double count, const float* gamma, const float* beta, float eps,
                     float momentum, float* running_mean, float* running_var, long long* num_batches_tracked,
                     float* mean, float* invstd, float* scale, float* shift, void* scratch, size_t scratch_bytes,
                     void* stream) {
  B200_REQUIRE(T > 0 && C > 0 && count > 0, "bn_finalize: bad sizes T=%d C=%d", T, C);
  B200_REQUIRE(C <= 256 * 32, "bn_finalize: C=%d exceeds 8192", C);
  B200_REQUIRE(scratch != nullptr && scratch_bytes >= b200_reduce_scratch_bytes(T, C), "bn_finalize: scratch too small");
  B200_LAUNCH(bn_finalize_kernel, dim3(dim3((C + 31) / 32, reduce_slices(T))), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      partial, T, C, count, gamma, beta, eps, momentum, running_mean, running_var, num_batches_tracked, mean, invstd,
      scale, shift, scratch);
  return OK;
}

int b200_bn_eval_coeffs(int C, const float* gamma, const float* beta, const float* running_mean,
                        const float* running_var, float eps, float* scale, float* shift, void* stream) {
  B200_LAUNCH(bn_eval_coeffs_kernel, dim3((C + 255) / 256), dim3(256), 0, static_cast<cudaStream_t>(stream), C, gamma, beta, running_mean,
                                                                                       running_var, eps, scale, shift);
  return OK;
}

int b200_bn_apply(const void* x, const void* residual, void* y, const float* scale, const float* shift, long long rows,
                  int C, int relu, void* stream) {
  B200_REQUIRE(C % 8 == 0, "bn_apply: C=%d must be a multiple of 8", C);
  const long long nvec = rows * (C / 8);
  B200_LAUNCH(bn_apply_kernel, dim3(capped_grid(nvec)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(x), static_cast<const uint4*>(residual), static_cast<uint4*>(y), scale, shift, nvec,
      C / 8, relu);
  return OK;
}

int b200_bn_bwd_blocks(long long rows, int C) {
  if (C % 8 != 0 || !pow2(C / 8) || C / 8 > 256) {
    set_error("bn_bwd_blocks: C=%d must be 8*2^k <= 2048", C);
    return -1;
  }
  return plan_bn_bwd(rows, C).blocks;
}

int b200_bn_bwd_reduce(const void* g, const void* x, const void* y_out, void* dz_out, const float* scale,
                       const float* shift, int relu, long long rows, int C, float* partial, void* stream) {
  B200_REQUIRE(C % 8 == 0 && pow2(C / 8) && C / 8 <= 256, "bn_bwd_reduce: C=%d must be 8*2^k <= 2048", C);
  const BnBwdPlan pl = plan_bn_bwd(rows, C);
  B200_LAUNCH(bn_bwd_reduce_kernel, dim3(pl.blocks), dim3(256), 256 * 17 * sizeof(float), static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(g), static_cast<const uint4*>(x), static_cast<const uint4*>(y_out),
      static_cast<uint4*>(dz_out), scale, shift, relu, rows, C / 8, pl.rows_per_block, partial);
  return OK;
}

int b200_bn_bwd_finalize(const float* partial, int T, int C, double count, float* dgamma, float* dbeta, int accumulate,
                         float* m1, float* m2, const float* mean, const float* invstd, void* scratch,
                         size_t scratch_bytes, void* stream) {
  B200_REQUIRE(T > 0 && C > 0 && C <= 256 * 32, "bn_bwd_finalize: bad sizes T=%d C=%d", T, C);
  B200_REQUIRE(scratch != nullptr && scratch_bytes >= b200_reduce_scratch_bytes(T, C), "bn_bwd_finalize: scratch too small");
  B200_LAUNCH(bn_bwd_finalize_kernel, dim3(dim3((C + 31) / 32, reduce_slices(T))), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      partial, T, C, count, dgamma, dbeta, accumulate, m1, m2, mean, invstd, scratch);
  return OK;
}

int b200_bn_bwd_apply(const void* g, const void* x, const void* y_out, int g_is_dz, void* dx, const float* scale,
                      const float* shift, const float* mean, const float* invstd, const float* m1, const float* m2,
                      int relu, long long rows, int C, void* stream) {
  B200_REQUIRE(rows >= 1 && C >= 8 && C % 8 == 0 && C <= kRvMaxC,
               "bn_bwd_apply: need rows >= 1 and C a multiple of 8 in [8, 8192] (rows=%lld C=%d)", rows, C);
  B200_REQUIRE(aligned16(g) && aligned16(x) && aligned16(dx) && aligned16(scale) && aligned16(shift) &&
                   aligned16(mean) && aligned16(invstd) && aligned16(m1) && aligned16(m2) &&
                   (y_out == nullptr || aligned16(y_out)),
               "bn_bwd_apply: g, x, dx, scale, shift, mean, invstd, m1, m2 (and y_out) must be non-null and 16-byte "
               "aligned");
  const RvGeom gm = repvgg_geom(rows, C);
  B200_LAUNCH(bn_bwd_apply_kernel, dim3(gm.blocks, gm.nchunk), dim3(256), 0,
      static_cast<cudaStream_t>(stream), static_cast<const uint4*>(g), static_cast<const uint4*>(x),
      static_cast<const uint4*>(y_out), g_is_dz, static_cast<uint4*>(dx), scale, shift, mean, invstd, m1, m2, relu, rows,
      C / 8, gm.rows_per_block, gm.gpc);
  return OK;
}

int b200_bn_relu_maxpool_fwd(const void* x, void* y, void* idx, const float* scale, const float* shift, int B, int H,
                             int W, int C, void* stream) {
  B200_REQUIRE(C % 8 == 0, "maxpool: C=%d must be a multiple of 8", C);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long nvec = static_cast<long long>(B) * Ho * Wo * (C / 8);
  B200_REQUIRE(static_cast<long long>(B) * H * W * (C / 8) < (1LL << 32), "maxpool: tensor too large");
  B200_LAUNCH(bn_relu_maxpool_fwd_kernel, dim3(capped_grid(nvec)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(x), static_cast<uint4*>(y), static_cast<unsigned long long*>(idx), scale, shift, B, H, W,
      C / 8);
  return OK;
}

int b200_maxpool_bwd(const void* g_out, const void* idx, void* g_in, int B, int H, int W, int C, void* stream) {
  B200_REQUIRE(C % 8 == 0, "maxpool_bwd: C=%d must be a multiple of 8", C);
  B200_REQUIRE(static_cast<long long>(B) * H * W * (C / 8) < (1LL << 32), "maxpool_bwd: tensor too large");
  const long long nvec = static_cast<long long>(B) * ((H - 1) / 2 + 1) * ((W - 1) / 2 + 1) * (C / 8);   // 2x2 input blocks
  B200_LAUNCH(maxpool_bwd_kernel, dim3(capped_grid(nvec)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(g_out), static_cast<const unsigned long long*>(idx), static_cast<uint4*>(g_in), B, H, W,
      C / 8);
  return OK;
}

int b200_avgpool_fwd(const void* x, void* y, int B, int HW, int C, void* stream) {
  B200_REQUIRE(C % 8 == 0, "avgpool: C=%d must be a multiple of 8", C);
  const long long nvec = static_cast<long long>(B) * (C / 8);
  B200_LAUNCH(avgpool_fwd_kernel, dim3(capped_grid(nvec, 128)), dim3(128), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(x), static_cast<uint4*>(y), B, HW, C / 8);
  return OK;
}
int b200_avgpool_bwd(const void* gy, void* gx, int B, int HW, int C, void* stream) {
  B200_REQUIRE(C % 8 == 0, "avgpool_bwd: C=%d must be a multiple of 8", C);
  const long long nvec = static_cast<long long>(B) * HW * (C / 8);
  B200_LAUNCH(avgpool_bwd_kernel, dim3(capped_grid(nvec)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(gy), static_cast<uint4*>(gx), B, HW, C / 8);
  return OK;
}

int b200_softmax_xent(const float* logits, long long ld, const long long* labels, int B, int N, float gscale,
                      float* loss_rows, void* dlogits, long long ld_d, int* correct, void* stream) {
  B200_REQUIRE(B > 0 && N > 0, "softmax_xent: empty input");
  B200_LAUNCH(softmax_xent_kernel, dim3(B), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      logits, ld, labels, N, gscale, loss_rows, static_cast<__nv_bfloat16*>(dlogits), ld_d, correct,
      static_cast<const float*>(nullptr), 0ll, 0.f);
  return OK;
}

int b200_softmax_xent_soft(const float* logits, long long ld, const long long* labels, const float* soft_targets,
                           long long ld_soft, float smoothing, int B, int N, float gscale, float* loss_rows, void* dlogits,
                           long long ld_d, int* correct, void* stream) {
  B200_REQUIRE(B > 0 && N > 0, "softmax_xent_soft: empty input");
  B200_REQUIRE(soft_targets != nullptr || labels != nullptr, "softmax_xent_soft: soft targets or labels are required");
  B200_REQUIRE(smoothing >= 0.f && smoothing < 1.f, "softmax_xent_soft: smoothing %f outside [0, 1)", smoothing);
  B200_LAUNCH(softmax_xent_kernel, dim3(B), dim3(256), 0, static_cast<cudaStream_t>(stream),
      logits, ld, labels, N, gscale, loss_rows, static_cast<__nv_bfloat16*>(dlogits), ld_d, correct, soft_targets, ld_soft,
      smoothing);
  return OK;
}

int b200_mean(const float* v, int n, float* out, void* stream) {
  B200_LAUNCH(mean_kernel, dim3(1), dim3(256), 0, static_cast<cudaStream_t>(stream), v, n, out);
  return OK;
}

int b200_colsum_bf16(const void* m, long long rows, long long ld, int cols, float* out, int accumulate, void* stream) {
  B200_LAUNCH(colsum_kernel, dim3((cols + 63) / 64), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(m), rows, ld, cols, out, accumulate);
  return OK;
}

int b200_pack_weight(const float* src, void* dst, int O, int I, int taps, int mode, long long ld_dst, void* stream) {
  B200_REQUIRE(mode == 0 || mode == 1 || mode == 3 || mode == 4, "pack_weight: mode %d", mode);
  B200_REQUIRE(mode < 3 || (O % 64 == 0 && I > 0 && 64 % I == 0),
               "pack_weight: grouped modes need C %% 64 == 0 and a group width dividing 64 (C=%d, Cg=%d)", O, I);
  const long long rows = mode == 1 ? I : O;
  const long long need = static_cast<long long>(taps) * (mode == 0 ? I : (mode == 1 ? O : 64));
  B200_REQUIRE(ld_dst >= need, "pack_weight: ld_dst %lld < %lld", ld_dst, need);
  B200_LAUNCH(pack_weight_kernel, dim3(capped_grid(rows * ld_dst)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      src, static_cast<__nv_bfloat16*>(dst), O, I, taps, mode, ld_dst);
  return OK;
}

int b200_pack_weights_multi(const void* table, int n_entries, int total_blocks, void* stream) {
  B200_REQUIRE(table != nullptr && n_entries > 0 && total_blocks > 0, "pack_weights_multi: empty table");
  B200_LAUNCH(pack_weights_multi_kernel, dim3(total_blocks), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const long long*>(table), n_entries);
  return OK;
}

int b200_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream) {
  B200_LAUNCH(cast_f32_bf16_kernel, dim3(capped_grid(n)), dim3(256), 0, static_cast<cudaStream_t>(stream), src, static_cast<__nv_bfloat16*>(dst),
                                                                                  n);
  return OK;
}
int b200_cast_bf16_to_f32(const void* src, float* dst, long long n, void* stream) {
  B200_LAUNCH(cast_bf16_f32_kernel, dim3(capped_grid(n)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(src), dst, n);
  return OK;
}

int b200_im2col_nchw(const float* x, void* a, int B, int Cin, int H, int W, int KH, int KW, int stride, int pad,
                     int ldk, void* stream) {
  B200_REQUIRE(ldk % 8 == 0 && ldk >= KH * KW * Cin, "im2col: ldk=%d must be a multiple of 8 and >= %d", ldk,
               KH * KW * Cin);
  const int Ho = (H + 2 * pad - KH) / stride + 1, Wo = (W + 2 * pad - KW) / stride + 1;
  const size_t smem = static_cast<size_t>(Cin) * KH * (W + 2 * pad) * sizeof(float) + static_cast<size_t>(ldk) * sizeof(int);
  B200_REQUIRE(smem <= 48 * 1024, "im2col: staged rows need %zu bytes of shared memory (> 48 KB)", smem);
  const int threads = (ldk / 8) * (256 / (ldk / 8) > 0 ? 256 / (ldk / 8) : 1);  // a multiple of the k-octet count
  B200_REQUIRE(ldk / 8 <= 256, "im2col: ldk=%d too large", ldk);
  B200_LAUNCH(im2col_nchw_kernel, dim3(B * Ho), dim3(threads), smem, static_cast<cudaStream_t>(stream), x, static_cast<uint4*>(a), B, Cin, H, W,
                                                                               KH, KW, stride, pad, Ho, Wo, ldk);
  return OK;
}

int b200_stem_wgrad_relayout(const float* src, float* dst, int Cout, int Cin, int taps, int ldk, int accumulate,
                              void* stream) {
  const long long total = static_cast<long long>(Cout) * Cin * taps;
  B200_LAUNCH(stem_wgrad_relayout_kernel, dim3(capped_grid(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), src, dst, Cout, Cin, taps,
                                                                                            ldk, accumulate);
  return OK;
}

int b200_sgd_momentum(float* p, const float* g, float* buf, long long n, float lr, const float* lr_dev, float momentum,
                      float weight_decay, float gscale, int first_step, const float* clip_coef, void* stream) {
  B200_LAUNCH(sgd_momentum_kernel, dim3(capped_grid(n)), dim3(256), 0, static_cast<cudaStream_t>(stream), p, g, buf, n, lr, lr_dev, momentum,
                                                                               weight_decay, gscale, first_step, clip_coef);
  return OK;
}

int b200_stem_s2d(const float* x, void* z, int B, int H, int W, void* stream) {
  B200_REQUIRE(B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "stem_s2d: H=%d W=%d must be even", H, W);
  const long long total = static_cast<long long>(B) * (H / 2 + 3) * (W / 2 + 3);
  B200_LAUNCH(stem_s2d_kernel, dim3(capped_grid(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), x, static_cast<uint4*>(z), B, H, W);
  return OK;
}

int b200_stem_s2d_wgrad_relayout(const float* g, float* dw, int accumulate, void* stream) {
  B200_LAUNCH(stem_s2d_wgrad_relayout_kernel, dim3((64 * 3 * 49 + 255) / 256), dim3(256), 0, static_cast<cudaStream_t>(stream), g, dw, accumulate);
  return OK;
}

int b200_rowscale_bf16(const void* x, const float* scale, void* y, long long n_samples, long long elems_per_sample,
                       void* stream) {
  B200_REQUIRE(n_samples > 0 && elems_per_sample > 0 && elems_per_sample % 8 == 0,
               "rowscale_bf16: elems_per_sample=%lld must be a positive multiple of 8", elems_per_sample);
  const long long nvec = n_samples * (elems_per_sample / 8);
  B200_LAUNCH(rowscale_bf16_kernel, dim3(capped_grid(nvec)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(x), scale, static_cast<uint4*>(y), nvec, elems_per_sample / 8);
  return OK;
}

int b200_tanh_fwd(const float* u, float* t, void* t_bf16, long long n, void* stream) {
  B200_REQUIRE(n > 0, "tanh_fwd: empty input");
  B200_LAUNCH(tanh_fwd_kernel, dim3(capped_grid(n)), dim3(256), 0, static_cast<cudaStream_t>(stream), u, t, static_cast<__nv_bfloat16*>(t_bf16), n);
  return OK;
}

int b200_tanh_bwd(const void* dt_bf16, const float* t, void* du_bf16, long long n, void* stream) {
  B200_REQUIRE(n > 0, "tanh_bwd: empty input");
  B200_LAUNCH(tanh_bwd_kernel, dim3(capped_grid(n)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dt_bf16), t, static_cast<__nv_bfloat16*>(du_bf16), n);
  return OK;
}

int b200_bn_gram_stats(const float* G, const float* s, const void* w_bf16, int N, int K, double count, const float* gamma,
                       const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                       long long* num_batches_tracked, float* mean, float* invstd, float* scale, float* shift, void* stream) {
  B200_REQUIRE(N > 0 && K >= 32 && K <= 256 && K % 32 == 0 && count > 0, "bn_gram_stats: N=%d K=%d (K must be 32..256, multiple of 32)", N, K);
  const size_t smem = static_cast<size_t>(32 + 8 + 1) * K * sizeof(float);
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(bn_gram_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 41 * 256 * 4));
    B200_CHECK_CUDA(cudaFuncSetAttribute(bn_conv1x1_bwd_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 40 * 256 * 4));
    configured = true;
  }
  B200_LAUNCH(bn_gram_stats_kernel, dim3((N + 7) / 8), dim3(256), smem, static_cast<cudaStream_t>(stream), 
      G, s, static_cast<const __nv_bfloat16*>(w_bf16), N, K, count, gamma, beta, eps, momentum, running_mean, running_var,
      num_batches_tracked, mean, invstd, scale, shift);
  return OK;
}

size_t b200_bn_conv1x1_bwd_scratch_bytes(int N, int K) {
  const size_t tiles = static_cast<size_t>(K / 32) * (K / 32);
  return static_cast<size_t>(2) * N * sizeof(float) + static_cast<size_t>(kAlgebraSlices) * tiles * 33 * 32 * sizeof(float);
}

int b200_bn_conv1x1_bwd(const float* dz_partial, int T, const float* D, const float* G, const float* s, const void* w_bf16,
                        const float* w_f32, int N, int K, double count, const float* gamma, const float* mean,
                        const float* invstd, float* dgamma, float* dbeta, float* dW, int accumulate, void* wcat, float* bias,
                        void* scratch, size_t scratch_bytes, void* tickets, void* stream) {
  B200_REQUIRE(N > 0 && T > 0 && K >= 32 && K <= 256 && K % 32 == 0 && count > 0, "bn_conv1x1_bwd: N=%d K=%d T=%d unsupported", N, K, T);
  B200_REQUIRE(scratch != nullptr && scratch_bytes >= b200_bn_conv1x1_bwd_scratch_bytes(N, K) && tickets != nullptr,
               "bn_conv1x1_bwd: scratch too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(bn_gram_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 41 * 256 * 4));
    B200_CHECK_CUDA(cudaFuncSetAttribute(bn_conv1x1_bwd_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 40 * 256 * 4));
    configured = true;
  }
  float2* coef = static_cast<float2*>(scratch);
  float* partial = reinterpret_cast<float*>(static_cast<char*>(scratch) + static_cast<size_t>(2) * N * sizeof(float));
  B200_LAUNCH(bn_conv1x1_bwd_rows_kernel, dim3((N + 7) / 8), dim3(256), static_cast<size_t>(32 + 8) * K * sizeof(float), st, 
      dz_partial, T, D, G, s, static_cast<const __nv_bfloat16*>(w_bf16), w_f32, N, K, count, gamma, mean, invstd, dgamma, dbeta,
      dW, accumulate, static_cast<__nv_bfloat16*>(wcat), coef);
  B200_LAUNCH(bn_conv1x1_bwd_m_kernel, dim3(dim3(K / 32, K / 32, kAlgebraSlices)), dim3(256), 0, st, 
      coef, static_cast<const __nv_bfloat16*>(w_bf16), w_f32, N, K, static_cast<__nv_bfloat16*>(wcat), bias,
      static_cast<unsigned int*>(tickets), partial);
  return OK;
}

int b200_stem_s2d_u8(const void* x_u8_nhwc, void* z, int B, int H, int W, const float* mean3, const float* std3, void* stream) {
  B200_REQUIRE(B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "stem_s2d_u8: H=%d W=%d must be even", H, W);
  B200_REQUIRE(mean3 != nullptr && std3 != nullptr, "stem_s2d_u8: host mean / std (3 floats each) required");
  float a[3], b[3];
  for (int c = 0; c < 3; ++c) {
    a[c] = 1.0f / (255.0f * std3[c]);
    b[c] = -mean3[c] / std3[c];
  }
  const long long total = static_cast<long long>(B) * (H / 2 + 3) * (W / 2 + 3);
  B200_LAUNCH(stem_s2d_u8_kernel, dim3(capped_grid(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const unsigned char*>(x_u8_nhwc), static_cast<uint4*>(z), B, H, W, a[0], a[1], a[2], b[0], b[1], b[2]);
  return OK;
}

int b200_normalize_u8_nhwc(const void* x_u8_nhwc, float* y_nchw, int B, int H, int W, const float* mean3, const float* std3,
                           void* stream) {
  B200_REQUIRE(B > 0 && H > 0 && W > 0 && mean3 != nullptr && std3 != nullptr, "normalize_u8_nhwc: bad arguments");
  float a[3], b[3];
  for (int c = 0; c < 3; ++c) {
    a[c] = 1.0f / (255.0f * std3[c]);
    b[c] = -mean3[c] / std3[c];
  }
  B200_LAUNCH(u8_nhwc_to_f32_nchw_kernel, dim3(capped_grid(static_cast<long long>(B) * H * W)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const unsigned char*>(x_u8_nhwc), y_nchw, B, H, W, a[0], a[1], a[2], b[0], b[1], b[2]);
  return OK;
}

int b200_subsample2(const void* x, void* xs, int B, int H, int W, int C, void* stream) {
  B200_REQUIRE(C % 8 == 0 && B > 0 && H > 0 && W > 0, "subsample2: C=%d must be a multiple of 8", C);
  B200_REQUIRE(static_cast<long long>(B) * H * W * (C / 8) < (1LL << 32), "subsample2: tensor too large");
  const long long total = static_cast<long long>(B) * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
  B200_LAUNCH(subsample2_kernel, dim3(capped_grid(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const uint4*>(x), static_cast<uint4*>(xs), B, H, W, C / 8);
  return OK;
}

int b200_add_even_pixels(void* gx, const void* gs, int B, int H, int W, int C, void* stream) {
  B200_REQUIRE(C % 8 == 0 && B > 0 && H > 0 && W > 0, "add_even_pixels: C=%d must be a multiple of 8", C);
  B200_REQUIRE(static_cast<long long>(B) * H * W * (C / 8) < (1LL << 32), "add_even_pixels: tensor too large");
  const long long total = static_cast<long long>(B) * ((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
  B200_LAUNCH(add_even_pixels_kernel, dim3(capped_grid(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<uint4*>(gx), static_cast<const uint4*>(gs), B, H, W, C / 8);
  return OK;
}

}  // extern "C"
