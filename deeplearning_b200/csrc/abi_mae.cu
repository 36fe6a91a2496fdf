// C-ABI entry points of the masked-autoencoder passes (see mae.cuh).  Every entry validates its shapes and pointers before
// it launches anything.
#include <stdint.h>

#include "../../include/b200cls.h"
#include "host_utils.h"
#include "mae.cuh"

using namespace b200;

namespace {
const char* mae_bad_split(int B, int P, int Nm, int D) {
  if (B < 1 || B > 65535) return "B must be in [1, 65535]";
  if (P < 2 || P > kMaeMaxP) return "P must be in [2, 1024]";
  if (Nm < 1 || Nm >= P) return "Nm must be in [1, P - 1]";
  if (D < 1 || D > 65536) return "D must be in [1, 65536]";
  return nullptr;
}
}  // namespace

#define MAE_REQUIRE_SPLIT(what, B, P, Nm, D)                                                                     \
  do {                                                                                                           \
    const char* _m = mae_bad_split(B, P, Nm, D);                                                                 \
    B200_REQUIRE(_m == nullptr, what ": %s (B=%d P=%d Nm=%d D=%d)", _m ? _m : "", B, P, Nm, D);                   \
  } while (0)

extern "C" {

int b200_mae_shuffle(const float* keys, int* ids, int* slot, int B, int P, void* stream) {
  MAE_REQUIRE_SPLIT("mae_shuffle", B, P, 1, 1);
  B200_REQUIRE(keys != nullptr && ids != nullptr && slot != nullptr, "mae_shuffle: keys, ids, slot must be non-null");
  B200_LAUNCH(mae_shuffle_kernel, dim3(B), dim3(256), 0, as_stream(stream), keys, P, ids, slot);
  return OK;
}

int b200_mae_patchify(const float* x, const int* ids, void* vis, float* tgt, int B, int C, int H, int W, int p, int Nm,
                      void* stream) {
  B200_REQUIRE(C >= 1 && p >= 1 && H >= p && W >= p && H % p == 0 && W % p == 0,
               "mae_patchify: H and W must be positive multiples of the patch size (C=%d H=%d W=%d p=%d)", C, H, W, p);
  const int P = (H / p) * (W / p);
  MAE_REQUIRE_SPLIT("mae_patchify", B, P, Nm, p * p * C);
  B200_REQUIRE(x != nullptr && ids != nullptr && vis != nullptr && tgt != nullptr,
               "mae_patchify: x, ids, vis, tgt must be non-null");
  const long long n = static_cast<long long>(B) * P * p * p * C;
  B200_LAUNCH(mae_patchify_kernel, dim3(capped_grid(n)), dim3(256), 0, as_stream(stream), x, ids, B, C, H, W, p,
              Nm, static_cast<__nv_bfloat16*>(vis), tgt);
  return OK;
}

int b200_mae_gather_rows(const float* src, long long src_rows_per_sample, int row_offset, const int* ids, int B, int P,
                         int s0, int n, int D, void* dst, int dst_f32, void* stream) {
  MAE_REQUIRE_SPLIT("mae_gather_rows", B, P, 1, D);
  B200_REQUIRE(s0 >= 0 && n >= 1 && s0 + n <= P, "mae_gather_rows: slots [s0, s0 + n) must lie in [0, P) (s0=%d n=%d P=%d)",
               s0, n, P);
  B200_REQUIRE(src_rows_per_sample >= 0 && row_offset >= 0, "mae_gather_rows: src_rows_per_sample and row_offset must be >= 0");
  B200_REQUIRE(src != nullptr && ids != nullptr && dst != nullptr, "mae_gather_rows: src, ids, dst must be non-null");
  const long long total = static_cast<long long>(B) * n * D;
  if (dst_f32)
    B200_LAUNCH(mae_gather_rows_kernel<float>, dim3(capped_grid(total)), dim3(256), 0, as_stream(stream), src,
                src_rows_per_sample, row_offset, ids, B, P, s0, n, D, static_cast<float*>(dst));
  else
    B200_LAUNCH(mae_gather_rows_kernel<__nv_bfloat16>, dim3(capped_grid(total)), dim3(256), 0, as_stream(stream),
                src, src_rows_per_sample, row_offset, ids, B, P, s0, n, D, static_cast<__nv_bfloat16*>(dst));
  return OK;
}

int b200_mae_assemble_fwd(const float* enc, const float* mask_embed, const float* dpos, const int* slot, float* dec, int B,
                          int P, int Nm, int D, void* stream) {
  MAE_REQUIRE_SPLIT("mae_assemble_fwd", B, P, Nm, D);
  B200_REQUIRE(enc != nullptr && mask_embed != nullptr && dpos != nullptr && slot != nullptr && dec != nullptr,
               "mae_assemble_fwd: enc, mask_embed, dpos, slot, dec must be non-null");
  const long long total = static_cast<long long>(B) * P * D;
  B200_LAUNCH(mae_assemble_fwd_kernel, dim3(capped_grid(total)), dim3(256), 0, as_stream(stream), enc,
              mask_embed, dpos, slot, B, P, Nm, D, dec);
  return OK;
}

int b200_mae_assemble_bwd(const void* g, const int* slot, void* g_enc, float* d_dpos, int B, int P, int Nm, int D,
                          void* stream) {
  MAE_REQUIRE_SPLIT("mae_assemble_bwd", B, P, Nm, D);
  B200_REQUIRE(g != nullptr && slot != nullptr && g_enc != nullptr && d_dpos != nullptr,
               "mae_assemble_bwd: g, slot, g_enc, d_dpos must be non-null");
  B200_LAUNCH(mae_assemble_bwd_kernel, dim3(P), dim3(256), 0, as_stream(stream),
              static_cast<const __nv_bfloat16*>(g), slot, B, P, Nm, D, static_cast<__nv_bfloat16*>(g_enc),
              d_dpos);
  return OK;
}

int b200_mae_pos_grad(const void* g, const int* slot, float* d_pos, int B, int P, int Nm, int D, void* stream) {
  MAE_REQUIRE_SPLIT("mae_pos_grad", B, P, Nm, D);
  B200_REQUIRE(g != nullptr && slot != nullptr && d_pos != nullptr, "mae_pos_grad: g, slot, d_pos must be non-null");
  B200_LAUNCH(mae_pos_grad_kernel, dim3(P + 1), dim3(256), 0, as_stream(stream),
              static_cast<const __nv_bfloat16*>(g), slot, B, P, Nm, D, d_pos);
  return OK;
}

int b200_mae_scatter_masked(const void* dh, const int* slot, void* g, int B, int P, int Nm, int D, void* stream) {
  MAE_REQUIRE_SPLIT("mae_scatter_masked", B, P, Nm, D);
  B200_REQUIRE(dh != nullptr && slot != nullptr && g != nullptr, "mae_scatter_masked: dh, slot, g must be non-null");
  const long long total = static_cast<long long>(B) * P * D;
  B200_LAUNCH(mae_scatter_masked_kernel, dim3(capped_grid(total)), dim3(256), 0, as_stream(stream),
              static_cast<const __nv_bfloat16*>(dh), slot, B, P, Nm, D, static_cast<__nv_bfloat16*>(g));
  return OK;
}

int b200_mae_mse_blocks(void) { return kMaeMseBlocks; }

int b200_mae_mse(const float* pred, const float* target, long long n, float grad_scale, void* grad, float* partial,
                 float* loss, void* stream) {
  B200_REQUIRE(n >= 1 && n <= (1ll << 40), "mae_mse: n must be in [1, 2^40] (n=%lld)", n);
  B200_REQUIRE(pred != nullptr && target != nullptr && grad != nullptr && partial != nullptr && loss != nullptr,
               "mae_mse: pred, target, grad, partial, loss must be non-null");
  B200_LAUNCH(mae_mse_kernel, dim3(kMaeMseBlocks), dim3(256), 0, as_stream(stream), pred, target, n, grad_scale,
              static_cast<__nv_bfloat16*>(grad), partial);
  B200_LAUNCH(mae_mse_finish_kernel, dim3(1), dim3(32), 0, as_stream(stream), static_cast<const float*>(partial),
              kMaeMseBlocks, 1.0 / static_cast<double>(n), loss);
  return OK;
}

}  // extern "C"
