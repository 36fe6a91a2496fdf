/* libb200cls.so - C ABI of the H100-native classification training step.
 *
 * The reference (KKKSQJ/DeepLearning) has no operator registry on this path: every op is a stock PyTorch call
 * (nn.Conv2d / nn.BatchNorm2d / nn.Linear / ... -> ATen -> cuDNN / cuBLAS, or oneDNN on CPU), and the only FFI it owns is
 * the pybind module `swin_window_process` (classification/swin_transformer/kernels/window_process/swin_window_process.cpp:70-131).
 * Each entry point below names the reference call site whose arithmetic it replaces.
 *
 * Conventions
 *   - plain C, no C++ types, no torch types; all pointers are DEVICE pointers unless stated otherwise.
 *   - activations are NHWC bf16 (channel count a multiple of 8); parameters/gradients/statistics are fp32.
 *   - the caller owns every buffer (inputs, outputs, workspaces); the library never allocates device memory.
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); no device synchronisation inside, so every call
 *     is CUDA-Graph capturable.
 *   - return 0 on success, negative on failure (B200_EINVAL / B200_EUNSUPPORTED / B200_ECUDA); b200_last_error() returns
 *     a thread-local message. Launch errors are detected with cudaPeekAtLastError only.
 */
#ifndef B200CLS_H_
#define B200CLS_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_EINVAL (-1)
#define B200_EUNSUPPORTED (-2)
#define B200_ECUDA (-3)

#define B200_ACT_NONE 0
#define B200_ACT_RELU 1
#define B200_ACT_GELU 2
#define B200_ACT_GELU_GRAD 3 /* multiply the accumulator by aux_in, which holds GELU'(pre-activation) as written through aux_out
                                by the forward GEMM with B200_ACT_GELU - backward of B200_ACT_GELU */

const char* b200_last_error(void);
int b200_abi_version(void);
/* Number of SMs of the current device (used by callers to size workspaces). */
int b200_sm_count(void);
/* Kernels launched by this library so far in this process (bench.py reports the per-step delta as gpu_launches). */
unsigned long long b200_launch_count(void);

/* ---- convolution / linear as implicit GEMM on wgmma (ksize in {1,3} pad ksize/2, stride in {1,2}; or 2x2/s2 unpadded) ----
 * forward:  y[B,Ho,Wo,Cout] = conv(x[B,H,W,Cin], w) (+bias) (act) (+residual)
 *   w        bf16 [Cout][ksize*ksize*Cin]   (b200_pack_weight mode 0)
 *   stats    optional fp32 [b200_conv2d_fwd_stats_rows()][2][Cout]: partial sum / sum of squares of y (as stored), one row
 *            per (persistent CTA group, 32-row quadrant) - a few hundred rows; feed them to b200_bn_finalize
 *   residual optional bf16, same shape as y, added after bias/act
 *   out_f32  optional fp32 [B*Ho*Wo][ld_out] - when given the result is written there instead of y (ksize 1 only)
 *   bn_scale, bn_shift  both NULL, or both set: fold BatchNorm with FIXED statistics into the epilogue,
 *            y = act(conv(x) * scale[c] + shift[c] (+ residual)) with act (0 / B200_ACT_RELU) applied after the residual
 *            add - the eval-mode forward of conv -> bn -> (+identity) -> relu (classification/resnet/models/networks.py:104-124,
 *            utils.py:61-83 `evaluate`) without any BatchNorm pass. scale / shift from b200_bn_eval_coeffs; Cout % 64 == 0,
 *            no bias, stats or out_f32.
 * replaces nn.Conv2d.forward / nn.Linear.forward: classification/resnet/models/networks.py:107,111,115,119,218;
 * classification/vision_transformer/vit_model.py:66,95,109,129,132. A linear layer is the case H=W=1, B=rows. */
int b200_conv2d_fwd(const void* x, const void* w, void* y, int B, int H, int W, int Cin, int Cout, int ksize, int stride,
                    float* stats, const float* bias, int act, const void* residual, float* out_f32, long long ld_out,
                    const float* bn_scale, const float* bn_shift, void* stream);
int b200_conv2d_fwd_stats_rows(int B, int H, int W, int Cout, int ksize, int stride);
/* Fused BatchNorm-backward mask of a dgrad GEMM (b200_conv2d_dgrad at stride 1, b200_conv2d_grouped_dgrad at stride 1,
 * b200_gemm_dual; NULL = off): the output is the gradient of relu(bn(x_raw)) - the kernel zeroes it where
 * x_raw * scale + shift <= 0 (dz) and writes the per-CTA partial rows stats[rows][2][C] = sum(dz), sum(dz * x_raw),
 * rows = b200_conv2d_fwd_stats_rows(B, H, W, C, ksize, 1) of the dx geometry: the reduce half of F.batch_norm's backward
 * (classification/resnet/models/networks.py:108,112 bn1 / bn2 under loss.backward(), utils.py:33) without a pass over the
 * gradient. Feed the rows to b200_bn_bwd_finalize, then b200_bn_bwd_apply(src_is_dz=1). The output channel count must be a
 * multiple of 64 and every field set. */
typedef struct {
  const void* x_raw;   /* bf16 raw output of the BatchNorm being differentiated, same geometry as the GEMM output */
  const float* scale;  /* b200_bn_finalize coefficients */
  const float* shift;
  float* stats;        /* [rows][2][C]: sum(dz), sum(dz * x_raw) */
} b200_bn_mask_t;
/* same convolution writing an fp32 NHWC output (+bias) through TMA - ConvNeXt downsample conv feeding the fp32 stream */
int b200_conv2d_fwd_f32(const void* x, const void* w, float* y, int B, int H, int W, int Cin, int Cout, int ksize,
                        int stride, const float* bias, void* stream);

/* data gradient: dx[B,H,W,Cin] = conv_transpose(dy[B,Ho,Wo,Cout], w) (+residual, same shape as dx; may alias dx)
 *   wd  bf16 [Cin][ksize*ksize*Cout]  (b200_pack_weight mode 1)
 *   ksize 1 & stride 2 writes only the even (h,w) pixels of dx; the others keep their previous contents.
 * replaces the cuDNN backward-data / cuBLAS dgrad autograd runs inside loss.backward() (classification/resnet/utils.py:43). */
int b200_conv2d_dgrad(const void* dy, const void* wd, void* dx, int B, int H, int W, int Cin, int Cout, int ksize,
                      int stride, const void* residual, const b200_bn_mask_t* bn_mask, void* stream);

/* weight gradient: dw[Cout][Cin][ksize][ksize] (fp32, OIHW) (+)= sum_pixels dy (x) x
 *   workspace: b200_conv2d_wgrad_workspace_bytes() bytes of scratch for the split-K partial tiles.
 *   bias_partial  optional: also produce the BIAS gradient = column sums of dy, as per-split partial sums
 *            fp32 [b200_conv2d_wgrad_splits()][2][Cout] (plane 0; fold with b200_bn_bwd_finalize). The dy tiles are summed
 *            from shared memory by four extra warps of the wgrad kernel: no separate pass over dy
 *            (replaces the bias part of loss.backward() for nn.Linear / nn.Conv2d(bias=True): vit_model.py:95,109,127-133).
 *   bias_out optional, requires bias_partial: the split reduction that follows the wgrad GEMM also folds bias_partial into
 *            the finished bias gradient bias_out[Cout] - no launch of its own.
 * replaces the cuDNN backward-filter / cuBLAS wgrad inside loss.backward(). */
int b200_conv2d_wgrad(const void* dy, const void* x, float* dw, void* workspace, size_t workspace_bytes, int B, int H,
                      int W, int Cin, int Cout, int ksize, int stride, int accumulate, float* bias_partial, float* bias_out,
                      void* stream);
size_t b200_conv2d_wgrad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, int stride);
int b200_conv2d_wgrad_splits(int B, int H, int W, int Cin, int Cout, int ksize, int stride);

/* ---- grouped 3x3 convolution (ResNeXt conv2: classification/resnet/models/networks.py:295-321, nn.Conv2d(groups=g)) ------
 * C input = C output channels, C % 64 == 0, group width Cg = C / groups in {4, 8, 16, 32, 64}, ksize 3 (pad 1), stride 1 / 2.
 * Anything else returns B200_EINVAL with a message and launches nothing.
 * forward: y[B,Ho,Wo,C] = conv(x[B,H,W,C], w) (act: 0 or B200_ACT_RELU); w bf16 [C][9*64] (b200_pack_weight mode 3);
 *   stats as for b200_conv2d_fwd, rows = b200_conv2d_grouped_fwd_stats_rows(); bn_scale / bn_shift as for b200_conv2d_fwd. */
int b200_conv2d_grouped_fwd(const void* x, const void* w, void* y, int B, int H, int W, int C, int groups, int ksize,
                            int stride, float* stats, int act, const float* bn_scale, const float* bn_shift, void* stream);
int b200_conv2d_grouped_fwd_stats_rows(int B, int H, int W, int C, int groups, int ksize, int stride);
/* data gradient dx[B,H,W,C] from dy[B,Ho,Wo,C]; wd bf16 [C][9*64] (b200_pack_weight mode 4). bn_mask as for
 * b200_conv2d_dgrad (stride 1), with rows = b200_conv2d_grouped_fwd_stats_rows(B, H, W, C, groups, 3, 1). */
int b200_conv2d_grouped_dgrad(const void* dy, const void* wd, void* dx, int B, int H, int W, int C, int groups, int ksize,
                              int stride, const b200_bn_mask_t* bn_mask, void* stream);
/* weight gradient dw[C][C/groups][3][3] (fp32, OIHW) (+)= sum_pixels dy (x) x within each group; workspace =
 * b200_conv2d_grouped_wgrad_workspace_bytes() bytes (0 for an unsupported shape). */
int b200_conv2d_grouped_wgrad(const void* dy, const void* x, float* dw, void* workspace, size_t workspace_bytes, int B,
                              int H, int W, int C, int groups, int ksize, int stride, int accumulate, void* stream);
size_t b200_conv2d_grouped_wgrad_workspace_bytes(int B, int H, int W, int C, int groups, int ksize, int stride);

/* ---- general GEMM with strided pixel views (transformer layers, patch embedding) ----------------------------------------
 * out[pixel, n] = epilogue( sum_k a[pixel, k] * w[n, k] ), pixels = dim[0] x dim[1] x dim[2] (w fastest), channel stride 1.
 * `a` and `out` must have identical pixel extents; strides are in elements and let `out`/`residual` be token-offset or
 * batch-broadcast views (e.g. ViT: rows 1.. of [B,197,D], residual = pos_embed with batch stride 0).
 * replaces nn.Linear / PatchEmbed conv + the surrounding bias / GELU / residual-add elementwise ops of
 * classification/vision_transformer/vit_model.py:66,95,109,127-133,159-160. */
typedef struct {
  const void* base;     /* first element of the view (bf16 unless stated otherwise) */
  long long dim[3];     /* pixel extents (w, h, n); use 1 for unused dims */
  long long stride[3];  /* element strides of the pixel dims */
} b200_view_t;

typedef struct {
  const void* w;               /* bf16 [N][K] (b200_pack_weight mode 0) */
  int N, K;
  const float* bias;           /* [N] or NULL */
  const float* colscale;       /* [N] multiplier applied after bias/act, before the residual (ConvNeXt layer scale), or NULL */
  int act;                     /* B200_ACT_* */
  int out_f32;                 /* 1: `out` is an fp32 tensor (residual stream) */
  const b200_view_t* residual; /* added after bias/act, or NULL */
  int residual_f32;
  const b200_view_t* aux_out;  /* second bf16 output kept for the backward pass, or NULL: with act == GELU it receives the derivative
                                  GELU'(pre-activation) (evaluated together with the value), otherwise the pre-activation itself */
  const b200_view_t* aux_in;   /* act == B200_ACT_GELU_GRAD: the GELU'(pre-activation) tensor a forward call wrote through aux_out */
  float* stats;                /* optional per-32-row-slab column sum / sum of squares, or NULL */
  const float* rowscale;       /* stochastic depth: per-SAMPLE multiplier [n_samples] applied after bias/act/colscale and
                                  before the residual (drop_path: convNext/models/networks.py:11-26, vit_model.py:12-40,
                                  swin_transformer.py:282,285), or NULL */
  int rows_per_sample;         /* output pixels per sample (sample = flat pixel index / rows_per_sample) */
} b200_gemm_args_t;

int b200_gemm_ex(const b200_view_t* a, const b200_view_t* out, const b200_gemm_args_t* args, void* stream);

/* ---- LayerNorm over the last dim, one warp per row (vit_model.py:194 eps 1e-6; swin_transformer.py:509 eps 1e-5) ------------
 * x is fp32 (x_f32) or bf16, y bf16; mean/rstd [rows] are kept for the backward pass.
 * backward: dx = rstd*(dy*gamma - mean(dy*gamma) - xhat*mean(dy*gamma*xhat)) (+ add), dx/add fp32 or bf16;
 * partial[b200_layernorm_bwd_blocks()][2][C] = per-block (sum dy, sum dy*xhat), folded by b200_bn_bwd_finalize. */
int b200_layernorm_fwd(const void* x, int x_f32, const float* gamma, const float* beta, void* y, int y_f32, float* mean,
                       float* rstd, long long rows, int C, float eps, void* stream);
int b200_layernorm_bwd_blocks(long long rows, int C);
int b200_layernorm_bwd(const void* dy, const void* x, int x_f32, const float* mean, const float* rstd, const float* gamma,
                       const void* add, void* dx, int dx_f32, float* partial, long long rows, int C, void* stream);

/* ---- ViT patch embedding helpers (vit_model.py:56-66,244-250) ---------------------------------------------------------------
 * patchify: NCHW fp32 -> bf16 [B*(H/ps)*(W/ps)][Cin*ps*ps] with k = c*ps*ps + kh*ps + kw (= conv weight.view(D,-1) order) */
int b200_patchify_nchw(const float* x, void* a, int B, int Cin, int H, int W, int ps, void* stream);
int b200_cls_row(const float* cls, const float* pos, float* tokens, int B, int T, int D, void* stream);
int b200_batch_rowsum(const void* g, int g_f32, long long stride_b, int B, int D, float* out, int accumulate,
                      void* stream);
/* strided 2-D copy (16-byte granularity), e.g. gathering the class-token rows of a [B,T,D] tensor */
int b200_copy_rows(const void* src, long long src_pitch_bytes, void* dst, long long dst_pitch_bytes, long long rows,
                   long long row_bytes, void* stream);
/* bias gradients of tall matrices: partial[b200_colsum_partial_slices(rows)][2][cols], folded by b200_bn_bwd_finalize */
int b200_colsum_partial_slices(long long rows);
int b200_colsum_partial(const void* m, long long rows, long long ld, int cols, float* partial, void* stream);

/* ---- multi-head self-attention, head_dim 64, T <= 256 tokens, with wgmma (vit_model.py:95-108) ---------------------------------
 * qkv bf16 [B][T][3][H][64] (the qkv Linear output as is), out bf16 [B][T][H*64], lse fp32 [B][H][T].
 * backward: dqkv bf16 [B][T][3][H][64]; delta fp32 [B][H][T] is scratch. Scores / probabilities never touch HBM. */
int b200_attention_fwd(const void* qkv, void* out, float* lse, int B, int T, int H, float scale, void* stream);
int b200_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta, void* dqkv,
                       int B, int T, int H, float scale, void* stream);

/* ---- Swin (classification/swin_transformer/models/swin_transformer.py) -----------------------------------------------------
 * Shifted-window attention, 7x7 windows, head_dim 32, with wgmma. qkv bf16 [B][H][W][3*nH*32] in natural (un-rolled) pixel
 * order; torch.roll / window_partition / window_reverse (:251-280) are folded into the gather / scatter addressing.
 * bias_tab = b200_window_bias_gather(): fp32 [nH][masked ? nW : 1][49 (query i)][64 (key j, 49 used)] holding
 *   log2(e) x ( relative_position_bias_table[relative_position_index[i][j]][h] (:131-134) plus, for shifted blocks, the
 *   attn_mask buffer value mask[w][i][j] (0 / -100, :215-238, :142-147) ) - one small launch per block and step; a soft-max thread
 *   (one query row) fetches its 256-byte row with 13 vector loads. masked = 1 when a mask was folded in.
 * Two windows are processed per tensor-core step (block-diagonal 128x128 score tile). lse fp32 [B][nW][nH][49] is the
 * base-2 log-sum-exp of the (scaled, biased) score rows - an opaque hand-over from forward to backward.
 * backward: dqkv same layout as qkv; dbias dense [nH][49 i][49 j] must be zeroed by the caller (atomics), then
 * b200_window_bias_scatter adds it into the table gradient. */
int b200_window_attention_fwd(const void* qkv, void* out, const float* bias_tab, int masked, float* lse, int B, int H,
                              int W, int nH, int shift, float scale, void* stream);
int b200_window_attention_bwd(const void* qkv, const void* out, const void* dout, const float* bias_tab, int masked,
                              const float* lse, void* dqkv, float* dbias, int B, int H, int W, int nH, int shift,
                              float scale, void* stream);
int b200_window_bias_gather(const float* table, const long long* index, const float* mask, int nW, float* bias_tab, int nH,
                            void* stream);
int b200_window_bias_scatter(const float* dbias, const long long* index, float* dtable, int nH, void* stream);
/* The reference's own operator FFI (kernels/window_process/swin_window_process.cpp:70-131), any 2/4-byte element type:
 *   partition: out[B*nW][ws][ws][C] = window_partition(roll(in[B][H][W][C], shifts=(shift, shift)))   (forward)
 *   merge:     out[B][H][W][C] = roll(window_reverse(in[B*nW][ws][ws][C]), shifts=(shift, shift))
 * roll_and_window_partition_backward(g, s) == merge(g, -s), window_merge_and_roll_backward(g, s) == partition(g, -s). */
int b200_window_partition(const void* in, void* out, int B, int H, int W, int C, int shift, int ws, int elem_bytes,
                          void* stream);
int b200_window_merge(const void* in, void* out, int B, int H, int W, int C, int shift, int ws, int elem_bytes,
                      void* stream);
/* PatchMerging front half (:333-343): 2x2 gather-concat of the fp32 stream + LayerNorm(4C) -> bf16 [B*H/2*W/2][4C] */
int b200_patch_merge_ln_fwd(const float* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd,
                            int B, int H, int W, int C, float eps, void* stream);
int b200_patch_merge_ln_bwd_blocks(long long rows);
int b200_patch_merge_ln_bwd(const void* dy, const float* x, const float* mean, const float* rstd, const float* gamma,
                            void* dx, float* partial, int B, int H, int W, int C, void* stream);

/* ---- ConvNeXt (classification/convNext/models/networks.py:92-105,160-165) ---------------------------------------------------
 * 7x7 depthwise conv, pad 3, NHWC: out = bias + sum_taps wt[tap][c]*in[...]; wt = tap-major [49][C] copy (b200_dwconv7_pack).
 * flip != 0 correlates with the flipped kernel (data gradient); `add` (same type as out) is summed into the result. */
int b200_dwconv7_pack(const float* w, float* wt, int C, void* stream);
int b200_dwconv7(const void* in, int in_f32, const float* wt, const float* bias, const void* add, void* out, int out_f32,
                 int flip, int B, int H, int W, int C, void* stream);
/* weight gradient dw [C][49] (+)= sum du * x_shifted; workspace = b200_dwconv7_wgrad_workspace_bytes() */
size_t b200_dwconv7_wgrad_workspace_bytes(int B, int H, int W, int C);
int b200_dwconv7_wgrad(const void* du, const float* x, float* dw, void* workspace, size_t workspace_bytes, int B, int H,
                       int W, int C, int accumulate, void* stream);
/* global average pool of [B][HW][C] (fp32 or bf16) -> fp32 [B][C] */
int b200_avgpool_any(const void* x, int x_f32, float* y, int B, int HW, int C, void* stream);
/* partial[b200_colsum_partial_slices(rows)][2][cols] of column sums of a*b (b optional): layer-scale / bias gradients */
int b200_colsum_prod_partial(const void* a, const void* b, long long rows, long long ld, int cols, float* partial,
                             void* stream);
/* layer-scale gradients from the unscaled pwconv2 weight gradient G [C][K]: dgamma, dW2 = gamma*G, db2 = gamma*gsum */
int b200_layerscale_grads(const float* G, const float* W2, const float* b2, const float* gsum, const float* gamma,
                          float* dW2, float* db2, float* dgamma, int C, int K, void* stream);
/* fused AdamW over flat fp32 arenas; wd = per-element weight decay (0 for the no-decay group, convNext/utils.py:144-166);
 * hyper = device {lr, 1-beta1^t, 1-beta2^t, beta1^t, beta2^t}; b200_adamw_tick advances t by one on the device
 * (initialise hyper to {lr, 0, 0, 1, 1}), so the whole update is CUDA-graph replayable. */
int b200_adamw_tick(float* hyper, float beta1, float beta2, void* stream);
int b200_adamw(float* p, const float* g, float* m, float* v, const float* wd, long long n, const float* hyper,
               float beta1, float beta2, float eps, float gscale, const float* clip_coef, void* stream);
/* Global-norm gradient clipping of the Swin recipe (torch.nn.utils.clip_grad_norm_: swin_transformer/utils/torch_utils.py:303-317,
 * main.py:197) without rewriting the gradients: clip[0] = min(1, max_norm / (gscale*||g||_2 + 1e-6)), clip[1] = the norm.
 * The optimizer entries multiply their gradient scale by clip_coef[0] when the pointer is non-null.
 * partial: fp32 scratch of b200_grad_clip_blocks() floats; g must be 16-byte aligned. */
int b200_grad_clip_blocks(void);
int b200_grad_clip_coef(const float* g, long long n, float gscale, float max_norm, float* partial, float* clip, void* stream);

/* ---- BatchNorm2d (train: batch statistics, eval: running statistics) ----------------------------------------------------
 * replaces nn.BatchNorm2d + nn.ReLU (+ residual add) of Bottleneck.forward, classification/resnet/models/networks.py:108-124 */
/* partial[T][2][C] column reductions run on a 2-D grid; `scratch` (b200_reduce_scratch_bytes(T, C) bytes, its first 1024
 * bytes zero on first use - the kernel leaves them zero) carries the slice sums and a ticket counter. One per stream. */
size_t b200_reduce_scratch_bytes(int T, int C);
int b200_bn_finalize(const float* partial, int T, int C, double count, const float* gamma, const float* beta, float eps,
                     float momentum, float* running_mean, float* running_var, long long* num_batches_tracked,
                     float* mean, float* invstd, float* scale, float* shift, void* scratch, size_t scratch_bytes,
                     void* stream);
int b200_bn_eval_coeffs(int C, const float* gamma, const float* beta, const float* running_mean,
                        const float* running_var, float eps, float* scale, float* shift, void* stream);
/* y = act(x*scale[c]+shift[c] (+residual)); x,y,residual bf16 [rows][C] */
int b200_bn_apply(const void* x, const void* residual, void* y, const float* scale, const float* shift, long long rows,
                  int C, int relu, void* stream);
/* backward pass 1: partial[b200_bn_bwd_blocks()][2][C] = per-block sums of dz and dz*x (raw x), dz = g*relu_mask;
 * b200_bn_bwd_finalize(mean, invstd) turns the second into sum(dz*xhat).
 *   y_out (optional) = saved post-activation output used for the mask; otherwise the mask is recomputed from x.
 *   dz_out (optional) receives dz as bf16. */
int b200_bn_bwd_reduce(const void* g, const void* x, const void* y_out, void* dz_out, const float* scale,
                       const float* shift, int relu, long long rows, int C, float* partial, void* stream);
int b200_bn_bwd_blocks(long long rows, int C);
int b200_bn_bwd_finalize(const float* partial, int T, int C, double count, float* dgamma, float* dbeta, int accumulate,
                         float* m1, float* m2, const float* mean, const float* invstd, void* scratch,
                         size_t scratch_bytes, void* stream);
/* backward pass 2: dx = scale*(dz - m1 - xhat*m2); g_is_dz != 0 means `g` already holds dz (mask applied). */
int b200_bn_bwd_apply(const void* g, const void* x, const void* y_out, int g_is_dz, void* dx, const float* scale,
                      const float* shift, const float* mean, const float* invstd, const float* m1, const float* m2,
                      int relu, long long rows, int C, void* stream);
/* ---- pooling ----------------------------------------------------------------------------------------------------------
 * stem: y[B,Ho,Wo,C] = maxpool3x3/s2/p1(relu(x*scale+shift)); idx = one byte arg-max tap per element (uint64 per 8 ch)
 * replaces bn1 -> relu -> maxpool, classification/resnet/models/networks.py:207-209 */
int b200_bn_relu_maxpool_fwd(const void* x, void* y, void* idx, const float* scale, const float* shift, int B, int H,
                             int W, int C, void* stream);
int b200_maxpool_bwd(const void* g_out, const void* idx, void* g_in, int B, int H, int W, int C, void* stream);
/* global average pool, classification/resnet/models/networks.py:216 */
int b200_avgpool_fwd(const void* x, void* y, int B, int HW, int C, void* stream);
int b200_avgpool_bwd(const void* gy, void* gx, int B, int HW, int C, void* stream);

/* ---- loss / misc ------------------------------------------------------------------------------------------------------
 * CrossEntropyLoss(mean) forward+backward; classification/resnet/train.py:104, utils.py:39-42.
 *   loss_rows[B] per-sample loss; dlogits (optional) bf16 [B][ld_d] = (softmax - onehot)*gscale; correct (optional) int[B] */
int b200_softmax_xent(const float* logits, long long ld, const long long* labels, int B, int N, float gscale,
                      float* loss_rows, void* dlogits, long long ld_d, int* correct, void* stream);
/* the same with a target DISTRIBUTION per sample: soft_targets fp32 [B][ld_soft] (timm SoftTargetCrossEntropy behind
 * Mixup / CutMix, classification/swin_transformer/main.py:111-113) or, with soft_targets == NULL, hard labels smoothed by
 * `smoothing` (LabelSmoothingCrossEntropy, main.py:114-115):  loss_b = sum_c t_c (lse - x_c),
 * dlogits = (softmax * sum_c t_c - t) * gscale; correct[b] compares the arg-max with the label (or the arg-max of t). */
int b200_softmax_xent_soft(const float* logits, long long ld, const long long* labels, const float* soft_targets,
                           long long ld_soft, float smoothing, int B, int N, float gscale, float* loss_rows, void* dlogits,
                           long long ld_d, int* correct, void* stream);
int b200_mean(const float* v, int n, float* out, void* stream);
int b200_colsum_bf16(const void* m, long long rows, long long ld, int cols, float* out, int accumulate, void* stream);

/* weight packing fp32 OIHW -> bf16 GEMM operand; mode 0: [O][taps*I] (pitch ld_dst), mode 1: [I][taps*O];
 * grouped convolution weight [C][Cg][taps] (O = C, I = Cg): mode 3 = block-diagonal forward operand [C][taps*64],
 * mode 4 = block-diagonal dgrad operand [C][taps*64] (transposed within each group, taps unflipped like mode 1) */
int b200_pack_weight(const float* src, void* dst, int O, int I, int taps, int mode, long long ld_dst, void* stream);
/* all weights of a model in one launch: table[n][10] int64 {src, dst, O, I, taps, mode, ld_dst, first_block, rows_out,
 * oscale (optional fp32 [O] multiplier per output channel, 0 = none)}; mode 0 = forward / wgrad operand [O][tap*I+i],
 * 1 = dgrad operand [I][tap*O+o], 2 = space-to-depth stem operand [O][256] of a [O][3][7][7] kernel, 3 / 4 = grouped
 * forward / dgrad operands as for b200_pack_weight (rows_out = O = C) */
int b200_pack_weights_multi(const void* table, int n_entries, int total_blocks, void* stream);
int b200_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream);
int b200_cast_bf16_to_f32(const void* src, float* dst, long long n, void* stream);
/* stem im2col from the user's NCHW fp32 batch: a bf16 [B*Ho*Wo][ldk], k=(kh*KW+kw)*Cin+c (networks.py:206 conv1 7x7/2) */
int b200_im2col_nchw(const float* x, void* a, int B, int Cin, int H, int W, int KH, int KW, int stride, int pad,
                     int ldk, void* stream);

/* Space-to-depth stem - the conv1 7x7 / stride 2 / pad 3 of ResNet (classification/resnet/models/networks.py:150,206) without a
 * patch matrix: b200_stem_s2d writes z bf16 [B][H/2+3][W/2+3][16] (zero-padded input, 2x2 pixel phase folded into 12 + 4
 * zero channels); the conv is then a 4x4 / stride-1 conv whose four x-taps are 64 contiguous elements of z, presented to the
 * implicit-GEMM kernels through a tensor map with overlapping rows. w = b200_pack_weights_multi mode 2 ([64][256]).
 * y bf16 [B][Ho][Wo][64] (Ho = H/2), stats as for b200_conv2d_fwd (rows: b200_conv2d_fwd_stats_rows(B, Ho, Wo, 64, 3, 1)).
 * wgrad: g fp32 [64][64][4] scratch gradient in the operand layout -> b200_stem_s2d_wgrad_relayout -> dW [64][3][7][7]. */
int b200_stem_s2d(const float* x, void* z, int B, int H, int W, void* stream);
/* GPU input pipeline (SURVEY 8(f)-1; replaces the CPU ToTensor + Normalize of classification/resnet/train.py:46-71):
 * decoded uint8 NHWC [B][H][W][3] -> the same space-to-depth operand (ResNet), or -> normalised fp32 NCHW (other families).
 * mean3 / std3 are HOST pointers to 3 floats each (the reference's [0.485, 0.456, 0.406] / [0.229, 0.224, 0.225]). */
int b200_stem_s2d_u8(const void* x_u8_nhwc, void* z, int B, int H, int W, const float* mean3, const float* std3, void* stream);
int b200_normalize_u8_nhwc(const void* x_u8_nhwc, float* y_nchw, int B, int H, int W, const float* mean3, const float* std3,
                           void* stream);
int b200_stem_s2d_conv_fwd(const void* z, const void* w, void* y, float* stats, int B, int Ho, int Wo, void* stream);
size_t b200_stem_s2d_conv_wgrad_workspace_bytes(int B, int Ho, int Wo);
int b200_stem_s2d_conv_wgrad(const void* dy, const void* z, float* g, void* workspace, size_t workspace_bytes, int B, int Ho,
                             int Wo, void* stream);
int b200_stem_s2d_wgrad_relayout(const float* g, float* dw, int accumulate, void* stream);

/* stem weight gradient [Cout][ldk] (k = tap*Cin + c, as produced by b200_conv2d_wgrad on the patch matrix) -> OIHW */
int b200_stem_wgrad_relayout(const float* src, float* dst, int Cout, int Cin, int taps, int ldk, int accumulate,
                              void* stream);

/* fused SGD(momentum) over a flat fp32 arena; torch.optim.SGD semantics (classification/resnet/train.py:96).
 * lr_dev (optional device float*) overrides lr, so a captured CUDA graph can follow the reference's LambdaLR schedule. */
int b200_sgd_momentum(float* p, const float* g, float* buf, long long n, float lr, const float* lr_dev, float momentum,
                      float weight_decay, float gscale, int first_step, const float* clip_coef, void* stream);

/* ---- train-mode BatchNorm folded through a 1x1 convolution (ResNet bottleneck conv3 -> bn3 -> +identity -> ReLU,
 * classification/resnet/models/networks.py:116-124): the wide conv output is never written; see csrc/bn_algebra.cuh.
 * forward: G = y2^T y2 (b200_conv2d_wgrad(y2, y2)), s = colsum(y2) -> b200_bn_gram_stats -> scale / shift ->
 *          b200_conv1x1_bn_act_fwd: y = relu(conv1x1(y2, w) * scale + shift + residual)       (w bf16 [Cout][Cin])
 * backward: dz = relu-mask * gradient (b200_conv1x1_dgrad_masked of the NEXT block, with its per-CTA column sums),
 *          D = dz^T y2 (b200_conv2d_wgrad) -> b200_bn_conv1x1_bwd -> dgamma, dbeta, dW, wcat [Cin][Cout + Cin] bf16, bias [Cin]
 *          -> b200_gemm_dual: g2 = [dz | y2] wcat^T + bias                                     */
int b200_bn_gram_stats(const float* G, const float* s, const void* w_bf16, int N, int K, double count, const float* gamma,
                       const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                       long long* num_batches_tracked, float* mean, float* invstd, float* scale, float* shift, void* stream);
int b200_conv1x1_bn_act_fwd(const void* x, const void* w, const float* scale, const float* shift, const void* residual,
                            void* y, long long pixels, int Cin, int Cout, int relu, void* stream);
/* y[pixels][Cout] = conv1x1(x, w) * scale + shift: the downsample branch conv -> BatchNorm (networks.py:118-119, 196-199) with the
 * batch statistics from b200_bn_gram_stats of its (compact, see b200_subsample2) input; no residual, no ReLU */
int b200_conv1x1_bn_fwd(const void* x, const void* w, const float* scale, const float* shift, void* y, long long pixels,
                        int Cin, int Cout, void* stream);
/* xs[b][i][j][:] = x[b][2i][2j][:] (the pixels a 1x1 / stride-2 convolution reads);  gx[b][2i][2j][:] += gs[b][i][j][:] */
int b200_subsample2(const void* x, void* xs, int B, int H, int W, int C, void* stream);
int b200_add_even_pixels(void* gx, const void* gs, int B, int H, int W, int C, void* stream);
/* dx[pixels][Cin] = (mask_src > 0) ? (dy[pixels][Cout] * wd^T + residual) : 0  (wd bf16 [Cin][Cout], b200_pack_weight mode 1);
 * stats fp32 [b200_conv1x1_dgrad_masked_stats_rows()][2][Cin]: per-CTA column sums (plane 0) of dx as stored */
int b200_conv1x1_dgrad_masked_stats_rows(long long pixels, int Cin, int Cout);
int b200_conv1x1_dgrad_masked(const void* dy, const void* wd, void* dx, long long pixels, int Cin, int Cout,
                              const void* residual, const void* mask_src, float* stats, void* stream);
/* dz_partial fp32 [T][2][N] (plane 0 = partial column sums of dz); scratch: b200_bn_conv1x1_bwd_scratch_bytes(N, K) bytes;
 * tickets: 64 uint32 counters, zero before the first call (the kernel leaves them zero) */
size_t b200_bn_conv1x1_bwd_scratch_bytes(int N, int K);
int b200_bn_conv1x1_bwd(const float* dz_partial, int T, const float* D, const float* G, const float* s, const void* w_bf16,
                        const float* w_f32, int N, int K, double count, const float* gamma, const float* mean,
                        const float* invstd, float* dgamma, float* dbeta, float* dW, int accumulate, void* wcat, float* bias,
                        void* scratch, size_t scratch_bytes, void* tickets, void* stream);
/* out[pixels][N] (bf16) = [a0[pixels][K0] | a1[pixels][K1]] * wcat[N][K0 + K1]^T + bias[N]; bn_mask as for b200_conv2d_dgrad */
int b200_gemm_dual(const void* a0, int K0, const void* a1, int K1, const void* wcat, const float* bias, void* out,
                   long long pixels, int N, const b200_bn_mask_t* bn_mask, void* stream);

/* ---- stochastic depth / pre_logits helpers -------------------------------------------------------------------------------
 * y[b, :] = x[b, :] * scale[b] over bf16 samples of elems_per_sample elements: the gradient entering a residual branch whose
 * forward was scaled per sample by drop_path (convNext/models/networks.py:11-26, vit_model.py:12-40, swin_transformer.py:282,285;
 * the forward scaling itself is b200_gemm_args_t::rowscale).  Samples with scale 0 are not read. */
int b200_rowscale_bf16(const void* x, const float* scale, void* y, long long n_samples, long long elems_per_sample,
                       void* stream);
/* ViT pre_logits = Linear + Tanh on the class-token row (vit_model.py:218-221): t = tanh(u) fp32 (kept for the backward) and
 * its bf16 copy (operand of the classifier GEMM); backward du = dt * (1 - t^2), bf16 in / out. */
int b200_tanh_fwd(const float* u, float* t, void* t_bf16, long long n, void* stream);
int b200_tanh_bwd(const void* dt_bf16, const float* t, void* du_bf16, long long n, void* stream);

/* ---- squeeze-and-excitation tail of an SE-ResNet block: SELayer (classification/seNet/models/se_module.py:15-19) between
 * the last BatchNorm and the residual add of SEBottleneck / SEBasicBlock (se_resnet.py:74-84 / :32-42):
 *     y = relu(u * gate[b][ch] + identity),  u = c * scale + shift,  gate = sigmoid(W2 relu(W1 mean_p(u)))
 * c bf16 [B][HW][C] is the raw conv output, scale / shift the BatchNorm coefficients (batch statistics in train mode, running
 * statistics in eval mode); per-image vectors are fp32 [B][C] (csum, pool, gate, A, R, dp) or [B][Cr] (h, dh); w1 = fc.0.weight
 * fp32 [Cr][C], w2 = fc.2.weight fp32 [C][Cr].  Scope: C % 64 == 0, 1 <= Cr <= 256, HW >= 1, 1 <= B <= 65535; other shapes
 * return B200_EINVAL with a message and launch nothing.  All sums are fp32 in a fixed order (no atomics).
 * forward:  squeeze  csum = sum_p c, pool = csum / HW * scale + shift          (one read of c)
 *           excite   h = relu(pool w1^T), gate = sigmoid(h w2^T)               (two small launches, fp32 CUDA cores)
 *           apply    y = relu(u * gate + identity)                              (one read of c and identity, one write of y)
 * backward (g = dL/dy):
 *           reduce   dz = g * [y > 0] (bf16, the identity branch's gradient), A = sum_p dz, R = sum_p dz * c
 *           coeffs   da = (scale R + shift A) gate (1 - gate), dW2 = da^T h, dh = (da w2) [h > 0], dW1 = dh^T pool,
 *                    dp = dh w1, dbeta = sum_b (gate A + dp), dgamma = invstd (sum_b (gate R + dp csum / HW) - mean dbeta),
 *                    m1 = dbeta / M, m2 = dgamma / M (M = B HW); dw1, dw2, dgamma, dbeta are written, not accumulated
 *           apply    dc = scale (dz gate + dp / HW - m1 - (c - mean) invstd m2)  (bf16) */
int b200_se_squeeze(const void* c, const float* scale, const float* shift, float* csum, float* pool, int B, int HW, int C,
                    void* stream);
int b200_se_excite(const float* pool, const float* w1, const float* w2, float* h, float* gate, int B, int C, int Cr,
                   void* stream);
int b200_se_apply(const void* c, const void* identity, void* y, const float* scale, const float* shift, const float* gate,
                  int B, int HW, int C, void* stream);
int b200_se_bwd_reduce(const void* g, const void* y, const void* c, void* dz, float* A, float* R, int B, int HW, int C,
                       void* stream);
int b200_se_bwd_coeffs(const float* A, const float* R, const float* csum, const float* pool, const float* h,
                       const float* gate, const float* w1, const float* w2, const float* scale, const float* shift,
                       const float* mean, const float* invstd, int B, int HW, int C, int Cr, float* dh, float* dp,
                       float* dw1, float* dw2, float* dgamma, float* dbeta, float* m1, float* m2, void* stream);
int b200_se_bwd_apply(const void* dz, const void* c, void* dc, const float* gate, const float* dp, const float* scale,
                      const float* mean, const float* invstd, const float* m1, const float* m2, int B, int HW, int C,
                      void* stream);

/* ---- RepVGG block (classification/RepVGG/models/repvgg.py RepVGGBlock, train form):
 *     y = relu(bn_dense(conv3x3(x)) + bn_1x1(conv1x1(x)) [+ bn_identity(x)])
 * c3 / c1 are the raw bf16 outputs of the two convolutions and x the block input, each [rows] rows of C channels at a row
 * pitch ld3 / ld1 / ldx (elements): the stem keeps [c3 | c1] in one [rows][2C] GEMM output.  co_* are fp32 [4][C] =
 * {mean, invstd, scale, shift} of a BatchNorm (b200_bn_finalize's outputs, contiguous), m_* fp32 [2][C] = {m1, m2} of
 * b200_bn_bwd_finalize.  The identity operands (x, co_id, m_id, dx) are all NULL for a block without an identity branch.
 * Scope: C a multiple of 8 in [8, 8192], rows >= 1, pitches multiples of 8 and >= C, 16-byte aligned pointers; anything
 * else returns B200_EINVAL with a message and launches nothing.  All sums are fp32 in a fixed order (no atomics).
 * partial_rows: T, the number of [2][C] partial rows the apply (stats) and reduce passes write for (rows, C); -1 if invalid.
 * apply:      y [rows][C] = relu(c3 s3 + c1 s1 [+ x s_id] + t3 + t1 [+ t_id]); stats (optional) fp32 [T][2][C] = sums of the
 *             stored bf16 y and y^2 (the batch statistics of the next block's identity BatchNorm, for b200_bn_finalize)
 * bwd_reduce: dz = g [y > 0]; partial fp32 [nb][T][2][C] (nb = 2, or 3 with x): branch b = dense, 1x1, identity holds
 *             {sum dz, sum dz * input_b}, the rows b200_bn_bwd_finalize reads with that branch's mean / invstd
 * bwd_apply:  dc_b = scale_b (dz - m1_b - (input_b - mean_b) invstd_b m2_b) for every branch (dz recomputed from g and y);
 *             dc3, dc1, dx are written at the pitches of c3, c1, x
 * fold:       eval-mode re-parameterisation (get_equivalent_kernel_bias, repvgg.py): wp bf16 [O][ldk], k = tap * I + i,
 *             = W3 t3 + pad(W1) t1 [+ I t_id] (zero for k >= 9 I), bias fp32 [O] = sum_b (beta_b - mean_b t_b),
 *             t = gamma / sqrt(running_var + eps); the identity BatchNorm (all four pointers NULL if absent) needs O == I */
int b200_repvgg_partial_rows(long long rows, int C);
int b200_repvgg_apply(const void* c3, long long ld3, const void* c1, long long ld1, const void* x, long long ldx,
                      const float* co3, const float* co1, const float* co_id, void* y, long long rows, int C, float* stats,
                      void* stream);
int b200_repvgg_bwd_reduce(const void* g, const void* y, const void* c3, long long ld3, const void* c1, long long ld1,
                           const void* x, long long ldx, long long rows, int C, float* partial, void* stream);
int b200_repvgg_bwd_apply(const void* g, const void* y, const void* c3, long long ld3, const void* c1, long long ld1,
                          const void* x, long long ldx, const float* co3, const float* m3, const float* co1, const float* m1,
                          const float* co_id, const float* m_id, void* dc3, void* dc1, void* dx, long long rows, int C,
                          void* stream);
int b200_repvgg_fold(const float* w3, const float* w1, const float* gamma3, const float* beta3, const float* mean3,
                     const float* var3, float eps3, const float* gamma1, const float* beta1, const float* mean1,
                     const float* var1, float eps1, const float* gamma_id, const float* beta_id, const float* mean_id,
                     const float* var_id, float eps_id, int O, int I, int ldk, void* wp, float* bias, void* stream);

/* ---- EfficientNet MBConv block (classification/efficientNet/models/network.py MBConv:176-242, SELayer:126-145,
 * ConvBNAction:97-122).  Activations are NHWC bf16 [B][H][W][C] (rows = B*H*W), 16-byte aligned; scale / shift are the
 * fp32 [C] coefficients of a BatchNorm (batch statistics in train mode, running statistics in eval mode), co fp32 [4][C] =
 * {mean, invstd, scale, shift} (b200_bn_finalize's outputs, contiguous), m fp32 [2][C] = {m1, m2} of b200_bn_bwd_finalize;
 * per-image vectors are fp32 [B][C] or [B][Cr].  Partial rows are fp32 [T][2][C] = {sum v, sum v * input}, the layout
 * b200_bn_finalize / b200_bn_bwd_finalize read.  Scope: C a multiple of 8 in [8, 8192], 1 <= B <= 65535, HW >= 1,
 * 1 <= Cr <= 256, depthwise k in {3, 5} with padding k/2 and stride 1 or 2 (any H, W >= 1); anything else returns
 * B200_EINVAL with a message and launches nothing.  All sums are fp32 in a fixed order (no atomics).
 * The streaming passes (silu_bn_bwd_reduce, tail_bwd_reduce) write b200_repvgg_partial_rows(rows, C) partial rows: they
 * share the RepVGG passes' row geometry.
 * dw_partial_rows: T of dw_fwd (rows = output pixels) and dw_dgrad (rows = input pixels); -1 if invalid
 * dw_fwd:      the dwconv of ConvBNAction(groups=C) (network.py:113-120): d = dwconv_kxk(in), w = the fp32 weight [C][k*k];
 *              in = silu(x * scale + shift) when scale is given (the previous BatchNorm + SiLU applied on load), else x;
 *              stats (optional) = sums of the stored d and d^2
 * dw_dgrad:    g_in = the data gradient of dw_fwd for dd = dL/dd; with scale (x = the raw input): dx = g_in silu'(x scale +
 *              shift) and partial = {sum dx, sum dx x}; otherwise dx = g_in (+ residual)
 * dw_wgrad:    dw fp32 [C][k*k] = sum over pixels of dd * in (in as in dw_fwd), written (not accumulated); ws is scratch of
 *              dw_wgrad_workspace_bytes
 * silu_bn_squeeze: SELayer.avg_pool / EfficientNet.avgpool (network.py:143, :359) of silu(d * scale + shift): pool fp32
 *              [B][C]; with mask fp32 [B][C] also out16 bf16 [B][C] = pool * mask (the classifier dropout, :340)
 * excite_fwd:  SELayer.fc (network.py:134-139): hpre = pool w1^T + b1 [B][Cr], gate = sigmoid(silu(hpre) w2^T + b2) [B][C];
 *              w1 fp32 [Cr][C], w2 fp32 [C][Cr]
 * excite_bwd:  from s = sum_p dL/da * silu(u) [B][C] (gate_reduce): dgp = s gate (1 - gate) [B][C] and dhp = (dgp w2)
 *              silu'(hpre) [B][Cr] (scratch the caller provides), dw1 [Cr][C], db1 [Cr], dw2 [C][Cr], db2 [C] (written,
 *              not accumulated) and dpool = dhp w1 [B][C]
 * gate_apply:  SELayer.forward's x * y (network.py:145): a = silu(d * scale + shift) * gate
 * gate_reduce: s [B][C] = sum_p da * silu(d * scale + shift)
 * silu_bn_bwd_reduce: dz = (da * gate + dpool / HW) * silu'(d * scale + shift) (da and gate optional together) stored bf16,
 *              partial = {sum dz, sum dz d}
 * tail_apply:  project BatchNorm, DropPath and shortcut (network.py:237-242): y = (c * scale + shift) * rs[b] (+ residual);
 *              rs fp32 [B] (the per-sample drop-connect multiplier) and residual optional
 * tail_bwd_reduce: dz = g * rs[b] stored bf16 (dz and rs both or neither; without them dz = g), partial = {sum dz, sum dz c}
 * bn_bwd_apply_dz: train-mode BatchNorm backward apply from a stored dz: dc = scale (dz - m1 - (c - mean) invstd m2) */
int b200_dw_partial_rows(long long rows, int C);
int b200_dw_fwd(const void* x, const float* w, const float* scale, const float* shift, void* d, float* stats, int B, int H,
                int W, int C, int k, int stride, void* stream);
int b200_dw_dgrad(const void* dd, const float* w, const void* x, const float* scale, const float* shift,
                  const void* residual, void* dx, float* partial, int B, int H, int W, int C, int k, int stride,
                  void* stream);
size_t b200_dw_wgrad_workspace_bytes(int B, int H, int W, int C, int k, int stride);
int b200_dw_wgrad(const void* dd, const void* x, const float* scale, const float* shift, float* dw, void* ws,
                  size_t ws_bytes, int B, int H, int W, int C, int k, int stride, void* stream);
int b200_silu_bn_squeeze(const void* d, const float* scale, const float* shift, const float* mask, float* pool,
                         void* out16, int B, int HW, int C, void* stream);
int b200_excite_fwd(const float* pool, const float* w1, const float* b1, const float* w2, const float* b2, float* hpre,
                    float* gate, int B, int C, int Cr, void* stream);
int b200_excite_bwd(const float* s, const float* pool, const float* hpre, const float* gate, const float* w1,
                    const float* w2, float* dgp, float* dhp, float* dw1, float* db1, float* dw2, float* db2, float* dpool,
                    int B, int C, int Cr, void* stream);
int b200_gate_apply(const void* d, const float* scale, const float* shift, const float* gate, void* a, int B, int HW, int C,
                    void* stream);
int b200_gate_reduce(const void* da, const void* d, const float* scale, const float* shift, float* s, int B, int HW, int C,
                     void* stream);
int b200_silu_bn_bwd_reduce(const void* da, const float* gate, const float* dpool, const void* d, const float* scale,
                            const float* shift, void* dz, float* partial, int B, int HW, int C, void* stream);
int b200_tail_apply(const void* c, const float* scale, const float* shift, const float* rs, const void* residual, void* y,
                    int B, int HW, int C, void* stream);
int b200_tail_bwd_reduce(const void* g, const float* rs, const void* c, void* dz, float* partial, int B, int HW, int C,
                         void* stream);
int b200_bn_bwd_apply_dz(const void* dz, const void* c, const float* co, const float* m, void* dc, long long rows, int C,
                         void* stream);

/* ---- VGG (classification/vggNet/models/network.py) passes the convolution GEMMs do not cover, and torch.optim.Adam.
 * Activations are NHWC bf16 [B][H][W][C], 16-byte aligned; scale / shift fp32 [C] are a BatchNorm's coefficients (batch
 * statistics in train mode, running statistics in eval mode).  Scope: 1 <= B <= 65535, C a multiple of 8 in [8, 8192]
 * (the adaptive pool: a multiple of 64), H, W >= 1 (the 2x2 pool: >= 2); anything else returns B200_EINVAL with a message
 * and launches nothing.  All sums are fp32 in a fixed order (no atomics).
 * pool_fwd:  MaxPool2d(2, 2) (floor mode) of x (plain: x = relu(conv + b), written by the GEMM) or of relu(x * scale + shift)
 *            (BN: x = the raw conv output; the full-resolution activation is never stored): y [B][H/2][W/2][C]; idx
 *            (optional, 8-byte aligned) one byte per element of y = the window tap 0..3 (row-major) of the maximum, ties
 *            resolved to the first
 * pool_bwd:  dx [B][H][W][C] = the pooled gradient g at the arg-max pixel of each window where the activation was positive,
 *            0 elsewhere (also in the row / column of an odd H / W that no window covers).  Plain: y = the pooled output
 *            (the mask is y > 0), c / scale / shift / partial NULL.  BN: y NULL, the mask is c * scale + shift > 0 and
 *            partial fp32 [pool_partial_rows][2][C] = {sum dx, sum dx c}, the rows b200_bn_bwd_finalize reads
 * avgpool7:  AdaptiveAvgPool2d((7, 7)) + torch.flatten: y bf16 [B][C * 49] with k = c * 49 + i * 7 + j, bin i spanning
 *            rows floor(i H / 7) .. ceil((i + 1) H / 7) - 1 (likewise columns); _bwd scatters gy [B][C * 49] back to
 *            gx [B][H][W][C]
 * dropout_fwd: y = x * mask over n elements (mask fp32, 0 or 1 / (1 - p)); n a multiple of 8
 * dropout_bwd: the backward of h = dropout(relu(pre)) from the stored h: dx = h > 0 ? g * scale : 0, scale = 1 / (1 - p)
 * adam:      torch.optim.Adam (L2 weight decay added to the gradient, every element decays by weight_decay) over flat
 *            fp32 arenas: g' = g gscale [clip_coef[0]] + weight_decay p, then b200_adamw's moments and bias-corrected step;
 *            hyper as b200_adamw's, advanced by b200_adamw_tick */
int b200_vgg_pool_partial_rows(int B, int H, int W, int C);
int b200_vgg_pool_fwd(const void* x, const float* scale, const float* shift, void* y, void* idx, int B, int H, int W, int C,
                      void* stream);
int b200_vgg_pool_bwd(const void* g, const void* idx, const void* y, const void* c, const float* scale, const float* shift,
                      void* dx, float* partial, int B, int H, int W, int C, void* stream);
int b200_vgg_avgpool7_fwd(const void* x, void* y, int B, int H, int W, int C, void* stream);
int b200_vgg_avgpool7_bwd(const void* gy, void* gx, int B, int H, int W, int C, void* stream);
int b200_vgg_dropout_fwd(const void* x, const float* mask, void* y, long long n, void* stream);
int b200_vgg_dropout_bwd(const void* g, const void* h, float scale, void* dx, long long n, void* stream);
int b200_adam(float* p, const float* g, float* m, float* v, long long n, const float* hyper, float beta1, float beta2,
              float eps, float weight_decay, float gscale, const float* clip_coef, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200CLS_H_ */
