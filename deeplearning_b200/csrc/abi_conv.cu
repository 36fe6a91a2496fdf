// C-ABI entry points for the wgmma implicit-GEMM kernels (forward / dgrad / wgrad). Host side only builds tensor maps,
// tap tables and tile geometry; see conv_gemm.cuh / wgrad_gemm.cuh for the device code.
#include <string.h>
#include "../../include/b200cls.h"
#include "conv_gemm.cuh"
#include "conv1x1_stream.cuh"
#include "conv_tap64.cuh"
#include "host_utils.h"
#include "wgrad_gemm.cuh"

using namespace b200;

namespace {

// wgmma shared-memory descriptor strides (bytes): K-major operands of conv_gemm / conv_tap64, MN-major operands of wgrad_gemm
constexpr uint32_t kFwdDescLbo = 16, kFwdDescSbo = 1024;
constexpr uint32_t kWgDescLbo = 8192, kWgDescSbo = 1024, kWgDescKstep = 2048;

struct Box3 {
  int b1, b2, b3;
};

// Factor P pixels (power of two) into a (w, h, n) box minimising padded work; ties -> longer w, then longer h.
Box3 choose_box(long long d1, long long d2, long long d3, int P) {
  Box3 best{P, 1, 1};
  double best_cost = -1;
  for (int b1 = 1; b1 <= P; b1 <<= 1) {
    for (int b2 = 1; b1 * b2 <= P; b2 <<= 1) {
      const int b3 = P / (b1 * b2);
      if (b1 > 256 || b2 > 256 || b3 > 256) continue;
      const double c1 = double((d1 + b1 - 1) / b1) * b1, c2 = double((d2 + b2 - 1) / b2) * b2,
                   c3 = double((d3 + b3 - 1) / b3) * b3;
      const double cost = c1 * c2 * c3;
      if (best_cost < 0 || cost < best_cost - 0.5 ||
          (cost < best_cost + 0.5 && (b1 > best.b1 || (b1 == best.b1 && b2 > best.b2)))) {
        best_cost = cost;
        best = Box3{b1, b2, b3};
      }
    }
  }
  return best;
}

inline int pad_of(int ksize) { return ksize == 2 ? 0 : ksize / 2; }  // 2x2/s2 patch-merging convs are unpadded
inline int out_dim(int in, int ksize, int stride) { return (in + 2 * pad_of(ksize) - ksize) / stride + 1; }

// Output pixel extents (w, h, n) of a convolution; a 1x1 / stride-1 one is a single flat run of B*H*W pixels.
struct Dims3 {
  long long d1, d2, d3;
};
Dims3 out_dims(int B, int H, int W, int ksize, int stride) {
  if (ksize == 1 && stride == 1) return Dims3{static_cast<long long>(B) * H * W, 1, 1};
  return Dims3{out_dim(W, ksize, stride), out_dim(H, ksize, stride), B};
}

// 4-D activation view descriptor (channels innermost).
struct View {
  const void* base;
  uint64_t dims[4];
  uint64_t strides[4];  // elements
};

// NHWC tensor [B][H][W][C] (contiguous) viewed with pixel phase (ph, pw) and step `s` along h/w.
View make_view(const void* base, int B, int H, int W, int C, int s, int ph, int pw) {
  View v;
  v.base = static_cast<const char*>(base) + (static_cast<long long>(ph) * W + pw) * C * 2;
  v.dims[0] = C;
  v.dims[1] = (W - pw + s - 1) / s;
  v.dims[2] = (H - ph + s - 1) / s;
  v.dims[3] = B;
  v.strides[0] = 1;
  v.strides[1] = static_cast<uint64_t>(s) * C;
  v.strides[2] = static_cast<uint64_t>(s) * W * C;
  v.strides[3] = static_cast<uint64_t>(H) * W * C;
  return v;
}
// Same tensor flattened to [B*H*W][C] (dims (C, M, 1, 1)).
View make_flat_view(const void* base, long long M, int C) {
  View v;
  v.base = base;
  v.dims[0] = C;
  v.dims[1] = M;
  v.dims[2] = 1;
  v.dims[3] = 1;
  v.strides[0] = 1;
  v.strides[1] = C;
  v.strides[2] = static_cast<uint64_t>(M) * C;
  v.strides[3] = static_cast<uint64_t>(M) * C;
  return v;
}
// The pixels of a GEMM operand / output, flattened for a 1x1 / stride-1 convolution.
View act_view(const void* base, int B, int H, int W, int C, bool flat) {
  return flat ? make_flat_view(base, static_cast<long long>(B) * H * W, C) : make_view(base, B, H, W, C, 1, 0, 0);
}
int encode_view(CUtensorMap* m, const View& v, const Box3& bx) {
  uint32_t box[4] = {64, (uint32_t)bx.b1, (uint32_t)bx.b2, (uint32_t)bx.b3};
  if (v.dims[1] == 0 || v.dims[2] == 0 || v.dims[3] == 0) {
    set_error("empty activation view");
    return EINVAL_;
  }
  return encode_tmap_bf16(m, v.base, 4, v.dims, v.strides, box);
}

// Row-major bf16 matrix [rows][cols] (e.g. a GEMM weight [N][K]) loaded in boxes of 64 columns x box_rows rows.
int encode_matrix(CUtensorMap* m, const void* base, long long cols, long long rows, int box_rows) {
  uint64_t dims[2] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(rows)};
  uint64_t strides[2] = {1, static_cast<uint64_t>(cols)};
  uint32_t box[2] = {64, static_cast<uint32_t>(box_rows)};
  return encode_tmap_bf16(m, base, 2, dims, strides, box);
}

// Activation operand x[B][H][W][C] of a ksize x ksize / `stride` convolution whose output pixels are tiled by `bx`: its
// tensor maps (one; or one per pixel phase at stride 2) and the tap table - tap t = kh * ksize + kw reads map tap_map[t]
// at offset (tap_o1[t], tap_o2[t]) from the output pixel.
template <class Params>
int encode_taps(Params& p, CUtensorMap (&maps)[4], const void* x, int B, int H, int W, int C, int ksize, int stride,
                const Box3& bx) {
  int rc;
  if (stride == 1) {
    if ((rc = encode_view(&maps[0], act_view(x, B, H, W, C, ksize == 1), bx))) return rc;
    for (int i = 1; i < 4; ++i) maps[i] = maps[0];
  } else {
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw)
        if ((rc = encode_view(&maps[ph * 2 + pw], make_view(x, B, H, W, C, 2, ph, pw), bx))) return rc;
  }
  // stride 2: tap (kh,kw) reads input row 2*oh + kh - pad -> phase ((kh-pad)&1), index oh + floor((kh-pad)/2)
  const int pad = pad_of(ksize);
  for (int kh = 0; kh < ksize; ++kh)
    for (int kw = 0; kw < ksize; ++kw) {
      const int t = kh * ksize + kw, dh = kh - pad, dw = kw - pad;
      const int ph = stride == 2 ? dh & 1 : 0, pw = stride == 2 ? dw & 1 : 0;
      p.tap_map[t] = static_cast<int8_t>(ph * 2 + pw);
      p.tap_o1[t] = static_cast<int8_t>((dw - pw) / stride);
      p.tap_o2[t] = static_cast<int8_t>((dh - ph) / stride);
    }
  return OK;
}

// The epilogue stores one quadrant (32 consecutive tile rows) per warp: split the 128-pixel box into 4 slabs along
// its slowest-varying dimensions (all box dims are powers of two, rows are ordered w fastest).
void quarter_box(const Box3& bx, Box3* qb, int (&o1)[4], int (&o2)[4], int (&o3)[4]) {
  for (int q = 0; q < 4; ++q) o1[q] = o2[q] = o3[q] = 0;
  if (bx.b3 >= 4) {
    *qb = Box3{bx.b1, bx.b2, bx.b3 / 4};
    for (int q = 0; q < 4; ++q) o3[q] = q * (bx.b3 / 4);
  } else if (bx.b3 == 2) {
    *qb = Box3{bx.b1, bx.b2 / 2, 1};  // b1*b2 = 64 -> b2 >= 2 unless b1 = 64
    if (bx.b2 >= 2) {
      for (int q = 0; q < 4; ++q) {
        o2[q] = (q & 1) * (bx.b2 / 2);
        o3[q] = q >> 1;
      }
    } else {
      *qb = Box3{bx.b1 / 2, 1, 1};
      for (int q = 0; q < 4; ++q) {
        o1[q] = (q & 1) * (bx.b1 / 2);
        o3[q] = q >> 1;
      }
    }
  } else if (bx.b2 >= 4) {
    *qb = Box3{bx.b1, bx.b2 / 4, 1};
    for (int q = 0; q < 4; ++q) o2[q] = q * (bx.b2 / 4);
  } else if (bx.b2 == 2) {
    *qb = Box3{bx.b1 / 2, 1, 1};
    for (int q = 0; q < 4; ++q) {
      o1[q] = (q & 1) * (bx.b1 / 2);
      o2[q] = q >> 1;
    }
  } else {
    *qb = Box3{bx.b1 / 4, 1, 1};
    for (int q = 0; q < 4; ++q) o1[q] = q * (bx.b1 / 4);
  }
}

// Tile geometry + output tensor map(s) of a GEMM whose output pixels are described by `dv`.
int setup_output(ConvGemmParams& p, const View& dv, int N, int out_f32, const View* auxv) {
  const long long d1 = dv.dims[1], d2 = dv.dims[2], d3 = dv.dims[3];
  const Box3 bx = choose_box(d1, d2, d3, 128);
  p.box1 = bx.b1, p.box2 = bx.b2, p.box3 = bx.b3;
  p.dim1 = static_cast<int>(d1), p.dim2 = static_cast<int>(d2), p.dim3 = static_cast<int>(d3);
  p.tiles1 = static_cast<int>((d1 + bx.b1 - 1) / bx.b1);
  p.tiles2 = static_cast<int>((d2 + bx.b2 - 1) / bx.b2);
  p.tiles3 = static_cast<int>((d3 + bx.b3 - 1) / bx.b3);
  p.N = N;
  const int BN = N <= 64 ? 64 : 128;
  p.n_tiles = (N + BN - 1) / BN;
  Box3 qb;
  quarter_box(bx, &qb, p.qoff1, p.qoff2, p.qoff3);
  p.out_f32 = out_f32;
  if (dv.base != nullptr) {
    uint32_t box[4] = {out_f32 ? 32u : 64u, (uint32_t)qb.b1, (uint32_t)qb.b2, (uint32_t)qb.b3};
    int rc = out_f32 ? encode_tmap_f32(&p.d_map, dv.base, 4, dv.dims, dv.strides, box)
                     : encode_tmap_bf16(&p.d_map, dv.base, 4, dv.dims, dv.strides, box);
    if (rc) return rc;
  }
  p.has_aux_out = 0;
  if (auxv != nullptr) {
    uint32_t box[4] = {64u, (uint32_t)qb.b1, (uint32_t)qb.b2, (uint32_t)qb.b3};
    int rc = encode_tmap_bf16(&p.aux_map, auxv->base, 4, auxv->dims, auxv->strides, box);
    if (rc) return rc;
    p.has_aux_out = 1;
  }
  return OK;
}
Box3 box_of(const ConvGemmParams& p) { return Box3{p.box1, p.box2, p.box3}; }

bool bn_mask_complete(const b200_bn_mask_t* m) { return m->x_raw && m->scale && m->shift && m->stats; }
// kEpiBnMask epilogue: mask the output (view dv; x_raw has the same layout) with relu'(bn(x_raw)) and write the sum(dz),
// sum(dz * x_raw) partial rows of that BatchNorm's backward.
void set_bn_mask(ConvGemmParams& p, const b200_bn_mask_t* m, const View& dv) {
  p.mask_in = static_cast<const __nv_bfloat16*>(m->x_raw);
  p.ms1 = static_cast<long long>(dv.strides[1]);
  p.ms2 = static_cast<long long>(dv.strides[2]);
  p.ms3 = static_cast<long long>(dv.strides[3]);
  p.bn_scale = m->scale, p.bn_shift = m->shift, p.stats = m->stats;
}

// Persistent grid. With BN statistics every CTA must keep seeing the same channel block (tile % n_tiles), so the grid is
// rounded down to a multiple of n_tiles.
int conv_grid(int tiles, int n_tiles, bool stats) {
  int grid = tiles < device_sm_count() ? tiles : device_sm_count();
  if (stats) grid = grid / n_tiles * n_tiles;
  return grid;
}

template <int BLOCK_N, int EPI>
int launch_conv_gemm_epi(const ConvGemmParams& q, int grid, cudaStream_t st) {
  using Cfg = ConvGemmCfg<BLOCK_N>;
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BLOCK_N, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES));
    configured = true;
  }
  B200_CHECK_CUDA(launch_pdl(conv_gemm_kernel<BLOCK_N, EPI>, dim3(grid), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, st, q));
  B200_LAUNCHED();
  return OK;
}

// Epilogue option set of a launch (bits of conv_gemm.cuh::kEpi*).
int epilogue_flags(const ConvGemmParams& p) {
  int f = 0;
  if (p.bias) f |= kEpiBias;
  if (p.colscale) f |= kEpiColscale;
  f |= (p.act & 3) << kEpiActShift;
  if (p.residual) f |= p.res_f32 ? kEpiResF32 : kEpiResBf16;
  if (p.has_aux_out) f |= kEpiAux;
  if (p.out_f32) f |= kEpiOutF32;
  if (p.out_direct) f |= kEpiDirect;
  if (p.stats) f |= kEpiStats;
  if (p.rowscale) f |= kEpiRowscale;
  if (p.affine) f = (f & ~(kEpiBias | kEpiColscale)) | kEpiAffine;   // colscale / bias carry the BatchNorm scale / shift
  if (p.mask_in) f |= p.bn_scale ? kEpiBnMask : kEpiMask;
  if (p.bn_scale) f &= ~kEpiStats;   // (kEpiBnMask always writes its two statistics rows)
  return f;
}

// The layer types on the four training paths get a compile-time epilogue; anything else runs the generic kernel.
#define B200_EPI_LIST(X)                                                                                  \
  X(kEpiStats)                                            /* ResNet conv -> BN statistics            */  \
  X(0)                                                    /* plain dgrad                             */  \
  X(kEpiResBf16)                                          /* dgrad + identity-branch gradient        */  \
  X(kEpiBias)                                             /* qkv / patch embedding                   */  \
  X(kEpiBias | kEpiResF32 | kEpiOutF32)                   /* proj, fc2: + residual stream (fp32)     */  \
  X(kEpiBias | kEpiColscale | kEpiResF32 | kEpiOutF32)    /* ConvNeXt pwconv2 * gamma + shortcut     */  \
  X(kEpiBias | (2 << kEpiActShift) | kEpiAux)             /* fc1 + GELU, keeps the pre-activation    */  \
  X(3 << kEpiActShift)                                    /* fc2 dgrad * GELU'(pre)                  */  \
  X((3 << kEpiActShift) | kEpiStats)                      /* ... + column sums = fc1 bias gradient   */  \
  X(kEpiOutF32)                                           /* Swin patch-merging reduction            */  \
  X(kEpiBias | kEpiOutF32)                                /* ConvNeXt downsample conv                */  \
  X(kEpiAffine | kEpiResBf16 | (1 << kEpiActShift))       /* bottleneck conv3: relu(bn(conv) + identity) */ \
  X(kEpiAffine | (1 << kEpiActShift))                     /* eval mode: relu(bn(conv))                   */ \
  X(kEpiAffine)                                           /* eval mode: bn(conv) (downsample branch)     */ \
  X(kEpiMask | kEpiResBf16 | kEpiStats)                   /* dgrad + identity gradient, ReLU mask, sum dz */ \
  X(kEpiBnMask)                                           /* 3x3 dgrad + reduce half of the producer's BN backward */ \
  X(kEpiBnMask | kEpiBias)                                /* the same behind the BN-algebra dual GEMM (bias = k W) */ \
  X(kEpiBias | (1 << kEpiActShift))                       /* VGG conv / classifier Linear + bias + ReLU  */ \
  X(kEpiBias | kEpiStats)                                 /* VGG _bn conv: + bias, BN statistics     */

// ---- 64 -> 64 channel convolutions with the weights resident in shared memory (conv_tap64.cuh): ResNet layer1's 3x3
// forward / dgrad and the space-to-depth stem.
bool tap64_ok(const ConvGemmParams& p) {
  const int f = epilogue_flags(p);
  return p.N == 64 && p.n_tiles == 1 && p.k_per_tap == 64 && p.k_blocks_per_tap == 1 && !p.var_taps && !p.chan_window &&
         p.num_taps >= 2 && p.num_taps <= 9 && (f == 0 || f == kEpiStats) && p.dim1 % p.box1 == 0 && p.dim2 % p.box2 == 0 &&
         p.dim3 % p.box3 == 0;
}
template <bool kStats>
int launch_tap64(const ConvGemmParams& q, int grid, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(conv_tap64_kernel<kStats>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTap64SmemBytes));
    configured = true;
  }
  B200_CHECK_CUDA(launch_pdl(conv_tap64_kernel<kStats>, dim3(grid), dim3(384), kTap64SmemBytes, st, q));
  B200_LAUNCHED();
  return OK;
}

template <int BLOCK_N>
int launch_conv_gemm(const ConvGemmParams& p, cudaStream_t st) {
  const int tiles = p.tiles1 * p.tiles2 * p.tiles3 * p.n_tiles;
  const int grid = conv_grid(tiles, p.n_tiles, p.stats != nullptr);
  B200_REQUIRE(grid > 0, "conv_gemm: %d channel blocks exceed the SM count (BN statistics need grid %% n_tiles == 0)", p.n_tiles);
  ConvGemmParams q = p;
  q.desc_lbo = kFwdDescLbo;
  q.desc_sbo = kFwdDescSbo;
  if constexpr (BLOCK_N == 64) {
    if (tap64_ok(p)) return p.stats != nullptr ? launch_tap64<true>(q, grid, st) : launch_tap64<false>(q, grid, st);
  }
  switch (epilogue_flags(p)) {
#define B200_EPI_CASE(F) \
  case (F):              \
    return launch_conv_gemm_epi<BLOCK_N, (F)>(q, grid, st);
    B200_EPI_LIST(B200_EPI_CASE)
#undef B200_EPI_CASE
    default:
      return launch_conv_gemm_epi<BLOCK_N, kEpiGeneric>(q, grid, st);
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Streaming kernel for the narrow-K -> wide-N 1x1 layers (conv1x1_stream.cuh): K in {64, 128, 256}, N % 256 == 0, pixels % 128 == 0.
bool stream_ok(long long pixels, int K, int N) {
  return (K == 64 || K == 128 || K == 256) && N % 256 == 0 && pixels % 128 == 0 && pixels / 128 < (1LL << 30);
}
int stream_grid(long long pixels, int N) {
  const int n_tiles = N / 256;
  const long long items = pixels / 128 * n_tiles;
  int grid = items < device_sm_count() ? static_cast<int>(items) : device_sm_count();
  return grid / n_tiles * n_tiles;
}

template <int KB, int MODE>
int launch_stream(const StreamParams& q, int grid, cudaStream_t st) {
  using Cfg = StreamCfg<KB, MODE>;
  static bool configured = false;
  if (!configured) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(conv1x1_stream_kernel<KB, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES));
    configured = true;
  }
  B200_CHECK_CUDA(launch_pdl(conv1x1_stream_kernel<KB, MODE>, dim3(grid), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, st, q));
  B200_LAUNCHED();
  return OK;
}

// a: [pixels][K], w: [N][K], out / res / mask: [pixels][N]
int run_stream(int mode, const void* a, const void* w, void* out, const void* res, const void* mask, const float* scale,
               const float* shift, float* stats, long long pixels, int K, int N, cudaStream_t st) {
  StreamParams q;
  memset(&q, 0, sizeof(q));
  int rc;
  if ((rc = encode_matrix(&q.a_map, a, K, pixels, 128))) return rc;
  if ((rc = encode_matrix(&q.b_map, w, K, N, 256))) return rc;
  if ((rc = encode_matrix(&q.out_map, out, N, pixels, 16))) return rc;
  if (res != nullptr && (rc = encode_matrix(&q.res_map, res, N, pixels, 16))) return rc;
  if (mask != nullptr && (rc = encode_matrix(&q.mask_map, mask, N, pixels, 16))) return rc;
  q.m_tiles = static_cast<int>(pixels / 128);
  q.n_tiles = N / 256;
  q.N = N;
  q.scale = scale, q.shift = shift, q.stats = stats;
  const int grid = stream_grid(pixels, N);
  if (mode == kStreamAffine)
    return K == 64 ? launch_stream<1, kStreamAffine>(q, grid, st)
                   : (K == 128 ? launch_stream<2, kStreamAffine>(q, grid, st) : launch_stream<4, kStreamAffine>(q, grid, st));
  if (mode == kStreamBnRelu)
    return K == 64 ? launch_stream<1, kStreamBnRelu>(q, grid, st)
                   : (K == 128 ? launch_stream<2, kStreamBnRelu>(q, grid, st) : launch_stream<4, kStreamBnRelu>(q, grid, st));
  return K == 64 ? launch_stream<1, kStreamMask>(q, grid, st)
                 : (K == 128 ? launch_stream<2, kStreamMask>(q, grid, st) : launch_stream<4, kStreamMask>(q, grid, st));
}

int dispatch_conv_gemm(ConvGemmParams& p, int N, cudaStream_t st) {
  if (N <= 64) return launch_conv_gemm<64>(p, st);
  return launch_conv_gemm<128>(p, st);
}
int block_n_for(int N) { return N <= 64 ? 64 : 128; }

template <int BLOCK_NG, bool kGrouped = false>
int launch_wgrad(const WgradParams& p, cudaStream_t st) {
  using Cfg = WgradCfg<BLOCK_NG>;
  static bool configured = false;
  if (!configured) {
    if constexpr (kGrouped) {
      B200_CHECK_CUDA(cudaFuncSetAttribute(wgrad_gemm_kernel<BLOCK_NG, false, true>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    } else {
      B200_CHECK_CUDA(cudaFuncSetAttribute(wgrad_gemm_kernel<BLOCK_NG, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           Cfg::SMEM_BYTES));
      B200_CHECK_CUDA(cudaFuncSetAttribute(wgrad_gemm_kernel<BLOCK_NG, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           Cfg::SMEM_BYTES));
    }
    configured = true;
  }
  const int items = p.mg_tiles * p.ng_tiles * p.num_taps * p.splits;
  const int grid = items < device_sm_count() ? items : device_sm_count();
  WgradParams q = p;
  q.desc_lbo = kWgDescLbo;
  q.desc_sbo = kWgDescSbo;
  q.desc_kstep = kWgDescKstep;
  if constexpr (kGrouped)
    B200_CHECK_CUDA(launch_pdl(wgrad_gemm_kernel<BLOCK_NG, false, true>, dim3(grid), dim3(kWgradThreads), Cfg::SMEM_BYTES, st, q));
  else if (q.bias_partial != nullptr)   // + four warps that sum the dY tiles' columns (the layer's bias gradient)
    B200_CHECK_CUDA(launch_pdl(wgrad_gemm_kernel<BLOCK_NG, true>, dim3(grid), dim3(kWgradThreads), Cfg::SMEM_BYTES, st, q));
  else
    B200_CHECK_CUDA(launch_pdl(wgrad_gemm_kernel<BLOCK_NG, false>, dim3(grid), dim3(kWgradThreads), Cfg::SMEM_BYTES, st, q));
  B200_LAUNCHED();
  return OK;
}

// partial[splits][Cout][taps*Cin] -> grad[Cout][Cin][taps] (+)=, see wgrad_gemm.cuh
int launch_wgrad_reduce(const float* partial, float* dw, int splits, int Cout, int Cin, int taps, int accumulate,
                        cudaStream_t st, const float* bias_partial = nullptr, float* bias_out = nullptr) {
  const long long total = static_cast<long long>(Cout) * Cin * taps;
  if (Cin % 8 == 0 && (reinterpret_cast<uintptr_t>(partial) & 15) == 0) {
    int chunk = taps == 1 ? 256 : 64;
    while (chunk > 16 && chunk / 2 >= Cin) chunk /= 2;  // (stays a multiple of 16: vector loads need 16 B alignment)
    while (chunk > 16 && static_cast<long long>(Cout) * ((Cin + chunk - 1) / chunk) < 2ll * device_sm_count()) chunk /= 2;
    const int SL = splits < 8 ? splits : 8;
    const size_t smem = static_cast<size_t>(SL) * taps * chunk * sizeof(float);
    if (smem <= 48 * 1024 && Cout <= 65535 * 32) {
      dim3 grid(Cout, (Cin + chunk - 1) / chunk);
      B200_CHECK_CUDA(launch_pdl(wgrad_reduce_rows_kernel, dim3(grid), dim3(256), smem, st, partial, dw, splits, Cout, Cin, taps, chunk, SL, accumulate, bias_partial, bias_out));
      return OK;
    }
  }
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  B200_CHECK_CUDA(launch_pdl(wgrad_reduce_flat_kernel, dim3(blocks), dim3(256), 0, st, partial, dw, splits, Cout, Cin, taps, accumulate, bias_partial, bias_out));
  return OK;
}

struct WgradPlan {
  int block_ng, mg_tiles, ng_tiles, taps;
  int merge_atoms;  // > 0: merged-tap mode (wgrad_gemm.cuh), the taps are columns of one N = 192 / 256 tile
  Box3 box;
  int tiles1, tiles2, tiles3, kb_total, splits, kb_per_split;
  int Ho, Wo;
};

// grouped: the kGrouped kernel of a 3x3 grouped convolution (Cin = 64: one channel block per row block; items of 3 taps)
WgradPlan plan_wgrad_geom(long long d1, long long d2, long long d3, int Cin, int Cout, int taps, bool grouped = false) {
  WgradPlan pl;
  pl.taps = taps;
  pl.Ho = static_cast<int>(d2), pl.Wo = static_cast<int>(d1);
  // 128 x 256 tiles halve the dY re-reads per Cin block (48 KB of operands per 2*128*256*64 flops instead of 32 KB per
  // 2*128*128*64): used whenever the padded operand traffic is lower than with 128-wide tiles.
  pl.block_ng = Cin <= 64 ? 64 : (((Cin + 255) / 256) * 48 < ((Cin + 127) / 128) * 32 ? 256 : 128);
  pl.mg_tiles = (Cout + 127) / 128;
  pl.ng_tiles = (Cin + pl.block_ng - 1) / pl.block_ng;
  pl.merge_atoms = 0;
  if (grouped) {
    pl.block_ng = 384;
    pl.ng_tiles = 1;
  } else if (Cin == 64 && taps > 1 && (taps % 4 == 0 || taps % 3 == 0)) {
    pl.merge_atoms = 1;
    pl.block_ng = taps % 4 == 0 ? 256 : 192;
    pl.ng_tiles = taps * 64 / pl.block_ng;
  }
  pl.box = choose_box(d1, d2, d3, 64);
  pl.tiles1 = static_cast<int>((d1 + pl.box.b1 - 1) / pl.box.b1);
  pl.tiles2 = static_cast<int>((d2 + pl.box.b2 - 1) / pl.box.b2);
  pl.tiles3 = static_cast<int>((d3 + pl.box.b3 - 1) / pl.box.b3);
  pl.kb_total = pl.tiles1 * pl.tiles2 * pl.tiles3;
  // Split-K factor: minimise (waves x pixel blocks per item x time per block) + the fp32 partial traffic it causes. The
  // per-block times are estimates of the kernel's L2-operand-bound time (us per 64-pixel block, by tile width).
  const int items_per_split = pl.mg_tiles * pl.ng_tiles * (pl.merge_atoms ? 1 : (grouped ? pl.taps / 3 : pl.taps));
  const int sms = device_sm_count();
  const double t_kb = pl.block_ng >= 256 ? 0.45 : (pl.block_ng == 192 ? 0.36 : (pl.block_ng == 128 ? 0.30 : 0.25));
  const double part_us = static_cast<double>(Cout) * Cin * taps * 4.0 * 2.0 / 3.0e6;  // write + read of one split at ~3 TB/s
  const int max_splits = pl.kb_total / 4 > 0 ? pl.kb_total / 4 : 1;
  int splits = 1;
  double best = 1e30;
  for (int s = 1; s <= max_splits; ++s) {
    const int kps = (pl.kb_total + s - 1) / s;
    const int s2 = (pl.kb_total + kps - 1) / kps;
    if (s2 != s) continue;
    const int waves = (items_per_split * s + sms - 1) / sms;
    if (waves > 2 && items_per_split <= sms) continue;   // never a third wave when one split's tiles fit on the SMs
    const double cost = waves * (kps * t_kb + 2.0) + s * part_us;
    if (cost < best) best = cost, splits = s;
    if (waves > 4 && s > 8) break;
  }
  pl.kb_per_split = (pl.kb_total + splits - 1) / splits;
  pl.splits = (pl.kb_total + pl.kb_per_split - 1) / pl.kb_per_split;
  return pl;
}

WgradPlan plan_wgrad(int B, int H, int W, int Cin, int Cout, int ksize, int stride, bool grouped = false) {
  const Dims3 d = out_dims(B, H, W, ksize, stride);
  WgradPlan pl = plan_wgrad_geom(d.d1, d.d2, d.d3, Cin, Cout, ksize * ksize, grouped);
  pl.Ho = out_dim(H, ksize, stride), pl.Wo = out_dim(W, ksize, stride);
  return pl;
}

// Bytes of the fp32 split-K partials [splits][Cout][taps * Cin] a weight-gradient launch writes to its workspace.
size_t wgrad_bytes(const WgradPlan& pl, int Cout, int Cin) {
  return static_cast<size_t>(pl.splits) * Cout * pl.taps * Cin * sizeof(float);
}

// Tile, split and partial-layout fields of a weight-gradient launch.
WgradParams wgrad_params(const WgradPlan& pl, int Cout, int Cin, void* workspace) {
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.num_taps = pl.merge_atoms ? 1 : pl.taps;
  p.merge_atoms = pl.merge_atoms;
  p.n_cols = pl.merge_atoms ? pl.taps * Cin : Cin;
  p.Cout = Cout, p.Cin = Cin;
  p.mg_tiles = pl.mg_tiles, p.ng_tiles = pl.ng_tiles;
  p.tiles1 = pl.tiles1, p.tiles2 = pl.tiles2, p.tiles3 = pl.tiles3;
  p.box1 = pl.box.b1, p.box2 = pl.box.b2, p.box3 = pl.box.b3;
  p.splits = pl.splits, p.kb_per_split = pl.kb_per_split, p.kb_total = pl.kb_total;
  p.ld_partial = static_cast<long long>(pl.taps) * Cin;
  p.partial = static_cast<float*>(workspace);
  return p;
}

// Tensor maps of dY and of the activation taps of a weight-gradient launch, and its tap table.
int setup_wgrad_maps(WgradParams& p, const WgradPlan& pl, const void* dy, const void* x, int B, int H, int W, int Cin,
                     int Cout, int ksize, int stride) {
  int rc;
  if ((rc = encode_view(&p.dy_map, act_view(dy, B, pl.Ho, pl.Wo, Cout, ksize == 1 && stride == 1), pl.box))) return rc;
  return encode_taps(p, p.x_maps, x, B, H, W, Cin, ksize, stride, pl.box);
}

// Space-to-depth stem (conv 7x7 / stride 2 / pad 3 on 3 channels, classification/resnet/models/networks.py:150,206):
// z[B][Ho+3][Wo+3][16] holds the zero-padded input with the 2x2 pixel phase folded into the channels (12 real + 4 zero), so
// the conv becomes a 4x4 / stride-1 conv. The four x-taps of a pixel are 64 CONTIGUOUS elements of z, therefore a tensor map
// whose rows overlap (row pitch 16 elements, row length 64) presents every k-block (one y-tap) as an ordinary 64-channel
// activation row: the implicit-GEMM kernels run unchanged with Cin = 64 and four taps (0, ky).
View stem_s2d_view(const void* z, int B, int Ho, int Wo) {
  const int Hz = Ho + 3, Wz = Wo + 3;
  View v;
  v.base = z;
  v.dims[0] = 64, v.dims[1] = Wo, v.dims[2] = Hz, v.dims[3] = B;
  v.strides[0] = 1, v.strides[1] = 16, v.strides[2] = static_cast<uint64_t>(Wz) * 16;
  v.strides[3] = static_cast<uint64_t>(Hz) * Wz * 16;
  return v;
}

}  // namespace

extern "C" {

// Statistics rows of a forward launch with BN-column tiles (see b200_conv2d_fwd_stats_rows).
static int fwd_stats_rows(int B, int H, int W, int Cout, int ksize, int stride, int BN) {
  const Dims3 d = out_dims(B, H, W, ksize, stride);
  const Box3 bx = choose_box(d.d1, d.d2, d.d3, 128);
  const long long m_tiles = ((d.d1 + bx.b1 - 1) / bx.b1) * ((d.d2 + bx.b2 - 1) / bx.b2) * ((d.d3 + bx.b3 - 1) / bx.b3);
  const int n_tiles = (Cout + BN - 1) / BN;
  const long long tiles = m_tiles * n_tiles;
  const int grid = conv_grid(tiles > (1 << 30) ? (1 << 30) : static_cast<int>(tiles), n_tiles, true);
  // one partial row per (CTA group, 32-row quadrant); with 64-channel tiles two, one per parity of the CTA's tile count
  // (the layout conv_tap64_kernel shares)
  return grid / n_tiles * (BN == 64 ? 8 : 4);
}

int b200_conv2d_fwd_stats_rows(int B, int H, int W, int Cout, int ksize, int stride) {
  return fwd_stats_rows(B, H, W, Cout, ksize, stride, block_n_for(Cout));
}

// y_f32: y is an fp32 tensor written through TMA (b200_conv2d_fwd_f32).
// bn_scale / bn_shift: y = act(conv * scale[c] + shift[c] (+ residual)) - BatchNorm with fixed (running) statistics folded
// into the epilogue; the activation moves AFTER the residual add (conv_gemm.cuh kEpiAffine).
// Cg > 0: grouped convolution of group width Cg (Cin == Cout, validated by the caller) in channel-window mode.
static int conv_fwd(const void* x, const void* w, void* y, int B, int H, int W, int Cin, int Cout, int ksize, int stride,
                    float* stats, const float* bias, int act, const void* residual, float* out_f32, long long ld_out,
                    const float* bn_scale, const float* bn_shift, int y_f32, int Cg, void* stream) {
  B200_REQUIRE(ksize == 1 || ksize == 3 || (ksize == 2 && stride == 2), "conv2d_fwd: ksize %d / stride %d unsupported", ksize, stride);
  B200_REQUIRE(stride == 1 || stride == 2, "conv2d_fwd: stride %d unsupported (1 or 2)", stride);
  B200_REQUIRE(Cin % 8 == 0 && Cout % 8 == 0, "conv2d_fwd: Cin=%d / Cout=%d must be multiples of 8", Cin, Cout);
  B200_REQUIRE(B > 0 && H > 0 && W > 0, "conv2d_fwd: empty input");
  B200_REQUIRE(stride == 1 || (H >= 2 && W >= 2), "conv2d_fwd: stride-2 needs H,W >= 2");
  B200_REQUIRE(out_f32 == nullptr || (ksize == 1 && stride == 1), "conv2d_fwd: fp32 output only for 1x1/s1");
  B200_REQUIRE((bn_scale == nullptr) == (bn_shift == nullptr), "conv2d_fwd: bn_scale and bn_shift go together");
  B200_REQUIRE(bn_scale == nullptr || (Cout % 64 == 0 && bias == nullptr && stats == nullptr && out_f32 == nullptr && act <= 1 && !y_f32),
               "conv2d_fwd + folded BN: Cout=%d must be a multiple of 64, no bias / statistics / fp32 output", Cout);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int Ho = out_dim(H, ksize, stride), Wo = out_dim(W, ksize, stride);
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  int rc;
  View dv = act_view(y, B, Ho, Wo, Cout, ksize == 1 && stride == 1);
  if (out_f32 != nullptr) dv.base = nullptr;  // direct fp32 stores, no TMA map
  if ((rc = setup_output(p, dv, Cout, y_f32, nullptr))) return rc;
  const int BN = Cg ? 64 : block_n_for(Cout);
  p.n_tiles = (Cout + BN - 1) / BN;
  p.chan_window = Cg ? 1 : 0;
  p.k_per_tap = Cg ? 64 : Cin;
  p.k_blocks_per_tap = Cg ? 1 : (Cin + 63) / 64;
  p.num_taps = ksize * ksize;
  if ((rc = encode_taps(p, p.a_maps, x, B, H, W, Cin, ksize, stride, box_of(p)))) return rc;
  for (int t = 0; t < p.num_taps; ++t) p.tap_w[t] = static_cast<int8_t>(t);
  if ((rc = encode_matrix(&p.b_map, w, static_cast<long long>(p.num_taps) * p.k_per_tap, Cout, BN))) return rc;
  p.stats = stats;
  p.bias = bias;
  p.act = act;
  p.residual = residual;
  p.rs1 = static_cast<long long>(dv.strides[1]);
  p.rs2 = static_cast<long long>(dv.strides[2]);
  p.rs3 = static_cast<long long>(dv.strides[3]);
  p.out_direct = out_f32;
  p.ld_out = ld_out;
  if (bn_scale != nullptr) {
    p.affine = 1;
    p.colscale = bn_scale;
    p.bias = bn_shift;
  }
  return Cg ? launch_conv_gemm<64>(p, st) : dispatch_conv_gemm(p, Cout, st);
}

int b200_conv2d_fwd(const void* x, const void* w, void* y, int B, int H, int W, int Cin, int Cout, int ksize, int stride,
                    float* stats, const float* bias, int act, const void* residual, float* out_f32, long long ld_out,
                    const float* bn_scale, const float* bn_shift, void* stream) {
  return conv_fwd(x, w, y, B, H, W, Cin, Cout, ksize, stride, stats, bias, act, residual, out_f32, ld_out, bn_scale, bn_shift,
                  0, 0, stream);
}

int b200_conv2d_fwd_f32(const void* x, const void* w, float* y, int B, int H, int W, int Cin, int Cout, int ksize,
                        int stride, const float* bias, void* stream) {
  return conv_fwd(x, w, y, B, H, W, Cin, Cout, ksize, stride, nullptr, bias, 0, nullptr, nullptr, 0, nullptr, nullptr, 1, 0,
                  stream);
}

// Cg > 0: grouped convolution of group width Cg (Cin == Cout, validated by the caller) in channel-window mode
static int conv_dgrad(const void* dy, const void* wd, void* dx, int B, int H, int W, int Cin, int Cout, int ksize,
                      int stride, const void* residual, const b200_bn_mask_t* bn_mask, int Cg, void* stream) {
  B200_REQUIRE(ksize == 1 || ksize == 3 || (ksize == 2 && stride == 2), "conv2d_dgrad: ksize %d / stride %d unsupported", ksize, stride);
  B200_REQUIRE(stride == 1 || stride == 2, "conv2d_dgrad: stride %d unsupported", stride);
  B200_REQUIRE(Cin % 8 == 0 && Cout % 8 == 0, "conv2d_dgrad: Cin=%d / Cout=%d must be multiples of 8", Cin, Cout);
  B200_REQUIRE(bn_mask == nullptr || (stride == 1 && Cin % 64 == 0 && bn_mask_complete(bn_mask)),
               "conv2d_dgrad: the fused BatchNorm-backward reduce needs stride 1, Cin %% 64 == 0 and every bn_mask field "
               "(Cin=%d, stride=%d)", Cin, stride);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int Ho = out_dim(H, ksize, stride), Wo = out_dim(W, ksize, stride);
  const bool flat = (ksize == 1 && stride == 1);
  const int BN = Cg ? 64 : block_n_for(Cin);
  const int k_per_tap = Cg ? 64 : Cout;
  int rc;
  CUtensorMap b_map;
  if ((rc = encode_matrix(&b_map, wd, static_cast<long long>(ksize * ksize) * k_per_tap, Cin, BN))) return rc;
  const int nphase = (stride == 2 && ksize >= 2) ? 2 : 1;  // phases per spatial dim that need their own launch
  for (int ph = 0; ph < nphase; ++ph) {
    for (int pw = 0; pw < nphase; ++pw) {
      ConvGemmParams p;
      memset(&p, 0, sizeof(p));
      p.b_map = b_map;
      // output (dx) view for this launch
      View dv = flat ? make_flat_view(dx, static_cast<long long>(B) * H * W, Cin)
                     : make_view(dx, B, H, W, Cin, stride, ph, pw);
      if ((rc = setup_output(p, dv, Cin, 0, nullptr))) return rc;
      p.n_tiles = (Cin + BN - 1) / BN;
      p.chan_window = Cg ? 1 : 0;
      p.k_per_tap = k_per_tap;
      p.k_blocks_per_tap = Cg ? 1 : (Cout + 63) / 64;
      if ((rc = encode_view(&p.a_maps[0], act_view(dy, B, Ho, Wo, Cout, flat), box_of(p)))) return rc;
      for (int i = 1; i < 4; ++i) p.a_maps[i] = p.a_maps[0];
      int nt = 0;
      if (ksize == 1) {
        p.tap_map[0] = 0, p.tap_o1[0] = 0, p.tap_o2[0] = 0, p.tap_w[0] = 0;
        nt = 1;
      } else if (stride == 1) {
        // dx[q] = sum_{kh,kw} W[kh,kw]^T dy[q - (kh-1, kw-1)]
        for (int kh = 0; kh < 3; ++kh)
          for (int kw = 0; kw < 3; ++kw) {
            p.tap_map[nt] = 0;
            p.tap_o1[nt] = static_cast<int8_t>(1 - kw);
            p.tap_o2[nt] = static_cast<int8_t>(1 - kh);
            p.tap_w[nt] = static_cast<int8_t>(kh * 3 + kw);
            ++nt;
          }
      } else if (ksize == 2) {
        // 2x2 / stride 2, unpadded: input pixel (2j+ph, 2i+pw) is touched by exactly one tap, (kh,kw) = (ph,pw), from (j,i)
        p.tap_map[0] = 0, p.tap_o1[0] = 0, p.tap_o2[0] = 0;
        p.tap_w[0] = static_cast<int8_t>(ph * 2 + pw);
        nt = 1;
      } else {
        // stride 2, 3x3, pad 1: input row ih = 2j+ph receives taps kh with (ih + 1 - kh) even, from oh = (ih+1-kh)/2
        for (int kh = 0; kh < 3; ++kh) {
          if (((ph + 1 - kh) & 1) != 0) continue;
          for (int kw = 0; kw < 3; ++kw) {
            if (((pw + 1 - kw) & 1) != 0) continue;
            p.tap_map[nt] = 0;
            p.tap_o1[nt] = static_cast<int8_t>((pw + 1 - kw) / 2);
            p.tap_o2[nt] = static_cast<int8_t>((ph + 1 - kh) / 2);
            p.tap_w[nt] = static_cast<int8_t>(kh * 3 + kw);
            ++nt;
          }
        }
      }
      p.num_taps = nt;
      if (residual != nullptr) {
        p.residual = static_cast<const char*>(residual) + (static_cast<const char*>(dv.base) - static_cast<const char*>(dx));
        p.rs1 = static_cast<long long>(dv.strides[1]);
        p.rs2 = static_cast<long long>(dv.strides[2]);
        p.rs3 = static_cast<long long>(dv.strides[3]);
      }
      if (bn_mask != nullptr) set_bn_mask(p, bn_mask, dv);
      if ((rc = Cg ? launch_conv_gemm<64>(p, st) : dispatch_conv_gemm(p, Cin, st))) return rc;
    }
  }
  return OK;
}

int b200_conv2d_dgrad(const void* dy, const void* wd, void* dx, int B, int H, int W, int Cin, int Cout, int ksize,
                      int stride, const void* residual, const b200_bn_mask_t* bn_mask, void* stream) {
  return conv_dgrad(dy, wd, dx, B, H, W, Cin, Cout, ksize, stride, residual, bn_mask, 0, stream);
}

int b200_gemm_ex(const b200_view_t* a, const b200_view_t* out, const b200_gemm_args_t* g, void* stream) {
  B200_REQUIRE(a != nullptr && out != nullptr && g != nullptr && g->w != nullptr, "gemm_ex: null argument");
  B200_REQUIRE(g->N % 8 == 0 && g->K % 8 == 0, "gemm_ex: N=%d / K=%d must be multiples of 8", g->N, g->K);
  for (int i = 0; i < 3; ++i)
    B200_REQUIRE(a->dim[i] == out->dim[i] && a->dim[i] > 0, "gemm_ex: a/out pixel extents differ in dim %d", i);
  B200_REQUIRE(!(g->aux_out != nullptr && g->out_f32), "gemm_ex: aux_out needs a bf16 primary output");
  B200_REQUIRE(!(g->stats != nullptr && g->out_f32), "gemm_ex: stats need a bf16 output");
  auto to_view = [](const b200_view_t* v, int C) {
    View r;
    r.base = v->base;
    r.dims[0] = C;
    r.strides[0] = 1;
    for (int i = 0; i < 3; ++i) {
      r.dims[i + 1] = static_cast<uint64_t>(v->dim[i]);
      r.strides[i + 1] = static_cast<uint64_t>(v->stride[i]);
    }
    return r;
  };
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  int rc;
  View dv = to_view(out, g->N);
  View auxv;
  if (g->aux_out) auxv = to_view(g->aux_out, g->N);
  if ((rc = setup_output(p, dv, g->N, g->out_f32, g->aux_out ? &auxv : nullptr))) return rc;
  const Box3 bx = box_of(p);
  // TMA needs non-zero strides that are multiples of 16 bytes for the activation operand
  if ((rc = encode_view(&p.a_maps[0], to_view(a, g->K), bx))) return rc;
  for (int i = 1; i < 4; ++i) p.a_maps[i] = p.a_maps[0];
  p.num_taps = 1;
  p.k_per_tap = g->K;
  p.k_blocks_per_tap = (g->K + 63) / 64;
  if ((rc = encode_matrix(&p.b_map, g->w, g->K, g->N, block_n_for(g->N)))) return rc;
  p.stats = g->stats;
  p.bias = g->bias;
  p.colscale = g->colscale;
  p.act = g->act;
  if (g->residual) {
    p.residual = g->residual->base;
    p.res_f32 = g->residual_f32;
    p.rs1 = g->residual->stride[0], p.rs2 = g->residual->stride[1], p.rs3 = g->residual->stride[2];
  }
  if (g->rowscale != nullptr) {
    B200_REQUIRE(g->rows_per_sample > 0, "gemm_ex: rowscale needs rows_per_sample > 0");
    p.rowscale = g->rowscale;
    p.rows_per_sample = g->rows_per_sample;
  }
  if (g->act == B200_ACT_GELU_GRAD) {
    B200_REQUIRE(g->aux_in != nullptr, "gemm_ex: B200_ACT_GELU_GRAD needs aux_in");
    p.aux_in = static_cast<const __nv_bfloat16*>(g->aux_in->base);
    p.as1 = g->aux_in->stride[0], p.as2 = g->aux_in->stride[1], p.as3 = g->aux_in->stride[2];
  }
  return dispatch_conv_gemm(p, g->N, static_cast<cudaStream_t>(stream));
}

int b200_conv2d_wgrad_splits(int B, int H, int W, int Cin, int Cout, int ksize, int stride) {
  return plan_wgrad(B, H, W, Cin, Cout, ksize, stride).splits;
}

size_t b200_conv2d_wgrad_workspace_bytes(int B, int H, int W, int Cin, int Cout, int ksize, int stride) {
  return wgrad_bytes(plan_wgrad(B, H, W, Cin, Cout, ksize, stride), Cout, Cin);
}

int b200_conv2d_wgrad(const void* dy, const void* x, float* dw, void* workspace, size_t workspace_bytes, int B, int H,
                      int W, int Cin, int Cout, int ksize, int stride, int accumulate, float* bias_partial, float* bias_out,
                      void* stream) {
  B200_REQUIRE(ksize == 1 || ksize == 3 || (ksize == 2 && stride == 2), "conv2d_wgrad: ksize %d / stride %d unsupported", ksize, stride);
  B200_REQUIRE(stride == 1 || stride == 2, "conv2d_wgrad: stride %d unsupported", stride);
  B200_REQUIRE(Cin % 8 == 0 && Cout % 8 == 0, "conv2d_wgrad: Cin=%d / Cout=%d must be multiples of 8", Cin, Cout);
  B200_REQUIRE(bias_out == nullptr || bias_partial != nullptr, "conv2d_wgrad: bias_out needs bias_partial");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const WgradPlan pl = plan_wgrad(B, H, W, Cin, Cout, ksize, stride);
  const size_t need = wgrad_bytes(pl, Cout, Cin);
  B200_REQUIRE(workspace != nullptr && workspace_bytes >= need, "conv2d_wgrad: workspace too small (%zu < %zu)",
               workspace_bytes, need);
  WgradParams p = wgrad_params(pl, Cout, Cin, workspace);
  p.bias_partial = bias_partial;
  int rc;
  if ((rc = setup_wgrad_maps(p, pl, dy, x, B, H, W, Cin, Cout, ksize, stride))) return rc;
  if (pl.block_ng == 64)
    rc = launch_wgrad<64>(p, st);
  else if (pl.block_ng == 128)
    rc = launch_wgrad<128>(p, st);
  else if (pl.block_ng == 192)
    rc = launch_wgrad<192>(p, st);
  else
    rc = launch_wgrad<256>(p, st);
  if (rc) return rc;
  if ((rc = launch_wgrad_reduce(p.partial, dw, pl.splits, Cout, Cin, pl.taps, accumulate, st, bias_partial, bias_out))) return rc;
  B200_LAUNCHED();
  return OK;
}

int b200_stem_s2d_conv_fwd(const void* z, const void* w, void* y, float* stats, int B, int Ho, int Wo, void* stream) {
  B200_REQUIRE(B > 0 && Ho > 0 && Wo > 0, "stem_s2d_conv_fwd: empty output");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int Cout = 64;
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  int rc;
  if ((rc = setup_output(p, make_view(y, B, Ho, Wo, Cout, 1, 0, 0), Cout, 0, nullptr))) return rc;
  const Box3 bx = box_of(p);
  p.k_per_tap = 64;
  p.k_blocks_per_tap = 1;
  p.num_taps = 4;
  if ((rc = encode_view(&p.a_maps[0], stem_s2d_view(z, B, Ho, Wo), bx))) return rc;
  for (int i = 1; i < 4; ++i) p.a_maps[i] = p.a_maps[0];
  for (int ky = 0; ky < 4; ++ky) {
    p.tap_map[ky] = 0, p.tap_o1[ky] = 0, p.tap_o2[ky] = static_cast<int8_t>(ky), p.tap_w[ky] = static_cast<int8_t>(ky);
  }
  if ((rc = encode_matrix(&p.b_map, w, 256, Cout, 64))) return rc;
  p.stats = stats;
  return dispatch_conv_gemm(p, Cout, st);
}

size_t b200_stem_s2d_conv_wgrad_workspace_bytes(int B, int Ho, int Wo) {
  return wgrad_bytes(plan_wgrad_geom(Wo, Ho, B, 64, 64, 4), 64, 64);
}

int b200_stem_s2d_conv_wgrad(const void* dy, const void* z, float* g, void* workspace, size_t workspace_bytes, int B, int Ho,
                             int Wo, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int Cout = 64, Cin = 64, taps = 4;
  const WgradPlan pl = plan_wgrad_geom(Wo, Ho, B, Cin, Cout, taps);
  const size_t need = wgrad_bytes(pl, Cout, Cin);
  B200_REQUIRE(workspace != nullptr && workspace_bytes >= need, "stem_s2d_conv_wgrad: workspace too small (%zu < %zu)",
               workspace_bytes, need);
  WgradParams p = wgrad_params(pl, Cout, Cin, workspace);
  int rc;
  if ((rc = encode_view(&p.dy_map, make_view(dy, B, Ho, Wo, Cout, 1, 0, 0), pl.box))) return rc;
  if ((rc = encode_view(&p.x_maps[0], stem_s2d_view(z, B, Ho, Wo), pl.box))) return rc;
  for (int i = 1; i < 4; ++i) p.x_maps[i] = p.x_maps[0];
  for (int ky = 0; ky < 4; ++ky) p.tap_map[ky] = 0, p.tap_o1[ky] = 0, p.tap_o2[ky] = static_cast<int8_t>(ky);
  if ((rc = launch_wgrad<256>(p, st))) return rc;  // merged-tap mode: the four y-taps are the four 64-column atoms
  // g[cout][k64][ky] (the generic "OIHW" layout of a 64-channel, 4-tap conv); b200_stem_s2d_wgrad_relayout maps it to [64,3,7,7]
  if ((rc = launch_wgrad_reduce(p.partial, g, pl.splits, Cout, Cin, taps, 0, st))) return rc;
  B200_LAUNCHED();
  return OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// BatchNorm folded through a 1x1 convolution (ResNet bottleneck conv3, engine/resnet.py "algebra" path).

int b200_conv1x1_bn_act_fwd(const void* x, const void* w, const float* scale, const float* shift, const void* residual,
                            void* y, long long pixels, int Cin, int Cout, int relu, void* stream) {
  B200_REQUIRE(pixels > 0 && Cin % 64 == 0 && Cout % 64 == 0, "conv1x1_bn_act_fwd: Cin=%d / Cout=%d must be multiples of 64", Cin, Cout);
  B200_REQUIRE(scale != nullptr && shift != nullptr && residual != nullptr && relu == 1,
               "conv1x1_bn_act_fwd: implemented for relu(bn(conv) + residual)");
  if (stream_ok(pixels, Cin, Cout))
    return run_stream(kStreamBnRelu, x, w, y, residual, nullptr, scale, shift, nullptr, pixels, Cin, Cout,
                      static_cast<cudaStream_t>(stream));
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  int rc;
  View dv = make_flat_view(y, pixels, Cout);
  if ((rc = setup_output(p, dv, Cout, 0, nullptr))) return rc;
  const Box3 bx = box_of(p);
  p.k_per_tap = Cin;
  p.k_blocks_per_tap = Cin / 64;
  p.num_taps = 1;
  if ((rc = encode_view(&p.a_maps[0], make_flat_view(x, pixels, Cin), bx))) return rc;
  for (int i = 1; i < 4; ++i) p.a_maps[i] = p.a_maps[0];
  if ((rc = encode_matrix(&p.b_map, w, Cin, Cout, block_n_for(Cout)))) return rc;
  p.affine = 1;
  p.colscale = scale;
  p.bias = shift;
  p.act = 1;
  p.residual = residual;
  p.rs1 = static_cast<long long>(dv.strides[1]);
  p.rs2 = static_cast<long long>(dv.strides[2]);
  p.rs3 = static_cast<long long>(dv.strides[3]);
  return dispatch_conv_gemm(p, Cout, static_cast<cudaStream_t>(stream));
}

int b200_conv1x1_bn_fwd(const void* x, const void* w, const float* scale, const float* shift, void* y, long long pixels,
                        int Cin, int Cout, void* stream) {
  B200_REQUIRE(pixels > 0 && Cin % 64 == 0 && Cout % 64 == 0, "conv1x1_bn_fwd: Cin=%d / Cout=%d must be multiples of 64", Cin, Cout);
  B200_REQUIRE(scale != nullptr && shift != nullptr, "conv1x1_bn_fwd: scale / shift required");
  if (stream_ok(pixels, Cin, Cout))
    return run_stream(kStreamAffine, x, w, y, nullptr, nullptr, scale, shift, nullptr, pixels, Cin, Cout,
                      static_cast<cudaStream_t>(stream));
  return conv_fwd(x, w, y, 1, 1, static_cast<int>(pixels), Cin, Cout, 1, 1, nullptr, nullptr, 0, nullptr, nullptr, 0, scale,
                  shift, 0, 0, stream);
}

int b200_conv1x1_dgrad_masked_stats_rows(long long pixels, int Cin, int Cout) {
  // one partial row per CTA group and 32-row quadrant of the kernel b200_conv1x1_dgrad_masked dispatches to: the streaming
  // kernel's groups own 256 channels, the generic kernel's 64 or 128
  if (stream_ok(pixels, Cout, Cin)) return stream_grid(pixels, Cin) / (Cin / 256) * 4;
  return b200_conv2d_fwd_stats_rows(1, 1, static_cast<int>(pixels), Cin, 1, 1);
}

int b200_conv1x1_dgrad_masked(const void* dy, const void* wd, void* dx, long long pixels, int Cin, int Cout,
                              const void* residual, const void* mask_src, float* stats, void* stream) {
  B200_REQUIRE(pixels > 0 && Cin % 64 == 0 && Cout % 64 == 0, "conv1x1_dgrad_masked: Cin=%d / Cout=%d must be multiples of 64", Cin, Cout);
  B200_REQUIRE(residual != nullptr && mask_src != nullptr && stats != nullptr, "conv1x1_dgrad_masked: residual, mask and stats are required");
  if (stream_ok(pixels, Cout, Cin))
    return run_stream(kStreamMask, dy, wd, dx, residual, mask_src, nullptr, nullptr, stats, pixels, Cout, Cin,
                      static_cast<cudaStream_t>(stream));
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  int rc;
  View dv = make_flat_view(dx, pixels, Cin);
  if ((rc = setup_output(p, dv, Cin, 0, nullptr))) return rc;
  const Box3 bx = box_of(p);
  p.k_per_tap = Cout;
  p.k_blocks_per_tap = Cout / 64;
  p.num_taps = 1;
  if ((rc = encode_view(&p.a_maps[0], make_flat_view(dy, pixels, Cout), bx))) return rc;
  for (int i = 1; i < 4; ++i) p.a_maps[i] = p.a_maps[0];
  if ((rc = encode_matrix(&p.b_map, wd, Cout, Cin, block_n_for(Cin)))) return rc;
  p.residual = residual;
  p.rs1 = static_cast<long long>(dv.strides[1]);
  p.rs2 = static_cast<long long>(dv.strides[2]);
  p.rs3 = static_cast<long long>(dv.strides[3]);
  p.mask_in = static_cast<const __nv_bfloat16*>(mask_src);
  p.ms1 = p.rs1, p.ms2 = p.rs2, p.ms3 = p.rs3;
  p.stats = stats;
  return dispatch_conv_gemm(p, Cin, static_cast<cudaStream_t>(stream));
}

int b200_gemm_dual(const void* a0, int K0, const void* a1, int K1, const void* wcat, const float* bias, void* out,
                   long long pixels, int N, const b200_bn_mask_t* bn_mask, void* stream) {
  B200_REQUIRE(pixels > 0 && K0 % 64 == 0 && K1 % 64 == 0 && N % 8 == 0, "gemm_dual: K0=%d / K1=%d must be multiples of 64", K0, K1);
  B200_REQUIRE(bn_mask == nullptr || (N % 64 == 0 && bn_mask_complete(bn_mask)),
               "gemm_dual: fused BN-backward reduce needs N %% 64 == 0 and every bn_mask field (N=%d)", N);
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  int rc;
  View dv = make_flat_view(out, pixels, N);
  if ((rc = setup_output(p, dv, N, 0, nullptr))) return rc;
  const Box3 bx = box_of(p);
  if ((rc = encode_view(&p.a_maps[0], make_flat_view(a0, pixels, K0), bx))) return rc;
  if ((rc = encode_view(&p.a_maps[1], make_flat_view(a1, pixels, K1), bx))) return rc;
  p.a_maps[2] = p.a_maps[0], p.a_maps[3] = p.a_maps[0];
  p.num_taps = 2;
  p.k_per_tap = K0;
  p.k_blocks_per_tap = K0 / 64;
  p.var_taps = 1;
  p.tap_map[0] = 0, p.tap_map[1] = 1;
  p.tap_kb[0] = static_cast<int16_t>(K0 / 64), p.tap_kb[1] = static_cast<int16_t>(K1 / 64);
  p.tap_k0[0] = 0, p.tap_k0[1] = K0;
  p.kb_total = (K0 + K1) / 64;
  if ((rc = encode_matrix(&p.b_map, wcat, K0 + K1, N, block_n_for(N)))) return rc;
  p.bias = bias;
  if (bn_mask != nullptr) set_bn_mask(p, bn_mask, dv);
  return dispatch_conv_gemm(p, N, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------------------------
// Grouped 3x3 convolutions (ResNeXt conv2, classification/resnet/models/networks.py:295-321): C input = C output channels,
// C % 64 == 0, group width Cg = C / groups in {4, 8, 16, 32, 64}, so no group straddles a 64-channel block. Forward and
// dgrad run conv_gemm_kernel<64> in channel-window mode on the block-diagonal operands of b200_pack_weight modes 3 / 4;
// the weight gradient runs the kGrouped mode of wgrad_gemm_kernel.

static int grouped_check(const char* fn, int C, int groups, int ksize, int stride) {
  B200_REQUIRE(ksize == 3, "%s: ksize %d unsupported (3x3 only)", fn, ksize);
  B200_REQUIRE(stride == 1 || stride == 2, "%s: stride %d unsupported (1 or 2)", fn, stride);
  B200_REQUIRE(groups > 0 && C > 0 && C % 64 == 0 && C % groups == 0, "%s: C=%d must be a multiple of 64 and of groups=%d",
               fn, C, groups);
  const int Cg = C / groups;
  B200_REQUIRE(Cg >= 4 && 64 % Cg == 0, "%s: group width C / groups = %d unsupported (4, 8, 16, 32 or 64)", fn, Cg);
  return OK;
}

int b200_conv2d_grouped_fwd_stats_rows(int B, int H, int W, int C, int groups, int ksize, int stride) {
  int rc;
  if ((rc = grouped_check("conv2d_grouped_fwd_stats_rows", C, groups, ksize, stride))) return rc;
  return fwd_stats_rows(B, H, W, C, ksize, stride, 64);
}

int b200_conv2d_grouped_fwd(const void* x, const void* w, void* y, int B, int H, int W, int C, int groups, int ksize,
                            int stride, float* stats, int act, const float* bn_scale, const float* bn_shift, void* stream) {
  int rc;
  if ((rc = grouped_check("conv2d_grouped_fwd", C, groups, ksize, stride))) return rc;
  B200_REQUIRE(act == 0 || act == 1, "conv2d_grouped_fwd: act %d unsupported (none or relu)", act);
  return conv_fwd(x, w, y, B, H, W, C, C, ksize, stride, stats, nullptr, act, nullptr, nullptr, 0, bn_scale, bn_shift, 0,
                  C / groups, stream);
}

int b200_conv2d_grouped_dgrad(const void* dy, const void* wd, void* dx, int B, int H, int W, int C, int groups, int ksize,
                              int stride, const b200_bn_mask_t* bn_mask, void* stream) {
  int rc;
  if ((rc = grouped_check("conv2d_grouped_dgrad", C, groups, ksize, stride))) return rc;
  return conv_dgrad(dy, wd, dx, B, H, W, C, C, ksize, stride, nullptr, bn_mask, C / groups, stream);
}

size_t b200_conv2d_grouped_wgrad_workspace_bytes(int B, int H, int W, int C, int groups, int ksize, int stride) {
  if (grouped_check("conv2d_grouped_wgrad_workspace_bytes", C, groups, ksize, stride)) return 0;
  return wgrad_bytes(plan_wgrad(B, H, W, 64, C, ksize, stride, true), C, 64);
}

int b200_conv2d_grouped_wgrad(const void* dy, const void* x, float* dw, void* workspace, size_t workspace_bytes, int B,
                              int H, int W, int C, int groups, int ksize, int stride, int accumulate, void* stream) {
  int rc;
  if ((rc = grouped_check("conv2d_grouped_wgrad", C, groups, ksize, stride))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const WgradPlan pl = plan_wgrad(B, H, W, 64, C, ksize, stride, true);
  const size_t need = wgrad_bytes(pl, C, 64);
  B200_REQUIRE(workspace != nullptr && workspace_bytes >= need, "conv2d_grouped_wgrad: workspace too small (%zu < %zu)",
               workspace_bytes, need);
  WgradParams p = wgrad_params(pl, C, 64, workspace);
  p.num_taps = pl.taps / 3;   // work items of three taps each
  p.n_cols = p.Cin = 3 * 64;
  if ((rc = setup_wgrad_maps(p, pl, dy, x, B, H, W, C, C, ksize, stride))) return rc;
  if ((rc = launch_wgrad<384, true>(p, st))) return rc;
  const long long total = static_cast<long long>(C) * (C / groups) * pl.taps;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  B200_CHECK_CUDA(launch_pdl(wgrad_reduce_grouped_kernel, dim3(blocks), dim3(256), 0, st, static_cast<const float*>(p.partial),
                             dw, pl.splits, C, C / groups, pl.taps, accumulate));
  B200_LAUNCHED();
  return OK;
}

}  // extern "C"
