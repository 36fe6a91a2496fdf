// ConvNeXt-specific passes: 7x7 depthwise convolution forward / backward (CUDA cores, register-tiled strips of 4 output
// pixels x 4 channels, NHWC), global average pool of the fp32 stream, column sums of an elementwise product (layer-scale
// gradient) and the fused AdamW update.
//
// Reference: Block.forward of classification/convNext/models/networks.py:92-105 (dwconv 7x7 pad 3 groups=dim WITH bias ->
// LN -> Linear -> GELU -> Linear -> gamma * x -> shortcut add), ConvNeXt.forward_features :160-165 (x.mean([-2,-1]) -> LN),
// AdamW with decay / no-decay groups: classification/convNext/train.py:96,102 and utils.py:144-166.
#pragma once
#include "common.cuh"

namespace b200 {

template <typename T>
__device__ __forceinline__ float4 ld4(const T* p);
template <>
__device__ __forceinline__ float4 ld4<float>(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}
template <>
__device__ __forceinline__ float4 ld4<__nv_bfloat16>(const __nv_bfloat16* p) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  return make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y));
}
template <typename T>
__device__ __forceinline__ void st4(T* p, const float4& v);
template <>
__device__ __forceinline__ void st4<float>(float* p, const float4& v) {
  *reinterpret_cast<float4*>(p) = v;
}
template <>
__device__ __forceinline__ void st4<__nv_bfloat16>(__nv_bfloat16* p, const float4& v) {
  uint2 u;
  u.x = pack_bf16x2(v.x, v.y);
  u.y = pack_bf16x2(v.z, v.w);
  *reinterpret_cast<uint2*>(p) = u;
}

// out[b,h,w,c] = bias[c] + sum_{kh,kw} wt[tap][c] * in[b, h+dh, w+dw, c]   (dh = kh-3, or 3-kh when FLIP) (+ add)
// wt is the tap-major copy [49][C] of the [C,1,7,7] parameter. One thread: 4 consecutive output pixels x 4 channels.
template <typename TIn, typename TOut, bool FLIP>
__global__ void __launch_bounds__(128) dwconv7_kernel(const TIn* __restrict__ in, const float* __restrict__ wt,
                                                       const float* __restrict__ bias, const TOut* __restrict__ add,
                                                       TOut* __restrict__ out, int B, int H, int W, int C) {
  pdl_wait();
  const int c4n = C >> 2;
  const int wstrips = (W + 3) >> 2;
  const long long total = static_cast<long long>(B) * H * wstrips * c4n;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % c4n) * 4;
    long long t = i / c4n;
    const int w0 = static_cast<int>(t % wstrips) * 4;
    t /= wstrips;
    const int h = static_cast<int>(t % H);
    const int b = static_cast<int>(t / H);
    float4 acc[4];
    const float4 bz = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = bz;
#pragma unroll 1
    for (int kh = 0; kh < 7; ++kh) {
      const int hh = h + kh - 3;
      if (hh < 0 || hh >= H) continue;
      const int krow = FLIP ? (6 - kh) : kh;
      float4 wv[7];
#pragma unroll
      for (int kw = 0; kw < 7; ++kw)
        wv[kw] = __ldg(reinterpret_cast<const float4*>(wt + static_cast<long long>(krow * 7 + (FLIP ? 6 - kw : kw)) * C + c));
      const TIn* rowp = in + ((static_cast<long long>(b) * H + hh) * W) * C + c;
#pragma unroll
      for (int iw = 0; iw < 10; ++iw) {
        const int ww = w0 + iw - 3;
        if (ww < 0 || ww >= W) continue;
        const float4 xv = ld4<TIn>(rowp + static_cast<long long>(ww) * C);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int kw = iw - j;
          if (kw >= 0 && kw < 7) {
            acc[j].x = fmaf(xv.x, wv[kw].x, acc[j].x);
            acc[j].y = fmaf(xv.y, wv[kw].y, acc[j].y);
            acc[j].z = fmaf(xv.z, wv[kw].z, acc[j].z);
            acc[j].w = fmaf(xv.w, wv[kw].w, acc[j].w);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (w0 + j < W) {
        const long long o = ((static_cast<long long>(b) * H + h) * W + w0 + j) * C + c;
        float4 v = acc[j];
        if (add != nullptr) {
          const float4 a = ld4<TOut>(add + o);
          v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
        }
        st4<TOut>(out + o, v);
      }
    }
  }
}

// Weight gradient partials: part[blockIdx.y][tap][c] = sum over this block's (b,h) rows of du[b,h,w,c] * x[b,h+kh-3,w+kw-3,c].
// Block = 32 channel-quads x 7 kernel rows (224 threads); a thread keeps its 7 (kw) x 4 (channel) accumulators in registers.
__global__ void __launch_bounds__(224) dwconv7_wgrad_kernel(const __nv_bfloat16* __restrict__ du, const float* __restrict__ x,
                                                            float* __restrict__ part, int B, int H, int W, int C,
                                                            int rows_per_block) {
  pdl_wait();
  const int cq = blockIdx.x * 32 + (threadIdx.x & 31);
  const int kh = threadIdx.x >> 5;  // 0..6
  const int c = cq * 4;
  const bool active = c < C;
  float4 acc[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  const long long nrows = static_cast<long long>(B) * H;
  const long long r0 = static_cast<long long>(blockIdx.y) * rows_per_block;
  const long long r1 = min(nrows, r0 + rows_per_block);
  if (active) {
    for (long long r = r0; r < r1; ++r) {
      const int h = static_cast<int>(r % H);
      const long long b = r / H;
      const int hh = h + kh - 3;
      if (hh < 0 || hh >= H) continue;
      const __nv_bfloat16* dup = du + (r * W) * C + c;
      const float* xp = x + ((b * H + hh) * W) * C + c;
      for (int w0 = 0; w0 < W; w0 += 4) {
        float4 d[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
          d[j] = (w0 + j < W) ? ld4<__nv_bfloat16>(dup + static_cast<long long>(w0 + j) * C) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int iw = 0; iw < 10; ++iw) {
          const int ww = w0 + iw - 3;
          if (ww < 0 || ww >= W) continue;
          const float4 xv = __ldg(reinterpret_cast<const float4*>(xp + static_cast<long long>(ww) * C));
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int kw = iw - j;
            if (kw >= 0 && kw < 7) {
              acc[kw].x = fmaf(d[j].x, xv.x, acc[kw].x);
              acc[kw].y = fmaf(d[j].y, xv.y, acc[kw].y);
              acc[kw].z = fmaf(d[j].z, xv.z, acc[kw].z);
              acc[kw].w = fmaf(d[j].w, xv.w, acc[kw].w);
            }
          }
        }
      }
    }
#pragma unroll
    for (int kw = 0; kw < 7; ++kw)
      *reinterpret_cast<float4*>(part + (static_cast<long long>(blockIdx.y) * 49 + kh * 7 + kw) * C + c) = acc[kw];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Tiled 7x7 depthwise kernels (H, W multiples of 14 and C a multiple of 32 - every ConvNeXt stage but the 7x7 one).
// A CTA stages the fp32 halo (20 x 20 pixels x 32 channels, zero padded) of a 14 x 14 output tile in shared memory; each of
// its 4 warps owns a 7 x 7 output block and each lane ONE channel, so every shared load is a conflict-free 128-byte row
// and the 49 filter taps of the lane's channel live in registers. Per input row a thread issues 13 shared loads for up
// to 343 FMAs (the naive strip kernel above: ~1 load per 11 FMAs from L1): the loop is FP32-FMA bound.
constexpr int kDwTile = 14, kDwHalo = 20, kDwCh = 32;

// 16 / 8-byte asynchronous global -> shared copies; src_bytes == 0 zero-fills the destination (the conv's zero padding)
__device__ __forceinline__ void dw_cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void dw_cp_async8(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void dw_cp_async_wait() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

// Stage ROWS x COLS pixels x 32 channels starting at (h0, w0) (zero outside the image) for a 128-thread CTA.
// fp32 sources are copied asynchronously as they are; bf16 sources are widened to fp32 on the way (RAW = keep bf16).
template <typename TIn, int ROWS, int COLS, bool RAW = false>
__device__ __forceinline__ void dw_fill_tile(void* s, const TIn* __restrict__ src, long long b, int h0, int w0, int H, int W,
                                             int C, int c0) {
  constexpr int N = ROWS * COLS * (kDwCh / 4);
  const int part = threadIdx.x & 7;
  const TIn* base = src + (b * H * W) * C + c0 + part * 4;
  const uint32_t s_u32 = static_cast<uint32_t>(__cvta_generic_to_shared(s));
#pragma unroll 5
  for (int k = threadIdx.x; k < N; k += 128) {
    const int pix = k >> 3;
    const int py = pix / COLS, px = pix - py * COLS;
    const int hh = h0 + py, ww = w0 + px;
    const bool ok = hh >= 0 && hh < H && ww >= 0 && ww < W;
    const TIn* g = ok ? base + (static_cast<long long>(hh) * W + ww) * C : base;
    if constexpr (sizeof(TIn) == 4) {
      dw_cp_async16(s_u32 + (pix * kDwCh + part * 4) * 4, g, ok ? 16 : 0);
    } else if constexpr (RAW) {
      dw_cp_async8(s_u32 + (pix * kDwCh + part * 4) * 2, g, ok ? 8 : 0);
    } else {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok) v = ld4<TIn>(g);
      *reinterpret_cast<float4*>(static_cast<float*>(s) + pix * kDwCh + part * 4) = v;
    }
  }
}

template <typename TIn, typename TOut, bool FLIP>
__global__ void __launch_bounds__(128, 4) dwconv7_tile_kernel(const TIn* __restrict__ in, const float* __restrict__ wt,
                                                              const float* __restrict__ bias, const TOut* __restrict__ add,
                                                              TOut* __restrict__ out, int B, int H, int W, int C) {
  pdl_wait();
  extern __shared__ float dw_smem[];  // [20][20][32]
  const int cgroups = C / kDwCh, tiles_w = W / kDwTile, tiles_h = H / kDwTile;
  int t = blockIdx.x;
  const int cg = t % cgroups;
  t /= cgroups;
  const int tw = t % tiles_w;
  t /= tiles_w;
  const int th = t % tiles_h;
  const long long b = t / tiles_h;
  const int c0 = cg * kDwCh;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  dw_fill_tile<TIn, kDwHalo, kDwHalo>(dw_smem, in, b, th * kDwTile - 3, tw * kDwTile - 3, H, W, C, c0);
  float w[49];
#pragma unroll
  for (int k = 0; k < 49; ++k) w[k] = __ldg(wt + static_cast<long long>(FLIP ? 48 - k : k) * C + c0 + lane);
  const float bz = bias ? __ldg(bias + c0 + lane) : 0.f;
  dw_cp_async_wait();
  __syncthreads();
  const int by = warp >> 1, bx = warp & 1;
  const float* sp = dw_smem + ((by * 7) * kDwHalo + bx * 7) * kDwCh + lane;
  float acc[7][7];
#pragma unroll
  for (int r = 0; r < 7; ++r)
#pragma unroll
    for (int q = 0; q < 7; ++q) acc[r][q] = bz;
#pragma unroll
  for (int i = 0; i < 13; ++i) {
    float xin[13];
#pragma unroll
    for (int j = 0; j < 13; ++j) xin[j] = sp[(i * kDwHalo + j) * kDwCh];
#pragma unroll
    for (int kh = 0; kh < 7; ++kh) {
      const int r = i - kh;
      if (r < 0 || r >= 7) continue;
#pragma unroll
      for (int q = 0; q < 7; ++q)
#pragma unroll
        for (int kw = 0; kw < 7; ++kw) acc[r][q] = fmaf(w[kh * 7 + kw], xin[q + kw], acc[r][q]);
    }
  }
  const int oh = th * kDwTile + by * 7, ow = tw * kDwTile + bx * 7;
#pragma unroll
  for (int r = 0; r < 7; ++r) {
#pragma unroll
    for (int q = 0; q < 7; ++q) {
      const long long o = ((b * H + oh + r) * W + ow + q) * C + c0 + lane;
      float v = acc[r][q];
      if (add != nullptr) v += static_cast<float>(add[o]);
      out[o] = static_cast<TOut>(v);
    }
  }
}

// Weight gradient on the same tiling: acc[kh][kw] += du[r][q] * x[r+kh][q+kw] over the lane's channel; a CTA walks
// `tiles_per_cta` tiles of one 32-channel group and writes one partial row part[blockIdx.y][tap][c].
__global__ void __launch_bounds__(128, 3) dwconv7_wgrad_tile_kernel(const __nv_bfloat16* __restrict__ du,
                                                                    const float* __restrict__ x, float* __restrict__ part,
                                                                    int B, int H, int W, int C, int tiles_per_cta) {
  pdl_wait();
  extern __shared__ float dw_smem[];  // x halo fp32 [20][20][32] | du tile bf16 [14][14][32]
  float* s_x = dw_smem;
  const __nv_bfloat16* s_d = reinterpret_cast<const __nv_bfloat16*>(dw_smem + kDwHalo * kDwHalo * kDwCh);
  const int tiles_w = W / kDwTile, tiles_h = H / kDwTile;
  const long long ntiles = static_cast<long long>(B) * tiles_h * tiles_w;
  const int c0 = blockIdx.x * kDwCh;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int by = warp >> 1, bx = warp & 1;
  float acc[49];
#pragma unroll
  for (int k = 0; k < 49; ++k) acc[k] = 0.f;
  const long long t0 = static_cast<long long>(blockIdx.y) * tiles_per_cta;
  const long long t1 = min(ntiles, t0 + tiles_per_cta);
  for (long long t = t0; t < t1; ++t) {
    const int tw = static_cast<int>(t % tiles_w);
    const int th = static_cast<int>((t / tiles_w) % tiles_h);
    const long long b = t / (static_cast<long long>(tiles_w) * tiles_h);
    __syncthreads();  // previous tile fully consumed
    dw_fill_tile<float, kDwHalo, kDwHalo>(s_x, x, b, th * kDwTile - 3, tw * kDwTile - 3, H, W, C, c0);
    dw_fill_tile<__nv_bfloat16, kDwTile, kDwTile, true>(dw_smem + kDwHalo * kDwHalo * kDwCh, du, b, th * kDwTile,
                                                        tw * kDwTile, H, W, C, c0);
    dw_cp_async_wait();
    __syncthreads();
    float d[7][7];
#pragma unroll
    for (int r = 0; r < 7; ++r)
#pragma unroll
      for (int q = 0; q < 7; ++q) d[r][q] = __bfloat162float(s_d[((by * 7 + r) * kDwTile + bx * 7 + q) * kDwCh + lane]);
    const float* sp = s_x + ((by * 7) * kDwHalo + bx * 7) * kDwCh + lane;
#pragma unroll
    for (int i = 0; i < 13; ++i) {
      float xin[13];
#pragma unroll
      for (int j = 0; j < 13; ++j) xin[j] = sp[(i * kDwHalo + j) * kDwCh];
#pragma unroll
      for (int kh = 0; kh < 7; ++kh) {
        const int r = i - kh;
        if (r < 0 || r >= 7) continue;
#pragma unroll
        for (int q = 0; q < 7; ++q)
#pragma unroll
          for (int kw = 0; kw < 7; ++kw) acc[kh * 7 + kw] = fmaf(d[r][q], xin[q + kw], acc[kh * 7 + kw]);
      }
    }
  }
  // fold the four warps (fixed order: deterministic), then one partial row per CTA
  __syncthreads();
  float* red = dw_smem;  // [4][49][32]
#pragma unroll
  for (int k = 0; k < 49; ++k) red[(warp * 49 + k) * 32 + lane] = acc[k];
  __syncthreads();
  for (int k = warp; k < 49; k += 4) {
    const float v = red[(0 * 49 + k) * 32 + lane] + red[(1 * 49 + k) * 32 + lane] + red[(2 * 49 + k) * 32 + lane] +
                    red[(3 * 49 + k) * 32 + lane];
    part[(static_cast<long long>(blockIdx.y) * 49 + k) * C + c0 + lane] = v;
  }
}

// dW[c][tap] (+)= sum_t part[t][tap][c]   ([C,1,7,7] parameter layout)
__global__ void dwconv7_wgrad_finalize_kernel(const float* __restrict__ part, int T, int C, float* __restrict__ dw,
                                              int accumulate) {
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over tap*C + c (coalesced reads)
  if (i >= 49 * C) return;
  const int c = i % C, tap = i / C;
  float s = 0.f;
  for (int t = 0; t < T; ++t) s += part[static_cast<long long>(t) * 49 * C + i];
  float* o = dw + static_cast<long long>(c) * 49 + tap;
  *o = accumulate ? *o + s : s;
}

// [C,1,7,7] fp32 parameter -> tap-major [49][C] copy
__global__ void dwconv7_pack_kernel(const float* __restrict__ w, float* __restrict__ wt, int C) {
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 49 * C) return;
  const int c = i % C, tap = i / C;
  wt[i] = w[static_cast<long long>(c) * 49 + tap];
}

// Global average pool of a [B][HW][C] tensor (fp32 or bf16) -> fp32 [B][C]; backward broadcasts g/HW (bf16 out).
template <typename TIn>
__global__ void avgpool_any_fwd_kernel(const TIn* __restrict__ x, float* __restrict__ y, int B, int HW, int C) {
  pdl_wait();
  const int c4n = C >> 2;
  const long long total = static_cast<long long>(B) * c4n;
  const float inv = 1.0f / HW;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % c4n) * 4;
    const long long b = i / c4n;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = 0; p < HW; ++p) {
      const float4 v = ld4<TIn>(x + (b * HW + p) * C + c);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    *reinterpret_cast<float4*>(y + b * C + c) = make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
  }
}

// partial[slice][2][cols]: plane 0 = column sums of a[r][c] * b[r][c] (b optional), plane 1 = 0
__global__ void colsum_prod_partial_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ bmat,
                                           long long rows, long long ld, int cols, float* __restrict__ partial) {
  pdl_wait();
  __shared__ float sh[4][64];
  const int cx = threadIdx.x & 63, ry = threadIdx.x >> 6;
  const int c = blockIdx.x * 64 + cx;
  const int S = gridDim.y;
  const long long chunk = (rows + S - 1) / S;
  const long long r0 = blockIdx.y * chunk, r1 = min(rows, r0 + chunk);
  float s = 0.f;
  if (c < cols)
    for (long long r = r0 + ry; r < r1; r += 4) {
      const float av = __bfloat162float(a[r * ld + c]);
      s += bmat ? av * __bfloat162float(bmat[r * ld + c]) : av;
    }
  sh[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && c < cols) {
    partial[(static_cast<long long>(blockIdx.y) * 2 + 0) * cols + c] = sh[0][cx] + sh[1][cx] + sh[2][cx] + sh[3][cx];
    partial[(static_cast<long long>(blockIdx.y) * 2 + 1) * cols + c] = 0.f;
  }
}

// Layer-scale bookkeeping of a ConvNeXt block, from the UNSCALED weight gradient G = g^T post of pwconv2 (out = gamma*(W2 post + b2)):
//   dgamma[c] = sum_k W2[c,k] G[c,k] + b2[c] * gsum[c] ;  dW2[c,:] = gamma[c] * G[c,:] ;  db2[c] = gamma[c] * gsum[c]
// (gsum = column sums of the upstream gradient g). One block per output channel c.
__global__ void layerscale_grads_kernel(const float* __restrict__ G, const float* __restrict__ W2,
                                        const float* __restrict__ b2, const float* __restrict__ gsum,
                                        const float* __restrict__ gamma, float* __restrict__ dW2, float* __restrict__ db2,
                                        float* __restrict__ dgamma, int C, int K) {
  pdl_wait();
  __shared__ float sh[8];
  const int c = blockIdx.x;
  const float ga = gamma ? gamma[c] : 1.0f;
  float dot = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float gv = G[static_cast<long long>(c) * K + k];
    dot = fmaf(W2[static_cast<long long>(c) * K + k], gv, dot);
    dW2[static_cast<long long>(c) * K + k] = ga * gv;
  }
  dot = warp_sum(dot);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = dot;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += sh[i];
    const float gs = gsum[c];
    if (dgamma) dgamma[c] = t + (b2 ? b2[c] : 0.f) * gs;
    if (db2) db2[c] = ga * gs;
  }
}

// Fused AdamW over flat fp32 arenas (torch.optim.AdamW semantics, amsgrad off):
//   p *= 1 - lr*wd[i];  m = b1*m + (1-b1)*g;  v = b2*v + (1-b2)*g*g;  p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps)
// hyper (device) = {lr, 1 - b1^t, 1 - b2^t}: kept on the device so a captured CUDA graph follows the schedule.
// hyper = {lr, 1-beta1^t, 1-beta2^t, beta1^t, beta2^t}: advances t by one (single thread), entirely on the device so the
// optimizer step can be replayed inside a CUDA graph.
__global__ void adamw_tick_kernel(float* __restrict__ hyper, float beta1, float beta2) {
  pdl_wait();
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const float p1 = hyper[3] * beta1, p2 = hyper[4] * beta2;
    hyper[3] = p1;
    hyper[4] = p2;
    hyper[1] = 1.0f - p1;
    hyper[2] = 1.0f - p2;
  }
}

// Global-norm gradient clipping (torch.nn.utils.clip_grad_norm_, used by the Swin recipe:
// classification/swin_transformer/utils/torch_utils.py:303-317, main.py:197) without a pass that rewrites the gradients:
//   pass 1: per-block sums of squares of the flat gradient arena;  pass 2 (one block): total_norm = gscale * sqrt(sum),
//   clip[0] = min(1, max_norm / (total_norm + 1e-6)), clip[1] = total_norm;  the optimizer kernels multiply by clip[0].
__global__ void __launch_bounds__(256) grad_sumsq_partial_kernel(const float* __restrict__ g, long long n,
                                                                 float* __restrict__ partial) {
  pdl_wait();
  __shared__ float red[8];
  float s = 0.f;
  const long long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 x = __ldg(g4 + i);
    s = fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, fmaf(x.w, x.w, s))));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float x = g[(n4 << 2) + threadIdx.x];
    s = fmaf(x, x, s);
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    partial[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(256) grad_clip_coef_kernel(const float* __restrict__ partial, int nblocks, float gscale,
                                                             float max_norm, float* __restrict__ clip) {
  pdl_wait();
  __shared__ double red[8];
  double s = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) s += static_cast<double>(partial[i]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    const float norm = gscale * static_cast<float>(sqrt(t));
    clip[0] = fminf(1.0f, max_norm / (norm + 1e-6f));
    clip[1] = norm;
  }
}

__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, const float* __restrict__ wd, long long n,
                             const float* __restrict__ hyper, float beta1, float beta2, float eps, float gscale,
                             const float* __restrict__ clip) {
  pdl_wait();
  if (clip != nullptr) gscale *= __ldg(clip);
  const float lr = __ldg(hyper), bc1 = __ldg(hyper + 1), bc2 = __ldg(hyper + 2);
  const float step = lr / bc1, rsq = rsqrtf(bc2);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float gi = g[i] * gscale;
    float pi = p[i] * (1.0f - lr * wd[i]);
    const float mi = fmaf(beta1, m[i], (1.0f - beta1) * gi);
    const float vi = fmaf(beta2, v[i], (1.0f - beta2) * gi * gi);
    m[i] = mi;
    v[i] = vi;
    pi -= step * mi / (sqrtf(vi) * rsq + eps);
    p[i] = pi;
  }
}

}  // namespace b200
