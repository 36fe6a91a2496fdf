// HBM-bound passes of the ViT / Swin / ConvNeXt paths: LayerNorm forward/backward (one warp per token row, statistics in
// fp32 registers), patch extraction from the user's NCHW fp32 batch, class-token row assembly.
//
// Reference semantics: nn.LayerNorm over the last dim (biased variance), eps 1e-6 in ViT
// (classification/vision_transformer/vit_model.py:194), 1e-5 in Swin (classification/swin_transformer/models/swin_transformer.py:509);
// PatchEmbed = Conv2d(3, D, p, p) -> flatten -> transpose (vit_model.py:56-66); cls/pos (vit_model.py:244-250).
#pragma once
#include "common.cuh"


namespace b200 {

template <typename T>
__device__ __forceinline__ void load_row8(const T* p, float (&f)[8]);
template <>
__device__ __forceinline__ void load_row8<float>(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <>
__device__ __forceinline__ void load_row8<__nv_bfloat16>(const __nv_bfloat16* p, float (&f)[8]) {
  unpack8(*reinterpret_cast<const uint4*>(p), f);
}
template <typename T>
__device__ __forceinline__ void store_row8(T* p, const float (&f)[8]);
template <>
__device__ __forceinline__ void store_row8<float>(float* p, const float (&f)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *(reinterpret_cast<float4*>(p) + 1) = make_float4(f[4], f[5], f[6], f[7]);
}
template <>
__device__ __forceinline__ void store_row8<__nv_bfloat16>(__nv_bfloat16* p, const float (&f)[8]) {
  *reinterpret_cast<uint4*>(p) = pack8(f);
}

// Sum over the LPR lanes (a power of two) that share a row.
template <int LPR>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int off = LPR / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// y = (x - mean) * rstd * gamma + beta.  LPR lanes per row (32 / LPR rows per warp: narrow rows such as C = 96 keep every
// lane busy); MAXV = max 8-element vectors per lane (C <= 8 * LPR * MAXV).
template <typename TIn, typename TY, int MAXV, int LPR = 32>
__global__ void layernorm_fwd_kernel(const TIn* __restrict__ x, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, TY* __restrict__ y,
                                     float* __restrict__ mean_out, float* __restrict__ rstd_out, long long rows, int C,
                                     float eps) {
  pdl_wait();
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane % LPR, grp = lane / LPR;
  const int nvec = C >> 3;
  const long long warp0 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long rb = warp0 * RPW; rb < rows; rb += nwarps * RPW) {
    const long long r = rb + grp;
    const bool live = r < rows;
    float v[MAXV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * LPR + sub;
      if (live && vi < nvec) {
        load_row8<TIn>(x + r * C + vi * 8, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    }
    s = group_sum<LPR>(s);
    const float mean = s / C;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * LPR + sub;
      if (live && vi < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          ss = fmaf(d, d, ss);
        }
      }
    }
    ss = group_sum<LPR>(ss);
    const float rstd = rsqrtf(ss / C + eps);
    if (live && sub == 0) {
      if (mean_out) mean_out[r] = mean;
      if (rstd_out) rstd_out[r] = rstd;
    }
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * LPR + sub;
      if (live && vi < nvec) {
        float g[8], b[8], o[8];
        load8f(gamma + vi * 8, g);
        load8f(beta + vi * 8, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf((v[i][j] - mean) * rstd, g[j], b[j]);
        store_row8<TY>(y + r * C + vi * 8, o);
      }
    }
  }
}

// dx = rstd * (dy*gamma - mean_c(dy*gamma) - xhat * mean_c(dy*gamma*xhat)) (+ add);  partial[block][2][C] = (sum dy, sum dy*xhat)
//   * every load of a row - x, dy and a bf16 residual gradient `add` - is issued before anything is computed, so each row
//     costs one exposed DRAM round trip.  The raw words stay in registers (x fp32 / dy, add bf16 packed) and xhat,
//     dy*gamma are recomputed for the output phase - two more FMAs per element;
//   * the per-column parameter-gradient accumulators live in shared memory (one private [2][C] slice per warp) so that the
//     register budget only has to hold one row.  Each [C] is split into a plane of the low and a plane of the high float4 of
//     every 8-channel vector, so that consecutive lanes touch consecutive 16-byte words (no bank conflict on the float4
//     read-modify-writes).
template <typename TIn, typename TOut, int MAXV, int LPR = 32>
__global__ void __launch_bounds__(256, 3)
layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const TIn* __restrict__ x, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const float* __restrict__ gamma, const TOut* __restrict__ add,
                     TOut* __restrict__ dx, float* __restrict__ partial, long long rows, int C) {
  pdl_wait();
  extern __shared__ float red[];  // [warps][rows per warp][2][C], each [C] = low float4 plane | high float4 plane
  constexpr int RPW = 32 / LPR;
  constexpr bool kEarlyAdd = sizeof(TOut) == 2;   // bf16 residual gradient: 4 registers per vector, fetched up front
  constexpr int XW = sizeof(TIn) == 4 ? 2 : 1;    // 16-byte words per 8-element vector of x
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int sub = lane % LPR, grp = lane / LPR;
  const int nvec = C >> 3, half = C >> 1;
  float* mine = red + (static_cast<long long>(warp) * RPW + grp) * 2 * C;
  for (int i = sub; i < 2 * C; i += LPR) mine[i] = 0.f;
  __syncwarp();
  const long long warp0 = blockIdx.x * static_cast<long long>(nw) + warp;
  const long long nwarps = static_cast<long long>(gridDim.x) * nw;
  auto decode_x = [](const uint4 (&w)[XW], float (&f)[8]) {
    if constexpr (XW == 2) {
      f[0] = __uint_as_float(w[0].x); f[1] = __uint_as_float(w[0].y); f[2] = __uint_as_float(w[0].z); f[3] = __uint_as_float(w[0].w);
      f[4] = __uint_as_float(w[1].x); f[5] = __uint_as_float(w[1].y); f[6] = __uint_as_float(w[1].z); f[7] = __uint_as_float(w[1].w);
    } else {
      unpack8(w[0], f);
    }
  };
  for (long long rb = warp0 * RPW; rb < rows; rb += nwarps * RPW) {
    const long long r = rb + grp;
    const bool live = r < rows;
    uint4 xr[MAXV][XW], dr[MAXV], ar[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * LPR + sub;
      if (live && vi < nvec) {
        const uint4* xp = reinterpret_cast<const uint4*>(x + r * C + vi * 8);
#pragma unroll
        for (int k = 0; k < XW; ++k) xr[i][k] = __ldg(xp + k);
        dr[i] = __ldg(reinterpret_cast<const uint4*>(dy + r * C + vi * 8));
        if constexpr (kEarlyAdd) {
          if (add != nullptr) ar[i] = __ldg(reinterpret_cast<const uint4*>(add + r * C + vi * 8));
        }
      }
    }
    const float mu = live ? mean[r] : 0.f, rs = live ? rstd[r] : 0.f;
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * LPR + sub;
      if (live && vi < nvec) {
        float xv[8], dv[8], g[8];
        decode_x(xr[i], xv);
        unpack8(dr[i], dv);
        load8f(gamma + vi * 8, g);
        float4* ab = reinterpret_cast<float4*>(mine) + vi;            // d beta : low plane, high plane at + half floats
        float4* ag = reinterpret_cast<float4*>(mine + C) + vi;        // d gamma
        float4 b0 = ab[0], b1 = ab[half >> 2], g0 = ag[0], g1 = ag[half >> 2];
        float xh[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[j] = (xv[j] - mu) * rs;
          const float dgj = dv[j] * g[j];
          s1 += dgj;
          s2 = fmaf(dgj, xh[j], s2);
        }
        b0.x += dv[0]; b0.y += dv[1]; b0.z += dv[2]; b0.w += dv[3];
        b1.x += dv[4]; b1.y += dv[5]; b1.z += dv[6]; b1.w += dv[7];
        g0.x = fmaf(dv[0], xh[0], g0.x); g0.y = fmaf(dv[1], xh[1], g0.y);
        g0.z = fmaf(dv[2], xh[2], g0.z); g0.w = fmaf(dv[3], xh[3], g0.w);
        g1.x = fmaf(dv[4], xh[4], g1.x); g1.y = fmaf(dv[5], xh[5], g1.y);
        g1.z = fmaf(dv[6], xh[6], g1.z); g1.w = fmaf(dv[7], xh[7], g1.w);
        ab[0] = b0; ab[half >> 2] = b1; ag[0] = g0; ag[half >> 2] = g1;
      }
    }
    s1 = group_sum<LPR>(s1) / C;
    s2 = group_sum<LPR>(s2) / C;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * LPR + sub;
      if (live && vi < nvec) {
        float xv[8], dv[8], g[8], o[8];
        decode_x(xr[i], xv);
        unpack8(dr[i], dv);
        load8f(gamma + vi * 8, g);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (dv[j] * g[j] - s1 - (xv[j] - mu) * rs * s2);
        if (add != nullptr) {
          float a[8];
          if constexpr (kEarlyAdd)
            unpack8(ar[i], a);
          else
            load_row8<TOut>(add + r * C + vi * 8, a);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += a[j];
        }
        store_row8<TOut>(dx + r * C + vi * 8, o);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) {
    const int sec = c >= C ? C : 0, cc = c - sec, j = cc & 7;
    const int pos = sec + (j < 4 ? (cc >> 3) * 4 + j : half + (cc >> 3) * 4 + j - 4);
    float s = 0.f;
    for (int w = 0; w < nw * RPW; ++w) s += red[static_cast<long long>(w) * 2 * C + pos];
    partial[static_cast<long long>(blockIdx.x) * 2 * C + c] = s;
  }
}

// Swin PatchMerging front half (classification/swin_transformer/models/swin_transformer.py:333-343): gather the 2x2 neighbourhood
// [x(0,0), x(1,0), x(0,1), x(1,1)] (row offset first, as the reference concatenates x0,x1,x2,x3) of the fp32 stream
// [B][H][W][C] into one 4C vector and LayerNorm it -> y bf16 [B*(H/2)*(W/2)][4C].  One warp per output row.
template <int MAXV>
__global__ void patch_merge_ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                          const float* __restrict__ beta, __nv_bfloat16* __restrict__ y,
                                          float* __restrict__ mean_out, float* __restrict__ rstd_out, int B, int H, int W,
                                          int C, float eps) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int C4 = 4 * C, nvec = C4 >> 3, cvec = C >> 3;
  const int Ho = H / 2, Wo = W / 2;
  const long long rows = static_cast<long long>(B) * Ho * Wo;
  const long long warp0 = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long r = warp0; r < rows; r += nwarps) {
    const int ow = static_cast<int>(r % Wo);
    const int oh = static_cast<int>((r / Wo) % Ho);
    const long long b = r / (static_cast<long long>(Wo) * Ho);
    float v[MAXV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * 32 + lane;
      if (vi < nvec) {
        const int seg = vi / cvec, cv = vi - seg * cvec;  // seg 0..3 -> (dh, dw) = (seg & 1, seg >> 1)
        const float* src = x + ((b * H + 2 * oh + (seg & 1)) * W + 2 * ow + (seg >> 1)) * C + cv * 8;
        load_row8<float>(src, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    }
    s = warp_sum(s);
    const float mean = s / C4;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * 32 + lane;
      if (vi < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          ss = fmaf(d, d, ss);
        }
      }
    }
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss / C4 + eps);
    if (lane == 0) {
      mean_out[r] = mean;
      rstd_out[r] = rstd;
    }
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * 32 + lane;
      if (vi < nvec) {
        float g[8], bb[8], o[8];
        load8f(gamma + vi * 8, g);
        load8f(beta + vi * 8, bb);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf((v[i][j] - mean) * rstd, g[j], bb[j]);
        *reinterpret_cast<uint4*>(y + r * C4 + vi * 8) = pack8(o);
      }
    }
  }
}

// Backward of the above: dx (bf16 [B][H][W][C], every pixel written exactly once) from dy bf16 [rows][4C];
// partial[block][2][4C] = (sum dy, sum dy*xhat) for the LayerNorm parameter gradients.
template <int MAXV>
__global__ void __launch_bounds__(256, 2)
patch_merge_ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                          const float* __restrict__ rstd, const float* __restrict__ gamma, __nv_bfloat16* __restrict__ dx,
                          float* __restrict__ partial, int B, int H, int W, int C) {
  pdl_wait();
  extern __shared__ float red[];  // [warps][2][4C]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int C4 = 4 * C, nvec = C4 >> 3, cvec = C >> 3;
  const int Ho = H / 2, Wo = W / 2;
  const long long rows = static_cast<long long>(B) * Ho * Wo;
  float* mine = red + static_cast<long long>(warp) * 2 * C4;
  for (int i = lane; i < 2 * C4; i += 32) mine[i] = 0.f;
  __syncwarp();
  const long long warp0 = blockIdx.x * static_cast<long long>(nw) + warp;
  const long long nwarps = static_cast<long long>(gridDim.x) * nw;
  for (long long r = warp0; r < rows; r += nwarps) {
    const int ow = static_cast<int>(r % Wo);
    const int oh = static_cast<int>((r / Wo) % Ho);
    const long long b = r / (static_cast<long long>(Wo) * Ho);
    const float mu = mean[r], rs = rstd[r];
    float xh[MAXV][8], dg[MAXV][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * 32 + lane;
      if (vi < nvec) {
        const int seg = vi / cvec, cv = vi - seg * cvec;
        float xv[8], dv[8], g[8];
        load_row8<float>(x + ((b * H + 2 * oh + (seg & 1)) * W + 2 * ow + (seg >> 1)) * C + cv * 8, xv);
        unpack8(*reinterpret_cast<const uint4*>(dy + r * C4 + vi * 8), dv);
        load8f(gamma + vi * 8, g);
        float4* ab = reinterpret_cast<float4*>(mine + vi * 8);
        float4* ag = reinterpret_cast<float4*>(mine + C4 + vi * 8);
        float4 b0 = ab[0], b1 = ab[1], g0 = ag[0], g1 = ag[1];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] = (xv[j] - mu) * rs;
          dg[i][j] = dv[j] * g[j];
          s1 += dg[i][j];
          s2 = fmaf(dg[i][j], xh[i][j], s2);
        }
        b0.x += dv[0]; b0.y += dv[1]; b0.z += dv[2]; b0.w += dv[3];
        b1.x += dv[4]; b1.y += dv[5]; b1.z += dv[6]; b1.w += dv[7];
        g0.x = fmaf(dv[0], xh[i][0], g0.x); g0.y = fmaf(dv[1], xh[i][1], g0.y);
        g0.z = fmaf(dv[2], xh[i][2], g0.z); g0.w = fmaf(dv[3], xh[i][3], g0.w);
        g1.x = fmaf(dv[4], xh[i][4], g1.x); g1.y = fmaf(dv[5], xh[i][5], g1.y);
        g1.z = fmaf(dv[6], xh[i][6], g1.z); g1.w = fmaf(dv[7], xh[i][7], g1.w);
        ab[0] = b0; ab[1] = b1; ag[0] = g0; ag[1] = g1;
      }
    }
    s1 = warp_sum(s1) / C4;
    s2 = warp_sum(s2) / C4;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int vi = i * 32 + lane;
      if (vi < nvec) {
        const int seg = vi / cvec, cv = vi - seg * cvec;
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (dg[i][j] - s1 - xh[i][j] * s2);
        *reinterpret_cast<uint4*>(dx + ((b * H + 2 * oh + (seg & 1)) * W + 2 * ow + (seg >> 1)) * C + cv * 8) = pack8(o);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C4; c += blockDim.x) {
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += red[static_cast<long long>(w) * 2 * C4 + c];
    partial[static_cast<long long>(blockIdx.x) * 2 * C4 + c] = s;
  }
}

// Patch extraction: x fp32 NCHW [B][Cin][H][W] -> a bf16 [B*(H/ps)*(W/ps)][Cin*ps*ps], k = c*ps*ps + kh*ps + kw
// (the flattening order of an OIHW conv weight, so the weight matrix is weight.view(D, -1) unchanged). ps % 8 == 0... or 4.
__global__ void patchify_nchw_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ a, int B, int Cin, int H,
                                     int W, int ps) {
  pdl_wait();
  const int ph = H / ps, pw = W / ps;
  const int K = Cin * ps * ps;
  const int kv = K / 4;  // 4 consecutive kw per thread (ps is a multiple of 4)
  const long long total = static_cast<long long>(B) * ph * pw * kv;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k4 = static_cast<int>(i % kv);
    long long t = i / kv;
    const int px = static_cast<int>(t % pw);
    t /= pw;
    const int py = static_cast<int>(t % ph);
    const int b = static_cast<int>(t / ph);
    const int k = k4 * 4;
    const int kw = k % ps, kh = (k / ps) % ps, c = k / (ps * ps);
    const float4 v = __ldg(reinterpret_cast<const float4*>(
        x + ((static_cast<long long>(b) * Cin + c) * H + py * ps + kh) * W + px * ps + kw));
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(a + (static_cast<long long>(b) * ph * pw + py * pw + px) * K + k) = o;
  }
}

// ViT class-token row: tokens[b][0][:] = cls[:] + pos[0][:]   (tokens fp32 [B][T][D])
__global__ void cls_row_kernel(const float* __restrict__ cls, const float* __restrict__ pos, float* __restrict__ tokens,
                               int B, int T, int D) {
  pdl_wait();
  const long long total = static_cast<long long>(B) * D;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(i % D);
    const long long b = i / D;
    tokens[b * T * D + d] = cls[d] + pos[d];
  }
}

// Strided 2-D copy of 16-byte vectors: dst[r][0:cols] = src[r][0:cols] with independent row pitches (in bytes).
__global__ void copy_rows_kernel(const uint8_t* __restrict__ src, long long src_pitch, uint8_t* __restrict__ dst,
                                 long long dst_pitch, long long rows, long long row_bytes) {
  pdl_wait();
  const long long vecs = row_bytes >> 4;
  const long long total = rows * vecs;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / vecs, v = i % vecs;
    *reinterpret_cast<uint4*>(dst + r * dst_pitch + (v << 4)) = __ldg(reinterpret_cast<const uint4*>(src + r * src_pitch + (v << 4)));
  }
}

// Column-sum partials of a bf16 matrix [rows][ld] (bias gradients): partial[slice][2][cols] (second plane zero), folded by
// the BN finalize machinery. 16-byte loads: a thread owns ONE 8-column vector (vector v = tid % vpr of column block
// blockIdx.x) and walks the rows of its slice with 8 independent loads in flight; 256/vpr row lanes per block are folded
// through shared memory. (The first version read one bf16 per thread from ~128 blocks: 1 TB/s; this one is HBM bound.)
__global__ void __launch_bounds__(256) colsum_partial_kernel(const __nv_bfloat16* __restrict__ m, long long rows, long long ld,
                                                             int cols, float* __restrict__ partial) {
  pdl_wait();
  __shared__ float sh[256 * 8];
  const int nvec = cols >> 3;                        // cols is a multiple of 8
  const int vpr = min(nvec - static_cast<int>(blockIdx.x) * 256, 256);   // vectors of this column block
  const int rpi = 256 / vpr;                         // row lanes
  const int v = threadIdx.x % vpr, lane_r = threadIdx.x / vpr;
  const bool active = lane_r < rpi;
  const int S = gridDim.y;
  const long long chunk = (rows + S - 1) / S;
  const long long r0 = blockIdx.y * chunk, r1 = min(rows, r0 + chunk);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (active) {
    const uint4* base = reinterpret_cast<const uint4*>(m) + blockIdx.x * 256 + v;
    const long long ldv = ld >> 3;
    long long r = r0 + lane_r;
    for (; r + 7 * rpi < r1; r += 8 * rpi) {
      uint4 x[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] = __ldg(base + (r + k * rpi) * ldv);
#pragma unroll
      for (int k = 0; k < 8; k += 2) {
        float f0[8], f1[8];
        unpack8(x[k], f0);
        unpack8(x[k + 1], f1);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f0[j] + f1[j];
      }
    }
    for (; r < r1; r += rpi) {
      float f[8];
      unpack8(__ldg(base + r * ldv), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sh[threadIdx.x * 8 + j] = active ? acc[j] : 0.f;
  __syncthreads();
  if (lane_r == 0) {
    for (int k = 1; k < rpi; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += sh[(k * vpr + v) * 8 + j];
    const int c = (blockIdx.x * 256 + v) * 8;
    float* p0 = partial + (static_cast<long long>(blockIdx.y) * 2 + 0) * cols + c;
    float* p1 = partial + (static_cast<long long>(blockIdx.y) * 2 + 1) * cols + c;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      p0[j] = acc[j];
      p1[j] = 0.f;
    }
  }
}

// Sum over the batch of a strided set of rows: out[d] (+)= sum_b g[b*stride_b + d]   (gradient of cls token / pos embed rows)
template <typename T>
__global__ void batch_rowsum_kernel(const T* __restrict__ g, long long stride_b, int B, int D, float* __restrict__ out,
                                    int accumulate) {
  pdl_wait();
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += static_cast<float>(g[b * stride_b + d]);
  out[d] = accumulate ? out[d] + s : s;
}

}  // namespace b200
