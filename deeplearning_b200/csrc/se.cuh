// Squeeze-and-excitation tail of an SE-ResNet block (classification/seNet/models/se_module.py:15-19, se_resnet.py:74-84 /
// :32-42): out = relu(u * gate + identity), u = bn(c) = c * scale + shift, gate = sigmoid(W2 relu(W1 mean_p(u))), one gate
// per (image, channel).  c is the raw bf16 conv output [B][HW][C] (C % 64 == 0), everything per channel or per image fp32.
//
// Streaming passes (squeeze, apply, backward reduce, backward apply) share one thread mapping: a CTA of 256 threads owns one
// image and one 64-channel block; thread t holds channel octet t & 7 (16 bytes, 8 threads cover a 128-byte pixel row) and
// walks pixel rows t >> 3, t >> 3 + 32, ...  Per-(image, channel) coefficients therefore live in registers, and the per-image
// sums of the two reduction passes are finished inside the CTA in a fixed order: no atomics, identical launches agree bit for
// bit.  The fully connected layers and the coefficient algebra are tiny (B x C x Cr) fp32 kernels on the CUDA cores that read
// the fp32 parameters directly.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int kSeRowsPerPass = 32;                     // pixel rows covered by one pass of a 256-thread CTA
constexpr int kSeApplyRows = 4 * kSeRowsPerPass;       // pixel rows per CTA of the apply passes (four in flight per thread)

// Per-CTA combine of the per-thread partial sums of NS quantities: red[NS][32 rows][65] (padded), result for channel t < 64
template <int NS>
__device__ __forceinline__ void se_rows_to_smem(float (*red)[kSeRowsPerPass][65], const float (&a)[NS][8]) {
  const int cg = threadIdx.x & 7, row = threadIdx.x >> 3;
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int j = 0; j < 8; ++j) red[s][row][cg * 8 + j] = a[s][j];
}

// ---- forward, squeeze: csum[b][ch] = sum_p c[b,p,ch]; pool[b][ch] = csum / HW * scale + shift (= mean_p u).
// grid (C / 64, B), block 256.
__global__ void __launch_bounds__(256) se_squeeze_kernel(const uint4* __restrict__ c, const float* __restrict__ scale,
                                                         const float* __restrict__ shift, float* __restrict__ csum,
                                                         float* __restrict__ pool, int HW, int cvec) {
  pdl_wait();
  __shared__ float red[1][kSeRowsPerPass][65];
  const int cg = threadIdx.x & 7, row = threadIdx.x >> 3;
  const int b = blockIdx.y;
  const uint4* src = c + static_cast<long long>(b) * HW * cvec + blockIdx.x * 8 + cg;
  float a[1][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[0][j] = 0.f;
  int p = row;
  for (; p + 3 * kSeRowsPerPass < HW; p += 4 * kSeRowsPerPass) {
    uint4 q[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) q[u] = __ldg(src + static_cast<long long>(p + u * kSeRowsPerPass) * cvec);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float f[8];
      unpack8(q[u], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[0][j] += f[j];
    }
  }
  for (; p < HW; p += kSeRowsPerPass) {
    float f[8];
    unpack8(__ldg(src + static_cast<long long>(p) * cvec), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[0][j] += f[j];
  }
  se_rows_to_smem<1>(red, a);
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
    for (int r = 0; r < kSeRowsPerPass; ++r) s += red[0][r][threadIdx.x];
    const int ch = blockIdx.x * 64 + threadIdx.x;
    const long long o = static_cast<long long>(b) * cvec * 8 + ch;
    csum[o] = s;
    pool[o] = fmaf(s / static_cast<float>(HW), scale[ch], shift[ch]);
  }
}

// ---- forward, excite 1: h[b][n] = relu(sum_k pool[b][k] * w1[n][k]) (w1 = fc.0.weight [Cr][C]).
// grid (ceil(Cr / 8), ceil(B / 8)), block 256: warp w computes output n = 8 * blockIdx.x + w for 8 images, lanes stride K.
__global__ void __launch_bounds__(256) se_fc1_kernel(const float* __restrict__ pool, const float* __restrict__ w1,
                                                     float* __restrict__ h, int B, int C, int Cr) {
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  const int b0 = blockIdx.y * 8;
  if (n >= Cr) return;
  const int nb = min(8, B - b0);
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const float4* wr = reinterpret_cast<const float4*>(w1 + static_cast<long long>(n) * C);
  const float4* xr = reinterpret_cast<const float4*>(pool + static_cast<long long>(b0) * C);
  const int k4 = C / 4;
  for (int k = lane; k < k4; k += 32) {
    const float4 w = __ldg(wr + k);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      // rows past the last image repeat it (always in bounds); their sums are discarded
      const float4 x = __ldg(xr + static_cast<long long>(min(i, nb - 1)) * k4 + k);
      acc[i] = fmaf(x.x, w.x, acc[i]);
      acc[i] = fmaf(x.y, w.y, acc[i]);
      acc[i] = fmaf(x.z, w.z, acc[i]);
      acc[i] = fmaf(x.w, w.w, acc[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float s = warp_sum(acc[i]);
    if (lane == i && i < nb) h[static_cast<long long>(b0 + i) * Cr + n] = fmaxf(s, 0.f);
  }
}

// ---- forward, excite 2: gate[b][n] = sigmoid(sum_j h[b][j] * w2[n][j]) (w2 = fc.2.weight [C][Cr]).
// grid (C / 32, ceil(B / 8)), block 256, dynamic smem (32 * (Cr + 1) + 8 * Cr) floats: the CTA's 32 rows of w2 and 8 rows
// of h are staged, thread (n = t & 31, image = t >> 5) computes one output.
__global__ void __launch_bounds__(256) se_fc2_kernel(const float* __restrict__ h, const float* __restrict__ w2,
                                                     float* __restrict__ gate, int B, int C, int Cr) {
  pdl_wait();
  extern __shared__ float se_smem[];
  float* ws = se_smem;                       // [32][Cr + 1]
  float* hs = se_smem + 32 * (Cr + 1);       // [8][Cr]
  const int n0 = blockIdx.x * 32, b0 = blockIdx.y * 8;
  const int nb = min(8, B - b0);
  const float* wsrc = w2 + static_cast<long long>(n0) * Cr;   // 32 contiguous rows
  for (int i = threadIdx.x; i < 32 * Cr; i += 256) {
    const int r = i / Cr;
    ws[r * (Cr + 1) + (i - r * Cr)] = __ldg(wsrc + i);
  }
  for (int i = threadIdx.x; i < nb * Cr; i += 256) hs[i] = __ldg(h + static_cast<long long>(b0) * Cr + i);
  __syncthreads();
  const int nl = threadIdx.x & 31, bi = threadIdx.x >> 5;
  if (bi >= nb) return;
  const float* wr = ws + nl * (Cr + 1);
  const float* hr = hs + bi * Cr;
  float acc = 0.f;
  for (int k = 0; k < Cr; ++k) acc = fmaf(hr[k], wr[k], acc);
  gate[static_cast<long long>(b0 + bi) * C + n0 + nl] = 1.f / (1.f + expf(-acc));
}

// ---- forward, gated apply: y = relu((c * scale + shift) * gate[b] + identity), bf16.
// grid (ceil(HW / 128), C / 64, B), block 256.
__global__ void __launch_bounds__(256) se_apply_kernel(const uint4* __restrict__ c, const uint4* __restrict__ identity,
                                                       uint4* __restrict__ y, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, const float* __restrict__ gate,
                                                       int HW, int cvec) {
  pdl_wait();
  const int cg = threadIdx.x & 7, row = threadIdx.x >> 3;
  const int b = blockIdx.z, v = blockIdx.y * 8 + cg;
  float sc[8], sh[8], gt[8];
  load8f(scale + v * 8, sc);
  load8f(shift + v * 8, sh);
  load8f(gate + static_cast<long long>(b) * cvec * 8 + v * 8, gt);
  const long long base = static_cast<long long>(b) * HW * cvec + v;
  const int p0 = blockIdx.x * kSeApplyRows + row;
  uint4 xq[4], rq[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int p = p0 + u * kSeRowsPerPass;
    if (p < HW) {
      xq[u] = __ldg(c + base + static_cast<long long>(p) * cvec);
      rq[u] = __ldg(identity + base + static_cast<long long>(p) * cvec);
    }
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int p = p0 + u * kSeRowsPerPass;
    if (p >= HW) break;
    float x[8], r[8];
    unpack8(xq[u], x);
    unpack8(rq[u], r);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = fmaxf(fmaf(fmaf(x[j], sc[j], sh[j]), gt[j], r[j]), 0.f);
    y[base + static_cast<long long>(p) * cvec] = pack8(x);
  }
}

// ---- backward, reduce: dz = g * [y > 0] (bf16, also the identity branch's gradient); A[b][ch] = sum_p dz,
// R[b][ch] = sum_p dz * c.  grid (C / 64, B), block 256.
__global__ void __launch_bounds__(256) se_bwd_reduce_kernel(const uint4* __restrict__ g, const uint4* __restrict__ y,
                                                            const uint4* __restrict__ c, uint4* __restrict__ dz,
                                                            float* __restrict__ A, float* __restrict__ R, int HW, int cvec) {
  pdl_wait();
  __shared__ float red[2][kSeRowsPerPass][65];
  const int cg = threadIdx.x & 7, row = threadIdx.x >> 3;
  const int b = blockIdx.y;
  const long long base = static_cast<long long>(b) * HW * cvec + blockIdx.x * 8 + cg;
  float a[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[0][j] = a[1][j] = 0.f;
  for (int p = row; p < HW; p += 4 * kSeRowsPerPass) {
    uint4 gq[4], yq[4], cq[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int pp = p + u * kSeRowsPerPass;
      if (pp < HW) {
        const long long i = base + static_cast<long long>(pp) * cvec;
        gq[u] = __ldg(g + i);
        yq[u] = __ldg(y + i);
        cq[u] = __ldg(c + i);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int pp = p + u * kSeRowsPerPass;
      if (pp >= HW) break;
      float gv[8], yv[8], xv[8];
      unpack8(gq[u], gv);
      unpack8(yq[u], yv);
      unpack8(cq[u], xv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        gv[j] = yv[j] > 0.f ? gv[j] : 0.f;
        a[0][j] += gv[j];
        a[1][j] = fmaf(gv[j], xv[j], a[1][j]);
      }
      dz[base + static_cast<long long>(pp) * cvec] = pack8(gv);
    }
  }
  se_rows_to_smem<2>(red, a);
  __syncthreads();
  if (threadIdx.x < 128) {
    const int s = threadIdx.x >> 6, chl = threadIdx.x & 63;
    float t = 0.f;
    for (int r = 0; r < kSeRowsPerPass; ++r) t += red[s][r][chl];
    (s == 0 ? A : R)[static_cast<long long>(b) * cvec * 8 + blockIdx.x * 64 + chl] = t;
  }
}

// da[b][ch] = dL/d(gate pre-activation) = (scale * R + shift * A) * gate * (1 - gate), where scale * R + shift * A is
// dL/dgate = sum_p dz * u
__device__ __forceinline__ float se_da(const float* __restrict__ A, const float* __restrict__ R,
                                       const float* __restrict__ gate, const float* __restrict__ scale,
                                       const float* __restrict__ shift, long long bc, int ch) {
  const float gt = __ldg(gate + bc);
  const float dgate = fmaf(__ldg(scale + ch), __ldg(R + bc), __ldg(shift + ch) * __ldg(A + bc));
  return dgate * gt * (1.f - gt);
}

// ---- backward, coefficients 1 (one launch, two kinds of CTA), 256 threads each:
//   blocks [0, nj * nbt):       dh[b][j] = (sum_ch da[b][ch] * w2[ch][j]) * [h > 0]   tile 8 images x 32 j, loop over ch
//   blocks [nj * nbt, + nj*C/32): dW2[ch][j] = sum_b da[b][ch] * h[b][j]            tile 32 ch x 32 j, loop over b
// with nj = ceil(Cr / 32), nbt = ceil(B / 8).  da is recomputed from (A, R, gate) where it is needed.
__global__ void __launch_bounds__(256) se_bwd_gate_kernel(const float* __restrict__ A, const float* __restrict__ R,
                                                          const float* __restrict__ gate, const float* __restrict__ h,
                                                          const float* __restrict__ w2, const float* __restrict__ scale,
                                                          const float* __restrict__ shift, float* __restrict__ dh,
                                                          float* __restrict__ dw2, int B, int C, int Cr) {
  pdl_wait();
  __shared__ float das[8][33];
  __shared__ float ts[32][33];
  const int nj = (Cr + 31) / 32, nbt = (B + 7) / 8;
  const int lo = threadIdx.x & 31, hi = threadIdx.x >> 5;
  const int n_dh = nj * nbt;
  if (static_cast<int>(blockIdx.x) < n_dh) {
    const int j0 = (blockIdx.x % nj) * 32, b0 = (blockIdx.x / nj) * 8;
    const int b = b0 + hi, j = j0 + lo;
    float acc = 0.f;
    for (int k0 = 0; k0 < C; k0 += 32) {
      das[hi][lo] = b < B ? se_da(A, R, gate, scale, shift, static_cast<long long>(b) * C + k0 + lo, k0 + lo) : 0.f;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = hi + 8 * u;   // ch row of the w2 tile
        ts[r][lo] = j < Cr ? __ldg(w2 + static_cast<long long>(k0 + r) * Cr + j) : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < 32; ++k) acc = fmaf(das[hi][k], ts[k][lo], acc);
      __syncthreads();
    }
    if (b < B && j < Cr) {
      const long long o = static_cast<long long>(b) * Cr + j;
      dh[o] = __ldg(h + o) > 0.f ? acc : 0.f;
    }
    return;
  }
  const int t = blockIdx.x - n_dh;
  const int j0 = (t % nj) * 32, c0 = (t / nj) * 32;
  const int j = j0 + lo;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int b0 = 0; b0 < B; b0 += 8) {
    const int b = b0 + hi;
    das[hi][lo] = b < B ? se_da(A, R, gate, scale, shift, static_cast<long long>(b) * C + c0 + lo, c0 + lo) : 0.f;
    ts[hi][lo] = (b < B && j < Cr) ? __ldg(h + static_cast<long long>(b) * Cr + j) : 0.f;
    __syncthreads();
#pragma unroll
    for (int bi = 0; bi < 8; ++bi) {
      const float hv = ts[bi][lo];
#pragma unroll
      for (int u = 0; u < 4; ++u) acc[u] = fmaf(das[bi][hi + 8 * u], hv, acc[u]);
    }
    __syncthreads();
  }
  if (j < Cr) {
#pragma unroll
    for (int u = 0; u < 4; ++u) dw2[static_cast<long long>(c0 + hi + 8 * u) * Cr + j] = acc[u];
  }
}

// ---- backward, coefficients 2: grid (C / 32, 1 + ceil(Cr / 8)), 256 threads, thread (ch = 32 * blockIdx.x + (t & 31),
// hi = t >> 5).  blockIdx.y == 0 (dynamic smem (32 + kSeDhRows) * Cr floats: w1 columns and a chunk of dh rows):
//   dp[b][ch]  = sum_j dh[b][j] * w1[j][ch]                      (dL/dpool), images b = hi + 8 i
//   dbeta      = sum_b (gate * A + dp),  S = sum_b (gate * R + dp * csum / HW)  (= sum du, sum du * c with du = dz*gate + dp/HW)
//   dgamma     = invstd * (S - mean * dbeta),  m1 = dbeta / M,  m2 = dgamma / M   (M = B * HW)
// blockIdx.y >= 1:  dW1[j][ch] = sum_b dh[b][j] * pool[b][ch] for j = 8 (blockIdx.y - 1) + hi
constexpr int kSeDhRows = 32;
__global__ void __launch_bounds__(256) se_bwd_bn_kernel(const float* __restrict__ A, const float* __restrict__ R,
                                                        const float* __restrict__ csum, const float* __restrict__ pool,
                                                        const float* __restrict__ gate, const float* __restrict__ dh,
                                                        const float* __restrict__ w1, const float* __restrict__ mean,
                                                        const float* __restrict__ invstd, float* __restrict__ dp,
                                                        float* __restrict__ dw1, float* __restrict__ dgamma,
                                                        float* __restrict__ dbeta, float* __restrict__ m1,
                                                        float* __restrict__ m2, int B, int HW, int C, int Cr) {
  pdl_wait();
  const int lo = threadIdx.x & 31, hi = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 32, ch = c0 + lo;
  if (blockIdx.y > 0) {
    const int j = (blockIdx.y - 1) * 8 + hi;
    if (j >= Cr) return;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};   // four interleaved partial sums over b (fixed order), loads kept in flight
    int b = 0;
    for (; b + 3 < B; b += 4) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
        acc[u] = fmaf(__ldg(dh + static_cast<long long>(b + u) * Cr + j), __ldg(pool + static_cast<long long>(b + u) * C + ch), acc[u]);
    }
    for (; b < B; ++b) acc[0] = fmaf(__ldg(dh + static_cast<long long>(b) * Cr + j), __ldg(pool + static_cast<long long>(b) * C + ch), acc[0]);
    dw1[static_cast<long long>(j) * C + ch] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
    return;
  }
  extern __shared__ float se_smem[];
  float* w1s = se_smem;                 // [Cr][32]
  float* dhs = se_smem + 32 * Cr;       // [kSeDhRows][Cr]
  __shared__ float red[2][8][32];
  for (int i = threadIdx.x; i < Cr * 32; i += 256) w1s[i] = __ldg(w1 + static_cast<long long>(i >> 5) * C + c0 + (i & 31));
  const float inv_hw = 1.f / static_cast<float>(HW);
  float sb = 0.f, sg = 0.f;
  for (int b0 = 0; b0 < B; b0 += kSeDhRows) {
    const int nrows = min(kSeDhRows, B - b0);
    __syncthreads();   // previous chunk consumed (and w1s staged on the first pass)
    for (int i = threadIdx.x; i < nrows * Cr; i += 256) dhs[i] = __ldg(dh + static_cast<long long>(b0) * Cr + i);
    __syncthreads();
    float acc[kSeDhRows / 8];
#pragma unroll
    for (int r = 0; r < kSeDhRows / 8; ++r) acc[r] = 0.f;
    for (int j = 0; j < Cr; ++j) {
      const float w = w1s[j * 32 + lo];
#pragma unroll
      for (int r = 0; r < kSeDhRows / 8; ++r) acc[r] = fmaf(dhs[(hi + 8 * r) * Cr + j], w, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < kSeDhRows / 8; ++r) {
      if (hi + 8 * r >= nrows) break;
      const long long o = static_cast<long long>(b0 + hi + 8 * r) * C + ch;
      dp[o] = acc[r];
      const float gt = __ldg(gate + o);
      sb += fmaf(gt, __ldg(A + o), acc[r]);
      sg += fmaf(gt, __ldg(R + o), acc[r] * __ldg(csum + o) * inv_hw);
    }
  }
  red[0][hi][lo] = sb;
  red[1][hi][lo] = sg;
  __syncthreads();
  if (hi == 0) {
    for (int i = 1; i < 8; ++i) {
      sb += red[0][i][lo];
      sg += red[1][i][lo];
    }
    const float M = static_cast<float>(B) * static_cast<float>(HW);
    const float dg = static_cast<float>(static_cast<double>(invstd[ch]) *
                                        (static_cast<double>(sg) - static_cast<double>(mean[ch]) * static_cast<double>(sb)));
    dbeta[ch] = sb;
    dgamma[ch] = dg;
    m1[ch] = sb / M;
    m2[ch] = dg / M;
  }
}

// ---- backward, apply: dc = scale * (du - m1 - xhat * m2), du = dz * gate + dp / HW, xhat = (c - mean) * invstd (bf16 out).
// grid (ceil(HW / 128), C / 64, B), block 256.
__global__ void __launch_bounds__(256) se_bwd_apply_kernel(const uint4* __restrict__ dz, const uint4* __restrict__ c,
                                                           uint4* __restrict__ dc, const float* __restrict__ gate,
                                                           const float* __restrict__ dp, const float* __restrict__ scale,
                                                           const float* __restrict__ mean, const float* __restrict__ invstd,
                                                           const float* __restrict__ m1, const float* __restrict__ m2, int HW,
                                                           int cvec) {
  pdl_wait();
  const int cg = threadIdx.x & 7, row = threadIdx.x >> 3;
  const int b = blockIdx.z, v = blockIdx.y * 8 + cg;
  float ka[8], kb[8], kc[8];
  {
    float sc[8], mu[8], is[8], q1[8], q2[8], gt[8], dpv[8];
    load8f(scale + v * 8, sc);
    load8f(mean + v * 8, mu);
    load8f(invstd + v * 8, is);
    load8f(m1 + v * 8, q1);
    load8f(m2 + v * 8, q2);
    load8f(gate + static_cast<long long>(b) * cvec * 8 + v * 8, gt);
    load8f(dp + static_cast<long long>(b) * cvec * 8 + v * 8, dpv);
    const float inv_hw = 1.f / static_cast<float>(HW);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // dc = ka * dz - kb * c + kc
      ka[j] = sc[j] * gt[j];
      kb[j] = sc[j] * is[j] * q2[j];
      kc[j] = sc[j] * (dpv[j] * inv_hw - q1[j] + mu[j] * is[j] * q2[j]);
    }
  }
  const long long base = static_cast<long long>(b) * HW * cvec + v;
  const int p0 = blockIdx.x * kSeApplyRows + row;
  uint4 zq[4], xq[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int p = p0 + u * kSeRowsPerPass;
    if (p < HW) {
      zq[u] = __ldg(dz + base + static_cast<long long>(p) * cvec);
      xq[u] = __ldg(c + base + static_cast<long long>(p) * cvec);
    }
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int p = p0 + u * kSeRowsPerPass;
    if (p >= HW) break;
    float zv[8], xv[8];
    unpack8(zq[u], zv);
    unpack8(xq[u], xv);
#pragma unroll
    for (int j = 0; j < 8; ++j) zv[j] = fmaf(ka[j], zv[j], fmaf(-kb[j], xv[j], kc[j]));
    dc[base + static_cast<long long>(p) * cvec] = pack8(zv);
  }
}

}  // namespace b200
