// Supervised contrastive learning passes (self-supervised/SupCon/models/model.py SupConModel, losses/SupConLoss.py
// SupConLoss): the row L2 normalisation of the embeddings and its backward, the SupCon loss over every pair of a batch and
// its backward, and the ReLU backward of the projection head.
//
// Loss convention: e fp32 [N][D] holds the contrast rows in cat(unbind(features, 1)) order and y int32 [N] their labels.
// With l_ij = e_i . e_j / tau, P_i = {j != i : y_j == y_i} and L_i = log sum_{j != i} exp l_ij,
//   loss_i = -(tau / base_tau) (sum_{j in P_i} l_ij / |P_i| - L_i),   loss = mean_i loss_i.
// L_i is a log-sum-exp with a running maximum, so it stays finite for any tau > 0 and any batch.  An anchor without a
// positive gives NaN, as the reference's 0 / 0 does.
//
// Every output element is written by exactly one thread and every sum runs over a fixed order (no atomics), so results
// are bitwise reproducible and every pass is capturable in a CUDA graph.
#pragma once
#include <math.h>

#include "common.cuh"

namespace b200 {

constexpr int kSupconBM = 16;       // anchor rows per CTA: warp w holds rows 2w, 2w + 1
constexpr int kSupconBN = 64;       // contrast rows per tile: lane l holds rows l, l + 32
constexpr int kSupconDK = 32;       // width chunk staged in shared memory
constexpr int kSupconMaxD = 2048;   // widest row the backward's shared-memory accumulator [kSupconBM][D] takes
constexpr float kSupconNormEps = 1e-12f;

// e = z / max(||z||, eps), nrm = ||z||; one warp per row, D a multiple of 4.
__global__ void __launch_bounds__(256) supcon_normalize_fwd_kernel(const float* __restrict__ z, int N, int D,
                                                                   float* __restrict__ e, float* __restrict__ nrm) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * 8ll + (threadIdx.x >> 5);
  if (row >= N) return;
  const float4* zr = reinterpret_cast<const float4*>(z + row * D);
  const int D4 = D >> 2;
  float acc = 0.f;
  for (int k = lane; k < D4; k += 32) {
    const float4 v = zr[k];
    acc = fmaf(v.x, v.x, acc);
    acc = fmaf(v.y, v.y, acc);
    acc = fmaf(v.z, v.z, acc);
    acc = fmaf(v.w, v.w, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  const float n = sqrtf(acc);
  const float d = fmaxf(n, kSupconNormEps);
  float4* er = reinterpret_cast<float4*>(e + row * D);
  for (int k = lane; k < D4; k += 32) {
    const float4 v = zr[k];
    er[k] = make_float4(v.x / d, v.y / d, v.z / d, v.w / d);
  }
  if (lane == 0) nrm[row] = n;
}

// dz = (de - e (e . de)) / ||z|| where ||z|| > eps, de / eps where the clamp was active; bf16 out, one warp per row.
__global__ void __launch_bounds__(256) supcon_normalize_bwd_kernel(const float* __restrict__ de, const float* __restrict__ e,
                                                                   const float* __restrict__ nrm, int N, int D,
                                                                   __nv_bfloat16* __restrict__ dz) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * 8ll + (threadIdx.x >> 5);
  if (row >= N) return;
  const float4* gr = reinterpret_cast<const float4*>(de + row * D);
  const float4* er = reinterpret_cast<const float4*>(e + row * D);
  const int D4 = D >> 2;
  float dot = 0.f;
  for (int k = lane; k < D4; k += 32) {
    const float4 g = gr[k], v = er[k];
    dot = fmaf(g.x, v.x, dot);
    dot = fmaf(g.y, v.y, dot);
    dot = fmaf(g.z, v.z, dot);
    dot = fmaf(g.w, v.w, dot);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  const float n = nrm[row];
  const bool clamped = !(n > kSupconNormEps);
  const float d = clamped ? kSupconNormEps : n;
  const float proj = clamped ? 0.f : dot;
  __nv_bfloat162* out = reinterpret_cast<__nv_bfloat162*>(dz + row * D);
  for (int k = lane; k < D4; k += 32) {
    const float4 g = gr[k], v = er[k];
    out[2 * k] = __floats2bfloat162_rn((g.x - v.x * proj) / d, (g.y - v.y * proj) / d);
    out[2 * k + 1] = __floats2bfloat162_rn((g.z - v.z * proj) / d, (g.w - v.w * proj) / d);
  }
}

// Dot products of one tile over the full width: s[a][b] = e[i0 + 2w + a] . e[j0 + l + 32 b] for warp w, lane l of a
// 256-thread CTA.  Rows past N read as zero.  Starts with a barrier, so the caller may reuse As / Bs right after a call.
__device__ __forceinline__ void supcon_tile_dots(const float* __restrict__ e, int N, int D, int i0, int j0,
                                                 float (*As)[kSupconDK + 1], float (*Bs)[kSupconDK + 1], float s[2][2]) {
  const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
  s[0][0] = s[0][1] = s[1][0] = s[1][1] = 0.f;
  for (int k0 = 0; k0 < D; k0 += kSupconDK) {
    __syncthreads();
    for (int t = tid; t < (kSupconBM + kSupconBN) * (kSupconDK / 4); t += 256) {
      const int r = t / (kSupconDK / 4), c = (t % (kSupconDK / 4)) * 4;
      const bool a_row = r < kSupconBM;
      const int row = a_row ? i0 + r : j0 + (r - kSupconBM);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < N && k0 + c < D) v = *reinterpret_cast<const float4*>(e + static_cast<long long>(row) * D + k0 + c);
      float* dst = a_row ? As[r] : Bs[r - kSupconBM];
      dst[c] = v.x;
      dst[c + 1] = v.y;
      dst[c + 2] = v.z;
      dst[c + 3] = v.w;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < kSupconDK; ++k) {
      const float a0 = As[2 * w][k], a1 = As[2 * w + 1][k];
      const float b0 = Bs[l][k], b1 = Bs[l + 32][k];
      s[0][0] = fmaf(a0, b0, s[0][0]);
      s[0][1] = fmaf(a0, b1, s[0][1]);
      s[1][0] = fmaf(a1, b0, s[1][0]);
      s[1][1] = fmaf(a1, b1, s[1][1]);
    }
  }
}

// (m, s) <- the log-sum-exp pair of the union of two sets of terms, each held as (max, sum of exp(term - max)).
__device__ __forceinline__ void supcon_lse_merge(float& m, float& s, float mo, float so) {
  const float mm = fmaxf(m, mo);
  if (mm == -INFINITY) return;
  s = s * expf(m - mm) + so * expf(mo - mm);
  m = mm;
}

// One CTA per kSupconBM anchor rows, sweeping the contrast rows in tiles of kSupconBN: L, npos = |P_i| and loss_i.
__global__ void __launch_bounds__(256) supcon_loss_fwd_kernel(const float* __restrict__ e, const int* __restrict__ y, int N,
                                                              int D, float inv_tau, float tau_ratio, float* __restrict__ L,
                                                              float* __restrict__ npos, float* __restrict__ row_loss) {
  pdl_wait();
  __shared__ float As[kSupconBM][kSupconDK + 1];
  __shared__ float Bs[kSupconBN][kSupconDK + 1];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int i0 = blockIdx.x * kSupconBM;
  int ia[2], ya[2];
  float m[2], s[2], ps[2], pc[2];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    ia[a] = i0 + 2 * w + a;
    ya[a] = ia[a] < N ? y[ia[a]] : 0;
    m[a] = -INFINITY;
    s[a] = ps[a] = pc[a] = 0.f;
  }
  for (int j0 = 0; j0 < N; j0 += kSupconBN) {
    float d[2][2];
    supcon_tile_dots(e, N, D, i0, j0, As, Bs, d);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int j = j0 + l + 32 * b;
      if (j >= N) continue;
      const int yj = y[j];
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        if (ia[a] >= N || j == ia[a]) continue;
        const float lg = d[a][b] * inv_tau;
        if (lg > m[a]) {
          s[a] = s[a] * expf(m[a] - lg) + 1.f;
          m[a] = lg;
        } else {
          s[a] += expf(lg - m[a]);
        }
        if (yj == ya[a]) {
          ps[a] += lg;
          pc[a] += 1.f;
        }
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 2; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float mo = __shfl_xor_sync(0xffffffffu, m[a], o), so = __shfl_xor_sync(0xffffffffu, s[a], o);
      ps[a] += __shfl_xor_sync(0xffffffffu, ps[a], o);
      pc[a] += __shfl_xor_sync(0xffffffffu, pc[a], o);
      supcon_lse_merge(m[a], s[a], mo, so);
    }
    if (l == 0 && ia[a] < N) {
      const float Li = m[a] + logf(s[a]);
      L[ia[a]] = Li;
      npos[ia[a]] = pc[a];
      row_loss[ia[a]] = -tau_ratio * (ps[a] / pc[a] - Li);
    }
  }
}

// loss[0] = mean of row_loss[0, N): per-thread strided sums, then a fixed-order tree, in double.
__global__ void __launch_bounds__(256) supcon_mean_kernel(const float* __restrict__ row_loss, int N, float* __restrict__ loss) {
  pdl_wait();
  __shared__ double red[256];
  double acc = 0.0;
  for (int i = threadIdx.x; i < N; i += 256) acc += row_loss[i];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = static_cast<float>(red[0] / N);
}

// de_i = c sum_j W_ij e_j with W_ij = exp(l_ij - L_i) + exp(l_ij - L_j) - [y_i == y_j] (1 / |P_i| + 1 / |P_j|) off the
// diagonal (G_ij + G_ji of the loss: l is symmetric, so no column reduction across CTAs is needed) and
// c = gout[0] * gscale.  One CTA per kSupconBM anchor rows; the [kSupconBM][D] accumulator lives in dynamic shared memory.
__global__ void __launch_bounds__(256, 1) supcon_loss_bwd_kernel(const float* __restrict__ e, const int* __restrict__ y,
                                                              const float* __restrict__ L, const float* __restrict__ npos,
                                                              const float* __restrict__ gout, float gscale, int N, int D,
                                                              float inv_tau, float* __restrict__ de) {
  pdl_wait();
  extern __shared__ float4 supcon_acc4[];
  float* acc = reinterpret_cast<float*>(supcon_acc4);
  __shared__ float As[kSupconBM][kSupconDK + 1];
  __shared__ float Bs[kSupconBN][kSupconDK + 1];
  __shared__ __align__(16) float Wt[kSupconBN][kSupconBM];
  const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
  const int i0 = blockIdx.x * kSupconBM;
  const float c = gout[0] * gscale;
  for (int t = tid; t < kSupconBM * D; t += 256) acc[t] = 0.f;
  int ia[2], ya[2];
  float La[2], pa[2];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    ia[a] = i0 + 2 * w + a;
    const bool ok = ia[a] < N;
    ya[a] = ok ? y[ia[a]] : 0;
    La[a] = ok ? L[ia[a]] : 0.f;
    pa[a] = ok ? npos[ia[a]] : 1.f;
  }
  for (int j0 = 0; j0 < N; j0 += kSupconBN) {
    float d[2][2];
    supcon_tile_dots(e, N, D, i0, j0, As, Bs, d);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int j = j0 + l + 32 * b;
      const bool jok = j < N;
      const int yj = jok ? y[j] : 0;
      const float Lj = jok ? L[j] : 0.f, pj = jok ? npos[j] : 1.f;
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        float wv = 0.f;
        if (jok && ia[a] < N && j != ia[a]) {
          const float lg = d[a][b] * inv_tau;
          const float pos = yj == ya[a] ? 1.f : 0.f;
          // pos / |P| is 0 / 0 = NaN for an anchor without a positive, as the reference's gradient is
          wv = c * (expf(lg - La[a]) + expf(lg - Lj) - pos / pa[a] - pos / pj);
        }
        Wt[l + 32 * b][2 * w + a] = wv;
      }
    }
    __syncthreads();
    const int jn = min(kSupconBN, N - j0);
    for (int dd = tid; dd < D; dd += 256) {
      float r[kSupconBM];
#pragma unroll
      for (int i = 0; i < kSupconBM; ++i) r[i] = acc[i * D + dd];
      const float* ej = e + static_cast<long long>(j0) * D + dd;
      for (int jj = 0; jj < jn; ++jj) {
        const float ev = ej[static_cast<long long>(jj) * D];
        const float4* w4 = reinterpret_cast<const float4*>(Wt[jj]);
#pragma unroll
        for (int q = 0; q < kSupconBM / 4; ++q) {
          const float4 wq = w4[q];
          r[4 * q] = fmaf(wq.x, ev, r[4 * q]);
          r[4 * q + 1] = fmaf(wq.y, ev, r[4 * q + 1]);
          r[4 * q + 2] = fmaf(wq.z, ev, r[4 * q + 2]);
          r[4 * q + 3] = fmaf(wq.w, ev, r[4 * q + 3]);
        }
      }
#pragma unroll
      for (int i = 0; i < kSupconBM; ++i) acc[i * D + dd] = r[i];
    }
    // (the next tile's supcon_tile_dots starts with a barrier before Wt is rewritten)
  }
  for (int dd = tid; dd < D; dd += 256) {
#pragma unroll
    for (int i = 0; i < kSupconBM; ++i)
      if (i0 + i < N) de[static_cast<long long>(i0 + i) * D + dd] = acc[i * D + dd];
  }
}

// dx = dy where the forward's ReLU output y is positive, else 0 (bf16).
__global__ void __launch_bounds__(256) supcon_relu_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                              const __nv_bfloat16* __restrict__ y, long long n,
                                                              __nv_bfloat16* __restrict__ dx) {
  pdl_wait();
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256)
    dx[i] = __bfloat162float(y[i]) > 0.f ? dy[i] : __float2bfloat16(0.f);
}

}  // namespace b200
