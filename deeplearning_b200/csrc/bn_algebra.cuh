// Train-mode BatchNorm folded THROUGH a 1x1 convolution (ResNet bottleneck conv3 -> bn3 -> (+identity) -> ReLU,
// classification/resnet/models/networks.py:116-124), so that the wide conv output c = y2 W^T is never written to HBM.
//
// With y2 [P x K] (the narrow input, K = 64..256 channels), W [N x K], c[p,o] = sum_j y2[p,j] W[o,j]:
//
//   forward statistics   sum_p c[p,o]   = W[o,:] . s            s = colsum(y2)          [K]
//                        sum_p c[p,o]^2 = W[o,:] G W[o,:]^T     G = y2^T y2             [K x K]  (one small tensor-core GEMM)
//     -> mean / invstd / scale / shift without a pass over c; the conv then applies  relu(acc * scale + shift + identity)
//        in its epilogue (conv_gemm.cuh kEpiAffine) and writes the block output directly.
//
//   backward  (dz = relu mask * upstream gradient,  dc = a dz + b c + k  per channel, the BatchNorm backward formula with
//              a = gamma invstd,  b = -a invstd mean(dz xhat),  k = -a mean(dz) - b mu)
//     D = dz^T y2 [N x K]   (the ordinary wgrad GEMM, on dz instead of dc)
//     sum_p dz c  = rowsum(W .* D)                      -> dgamma, dbeta, a, b, k        (no pass over c)
//     dW = a D + b (W G) + k s^T                         (weight gradient of the conv)
//     g2 = dc W = dz (diag(a) W) + y2 (W^T diag(b) W) + k W   -> ONE GEMM over [dz | y2] with the packed operand
//          Wcat[i][0..N) = a_o W[o,i],  Wcat[i][N + j] = M[j][i] = sum_o b_o W[o,j] W[o,i],  bias[i] = sum_o k_o W[o,i]
//
// c enters only through exact (fp32-accumulated) products of y2 and the bf16 weights the tensor cores used, i.e. the
// un-rounded conv output: closer to the fp32 reference than statistics of a bf16-rounded c.  Small-matrix work below runs
// in fp64 / fp32 on the CUDA cores (N K^2 MACs: 1 M for layer1 ... 67 M for layer3).
#pragma once
#include "common.cuh"

namespace b200 {

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- q = w G for 8 channels per block (one per warp), G staged through shared memory in chunks of 32 rows --------------------
// All 256 threads load a 32 x K chunk of G with coalesced 16-byte loads (one round of latency per chunk instead of one per
// row), then every warp accumulates its channel:  acc[x] = sum_i w_i * (G[i][j] * inv_n - m_i * m_j),  j = lane + 32 x.
// kCov = false drops the mean correction (plain q = w G).  w: this warp's K weights in shared memory, m: K means (kCov).
template <bool kCov>
__device__ __forceinline__ void warp_wG(const float* __restrict__ G, int K, float* Gs /* [32][K] */, const float* w,
                                        const float* m, float inv_n, float (&acc)[8]) {
  const int lane = threadIdx.x & 31;
  const int nq = K / 32;
  __syncthreads();   // w / m were just written by other threads of the block
  float mj[8];
#pragma unroll
  for (int x = 0; x < 8; ++x) {
    acc[x] = 0.f;
    mj[x] = (kCov && x < nq) ? m[lane + 32 * x] : 0.f;
  }
  // a 32 x K chunk is K / 32 = nq float4 per thread: all of them are loaded at once, one chunk AHEAD of the one being
  // consumed (the serial load -> store loop this replaces spent 8 L2 round trips per chunk: 51 -> ~20 us at N=1024, K=256)
  float4 pre[8];
  auto issue = [&](int r0) {
    const float4* src = reinterpret_cast<const float4*>(G + static_cast<long long>(r0) * K) + threadIdx.x;
#pragma unroll
    for (int x = 0; x < 8; ++x)
      if (x < nq) pre[x] = __ldg(src + 256 * x);
  };
  issue(0);
  for (int r0 = 0; r0 < K; r0 += 32) {
    __syncthreads();   // previous chunk consumed
#pragma unroll
    for (int x = 0; x < 8; ++x)
      if (x < nq) reinterpret_cast<float4*>(Gs)[threadIdx.x + 256 * x] = pre[x];
    __syncthreads();
    if (r0 + 32 < K) issue(r0 + 32);
#pragma unroll 4
    for (int r = 0; r < 32; ++r) {
      const float wi = w[r0 + r];
      const float mi = kCov ? m[r0 + r] : 0.f;
      const float* grow = Gs + r * K + lane;
#pragma unroll
      for (int x = 0; x < 8; ++x) {
        if (x < nq) {
          const float g = grow[32 * x];
          acc[x] = fmaf(wi, kCov ? fmaf(g, inv_n, -mi * mj[x]) : g, acc[x]);
        }
      }
    }
  }
}

// One warp per output channel o (8 per block).  G fp32 [K][K] (symmetric), s fp32 [K], Wb bf16 [N][K] (the forward operand).
// Writes mean / invstd / scale / shift and updates the running statistics like nn.BatchNorm2d (momentum, unbiased var).
__global__ void __launch_bounds__(256) bn_gram_stats_kernel(const float* __restrict__ G, const float* __restrict__ s,
                                                            const __nv_bfloat16* __restrict__ Wb, int N, int K, double count,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            float eps, float momentum, float* running_mean,
                                                            float* running_var, long long* num_batches, float* mean_out,
                                                            float* invstd_out, float* scale_out, float* shift_out) {
  pdl_wait();
  extern __shared__ float sm_gs[];   // [32][K] chunk of G | [8 warps][K] weights | [K] column means
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int o = blockIdx.x * 8 + warp;
  float* Gs = sm_gs;
  float* w = sm_gs + 32 * K + warp * K;
  float* m = sm_gs + 32 * K + 8 * K;
  const double inv_n = 1.0 / count;
  for (int j = threadIdx.x; j < K; j += blockDim.x) m[j] = static_cast<float>(static_cast<double>(s[j]) * inv_n);
  for (int j = lane; j < K; j += 32) w[j] = o < N ? __bfloat162float(Wb[static_cast<long long>(o) * K + j]) : 0.f;
  // (warp_wG starts with a block barrier: m and w are visible to everyone)
  float acc[8];
  warp_wG<true>(G, K, Gs, w, m, static_cast<float>(inv_n), acc);
  if (o >= N) return;
  const int nq = K / 32;
  double var = 0.0, mean = 0.0;
#pragma unroll
  for (int x = 0; x < 8; ++x) {
    if (x < nq) {
      const int j = lane + 32 * x;
      var += static_cast<double>(acc[x]) * static_cast<double>(w[j]);
      mean += static_cast<double>(w[j]) * static_cast<double>(m[j]);
    }
  }
  var = warp_sum_d(var);
  mean = warp_sum_d(mean);
  if (lane == 0) {
    if (var < 0.0) var = 0.0;
    const double invstd = 1.0 / sqrt(var + static_cast<double>(eps));
    const float g = gamma ? gamma[o] : 1.0f, b = beta ? beta[o] : 0.0f;
    mean_out[o] = static_cast<float>(mean);
    invstd_out[o] = static_cast<float>(invstd);
    scale_out[o] = static_cast<float>(g * invstd);
    shift_out[o] = static_cast<float>(b - mean * g * invstd);
    if (running_mean) {
      const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
      running_mean[o] = static_cast<float>((1.0 - momentum) * running_mean[o] + momentum * mean);
      running_var[o] = static_cast<float>((1.0 - momentum) * running_var[o] + momentum * unbiased);
    }
    if (num_batches && o == 0) *num_batches += 1;
  }
}

// Backward, per output channel o (one warp each, 8 per block):
//   sum_dz from the partial rows dz_partial[T][2][N] (plane 0), D fp32 [N][K] (raw dz^T y2), G, s, Wb as above, W fp32 [N][K]
//   (the master weights, for the data-gradient operand), mean / invstd / gamma of the BatchNorm.
// Writes dgamma[o], dbeta[o] (optionally accumulating), dW[o][:] = a D + b (Wb G) + k s (optionally accumulating),
// the bf16 column o of the dgrad operand wcat[i][o] = a_o W[o][i] (ld = N + K) and coef[o] = {b_o, k_o} for the M kernel.
__global__ void __launch_bounds__(256) bn_conv1x1_bwd_rows_kernel(
    const float* __restrict__ dz_partial, int T, const float* __restrict__ D, const float* __restrict__ G,
    const float* __restrict__ s, const __nv_bfloat16* __restrict__ Wb, const float* __restrict__ W, int N, int K, double count,
    const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ invstd, float* dgamma,
    float* dbeta, float* dW, int accumulate, __nv_bfloat16* __restrict__ wcat, float2* __restrict__ coef) {
  pdl_wait();
  extern __shared__ float sm_f[];   // [32][K] chunk of G | [8 warps][K] bf16 weights (as float) of the warp's channel
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int o = blockIdx.x * 8 + warp;
  const bool live = o < N;
  float* Gs = sm_f;
  float* wb = sm_f + 32 * K + warp * K;
  const long long row = static_cast<long long>(live ? o : 0) * K;
  const int nq = K / 32;
  float dv[8], wv[8];
  double t = 0.0;   // sum_j Wb[o][j] D[o][j] = sum_p dz[p,o] c[p,o]
#pragma unroll
  for (int x = 0; x < 8; ++x) {
    if (x < nq) {
      const int j = lane + 32 * x;
      const float v = live ? __bfloat162float(Wb[row + j]) : 0.f;
      wb[j] = v;
      dv[x] = D[row + j];
      wv[x] = W[row + j];
      t += static_cast<double>(v) * static_cast<double>(dv[x]);
    }
  }
  // column sum of dz: T partial rows, 8 independent loads in flight per lane
  float sd[8];
#pragma unroll
  for (int x = 0; x < 8; ++x) sd[x] = 0.f;
  if (live) {
    for (int r0 = lane; r0 < T; r0 += 256) {
#pragma unroll
      for (int x = 0; x < 8; ++x) {
        const int r = r0 + 32 * x;
        if (r < T) sd[x] += __ldg(dz_partial + (static_cast<long long>(r) * 2) * N + o);
      }
    }
  }
  double sdz = 0.0;
#pragma unroll
  for (int x = 0; x < 8; ++x) sdz += static_cast<double>(sd[x]);
  t = warp_sum_d(t);
  sdz = warp_sum_d(sdz);
  // q_j = sum_i Wb[o][i] G[i][j]   (starts with a block barrier: wb is visible)
  float q[8];
  warp_wG<false>(G, K, Gs, wb, nullptr, 0.f, q);
  if (!live) return;
  const double mu = mean[o], is = invstd[o], g = gamma ? gamma[o] : 1.0f;
  const double dg = is * (t - mu * sdz);   // sum dz * xhat
  const double a = g * is;
  const double b = -a * is * (dg / count);
  const double k = -a * (sdz / count) - b * mu;
  if (lane == 0) {
    dgamma[o] = accumulate ? dgamma[o] + static_cast<float>(dg) : static_cast<float>(dg);
    dbeta[o] = accumulate ? dbeta[o] + static_cast<float>(sdz) : static_cast<float>(sdz);
    coef[o] = make_float2(static_cast<float>(b), static_cast<float>(k));
  }
  const float af = static_cast<float>(a), bf = static_cast<float>(b), kf = static_cast<float>(k);
  const int ld = N + K;
#pragma unroll
  for (int x = 0; x < 8; ++x) {
    if (x < nq) {
      const int j = lane + 32 * x;
      const float v = af * dv[x] + bf * q[x] + kf * s[j];
      dW[row + j] = accumulate ? dW[row + j] + v : v;
      wcat[static_cast<long long>(j) * ld + o] = __float2bfloat16(af * wv[x]);
    }
  }
}

// M[j][i] = sum_o b_o Wb[o][j] W[o][i]  ->  wcat[i][N + j];   bias[i] = sum_o k_o W[o][i].
// grid (K/32, K/32, S): a block computes a 32 x 32 tile of M over ITS slice of the channels o (N / S of them, staged through
// shared memory 32 rows at a time) and publishes the partial tile; the last block of a tile to finish (ticket counter, reset
// for the next launch) adds the S partials in a fixed order - deterministic - and writes the bf16 operand.  Thread = (i, 4 j's).
// Tiles with blockIdx.y == 0 also carry the 32 bias entries of their i range.
// scratch: [K/32 * K/32] uint32 tickets (zero before the first launch) | partial [S][K/32*K/32][33][32] floats.
constexpr int kAlgebraSlices = 8;
__global__ void __launch_bounds__(256) bn_conv1x1_bwd_m_kernel(const float2* __restrict__ coef, const __nv_bfloat16* __restrict__ Wb,
                                                               const float* __restrict__ W, int N, int K,
                                                               __nv_bfloat16* __restrict__ wcat, float* __restrict__ bias,
                                                               unsigned int* __restrict__ tickets, float* __restrict__ partial) {
  pdl_wait();
  __shared__ float sa[32][33];   // b_o * Wb[o][j0 + .]
  __shared__ float sw[32][33];   // W[o][i0 + .]
  __shared__ float sk[32];       // k_o
  __shared__ int is_last;
  const int ti = threadIdx.x & 31, tq = threadIdx.x >> 5;   // i = i0 + ti; j = j0 + tq * 4 + {0..3}
  const int i0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
  const int S = gridDim.z, z = blockIdx.z;
  const int per = (N + S - 1) / S;
  const int o_begin = z * per, o_end = min(N, o_begin + per);
  const int tile = blockIdx.y * gridDim.x + blockIdx.x, n_tile = gridDim.x * gridDim.y;
  float acc[4] = {0.f, 0.f, 0.f, 0.f}, accb = 0.f;
  // the 32 channels of the NEXT round are fetched into registers while the current round is multiplied
  float av[4], wv4[4], kv[4];
  auto fetch = [&](int o0) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int o = o0 + tq * 4 + r;
      av[r] = wv4[r] = kv[r] = 0.f;
      if (o < o_end) {
        const long long base = static_cast<long long>(o) * K;
        const float2 c = coef[o];
        av[r] = c.x * __bfloat162float(Wb[base + j0 + ti]);
        wv4[r] = W[base + i0 + ti];
        kv[r] = c.y;
      }
    }
  };
  fetch(o_begin);
  for (int o0 = o_begin; o0 < o_end; o0 += 32) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      sa[tq * 4 + r][ti] = av[r];
      sw[tq * 4 + r][ti] = wv4[r];
      if (ti == 0) sk[tq * 4 + r] = kv[r];
    }
    __syncthreads();
    if (o0 + 32 < o_end) fetch(o0 + 32);
#pragma unroll
    for (int o = 0; o < 32; ++o) {
      const float wv = sw[o][ti];
#pragma unroll
      for (int x = 0; x < 4; ++x) acc[x] = fmaf(sa[o][tq * 4 + x], wv, acc[x]);
      if (tq == 0) accb = fmaf(sk[o], wv, accb);
    }
    __syncthreads();
  }
  // publish this slice's partial tile: [z][tile][row 0..31 = j, row 32 = bias][i]
  float* mine = partial + (static_cast<long long>(z) * n_tile + tile) * 33 * 32;
#pragma unroll
  for (int x = 0; x < 4; ++x) mine[(tq * 4 + x) * 32 + ti] = acc[x];
  if (tq == 0) mine[32 * 32 + ti] = accb;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(&tickets[tile], 1u);
    is_last = (t == static_cast<unsigned int>(S - 1));
    if (is_last) tickets[tile] = 0;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  float fin[4] = {0.f, 0.f, 0.f, 0.f}, finb = 0.f;
  for (int zz = 0; zz < S; ++zz) {
    const float* src = partial + (static_cast<long long>(zz) * n_tile + tile) * 33 * 32;
#pragma unroll
    for (int x = 0; x < 4; ++x) fin[x] += __ldcg(src + (tq * 4 + x) * 32 + ti);
    if (tq == 0) finb += __ldcg(src + 32 * 32 + ti);
  }
  const long long ld = N + K;
#pragma unroll
  for (int x = 0; x < 4; ++x) wcat[static_cast<long long>(i0 + ti) * ld + N + j0 + tq * 4 + x] = __float2bfloat16(fin[x]);
  if (blockIdx.y == 0 && tq == 0) bias[i0 + ti] = finb;
}

}  // namespace b200
