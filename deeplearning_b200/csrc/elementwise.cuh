// HBM-bound passes of the classification training step (NHWC bf16 activations, fp32 statistics):
// train/eval BatchNorm finalize + apply(+ReLU)(+residual), BatchNorm backward (reduce / finalize / apply),
// stem max-pool forward/backward, global average pool, soft-max cross-entropy, layout packing and the fused SGD update.
// All kernels move 16-byte vectors (8 bf16 channels per thread) and use grid-stride loops over a grid sized from the SM count.
//
// Reference semantics: nn.BatchNorm2d defaults (eps 1e-5, momentum 0.1, biased var to normalise, unbiased running_var)
// as used at classification/resnet/models/networks.py:45,91,134; MaxPool2d(3,2,1) :152; AdaptiveAvgPool2d(1) :160;
// CrossEntropyLoss (classification/resnet/train.py:104); SGD momentum (classification/resnet/train.py:96).
#pragma once
#include "row_passes.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------------------------------
// Column reduction of per-tile partials partial[T][2][C] -> two per-channel sums (double), parallel over T:
// grid = (ceil(C/32), S); every block reduces its slice of T for 32 channels and publishes it to `scratch`; the last
// block to finish (ticket counter, reset to zero for the next call) folds the S slices and returns true.
// scratch layout: [256 x uint32 counters][S][2][C] doubles.
__device__ __forceinline__ bool reduce_partials_last_block(const float* __restrict__ partial, int T, int C, void* scratch,
                                                           double& s_out, double& ss_out) {
  __shared__ double sh[2][8][32];
  __shared__ int is_last;
  unsigned int* counters = static_cast<unsigned int*>(scratch);
  double* slices = reinterpret_cast<double*>(static_cast<char*>(scratch) + 1024);
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const int S = gridDim.y;
  const int chunk = (T + S - 1) / S;
  const int t0 = blockIdx.y * chunk, t1 = min(T, t0 + chunk);
  double s = 0.0, ss = 0.0;
  if (c < C) {
    // four rows (eight loads) in flight per thread: the kernel is a chain of L2 round trips, not bandwidth
    int t = t0 + ry;
    for (; t + 24 < t1; t += 32) {
      float v[4][2];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        v[u][0] = __ldg(partial + (static_cast<long long>(t + 8 * u) * 2 + 0) * C + c);
        v[u][1] = __ldg(partial + (static_cast<long long>(t + 8 * u) * 2 + 1) * C + c);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        s += static_cast<double>(v[u][0]);
        ss += static_cast<double>(v[u][1]);
      }
    }
    for (; t < t1; t += 8) {
      s += static_cast<double>(__ldg(partial + (static_cast<long long>(t) * 2 + 0) * C + c));
      ss += static_cast<double>(__ldg(partial + (static_cast<long long>(t) * 2 + 1) * C + c));
    }
  }
  sh[0][ry][cx] = s;
  sh[1][ry][cx] = ss;
  __syncthreads();
  if (ry == 0 && c < C) {
    for (int i = 1; i < 8; ++i) {
      s += sh[0][i][cx];
      ss += sh[1][i][cx];
    }
    slices[(static_cast<long long>(blockIdx.y) * 2 + 0) * C + c] = s;
    slices[(static_cast<long long>(blockIdx.y) * 2 + 1) * C + c] = ss;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(&counters[blockIdx.x], 1u);
    is_last = (ticket == static_cast<unsigned int>(S - 1));
    if (is_last) counters[blockIdx.x] = 0;  // ready for the next launch on this stream
  }
  __syncthreads();
  if (!is_last) return false;
  __threadfence();
  s = 0.0;
  ss = 0.0;
  if (c < C) {
    for (int k = ry; k < S; k += 8) {
      s += slices[(static_cast<long long>(k) * 2 + 0) * C + c];
      ss += slices[(static_cast<long long>(k) * 2 + 1) * C + c];
    }
  }
  __syncthreads();
  sh[0][ry][cx] = s;
  sh[1][ry][cx] = ss;
  __syncthreads();
  if (ry == 0) {
    for (int i = 1; i < 8; ++i) {
      s += sh[0][i][cx];
      ss += sh[1][i][cx];
    }
  }
  s_out = s;
  ss_out = ss;
  return ry == 0 && c < C;
}

// BatchNorm statistics finalize: partial[T][2][C] (sum, sum of squares per tile) -> mean/invstd/scale/shift,
// running-stat update (double accumulation).
__global__ void bn_finalize_kernel(const float* __restrict__ partial, int T, int C, double count,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   float momentum, float* running_mean, float* running_var, long long* num_batches,
                                   float* mean_out, float* invstd_out, float* scale_out, float* shift_out,
                                   void* scratch) {
  pdl_wait();
  double s, ss;
  const bool owner = reduce_partials_last_block(partial, T, C, scratch, s, ss);
  if (owner) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const double mean = s / count;
    double var = ss / count - mean * mean;
    if (var < 0.0) var = 0.0;
    const double invstd = 1.0 / sqrt(var + static_cast<double>(eps));
    const float g = gamma ? gamma[c] : 1.0f, b = beta ? beta[c] : 0.0f;
    mean_out[c] = static_cast<float>(mean);
    invstd_out[c] = static_cast<float>(invstd);
    scale_out[c] = static_cast<float>(g * invstd);
    shift_out[c] = static_cast<float>(b - mean * g * invstd);
    if (running_mean) {
      const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
      running_mean[c] = static_cast<float>((1.0 - momentum) * running_mean[c] + momentum * mean);
      running_var[c] = static_cast<float>((1.0 - momentum) * running_var[c] + momentum * unbiased);
    }
    if (num_batches && c == 0) *num_batches += 1;
  }
}

// Eval-mode BN: scale/shift from running statistics.
__global__ void bn_eval_coeffs_kernel(int C, const float* __restrict__ gamma, const float* __restrict__ beta,
                                      const float* __restrict__ running_mean, const float* __restrict__ running_var,
                                      float eps, float* scale_out, float* shift_out) {
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    const float invstd = 1.0f / sqrtf(running_var[c] + eps);
    const float sc = gamma[c] * invstd;
    scale_out[c] = sc;
    shift_out[c] = beta[c] - running_mean[c] * sc;
  }
}

// y = act(x * scale[c] + shift[c] (+ residual)); x,y,residual bf16 [rows][C].
__global__ void __launch_bounds__(256) bn_apply_kernel(const uint4* __restrict__ x, const uint4* __restrict__ residual,
                                                       uint4* __restrict__ y, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, long long nvec, int cvec, int relu) {
  pdl_wait();
  // four independent 16-byte vectors (plus their residuals) per thread and iteration: ~100 KB of loads in flight per SM,
  // which is what HBM3e needs to stay busy (one vector per iteration left the kernel at ~5.2 of 6.5 TB/s)
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i0 = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i0 < nvec; i0 += 4 * stride) {
    uint4 xv[4], rv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long i = i0 + u * stride;
      if (i < nvec) {
        xv[u] = __ldg(x + i);
        if (residual) rv[u] = __ldg(residual + i);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long i = i0 + u * stride;
      if (i >= nvec) break;
      const int cg = static_cast<int>(i % cvec);
      float sc[8], sh[8], v[8];
      load8f(scale + cg * 8, sc);
      load8f(shift + cg * 8, sh);
      unpack8(xv[u], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaf(v[j], sc[j], sh[j]);
      if (residual) {
        float r[8];
        unpack8(rv[u], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += r[j];
      }
      if (relu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f);
      }
      y[i] = pack8(v);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// BatchNorm backward, pass 1: dz = g * relu_mask; per-channel partial sums of dz and dz * xhat.
//   mask source: y_out (saved post-activation output, used when a residual was added) if given, else recomputed from
//   x*scale+shift > 0; relu == 0 -> no mask.  Optionally stores dz (bf16) for reuse (identity-branch gradient).
// Block = 256 threads; each thread owns one 8-channel group and strides over rows. partial[blocks][2][C].
__global__ void __launch_bounds__(256, 2)
bn_bwd_reduce_kernel(const uint4* __restrict__ g, const uint4* __restrict__ x, const uint4* __restrict__ y_out,
                     uint4* __restrict__ dz_out, const float* __restrict__ scale, const float* __restrict__ shift, int relu,
                     long long rows, int cvec, int rows_per_block, float* __restrict__ partial) {
  pdl_wait();
  extern __shared__ float red[];  // [256][17]
  const int tpr = cvec;                  // threads per row (power of two, <= 256)
  const int rpi = 256 / tpr;             // rows per iteration
  const int cg = threadIdx.x % tpr;
  const int rsub = threadIdx.x / tpr;
  const bool mask_from_y = relu && (y_out != nullptr);
  const bool mask_from_x = relu && (y_out == nullptr);
  float sc[8], sh[8];
  if (mask_from_x) {
    load8f(scale + cg * 8, sc);
    load8f(shift + cg * 8, sh);
  }
  // accumulates sum(dz) and sum(dz * x) with the RAW x; the finalize kernel turns the latter into sum(dz * xhat)
  float a1[8], a2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a1[j] = a2[j] = 0.f;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  // four rows in flight per thread (8-12 independent 16-byte loads)
  for (long long r = r0 + rsub; r < r1; r += 4 * rpi) {
    uint4 gq[4], xq[4], yq[4];
    bool has[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const long long rr = r + h * rpi;
      has[h] = rr < r1;
      if (has[h]) {
        const long long i = rr * cvec + cg;
        gq[h] = __ldg(g + i);
        xq[h] = __ldg(x + i);
        if (mask_from_y) yq[h] = __ldg(y_out + i);
      }
    }
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      if (!has[h]) break;
      float gv[8], xv[8];
      unpack8(gq[h], gv);
      unpack8(xq[h], xv);
      if (mask_from_y) {
        float yv[8];
        unpack8(yq[h], yv);
#pragma unroll
        for (int j = 0; j < 8; ++j) gv[j] = yv[j] > 0.f ? gv[j] : 0.f;
      } else if (mask_from_x) {
#pragma unroll
        for (int j = 0; j < 8; ++j) gv[j] = fmaf(xv[j], sc[j], sh[j]) > 0.f ? gv[j] : 0.f;
      }
      if (dz_out) dz_out[(r + h * rpi) * cvec + cg] = pack8(gv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        a1[j] += gv[j];
        a2[j] = fmaf(gv[j], xv[j], a2[j]);
      }
    }
  }
  float* my = red + threadIdx.x * 17;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    my[j] = a1[j];
    my[8 + j] = a2[j];
  }
  __syncthreads();
  if (rsub == 0) {
    for (int k = 1; k < rpi; ++k) {
      const float* o = red + (k * tpr + cg) * 17;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        a1[j] += o[j];
        a2[j] += o[8 + j];
      }
    }
    const int C = cvec * 8;
    float* p1 = partial + (static_cast<long long>(blockIdx.x) * 2 + 0) * C + cg * 8;
    float* p2 = partial + (static_cast<long long>(blockIdx.x) * 2 + 1) * C + cg * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      p1[j] = a1[j];
      p2[j] = a2[j];
    }
  }
}

// BN backward finalize: partial[T][2][C] -> dbeta = sum dz, dgamma = sum dz*xhat, and the per-channel means used by
// the apply pass: m1 = dbeta / count, m2 = dgamma / count.
__global__ void bn_bwd_finalize_kernel(const float* __restrict__ partial, int T, int C, double count,
                                       float* __restrict__ dgamma, float* __restrict__ dbeta, int accumulate,
                                       float* __restrict__ m1, float* __restrict__ m2, const float* __restrict__ mean,
                                       const float* __restrict__ invstd, void* scratch) {
  pdl_wait();
  double s, ss;
  const bool owner = reduce_partials_last_block(partial, T, C, scratch, s, ss);
  if (owner) {
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    // the reduce pass accumulated sum(dz * x) with the raw x: sum(dz * xhat) = invstd * (sum(dz*x) - mean * sum(dz))
    if (mean != nullptr) ss = static_cast<double>(invstd[c]) * (ss - static_cast<double>(mean[c]) * s);
    if (dbeta) dbeta[c] = accumulate ? dbeta[c] + static_cast<float>(s) : static_cast<float>(s);
    if (dgamma) dgamma[c] = accumulate ? dgamma[c] + static_cast<float>(ss) : static_cast<float>(ss);
    if (m1) m1[c] = static_cast<float>(s / count);
    if (m2) m2[c] = static_cast<float>(ss / count);
  }
}

// BN backward, pass 2: dx = scale * (dz - m1 - xhat * m2), dz recomputed exactly as in pass 1 (or read from g when
// g_is_dz).  Row geometry of row_passes.cuh (repvgg_geom): gridDim.y chunks of gpc 8-channel groups, so any C % 8 == 0 up
// to 8192 runs; for C = 8 * 2^k <= 2048 that is pass 1's grid and thread mapping.
__global__ void bn_bwd_apply_kernel(const uint4* __restrict__ g, const uint4* __restrict__ x,
                                    const uint4* __restrict__ y_out, int g_is_dz, uint4* __restrict__ dx,
                                    const float* __restrict__ scale, const float* __restrict__ shift,
                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                    const float* __restrict__ m1, const float* __restrict__ m2, int relu,
                                    long long rows, int cvec, int rows_per_block, int gpc) {
  pdl_wait();
  const int rpi = 256 / gpc;
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;
  const int cg = blockIdx.y * gpc + lane_g;
  if (rsub >= rpi || cg >= cvec) return;
  // dx = a * dz - bq * x + cq, a = scale
  float a[8], bq[8], cq[8], sh[8];
  rv_bwd_coeffs(mean, invstd, scale, m1, m2, cg, a, bq, cq);
  const bool mask_from_x = relu && !g_is_dz && (y_out == nullptr);
  const bool mask_from_y = relu && !g_is_dz && (y_out != nullptr);
  if (mask_from_x) load8f(shift + cg * 8, sh);
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  // four rows in flight per thread (8-12 independent 16-byte loads): the two-row version left HBM at ~4.7 TB/s
  for (long long r = r0 + rsub; r < r1; r += 4 * rpi) {
    uint4 gq[4], xq[4], yq[4];
    bool has[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const long long rr = r + h * rpi;
      has[h] = rr < r1;
      if (has[h]) {
        const long long i = rr * cvec + cg;
        gq[h] = __ldg(g + i);
        xq[h] = __ldg(x + i);
        if (mask_from_y) yq[h] = __ldg(y_out + i);
      }
    }
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      if (!has[h]) break;
      float gv[8], xv[8], o[8];
      unpack8(gq[h], gv);
      unpack8(xq[h], xv);
      if (mask_from_y) {
        float yv[8];
        unpack8(yq[h], yv);
#pragma unroll
        for (int j = 0; j < 8; ++j) gv[j] = yv[j] > 0.f ? gv[j] : 0.f;
      } else if (mask_from_x) {
#pragma unroll
        for (int j = 0; j < 8; ++j) gv[j] = fmaf(xv[j], a[j], sh[j]) > 0.f ? gv[j] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf(a[j], gv[j], fmaf(-bq[j], xv[j], cq[j]));
      dx[(r + h * rpi) * cvec + cg] = pack8(o);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Stem: y = maxpool3x3s2p1(relu(x*scale+shift)); also records the arg-max tap (0..8) for the backward pass.
// All nine taps are loaded before any arithmetic (nine independent 16-byte loads in flight per thread); the arg-max is taken
// over the fp32 activations - rounding to bf16 is monotonic, so the pooled VALUE equals the max of the rounded activations a
// stand-alone BN+ReLU pass would have stored, and ties between activations that only coincide after rounding go to the
// larger fp32 value, which is what the fp32 reference does.  Index arithmetic in 32 bits.
__global__ void __launch_bounds__(256) bn_relu_maxpool_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y,
                                                                  unsigned long long* __restrict__ idx,
                                                                  const float* __restrict__ scale,
                                                                  const float* __restrict__ shift, int B, int H, int W, int cvec) {
  pdl_wait();
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const unsigned nvec = static_cast<unsigned>(B) * Ho * Wo * cvec;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x) {
    const unsigned cg = i % cvec;
    unsigned t = i / cvec;
    const int ow = static_cast<int>(t % Wo);
    t /= Wo;
    const int oh = static_cast<int>(t % Ho);
    const unsigned b = t / Ho;
    uint4 v[9];
    bool ok[9];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int ih = oh * 2 - 1 + kh, iw = ow * 2 - 1 + kw;
        ok[kh * 3 + kw] = ih >= 0 && ih < H && iw >= 0 && iw < W;
        v[kh * 3 + kw] = ok[kh * 3 + kw] ? __ldg(x + ((b * H + ih) * W + iw) * cvec + cg) : zero;
      }
    }
    float sc[8], sh[8], best[8];
    int bi[8];
    load8f(scale + cg * 8, sc);
    load8f(shift + cg * 8, sh);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      best[j] = -INFINITY;
      bi[j] = 0;
    }
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      if (!ok[tap]) continue;
      float f[8];
      unpack8(v[tap], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float a = fmaxf(fmaf(f[j], sc[j], sh[j]), 0.f);
        if (a > best[j]) {
          best[j] = a;
          bi[j] = tap;
        }
      }
    }
    y[i] = pack8(best);
    unsigned long long packed = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) packed |= static_cast<unsigned long long>(bi[j] & 0xFF) << (8 * j);
    idx[i] = packed;
  }
}

// Max-pool backward: g_in[b,h,w,c] = sum over the (<=4) windows covering (h,w) whose arg-max is this pixel.
// One thread produces the 2x2 input block (2a..2a+1, 2b..2b+1) of one 8-channel group: exactly the four windows
// (a,b), (a,b+1), (a+1,b), (a+1,b+1) touch it - (even,even) belongs to tap (1,1) of window (a,b) only, the odd row / column
// pixels to two, the (odd,odd) pixel to all four - so four (arg-max, gradient) loads feed four outputs (the per-pixel
// version loaded nine and spent ~3x the instructions).
__global__ void __launch_bounds__(256) maxpool_bwd_kernel(const uint4* __restrict__ g_out,
                                                          const unsigned long long* __restrict__ idx, uint4* __restrict__ g_in,
                                                          int B, int H, int W, int cvec) {
  pdl_wait();
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;   // = H / 2, W / 2
  const unsigned nblk = static_cast<unsigned>(B) * Ho * Wo * cvec;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < nblk; i += gridDim.x * blockDim.x) {
    const unsigned cg = i % cvec;
    unsigned t = i / cvec;
    const int bw = static_cast<int>(t % Wo);
    t /= Wo;
    const int ah = static_cast<int>(t % Ho);
    const unsigned b = t / Ho;
    // windows (ah + dy, bw + dx), dy, dx in {0, 1}
    uint4 gq[4];
    unsigned long long pk[4];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int oh = ah + (d >> 1), ow = bw + (d & 1);
      const bool ok = oh < Ho && ow < Wo;
      const unsigned o = ((b * Ho + (ok ? oh : ah)) * Wo + (ok ? ow : bw)) * cvec + cg;
      gq[d] = ok ? __ldg(g_out + o) : make_uint4(0u, 0u, 0u, 0u);
      pk[d] = ok ? __ldg(idx + o) : 0xFFFFFFFFFFFFFFFFull;   // tap 255: never matches
    }
    float g[4][8];
#pragma unroll
    for (int d = 0; d < 4; ++d) unpack8(gq[d], g[d]);
    float o00[8], o01[8], o10[8], o11[8];   // input pixels (2a, 2b), (2a, 2b+1), (2a+1, 2b), (2a+1, 2b+1)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int t0 = static_cast<int>((pk[0] >> (8 * j)) & 0xFF), t1 = static_cast<int>((pk[1] >> (8 * j)) & 0xFF);
      const int t2 = static_cast<int>((pk[2] >> (8 * j)) & 0xFF), t3 = static_cast<int>((pk[3] >> (8 * j)) & 0xFF);
      // window (a,b): taps (kh,kw) -> input (2a-1+kh, 2b-1+kw): (1,1)->(2a,2b) (1,2)->(2a,2b+1) (2,1)->(2a+1,2b) (2,2)->(2a+1,2b+1)
      o00[j] = (t0 == 4) ? g[0][j] : 0.f;
      o01[j] = ((t0 == 5) ? g[0][j] : 0.f) + ((t1 == 3) ? g[1][j] : 0.f);                 // window (a,b+1): tap (1,0)
      o10[j] = ((t0 == 7) ? g[0][j] : 0.f) + ((t2 == 1) ? g[2][j] : 0.f);                 // window (a+1,b): tap (0,1)
      o11[j] = ((t0 == 8) ? g[0][j] : 0.f) + ((t1 == 6) ? g[1][j] : 0.f) +               // (a,b+1): tap (2,0)
               ((t2 == 2) ? g[2][j] : 0.f) + ((t3 == 0) ? g[3][j] : 0.f);                 // (a+1,b): (0,2); (a+1,b+1): (0,0)
    }
    const unsigned base = ((b * H + 2 * ah) * W + 2 * bw) * cvec + cg;
    const bool w1 = 2 * bw + 1 < W, h1 = 2 * ah + 1 < H;   // (odd H / W: the last block is half outside)
    g_in[base] = pack8(o00);
    if (w1) g_in[base + cvec] = pack8(o01);
    if (h1) g_in[base + W * cvec] = pack8(o10);
    if (h1 && w1) g_in[base + W * cvec + cvec] = pack8(o11);
  }
}

// Global average pool over HW: x [B][HW][C] bf16 -> y [B][C] bf16.
__global__ void avgpool_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int B, int HW, int cvec) {
  pdl_wait();
  const long long nvec = static_cast<long long>(B) * cvec;
  const float inv = 1.0f / HW;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % cvec);
    const long long b = i / cvec;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int p = 0; p < HW; ++p) {
      float v[8];
      unpack8(__ldg(x + (b * HW + p) * cvec + cg), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    y[i] = pack8(acc);
  }
}
// Backward: g_x[b][p][c] = g_y[b][c] / HW.
__global__ void avgpool_bwd_kernel(const uint4* __restrict__ gy, uint4* __restrict__ gx, int B, int HW, int cvec) {
  pdl_wait();
  const long long nvec = static_cast<long long>(B) * HW * cvec;
  const float inv = 1.0f / HW;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % cvec);
    const long long b = i / (static_cast<long long>(HW) * cvec);
    float v[8];
    unpack8(__ldg(gy + b * cvec + cg), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= inv;
    gx[i] = pack8(v);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Soft-max cross-entropy (mean reduction) forward + backward in one pass. One block per row.
//   logits fp32 [B][ld], labels int64 -> loss_rows[B] (fp32, un-normalised), dlogits bf16 [B][ld_d] = (p - onehot)*gscale
// Soft targets (timm SoftTargetCrossEntropy behind Mixup / CutMix, swin_transformer/main.py:111-113) and label smoothing
// (LabelSmoothingCrossEntropy, main.py:114-115) are the same kernel with target distribution t instead of a one-hot:
//   t_c = soft[b][c]                      (soft != null), or
//   t_c = (1 - eps) [c == label] + eps/N  (smoothing eps),
//   loss_b = sum_c t_c (lse - x_c),  dlogits = (p_c * sum_c t_c - t_c) * gscale.
__global__ void softmax_xent_kernel(const float* __restrict__ logits, long long ld, const long long* __restrict__ labels,
                                    int N, float gscale, float* __restrict__ loss_rows,
                                    __nv_bfloat16* __restrict__ dlogits, long long ld_d, int* __restrict__ correct,
                                    const float* __restrict__ soft, long long ld_soft, float smoothing) {
  pdl_wait();
  __shared__ float sh[32];
  __shared__ int shi[32];
  const int b = blockIdx.x;
  const float* row = logits + b * ld;
  float mx = -INFINITY;
  int amax = 0;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const float v = row[j];
    if (v > mx) {
      mx = v;
      amax = j;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oa = __shfl_xor_sync(0xffffffffu, amax, o);
    if (om > mx || (om == mx && oa < amax)) {
      mx = om;
      amax = oa;
    }
  }
  if ((threadIdx.x & 31) == 0) {
    sh[threadIdx.x >> 5] = mx;
    shi[threadIdx.x >> 5] = amax;
  }
  __syncthreads();
  const int nw = blockDim.x >> 5;
  mx = sh[0];
  amax = shi[0];
  for (int i = 1; i < nw; ++i)
    if (sh[i] > mx || (sh[i] == mx && shi[i] < amax)) {
      mx = sh[i];
      amax = shi[i];
    }
  __syncthreads();
  float s = 0.f;
  for (int j = threadIdx.x; j < N; j += blockDim.x) s += __expf(row[j] - mx);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
  for (int i = 0; i < nw; ++i) s += sh[i];
  const float lse = mx + logf(s);
  if (soft != nullptr || smoothing > 0.f) {
    // general target distribution: sum_c t_c and sum_c t_c x_c by a block reduction, arg-max of t as the "label"
    const float* trow = soft ? soft + b * ld_soft : nullptr;
    const int hard = labels ? static_cast<int>(labels[b]) : -1;
    const float off = smoothing / static_cast<float>(N), on = 1.f - smoothing;
    auto target = [&](int j) { return trow ? trow[j] : (off + (j == hard ? on : 0.f)); };
    float st = 0.f, stx = 0.f, tmx = -INFINITY;
    int tam = 0;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      const float t = target(j);
      st += t;
      stx = fmaf(t, row[j], stx);
      if (t > tmx) tmx = t, tam = j;
    }
    st = warp_sum(st);
    stx = warp_sum(stx);
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, tmx, o);
      const int oa = __shfl_xor_sync(0xffffffffu, tam, o);
      if (om > tmx || (om == tmx && oa < tam)) tmx = om, tam = oa;
    }
    __shared__ float sh2[2][32];
    __syncthreads();
    if ((threadIdx.x & 31) == 0) {
      sh2[0][threadIdx.x >> 5] = st;
      sh2[1][threadIdx.x >> 5] = stx;
      sh[threadIdx.x >> 5] = tmx;
      shi[threadIdx.x >> 5] = tam;
    }
    __syncthreads();
    st = stx = 0.f;
    tmx = sh[0], tam = shi[0];
    for (int i = 0; i < nw; ++i) {
      st += sh2[0][i];
      stx += sh2[1][i];
      if (sh[i] > tmx || (sh[i] == tmx && shi[i] < tam)) tmx = sh[i], tam = shi[i];
    }
    if (threadIdx.x == 0) {
      loss_rows[b] = lse * st - stx;
      if (correct) correct[b] = (amax == (hard >= 0 ? hard : tam)) ? 1 : 0;
    }
    if (dlogits) {
      const float inv = st / s;
      for (int j = threadIdx.x; j < ld_d; j += blockDim.x) {
        float d = 0.f;
        if (j < N) d = (__expf(row[j] - mx) * inv - target(j)) * gscale;
        dlogits[b * ld_d + j] = __float2bfloat16_rn(d);
      }
    }
    return;
  }
  const int label = static_cast<int>(labels[b]);
  if (threadIdx.x == 0) {
    loss_rows[b] = lse - row[label];
    if (correct) correct[b] = (amax == label) ? 1 : 0;
  }
  if (dlogits) {
    const float inv = 1.0f / s;
    for (int j = threadIdx.x; j < ld_d; j += blockDim.x) {
      float d = 0.f;
      if (j < N) d = (__expf(row[j] - mx) * inv - (j == label ? 1.f : 0.f)) * gscale;
      dlogits[b * ld_d + j] = __float2bfloat16_rn(d);
    }
  }
}

// mean of n floats -> out[0] (single block)
__global__ void mean_kernel(const float* __restrict__ v, int n, float* __restrict__ out) {
  pdl_wait();
  __shared__ float sh[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += v[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += sh[i];
    out[0] = t / n;
  }
}

// Column sums of a bf16 matrix [rows][ld] -> fp32 out[cols] (bias gradients). One block per 64 columns.
__global__ void colsum_kernel(const __nv_bfloat16* __restrict__ m, long long rows, long long ld, int cols,
                              float* __restrict__ out, int accumulate) {
  pdl_wait();
  __shared__ float sh[4][64];
  const int cx = threadIdx.x & 63, ry = threadIdx.x >> 6;
  const int c = blockIdx.x * 64 + cx;
  float s = 0.f;
  if (c < cols)
    for (long long r = ry; r < rows; r += 4) s += __bfloat162float(m[r * ld + c]);
  sh[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && c < cols) {
    s = sh[0][cx] + sh[1][cx] + sh[2][cx] + sh[3][cx];
    out[c] = accumulate ? out[c] + s : s;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Weight packing: fp32 OIHW master parameter -> bf16 GEMM operand.
//   mode 0 (forward / wgrad layout): dst[o][tap*I + i]      (row pitch ld_dst, zero padded)
//   mode 1 (dgrad layout):           dst[i][tap*O + o]
//   modes 3 / 4: grouped convolution, src [C][Cg][taps] (O = C, I = Cg, 64 % Cg == 0) -> block-diagonal [C][taps*64]
//     mode 3 (forward): dst[o][tap*64 + j] = W[o][c - g*Cg][tap] with input channel c = (o & ~63) + j, if c is in o's group g
//     mode 4 (dgrad):   dst[c][tap*64 + j] = W[o][c - g*Cg][tap] with output channel o = (c & ~63) + j, if o is in c's group g
//     (taps unflipped as in mode 1; everything outside the group is zero)
__device__ __forceinline__ float grouped_pack_value(const float* __restrict__ src, int Cg, int taps, int mode, long long r,
                                                    long long k) {
  if (k >= static_cast<long long>(taps) * 64) return 0.f;
  const int tap = static_cast<int>(k >> 6);
  const long long other = (r & ~63ll) + (k & 63);   // the channel of the other side in the same 64-channel block
  if (r / Cg != other / Cg) return 0.f;
  const long long o = mode == 3 ? r : other, c = mode == 3 ? other : r;
  return src[(o * Cg + c % Cg) * taps + tap];
}

__global__ void pack_weight_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int O, int I,
                                   int taps, int mode, long long ld_dst) {
  pdl_wait();
  const long long rows = mode == 1 ? I : O;
  const long long total = rows * ld_dst;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = idx / ld_dst;
    const long long k = idx % ld_dst;
    float v = 0.f;
    if (mode >= 3) {
      v = grouped_pack_value(src, I, taps, mode, r, k);
    } else if (mode == 0) {
      if (k < static_cast<long long>(taps) * I) {
        const int tap = static_cast<int>(k / I), i = static_cast<int>(k % I);
        v = src[(r * I + i) * taps + tap];
      }
    } else {
      if (k < static_cast<long long>(taps) * O) {
        const int tap = static_cast<int>(k / O), o = static_cast<int>(k % O);
        v = src[(static_cast<long long>(o) * I + r) * taps + tap];
      }
    }
    dst[idx] = __float2bfloat16_rn(v);
  }
}

// fp32 -> bf16 cast of a flat buffer (n multiple of 1 element; scalar tail-safe).
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = __float2bfloat16_rn(src[i]);
}
__global__ void cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, long long n) {
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = __bfloat162float(src[i]);
}

// Stem im2col: x fp32 NCHW [B][Cin][H][W] -> A bf16 [B*Ho*Wo][ldk], k = (kh*KW + kw)*Cin + c, zero padded to ldk.
// One block per output row (b, oh): the KH input rows of every channel are staged in shared memory with coalesced loads
// (zero padded left/right), then each thread assembles 16-byte output vectors from shared memory.
__global__ void im2col_nchw_kernel(const float* __restrict__ x, uint4* __restrict__ a, int B, int Cin, int H, int W,
                                   int KH, int KW, int stride, int pad, int Ho, int Wo, int ldk) {
  pdl_wait();
  extern __shared__ float srow[];  // [Cin][KH][W + 2*pad] floats, then int lut[ldk]
  const int Wp = W + 2 * pad;
  const int b = blockIdx.x / Ho, oh = blockIdx.x % Ho;
  const int n_in = Cin * KH * Wp;
  int* lut = reinterpret_cast<int*>(srow + n_in);  // k -> offset of tap (kh,kw), channel c inside srow (or -1)
  const int K = KH * KW * Cin;
  for (int k = threadIdx.x; k < ldk; k += blockDim.x) {
    int off = -1;
    if (k < K) {
      const int c = k % Cin, tap = k / Cin;
      off = (c * KH + tap / KW) * Wp + tap % KW;
    }
    lut[k] = off;
  }
  for (int i = threadIdx.x; i < n_in; i += blockDim.x) {
    const int wp = i % Wp;
    const int kh = (i / Wp) % KH;
    const int c = i / (Wp * KH);
    const int ih = oh * stride - pad + kh, iw = wp - pad;
    float v = 0.f;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = __ldg(x + ((static_cast<long long>(b) * Cin + c) * H + ih) * W + iw);
    srow[i] = v;
  }
  __syncthreads();
  const int kvec = ldk / 8;
  uint4* out = a + (static_cast<long long>(b) * Ho + oh) * Wo * kvec;
  // thread -> fixed k-octet (its 8 lut entries stay in registers), strides over output pixels
  const int kv = threadIdx.x % kvec;
  const int ow0 = threadIdx.x / kvec, ow_step = blockDim.x / kvec;
  if (ow0 < ow_step) {
    int off[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) off[j] = lut[kv * 8 + j];
    for (int ow = ow0; ow < Wo; ow += ow_step) {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = off[j] >= 0 ? srow[off[j] + ow * stride] : 0.f;
      out[ow * kvec + kv] = pack8(v);
    }
  }
}

// Multi-tensor weight packing: one launch packs every conv / linear weight of a model.
// table[e] = {src, dst, O, I, taps, mode, ld_dst, first_block, rows_out, oscale} (int64 each); grid = total blocks.
// oscale (optional fp32 [O]) multiplies every weight of output channel o (layer scale folded into the dgrad operand).
// Every layout goes through a shared-memory tile so that the fp32 parameter is read in contiguous runs and the bf16
// operand is written in contiguous runs (the first version walked the destination with 64-bit div/mod per element and
// stride-`taps` / stride-`I*taps` reads: 0.24 ms per step, now bandwidth bound):
//   mode 0, taps > 1 : per output channel, a run of i's x all taps  ([i][tap] -> [tap][i])
//   mode 1           : 32 (o) x 32 (i) x taps tiles                 ([o][i][tap] -> [i][tap][o])
//   mode 0, taps = 1 : straight row copy
constexpr int kPackTileFloats = 32 * (32 * 9 + 1);

__device__ __forceinline__ void pack_zero_pad(__nv_bfloat16* dst, long long rows_src, long long rows_out, long long cols,
                                              long long ld, long long b, long long nblk) {
  // columns [cols, ld) of the live rows, then the rows [rows_src, rows_out)
  const long long padc = ld - cols;
  const __nv_bfloat16 z = __float2bfloat16_rn(0.f);
  if (padc > 0)
    for (long long idx = b * blockDim.x + threadIdx.x; idx < rows_src * padc; idx += nblk * blockDim.x)
      dst[(idx / padc) * ld + cols + idx % padc] = z;
  for (long long idx = b * blockDim.x + threadIdx.x; idx < (rows_out - rows_src) * ld; idx += nblk * blockDim.x)
    dst[rows_src * ld + idx] = z;
}

__global__ void __launch_bounds__(256) pack_weights_multi_kernel(const long long* __restrict__ table, int n_entries) {
  pdl_wait();
  __shared__ int entry;
  __shared__ float sm[kPackTileFloats];
  if (threadIdx.x == 0) {
    // last entry whose first block is <= blockIdx.x (binary search: the table holds ~100-200 entries)
    int lo = 0, hi = n_entries - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (table[mid * 10 + 7] <= static_cast<long long>(blockIdx.x)) lo = mid; else hi = mid - 1;
    }
    entry = lo;
  }
  __syncthreads();
  const long long* t = table + entry * 10;
  const float* __restrict__ src = reinterpret_cast<const float*>(t[0]);
  __nv_bfloat16* __restrict__ dst = reinterpret_cast<__nv_bfloat16*>(t[1]);
  const int O = static_cast<int>(t[2]), I = static_cast<int>(t[3]), taps = static_cast<int>(t[4]);
  const int mode = static_cast<int>(t[5]);
  const long long ld = t[6], first = t[7], rows_out = t[8];
  const float* __restrict__ oscale = reinterpret_cast<const float*>(t[9]);
  const long long next_first = (entry + 1 < n_entries) ? table[(entry + 1) * 10 + 7] : static_cast<long long>(gridDim.x);
  const int nblk = static_cast<int>(next_first - first);
  const int blk = static_cast<int>(blockIdx.x - first);
  const int tid = threadIdx.x;

  if (mode == 2) {
    // space-to-depth stem operand: src [O][3][7][7] -> dst [O][256], k = ky4*64 + kx4*16 + (dy*2+dx)*3 + c with
    // kernel row 2*ky4+dy and column 2*kx4+dx (taps that fall outside the 7x7 kernel and channels 12..15 are zero)
    const int total = static_cast<int>(rows_out * ld);
    for (int idx = blk * 256 + tid; idx < total; idx += nblk * 256) {
      const int r = idx / static_cast<int>(ld), k = idx % static_cast<int>(ld);
      float v = 0.f;
      if (r < O && k < 256) {
        const int ky4 = k >> 6, kx4 = (k >> 4) & 3, q = k & 15;
        if (q < 12) {
          const int d = q / 3, c = q - d * 3;
          const int kh = 2 * ky4 + (d >> 1), kw = 2 * kx4 + (d & 1);
          if (kh < 7 && kw < 7) v = src[((r * 3 + c) * 7 + kh) * 7 + kw];
        }
      }
      dst[idx] = __float2bfloat16_rn(v);
    }
    return;
  }

  if (mode >= 3) {
    // grouped convolution operands (see grouped_pack_value): rows_out = O = C
    for (long long idx = blk * 256ll + tid; idx < rows_out * ld; idx += nblk * 256ll) {
      const long long r = idx / ld, k = idx % ld;
      dst[idx] = __float2bfloat16_rn(r < O ? grouped_pack_value(src, I, taps, mode, r, k) : 0.f);
    }
    return;
  }

  if (mode == 0 && taps == 1) {
    // dst[o][i] = src[o][i]: contiguous rows; 8 floats -> one 16-byte store per thread when the row allows it
    const bool vec = (I % 8 == 0) && (ld % 8 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
    for (int o = blk; o < O; o += nblk) {
      const float sc = oscale ? oscale[o] : 1.f;
      const float* s0 = src + static_cast<long long>(o) * I;
      __nv_bfloat16* d0 = dst + o * ld;
      if (vec) {
        for (int i = tid * 8; i < I; i += 256 * 8) {
          float f[8];
          load8f(s0 + i, f);
#pragma unroll
          for (int k = 0; k < 8; ++k) f[k] *= sc;
          *reinterpret_cast<uint4*>(d0 + i) = pack8(f);
        }
      } else {
        for (int i = tid; i < I; i += 256) d0[i] = __float2bfloat16_rn(s0[i] * sc);
      }
    }
    pack_zero_pad(dst, O, rows_out, I, ld, blk, nblk);
    return;
  }

  if (mode == 1 && taps == 1 && O % 8 == 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    // plain transpose [O][I] -> [I][O] (every linear layer's dgrad operand): 32 (i) x 64 (o) tiles, reads run along i
    // (128-byte rows), every thread writes 8 consecutive o of one i as ONE 16-byte store
    constexpr int TP = 33;                       // pitch of sm[o][i]
    const int tiles_o = (O + 63) / 64, tiles_i = (I + 31) / 32;
    for (int w = blk; w < tiles_o * tiles_i; w += nblk) {
      const int o0 = (w % tiles_o) * 64, i0 = (w / tiles_o) * 32;
      const int no = min(64, O - o0), ni = min(32, I - i0);
      __syncthreads();
      for (int e = tid; e < 64 * 32; e += 256) {
        const int oo = e >> 5, ii = e & 31;
        float v = 0.f;
        if (oo < no && ii < ni) {
          v = src[static_cast<long long>(o0 + oo) * I + i0 + ii];
          if (oscale) v *= oscale[o0 + oo];
        }
        sm[oo * TP + ii] = v;
      }
      __syncthreads();
      {
        const int ii = tid >> 3, og = (tid & 7) * 8;     // 32 i x 8 groups of 8 o
        if (ii < ni && og < no) {                        // (O % 8 == 0: a group is all-valid or all-invalid)
          float f[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) f[k] = sm[(og + k) * TP + ii];
          *reinterpret_cast<uint4*>(dst + static_cast<long long>(i0 + ii) * ld + o0 + og) = pack8(f);
        }
      }
    }
    pack_zero_pad(dst, I, rows_out, static_cast<long long>(O), ld, blk, nblk);
    return;
  }

  if (mode == 0 && taps <= 64) {
    // per output channel o and run of `piece` input channels: src[(o*I + i)*taps + tap] is one contiguous run
    const int piece = (kPackTileFloats - 64) / taps;
    const int pieces = (I + piece - 1) / piece;
    for (int w = blk; w < O * pieces; w += nblk) {
      const int o = w / pieces, i0 = (w - o * pieces) * piece;
      const int ni = min(piece, I - i0);
      const float* s0 = src + (static_cast<long long>(o) * I + i0) * taps;
      const float sc = oscale ? oscale[o] : 1.f;
      __syncthreads();
      for (int e = tid; e < ni * taps; e += 256) sm[e] = s0[e] * sc;
      __syncthreads();
      __nv_bfloat16* d0 = dst + o * ld + i0;
      if ((ni & 1) == 0 && (I & 1) == 0 && (i0 & 1) == 0 && (ld & 1) == 0) {
        // two neighbouring input channels per 4-byte store (half the store instructions; 128-byte runs per warp)
        const int hn = ni >> 1;
        for (int e = tid; e < hn * taps; e += 256) {
          const int tap = e / hn, i = (e - tap * hn) * 2;
          *reinterpret_cast<uint32_t*>(d0 + static_cast<long long>(tap) * I + i) =
              pack_bf16x2(sm[i * taps + tap], sm[(i + 1) * taps + tap]);
        }
      } else {
        for (int e = tid; e < ni * taps; e += 256) {
          const int tap = e / ni, i = e - tap * ni;
          d0[static_cast<long long>(tap) * I + i] = __float2bfloat16_rn(sm[i * taps + tap]);
        }
      }
    }
    pack_zero_pad(dst, O, rows_out, static_cast<long long>(taps) * I, ld, blk, nblk);
    return;
  }

  if (mode == 1 && taps <= 9) {
    // 32 (o) x 32 (i) x taps tiles: reads run along [i][tap] of one o, writes run along o
    const int pitch = 32 * taps + 1;
    const int tiles_o = (O + 31) / 32, tiles_i = (I + 31) / 32;
    for (int w = blk; w < tiles_o * tiles_i; w += nblk) {
      const int o0 = (w % tiles_o) * 32, i0 = (w / tiles_o) * 32;
      const int no = min(32, O - o0), ni = min(32, I - i0);
      const int run = ni * taps;
      __syncthreads();
      for (int e = tid; e < no * run; e += 256) {
        const int oo = e / run, rem = e - oo * run;
        float v = src[(static_cast<long long>(o0 + oo) * I + i0) * taps + rem];
        if (oscale) v *= oscale[o0 + oo];
        sm[oo * pitch + rem] = v;
      }
      __syncthreads();
      if ((no & 1) == 0 && (O & 1) == 0 && (ld & 1) == 0) {
        for (int e = tid; e < run * 16; e += 256) {
          const int oo = (e & 15) * 2, rem = e >> 4;   // rem = ii * taps + tap; two neighbouring output channels per store
          if (oo < no) {
            const int ii = rem / taps, tap = rem - ii * taps;
            *reinterpret_cast<uint32_t*>(dst + (i0 + ii) * ld + static_cast<long long>(tap) * O + o0 + oo) =
                pack_bf16x2(sm[oo * pitch + rem], sm[(oo + 1) * pitch + rem]);
          }
        }
      } else {
        for (int e = tid; e < run * 32; e += 256) {
          const int oo = e & 31, rem = e >> 5;   // rem = ii * taps + tap
          if (oo < no) {
            const int ii = rem / taps, tap = rem - ii * taps;
            dst[(i0 + ii) * ld + static_cast<long long>(tap) * O + o0 + oo] = __float2bfloat16_rn(sm[oo * pitch + rem]);
          }
        }
      }
    }
    pack_zero_pad(dst, I, rows_out, static_cast<long long>(taps) * O, ld, blk, nblk);
    return;
  }

  // generic fallback (any tap count)
  const long long total = rows_out * ld;
  const long long rows_src = mode == 0 ? O : I;
  for (long long idx = static_cast<long long>(blk) * 256 + tid; idx < total; idx += nblk * 256ll) {
    const long long r = idx / ld;
    const long long k = idx % ld;
    float v = 0.f;
    if (r < rows_src) {
      if (mode == 0) {
        if (k < static_cast<long long>(taps) * I) {
          const int tap = static_cast<int>(k / I), i = static_cast<int>(k % I);
          v = src[(r * I + i) * taps + tap];
          if (oscale) v *= oscale[r];
        }
      } else {
        if (k < static_cast<long long>(taps) * O) {
          const int tap = static_cast<int>(k / O), o = static_cast<int>(k % O);
          v = src[(static_cast<long long>(o) * I + r) * taps + tap];
          if (oscale) v *= oscale[o];
        }
      }
    }
    dst[idx] = __float2bfloat16_rn(v);
  }
}

// Stem weight gradient: patch-matrix layout [Cout][ldk] with k = tap*Cin + c  ->  OIHW [Cout][Cin][taps].
__global__ void stem_wgrad_relayout_kernel(const float* __restrict__ src, float* __restrict__ dst, int Cout, int Cin,
                                           int taps, int ldk, int accumulate) {
  pdl_wait();
  const long long total = static_cast<long long>(Cout) * Cin * taps;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(i % taps);
    const int c = static_cast<int>((i / taps) % Cin);
    const int o = static_cast<int>(i / (static_cast<long long>(taps) * Cin));
    const float v = src[static_cast<long long>(o) * ldk + t * Cin + c];
    dst[i] = accumulate ? dst[i] + v : v;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Fused SGD with momentum over a flat fp32 arena (torch.optim.SGD semantics, dampening 0, no nesterov):
//   g' = g*gscale + wd*p ; buf = first ? g' : mu*buf + g' ; p -= lr*buf
__global__ void sgd_momentum_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf,
                                    long long n, float lr, const float* __restrict__ lr_dev, float momentum, float wd,
                                    float gscale, int first_step, const float* __restrict__ clip) {
  pdl_wait();
  if (lr_dev != nullptr) lr = __ldg(lr_dev);  // device-resident learning rate: lets a captured CUDA graph follow a schedule
  if (clip != nullptr) gscale *= __ldg(clip);  // global-norm clipping coefficient (b200_grad_clip_coef)
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float pv = p[i];
    const float gg = fmaf(wd, pv, g[i] * gscale);
    const float bv = first_step ? gg : fmaf(momentum, buf[i], gg);
    buf[i] = bv;
    p[i] = pv - lr * bv;
  }
}

// Space-to-depth input of the stem: x fp32 NCHW [B][3][H][W] (H, W even) -> z bf16 [B][H/2+3][W/2+3][16],
// z[b][Y][X][(dy*2+dx)*3 + c] = xpad[b][c][2Y+dy][2X+dx] with xpad = x zero-padded by 3 pixels; channels 12..15 = 0.
__global__ void stem_s2d_kernel(const float* __restrict__ x, uint4* __restrict__ z, int B, int H, int W) {
  pdl_wait();
  const int Hz = H / 2 + 3, Wz = W / 2 + 3;
  const long long total = static_cast<long long>(B) * Hz * Wz;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int X = static_cast<int>(i % Wz);
    const int Y = static_cast<int>((i / Wz) % Hz);
    const long long b = i / (static_cast<long long>(Wz) * Hz);
    float v[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) v[q] = 0.f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const int h = 2 * Y + dy - 3;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int w = 2 * X + dx - 3;
        if (w < 0 || w >= W) continue;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[(dy * 2 + dx) * 3 + c] = __ldg(x + ((b * 3 + c) * H + h) * W + w);
      }
    }
    float lo[8], hi[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) lo[q] = v[q], hi[q] = v[8 + q];
    z[2 * i] = pack8(lo);
    z[2 * i + 1] = pack8(hi);
  }
}

// Stride-2 helpers of the downsample branch on the BatchNorm-algebra path (engine/resnet.py): the 1x1 / stride-2 convolution
// only ever sees the even pixels of its input, so the branch runs on a COMPACT copy xs[b][i][j][:] = x[b][2i][2j][:] (a quarter
// of x) as a flat GEMM, and its data gradient is added back onto the even pixels: gx[b][2i][2j][:] += gs[b][i][j][:].
__global__ void __launch_bounds__(256) subsample2_kernel(const uint4* __restrict__ x, uint4* __restrict__ xs, int B, int H, int W,
                                                         int cvec) {
  pdl_wait();
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const unsigned total = static_cast<unsigned>(B) * Ho * Wo * cvec;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned c = i % cvec;
    unsigned t = i / cvec;
    const unsigned ow = t % Wo;
    t /= Wo;
    const unsigned oh = t % Ho;
    const unsigned b = t / Ho;
    xs[i] = __ldg(x + ((b * H + 2 * oh) * W + 2 * ow) * cvec + c);
  }
}
__global__ void __launch_bounds__(256) add_even_pixels_kernel(uint4* __restrict__ gx, const uint4* __restrict__ gs, int B, int H,
                                                              int W, int cvec) {
  pdl_wait();
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const unsigned total = static_cast<unsigned>(B) * Ho * Wo * cvec;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned c = i % cvec;
    unsigned t = i / cvec;
    const unsigned ow = t % Wo;
    t /= Wo;
    const unsigned oh = t % Ho;
    const unsigned b = t / Ho;
    uint4* dst = gx + ((b * H + 2 * oh) * W + 2 * ow) * cvec + c;
    float a[8], d[8];
    unpack8(*dst, a);
    unpack8(__ldg(gs + i), d);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] += d[k];
    *dst = pack8(a);
  }
}

// GPU input pipeline (SURVEY 8(f)-1): the same space-to-depth operand straight from the DECODED image batch,
// x uint8 NHWC [B][H][W][3] (what a JPEG decoder / PIL produces), with the reference's ToTensor + Normalize
// (classification/resnet/train.py:46-71: x / 255, then (x - mean[c]) / std[c]) fused in: z = bf16((u8 * a[c]) + b[c]),
// a = 1 / (255 std), b = -mean / std.  The host->device copy shrinks 4x (1 byte instead of 4 per value) and the
// fp32 NCHW batch never exists.
__global__ void stem_s2d_u8_kernel(const unsigned char* __restrict__ x, uint4* __restrict__ z, int B, int H, int W, float a0,
                                   float a1, float a2, float b0, float b1, float b2) {
  pdl_wait();
  const int Hz = H / 2 + 3, Wz = W / 2 + 3;
  const long long total = static_cast<long long>(B) * Hz * Wz;
  const float a[3] = {a0, a1, a2}, bb[3] = {b0, b1, b2};
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int X = static_cast<int>(i % Wz);
    const int Y = static_cast<int>((i / Wz) % Hz);
    const long long b = i / (static_cast<long long>(Wz) * Hz);
    float v[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) v[q] = 0.f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const int h = 2 * Y + dy - 3;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int w = 2 * X + dx - 3;
        if (w < 0 || w >= W) continue;
        const unsigned char* px = x + ((b * H + h) * W + w) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[(dy * 2 + dx) * 3 + c] = fmaf(static_cast<float>(px[c]), a[c], bb[c]);
      }
    }
    float lo[8], hi[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) lo[q] = v[q], hi[q] = v[8 + q];
    z[2 * i] = pack8(lo);
    z[2 * i + 1] = pack8(hi);
  }
}

// The same ToTensor + Normalize for the other families: uint8 NHWC -> fp32 NCHW (the layout their patch-embedding kernels read).
__global__ void u8_nhwc_to_f32_nchw_kernel(const unsigned char* __restrict__ x, float* __restrict__ y, int B, int H, int W,
                                           float a0, float a1, float a2, float b0, float b1, float b2) {
  pdl_wait();
  const long long total = static_cast<long long>(B) * H * W;
  const long long plane = static_cast<long long>(H) * W;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / plane, p = i - b * plane;
    const unsigned char* px = x + i * 3;
    float* o = y + b * 3 * plane + p;
    o[0] = fmaf(static_cast<float>(px[0]), a0, b0);
    o[plane] = fmaf(static_cast<float>(px[1]), a1, b1);
    o[2 * plane] = fmaf(static_cast<float>(px[2]), a2, b2);
  }
}

// Weight gradient of the space-to-depth stem: g[64][k64 = kx4*16 + (dy*2+dx)*3 + c][ky4] -> dW [64][3][7][7] (OIHW).
__global__ void stem_s2d_wgrad_relayout_kernel(const float* __restrict__ g, float* __restrict__ dw, int accumulate) {
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 64 * 3 * 49) return;
  const int kw = i % 7, kh = (i / 7) % 7, c = (i / 49) % 3, o = i / 147;
  const int ky4 = kh >> 1, dy = kh & 1, kx4 = kw >> 1, dx = kw & 1;
  const float v = g[(o * 64 + kx4 * 16 + (dy * 2 + dx) * 3 + c) * 4 + ky4];
  dw[i] = accumulate ? dw[i] + v : v;
}

// Stochastic depth (drop_path of the reference: classification/convNext/models/networks.py:11-26, vision_transformer/
// vit_model.py:12-40, timm DropPath in swin_transformer.py:282,285): y[b, ...] = x[b, ...] * scale[b], scale[b] =
// floor(keep + U_b) / keep.  Used on the BACKWARD side (the gradient entering a dropped residual branch); the forward side
// lives in the GEMM epilogue (ConvGemmParams::rowscale).  vec_per_sample = elements per sample / 8.
__global__ void __launch_bounds__(256) rowscale_bf16_kernel(const uint4* __restrict__ x, const float* __restrict__ scale,
                                                            uint4* __restrict__ y, long long nvec, long long vec_per_sample) {
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float s = __ldg(scale + i / vec_per_sample);
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (s != 0.f) {   // a dropped sample: no read of x at all
      float f[8];
      unpack8(__ldg(x + i), f);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] *= s;
      o = pack8(f);
    }
    y[i] = o;
  }
}

// ViT pre_logits activation (vit_model.py:218-221: Linear -> Tanh on the class-token row).  t = tanh(u) (fp32, kept for the
// backward) and its bf16 copy for the classifier GEMM;  backward: du = dt * (1 - t^2)  (bf16 in / out).
__global__ void __launch_bounds__(256) tanh_fwd_kernel(const float* __restrict__ u, float* __restrict__ t,
                                                       __nv_bfloat16* __restrict__ t16, long long n) {
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = tanhf(u[i]);
    t[i] = v;
    t16[i] = __float2bfloat16(v);
  }
}
__global__ void __launch_bounds__(256) tanh_bwd_kernel(const __nv_bfloat16* __restrict__ dt, const float* __restrict__ t,
                                                       __nv_bfloat16* __restrict__ du, long long n) {
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = t[i];
    du[i] = __float2bfloat16(__bfloat162float(dt[i]) * (1.0f - v * v));
  }
}

}  // namespace b200
