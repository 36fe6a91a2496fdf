// RepVGG block passes (classification/RepVGG/models/repvgg.py RepVGGBlock): three BatchNorms on three branches feed ONE
// sum, so each direction makes one pass over the block's tensors instead of one per branch.
//
//   forward   y = relu(c3 * s3 + c1 * s1 [+ x * s_id] + (t3 + t1 [+ t_id]))      c3 / c1: raw 3x3 / 1x1 conv outputs
//             (+ per-CTA sums of the stored bf16 y and y^2: the batch statistics of the next block's identity BatchNorm)
//   backward  reduce: dz = g * [y > 0]; per channel sum(dz), sum(dz * c3), sum(dz * c1) [, sum(dz * x)]
//             apply:  dc_b = scale_b * (dz - m1_b - xhat_b * m2_b) for every branch b (b200_bn_bwd_finalize's m1 / m2)
//   eval      fold: K = W3 t3 + pad(W1) t1 [+ I t_id], b = sum_b (beta_b - mean_b t_b), t = gamma / sqrt(var + eps)
//
// The backward apply recomputes dz from g and y instead of reading a dz the reduce pass stored: with an identity branch
// both choices move 13 bf16 tensor-sized streams (reduce 5 reads; apply 5 reads + 3 writes, or reduce 5 reads + 1 write;
// apply 4 reads + 3 writes), without one both move 10, so recomputing costs no traffic and saves a buffer.
//
// Thread mapping of the three streaming passes: a thread owns one 8-channel group (16-byte vectors) of a channel chunk
// (gridDim.y chunks of <= 256 groups) and strides over the rows of its CTA's row range; the rpi = 256 / gpc threads of a
// group reduce their sums through shared memory in a fixed order (no atomics), one [2][C] partial row per CTA row range.
#pragma once
#include "row_passes.cuh"

namespace b200 {

// ---------------------------------------------------------------------------------------------------------- forward
template <bool ID, bool STATS>
__global__ void __launch_bounds__(256, 2) repvgg_apply_kernel(
    const __nv_bfloat16* __restrict__ c3, long long ld3, const __nv_bfloat16* __restrict__ c1, long long ld1,
    const __nv_bfloat16* __restrict__ x, long long ldx, const float* __restrict__ co3, const float* __restrict__ co1,
    const float* __restrict__ coid, uint4* __restrict__ y, long long rows, int C, int rows_per_block, int gpc,
    float* __restrict__ stats) {
  pdl_wait();
  const int cvec = C / 8, rpi = 256 / gpc;
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;
  const int cg = blockIdx.y * gpc + lane_g;
  const bool live = rsub < rpi && cg < cvec;
  float acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
  if (live) {
    float s3[8], s1[8], sid[8], sh[8], t[8];
    load8f(co3 + 2 * C + cg * 8, s3);
    load8f(co1 + 2 * C + cg * 8, s1);
    load8f(co3 + 3 * C + cg * 8, sh);
    load8f(co1 + 3 * C + cg * 8, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) sh[j] += t[j];
    if constexpr (ID) {
      load8f(coid + 2 * C + cg * 8, sid);
      load8f(coid + 3 * C + cg * 8, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) sh[j] += t[j];
    }
    const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
    const long long r1 = min(rows, r0 + rows_per_block);
    for (long long r = r0 + rsub; r < r1; r += 4 * rpi) {
      uint4 q3[4], q1[4], qx[4];
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const long long rr = r + h * rpi;
        if (rr < r1) {
          q3[h] = rv_ld(c3, ld3, rr, cg);
          q1[h] = rv_ld(c1, ld1, rr, cg);
          if constexpr (ID) qx[h] = rv_ld(x, ldx, rr, cg);
        }
      }
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const long long rr = r + h * rpi;
        if (rr >= r1) break;
        float a[8], b[8], v[8];
        unpack8(q3[h], a);
        unpack8(q1[h], b);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = sh[j];
        if constexpr (ID) {
          float xv[8];
          unpack8(qx[h], xv);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = fmaf(xv[j], sid[j], v[j]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(fmaf(a[j], s3[j], fmaf(b[j], s1[j], v[j])), 0.f);
        const uint4 o = pack8(v);
        y[rr * cvec + cg] = o;
        if constexpr (STATS) {
          unpack8(o, v);   // statistics of the stored bf16 values, which are what the next block normalises
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            acc[0][j] += v[j];
            acc[1][j] = fmaf(v[j], v[j], acc[1][j]);
          }
        }
      }
    }
  }
  if constexpr (STATS) {
    if (rv_cta_reduce<2>(acc, gpc, rpi, lane_g, rsub) && live) {
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int j = 0; j < 8; ++j) stats[(static_cast<long long>(blockIdx.x) * 2 + s) * C + cg * 8 + j] = acc[s][j];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- backward
// partial[b][T][2][C], b = 0 dense, 1 1x1, 2 identity: {sum dz, sum dz * input of branch b}, the rows b200_bn_bwd_finalize
// reads (with the branch's mean / invstd it turns sum(dz * c) into sum(dz * xhat)).
template <bool ID>
__global__ void __launch_bounds__(256, 2) repvgg_bwd_reduce_kernel(
    const uint4* __restrict__ g, const uint4* __restrict__ y, const __nv_bfloat16* __restrict__ c3, long long ld3,
    const __nv_bfloat16* __restrict__ c1, long long ld1, const __nv_bfloat16* __restrict__ x, long long ldx, long long rows,
    int C, int rows_per_block, int gpc, float* __restrict__ partial) {
  pdl_wait();
  constexpr int NS = ID ? 4 : 3;
  const int cvec = C / 8, rpi = 256 / gpc;
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;
  const int cg = blockIdx.y * gpc + lane_g;
  const bool live = rsub < rpi && cg < cvec;
  float acc[NS][8];
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[s][j] = 0.f;
  if (live) {
    const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
    const long long r1 = min(rows, r0 + rows_per_block);
    for (long long r = r0 + rsub; r < r1; r += 2 * rpi) {
      uint4 qg[2], qy[2], q3[2], q1[2], qx[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long rr = r + h * rpi;
        if (rr < r1) {
          qg[h] = __ldg(g + rr * cvec + cg);
          qy[h] = __ldg(y + rr * cvec + cg);
          q3[h] = rv_ld(c3, ld3, rr, cg);
          q1[h] = rv_ld(c1, ld1, rr, cg);
          if constexpr (ID) qx[h] = rv_ld(x, ldx, rr, cg);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (r + h * rpi >= r1) break;
        float dz[8], yv[8], a[8], b[8];
        unpack8(qg[h], dz);
        unpack8(qy[h], yv);
        unpack8(q3[h], a);
        unpack8(q1[h], b);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          dz[j] = yv[j] > 0.f ? dz[j] : 0.f;
          acc[0][j] += dz[j];
          acc[1][j] = fmaf(dz[j], a[j], acc[1][j]);
          acc[2][j] = fmaf(dz[j], b[j], acc[2][j]);
        }
        if constexpr (ID) {
          float xv[8];
          unpack8(qx[h], xv);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[NS - 1][j] = fmaf(dz[j], xv[j], acc[NS - 1][j]);
        }
      }
    }
  }
  if (rv_cta_reduce<NS>(acc, gpc, rpi, lane_g, rsub) && live) {
    const long long T = gridDim.x;
#pragma unroll
    for (int b = 0; b < NS - 1; ++b) {
      float* p = partial + (static_cast<long long>(b) * T + blockIdx.x) * 2 * C + cg * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        p[j] = acc[0][j];
        p[C + j] = acc[b + 1][j];
      }
    }
  }
}

template <bool ID>
__global__ void __launch_bounds__(256) repvgg_bwd_apply_kernel(
    const uint4* __restrict__ g, const uint4* __restrict__ y, const __nv_bfloat16* __restrict__ c3, long long ld3,
    const __nv_bfloat16* __restrict__ c1, long long ld1, const __nv_bfloat16* __restrict__ x, long long ldx,
    const float* __restrict__ co3, const float* __restrict__ m3, const float* __restrict__ co1, const float* __restrict__ m1,
    const float* __restrict__ coid, const float* __restrict__ mid, __nv_bfloat16* __restrict__ dc3,
    __nv_bfloat16* __restrict__ dc1, __nv_bfloat16* __restrict__ dx, long long rows, int C, int rows_per_block, int gpc) {
  pdl_wait();
  const int cvec = C / 8, rpi = 256 / gpc;
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;
  const int cg = blockIdx.y * gpc + lane_g;
  if (rsub >= rpi || cg >= cvec) return;
  float a3[8], b3[8], k3[8], a1[8], b1[8], k1[8], ai[8], bi[8], ki[8];
  rv_bwd_coeffs(co3, co3 + C, co3 + 2 * C, m3, m3 + C, cg, a3, b3, k3);
  rv_bwd_coeffs(co1, co1 + C, co1 + 2 * C, m1, m1 + C, cg, a1, b1, k1);
  if constexpr (ID) rv_bwd_coeffs(coid, coid + C, coid + 2 * C, mid, mid + C, cg, ai, bi, ki);
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  for (long long r = r0 + rsub; r < r1; r += 2 * rpi) {
    uint4 qg[2], qy[2], q3[2], q1[2], qx[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long rr = r + h * rpi;
      if (rr < r1) {
        qg[h] = __ldg(g + rr * cvec + cg);
        qy[h] = __ldg(y + rr * cvec + cg);
        q3[h] = rv_ld(c3, ld3, rr, cg);
        q1[h] = rv_ld(c1, ld1, rr, cg);
        if constexpr (ID) qx[h] = rv_ld(x, ldx, rr, cg);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long rr = r + h * rpi;
      if (rr >= r1) break;
      float dz[8], yv[8], u[8];
      unpack8(qg[h], dz);
      unpack8(qy[h], yv);
#pragma unroll
      for (int j = 0; j < 8; ++j) dz[j] = yv[j] > 0.f ? dz[j] : 0.f;
      unpack8(q3[h], u);
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = fmaf(a3[j], dz[j], fmaf(-b3[j], u[j], k3[j]));
      *reinterpret_cast<uint4*>(dc3 + rr * ld3 + cg * 8) = pack8(u);
      unpack8(q1[h], u);
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = fmaf(a1[j], dz[j], fmaf(-b1[j], u[j], k1[j]));
      *reinterpret_cast<uint4*>(dc1 + rr * ld1 + cg * 8) = pack8(u);
      if constexpr (ID) {
        unpack8(qx[h], u);
#pragma unroll
        for (int j = 0; j < 8; ++j) u[j] = fmaf(ai[j], dz[j], fmaf(-bi[j], u[j], ki[j]));
        *reinterpret_cast<uint4*>(dx + rr * ldx + cg * 8) = pack8(u);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- eval fold
// wp bf16 [O][ldk], k = tap * I + i (the b200_pack_weight mode-0 layout; zero for k >= 9 * I), bias fp32 [O].
struct RvFoldBn {
  const float *gamma, *beta, *mean, *var;
  float eps;
};

__device__ __forceinline__ float rv_fold_t(const RvFoldBn& bn, int o) {
  return bn.gamma[o] / sqrtf(bn.var[o] + bn.eps);
}
// beta - mean * gamma / std, rounded as _fuse_bn_tensor of the reference computes it
__device__ __forceinline__ float rv_fold_b(const RvFoldBn& bn, int o) {
  return bn.beta[o] - bn.mean[o] * bn.gamma[o] / sqrtf(bn.var[o] + bn.eps);
}

__global__ void __launch_bounds__(256) repvgg_fold_kernel(const float* __restrict__ w3, const float* __restrict__ w1,
                                                          RvFoldBn bn3, RvFoldBn bn1, RvFoldBn bnid, int O, int I,
                                                          int ldk, __nv_bfloat16* __restrict__ wp,
                                                          float* __restrict__ bias) {
  pdl_wait();
  const long long total = static_cast<long long>(O) * ldk;
  for (long long idx = blockIdx.x * 256ll + threadIdx.x; idx < total; idx += static_cast<long long>(gridDim.x) * 256) {
    const int o = static_cast<int>(idx / ldk), k = static_cast<int>(idx % ldk);
    const int tap = k / I, i = k - tap * I;
    float v = 0.f;
    if (tap < 9) {
      v = w3[(static_cast<long long>(o) * I + i) * 9 + tap] * rv_fold_t(bn3, o);
      if (tap == 4) {
        v += w1[static_cast<long long>(o) * I + i] * rv_fold_t(bn1, o);
        if (bnid.gamma != nullptr && i == o) v += rv_fold_t(bnid, o);
      }
    }
    wp[idx] = __float2bfloat16_rn(v);
    if (k == 0) {
      float b = rv_fold_b(bn3, o) + rv_fold_b(bn1, o);
      if (bnid.gamma != nullptr) b += rv_fold_b(bnid, o);
      bias[o] = b;
    }
  }
}

}  // namespace b200
