// Helpers of the row-streaming BatchNorm passes (repvgg.cuh, mbconv.cuh, elementwise.cuh's BatchNorm backward apply): the
// thread / CTA geometry over [rows][C] NHWC tensors, the fixed-order CTA reduction of per-channel sums into one [2][C]
// partial row per CTA, and the coefficients of the BatchNorm backward apply.
//
// Thread mapping: a thread owns one 8-channel group (16-byte vectors) of a channel chunk (gridDim.y chunks of <= 256 groups)
// and strides over the rows of its CTA's row range; the rpi = 256 / gpc threads of a group reduce their sums through shared
// memory in a fixed order (no atomics).
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int kRvMaxC = 8192;     // bn_finalize / bn_bwd_finalize limit
constexpr int kRvTargetCtas = kNumSMs * 8;

struct RvGeom {
  int nchunk, gpc, rpi, blocks, rows_per_block;
};

// gridDim = (blocks, nchunk); independent of the device so that the partial-row count is known without one
__host__ __device__ inline RvGeom repvgg_geom(long long rows, int C) {
  RvGeom g;
  const int cvec = C / 8;
  g.nchunk = (cvec + 255) / 256;
  g.gpc = (cvec + g.nchunk - 1) / g.nchunk;
  g.rpi = 256 / g.gpc;
  long long blocks = kRvTargetCtas / g.nchunk;
  if (blocks < 1) blocks = 1;
  long long rpb = (rows + blocks - 1) / blocks;
  rpb = ((rpb + g.rpi - 1) / g.rpi) * g.rpi;
  blocks = (rows + rpb - 1) / rpb;
  g.blocks = static_cast<int>(blocks);
  g.rows_per_block = static_cast<int>(rpb);
  return g;
}

__device__ __forceinline__ uint4 rv_ld(const __nv_bfloat16* __restrict__ base, long long ld, long long r, int cg) {
  return __ldg(reinterpret_cast<const uint4*>(base + r * ld + cg * 8));
}

// Fixed-order reduction of NS per-thread sums of 8 channels over the rpi threads of each channel group; the rsub == 0
// thread of the group returns true with the CTA's totals in acc.
template <int NS>
__device__ __forceinline__ bool rv_cta_reduce(float (&acc)[NS][8], int gpc, int rpi, int lane_g, int rsub) {
  __shared__ float red[256][NS * 8 + 1];
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int j = 0; j < 8; ++j) red[threadIdx.x][s * 8 + j] = acc[s][j];
  __syncthreads();
  if (rsub != 0 || rsub >= rpi) return false;
  for (int k = 1; k < rpi; ++k) {
    const float* o = red[k * gpc + lane_g];
#pragma unroll
    for (int s = 0; s < NS; ++s)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[s][j] += o[s * 8 + j];
  }
  return true;
}

// dc = a * dz - bq * c + cq with a = scale, bq = scale * invstd * m2, cq = scale * (mean * invstd * m2 - m1): the
// BatchNorm backward apply, dc = scale * (dz - m1 - (c - mean) * invstd * m2), for channel group cg
__device__ __forceinline__ void rv_bwd_coeffs(const float* __restrict__ mean, const float* __restrict__ invstd,
                                              const float* __restrict__ scale, const float* __restrict__ m1,
                                              const float* __restrict__ m2, int cg, float (&a)[8], float (&bq)[8],
                                              float (&cq)[8]) {
  float mu[8], is[8], q1[8], q2[8];
  load8f(mean + cg * 8, mu);
  load8f(invstd + cg * 8, is);
  load8f(scale + cg * 8, a);
  load8f(m1 + cg * 8, q1);
  load8f(m2 + cg * 8, q2);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    bq[j] = a[j] * is[j] * q2[j];
    cq[j] = a[j] * (mu[j] * is[j] * q2[j] - q1[j]);
  }
}

}  // namespace b200
