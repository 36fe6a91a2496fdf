// Multi-head self-attention for short sequences (T <= 256 tokens, head_dim 64): the parameters shared by the forward kernel
// (attention_fwd2.cuh) and the backward kernels (attention_bwd.cuh, attn_delta_kernel below).
#pragma once
#include "common.cuh"

namespace b200 {

__device__ __forceinline__ float attn_ex2(float x) {  // MUFU.EX2; exp2f() adds a denormal-range fix-up per element
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct alignas(64) AttnFwdParams {
  CUtensorMap q_map;    // qkv as (3*H*64, T, B), box (64, 128, 1)
  CUtensorMap kv_map;   // same tensor, box (64, Tpad, 1): keys beyond T are zero-filled
  CUtensorMap o_map;    // out as (H*64, T, B), box (64, 128, 1)
  int B, H, T, Tpad, mblocks;   // Tpad = T rounded up to 64 (the key tile), mblocks = 128-query blocks
  float scale_log2e;    // scale * log2(e)
  float scale;
  float* lse;           // [B][H][T] natural-log LSE of the scaled scores
};

}  // namespace b200

namespace b200 {

// ------------------------------------------------------------------------------------------------------------------
// Backward: attention_bwd.cuh (attn_bwd_kernel); the row term delta_i = sum_d dO[i,d] O[i,d] it needs is
// produced by attn_delta_kernel below.

// delta[b][h][t] = sum_d dO[b,t,h,d] * O[b,t,h,d].  Eight lanes per (b,t,h) row (one 16-byte vector of dO and of O each, the
// row sum by three shuffles), four rows in flight per lane: every load instruction of a warp covers 512 contiguous bytes.
// (The one-thread-per-row version this replaces touched 32 different 128-byte lines per instruction: 2.9 TB/s.)
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* __restrict__ dO, const __nv_bfloat16* __restrict__ O,
                                                         float* __restrict__ delta, int B, int T, int H) {
  pdl_wait();
  const long long total = static_cast<long long>(B) * T * H;
  const int sub = threadIdx.x & 7;
  const long long rows_per_pass = static_cast<long long>(gridDim.x) * (blockDim.x >> 3);
  // (the loop bound is warp-uniform: the shuffles below run with the full mask)
  for (long long rw = blockIdx.x * static_cast<long long>(blockDim.x >> 3) + ((threadIdx.x >> 5) << 2); rw < total;
       rw += 4 * rows_per_pass) {
    const long long r0 = rw + ((threadIdx.x & 31) >> 3);
    uint4 a[4], o[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long row = r0 + u * rows_per_pass;
      if (row < total) {
        a[u] = __ldg(reinterpret_cast<const uint4*>(dO + row * 64) + sub);
        o[u] = __ldg(reinterpret_cast<const uint4*>(O + row * 64) + sub);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long row = r0 + u * rows_per_pass;
      float s = 0.f;
      if (row < total) {
        float x[8], y[8];
        unpack8(a[u], x);
        unpack8(o[u], y);
#pragma unroll
        for (int j = 0; j < 8; ++j) s = fmaf(x[j], y[j], s);
      }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      if (sub == 0 && row < total) {
        const int h = static_cast<int>(row % H);
        const long long bt = row / H;
        const int t = static_cast<int>(bt % T);
        const long long b = bt / T;
        delta[(b * H + h) * T + t] = s;
      }
    }
  }
}

}  // namespace b200
