// Multi-head self-attention forward for short sequences (T <= 256 tokens, head dim 64), persistent, with wgmma:
//
//   O[b, t, h, :] = softmax_j( scale * Q[b,t,h,:] . K[b,j,h,:] ) V[b,j,h,:]
//
// ONE CTA per SM walks (batch, head) items:
//   * a producer warp fetches Q (both 128-query blocks) and K of an item, and V, with TMA (rows beyond T are zero-filled);
//     Q / K of item i+1 land as soon as every S product of item i has retired, V once its P V products have;
//   * query block g is owned by warpgroup 1 + g, which works through its 128 rows as two 64-row halves:
//     S = Q K^T (m64 x NT keys, K = 64) in registers, the soft-max on the accumulator fragment (a row lives in the four
//     lanes of a quad: two shuffles per row reduction), P as bf16 into the 128B-swizzled K-major layout, O = P V (V used in
//     place as an MN-major operand), O / rowsum -> bf16 -> staging -> one TMA store per block;
//   * S / P never touch HBM; only the per-row log-sum-exp is kept for the backward pass.
//
// Shared memory: Q 2 x 16 KB, K 32 KB, V 32 KB, P 2 x 64 KB (the first 16 KB of a block's P double as its O staging slab).
//
// Replaces the eager sequence of vit_model.py:95-108 (classification/vision_transformer): qkv split, (q@k^T)*scale, softmax,
// attn@v, transpose/reshape, which materialises the [B,12,197,197] score tensor three times in HBM.
#pragma once
#include "attention.cuh"

namespace b200 {

constexpr int kAttn2SmemBytes = 2 * 16384 /*Q*/ + 32768 /*K*/ + 32768 /*V*/ + 2 * 65536 /*P*/ + 256 + 1024;
constexpr int kAttn2Threads = 384;   // warpgroup 0: TMA producer (warp 0), warpgroups 1-2: query blocks 0 / 1
static_assert(kAttn2SmemBytes <= 227 * 1024, "shared memory of one H100 block");

// NT = the key tile (p.Tpad: T rounded up to 64, <= 256)
template <int NT>
__global__ void __launch_bounds__(kAttn2Threads, 1) attn_fwd2_kernel(const __grid_constant__ AttnFwdParams p) {
  pdl_wait();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                       // [2][128][128B]
  uint8_t* sK = smem + 32768;               // [NT][128B]
  uint8_t* sV = smem + 65536;               // [NT][128B]
  uint8_t* sP = smem + 98304;               // [2 blocks][4 key blocks][128][128B]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 98304 + 131072);
  uint64_t* bar_qk_full = bars + 0;         // Q (all blocks) and K of the current item landed
  uint64_t* bar_qk_empty = bars + 1;        // every block's S products retired: Q / K may be overwritten (count = mblocks)
  uint64_t* bar_v_full = bars + 2;
  uint64_t* bar_v_empty = bars + 3;         // every block's P V products retired                           (count = mblocks)

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int items = p.B * p.H;
  const int HD = p.H * 64;
  const int mblocks = p.mblocks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.q_map);
    tma_prefetch_desc(&p.kv_map);
    tma_prefetch_desc(&p.o_map);
    mbar_init(bar_qk_full, 1);
    mbar_init(bar_qk_empty, mblocks);
    mbar_init(bar_v_full, 1);
    mbar_init(bar_v_empty, mblocks);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    // ---------------- TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int it = 0;
      for (int item = blockIdx.x; item < items; item += gridDim.x, ++it) {
        const int h = item % p.H, b = item / p.H;
        if (it > 0) mbar_wait_backoff(bar_qk_empty, (it - 1) & 1);
        mbar_expect_tx(bar_qk_full, mblocks * 16384 + NT * 128);
        for (int g = 0; g < mblocks; ++g) tma_load_3d(sQ + g * 16384, &p.q_map, bar_qk_full, h * 64, g * 128, b);
        tma_load_3d(sK, &p.kv_map, bar_qk_full, HD + h * 64, 0, b);
        if (it > 0) mbar_wait_backoff(bar_v_empty, (it - 1) & 1);
        mbar_expect_tx(bar_v_full, NT * 128);
        tma_load_3d(sV, &p.kv_map, bar_v_full, 2 * HD + h * 64, 0, b);
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int g = (warp_idx >> 2) - 1;
    if (g < mblocks) {
      // ---------------- query block g: S -> soft-max -> P -> P V -> O, in two halves of 64 rows
      const int t = threadIdx.x & 127;
      const bool leader = t == 0;
      const int r0 = 16 * (t >> 5) + (lane >> 2);   // fragment rows r0, r0 + 8 of a half
      const int cq = 2 * (lane & 3);                // fragment column offset inside an 8-column group
      uint8_t* sPg = sP + g * 65536;
      const uint32_t q_addr = smem_u32(sQ + g * 16384), k_addr = smem_u32(sK), v_addr = smem_u32(sV);
      const uint32_t p_addr = smem_u32(sPg);
      int it = 0;
      for (int item = blockIdx.x; item < items; item += gridDim.x, ++it) {
        const uint32_t ph = it & 1;
        const int h = item % p.H, b = item / p.H;
        // The first 16 KB of this block's P buffer were the staging slab of the previous item's O store: that store must
        // have finished READING shared memory before P is written again.
        if (it > 0) {
          if (leader) tma_store_wait_read<0>();
          named_bar_sync(2 + g, 128);
        }
        mbar_wait(bar_qk_full, ph);
#pragma unroll 1
        for (int hf = 0; hf < 2; ++hf) {
          // a half whose 64 query rows all lie beyond T only keeps the barrier protocol alive (TMA clips its O rows)
          const bool live = g * 128 + hf * 64 < p.T;
          float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
          if (live) {
            float sacc[NT / 2];
#pragma unroll
            for (int i = 0; i < NT / 2; ++i) sacc[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)
              Wgmma<NT, 0, 0>::mma(sacc, make_smem_desc_sw128(q_addr + hf * 8192 + k * 32, 16, 1024),
                                   make_smem_desc_sw128(k_addr + k * 32, 16, 1024), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_reg_fence(sacc);
            // row maxima over the valid keys, then P = exp2(scale * log2e * s - max) (bf16, unnormalised), keys >= T zero
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                if (8 * j + cq + (i & 1) < p.T) mx[i >> 1] = fmaxf(mx[i >> 1], sacc[4 * j + i]);
              }
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
              mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
            }
            const float mxs[2] = {mx[0] * p.scale_log2e, mx[1] * p.scale_log2e};
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
#pragma unroll
              for (int hh = 0; hh < 2; ++hh) {
                const int c = 8 * j + cq;
                const float e0 = c < p.T ? attn_ex2(fmaf(sacc[4 * j + 2 * hh], p.scale_log2e, -mxs[hh])) : 0.f;
                const float e1 = c + 1 < p.T ? attn_ex2(fmaf(sacc[4 * j + 2 * hh + 1], p.scale_log2e, -mxs[hh])) : 0.f;
                // row sum of the unrounded exponentials (differs from the sum of the bf16-rounded P the tensor core sees
                // by ~2^-9 / sqrt(T) relative, far below the bf16 output)
                sum[hh] += e0 + e1;
                const int R = hf * 64 + r0 + 8 * hh;
                *reinterpret_cast<uint32_t*>(sPg + (j >> 3) * 16384 + R * 128 + (((j & 7) ^ (R & 7)) << 4) + (lane & 3) * 4) =
                    pack_bf16x2(e0, e1);
              }
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              sum[hh] += __shfl_xor_sync(0xffffffffu, sum[hh], 1);
              sum[hh] += __shfl_xor_sync(0xffffffffu, sum[hh], 2);
            }
          }
          if (hf == 1 && leader) mbar_arrive(bar_qk_empty);   // both S products of this block have retired
          fence_proxy_async_smem();
          named_bar_sync(2 + g, 128);   // P of this half complete
          if (live) {
            // ---- O = P V : A = P (K-major, key blocks of 64), B = V (MN-major: rows = keys, 64 contiguous d), K = NT keys
            if (hf == 0) mbar_wait(bar_v_full, ph);
            float o[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) o[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < NT / 16; ++ks)
              Wgmma<64, 0, 1>::mma(o, make_smem_desc_sw128(p_addr + (ks >> 2) * 16384 + hf * 8192 + (ks & 3) * 32, 16, 1024),
                                   make_smem_desc_sw128(v_addr + ks * 2048, 8192, 1024), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_reg_fence(o);
            // O / sum -> bf16 -> staging rows of this half (their P rows in key block 0 have just been consumed)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const float inv = 1.0f / sum[hh];
              const int R = hf * 64 + r0 + 8 * hh;
#pragma unroll
              for (int j = 0; j < 8; ++j)
                *reinterpret_cast<uint32_t*>(sPg + R * 128 + ((j ^ (R & 7)) << 4) + (lane & 3) * 4) =
                    pack_bf16x2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
              const int tq = g * 128 + R;
              if ((lane & 3) == 0 && tq < p.T && p.lse != nullptr)
                p.lse[(static_cast<long long>(b) * p.H + h) * p.T + tq] = mx[hh] * p.scale + logf(sum[hh]);
            }
          }
        }
        if (leader) mbar_arrive(bar_v_empty);   // both P V products of this block have retired
        fence_proxy_async_smem();
        named_bar_sync(2 + g, 128);
        if (leader) {
          tma_store_3d(&p.o_map, sPg, h * 64, g * 128, b);
          tma_store_commit();
        }
      }
      if (leader) tma_store_wait_all<0>();
    }
  }
}

}  // namespace b200
