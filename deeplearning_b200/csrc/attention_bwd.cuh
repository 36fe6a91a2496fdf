// ViT multi-head attention backward for sm_90a (T <= 256 tokens, head dim 64), the backward of attn_fwd2_kernel
// (attention_fwd2.cuh); replaces autograd through classification/vision_transformer/vit_model.py:97-108.
//
//   S  = Q K^T                    -> P = exp(scale*S - lse)            (recomputed from the saved log-sum-exp, never in HBM)
//   dP = dO V^T                   -> dS = scale * P * (dP - delta),  delta_i = sum_d dO[i,d] O[i,d] (attn_delta_kernel)
//   dV += P^T dO ,  dK += dS^T Q ,  dQ = dS K
//
// One CTA per (batch, head) walks the keys in blocks of 128:
//
//   for key block j (128 keys):      K_j, V_j resident (16 KB each), dK_j / dV_j accumulate in registers
//     for query block mb (128 rows): S = Q K_j^T (128 columns) -> P -> dP = dO V_j^T -> dS (in place over P)
//                                    dV_j += P^T dO, dK_j += dS^T Q, dQ_part = dS K_j
//
//   Warp 0 is the TMA producer; warpgroups 1 and 2 own query rows (S, dP, dQ) and keys (dK, dV) 64 wg .. 64 wg + 63 each,
//   issue their wgmma products themselves and hand S / dP / dQ to the soft-max threads (one row each; the two warps of a
//   32-row quadrant split the columns in half) through a 128 x 128 fp32 image in shared memory.
//   dQ of a query block is the sum over the key blocks: block 0 stores its part (bf16) through the normal dQ path, later
//   blocks TMA-load that part back (same CTA, so program order + wait_group make it visible), add their fp32 accumulator
//   and store the sum - deterministic, no atomics.
//
// P and dS live in shared memory as bf16 in the key-blocked 128B-swizzled layout, which serves both as a K-major A operand
// (dQ = dS K) and as an MN-major A operand (P^T dO, dS^T Q) without any transpose; K, V, Q, dO tiles are likewise consumed
// in place as K-major or MN-major B operands.
#pragma once
#include "attention.cuh"

namespace b200 {

struct alignas(64) AttnBwdParams {
  CUtensorMap qkv_map;   // qkv (3*H*64, T, B), box (64, 128, 1): Q, K and V tiles
  CUtensorMap do_map;    // dO (H*64, T, B), box (64, 128, 1)
  CUtensorMap dqkv_map;  // dqkv (3*H*64, T, B), box (64, 128, 1): stores, and loads of the partial dQ
  int B, H, T, nblk;     // nblk = ceil(T / 128) query blocks = key blocks
  float scale, scale_log2e;
  const float* lse;      // [B][H][T]
  const float* delta;    // [B][H][T]
};

constexpr int kAttnBwdSmemBytes = 4 * 16384 + 32768 + 128 * 128 * 4 + 256 + 1024;
constexpr int kAttnBwdThreads = 384;   // warpgroup 0: TMA producer (warp 0), warpgroups 1-2: rows 0-63 / 64-127
static_assert(kAttnBwdSmemBytes <= 227 * 1024, "shared memory of one H100 block");

__global__ void __launch_bounds__(kAttnBwdThreads, 1) attn_bwd_kernel(const __grid_constant__ AttnBwdParams p) {
  pdl_wait();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = smem + 16384;
  uint8_t* sQ = smem + 32768;    // also the landing buffer of the partial dQ (Q is dead once both dK products retired)
  uint8_t* sdO = smem + 49152;   // also the dQ staging buffer
  uint8_t* sP = smem + 65536;    // [2 key blocks of 64][128 q rows][64 keys] bf16: P, then dS in place; dK_j | dV_j staging
  uint8_t* sImg = smem + 98304;  // [128][128] fp32: S, dP, dQ_part
  uint64_t* bars = reinterpret_cast<uint64_t*>(sImg + 128 * 128 * 4);
  uint64_t* bar_kv = bars + 0;      // K_j / V_j landed
  uint64_t* bar_q = bars + 1;       // Q / dO of the current query block landed
  uint64_t* bar_free = bars + 2;    // dQ_part stored: Q / dO / P buffers reusable (8 warp arrivals)
  uint64_t* bar_kvfree = bars + 3;  // dK_j / dV_j stored (8 warp arrivals): K / V reusable
  uint64_t* bar_part = bars + 4;    // partial dQ landed in sQ

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x % p.H;
  const int b = blockIdx.x / p.H;
  const int HD = p.H * 64;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.qkv_map);
    tma_prefetch_desc(&p.do_map);
    tma_prefetch_desc(&p.dqkv_map);
    mbar_init(bar_kv, 1);
    mbar_init(bar_q, 1);
    mbar_init(bar_free, 8);
    mbar_init(bar_kvfree, 8);
    mbar_init(bar_part, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp_idx < 4) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int it = 0;
      for (int j = 0; j < p.nblk; ++j) {
        if (j > 0) mbar_wait_backoff(bar_kvfree, (j - 1) & 1);
        mbar_expect_tx(bar_kv, 2 * 16384);
        tma_load_3d(sK, &p.qkv_map, bar_kv, HD + h * 64, j * 128, b);
        tma_load_3d(sV, &p.qkv_map, bar_kv, 2 * HD + h * 64, j * 128, b);
        for (int mb = 0; mb < p.nblk; ++mb, ++it) {
          if (it > 0) mbar_wait_backoff(bar_free, (it - 1) & 1);   // previous dQ_part stored: Q / dO / P reusable
          mbar_expect_tx(bar_q, 2 * 16384);
          tma_load_3d(sQ, &p.qkv_map, bar_q, h * 64, mb * 128, b);
          tma_load_3d(sdO, &p.do_map, bar_q, h * 64, mb * 128, b);
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int ew = warp_idx - 4;
    const int wg = ew >> 2;
    const int quad = 2 * wg + (ew & 1);   // 32-row quadrant of the 128 rows (inside this warpgroup's 64)
    const int pair = (ew >> 1) & 1;       // the two warps of a quadrant split the columns of every row in half
    const int row = quad * 32 + lane;
    const int t128 = threadIdx.x & 127;
    const uint32_t img = smem_u32(sImg);
    const uint32_t k_addr = smem_u32(sK), v_addr = smem_u32(sV), q_addr = smem_u32(sQ), do_addr = smem_u32(sdO);
    const uint32_t p_addr = smem_u32(sP);
    const long long bh = static_cast<long long>(b) * p.H + h;
    constexpr uint32_t kAll = 1, kBarWg = 2;   // named barriers: all 256 consumer threads / this warpgroup
    int it = 0;
    uint32_t part_phase = 0;
    for (int j = 0; j < p.nblk; ++j) {
      float dv[32], dk[32];   // dV_j / dK_j rows (keys) 64 wg .. + 63
#pragma unroll
      for (int i = 0; i < 32; ++i) dv[i] = 0.f, dk[i] = 0.f;
      for (int mb = 0; mb < p.nblk; ++mb, ++it) {
        const uint32_t ph = it & 1;
        const int t = mb * 128 + row;
        const bool valid = t < p.T;
        const float lse2 = valid ? p.lse[bh * p.T + t] * 1.4426950408889634f : INFINITY;
        const float delta = valid ? p.delta[bh * p.T + t] : 0.f;
        if (mb == 0) mbar_wait(bar_kv, j & 1);
        mbar_wait(bar_q, ph);
        {
          // S = Q K_j^T : rows 64 wg .. of Q (K-major), K_j (K-major, N = 128 keys), K = 64
          float sacc[64];
#pragma unroll
          for (int i = 0; i < 64; ++i) sacc[i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            Wgmma<128, 0, 0>::mma(sacc, make_smem_desc_sw128(q_addr + wg * 8192 + k * 32, 16, 1024),
                                  make_smem_desc_sw128(k_addr + k * 32, 16, 1024), 1u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_reg_fence(sacc);
          named_bar_sync(kBarWg + wg, 128);   // the previous iteration's dQ_part has been read out of the image
          acc_to_img<128>(sacc, img, 128, 64 * wg, 0);
          named_bar_sync(kBarWg + wg, 128);
        }
        // ---- P = exp2(S*scale*log2e - lse*log2e), keys >= T masked
#pragma unroll 1
        for (int c = pair * 2; c < pair * 2 + 2; ++c) {
          uint32_t v[32];
          img_ld32(img, 128, row, c * 32, v);
          const int key0 = j * 128 + c * 32;            // first key of this chunk
          const bool crosses = key0 + 32 > p.T;         // warp-uniform
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            float e[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) e[i] = attn_ex2(fmaf(__uint_as_float(v[g * 8 + i]), p.scale_log2e, -lse2));
            if (crosses) {
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (key0 + g * 8 + i >= p.T) e[i] = 0.f;
            }
            const int col = c * 32 + g * 8;
            *reinterpret_cast<uint4*>(sP + (col >> 6) * 16384 + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4)) = pack8(e);
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(kAll, 256);   // all 128 rows of P written (dV reads every row); S read out of the image
        {
          // dP = dO V_j^T (rows 64 wg ..), into the image; dV_j += P^T dO (keys 64 wg ..: key atom wg of P, MN-major)
          float dp[64];
#pragma unroll
          for (int i = 0; i < 64; ++i) dp[i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            Wgmma<128, 0, 0>::mma(dp, make_smem_desc_sw128(do_addr + wg * 8192 + k * 32, 16, 1024),
                                  make_smem_desc_sw128(v_addr + k * 32, 16, 1024), 1u);
#pragma unroll
          for (int ks = 0; ks < 8; ++ks)   // 128 queries = 8 steps of 16
            Wgmma<64, 1, 1>::mma(dv, make_smem_desc_sw128(p_addr + wg * 16384 + ks * 2048, 16384, 1024),
                                 make_smem_desc_sw128(do_addr + ks * 2048, 8192, 1024), 1u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_reg_fence(dp);
          wgmma_reg_fence(dv);
          acc_to_img<128>(dp, img, 128, 64 * wg, 0);
        }
        named_bar_sync(kAll, 256);   // dP in the image; every dV product has read P
        // ---- dS = scale * P * (dP - delta), in place
#pragma unroll 1
        for (int c = pair * 2; c < pair * 2 + 2; ++c) {
          uint32_t v[32];
          img_ld32(img, 128, row, c * 32, v);
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const int col = c * 32 + g * 8;
            uint4* slot = reinterpret_cast<uint4*>(sP + (col >> 6) * 16384 + row * 128 + ((((col & 63) >> 3) ^ (row & 7)) << 4));
            float pv[8], e[8];
            unpack8(*slot, pv);
#pragma unroll
            for (int i = 0; i < 8; ++i) e[i] = p.scale * pv[i] * (__uint_as_float(v[g * 8 + i]) - delta);
            *slot = pack8(e);
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(kAll, 256);   // all rows of dS written (dK reads every row); dP read out of the image
        {
          // dQ_part = dS K_j (rows 64 wg ..: dS K-major, K_j MN-major), dK_j += dS^T Q (key atom wg of dS, MN-major)
          float dq[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) dq[i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 8; ++ks)   // 128 keys = 8 steps of 16
            Wgmma<64, 0, 1>::mma(dq, make_smem_desc_sw128(p_addr + (ks >> 2) * 16384 + wg * 8192 + (ks & 3) * 32, 16, 1024),
                                 make_smem_desc_sw128(k_addr + ks * 2048, 8192, 1024), 1u);
#pragma unroll
          for (int ks = 0; ks < 8; ++ks)
            Wgmma<64, 1, 1>::mma(dk, make_smem_desc_sw128(p_addr + wg * 16384 + ks * 2048, 16384, 1024),
                                 make_smem_desc_sw128(q_addr + ks * 2048, 8192, 1024), 1u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_reg_fence(dq);
          wgmma_reg_fence(dk);
          acc_to_img<64>(dq, img, 128, 64 * wg, 0);
        }
        named_bar_sync(kAll, 256);   // dQ_part in the image; every product has read Q / dS: sQ may take the partial dQ
        // ---- dQ_part (+ the parts of the previous key blocks) -> bf16 -> staging -> TMA store
        if (j > 0) {
          if (threadIdx.x == 128) {
            tma_store_wait_all<0>();   // this thread's earlier dQ stores are complete (not just read) before the reload
            mbar_expect_tx(bar_part, 16384);
            tma_load_3d(sQ, &p.dqkv_map, bar_part, h * 64, mb * 128, b);
          }
          mbar_wait(bar_part, part_phase);
          part_phase ^= 1;
        }
        uint8_t* stg = sdO;
        {
          const int c = pair;   // each warp of the pair drains one 32-column half of dQ_part
          uint32_t v[32];
          img_ld32(img, 128, row, c * 32, v);
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const int off = row * 128 + (((c * 4 + g) ^ (row & 7)) << 4);
            float e[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) e[i] = __uint_as_float(v[g * 8 + i]);
            if (j > 0) {
              float prev[8];
              unpack8(*reinterpret_cast<const uint4*>(sQ + off), prev);
#pragma unroll
              for (int i = 0; i < 8; ++i) e[i] += prev[i];
            }
            *reinterpret_cast<uint4*>(stg + off) = pack8(e);
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(kAll, 256);
        if (threadIdx.x == 128) {
          tma_store_3d(&p.dqkv_map, stg, h * 64, mb * 128, b);
          tma_store_commit();
          tma_store_wait_read<0>();
        }
        named_bar_sync(kAll, 256);
        if (lane == 0) mbar_arrive(bar_free);
      }
      // ---- dK_j, dV_j (rows = keys 64 wg ..) -> bf16 -> staging in the P region (free after the last products) -> TMA store
      {
        const int r0 = 64 * wg + 16 * (t128 >> 5) + (lane >> 2);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int R = r0 + 8 * hh;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int off = R * 128 + ((jj ^ (R & 7)) << 4) + (lane & 3) * 4;
            *reinterpret_cast<uint32_t*>(sP + off) = pack_bf16x2(dk[4 * jj + 2 * hh], dk[4 * jj + 2 * hh + 1]);
            *reinterpret_cast<uint32_t*>(sP + 16384 + off) = pack_bf16x2(dv[4 * jj + 2 * hh], dv[4 * jj + 2 * hh + 1]);
          }
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(kAll, 256);
      if (threadIdx.x == 128) {
        tma_store_3d(&p.dqkv_map, sP, HD + h * 64, j * 128, b);
        tma_store_3d(&p.dqkv_map, sP + 16384, 2 * HD + h * 64, j * 128, b);
        tma_store_commit();
        tma_store_wait_read<0>();
      }
      named_bar_sync(kAll, 256);
      if (lane == 0) mbar_arrive(bar_kvfree);
    }
    if (threadIdx.x == 128) tma_store_wait_all<0>();
  }
}

}  // namespace b200
