// Implicit-GEMM convolution for the 64 -> 64 channel layers (ResNet layer1 3x3 forward / dgrad, the space-to-depth stem) with
// the WEIGHTS RESIDENT in shared memory:
//
//   out[pixel, 0..63] = sum_tap A_tap[pixel + tap offset, 0..63] * W[0..63][tap*64 + c]^T       (num_taps <= 9)
//
// These layers have N = 64 and K = 64 per tap: per 128-pixel tile the generic kernel (conv_gemm.cuh) streams 16 KB of
// activations AND 8 KB of weights per tap through its ring, so a third of its L2 -> shared-memory traffic is the same
// 72 KB of weights fetched again for every tile (the layer is L2-bound: nine taps re-read the activation tile).  Here the
// taps' weight slices (<= 72 KB) are loaded once per CTA, the activation taps stream through a 5-deep ring of 16 KB slots,
// two consumer warpgroups multiply 64 rows each with wgmma (N = 64) and hand the accumulator to their warps through a shared-
// memory image; the warps of quadrant q take alternate tiles, convert, take the BatchNorm statistics from the staged slab
// and store by TMA (full tiles only: no predicates).  Same tensor maps, tap tables and statistics layout as
// conv_gemm_kernel<64>: the host code of b200_conv2d_fwd / b200_conv2d_dgrad / b200_stem_s2d_conv_fwd prepares ONE
// ConvGemmParams and dispatches here when the shape qualifies (abi_conv.cu tap64_ok).
#pragma once
#include "conv_gemm.cuh"

namespace b200 {

constexpr int kTap64Stages = 5;
constexpr int kTap64SmemBytes = 9 * 8192 + kTap64Stages * 16384 + 8 * 4096 + 128 * 64 * 4 + 512 + 1024;
static_assert(kTap64SmemBytes <= 227 * 1024, "shared memory of one H100 block");

template <bool kStats>
__global__ void __launch_bounds__(384, 1) conv_tap64_kernel(const __grid_constant__ ConvGemmParams p) {
  constexpr int STAGES = kTap64Stages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sB = smem;                         // [9 taps][64 rows x 128 B]
  uint8_t* sA = sB + 9 * 8192;                // ring of 128-pixel x 64-channel tap tiles
  uint8_t* sOut = sA + STAGES * 16384;        // [8 warps][32 rows x 128 B]
  uint8_t* sImg = sOut + 8 * 4096;            // fp32 accumulator image [128][64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sImg + 128 * 64 * 4);
  uint64_t* a_full = bars;                    // [STAGES]
  uint64_t* a_empty = bars + STAGES;          // [STAGES]
  uint64_t* b_full = bars + 2 * STAGES;

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = p.tiles1 * p.tiles2 * p.tiles3;
  const int taps = p.num_taps;

  if (warp_idx == 0 && lane == 0) {
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(&p.a_maps[i]);
    tma_prefetch_desc(&p.b_map);
    tma_prefetch_desc(&p.d_map);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], 2);   // one arrive per consumer warpgroup
    }
    mbar_init(b_full, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // everything above touched only this CTA's shared memory and the kernel parameters

  if (warp_idx < 4) {
    // ===================== TMA producer (warp 0): the weight slices once, then the activation taps =====================
    setmaxnreg_dec<40>();
    if (warp_idx == 0 && lane == 0) {
      mbar_expect_tx(b_full, static_cast<uint32_t>(taps) * 8192u);
      for (int t = 0; t < taps; ++t) tma_load_2d(sB + t * 8192, &p.b_map, b_full, p.tap_w[t] * p.k_per_tap, 0);
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < m_tiles; tile += gridDim.x) {
        const int t1 = tile % p.tiles1;
        const int t2 = (tile / p.tiles1) % p.tiles2;
        const int t3 = tile / (p.tiles1 * p.tiles2);
        const int c1 = t1 * p.box1, c2 = t2 * p.box2, c3 = t3 * p.box3;
        for (int t = 0; t < taps; ++t) {
          mbar_wait_backoff(&a_empty[stage], phase ^ 1);
          mbar_expect_tx(&a_full[stage], 16384);
          tma_load_4d(sA + stage * 16384, &p.a_maps[p.tap_map[t]], &a_full[stage], 0, c1 + p.tap_o1[t], c2 + p.tap_o2[t], c3);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== Two consumer warpgroups (rows 64 wg ..): wgmma, then the epilogue of alternate tiles ===========
    setmaxnreg_inc<232>();
    const int ew = warp_idx - 4;
    const int wg = ew >> 2;
    const int q = 2 * wg + (ew & 1);   // 32-row quadrant of the tile
    const int pair = (ew >> 1) & 1;    // the two warps of a quadrant take alternate tiles
    const int row = q * 32 + lane;
    const uint32_t img_s = smem_u32(sImg);
    const uint64_t desc_a0 = make_smem_desc_sw128(smem_u32(sA) + wg * 8192, p.desc_lbo, p.desc_sbo);
    const uint64_t desc_b0 = make_smem_desc_sw128(smem_u32(sB), p.desc_lbo, p.desc_sbo);
    const uint32_t os = smem_u32(sOut + ew * 4096);
    const uint32_t row_s = lane * 128;
    const uint32_t sw = (lane & 7) << 4;
    uint32_t stat_off[8];
#pragma unroll
    for (int m = 0; m < 8; ++m) stat_off[m] = m * 128 + ((((lane >> 2) ^ m) << 4) | ((lane & 3) << 2));
    uint64_t run_s = 0, run_q = 0;
    mbar_wait(b_full, 0);
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < m_tiles; tile += gridDim.x, ++it) {
      float acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int t = 0; t < taps; ++t) {
        mbar_wait(&a_full[stage], phase);
        wgmma_fence();
        const uint64_t da = desc_a0 + static_cast<uint64_t>(stage) * (16384 >> 4);
        const uint64_t db = desc_b0 + static_cast<uint64_t>(t) * (8192 >> 4);
#pragma unroll
        for (int k = 0; k < 4; ++k) Wgmma<64, 0, 0>::mma(acc, da + 2 * k, db + 2 * k, 1u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&a_empty[prev]);
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&a_empty[prev]);
      named_bar_sync(1 + wg, 128);   // the previous tile's image has been read
      acc_to_img<64>(acc, img_s, 64, 64 * wg, 0);
      named_bar_sync(1 + wg, 128);
      if ((it & 1) != pair) continue;
      const int t1 = tile % p.tiles1;
      const int t2 = (tile / p.tiles1) % p.tiles2;
      const int t3 = tile / (p.tiles1 * p.tiles2);
      const int s1 = t1 * p.box1 + p.qoff1[q], s2 = t2 * p.box2 + p.qoff2[q], s3 = t3 * p.box3 + p.qoff3[q];
      if (lane == 0) tma_store_wait_read<0>();   // this warp's previous store has finished reading the slab
      __syncwarp();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint32_t v[32];
        img_ld32(img_s, 64, row, h * 32, v);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          sts128(os + row_s + (((h * 4 + j) << 4) ^ sw),
                 pack_bf16x2(__uint_as_float(v[j * 8 + 0]), __uint_as_float(v[j * 8 + 1])),
                 pack_bf16x2(__uint_as_float(v[j * 8 + 2]), __uint_as_float(v[j * 8 + 3])),
                 pack_bf16x2(__uint_as_float(v[j * 8 + 4]), __uint_as_float(v[j * 8 + 5])),
                 pack_bf16x2(__uint_as_float(v[j * 8 + 6]), __uint_as_float(v[j * 8 + 7])));
      }
      __syncwarp();
      if constexpr (kStats) {
        // column sums / sums of squares over this warp's 32 rows, from the (bf16-rounded) slab: lane owns columns 2l, 2l + 1
        uint64_t a_s = 0, a_q = 0;
#pragma unroll
        for (int r = 0; r < 32; ++r) {
          const uint32_t w = lds32(os + (r >> 3) * 1024 + stat_off[r & 7]);
          const uint64_t x2 = f2_pack(bf16_lo(w), bf16_hi(w));
          a_s = f2_add(a_s, x2);
          a_q = f2_fma(x2, x2, a_q);
        }
        run_s = f2_add(run_s, a_s);
        run_q = f2_add(run_q, a_q);
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                         reinterpret_cast<uint64_t>(&p.d_map)),
                     "r"(os), "r"(0), "r"(s1), "r"(s2), "r"(s3)
                     : "memory");
        tma_store_commit();
      }
    }
    if constexpr (kStats) {
      // the statistics layout of conv_gemm_kernel<64>: two partial rows per (CTA, quadrant), one per warp of the quadrant
      const long long srow = (static_cast<long long>(blockIdx.x) * 4 + q) * 2 + pair;
      float s_lo, s_hi, q_lo, q_hi;
      f2_unpack(run_s, s_lo, s_hi);
      f2_unpack(run_q, q_lo, q_hi);
      float* sp = p.stats + srow * 2 * p.N + 2 * lane;
      *reinterpret_cast<float2*>(sp) = make_float2(s_lo, s_hi);
      *reinterpret_cast<float2*>(sp + p.N) = make_float2(q_lo, q_hi);
    }
    if (lane == 0) tma_store_wait_all<0>();
  }
}

}  // namespace b200
