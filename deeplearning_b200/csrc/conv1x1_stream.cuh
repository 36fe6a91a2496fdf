// Streaming 1x1-convolution GEMM for the HBM-bound "narrow K -> wide N" layers of a ResNet bottleneck (sm_90a):
//
//   out[P][N] = epilogue( A[P][K] * W[N][K]^T ),   K = 64, 128 or 256 (KB = 1, 2, 4 k-blocks), N a multiple of 256, P a multiple of 128
//
//   kStreamBnRelu : out = relu(acc * scale[n] + shift[n] + residual)         conv3 -> bn3 -> + identity -> ReLU
//                   (classification/resnet/models/networks.py:116-124, BatchNorm folded through the conv: bn_algebra.cuh)
//   kStreamMask   : out = mask > 0 ? acc + residual : 0,  + per-CTA column sums  dgrad of conv1 + identity gradient, masked by
//                   the ReLU of the block input; the sums are sum(dz) of the previous block's BatchNorm backward
//   kStreamAffine : out = acc * scale[n] + shift[n]                            downsample conv -> BatchNorm (no residual, no ReLU)
//
// These layers move far more bytes of activations than they do arithmetic per byte, so everything that touches HBM is a bulk
// tensor copy:
//   * K <= 128: W (32 / 64 KB) is loaded ONCE per CTA and stays in shared memory (a CTA always works on the same 256-channel
//     block) and the A tiles (16 / 32 KB) stream through a 4- / 2-deep TMA ring;  K = 256 (layer3): W no longer fits beside
//     the slab rings, so (A, W) k-blocks of 16 + 32 KB stream through a 3-deep ring as in the generic kernel;
//   * two consumer warpgroups multiply 64 rows x 256 columns each with wgmma; the epilogue is elementwise, so it works on the
//     accumulator fragment in place: every consumer warp owns 16 rows of the tile, prefetches its own 16-row x 64-channel
//     residual / mask slabs by TMA into a private ring (no cross-warp synchronisation), two or three slabs ahead, and
//     stores its output slab by TMA;
//   * full tiles only: no row / column predicates anywhere.
#pragma once
#include "common.cuh"

namespace b200 {

enum : int { kStreamBnRelu = 0, kStreamMask = 1, kStreamAffine = 2 };

struct alignas(64) StreamParams {
  CUtensorMap a_map;     // A   [P][K] bf16, box {64, 128}
  CUtensorMap b_map;     // W   [N][K] bf16, box {64, 256}
  CUtensorMap out_map;   // out [P][N] bf16, box {64, 16}
  CUtensorMap res_map;   // residual [P][N] bf16, box {64, 16}
  CUtensorMap mask_map;  // kStreamMask: ReLU output whose zeros kill the gradient [P][N] bf16, box {64, 16}
  int m_tiles, n_tiles;  // P / 128, N / 256
  int N;
  const float* scale;    // kStreamBnRelu: [N]
  const float* shift;
  float* stats;          // kStreamMask: [gridDim.x / n_tiles * 4][2][N] (plane 0 = column sums of `out` as stored, plane 1 = 0):
                         // one row per 32-row quadrant of the tile, as conv_gemm_kernel writes them
};

template <int KB, int MODE>
struct StreamCfg {
  static constexpr bool STREAM_B = KB > 2;                                 // W streamed with A instead of resident
  static constexpr int A_STAGE = STREAM_B ? 16384 + 32768 : KB * 16384;    // STREAM_B: one k-block of A and of W
  static constexpr int STAGES = STREAM_B ? 3 : (KB == 1 ? 4 : 2);
  static constexpr int B_BYTES = STREAM_B ? 0 : KB * 32768;
  static constexpr int NBUF = (KB >= 2 && (MODE == kStreamMask || STREAM_B)) ? 2 : 3;   // slabs in flight per warp and source
  static constexpr int SLAB = 2048;                                        // 16 rows x 128 B
  static constexpr int RES_BYTES = MODE == kStreamAffine ? 0 : 8 * NBUF * SLAB;
  static constexpr int MASK_BYTES = MODE == kStreamMask ? RES_BYTES : 0;
  static constexpr int OUT_SLABS = (STREAM_B && MODE == kStreamMask) ? 1 : 2;   // output slabs per warp (shared memory is full)
  static constexpr int OUT_BYTES = 8 * OUT_SLABS * SLAB;
  static constexpr int COEF_BYTES = MODE != kStreamMask ? 2 * 256 * 4 : 0;
  static constexpr int BAR_BYTES = 512;
  static constexpr int SMEM_BYTES = B_BYTES + STAGES * A_STAGE + RES_BYTES + MASK_BYTES + OUT_BYTES + COEF_BYTES + BAR_BYTES + 1024;
  static constexpr int THREADS = 384;   // warpgroup 0: TMA producer (warp 0), warpgroups 1-2: consumers
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one H100 block");
};

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src_smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src_smem), "r"(c0), "r"(c1)
               : "memory");
}

template <int KB, int MODE>
__global__ void __launch_bounds__(384, 1) conv1x1_stream_kernel(const __grid_constant__ StreamParams p) {
  using Cfg = StreamCfg<KB, MODE>;
  constexpr int STAGES = Cfg::STAGES, NBUF = Cfg::NBUF;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sB = smem;
  uint8_t* sA = sB + Cfg::B_BYTES;
  uint8_t* sRes = sA + STAGES * Cfg::A_STAGE;
  uint8_t* sMask = sRes + Cfg::RES_BYTES;
  uint8_t* sOut = sMask + Cfg::MASK_BYTES;
  float* sCoef = reinterpret_cast<float*>(sOut + Cfg::OUT_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sCoef) + Cfg::COEF_BYTES);
  uint64_t* a_full = bars;                        // [STAGES]
  uint64_t* a_empty = bars + STAGES;              // [STAGES]
  uint64_t* b_full = bars + 2 * STAGES;           // [1]
  uint64_t* slab_full = bars + 2 * STAGES + 1;    // [8 warps][NBUF]

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tile = blockIdx.x % p.n_tiles;
  const int m_first = blockIdx.x / p.n_tiles, m_step = gridDim.x / p.n_tiles;
  const int my_tiles = m_first < p.m_tiles ? (p.m_tiles - m_first + m_step - 1) / m_step : 0;

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&p.a_map);
    tma_prefetch_desc(&p.b_map);
    tma_prefetch_desc(&p.out_map);
    if constexpr (MODE != kStreamAffine) tma_prefetch_desc(&p.res_map);
    if constexpr (MODE == kStreamMask) tma_prefetch_desc(&p.mask_map);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], 2);   // one arrive per consumer warpgroup
    }
    mbar_init(b_full, 1);
    for (int i = 0; i < 8 * NBUF; ++i) mbar_init(&slab_full[i], 1);
    fence_mbar_init();
  }
  pdl_wait();   // everything above touched only this CTA's shared memory and the kernel parameters
  if constexpr (MODE != kStreamMask) {
    // this CTA's 256 scale / shift values (its channel block never changes)
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
      sCoef[i] = __ldg(p.scale + n_tile * 256 + i);
      sCoef[256 + i] = __ldg(p.shift + n_tile * 256 + i);
    }
  }
  __syncthreads();

  if (warp_idx < 4) {
    // ===================== TMA producer (warp 0): W once, then the A tiles =====================
    setmaxnreg_dec<40>();
    if (warp_idx == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      if constexpr (Cfg::STREAM_B) {
        for (int t = 0; t < my_tiles; ++t) {
          const int m_tile = m_first + t * m_step;
          for (int kb = 0; kb < KB; ++kb) {
            mbar_wait_backoff(&a_empty[stage], phase ^ 1);
            mbar_expect_tx(&a_full[stage], Cfg::A_STAGE);
            tma_load_2d(sA + stage * Cfg::A_STAGE, &p.a_map, &a_full[stage], kb * 64, m_tile * 128);
            tma_load_2d(sA + stage * Cfg::A_STAGE + 16384, &p.b_map, &a_full[stage], kb * 64, n_tile * 256);
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      } else {
        mbar_expect_tx(b_full, Cfg::B_BYTES);
        for (int kb = 0; kb < KB; ++kb) tma_load_2d(sB + kb * 32768, &p.b_map, b_full, kb * 64, n_tile * 256);
        for (int t = 0; t < my_tiles; ++t) {
          const int m_tile = m_first + t * m_step;
          mbar_wait_backoff(&a_empty[stage], phase ^ 1);
          mbar_expect_tx(&a_full[stage], Cfg::A_STAGE);
          for (int kb = 0; kb < KB; ++kb)
            tma_load_2d(sA + stage * Cfg::A_STAGE + kb * 16384, &p.a_map, &a_full[stage], kb * 64, m_tile * 128);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup wg multiplies rows 64 wg .. + 63, warp ew drains 16 of them ===============
    setmaxnreg_inc<232>();
    const int ew = warp_idx - 4;       // 0..7: rows 16 ew .. 16 ew + 15 of the tile
    const int wg = ew >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    const uint64_t desc_b0 = make_smem_desc_sw128(smem_u32(sB), 16, 1024);
    const uint64_t desc_a0 = make_smem_desc_sw128(smem_u32(sA) + wg * 8192, 16, 1024);
    const uint32_t res_s = smem_u32(sRes + ew * NBUF * Cfg::SLAB);
    const uint32_t mask_s = smem_u32(sMask + ew * NBUF * Cfg::SLAB);
    const uint32_t out_s = smem_u32(sOut + ew * Cfg::OUT_SLABS * Cfg::SLAB);
    uint64_t* my_full = slab_full + ew * NBUF;
    // the fragment element pair (row lane / 4 + 8 h, columns 8 jj + 2 (lane % 4) + {0, 1}) of a 64-column unit sits at
    // byte frag_off + h * 1024 + ((jj ^ (lane / 4)) << 4) of a 16-row x 128 B swizzled slab
    const uint32_t frag_off = (lane >> 2) * 128 + (lane & 3) * 4;
    const uint32_t fsw = lane >> 2;
    const int col0 = n_tile * 256;
    const int total_units = my_tiles * 4;
    constexpr uint32_t kSlabTx = MODE == kStreamMask ? 2 * Cfg::SLAB : Cfg::SLAB;

    auto issue_unit = [&](int g) {   // lane 0: TMA loads of unit g (tile g / 4, 64-column unit g % 4) into ring slot g % NBUF
      const int slot = g % NBUF;
      const int row = (m_first + (g >> 2) * m_step) * 128 + ew * 16;
      const int col = col0 + (g & 3) * 64;
      mbar_expect_tx(&my_full[slot], kSlabTx);
      tma_load_2d(reinterpret_cast<void*>(sRes + (ew * NBUF + slot) * Cfg::SLAB), &p.res_map, &my_full[slot], col, row);
      if constexpr (MODE == kStreamMask)
        tma_load_2d(reinterpret_cast<void*>(sMask + (ew * NBUF + slot) * Cfg::SLAB), &p.mask_map, &my_full[slot], col, row);
    };
    if constexpr (MODE != kStreamAffine) {
      if (lane == 0)
        for (int g = 0; g < NBUF && g < total_units; ++g) issue_unit(g);
    }

    // column sums (kStreamMask): lane owns columns 2*lane, 2*lane + 1 of each of the four 64-column units
    uint32_t stat_off[8];
#pragma unroll
    for (int m = 0; m < 8; ++m) stat_off[m] = m * 128 + ((((lane >> 2) ^ m) << 4) | ((lane & 3) << 2));
    uint64_t run_s[4] = {0, 0, 0, 0};
    if constexpr (!Cfg::STREAM_B) mbar_wait(b_full, 0);

    int g = 0, stage = 0;
    uint32_t phase = 0;
    for (int t = 0; t < my_tiles; ++t) {
      const int row0 = (m_first + t * m_step) * 128 + ew * 16;
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      if constexpr (Cfg::STREAM_B) {
        int prev = -1;
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&a_full[stage], phase);
          wgmma_fence();
          const uint64_t da = desc_a0 + static_cast<uint64_t>((stage * Cfg::A_STAGE) >> 4);
          const uint64_t db = da - static_cast<uint64_t>((wg * 8192) >> 4) + static_cast<uint64_t>(16384 >> 4);
#pragma unroll
          for (int k = 0; k < 4; ++k) Wgmma<256, 0, 0>::mma(acc, da + 2 * k, db + 2 * k, 1u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && leader) mbar_arrive(&a_empty[prev]);
          prev = stage;
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
        wgmma_wait<0>();
        if (leader) mbar_arrive(&a_empty[prev]);
      } else {
        mbar_wait(&a_full[stage], phase);
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < KB; ++kb) {
          const uint64_t da = desc_a0 + static_cast<uint64_t>((stage * Cfg::A_STAGE + kb * 16384) >> 4);
          const uint64_t db = desc_b0 + static_cast<uint64_t>((kb * 32768) >> 4);
#pragma unroll
          for (int k = 0; k < 4; ++k) Wgmma<256, 0, 0>::mma(acc, da + 2 * k, db + 2 * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (leader) mbar_arrive(&a_empty[stage]);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_reg_fence(acc);
#pragma unroll
      for (int u = 0; u < 4; ++u, ++g) {
        const int slot = g % NBUF;
        const uint32_t rs = res_s + slot * Cfg::SLAB, ms = mask_s + slot * Cfg::SLAB;
        const uint32_t os = out_s + (Cfg::OUT_SLABS == 2 ? (g & 1) : 0) * Cfg::SLAB;
        // the TMA store that last used this output slab (two units ago; one with a single slab) has finished reading it
        if (lane == 0) {
          if constexpr (Cfg::OUT_SLABS == 2) tma_store_wait_read<1>(); else tma_store_wait_read<0>();
        }
        if constexpr (MODE != kStreamAffine) mbar_wait(&my_full[slot], (g / NBUF) & 1);
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const uint32_t off = frag_off + h * 1024 + ((jj ^ fsw) << 4);
            const int j = u * 8 + jj;
            float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
            const uint32_t rw = MODE != kStreamAffine ? lds32(rs + off) : 0u;
            const int c = u * 64 + jj * 8 + 2 * (lane & 3);
            if constexpr (MODE == kStreamBnRelu) {
              const float2 sc = *reinterpret_cast<const float2*>(sCoef + c);
              const float2 sh = *reinterpret_cast<const float2*>(sCoef + 256 + c);
              f0 = fmaxf(fmaf(f0, sc.x, sh.x) + bf16_lo(rw), 0.0f);
              f1 = fmaxf(fmaf(f1, sc.y, sh.y) + bf16_hi(rw), 0.0f);
            } else if constexpr (MODE == kStreamAffine) {
              const float2 sc = *reinterpret_cast<const float2*>(sCoef + c);
              const float2 sh = *reinterpret_cast<const float2*>(sCoef + 256 + c);
              f0 = fmaf(f0, sc.x, sh.x);
              f1 = fmaf(f1, sc.y, sh.y);
            } else {
              const uint32_t mw = lds32(ms + off);
              f0 = (mw & 0x7fffu) ? f0 + bf16_lo(rw) : 0.0f;
              f1 = (mw & 0x7fff0000u) ? f1 + bf16_hi(rw) : 0.0f;
            }
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(os + off), "r"(pack_bf16x2(f0, f1)) : "memory");
          }
        }
        __syncwarp();
        if constexpr (MODE == kStreamMask) {
          uint64_t a_s = 0;
#pragma unroll
          for (int r = 0; r < 16; ++r) {
            const uint32_t w = lds32(os + (r >> 3) * 1024 + stat_off[r & 7]);
            a_s = f2_add(a_s, f2_pack(bf16_lo(w), bf16_hi(w)));
          }
          run_s[u] = f2_add(run_s[u], a_s);
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          tma_store_2d(&p.out_map, os, col0 + u * 64, row0);
          tma_store_commit();
          if constexpr (MODE != kStreamAffine) {
            if (g + NBUF < total_units) issue_unit(g + NBUF);   // all lanes have consumed ring slot `slot` (__syncwarp above)
          }
        }
      }
    }
    if constexpr (MODE == kStreamMask) {
      // one statistics row per 32-row quadrant q = ew / 2: the two warps of a quadrant add up through the (now idle) residual
      // ring of the odd warp (every slab loaded into it has been consumed: the loads were waited for)
      float2* xch = reinterpret_cast<float2*>(sRes + (ew | 1) * NBUF * Cfg::SLAB);
      if (ew & 1) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float lo, hi;
          f2_unpack(run_s[u], lo, hi);
          xch[u * 32 + lane] = make_float2(lo, hi);
        }
      }
      named_bar_sync(1, 256);
      if (!(ew & 1)) {
        const int srow = (blockIdx.x / p.n_tiles) * 4 + (ew >> 1);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float lo, hi;
          f2_unpack(run_s[u], lo, hi);
          const float2 o = xch[u * 32 + lane];
          float* sp = p.stats + static_cast<long long>(srow) * 2 * p.N + col0 + u * 64 + 2 * lane;
          *reinterpret_cast<float2*>(sp) = make_float2(lo + o.x, hi + o.y);
          *reinterpret_cast<float2*>(sp + p.N) = make_float2(0.f, 0.f);
        }
      }
    }
    if (lane == 0) tma_store_wait_all<0>();
  }
}

}  // namespace b200
