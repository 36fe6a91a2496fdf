// Weight-gradient GEMM for sm_90a:   dW[cout, tap, cin] = sum_pixels dY[pixel, cout] * X_tap[pixel (+tap offset), cin]
//
// The reduction runs over pixels, so both operands are "MN-major" for the tensor core: a TMA box of 64 pixels x 64 channels
// (64 rows of 128 B, 128B swizzle) is exactly one canonical MN-major SWIZZLE_128B atom column (K = pixel rows). The same
// NHWC activation tensors and the same tap/phase tensor maps as the forward kernel are used - no transposes, no im2col.
// The pixel range is split across CTAs (split-K); each CTA writes its fp32 partial tile to a workspace which
// wgrad_reduce_rows_kernel sums deterministically (no atomics) into the OIHW gradient.
//
// 64-channel inputs with several taps (ResNet layer1 3x3, the space-to-depth stem) run in MERGED-TAP mode: the 64-column
// atoms of one B tile belong to DIFFERENT taps (same pixels, shifted TMA coordinates), so one dY tile feeds an N = 192 / 256
// MMA instead of one N = 64 MMA per tap.
//
// GROUPED mode (kGrouped, 3x3 grouped convolutions whose groups never straddle a 64-channel block): dW of such a layer only
// needs the diagonal 64 x 64 blocks of dY^T X_tap. Each consumer warpgroup owns one 64-channel block and multiplies its dY
// atom with X atoms of the SAME channel block for three taps (BLOCK_NG / 2 = 192 columns per warpgroup); a work item is one
// (split, 128-channel pair, tap triple). The dense C x C product is never formed; wgrad_reduce_grouped_kernel picks the
// in-group columns.
//
// Two consumer warpgroups multiply with wgmma (64 output channels each: one dY atom) and store their fp32 fragments straight
// to the partial rows; warp 0 is the TMA producer.
//
// Replaces the cuDNN backward-filter / cuBLAS calls autograd issues for nn.Conv2d / nn.Linear in the reference
// (loss.backward(): classification/resnet/utils.py:43).
#pragma once
#include "common.cuh"
#include "conv_gemm.cuh"
#include "conv1x1_stream.cuh"   // lds128

namespace b200 {

struct alignas(64) WgradParams {
  CUtensorMap dy_map;     // 4-D (Cout, d1, d2, d3), box (64, b1, b2, b3), b1*b2*b3 = 64 pixels
  CUtensorMap x_maps[4];  // 4-D (Cin, ...), same box
  int num_taps;     // taps that are separate work items (1 in merged-tap mode)
  int merge_atoms;  // merged-tap mode: 64-channel atoms per tap (Cin / 64); 0 = one tap per work item
  int n_cols;       // valid columns of one partial row segment: Cin, or taps * Cin in merged-tap mode
  int Cout, Cin;
  int mg_tiles, ng_tiles;
  int tiles1, tiles2, tiles3;
  int box1, box2, box3;
  int splits, kb_per_split, kb_total;
  long long ld_partial;  // taps * Cin (row pitch of the partial matrix, in floats)
  int8_t tap_map[kMaxTaps];
  int8_t tap_o1[kMaxTaps];
  int8_t tap_o2[kMaxTaps];
  float* partial;  // [splits][Cout][taps*Cin]
  uint32_t desc_lbo, desc_sbo, desc_kstep;  // MN-major smem descriptor strides (bytes): 8192 / 1024 / 2048
  // kBias kernels: per-split column sums of dY (= the bias gradient of the layer), [splits][2][Cout] (plane 0 = sums,
  // plane 1 = 0: the layout b200_bn_bwd_finalize folds).  The dY tiles are already in shared memory for the tensor core:
  // the consumer warps add up their rows, so the bias gradient costs no pass over dY.
  float* bias_partial;
};

template <int BLOCK_NG>
struct WgradCfg {
  static constexpr int BLOCK_K = 64;                       // pixels per stage
  static constexpr int A_BYTES = 2 * 64 * 128;             // two 64-channel atoms of dY
  static constexpr int B_BYTES = (BLOCK_NG / 64) * 64 * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BLOCK_NG == 384 ? 3 : (BLOCK_NG == 256 ? 4 : (BLOCK_NG == 192 ? 5 : (BLOCK_NG == 128 ? 6 : 8)));
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one H100 block");
};
constexpr int kWgradThreads = 384;   // warpgroup 0: TMA producer (warp 0), warpgroups 1-2: consumers

template <int BLOCK_NG, bool kBias = false, bool kGrouped = false>
__global__ void __launch_bounds__(kWgradThreads, 1) wgrad_gemm_kernel(const __grid_constant__ WgradParams p) {
  static_assert(!kGrouped || (BLOCK_NG == 384 && !kBias), "grouped mode: two warpgroups x three 64-column taps");
  using Cfg = WgradCfg<BLOCK_NG>;
  constexpr int NW = kGrouped ? BLOCK_NG / 2 : BLOCK_NG;   // columns of one warpgroup's MMA
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  __shared__ float bias_red[2][16][64];      // kBias: per-row-group column sums of the two dY atoms

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // work item = (split, mg, ng, tap); tap fastest so CTAs sharing the same pixels run together (L2 reuse)
  const int items_per_split = p.mg_tiles * p.ng_tiles * p.num_taps;
  const int num_items = items_per_split * p.splits;

  if (warp_idx == 0 && lane == 0) {
    tma_prefetch_desc(&p.dy_map);
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(&p.x_maps[i]);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kBias ? 8 : 2);   // one arrive per consumer warpgroup (kBias: per consumer warp)
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // everything above touched only this CTA's shared memory and the kernel parameters

  if (warp_idx < 4) {
    setmaxnreg_dec<40>();
    if (warp_idx == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int split = item / items_per_split;
        int r = item - split * items_per_split;
        const int tap = r % p.num_taps;
        r /= p.num_taps;
        const int ng = r % p.ng_tiles;
        const int mg = r / p.ng_tiles;
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
        // per 64-column atom of the B tile: tensor map, channel offset and tap shift
        const CUtensorMap* xm[BLOCK_NG / 64];
        int ch0[BLOCK_NG / 64], o1[BLOCK_NG / 64], o2[BLOCK_NG / 64];
#pragma unroll
        for (int j = 0; j < BLOCK_NG / 64; ++j) {
          int tp = tap, ca = ng * (BLOCK_NG / 64) + j;
          if constexpr (kGrouped) {
            // atom j: tap 3 * tap + j % 3 of channel block 2 mg + j / 3 (the dY atom of consumer warpgroup j / 3)
            tp = tap * 3 + j % 3;
            ca = mg * 2 + j / 3;
          } else if (p.merge_atoms) {
            tp = ca / p.merge_atoms;
            ca -= tp * p.merge_atoms;
          }
          xm[j] = &p.x_maps[p.tap_map[tp]];
          ch0[j] = ca * 64;
          o1[j] = p.tap_o1[tp], o2[j] = p.tap_o2[tp];
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          const int t1 = kb % p.tiles1;
          const int t2 = (kb / p.tiles1) % p.tiles2;
          const int t3 = kb / (p.tiles1 * p.tiles2);
          const int c1 = t1 * p.box1, c2 = t2 * p.box2, c3 = t3 * p.box3;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* a_dst = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* b_dst = a_dst + Cfg::A_BYTES;
          mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          tma_load_4d(a_dst, &p.dy_map, &full_bar[stage], mg * 128, c1, c2, c3);
          tma_load_4d(a_dst + 8192, &p.dy_map, &full_bar[stage], mg * 128 + 64, c1, c2, c3);
#pragma unroll
          for (int j = 0; j < BLOCK_NG / 64; ++j)
            tma_load_4d(b_dst + j * 8192, xm[j], &full_bar[stage], ch0[j], c1 + o1[j], c2 + o2[j], c3);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== consumer warpgroups: rows (output channels) mg * 128 + 64 wg .. + 63 =====================
    setmaxnreg_inc<232>();
    const int wg = (warp_idx >> 2) - 1;
    const bool leader = (threadIdx.x & 127) == 0;
    // A = dY atom wg (64 output channels, MN-major), B = BLOCK_NG / 64 atoms of X (MN-major): 16 pixel rows per K step
    const uint64_t desc_a0 = make_smem_desc_sw128(smem_u32(smem) + wg * 8192, p.desc_lbo, p.desc_sbo);
    const uint64_t desc_b0 =
        make_smem_desc_sw128(smem_u32(smem) + Cfg::A_BYTES + (kGrouped ? wg * NW * 128 : 0), p.desc_lbo, p.desc_sbo);
    const uint64_t kstep = p.desc_kstep >> 4;
    const int t = threadIdx.x & 127;
    const int frow = 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2);   // fragment row of d[4j], d[4j+1]; d[4j+2..3]: + 8
    const int fcol = 2 * (t & 3);
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      const int split = item / items_per_split;
      int r = item - split * items_per_split;
      const int tap = r % p.num_taps;
      r /= p.num_taps;
      const int ng = r % p.ng_tiles;
      const int mg = r / p.ng_tiles;
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
      // kBias: the (ng == 0, tap == 0) item of every (split, mg) pair also sums the columns of its dY tiles (the layer's bias
      // gradient) while they are in shared memory for the tensor core: thread t of a warpgroup adds up 4 rows of ONE 16-byte
      // chunk (8 channels) of its atom, chunk cc = t % 8 (XOR-swizzled by row & 7), rows (t / 8) * 4 .. + 4.
      const bool summed = kBias && ng == 0 && tap == 0;
      const int cc = t & 7, rg = t >> 3;
      float bsum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      float acc[NW / 2];
#pragma unroll
      for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        const uint64_t soff = static_cast<uint64_t>(stage) * (Cfg::STAGE_BYTES >> 4);
        const uint64_t da = desc_a0 + soff, db = desc_b0 + soff;
#pragma unroll
        for (int k = 0; k < 4; ++k) Wgmma<NW, 1, 1>::mma(acc, da + k * kstep, db + k * kstep, 1u);
        wgmma_commit();
        if (summed) {
          const uint32_t base = smem_u32(smem + stage * Cfg::STAGE_BYTES) + wg * 8192;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int r = rg * 4 + i;
            float f[8];
            unpack8(lds128(base + r * 128 + ((static_cast<uint32_t>(cc) ^ static_cast<uint32_t>(r & 7)) << 4)), f);
#pragma unroll
            for (int j = 0; j < 8; ++j) bsum[j] += f[j];
          }
        }
        wgmma_wait<1>();   // the k-block before this one has been read: release its slot
        if constexpr (kBias) {
          __syncwarp();
          if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        } else {
          if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      // (the host guarantees every split owns at least one pixel block)
      if constexpr (kBias) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      } else {
        if (leader) mbar_arrive(&empty_bar[prev]);
      }
      if (summed) {
        // fold the 16 row groups (fixed order: deterministic) and write this split's partial sums
        named_bar_sync(1 + wg, 128);   // the previous item's readers are done with bias_red
#pragma unroll
        for (int j = 0; j < 8; ++j) bias_red[wg][rg][cc * 8 + j] = bsum[j];
        named_bar_sync(1 + wg, 128);
        if (t < 64) {
          float tot = 0.f;
#pragma unroll
          for (int g2 = 0; g2 < 16; ++g2) tot += bias_red[wg][g2][t];
          const int cout = mg * 128 + wg * 64 + t;
          if (cout < p.Cout) {
            p.bias_partial[(static_cast<long long>(split) * 2) * p.Cout + cout] = tot;
            p.bias_partial[(static_cast<long long>(split) * 2 + 1) * p.Cout + cout] = 0.f;
          }
        }
      }
      const int ncol = p.n_cols - ng * BLOCK_NG;   // valid columns of this tile (a multiple of 8)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int cout = mg * 128 + frow + 8 * h;
        if (cout < p.Cout) {
          float* out_row = p.partial + (static_cast<long long>(split) * p.Cout + cout) * p.ld_partial +
                           static_cast<long long>(tap) * p.Cin + ng * BLOCK_NG;
#pragma unroll
          for (int j = 0; j < NW / 8; ++j)
            if (8 * j + fcol < ncol)
              *reinterpret_cast<float2*>(out_row + 8 * j + fcol) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

// grad[cout][cin][tap] (OIHW, fp32) (+)= sum_s partial[s][cout][tap*Cin + cin]
// Row-block reduction: one block owns `chunk` input channels of one output channel for ALL taps, i.e. a contiguous run of
// chunk * taps gradient elements. The split range is folded by `SL` thread slices with float4 loads (coalesced along cin in
// the partial layout, two independent loads in flight per thread), staged in shared memory as [slice][tap][cin] and written
// out tap-innermost, so that both the partial reads and the OIHW gradient writes are fully coalesced. Fixed summation order.
__global__ void __launch_bounds__(256) wgrad_reduce_rows_kernel(const float* __restrict__ partial, float* __restrict__ grad,
                                                                int splits, int Cout, int Cin, int taps, int chunk, int SL,
                                                                int accumulate, const float* __restrict__ bias_partial,
                                                                float* __restrict__ bias_out) {
  pdl_wait();
  extern __shared__ float4 rows_sm4[];
  const int cout = blockIdx.x;
  // the layer's bias gradient: the per-split column sums of dY the kBias wgrad kernel left in bias_partial[splits][2][Cout],
  // folded in split order by the first block of each output channel (it used to be a launch of its own per layer)
  if (bias_out != nullptr && blockIdx.y == 0 && threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += bias_partial[static_cast<long long>(k) * 2 * Cout + cout];
    bias_out[cout] = s;
  }
  const int c0 = blockIdx.y * chunk;
  const int cw = min(chunk, Cin - c0);
  const int vpt = cw >> 2;          // float4 vectors per tap
  const int nvec = taps * vpt;
  const long long slice4 = static_cast<long long>(Cout) * taps * Cin / 4;
  const float4* row4 = reinterpret_cast<const float4*>(partial + static_cast<long long>(cout) * taps * Cin + c0);
  const int cin4 = Cin >> 2;
  for (int w = threadIdx.x; w < nvec * SL; w += blockDim.x) {
    const int sl = w / nvec;
    const int v = w - sl * nvec;
    const int tap = v / vpt;
    const int cv = v - tap * vpt;
    const float4* src = row4 + tap * cin4 + cv;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    int k = sl;
    for (; k + SL < splits; k += 2 * SL) {
      const float4 x = __ldcs(src + k * slice4);
      const float4 y = __ldcs(src + (k + SL) * slice4);
      a.x += x.x, a.y += x.y, a.z += x.z, a.w += x.w;
      b.x += y.x, b.y += y.y, b.z += y.z, b.w += y.w;
    }
    if (k < splits) {
      const float4 x = __ldcs(src + k * slice4);
      a.x += x.x, a.y += x.y, a.z += x.z, a.w += x.w;
    }
    rows_sm4[w] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
  __syncthreads();
  const float* sm = reinterpret_cast<const float*>(rows_sm4);
  float* out = grad + (static_cast<long long>(cout) * Cin + c0) * taps;
  for (int e = threadIdx.x; e < cw * taps; e += blockDim.x) {
    const int cin = e / taps;
    const int tap = e - cin * taps;
    float s = 0.f;
    for (int sl = 0; sl < SL; ++sl) s += sm[(sl * nvec) * 4 + tap * cw + cin];
    out[e] = accumulate ? out[e] + s : s;
  }
}

// Same reduction, one thread per element walking the splits: fallback for shapes the row kernel does not take.
__global__ void wgrad_reduce_flat_kernel(const float* __restrict__ partial, float* __restrict__ grad, int splits, int Cout,
                                    int Cin, int taps, int accumulate, const float* __restrict__ bias_partial,
                                    float* __restrict__ bias_out) {
  pdl_wait();
  const long long total = static_cast<long long>(Cout) * Cin * taps;
  const long long slice = total;
  if (bias_out != nullptr) {
    for (int cout = blockIdx.x * blockDim.x + threadIdx.x; cout < Cout; cout += gridDim.x * blockDim.x) {
      float s = 0.f;
      for (int k = 0; k < splits; ++k) s += bias_partial[static_cast<long long>(k) * 2 * Cout + cout];
      bias_out[cout] = s;
    }
  }
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // i indexes the partial layout (coalesced reads): [cout][tap][cin]
    const int cin = static_cast<int>(i % Cin);
    const long long t = i / Cin;
    const int tap = static_cast<int>(t % taps);
    const int cout = static_cast<int>(t / taps);
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += partial[k * slice + i];
    const long long o = (static_cast<long long>(cout) * Cin + cin) * taps + tap;
    grad[o] = accumulate ? grad[o] + s : s;
  }
}

// Grouped mode: grad[co][ci][tap] (OIHW [C][Cg][taps]) (+)= sum_s partial[s][co][tap * 64 + (co % 64) / Cg * Cg + ci], the
// in-group columns of the diagonal blocks the kGrouped wgrad kernel wrote. One thread per gradient element, splits summed
// in order (deterministic).
__global__ void wgrad_reduce_grouped_kernel(const float* __restrict__ partial, float* __restrict__ grad, int splits, int C,
                                            int Cg, int taps, int accumulate) {
  pdl_wait();
  const long long total = static_cast<long long>(C) * Cg * taps;
  const long long slice = static_cast<long long>(C) * taps * 64;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int tap = static_cast<int>(i % taps);
    const int ci = static_cast<int>((i / taps) % Cg);
    const int co = static_cast<int>(i / (static_cast<long long>(taps) * Cg));
    const float* src = partial + static_cast<long long>(co) * taps * 64 + tap * 64 + (co & 63) / Cg * Cg + ci;
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += src[k * slice];
    grad[i] = accumulate ? grad[i] + s : s;
  }
}


}  // namespace b200
