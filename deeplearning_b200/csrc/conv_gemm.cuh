// Implicit-GEMM convolution / linear forward kernel for sm_90a.
//
//   D[pixel, n] = sum_{tap, c} A_tap[pixel (+tap offset), c] * Wt[n, tap*Cin + c]        (bf16 in, fp32 accumulate)
//
// * A (activations, NHWC bf16) is fetched by TMA as 4-D boxes (64 channels x b1 x b2 x b3 pixels = 128 rows of 128 B,
//   128B-swizzled) straight into the layout wgmma consumes (K-major). A filter tap is just a coordinate offset;
//   out-of-image pixels are zero-filled by the TMA unit, which is the convolution's zero padding. Stride-2 convolutions
//   pass up to four "phase" views (even/odd rows x cols) of the input as separate tensor maps.
// * B (weights, [Cout][taps*Cin] bf16) is a 2-D TMA box of BLOCK_N rows x 64 k.
// * Two MMA warpgroups each multiply 64 rows of the 128-row tile with wgmma (m64 x BLOCK_N x k16) into registers; the
//   TMA producer (warpgroup 0) keeps a ring of k-block stages full. The kernel is persistent: grid = min(tiles, #SM).
// * Epilogue: the MMA warpgroups store their accumulator into a shared-memory image (mbarrier img_full) and go straight on
//   to the next tile's main loop; a dedicated epilogue warpgroup drains the image one row per thread (mbarrier img_empty
//   hands it back): (+bias, activation, +residual) -> bf16 -> swizzled smem staging -> TMA store, plus optional
//   per-channel sum / sum-of-squares partials (train-mode BatchNorm statistics). The tensor cores therefore only wait for
//   the epilogue when it takes longer than a main loop.
//
// Replaces the cuDNN/cuBLAS calls behind nn.Conv2d / nn.Linear on the reference's hot path
// (classification/resnet/models/networks.py:27-35,104-124; classification/vision_transformer/vit_model.py:95,109,127-133).
#pragma once
#include <cstdio>
#include "common.cuh"

namespace b200 {

constexpr int kMaxTaps = 16;

struct alignas(64) ConvGemmParams {
  CUtensorMap a_maps[4];
  CUtensorMap b_map;
  CUtensorMap d_map;    // output, box = one warp's slab: (64 bf16 | 32 fp32 channels) x 32 pixels (a quarter of the tile box)
  CUtensorMap aux_map;  // optional second output (pre-activation), same geometry as d_map (bf16)
  int num_taps;
  int k_per_tap;         // Cin (elements of K per tap)
  int k_blocks_per_tap;  // ceil(Cin / 64)
  int tiles1, tiles2, tiles3;
  int box1, box2, box3;
  int dim1, dim2, dim3;  // output pixel extents (row -> pixel mapping of the residual / aux / fp32 paths)
  int qoff1[4], qoff2[4], qoff3[4];  // pixel offset of quadrant q's 32-row slab (tile rows 32q ..) inside the tile box
  int n_tiles;
  int N;
  int8_t tap_map[kMaxTaps];  // which activation view (phase) the tap reads
  int8_t tap_o1[kMaxTaps];   // pixel offset along dim1 (w)
  int8_t tap_o2[kMaxTaps];   // pixel offset along dim2 (h)
  int8_t tap_w[kMaxTaps];    // which k_per_tap-wide slice of the weight matrix the tap multiplies
  float* stats;             // [stats_rows][2][N] per-CTA partial sums (see conv_stats_rows), or null; needs grid % n_tiles == 0
  const float* bias;        // [N] or null
  const float* colscale;    // [N] per-channel multiplier applied after bias/activation (layer scale), or null
  int act;                  // 0 none, 1 relu, 2 gelu(erf), 3 multiply by aux_in = GELU'(pre) saved by the forward (backward of 2)
  int out_f32;              // 1: d_map is fp32 (32-channel slabs)
  int res_f32;              // 1: residual tensor is fp32
  int has_aux_out;          // 1: second output through aux_map: the pre-activation (act 0/1) or GELU'(pre) (act 2)
  const void* residual;     // tensor added in the epilogue (pixel strides rs1..rs3, in elements) or null
  long long rs1, rs2, rs3;
  const __nv_bfloat16* aux_in;  // act == 3: GELU'(pre) tensor written by the forward GEMM (pixel strides as1..as3)
  long long as1, as2, as3;
  uint32_t desc_lbo, desc_sbo;  // K-major smem descriptor strides (bytes): 16 / 1024
  float* out_direct;        // direct fp32 output ([pixels][ld_out]) for tiny N (logits) or null
  long long ld_out;
  // --- stochastic depth (generic epilogue only): per-SAMPLE multiplier applied after bias / act / colscale, before the
  // residual add: sample = flat output pixel / rows_per_sample  (drop_path of the reference: convNext/models/networks.py:11-26)
  const float* rowscale;
  int rows_per_sample;
  // --- K made of several sources of different widths (dual-source dgrad of the BN-algebra path, [dz | y2] x [aW | M]^T):
  // with var_taps != 0 tap t spans tap_kb[t] k-blocks of activation view tap_map[t] (channel offset cb * 64) and multiplies
  // the weight columns starting at tap_k0[t]; kb_total = sum of tap_kb.
  int var_taps;
  int kb_total;
  int16_t tap_kb[kMaxTaps];
  int32_t tap_k0[kMaxTaps];
  // --- kEpiMask: tensor whose sign decides which outputs survive (ReLU mask of the block output), pixel strides ms1..ms3
  const __nv_bfloat16* mask_in;
  long long ms1, ms2, ms3;
  int affine;               // host-side: kEpiAffine (colscale = BN scale, bias = BN shift)
  // --- kEpiBnMask: the output is the gradient of relu(bn(x)); mask_in holds the RAW convolution output x of that BatchNorm,
  // alive = x * bn_scale + bn_shift > 0; the statistics rows carry sum(dz) and sum(dz * x) (what bn_bwd_reduce produces)
  const float* bn_scale;
  const float* bn_shift;
  // --- grouped convolution whose groups never straddle a 64-channel block (BLOCK_N = 64 only): output channel block n
  // reads only input channel block n, so the activation box of every k-block starts at channel n_tile * 64 (one k-block
  // per tap) and B is the block-diagonal [C][taps * 64] operand (b200_pack_weight mode 3 / 4)
  int chan_window;
};

template <int BLOCK_N>
struct ConvGemmCfg {
  static constexpr int BLOCK_M = 128;
  static constexpr int BLOCK_K = 64;
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGES = BLOCK_N == 128 ? 4 : 5;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EPI_WARPS = 4;
  static constexpr int SLAB_BYTES = 32 * 128;                       // one warp's 32 rows x 128 B
  static constexpr int STAGING_BYTES = EPI_WARPS * 2 * SLAB_BYTES;  // double-buffered per warp
  static constexpr int IMG_BYTES = BLOCK_M * BLOCK_N * 4;           // fp32 accumulator image
  // 64-column tiles have room for a second image: the MMA warpgroups can hand over the next tile while the epilogue
  // still drains this one (128-column tiles use that room for a fourth k-stage instead)
  static constexpr int IMGS = BLOCK_N == 128 ? 1 : 2;
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + IMGS * IMG_BYTES + BAR_BYTES + 1024;
  static constexpr int THREADS = 512;   // warpgroup 0: TMA producer, 1-2: MMA, 3: epilogue
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one H100 block");
  static_assert(2 * STAGES + 2 * IMGS <= BAR_BYTES / 8, "mbarriers");
};

// Exact-erf GELU (nn.GELU() of the reference: vit_model.py:121, swin_transformer.py:20, convNext/models/networks.py:84) with
// erf from Abramowitz & Stegun 7.1.26 (|abs error| <= 1.5e-7, far below the bf16 rounding of the stored activation):
// one reciprocal, one exp2 and six FMAs instead of erff()'s two-range polynomial (~3x fewer epilogue instructions).
//   t = 1 / (1 + p |z|),  erf(|z|) = 1 - (a1 t + a2 t^2 + a3 t^3 + a4 t^4 + a5 t^5) exp(-z^2),   z = x / sqrt(2)
// Returns erfc(|z|) / 2 = (1 - erf|z|) / 2 in `tail` and exp(-x^2 / 2) in `e` so that value and derivative share the work.
__device__ __forceinline__ void gelu_parts(float x, float& tail, float& e) {
  const float az = fabsf(x) * 0.70710678118654752f;
  float t;  // MUFU.RCP (1 ulp) - __frcp_rn would expand into a Newton iteration
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, az, 1.0f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * az * az));  // MUFU.EX2 (2 ulp)
  tail = 0.5f * poly * t * e;
}
__device__ __forceinline__ float gelu_erf(float x) {
  float tail, e;
  gelu_parts(x, tail, e);
  // Phi(x) = 1 - tail for x >= 0, tail for x < 0
  return x * (x >= 0.f ? 1.0f - tail : tail);
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  float tail, e;
  gelu_parts(x, tail, e);
  const float cdf = x >= 0.f ? 1.0f - tail : tail;
  return fmaf(x * 0.3989422804014327f, e, cdf);
}

// Two GELUs at once on fp32x2 values (common.cuh f2_*: per-lane IEEE fp32 operations, the same results as the scalar version).
// cdf = 0.5 + sign(x) * (0.5 - tail) replaces the compare / select of the scalar version.
__device__ __forceinline__ void gelu_parts2(float x0, float x1, uint64_t& cdf, uint64_t& e) {
  const uint64_t az = f2_pack(fabsf(x0) * 0.70710678118654752f, fabsf(x1) * 0.70710678118654752f);
  float d0, d1, t0, t1, g0, g1, e0, e1, h0, h1;
  f2_unpack(f2_fma(f2_bcast(0.3275911f), az, f2_bcast(1.0f)), d0, d1);
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(d0));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(d1));
  const uint64_t t = f2_pack(t0, t1);
  uint64_t poly = f2_fma(f2_bcast(1.061405429f), t, f2_bcast(-1.453152027f));
  poly = f2_fma(poly, t, f2_bcast(1.421413741f));
  poly = f2_fma(poly, t, f2_bcast(-0.284496736f));
  poly = f2_fma(poly, t, f2_bcast(0.254829592f));
  f2_unpack(f2_mul(f2_mul(az, az), f2_bcast(-1.4426950408889634f)), g0, g1);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(g0));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(g1));
  e = f2_pack(e0, e1);
  // 0.5 - tail = 0.5 - 0.5 * poly * t * e  (>= 0), then the sign of x
  f2_unpack(f2_fma(f2_mul(f2_mul(poly, t), e), f2_bcast(-0.5f), f2_bcast(0.5f)), h0, h1);
  cdf = f2_add(f2_pack(copysignf(h0, x0), copysignf(h1, x1)), f2_bcast(0.5f));
}
__device__ __forceinline__ void gelu_erf2(float& x0, float& x1) {
  uint64_t cdf, e;
  gelu_parts2(x0, x1, cdf, e);
  f2_unpack(f2_mul(f2_pack(x0, x1), cdf), x0, x1);
}
// x <- GELU(x), g <- GELU'(x) = Phi(x) + x phi(x) for two values: the derivative shares the cdf / exp work of the value (two
// more packed instructions), which is why the FORWARD GEMM of an MLP saves GELU'(pre) for the backward pass instead of the
// pre-activation itself - the dgrad epilogue of the following layer then only multiplies (it used to re-evaluate the whole
// erf polynomial per element, which made that epilogue instruction-issue bound).
__device__ __forceinline__ void gelu_erf_val_grad2(float& x0, float& x1, float& g0, float& g1) {
  uint64_t cdf, e;
  gelu_parts2(x0, x1, cdf, e);
  const uint64_t x = f2_pack(x0, x1);
  f2_unpack(f2_fma(f2_mul(x, f2_bcast(0.3989422804014327f)), e, cdf), g0, g1);
  f2_unpack(f2_mul(x, cdf), x0, x1);
}

// Optional phase timers (-DCONV_PROFILE): CTA 0 prints average cycles per tile of every wait / work phase of each role.
#ifdef CONV_PROFILE
#define CPROF_DECL(N) long long cp_t[N] = {}; long long cp_0 = clock64(), cp_1;
#define CPROF_TICK(i) { cp_1 = clock64(); cp_t[i] += cp_1 - cp_0; cp_0 = cp_1; }
#else
#define CPROF_DECL(N)
#define CPROF_TICK(i)
#endif

// One step of the warp's column-sum butterfly: px[i] += the partner lane's px[i + S] (or px[i] for the upper half), so that
// after steps 16 .. 1 px[0] of lane l holds column l summed over the 32 lanes. A template so that the loop is unrolled and
// px stays in registers (with a run-time step it was placed in local memory).
template <int S>
__device__ __forceinline__ void butterfly_step(float (&px)[32], int lane) {
  const bool up = (lane & S) != 0;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    const float send = up ? px[i] : px[i + S];
    const float keep = up ? px[i + S] : px[i];
    px[i] = keep + __shfl_xor_sync(0xffffffffu, send, S);
  }
}

// Epilogue specialisation: EPI < 0 keeps every epilogue option a run-time flag (generic fallback); EPI >= 0 is a bit set
// of compile-time options so that the hot layer types get a branch-free epilogue without the unused operand loads.
constexpr int kEpiGeneric = -1;
constexpr int kEpiBias = 1, kEpiColscale = 2, kEpiActShift = 2 /* 2 bits */, kEpiResBf16 = 16, kEpiResF32 = 32,
              kEpiAux = 64, kEpiOutF32 = 128, kEpiDirect = 256, kEpiStats = 512,
              kEpiRowscale = 1024 /* never specialised: selects the generic kernel */,
              // BatchNorm folded into a 1x1 convolution (specialised kernels only):
              //   kEpiAffine: f = f * colscale[n] + bias[n]  (scale / shift of the batch statistics) BEFORE the residual add,
              //               and the ReLU (act == 1) moves AFTER the residual add:  y = relu(bn(conv) + identity)
              //   kEpiMask:   after the residual add, f = mask_in > 0 ? f : 0      (dz = relu'(y) * (dgrad + identity gradient))
              //   kEpiBnMask: after everything else, f = (mask_in * bn_scale + bn_shift > 0) ? f : 0 and the statistics rows
              //               hold sum(f), sum(f * mask_in): the reduce half of the BatchNorm(+ReLU) backward of the PRODUCER of
              //               this gradient, which therefore needs no pass of its own (bn_bwd_reduce in elementwise.cuh)
              kEpiAffine = 2048, kEpiMask = 4096, kEpiBnMask = 8192;

template <int BLOCK_N, int EPI = kEpiGeneric>
__global__ void __launch_bounds__(512, 1) conv_gemm_kernel(const __grid_constant__ ConvGemmParams p) {
  static_assert(BLOCK_N == 64 || BLOCK_N == 128, "64- or 128-column tiles");
  using Cfg = ConvGemmCfg<BLOCK_N>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int IMGS = Cfg::IMGS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_base = smem;
  uint8_t* staging = smem + STAGES * Cfg::STAGE_BYTES;
  uint8_t* img = staging + Cfg::STAGING_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(img + IMGS * Cfg::IMG_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* img_full = bars + 2 * STAGES;           // image i holds a finished accumulator (8 MMA warps arrive)
  uint64_t* img_empty = bars + 2 * STAGES + IMGS;   // image i has been read by the epilogue (4 epilogue warps arrive)

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_tiles = p.tiles1 * p.tiles2 * p.tiles3;
  const int num_tiles = m_tiles * p.n_tiles;
  const int num_kb = p.var_taps ? p.kb_total : p.num_taps * p.k_blocks_per_tap;

  if (warp_idx == 0 && lane == 0) {
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(&p.a_maps[i]);
    tma_prefetch_desc(&p.b_map);
    tma_prefetch_desc(&p.d_map);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrive per MMA warpgroup
    }
    for (int i = 0; i < IMGS; ++i) {
      mbar_init(&img_full[i], 8);
      mbar_init(&img_empty[i], Cfg::EPI_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // everything above touched only this CTA's shared memory and the kernel parameters

  if (warp_idx < 4) {
    // ===================== TMA producer (warp 0 of warpgroup 0) =====================
    setmaxnreg_dec<40>();
    if (warp_idx == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      CPROF_DECL(2)
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n_tile = tile % p.n_tiles;
        const int m_tile = tile / p.n_tiles;
        const int t1 = m_tile % p.tiles1;
        const int t2 = (m_tile / p.tiles1) % p.tiles2;
        const int t3 = m_tile / (p.tiles1 * p.tiles2);
        const int c1 = t1 * p.box1, c2 = t2 * p.box2, c3 = t3 * p.box3;
        int tap = 0, cb = 0;   // running (tap, channel block) of k-block kb: no division in the single-thread issue loop
        int kb_in_tap = p.var_taps ? p.tap_kb[0] : p.k_blocks_per_tap;
        for (int kb = 0; kb < num_kb; ++kb, ++cb) {
          if (cb == kb_in_tap) {
            cb = 0;
            ++tap;
            if (p.var_taps) kb_in_tap = p.tap_kb[tap];
          }
          const int wk = p.var_taps ? p.tap_k0[tap] + cb * 64 : p.tap_w[tap] * p.k_per_tap + cb * 64;
          CPROF_TICK(1)
          mbar_wait_backoff(&empty_bar[stage], phase ^ 1);
          CPROF_TICK(0)
          uint8_t* a_dst = stage_base + stage * Cfg::STAGE_BYTES;
          uint8_t* b_dst = a_dst + Cfg::A_BYTES;
          mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          tma_load_4d(a_dst, &p.a_maps[p.tap_map[tap]], &full_bar[stage], p.chan_window ? n_tile * BLOCK_N : cb * 64, c1 + p.tap_o1[tap],
                      c2 + p.tap_o2[tap], c3);
          tma_load_2d(b_dst, &p.b_map, &full_bar[stage], wk, n_tile * BLOCK_N);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
#ifdef CONV_PROFILE
      if (blockIdx.x == 0) {
        const int nt = (num_tiles - 1) / gridDim.x + 1;
        printf("conv producer: wait_empty %lld issue %lld  (cycles/tile, %d tiles, %d k-blocks)\n", cp_t[0] / nt, cp_t[1] / nt, nt, num_kb);
      }
#endif
    }
  } else if (warp_idx < 12) {
    // ===================== Two MMA warpgroups: wgmma main loop, accumulator -> image =====================
    // Warpgroup wg owns tile rows 64 wg .. 64 wg + 63. It waits for the epilogue only right before it overwrites an image
    // the epilogue has not finished reading.
    setmaxnreg_dec<112>();
    const int wg = (warp_idx - 4) >> 2;
    const uint64_t desc_a0 = make_smem_desc_sw128(smem_u32(stage_base) + wg * 8192, p.desc_lbo, p.desc_sbo);
    const uint64_t desc_b0 = make_smem_desc_sw128(smem_u32(stage_base) + Cfg::A_BYTES, p.desc_lbo, p.desc_sbo);
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    CPROF_DECL(3)
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      // ---- main loop: 64 rows x BLOCK_N of this warpgroup, K in 64-wide k-blocks of four wgmma K steps each
      float acc[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;   // (also ends the live range of the previous tile's values)
      int prev = -1;
      CPROF_TICK(2)
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence();
        const uint64_t soff = static_cast<uint64_t>(stage) * (Cfg::STAGE_BYTES >> 4);
        const uint64_t da = desc_a0 + soff, db = desc_b0 + soff;
#pragma unroll
        for (int k = 0; k < 4; ++k) Wgmma<BLOCK_N, 0, 0>::mma(acc, da + 2 * k, db + 2 * k, 1u);   // +32 B per 16-element K step
        wgmma_commit();
        wgmma_wait<1>();   // the k-block before this one has been read: release its slot
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      CPROF_TICK(0)
      const int b = IMGS == 1 ? 0 : it % IMGS;
      mbar_wait(&img_empty[b], ((it / IMGS) & 1) ^ 1);   // (passes at once on the first use of each image)
      CPROF_TICK(1)
      acc_to_img<BLOCK_N>(acc, smem_u32(img + b * Cfg::IMG_BYTES), BLOCK_N, 64 * wg, 0);
      __syncwarp();   // the warp's image stores happen before lane 0's (release) arrive
      if (lane == 0) mbar_arrive(&img_full[b]);
    }
#ifdef CONV_PROFILE
    if (blockIdx.x == 0 && lane == 0 && (warp_idx & 3) == 0) {
      const int nt = (num_tiles - 1) / gridDim.x + 1;
      printf("conv mma wg %d: main loop %lld wait img_empty %lld acc->img %lld  (cycles/tile)\n", wg, cp_t[0] / nt, cp_t[1] / nt,
             cp_t[2] / nt);
    }
#endif
  } else {
    // ===================== Epilogue warpgroup: drains the image one row per thread =====================
    // Warp q owns the 32-row quadrant q of every tile, over all of its column units.
    setmaxnreg_inc<248>();
    const int q = warp_idx - 12;
    const int row = q * 32 + lane;
    const uint32_t stage_s = smem_u32(staging + q * 2 * Cfg::SLAB_BYTES);
    const uint32_t row_s = lane * 128;          // this thread's row inside a slab
    const uint32_t sw = (lane & 7) << 4;        // 128B-swizzle XOR term of that row
    // statistics read-back: lane owns columns 2*lane, 2*lane+1 -> 4-byte word `lane` of every row
    uint32_t stat_off[8];
#pragma unroll
    for (int m = 0; m < 8; ++m) stat_off[m] = m * 128 + ((((lane >> 2) ^ m) << 4) | ((lane & 3) << 2));
    // kernel parameters used in the inner loops, hoisted into registers
    constexpr bool G = EPI < 0;
    constexpr bool kAffine = !G && (EPI & kEpiAffine) != 0;   // BatchNorm scale / shift, ReLU after the residual add
    constexpr bool kBnMask = !G && (EPI & kEpiBnMask) != 0;   // ReLU mask recomputed from the raw BN input + sum(dz * x)
    constexpr bool kMask = !G && (EPI & (kEpiMask | kEpiBnMask)) != 0;   // a second tensor decides which outputs survive
    const int N = p.N;
    const float* const bias = (!kAffine && (G || (EPI & kEpiBias))) ? p.bias : nullptr;
    const float* const colscale = (!kAffine && (G || (EPI & kEpiColscale))) ? p.colscale : nullptr;
    const int act_bits = G ? p.act : ((EPI >> kEpiActShift) & 3);
    const int act = kAffine ? 0 : act_bits;                   // (kAffine: the activation is applied after the residual)
    const bool has_res = G ? (p.residual != nullptr) : ((EPI & (kEpiResBf16 | kEpiResF32)) != 0);
    const bool res_f32 = G ? (p.res_f32 != 0) : ((EPI & kEpiResF32) != 0);
    const bool has_aux = G ? (p.has_aux_out != 0) : ((EPI & kEpiAux) != 0);
    const bool out_f32 = G ? (p.out_f32 != 0) : ((EPI & kEpiOutF32) != 0);
    float* const out_direct = (G || (EPI & kEpiDirect)) ? p.out_direct : nullptr;
    float* const stats = (G || (EPI & (kEpiStats | kEpiBnMask))) ? p.stats : nullptr;
    const float* const rowscale = G ? p.rowscale : nullptr;
    const bool need_rowmap = has_res || act == 3 || kMask || out_direct != nullptr || rowscale != nullptr || p.dim1 % p.box1 != 0 ||
                             p.dim2 % p.box2 != 0 || p.dim3 % p.box3 != 0;
    const bool full_cols = (N % BLOCK_N) == 0;  // no partially valid 32-column group anywhere
    uint32_t store_counter = 0;
    // Work units: 64 bf16 (or 32 fp32) channels x the warp's 32 rows
    const int unit_cols = out_f32 ? 32 : 64;
    const int units = BLOCK_N / unit_cols;
    const int nsub = out_f32 ? 1 : 2;  // 32-column image loads per unit
    // Train-mode BN statistics: every epilogue warp keeps running column sums of the slabs it stored (the launch guarantees
    // grid % n_tiles == 0, so a CTA always sees the same channel block) and writes them out at the end of the kernel, in
    // one of two slots: the 64-column unit of a 128-column tile (both slots share a partial row), or for 64-column tiles
    // the parity of the CTA's tile count (two partial rows per quadrant, the layout conv_tap64_kernel shares).
    constexpr int SLOTS = 2;
    uint64_t run_s[SLOTS], run_q[SLOTS];
    float run_x[SLOTS][2];   // kBnMask: sum(dz * x) of column (slot k, half h, lane)
#pragma unroll
    for (int k = 0; k < SLOTS; ++k) run_s[k] = 0, run_q[k] = 0, run_x[k][0] = run_x[k][1] = 0.f;
    int it = 0;
    CPROF_DECL(2)
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int b = IMGS == 1 ? 0 : it % IMGS;
      const uint32_t img_s = smem_u32(img + b * Cfg::IMG_BYTES);
      const int n_tile = tile % p.n_tiles;
      const int m_tile = tile / p.n_tiles;
      const int t1 = m_tile % p.tiles1;
      const int t2 = (m_tile / p.tiles1) % p.tiles2;
      const int t3 = m_tile / (p.tiles1 * p.tiles2);
      const int c1 = t1 * p.box1, c2 = t2 * p.box2, c3 = t3 * p.box3;
      int p1 = 0, p2 = 0, p3 = 0;
      bool row_ok = true;
      if (need_rowmap) {
        const int i1 = row % p.box1;
        const int i2 = (row / p.box1) % p.box2;
        const int i3 = row / (p.box1 * p.box2);
        p1 = c1 + i1, p2 = c2 + i2, p3 = c3 + i3;
        row_ok = (p1 < p.dim1) && (p2 < p.dim2) && (p3 < p.dim3);
      }
      const int s1 = c1 + p.qoff1[q], s2 = c2 + p.qoff2[q], s3 = c3 + p.qoff3[q];

      // Global operands of the epilogue (residual / saved pre-activation) run ONE 32-column group ahead: the group's loads
      // are issued while the previous group is converted and stored, so every epilogue warp always has 64-128 B per lane in
      // flight towards HBM.
      uint4 nx_b[4];   // bf16 residual or aux_in: 32 x bf16
      float4 nx_f[8];  // fp32 residual: 32 x fp32
      uint4 nx_m[4];   // kMask: 32 x bf16 of the mask tensor
      auto issue_pre = [&](int u, int h) {
        const int ncp = n_tile * BLOCK_N + u * unit_cols + h * 32;
        if (n_tile * BLOCK_N + u * unit_cols >= N || !row_ok) return;
        if (has_res) {
          const long long off = p3 * p.rs3 + p2 * p.rs2 + p1 * p.rs1 + ncp;
          if (res_f32) {
            const float4* rp = reinterpret_cast<const float4*>(static_cast<const float*>(p.residual) + off);
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (full_cols || ncp + j * 4 < N) nx_f[j] = __ldg(rp + j);
          } else {
            const uint4* rp = reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(p.residual) + off);
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (full_cols || ncp + j * 8 < N) nx_b[j] = __ldg(rp + j);
          }
        }
        if (act == 3) {
          const uint4* ap = reinterpret_cast<const uint4*>(p.aux_in + p3 * p.as3 + p2 * p.as2 + p1 * p.as1 + ncp);
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (full_cols || ncp + j * 8 < N) nx_b[j] = __ldg(ap + j);
        }
        if constexpr (kMask) {
          const uint4* mp = reinterpret_cast<const uint4*>(p.mask_in + p3 * p.ms3 + p2 * p.ms2 + p1 * p.ms1 + ncp);
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (full_cols || ncp + j * 8 < N) nx_m[j] = __ldg(mp + j);
        }
      };
      if (has_res || act == 3 || kMask) issue_pre(0, 0);   // (they do not depend on the accumulator)
      CPROF_TICK(1)
      mbar_wait(&img_full[b], (it / IMGS) & 1);
      CPROF_TICK(0)

#pragma unroll 1
      for (int u = 0; u < units; ++u) {
        const int n0 = n_tile * BLOCK_N + u * unit_cols;
        const bool chunk_live = n0 < N;  // warp-uniform
        const uint32_t buf_s = stage_s + (store_counter & 1) * Cfg::SLAB_BYTES;
        const uint32_t aux_s = stage_s + ((store_counter + 1) & 1) * Cfg::SLAB_BYTES;
        if (chunk_live && out_direct == nullptr) {
          // the TMA store that last used this slab (two stores ago) must have finished reading it
          if (lane == 0) {
            if (has_aux) tma_store_wait_read<0>(); else tma_store_wait_read<1>();
          }
          __syncwarp();
        }
#pragma unroll 1
        for (int h = 0; h < nsub; ++h) {
          uint32_t v[32];
          img_ld32(img_s, BLOCK_N, row, u * unit_cols + h * 32, v);
          if (u == units - 1 && h == nsub - 1) {
            // the last image read of this tile: the MMA warpgroups may overwrite the image (release orders the loads)
            __syncwarp();
            if (lane == 0) mbar_arrive(&img_empty[b]);
          }
          uint4 pre_b[4];
          float4 pre_f[8];
          uint4 pre_m[4];
          if (has_res || act == 3 || kMask) {
#pragma unroll
            for (int j = 0; j < 4; ++j) pre_b[j] = nx_b[j];
#pragma unroll
            for (int j = 0; j < 8; ++j) pre_f[j] = nx_f[j];
            if constexpr (kMask) {
#pragma unroll
              for (int j = 0; j < 4; ++j) pre_m[j] = nx_m[j];
            }
            if (h + 1 < nsub)
              issue_pre(u, h + 1);
            else if (u + 1 < units)
              issue_pre(u + 1, 0);
          }
          if (!chunk_live) continue;
          const int nc = n0 + h * 32;  // first channel of this 32-column group
          float f[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]);
          if constexpr (kAffine) {
            // train / eval BatchNorm of the convolution output: f * scale[n] + shift[n]  (channel counts are multiples of 32)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 s4 = __ldg(reinterpret_cast<const float4*>(p.colscale + nc) + j);
              const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + nc) + j);
              f2_unpack(f2_fma(f2_pack(f[j * 4 + 0], f[j * 4 + 1]), f2_pack(s4.x, s4.y), f2_pack(b4.x, b4.y)), f[j * 4 + 0], f[j * 4 + 1]);
              f2_unpack(f2_fma(f2_pack(f[j * 4 + 2], f[j * 4 + 3]), f2_pack(s4.z, s4.w), f2_pack(b4.z, b4.w)), f[j * 4 + 2], f[j * 4 + 3]);
            }
          }
          if (bias != nullptr) {
            if (full_cols) {
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + nc) + j);
                f2_unpack(f2_add(f2_pack(f[j * 4 + 0], f[j * 4 + 1]), f2_pack(b4.x, b4.y)), f[j * 4 + 0], f[j * 4 + 1]);
                f2_unpack(f2_add(f2_pack(f[j * 4 + 2], f[j * 4 + 3]), f2_pack(b4.z, b4.w)), f[j * 4 + 2], f[j * 4 + 3]);
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j) f[j] += (nc + j < N) ? __ldg(bias + nc + j) : 0.0f;
            }
          }
          if (has_aux) {
            // second output (bf16) for the backward pass: the pre-activation, or - when the activation is GELU - its
            // derivative GELU'(pre), computed together with the value (what act == 3 of the next layer's dgrad multiplies by)
            const uint32_t z = row_ok ? 0xffffffffu : 0u;
            if (act == 2) {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float g[8];
#pragma unroll
                for (int i = 0; i < 8; i += 2) gelu_erf_val_grad2(f[j * 8 + i], f[j * 8 + i + 1], g[i], g[i + 1]);
                sts128(aux_s + row_s + ((((h * 4 + j) << 4)) ^ sw), pack_bf16x2(g[0], g[1]) & z, pack_bf16x2(g[2], g[3]) & z,
                       pack_bf16x2(g[4], g[5]) & z, pack_bf16x2(g[6], g[7]) & z);
              }
            } else {
#pragma unroll
              for (int j = 0; j < 4; ++j)
                sts128(aux_s + row_s + ((((h * 4 + j) << 4)) ^ sw), pack_bf16x2(f[j * 8 + 0], f[j * 8 + 1]) & z,
                       pack_bf16x2(f[j * 8 + 2], f[j * 8 + 3]) & z, pack_bf16x2(f[j * 8 + 4], f[j * 8 + 5]) & z,
                       pack_bf16x2(f[j * 8 + 6], f[j * 8 + 7]) & z);
            }
          }
          if (act == 1) {
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j], 0.0f);
          } else if (act == 2) {
            if (!has_aux) {   // (with a second output the value was computed together with the derivative above)
#pragma unroll
              for (int j = 0; j < 32; j += 2) gelu_erf2(f[j], f[j + 1]);
            }
          } else if (act == 3 && row_ok) {
            // backward of GELU: aux_in holds GELU'(pre) as saved by the forward GEMM
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (full_cols || nc + j * 8 < N) {
                float a[8];
                unpack8(pre_b[j], a);
#pragma unroll
                for (int i = 0; i < 8; i += 2)
                  f2_unpack(f2_mul(f2_pack(f[j * 8 + i], f[j * 8 + i + 1]), f2_pack(a[i], a[i + 1])), f[j * 8 + i],
                            f[j * 8 + i + 1]);
              }
            }
          }
          if (colscale != nullptr) {
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] *= (full_cols || nc + j < N) ? __ldg(colscale + nc + j) : 0.0f;
          }
          if (rowscale != nullptr && row_ok) {
            const long long pix = (static_cast<long long>(p3) * p.dim2 + p2) * p.dim1 + p1;
            const float rs = __ldg(rowscale + pix / p.rows_per_sample);
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] *= rs;
          }
          if (has_res && row_ok) {
            if (res_f32) {
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                if (full_cols || nc + j * 4 < N) {
                  const float4 r = pre_f[j];
                  f2_unpack(f2_add(f2_pack(f[j * 4 + 0], f[j * 4 + 1]), f2_pack(r.x, r.y)), f[j * 4 + 0], f[j * 4 + 1]);
                  f2_unpack(f2_add(f2_pack(f[j * 4 + 2], f[j * 4 + 3]), f2_pack(r.z, r.w)), f[j * 4 + 2], f[j * 4 + 3]);
                }
              }
            } else {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                if (full_cols || nc + j * 8 < N) {
                  float r[8];
                  unpack8(pre_b[j], r);
#pragma unroll
                  for (int i = 0; i < 8; i += 2)
                    f2_unpack(f2_add(f2_pack(f[j * 8 + i], f[j * 8 + i + 1]), f2_pack(r[i], r[i + 1])), f[j * 8 + i],
                              f[j * 8 + i + 1]);
                }
              }
            }
          }
          if constexpr (kAffine) {
            if (act_bits == 1) {
#pragma unroll
              for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j], 0.0f);
            }
          }
          if constexpr (kBnMask) {
            // BatchNorm(+ReLU) backward of the layer that produced this gradient's argument: alive iff x * scale + shift > 0
            // (exactly the forward's ReLU input), and the column sums of dz * x by a 5-step butterfly over the warp's 32 rows
            float px[32];
            if (row_ok) {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float x8[8];
                unpack8(pre_m[j], x8);
#pragma unroll
                for (int i = 0; i < 8; ++i) px[j * 8 + i] = x8[i];
              }
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float4 s4 = __ldg(reinterpret_cast<const float4*>(p.bn_scale + nc) + j);
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bn_shift + nc) + j);
                const float sc4[4] = {s4.x, s4.y, s4.z, s4.w}, sh4[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  // (rounded to the stored bf16 value first: both sums are sums over dz exactly as bn_bwd_apply will read it)
                  const float fm =
                      fmaf(px[j * 4 + i], sc4[i], sh4[i]) > 0.f ? __bfloat162float(__float2bfloat16_rn(f[j * 4 + i])) : 0.f;
                  f[j * 4 + i] = fm;
                  px[j * 4 + i] *= fm;
                }
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j) px[j] = 0.f;
            }
            butterfly_step<16>(px, lane);
            butterfly_step<8>(px, lane);
            butterfly_step<4>(px, lane);
            butterfly_step<2>(px, lane);
            butterfly_step<1>(px, lane);
            const int slot = units == 1 ? (it & 1) : u;
#pragma unroll
            for (int k = 0; k < SLOTS; ++k) {
              if (k == slot) {
                run_x[k][0] += h == 0 ? px[0] : 0.f;
                run_x[k][1] += h == 0 ? 0.f : px[0];
              }
            }
          } else if constexpr (kMask) {
            // the mask tensor is a ReLU output (>= 0): an element is alive iff its bf16 bits are non-zero
            if (row_ok) {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const uint32_t w[4] = {pre_m[j].x, pre_m[j].y, pre_m[j].z, pre_m[j].w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  if ((w[i] & 0x7fffu) == 0u) f[j * 8 + 2 * i] = 0.f;
                  if ((w[i] & 0x7fff0000u) == 0u) f[j * 8 + 2 * i + 1] = 0.f;
                }
              }
            }
          }
          if (out_direct != nullptr) {
            if (row_ok) {
              const long long pix = (static_cast<long long>(p3) * p.dim2 + p2) * p.dim1 + p1;
              float* op = out_direct + pix * p.ld_out + nc;
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (nc + j < N) op[j] = f[j];
            }
            continue;
          }
          if (!row_ok) {
            // rows of a partial pixel box: clipped by the TMA store, and must not pollute the BN statistics
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = 0.f;
          }
          if (out_f32) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
              sts128(buf_s + row_s + ((j << 4) ^ sw), __float_as_uint(f[j * 4 + 0]), __float_as_uint(f[j * 4 + 1]),
                     __float_as_uint(f[j * 4 + 2]), __float_as_uint(f[j * 4 + 3]));
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              sts128(buf_s + row_s + (((h * 4 + j) << 4) ^ sw), pack_bf16x2(f[j * 8 + 0], f[j * 8 + 1]),
                     pack_bf16x2(f[j * 8 + 2], f[j * 8 + 3]), pack_bf16x2(f[j * 8 + 4], f[j * 8 + 5]),
                     pack_bf16x2(f[j * 8 + 6], f[j * 8 + 7]));
          }
        }
        if (!chunk_live || out_direct != nullptr) continue;
        __syncwarp();
        if (stats != nullptr) {
          // Column sums over this warp's 32 rows, read back from the (bf16-rounded) slab: lane l owns columns 2l, 2l+1;
          // bank-conflict-free thanks to the 128B swizzle; packed fp32x2 adds / fmas, folded into the running sums.
          uint64_t a_s = 0, a_q = 0;
#pragma unroll
          for (int r = 0; r < 32; ++r) {
            const uint32_t w = lds32(buf_s + (r >> 3) * 1024 + stat_off[r & 7]);
            const uint64_t x2 = f2_pack(bf16_lo(w), bf16_hi(w));
            a_s = f2_add(a_s, x2);
            a_q = f2_fma(x2, x2, a_q);
          }
          const int slot = units == 1 ? (it & 1) : u;
#pragma unroll
          for (int k = 0; k < SLOTS; ++k) {
            if (k == slot) {
              run_s[k] = f2_add(run_s[k], a_s);
              run_q[k] = f2_add(run_q[k], a_q);
            }
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          // (cp.async.bulk takes a shared-window address: reuse the 32-bit slab address)
          asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                           reinterpret_cast<uint64_t>(&p.d_map)),
                       "r"(buf_s), "r"(n0), "r"(s1), "r"(s2), "r"(s3)
                       : "memory");
          tma_store_commit();
          if (has_aux) {
            asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                             reinterpret_cast<uint64_t>(&p.aux_map)),
                         "r"(aux_s), "r"(n0), "r"(s1), "r"(s2), "r"(s3)
                         : "memory");
            tma_store_commit();
          }
        }
        store_counter += has_aux ? 2 : 1;
      }
    }
#ifdef CONV_PROFILE
    if (blockIdx.x == 0 && lane == 0 && q == 0) {
      const int nt = (num_tiles - 1) / gridDim.x + 1;
      printf("conv epilogue: wait img_full %lld drain %lld  (cycles/tile)\n", cp_t[0] / nt, cp_t[1] / nt);
    }
#endif
    if (stats != nullptr) {
      const int cta = static_cast<int>(blockIdx.x);
      const int n_tile = cta % p.n_tiles;
      const int grp = cta / p.n_tiles;
#pragma unroll
      for (int k = 0; k < SLOTS; ++k) {
        const int srow = units == 1 ? (grp * 4 + q) * 2 + k : grp * 4 + q;
        const int col = n_tile * BLOCK_N + (units == 1 ? 0 : k * unit_cols) + 2 * lane;
        if (col < N) {
          float s_lo, s_hi, q_lo, q_hi;
          f2_unpack(run_s[k], s_lo, s_hi);
          f2_unpack(run_q[k], q_lo, q_hi);
          float* sp = stats + static_cast<long long>(srow) * 2 * N + col;
          *reinterpret_cast<float2*>(sp) = make_float2(s_lo, s_hi);
          if constexpr (kBnMask) {
            sp += N - lane;   // second row: this lane owns column `lane` of each 32-column half
            sp[0] = run_x[k][0];
            sp[32] = run_x[k][1];
          } else {
            *reinterpret_cast<float2*>(sp + N) = make_float2(q_lo, q_hi);
          }
        }
      }
    }
    if (lane == 0) tma_store_wait_all<0>();
  }
}

}  // namespace b200
