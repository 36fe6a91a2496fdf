// Shifted-window multi-head self-attention (Swin), head_dim 32, 7x7 windows (49 tokens), with wgmma - forward and backward.
//
//   attn = softmax( scale * q k^T + relative_position_bias[h] (+ shift mask[window]) ) ;  out = attn v
//
// The cyclic shift (torch.roll), window_partition and window_reverse of the reference are folded into the addressing:
// a window's 49 tokens are gathered with 16-byte cp.async copies straight from the un-rolled qkv tensor [B,H,W,3C]
// (pixel ((wy*7+i+shift)%H, (wx*7+j+shift)%W)) into the 128B-swizzled operand layout, and the result rows are scattered
// back to the same pixels, so none of the four full-tensor permutation passes of the reference is executed.
// Per (batch, window, head): S = Q K^T (64 query rows with 49 valid, N=64 keys, K=32) by wgmma, handed to the soft-max
// threads (one query row each) through a shared-memory image; P (bf16) goes through shared memory into O = P V. Scores never touch HBM; only the row log-sum-exp is kept.
// CTAs are persistent over (batch, window) pairs of ONE head so that the backward pass can accumulate the gradient of the
// relative-position bias in registers and flush it with one atomicAdd per element per CTA.
//
// Replaces WindowAttention.forward and the roll / window_partition / window_reverse / roll sequence of
// SwinTransformerBlock.forward (classification/swin_transformer/models/swin_transformer.py:118-149, :251-280), including the
// optional fused kernels of kernels/window_process (the --fused_window_process path).
#pragma once
#include "common.cuh"

namespace b200 {

struct WAttnParams {
  const __nv_bfloat16* qkv;   // [B][H][W][3*C]
  __nv_bfloat16* out;         // fwd: [B][H][W][C]
  const float* bias;          // [nH][masked ? nW : 1][49 queries i][64 (key j, 49 used)]: bias[h][i][j] (+ mask[w][i][j]), see
                              // wattn_bias_gather_kernel - 256-byte rows so that a soft-max thread fetches its row as 13 float4
  int masked;                 // 1: the table holds one slice per window (shifted blocks)
  float* lse;                 // [B][nW][nH][49], base-2 log-sum-exp of the scaled, biased scores
  int B, H, W, nH, shift;
  float scale;
  // backward only
  const __nv_bfloat16* o;     // forward output [B][H][W][C]
  const __nv_bfloat16* dout;  // [B][H][W][C]
  __nv_bfloat16* dqkv;        // [B][H][W][3*C]
  float* dbias;               // dense [nH][49][49], accumulated with atomics (zeroed by the caller)
};

constexpr int kWS = 7, kWT = 49;

// Optional phase timers (-DWATTN_PROFILE): CTA 0 prints the average cycles per step of every wait / compute phase.
#ifdef WATTN_PROFILE
#define WPROF_DECL(N) long long wp_t[N] = {}; long long wp_0 = clock64(), wp_1;
#define WPROF_TICK(i) { wp_1 = clock64(); wp_t[i] += wp_1 - wp_0; wp_0 = wp_1; }
#else
#define WPROF_DECL(N)
#define WPROF_TICK(i)
#endif

__device__ __forceinline__ float wattn_ex2(float x) {  // MUFU.EX2 without the denormal-range fix-up of exp2f / __expf
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

// pixel offset (in pixels) of token t of window (wy, wx) in the un-rolled image
__device__ __forceinline__ long long wattn_pixel(const WAttnParams& p, int b, int wy, int wx, int t) {
  const int i = t / kWS, j = t - i * kWS;
  int y = wy * kWS + i + p.shift, x = wx * kWS + j + p.shift;
  if (y >= p.H) y -= p.H;
  if (x >= p.W) x -= p.W;
  return (static_cast<long long>(b) * p.H + y) * p.W + x;
}

// Gather one 49 x 32 bf16 tile (64 B per token) into a [64][128B] 128B-swizzled tile (only the first 4 chunks of a row are used).
__device__ __forceinline__ void wattn_gather(uint32_t tile_s, const __nv_bfloat16* base, long long row_stride, int col0,
                                             const WAttnParams& p, int b, int wy, int wx, int tid, int nthreads) {
  for (int idx = tid; idx < kWT * 4; idx += nthreads) {
    const int t = idx >> 2, c = idx & 3;
    const long long pix = wattn_pixel(p, b, wy, wx, t);
    cp_async16(tile_s + t * 128 + ((c ^ (t & 7)) << 4), base + pix * row_stride + col0 + c * 8);
  }
}

// Two windows per step: rows 0..63 of every operand tile belong to window "A" of the pair, rows 64..127 to window "B"
// (49 real tokens + 15 zero rows each). A soft-max group (one warpgroup) multiplies the two diagonal 64 x 64 blocks with
// wgmma (one m64 product per window), so every product of a step is two m64 MMAs; P is written block-diagonally into a
// 128-row tile whose off-diagonal halves are zeroed once and never touched.
constexpr int kWAttnStages = 3;  // operand ring: the gathers run up to two steps ahead of the tensor core
constexpr int kWAttnImg = 128 * 64 * 4;   // per group: fp32 image of one 128 x 64 accumulator pair
constexpr int kWAttnFwdSmem = kWAttnStages * 2 * 16384 + 2 * 32768 + 2 * kWAttnImg + 256 + 1024;
// warps 0-1: gather, warps 4-7 / 8-11: soft-max groups 0 / 1 (warpgroups 1 and 2)
constexpr int kWAttnFwdThreads = 12 * 32;
constexpr int kWAttnGatherThreads = 64;
static_assert(kWAttnFwdSmem <= 227 * 1024, "shared memory of one H100 block");

__device__ __forceinline__ void wattn_item(const WAttnParams& p, int item, int nW, int nWx, int& b, int& win, int& wy, int& wx) {
  b = item / nW;
  win = item - b * nW;
  wy = win / nWx;
  wx = win - wy * nWx;
}

// Both m64 products of a step for one group: window w (rows 64 w ..) of D = A B, K = 16 * KSTEPS. A / B descriptors of
// window w: (a0 + w * a_win + k * a_k, b0 + w * b_win + k * b_k) in 16-byte units.
template <int N, int TA, int TB, int KSTEPS>
__device__ __forceinline__ void wattn_mma2(float (&d0)[N / 2], float (&d1)[N / 2], uint64_t a0, uint64_t a_win, uint64_t a_k,
                                           uint64_t b0, uint64_t b_win, uint64_t b_k) {
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d0[i] = 0.f, d1[i] = 0.f;
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) {
    Wgmma<N, TA, TB>::mma(d0, a0 + k * a_k, b0 + k * b_k, 1u);
    Wgmma<N, TA, TB>::mma(d1, a0 + a_win + k * a_k, b0 + b_win + k * b_k, 1u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_reg_fence(d0);
  wgmma_reg_fence(d1);
}
__device__ __forceinline__ uint64_t wdesc(uint32_t addr, uint32_t lbo) { return make_smem_desc_sw128(addr, lbo, 1024); }

// Forward, warp specialised. A step = one PAIR of windows of this CTA's head (see above).
//   gather warps (0, 1): tokens i and i+64 of the pair -> 12 cp.async (q, k, v x 4 chunks) into ring stage n%3, then arrive full
//   soft-max group g (warpgroup 1 + g) owns the steps with n&1 == g: S = Q K^T -> P (bf16, block diagonal) -> O = P V ->
//   write out, so the gathers of step n+1 and the two groups' steps overlap.
__global__ void __launch_bounds__(kWAttnFwdThreads, 1) wattn_fwd_kernel(const WAttnParams p) {
  pdl_wait();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // stage s: two tiles [128][128B] (rows 0..48: window A, 64..112: window B). A head row is only 64 B, so Q and K share
  // a tile (Q = 16-byte chunks 0..3 of a row, K = chunks 4..7: the K descriptor simply starts 64 B later) and V takes the
  // first half of the second tile; then P[g], then the accumulator images
  constexpr int kStage = 2 * 16384;
  constexpr int NS = kWAttnStages;
  uint8_t* sP = smem + NS * kStage;   // [2 groups][2 key atoms][128][128B]
  uint8_t* sImg = sP + 2 * 32768;     // [2 groups][128][64] fp32
  uint64_t* bars = reinterpret_cast<uint64_t*>(sImg + 2 * kWAttnImg);
  uint64_t* full = bars;        // [NS] gather complete (64 arrivals)
  uint64_t* empty = bars + 4;   // [NS] stage consumed (the group's P V product retired)
  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int C = p.nH * 32;
  const int nWy = p.H / kWS, nWx = p.W / kWS, nW = nWy * nWx;

  // zero everything once: pad rows of K / V and the off-diagonal halves of P must be finite zeros for every step
  for (int i = threadIdx.x; i < (NS * kStage + 2 * 32768) / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0) {
    for (int i = 0; i < NS; ++i) {
      mbar_init(&full[i], kWAttnGatherThreads);
      mbar_init(&empty[i], 1);
    }
    fence_mbar_init();
  }
  fence_proxy_async_smem();   // the zero fill above must be visible to the tensor core (async proxy)
  __syncthreads();

  const int head = blockIdx.x % p.nH;
  const int lanes = gridDim.x / p.nH;           // CTAs sharing this head
  const int total = p.B * nW;
  const int npairs = (total + 1) / 2;
  const int first = blockIdx.x / p.nH;
  const int nsteps = first < npairs ? (npairs - first + lanes - 1) / lanes : 0;

  if (warp_idx < 2) {
    // ===================== gather warps: one thread per token of the pair =====================
    const int i0 = threadIdx.x;   // 0..63; tokens i0 and i0 + 64 of the 98
    for (int n = 0; n < nsteps; ++n) {
      const int s = n % NS;
      const uint32_t ph = (n / NS) & 1;
      mbar_wait(&empty[s], ph ^ 1);
#pragma unroll
      for (int rep = 0; rep < 2; ++rep) {
        const int i = i0 + rep * kWAttnGatherThreads;
        const int slot = i / kWT, tok = i - slot * kWT;
        const int item = 2 * (first + n * lanes) + slot;
        if (i < 2 * kWT && item < total) {
          int b, win, wy, wx;
          wattn_item(p, item, nW, nWx, b, win, wy, wx);
          const __nv_bfloat16* src = p.qkv + wattn_pixel(p, b, wy, wx, tok) * 3 * C + head * 32;
          const int r = slot * 64 + tok;
          const uint32_t dst = smem_u32(smem + s * kStage) + r * 128;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            cp_async16(dst + ((c ^ (r & 7)) << 4), src + c * 8);                        // q
            cp_async16(dst + (((4 + c) ^ (r & 7)) << 4), src + C + c * 8);              // k
            cp_async16(dst + 16384 + ((c ^ (r & 7)) << 4), src + 2 * C + c * 8);        // v
          }
        }
      }
      cp_async_wait_all();
      fence_proxy_async_smem();
      mbar_arrive(&full[s]);
    }
  } else if (warp_idx >= 4) {
    // ===================== soft-max groups: thread = query row of window `slot` =====================
    const int g = (warp_idx >> 2) - 1;
    const int row = (warp_idx & 3) * 32 + lane;
    const int slot = row >> 6, tok = row & 63;
    const uint32_t img = smem_u32(sImg + g * kWAttnImg);
    const uint32_t p_g = smem_u32(sP + g * 32768);
    const uint32_t p_s = p_g + slot * 16384 + row * 128;  // this row's 64 keys (key atom `slot`)
    for (int n = g; n < nsteps; n += 2) {
      const int s = n % NS;
      const int item = 2 * (first + n * lanes) + slot;
      const bool valid = tok < kWT && item < total;
      int b = 0, win = 0, wy = 0, wx = 0;
      if (item < total) wattn_item(p, item, nW, nWx, b, win, wy, wx);
      // this row's bias (+ mask) values: requested before the wait so that their latency hides behind the gather / MMA
      const float4* brow = reinterpret_cast<const float4*>(
          p.bias + ((static_cast<long long>(head) * (p.masked ? nW : 1) + (p.masked ? win : 0)) * kWT + (valid ? tok : 0)) * 64);
      float4 bv[13];
#pragma unroll
      for (int c = 0; c < 13; ++c) bv[c] = __ldg(brow + c);
      const float* bf = reinterpret_cast<const float*>(bv);
      mbar_wait(&full[s], (n / NS) & 1);
      const uint32_t q_s = smem_u32(smem + s * kStage), k_s = q_s + 64, v_s = q_s + 16384;
      {
        // S = Q K^T of both windows (K = 32: two steps), into the image
        float s0[32], s1[32];
        wattn_mma2<64, 0, 0, 2>(s0, s1, wdesc(q_s, 16), 8192 >> 4, 2, wdesc(k_s, 16), 8192 >> 4, 2);
        named_bar_sync(1 + g, 128);   // the previous step's O has been read out of the image
        acc_to_img<64>(s0, img, 64, 0, 0);
        acc_to_img<64>(s1, img, 64, 64, 0);
        named_bar_sync(1 + g, 128);
      }
      uint32_t v[64];
      {
        uint32_t(&lo)[32] = *reinterpret_cast<uint32_t(*)[32]>(&v[0]);
        uint32_t(&hi)[32] = *reinterpret_cast<uint32_t(*)[32]>(&v[32]);
        img_ld32(img, 64, row, 0, lo);
        img_ld32(img, 64, row, 32, hi);
      }
      // log2 domain, branch free: rows outside the window (zero Q rows -> finite scores) get max = +inf -> all-zero P
      const float scale2 = p.scale * 1.4426950408889634f;
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < kWT; ++j) {
        const float sc = fmaf(__uint_as_float(v[j]), scale2, bf[j]);
        v[j] = __float_as_uint(sc);
        mx = fmaxf(mx, sc);
      }
      const float mxe = valid ? mx : INFINITY;
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 64; j += 2) {
        const float e0 = j < kWT ? wattn_ex2(__uint_as_float(v[j]) - mxe) : 0.f;
        const float e1 = j + 1 < kWT ? wattn_ex2(__uint_as_float(v[j + 1]) - mxe) : 0.f;
        const uint32_t w = pack_bf16x2(e0, e1);
        sum += bf16_lo(w) + bf16_hi(w);
        v[j >> 1] = w;  // in place: slot j/2 has already been consumed
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) sts128(p_s + ((c ^ (row & 7)) << 4), v[c * 4], v[c * 4 + 1], v[c * 4 + 2], v[c * 4 + 3]);
      if (valid) p.lse[((static_cast<long long>(b) * nW + win) * p.nH + head) * kWT + tok] = mx + __log2f(sum);  // log2 units
      fence_proxy_async_smem();
      named_bar_sync(1 + g, 128);   // P complete; every row has read S out of the image
      {
        // O = P V of both windows: A = P (K-major, the window's own key atom), B = V (MN-major), K = 64 keys
        float o0[16], o1[16];
        wattn_mma2<32, 0, 1, 4>(o0, o1, wdesc(p_g, 16), (16384 + 8192) >> 4, 2, wdesc(v_s, 8192), 8192 >> 4, 2048 >> 4);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);   // Q / K / V of this stage are no longer read
        acc_to_img<32>(o0, img, 64, 0, 0);
        acc_to_img<32>(o1, img, 64, 64, 0);
        named_bar_sync(1 + g, 128);
      }
      uint32_t ov[32];
      img_ld32(img, 64, row, 0, ov);
      if (valid) {
        const float inv = 1.0f / sum;
        __nv_bfloat16* dst = p.out + wattn_pixel(p, b, wy, wx, tok) * C + head * 32;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          uint4 w;
          w.x = pack_bf16x2(__uint_as_float(ov[c * 8 + 0]) * inv, __uint_as_float(ov[c * 8 + 1]) * inv);
          w.y = pack_bf16x2(__uint_as_float(ov[c * 8 + 2]) * inv, __uint_as_float(ov[c * 8 + 3]) * inv);
          w.z = pack_bf16x2(__uint_as_float(ov[c * 8 + 4]) * inv, __uint_as_float(ov[c * 8 + 5]) * inv);
          w.w = pack_bf16x2(__uint_as_float(ov[c * 8 + 6]) * inv, __uint_as_float(ov[c * 8 + 7]) * inv);
          *reinterpret_cast<uint4*>(dst + c * 8) = w;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Backward. Per (batch, window, head), two windows per step as in the forward kernel:
//   P = exp(scale*S + bias + mask - lse);  dP = dO V^T;  dS = P*(dP - delta), delta_i = <dO_i, O_i>;  dbias += dS
//   dV = P^T dO;  dQ = scale * dS K;  dK = scale * dS^T Q          (dS is stored pre-multiplied by scale)
constexpr int kWAttnBwdSmem = kWAttnFwdSmem;

// Same warp-specialised pipeline as the forward kernel (Q/K/V/dO ring, two soft-max groups with their own P/dS tile and
// accumulator image); each group issues its step's products itself: S = Q K^T, then dP = dO V^T with dV = P^T dO, then
// dQ = dS K with dK = dS^T Q (block diagonal: only the two 64 x 64 window blocks are multiplied).
__global__ void __launch_bounds__(kWAttnFwdThreads, 1) wattn_bwd_kernel(const WAttnParams p) {
  pdl_wait();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int kStage = 2 * 16384;   // tile 0: Q (chunks 0..3 of a row) | K (chunks 4..7); tile 1: V | dO
  constexpr int NS = kWAttnStages;
  uint8_t* sP = smem + NS * kStage;   // [2 groups][2 key atoms][128][128B]: P, then dS in place (block diagonal)
  uint8_t* sImg = sP + 2 * 32768;     // [2 groups][128][64] fp32
  uint64_t* bars = reinterpret_cast<uint64_t*>(sImg + 2 * kWAttnImg);
  uint64_t* full = bars;         // [NS]
  uint64_t* empty = bars + 4;    // [NS]
  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int C = p.nH * 32;
  const int nWy = p.H / kWS, nWx = p.W / kWS, nW = nWy * nWx;

  for (int i = threadIdx.x; i < (NS * kStage + 2 * 32768) / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0) {
    for (int i = 0; i < NS; ++i) {
      mbar_init(&full[i], kWAttnGatherThreads);
      mbar_init(&empty[i], 1);
    }
    fence_mbar_init();
  }
  fence_proxy_async_smem();
  __syncthreads();

  const int head = blockIdx.x % p.nH;
  const int lanes = gridDim.x / p.nH;
  const int total = p.B * nW;
  const int npairs = (total + 1) / 2;
  const int first = blockIdx.x / p.nH;
  const int nsteps = first < npairs ? (npairs - first + lanes - 1) / lanes : 0;

  if (warp_idx < 4) {
    setmaxnreg_dec<56>();
    if (warp_idx < 2) {
    // ===================== gather warps: one thread per token of the pair (q, k, v, dO rows) =====================
    const int i0 = threadIdx.x;
    WPROF_DECL(3)
    for (int n = 0; n < nsteps; ++n) {
      const int s = n % NS;
      WPROF_TICK(2)
      mbar_wait(&empty[s], ((n / NS) & 1) ^ 1);
      WPROF_TICK(0)
#pragma unroll
      for (int rep = 0; rep < 2; ++rep) {
        const int i = i0 + rep * kWAttnGatherThreads;
        const int slot = i / kWT, tok = i - slot * kWT;
        const int item = 2 * (first + n * lanes) + slot;
        if (i < 2 * kWT && item < total) {
          int b, win, wy, wx;
          wattn_item(p, item, nW, nWx, b, win, wy, wx);
          const long long pix = wattn_pixel(p, b, wy, wx, tok);
          const __nv_bfloat16* src = p.qkv + pix * 3 * C + head * 32;
          const __nv_bfloat16* dsrc = p.dout + pix * C + head * 32;
          const int r = slot * 64 + tok;
          const uint32_t dst = smem_u32(smem + s * kStage) + r * 128;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            cp_async16(dst + ((c ^ (r & 7)) << 4), src + c * 8);                          // q
            cp_async16(dst + (((4 + c) ^ (r & 7)) << 4), src + C + c * 8);                // k
            cp_async16(dst + 16384 + ((c ^ (r & 7)) << 4), src + 2 * C + c * 8);          // v
            cp_async16(dst + 16384 + (((4 + c) ^ (r & 7)) << 4), dsrc + c * 8);           // dO
          }
        }
      }
      WPROF_TICK(1)
      cp_async_wait_all();
      fence_proxy_async_smem();
      mbar_arrive(&full[s]);
    }
#ifdef WATTN_PROFILE
    if (blockIdx.x == 0 && threadIdx.x == 0 && nsteps > 0)
      printf("bwd gather : wait_empty %lld  issue %lld  wait_data %lld\n", wp_t[0] / nsteps, wp_t[1] / nsteps, wp_t[2] / nsteps);
#endif
    }
  } else {
    // ===================== soft-max groups =====================
    setmaxnreg_inc<224>();
    const int g = (warp_idx >> 2) - 1;
    const int row = (warp_idx & 3) * 32 + lane;
    const int slot = row >> 6, tok = row & 63;
    const uint32_t img = smem_u32(sImg + g * kWAttnImg);
    const uint32_t p_g = smem_u32(sP + g * 32768);
    uint8_t* const prow = sP + g * 32768 + slot * 16384 + row * 128;   // this row's 64 keys (key atom `slot`)
    const uint32_t prow_s = smem_u32(prow);
    WPROF_DECL(14)
    float db[kWT];  // gradient of bias[head][tok][:] accumulated over this thread's steps
#pragma unroll
    for (int j = 0; j < kWT; ++j) db[j] = 0.f;
    for (int n = g; n < nsteps; n += 2) {
      const int s = n % NS;
      const int item = 2 * (first + n * lanes) + slot;
      const bool valid = tok < kWT && item < total;
      int b = 0, win = 0, wy = 0, wx = 0;
      if (item < total) wattn_item(p, item, nW, nWx, b, win, wy, wx);
      const long long pix = wattn_pixel(p, b, wy, wx, valid ? tok : 0);
      // log2-domain row log-sum-exp; +inf for rows outside the window makes their P exactly zero without a branch
      const float lse = valid ? p.lse[((static_cast<long long>(b) * nW + win) * p.nH + head) * kWT + tok] : INFINITY;
      const float scale2 = p.scale * 1.4426950408889634f;
      const float4* brow = reinterpret_cast<const float4*>(
          p.bias + ((static_cast<long long>(head) * (p.masked ? nW : 1) + (p.masked ? win : 0)) * kWT + (valid ? tok : 0)) * 64);
      float4 bv[13];  // this row's bias (+ mask) values, requested before the wait
#pragma unroll
      for (int c = 0; c < 13; ++c) bv[c] = __ldg(brow + c);
      const float* bf = reinterpret_cast<const float*>(bv);
      uint4 orow[4];  // forward output row (64 B), requested early: only needed for delta
      if (valid) {
        const uint4* op = reinterpret_cast<const uint4*>(p.o + pix * C + head * 32);
#pragma unroll
        for (int c = 0; c < 4; ++c) orow[c] = __ldg(op + c);
      }
      WPROF_TICK(13)
      mbar_wait(&full[s], (n / NS) & 1);
      WPROF_TICK(0)
      const uint32_t q_s = smem_u32(smem + s * kStage), k_s = q_s + 64, v_s = q_s + 16384, do_s = v_s + 64;
      {
        // S = Q K^T (both windows) into the image
        float s0[32], s1[32];
        wattn_mma2<64, 0, 0, 2>(s0, s1, wdesc(q_s, 16), 8192 >> 4, 2, wdesc(k_s, 16), 8192 >> 4, 2);
        named_bar_sync(1 + g, 128);   // the previous step's gradients have been read out of the image
        acc_to_img<64>(s0, img, 64, 0, 0);
        acc_to_img<64>(s1, img, 64, 64, 0);
        named_bar_sync(1 + g, 128);
      }
      // ---- P
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {   // two 32-key halves keep the live register set small
        uint32_t v[32];
        img_ld32(img, 64, row, hf * 32, v);
        WPROF_TICK(1)
#pragma unroll
        for (int jj = 0; jj < 32; jj += 2) {
          const int j = hf * 32 + jj;
          float e0 = 0.f, e1 = 0.f;
          if (j < kWT) e0 = wattn_ex2(fmaf(__uint_as_float(v[jj]), scale2, bf[j]) - lse);
          if (j + 1 < kWT) e1 = wattn_ex2(fmaf(__uint_as_float(v[jj + 1]), scale2, bf[j + 1 < 52 ? j + 1 : 51]) - lse);
          v[jj >> 1] = pack_bf16x2(e0, e1);
        }
        WPROF_TICK(2)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          sts128(prow_s + (((hf * 4 + c) ^ (row & 7)) << 4), v[c * 4], v[c * 4 + 1], v[c * 4 + 2], v[c * 4 + 3]);
        WPROF_TICK(3)
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + g, 128);   // P complete; S read out of the image
      WPROF_TICK(4)
      // dP = dO V^T (both windows) into the image, dV = P^T dO (A = P^T: the window's key atom, MN-major) kept in registers
      float gv0[16], gv1[16];
      {
        float d0[32], d1[32];
        wattn_mma2<64, 0, 0, 2>(d0, d1, wdesc(do_s, 16), 8192 >> 4, 2, wdesc(v_s, 16), 8192 >> 4, 2);
        acc_to_img<64>(d0, img, 64, 0, 0);
        acc_to_img<64>(d1, img, 64, 64, 0);
        wattn_mma2<32, 1, 1, 4>(gv0, gv1, wdesc(p_g, 16384), (16384 + 8192) >> 4, 2048 >> 4, wdesc(do_s, 8192), 8192 >> 4,
                             2048 >> 4);
      }
      // delta_i = <dO_i, O_i>: dO from the gathered tile (stage s stays valid until this step's last products retire)
      float delta = 0.f;
      if (valid) {
        const uint8_t* drow = smem + s * kStage + 16384 + row * 128;   // dO = chunks 4..7 of the V|dO tile row
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float a[8], o[8];
          unpack8(*reinterpret_cast<const uint4*>(drow + (((4 + c) ^ (row & 7)) << 4)), a);
          unpack8(orow[c], o);
#pragma unroll
          for (int e = 0; e < 8; ++e) delta = fmaf(a[e], o[e], delta);
        }
      }
      named_bar_sync(1 + g, 128);   // dP in the image
      // ---- dS (in place over P)
      WPROF_TICK(6)
      {
        uint32_t v[64];
        uint32_t(&lo)[32] = *reinterpret_cast<uint32_t(*)[32]>(&v[0]);
        uint32_t(&hi)[32] = *reinterpret_cast<uint32_t(*)[32]>(&v[32]);
        img_ld32(img, 64, row, 0, lo);
        img_ld32(img, 64, row, 32, hi);
        WPROF_TICK(7)
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const uint32_t off = (c ^ (row & 7)) << 4;
          float pv[8];
          unpack8(*reinterpret_cast<const uint4*>(prow + off), pv);  // P of this row (bf16, as the tensor core saw it)
          float d[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int j = c * 8 + e;
            d[e] = pv[e] * (__uint_as_float(v[j]) - delta);   // rows outside the window have P == 0 (and finite dP)
            if (j < kWT) db[j] += d[e];
            d[e] *= p.scale;
          }
          sts128(prow_s + off, pack_bf16x2(d[0], d[1]), pack_bf16x2(d[2], d[3]), pack_bf16x2(d[4], d[5]), pack_bf16x2(d[6], d[7]));
        }
      }
      WPROF_TICK(8)
      fence_proxy_async_smem();
      named_bar_sync(1 + g, 128);   // dS complete; dP read out of the image
      // dQ = dS K (A = dS K-major, B = K MN-major) and dK = dS^T Q (both MN-major), then the gradients through the image
      {
        float q0[16], q1[16], k0[16], k1[16];
        wattn_mma2<32, 0, 1, 4>(q0, q1, wdesc(p_g, 16), (16384 + 8192) >> 4, 2, wdesc(k_s, 8192), 8192 >> 4, 2048 >> 4);
        wattn_mma2<32, 1, 1, 4>(k0, k1, wdesc(p_g, 16384), (16384 + 8192) >> 4, 2048 >> 4, wdesc(q_s, 8192), 8192 >> 4,
                             2048 >> 4);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);   // the stage is no longer read
        acc_to_img<32>(q0, img, 64, 0, 0);
        acc_to_img<32>(q1, img, 64, 64, 0);
        acc_to_img<32>(k0, img, 64, 0, 32);
        acc_to_img<32>(k1, img, 64, 64, 32);
      }
      named_bar_sync(1 + g, 128);
      WPROF_TICK(10)
      uint32_t gq[32], gk[32], gv[32];
      img_ld32(img, 64, row, 0, gq);
      {
        uint32_t t2[32];
        img_ld32(img, 64, row, 32, t2);
#pragma unroll
        for (int i = 0; i < 32; ++i) gk[i] = t2[i];
      }
      named_bar_sync(1 + g, 128);
      acc_to_img<32>(gv0, img, 64, 0, 0);
      acc_to_img<32>(gv1, img, 64, 64, 0);
      named_bar_sync(1 + g, 128);
      img_ld32(img, 64, row, 0, gv);
      WPROF_TICK(11)
      if (valid) {
        __nv_bfloat16* dst = p.dqkv + pix * 3 * C + head * 32;
#pragma unroll
        for (int which = 0; which < 3; ++which) {
          const uint32_t* gg = which == 0 ? gq : (which == 1 ? gk : gv);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            uint4 w;
            w.x = pack_bf16x2(__uint_as_float(gg[c * 8 + 0]), __uint_as_float(gg[c * 8 + 1]));
            w.y = pack_bf16x2(__uint_as_float(gg[c * 8 + 2]), __uint_as_float(gg[c * 8 + 3]));
            w.z = pack_bf16x2(__uint_as_float(gg[c * 8 + 4]), __uint_as_float(gg[c * 8 + 5]));
            w.w = pack_bf16x2(__uint_as_float(gg[c * 8 + 6]), __uint_as_float(gg[c * 8 + 7]));
            *reinterpret_cast<uint4*>(dst + which * C + c * 8) = w;
          }
        }
      }
      WPROF_TICK(12)
    }
#ifdef WATTN_PROFILE
    WPROF_TICK(12)
    if (blockIdx.x == 0 && lane == 0 && (warp_idx & 3) == 0 && nsteps > 1) {
      const int ns = (nsteps - g + 1) / 2;
      printf("bwd softmax g%d: wait_s %lld | P: ld %lld math %lld sts %lld fence %lld | dS: ld %lld math %lld | "
             "grad: mma %lld ld %lld store %lld | prologue %lld\n", g, wp_t[0] / ns, wp_t[1] / ns, wp_t[2] / ns, wp_t[3] / ns,
             wp_t[4] / ns, wp_t[7] / ns, wp_t[8] / ns, wp_t[10] / ns, wp_t[11] / ns, wp_t[12] / ns, wp_t[13] / ns);
    }
#endif
    if (tok < kWT) {
      float* dbp = p.dbias + (static_cast<long long>(head) * kWT + tok) * kWT;
#pragma unroll
      for (int j = 0; j < kWT; ++j) atomicAdd(dbp + j, db[j]);
    }
  }
}

// tab[h][w][i][j] = log2(e) * (table[index[i][j]][h] (+ mask[w][i][j]))      (WindowAttention.forward :131-147), j padded to 64
// One launch per block and step folds the relative-position bias gather and the shift mask into one table of 256-byte
// rows (one per query) that the soft-max threads read with 13 vector loads.
__global__ void wattn_bias_gather_kernel(const float* __restrict__ table, const long long* __restrict__ index,
                                         const float* __restrict__ mask, int nWm, float* __restrict__ tab, int nH) {
  pdl_wait();
  const long long n = static_cast<long long>(nH) * nWm * kWT * 64;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(e & 63);
    long long t = e >> 6;
    const int i = static_cast<int>(t % kWT);
    t /= kWT;
    const int w = static_cast<int>(t % nWm);
    const int h = static_cast<int>(t / nWm);
    float v = 0.f;
    if (j < kWT) {
      v = table[index[i * kWT + j] * nH + h];
      if (mask != nullptr) v += mask[(static_cast<long long>(w) * kWT + i) * kWT + j];
      v *= 1.4426950408889634f;   // the kernels work in the log2 domain: p = 2^(s*scale*log2e + tab - lse2)
    }
    tab[e] = v;
  }
}
// dtable[index[i][j]][h] (+)= dbias[h][i][j]   (dtable zeroed / holding the running gradient)
__global__ void wattn_bias_scatter_kernel(const float* __restrict__ dbias, const long long* __restrict__ index,
                                          float* __restrict__ dtable, int nH) {
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nH * kWT * kWT) return;
  const int h = i / (kWT * kWT), ij = i - h * kWT * kWT;
  atomicAdd(dtable + index[ij] * nH + h, dbias[i]);
}

// ------------------------------------------------------------------------------------------------------------------
// Stand-alone permutations of kernels/window_process (the reference's only first-party CUDA; B2 seam), 16-byte vectors:
//   partition: out[b*nW + win][wy][wx][:] = in[b][(wh*ws + wy - shift) mod H][(ww*ws + wx - shift) mod W][:]
//   merge:     out[b][h][w][:] = in[b*nW + win(h', w')][h' % ws][w' % ws][:],  (h', w') = ((h - shift) mod H, (w - shift) mod W)
// Each thread moves four independent 16-byte vectors per iteration (index arithmetic in 32 bits: the tensors of this path hold
// far fewer than 2^32 vectors), so ~64 B per thread are in flight - a permutation kernel is pure HBM latency hiding.
template <bool kMerge>
__global__ void __launch_bounds__(256) window_permute_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int B, int H,
                                                             int W, int cvec, int shift, int ws) {
  pdl_wait();
  const unsigned nWx = W / ws, nWy = H / ws;
  const unsigned total = static_cast<unsigned>(B) * H * W * cvec;
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < total; i0 += 4 * stride) {
    uint4 v[4];
    unsigned src[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const unsigned i = i0 + u * stride;
      if (i >= total) break;
      const unsigned c = i % cvec;
      unsigned t = i / cvec;
      if (kMerge) {
        // out[b][h][w] = in[b*nW + win(h', w')][h' % ws][w' % ws],  (h', w') = ((h - shift) mod H, (w - shift) mod W)
        const unsigned w = t % W;
        t /= W;
        const unsigned h = t % H;
        const unsigned b = t / H;
        int y = (static_cast<int>(h) - shift) % H, x = (static_cast<int>(w) - shift) % W;
        if (y < 0) y += H;
        if (x < 0) x += W;
        const unsigned win = (b * nWy + y / ws) * nWx + x / ws;
        src[u] = ((win * ws + y % ws) * ws + x % ws) * cvec + c;
      } else {
        // out[b*nW + win][wy][wx] = in[b][(wh*ws + wy - shift) mod H][(ww*ws + wx - shift) mod W]
        const unsigned wx = t % ws;
        t /= ws;
        const unsigned wy = t % ws;
        t /= ws;
        const unsigned ww = t % nWx;
        t /= nWx;
        const unsigned wh = t % nWy;
        const unsigned b = t / nWy;
        int y = (static_cast<int>(wh * ws + wy) - shift) % H, x = (static_cast<int>(ww * ws + wx) - shift) % W;
        if (y < 0) y += H;
        if (x < 0) x += W;
        src[u] = ((b * H + y) * W + x) * cvec + c;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (i0 + u * stride < total) v[u] = __ldg(in + src[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (i0 + u * stride < total) out[i0 + u * stride] = v[u];
  }
}

}  // namespace b200
