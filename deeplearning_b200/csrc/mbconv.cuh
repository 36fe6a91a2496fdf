// MBConv block passes of EfficientNet (classification/efficientNet/models/network.py MBConv:176-242, SELayer:126-145):
//
//   forward   d = dwconv_kxk(silu(c_e * s_e + t_e))      the expand BatchNorm + SiLU applied on load, never stored
//             pool = mean_p silu(d * s_d + t_d)          squeeze
//             gate = sigmoid(W2 silu(W1 pool + b1) + b2) excite (fp32, biased 1x1 convolutions of the pooled vector)
//             a = silu(d * s_d + t_d) * gate             gate apply: the input of the project GEMM
//             y = (c_p * s_p + t_p) * r_b (+ x)          tail apply: drop-connect multiplier r_b, residual x
//   backward  tail reduce      dz = g r_b, {sum dz, sum dz c_p}
//             gate reduce      S = sum_p da silu(u_d)   (u = the BatchNorm output)
//             excite backward  dW1, db1, dW2, db2 and dpool from S
//             SiLU-BN reduce   dz = (da gate + dpool / HW) silu'(u_d), {sum dz, sum dz d}
//             BN apply from dz dc = scale (dz - m1 - xhat m2)   (b200_bn_bwd_apply, elementwise.cuh)
//             depthwise dgrad  (+ residual) or x silu'(u_in) with the input BatchNorm's {sum dz, sum dz x}
//             depthwise wgrad  dW [C][k*k]
//
// The streaming passes use the row geometry of row_passes.cuh.  The depthwise passes use 64-channel CTAs (8 groups of 8
// channels x 32 row lanes) so that the block's k*k taps of 64 channels fit in shared memory; each thread reads the taps of
// its 8 channels as two float4s per tap.
#pragma once
#include "row_passes.cuh"

namespace b200 {

__device__ __forceinline__ float mb_sigmoid(float u) { return 1.f / (1.f + __expf(-u)); }
__device__ __forceinline__ float mb_silu(float u) { return u * mb_sigmoid(u); }
__device__ __forceinline__ float mb_dsilu(float u) {
  const float s = mb_sigmoid(u);
  return s * (1.f + u * (1.f - s));
}

// ------------------------------------------------------------------------------------------------ depthwise geometry
constexpr int kDwLanes = 32;   // row lanes per CTA; 8 channel groups x 32 lanes = 256 threads

struct DwGeom {
  int nchunk, blocks, rows_per_block;
};

__host__ __device__ inline DwGeom dw_geom(long long rows, int C) {
  DwGeom g;
  g.nchunk = (C + 63) / 64;
  long long blocks = kRvTargetCtas / g.nchunk;
  if (blocks < 1) blocks = 1;
  long long rpb = (rows + blocks - 1) / blocks;
  rpb = ((rpb + kDwLanes - 1) / kDwLanes) * kDwLanes;
  blocks = (rows + rpb - 1) / rpb;
  g.blocks = static_cast<int>(blocks);
  g.rows_per_block = static_cast<int>(rpb);
  return g;
}

// taps of the CTA's 64 channels, [k*k][64] (zero past C)
template <int K>
__device__ __forceinline__ void dw_stage_taps(const float* __restrict__ w, int C, float (*ws)[64]) {
  const int c0 = blockIdx.y * 64;
  for (int i = threadIdx.x; i < K * K * 64; i += 256) {
    const int cc = i / (K * K), tap = i % (K * K);
    ws[tap][cc] = c0 + cc < C ? __ldg(w + static_cast<long long>(c0 + cc) * K * K + tap) : 0.f;
  }
  __syncthreads();
}

__device__ __forceinline__ void dw_tap8(const float (*ws)[64], int tap, int lane_g, float (&t)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(&ws[tap][lane_g * 8]);
  const float4 b = *reinterpret_cast<const float4*>(&ws[tap][lane_g * 8 + 4]);
  t[0] = a.x; t[1] = a.y; t[2] = a.z; t[3] = a.w;
  t[4] = b.x; t[5] = b.y; t[6] = b.z; t[7] = b.w;
}

// What the depthwise passes apply to their input on load (template argument PRE): nothing, the previous BatchNorm + SiLU
// (EfficientNet), or the previous BatchNorm + ReLU (ShuffleNet, shufflenet.cuh).  A bool true selects kDwSilu.
constexpr int kDwRaw = 0, kDwSilu = 1, kDwRelu = 2;

// 8 input channels at (b, ih, iw), with silu / relu(x * sc + sh) applied when PRE
template <int PRE>
__device__ __forceinline__ void dw_load_in(const __nv_bfloat16* __restrict__ x, long long pix, int C, int cg,
                                           const float (&sc)[8], const float (&sh)[8], float (&v)[8]) {
  unpack8(__ldg(reinterpret_cast<const uint4*>(x + pix * C) + cg), v);
  if constexpr (PRE == kDwSilu) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = mb_silu(fmaf(v[j], sc[j], sh[j]));
  } else if constexpr (PRE == kDwRelu) {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = fmaxf(fmaf(v[j], sc[j], sh[j]), 0.f);
  }
}

// derivative of the on-load activation at u = x * sc + sh (relu'(0) = 0, as torch's ReLU backward)
template <int PRE>
__device__ __forceinline__ float dw_dact(float u) {
  if constexpr (PRE == kDwRelu) return u > 0.f ? 1.f : 0.f;
  else return mb_dsilu(u);
}

// ---------------------------------------------------------------------------------------------- depthwise forward
// d[b][oh][ow][c] = sum_taps in(b, oh*S - K/2 + kh, ow*S - K/2 + kw, c) w[c][kh][kw]; stats [T][2][C] = sums of the stored
// bf16 d and d^2 per CTA row range.
template <int K, int S, int PRE, bool STATS>
__global__ void __launch_bounds__(256, 2) dw_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w,
                                                     const float* __restrict__ scale, const float* __restrict__ shift,
                                                     __nv_bfloat16* __restrict__ d, float* __restrict__ stats, int B, int H,
                                                     int W, int Ho, int Wo, int C, int rows_per_block) {
  __shared__ __align__(16) float ws[K * K][64];
  pdl_wait();
  dw_stage_taps<K>(w, C, ws);
  const int lane_g = threadIdx.x % 8, rsub = threadIdx.x / 8;
  const int cg = blockIdx.y * 8 + lane_g;
  const bool live = cg < C / 8;
  float acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
  if (live) {
    float sc[8], sh[8];
    if constexpr (PRE) {
      load8f(scale + cg * 8, sc);
      load8f(shift + cg * 8, sh);
    }
    const long long rows = static_cast<long long>(B) * Ho * Wo;
    const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
    const long long r1 = min(rows, r0 + rows_per_block);
    for (long long r = r0 + rsub; r < r1; r += kDwLanes) {
      const int ow = static_cast<int>(r % Wo);
      const long long t = r / Wo;
      const int oh = static_cast<int>(t % Ho);
      const long long b = t / Ho;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = 0.f;
#pragma unroll
      for (int kh = 0; kh < K; ++kh) {
        const int ih = oh * S - K / 2 + kh;
        if (ih < 0 || ih >= H) continue;
#pragma unroll
        for (int kw = 0; kw < K; ++kw) {
          const int iw = ow * S - K / 2 + kw;
          if (iw < 0 || iw >= W) continue;
          float v[8], tp[8];
          dw_load_in<PRE>(x, (b * H + ih) * W + iw, C, cg, sc, sh, v);
          dw_tap8(ws, kh * K + kw, lane_g, tp);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = fmaf(v[j], tp[j], o[j]);
        }
      }
      const uint4 q = pack8(o);
      reinterpret_cast<uint4*>(d + r * C)[cg] = q;
      if constexpr (STATS) {
        unpack8(q, o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc[0][j] += o[j];
          acc[1][j] = fmaf(o[j], o[j], acc[1][j]);
        }
      }
    }
  }
  if constexpr (STATS) {
    if (rv_cta_reduce<2>(acc, 8, kDwLanes, lane_g, rsub) && live) {
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int j = 0; j < 8; ++j) stats[(static_cast<long long>(blockIdx.x) * 2 + s) * C + cg * 8 + j] = acc[s][j];
    }
  }
}

// --------------------------------------------------------------------------------------------- depthwise data gradient
// g_in[b][ih][iw][c] = sum over the taps that read (ih, iw) of dd[b][oh][ow][c] w[c][kh][kw], rows = input pixels.
// PRE (the input was normalised on load): dx = g_in act'(x sc + sh) and partial [T][2][C] = {sum dx, sum dx x} of the
// stored bf16 dx; RES: dx = g_in + residual.
template <int K, int S, int PRE, bool RES>
__global__ void __launch_bounds__(256, 2) dw_dgrad_kernel(const __nv_bfloat16* __restrict__ dd, const float* __restrict__ w,
                                                       const __nv_bfloat16* __restrict__ x, const float* __restrict__ scale,
                                                       const float* __restrict__ shift,
                                                       const __nv_bfloat16* __restrict__ res, __nv_bfloat16* __restrict__ dx,
                                                       float* __restrict__ partial, int B, int H, int W, int Ho, int Wo,
                                                       int C, int rows_per_block) {
  __shared__ __align__(16) float ws[K * K][64];
  pdl_wait();
  dw_stage_taps<K>(w, C, ws);
  const int lane_g = threadIdx.x % 8, rsub = threadIdx.x / 8;
  const int cg = blockIdx.y * 8 + lane_g;
  const bool live = cg < C / 8;
  float acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
  if (live) {
    float sc[8], sh[8];
    if constexpr (PRE) {
      load8f(scale + cg * 8, sc);
      load8f(shift + cg * 8, sh);
    }
    const long long rows = static_cast<long long>(B) * H * W;
    const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
    const long long r1 = min(rows, r0 + rows_per_block);
    for (long long r = r0 + rsub; r < r1; r += kDwLanes) {
      const int iw = static_cast<int>(r % W);
      const long long t = r / W;
      const int ih = static_cast<int>(t % H);
      const long long b = t / H;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = 0.f;
#pragma unroll
      for (int kh = 0; kh < K; ++kh) {
        const int th = ih + K / 2 - kh;
        if (th < 0 || (S == 2 && (th & 1))) continue;
        const int oh = th / S;
        if (oh >= Ho) continue;
#pragma unroll
        for (int kw = 0; kw < K; ++kw) {
          const int tw = iw + K / 2 - kw;
          if (tw < 0 || (S == 2 && (tw & 1))) continue;
          const int ow = tw / S;
          if (ow >= Wo) continue;
          float g[8], tp[8];
          unpack8(__ldg(reinterpret_cast<const uint4*>(dd + ((b * Ho + oh) * Wo + ow) * C) + cg), g);
          dw_tap8(ws, kh * K + kw, lane_g, tp);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = fmaf(g[j], tp[j], o[j]);
        }
      }
      if constexpr (PRE) {
        float xv[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(x + r * C) + cg), xv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] *= dw_dact<PRE>(fmaf(xv[j], sc[j], sh[j]));
        const uint4 q = pack8(o);
        reinterpret_cast<uint4*>(dx + r * C)[cg] = q;
        unpack8(q, o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc[0][j] += o[j];
          acc[1][j] = fmaf(o[j], xv[j], acc[1][j]);
        }
      } else {
        if constexpr (RES) {
          float rv[8];
          unpack8(__ldg(reinterpret_cast<const uint4*>(res + r * C) + cg), rv);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += rv[j];
        }
        reinterpret_cast<uint4*>(dx + r * C)[cg] = pack8(o);
      }
    }
  }
  if constexpr (PRE) {
    if (rv_cta_reduce<2>(acc, 8, kDwLanes, lane_g, rsub) && live) {
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int j = 0; j < 8; ++j) partial[(static_cast<long long>(blockIdx.x) * 2 + s) * C + cg * 8 + j] = acc[s][j];
    }
  }
}

// ------------------------------------------------------------------------------------------- depthwise weight gradient
// CTA (row range, 64-channel block, kernel row kh = blockIdx.z): ws[T][kh][kw][C] = sum over its output pixels of
// dd[b][oh][ow][c] in(b, oh*S - K/2 + kh, ow*S - K/2 + kw, c); dw_wgrad_reduce_kernel sums the T slabs in order.
// (ptxas' default register budget spills the ReLU mode; a one-CTA minimum lifts it and leaves the other modes' code as is)
template <int K, int S, int PRE>
__global__ void __launch_bounds__(256, PRE == kDwRelu ? 1 : 0) dw_wgrad_kernel(const __nv_bfloat16* __restrict__ dd,
                                                       const __nv_bfloat16* __restrict__ x, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, float* __restrict__ ws, int B, int H,
                                                       int W, int Ho, int Wo, int C, int rows_per_block) {
  pdl_wait();
  const int kh = blockIdx.z;
  const int lane_g = threadIdx.x % 8, rsub = threadIdx.x / 8;
  const int cg = blockIdx.y * 8 + lane_g;
  const bool live = cg < C / 8;
  float acc[K][8];
#pragma unroll
  for (int s = 0; s < K; ++s)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[s][j] = 0.f;
  if (live) {
    float sc[8], sh[8];
    if constexpr (PRE) {
      load8f(scale + cg * 8, sc);
      load8f(shift + cg * 8, sh);
    }
    const long long rows = static_cast<long long>(B) * Ho * Wo;
    const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
    const long long r1 = min(rows, r0 + rows_per_block);
    for (long long r = r0 + rsub; r < r1; r += kDwLanes) {
      const int ow = static_cast<int>(r % Wo);
      const long long t = r / Wo;
      const int oh = static_cast<int>(t % Ho);
      const long long b = t / Ho;
      const int ih = oh * S - K / 2 + kh;
      if (ih < 0 || ih >= H) continue;
      float g[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(dd + r * C) + cg), g);
#pragma unroll
      for (int kw = 0; kw < K; ++kw) {
        const int iw = ow * S - K / 2 + kw;
        if (iw < 0 || iw >= W) continue;
        float v[8];
        dw_load_in<PRE>(x, (b * H + ih) * W + iw, C, cg, sc, sh, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[kw][j] = fmaf(g[j], v[j], acc[kw][j]);
      }
    }
  }
  if (rv_cta_reduce<K>(acc, 8, kDwLanes, lane_g, rsub) && live) {
#pragma unroll
    for (int kw = 0; kw < K; ++kw)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        ws[(static_cast<long long>(blockIdx.x) * K * K + kh * K + kw) * C + cg * 8 + j] = acc[kw][j];
  }
}

// dw[c][tap] = sum_t ws[t][tap][c] in a fixed order: a CTA owns 32 consecutive (tap, c) outputs; its 8 slab lanes sum the
// slabs t = j, j + 8, ... in ascending order, and the 8 lane sums are added in lane order.
constexpr int kDwRedLanes = 8;

__global__ void __launch_bounds__(256) dw_wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, int T,
                                                              int taps, int C) {
  __shared__ float red[kDwRedLanes][32];
  pdl_wait();
  const long long n = static_cast<long long>(taps) * C;
  const int lane = threadIdx.x % 32, j = threadIdx.x / 32;
  const long long i = blockIdx.x * 32ll + lane;
  float s = 0.f;
  if (i < n)
    for (int t = j; t < T; t += kDwRedLanes) s += ws[static_cast<long long>(t) * n + i];
  red[j][lane] = s;
  __syncthreads();
  if (j == 0 && i < n) {
    for (int q = 1; q < kDwRedLanes; ++q) s += red[q][lane];
    const int tap = static_cast<int>(i / C), c = static_cast<int>(i % C);
    dw[static_cast<long long>(c) * taps + tap] = s;
  }
}

// --------------------------------------------------------------------------------------------------- per-image sums
// grid (B, nchunk) of the row geometry over one image's HW pixels.  GATE == false (squeeze): pool[b][c] = mean_p
// silu(u), u = d sc + sh, and with a mask out16[b][c] = bf16(pool mask); GATE (gate reduce): s[b][c] = sum_p da silu(u).
template <bool GATE, bool MASK>
__global__ void __launch_bounds__(256) mb_image_sum_kernel(const uint4* __restrict__ da, const uint4* __restrict__ d,
                                                           const float* __restrict__ scale, const float* __restrict__ shift,
                                                           const float* __restrict__ mask, float* __restrict__ out,
                                                           __nv_bfloat16* __restrict__ out16, int HW, int C, int gpc) {
  pdl_wait();
  const int cvec = C / 8, rpi = 256 / gpc;
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;
  const int cg = blockIdx.y * gpc + lane_g;
  const bool live = rsub < rpi && cg < cvec;
  const long long b = blockIdx.x;
  float acc[1][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = 0.f;
  if (live) {
    float sc[8], sh[8];
    load8f(scale + cg * 8, sc);
    load8f(shift + cg * 8, sh);
    for (int p = rsub; p < HW; p += rpi) {
      const long long r = b * HW + p;
      float v[8];
      unpack8(__ldg(d + r * cvec + cg), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = mb_silu(fmaf(v[j], sc[j], sh[j]));
      if constexpr (GATE) {
        float g[8];
        unpack8(__ldg(da + r * cvec + cg), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[0][j] = fmaf(g[j], v[j], acc[0][j]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[0][j] += v[j];
      }
    }
  }
  if (rv_cta_reduce<1>(acc, gpc, rpi, lane_g, rsub) && live) {
    const float inv = GATE ? 1.f : 1.f / static_cast<float>(HW);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const long long i = b * C + cg * 8 + j;
      const float v = acc[0][j] * inv;
      out[i] = v;
      if constexpr (MASK) out16[i] = __float2bfloat16_rn(v * mask[i]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------ excite
// One CTA per image: hpre = W1 pool + b1 [Cr] (one warp per output, fixed shuffle order), gate = sigmoid(W2 silu(hpre) + b2).
__global__ void __launch_bounds__(256) mb_excite_fwd_kernel(const float* __restrict__ pool, const float* __restrict__ w1,
                                                            const float* __restrict__ b1, const float* __restrict__ w2,
                                                            const float* __restrict__ b2, float* __restrict__ hpre,
                                                            float* __restrict__ gate, int C, int Cr) {
  extern __shared__ float mb_sm[];
  float* p = mb_sm;
  float* h = mb_sm + C;
  pdl_wait();
  const long long b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += 256) p[c] = pool[b * C + c];
  __syncthreads();
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  for (int r = warp; r < Cr; r += 8) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(w1[static_cast<long long>(r) * C + c], p[c], s);
    s = warp_sum(s) + b1[r];
    if (lane == 0) {
      hpre[b * Cr + r] = s;
      h[r] = mb_silu(s);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    float s = b2[c];
    for (int r = 0; r < Cr; ++r) s = fmaf(w2[static_cast<long long>(c) * Cr + r], h[r], s);
    gate[b * C + c] = mb_sigmoid(s);
  }
}

// One CTA per image: dgp = S gate (1 - gate) [C] (gradient of the W2 output), dhp = (dgp W2) silu'(hpre) [Cr].
__global__ void __launch_bounds__(256) mb_excite_bwd_image_kernel(const float* __restrict__ S, const float* __restrict__ gate,
                                                                  const float* __restrict__ hpre, const float* __restrict__ w2,
                                                                  float* __restrict__ dgp, float* __restrict__ dhp, int C,
                                                                  int Cr) {
  extern __shared__ float mb_sm[];
  pdl_wait();
  const long long b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float g = gate[b * C + c];
    const float v = S[b * C + c] * g * (1.f - g);
    mb_sm[c] = v;
    dgp[b * C + c] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  for (int r = warp; r < Cr; r += 8) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(mb_sm[c], w2[static_cast<long long>(c) * Cr + r], s);
    s = warp_sum(s);
    if (lane == 0) dhp[b * Cr + r] = s * mb_dsilu(hpre[b * Cr + r]);
  }
}

// Sums over the batch (b ascending) and over Cr: one thread per output of
//   dW2[c][r] = sum_b dgp[b][c] silu(hpre[b][r]),  db2[c] = sum_b dgp[b][c],
//   dW1[r][c] = sum_b dhp[b][r] pool[b][c],        db1[r] = sum_b dhp[b][r],
//   dpool[b][c] = sum_r dhp[b][r] W1[r][c]
__global__ void __launch_bounds__(256) mb_excite_bwd_params_kernel(
    const float* __restrict__ dgp, const float* __restrict__ dhp, const float* __restrict__ hpre,
    const float* __restrict__ pool, const float* __restrict__ w1, float* __restrict__ dw1, float* __restrict__ db1,
    float* __restrict__ dw2, float* __restrict__ db2, float* __restrict__ dpool, int B, int C, int Cr) {
  pdl_wait();
  const long long n_w = static_cast<long long>(C) * Cr;
  const long long total = 2 * n_w + C + Cr + static_cast<long long>(B) * C;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * 256) {
    float s = 0.f;
    if (i < n_w) {
      const int c = static_cast<int>(i / Cr), r = static_cast<int>(i % Cr);
      for (int b = 0; b < B; ++b)
        s = fmaf(dgp[static_cast<long long>(b) * C + c], mb_silu(hpre[static_cast<long long>(b) * Cr + r]), s);
      dw2[i] = s;
    } else if (i < 2 * n_w) {
      const long long k = i - n_w;
      const int r = static_cast<int>(k / C), c = static_cast<int>(k % C);
      for (int b = 0; b < B; ++b)
        s = fmaf(dhp[static_cast<long long>(b) * Cr + r], pool[static_cast<long long>(b) * C + c], s);
      dw1[k] = s;
    } else if (i < 2 * n_w + C) {
      const int c = static_cast<int>(i - 2 * n_w);
      for (int b = 0; b < B; ++b) s += dgp[static_cast<long long>(b) * C + c];
      db2[c] = s;
    } else if (i < 2 * n_w + C + Cr) {
      const int r = static_cast<int>(i - 2 * n_w - C);
      for (int b = 0; b < B; ++b) s += dhp[static_cast<long long>(b) * Cr + r];
      db1[r] = s;
    } else {
      const long long k = i - 2 * n_w - C - Cr;
      const long long b = k / C;
      const int c = static_cast<int>(k % C);
      for (int r = 0; r < Cr; ++r) s = fmaf(dhp[b * Cr + r], w1[static_cast<long long>(r) * C + c], s);
      dpool[k] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------------ streaming passes
// Row r of a [B][HW][C] tensor belongs to image r / HW.
#define MB_ROWS_PROLOGUE                                                          \
  const int cvec = C / 8, rpi = 256 / gpc;                                        \
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;                 \
  const int cg = blockIdx.y * gpc + lane_g;                                       \
  const bool live = rsub < rpi && cg < cvec;                                      \
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;       \
  const long long r1 = min(rows, r0 + rows_per_block)

// GATE: a = silu(d sc + sh) gate[b][c];  else (tail): y = (d sc + sh) rs[b] (+ residual), rs optional
template <bool GATE, bool RS, bool RES>
__global__ void __launch_bounds__(256) mb_apply_kernel(const uint4* __restrict__ d, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, const float* __restrict__ vec,
                                                       const uint4* __restrict__ res, uint4* __restrict__ y, long long rows,
                                                       int HW, int C, int rows_per_block, int gpc) {
  pdl_wait();
  MB_ROWS_PROLOGUE;
  if (!live) return;
  float sc[8], sh[8];
  load8f(scale + cg * 8, sc);
  load8f(shift + cg * 8, sh);
  for (long long r = r0 + rsub; r < r1; r += rpi) {
    const long long b = r / HW;
    float v[8];
    unpack8(__ldg(d + r * cvec + cg), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = fmaf(v[j], sc[j], sh[j]);
    if constexpr (GATE) {
      float g[8];
      load8f(vec + b * C + cg * 8, g);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = mb_silu(v[j]) * g[j];
    } else {
      if constexpr (RS) {
        const float s = __ldg(vec + b);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] *= s;
      }
      if constexpr (RES) {
        float x[8];
        unpack8(__ldg(res + r * cvec + cg), x);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += x[j];
      }
    }
    y[r * cvec + cg] = pack8(v);
  }
}

// Backward reduces; dz (stored bf16 when dz != nullptr) and partial [T][2][C] = {sum dz, sum dz c} of the stored values.
//   SILU == false (tail):  dz = g rs[b]  (RS; else dz = g, not stored)              g = dL/dy, c = c_p
//   SILU (SiLU-BN):        dz = (da gate[b][c] (DA) + dpool[b][c] / HW) silu'(c sc + sh)   c = d
template <bool SILU, bool OPT>
__global__ void __launch_bounds__(256, 2) mb_bwd_reduce_kernel(
    const uint4* __restrict__ g, const float* __restrict__ vec, const float* __restrict__ dpool,
    const uint4* __restrict__ c, const float* __restrict__ scale, const float* __restrict__ shift, uint4* __restrict__ dz,
    float* __restrict__ partial, long long rows, int HW, int C, int rows_per_block, int gpc) {
  pdl_wait();
  MB_ROWS_PROLOGUE;
  float acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
  if (live) {
    float sc[8], sh[8];
    if constexpr (SILU) {
      load8f(scale + cg * 8, sc);
      load8f(shift + cg * 8, sh);
    }
    const float inv_hw = 1.f / static_cast<float>(HW);
    for (long long r = r0 + rsub; r < r1; r += rpi) {
      const long long b = r / HW;
      float v[8], cv[8];
      unpack8(__ldg(c + r * cvec + cg), cv);
      if constexpr (SILU) {
        float dp[8];
        load8f(dpool + b * C + cg * 8, dp);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = dp[j] * inv_hw;
        if constexpr (OPT) {
          float a[8], gt[8];
          unpack8(__ldg(g + r * cvec + cg), a);
          load8f(vec + b * C + cg * 8, gt);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = fmaf(a[j], gt[j], v[j]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] *= mb_dsilu(fmaf(cv[j], sc[j], sh[j]));
      } else {
        unpack8(__ldg(g + r * cvec + cg), v);
        if constexpr (OPT) {
          const float s = __ldg(vec + b);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] *= s;
        }
      }
      if (SILU || OPT) {
        const uint4 q = pack8(v);
        dz[r * cvec + cg] = q;
        unpack8(q, v);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[0][j] += v[j];
        acc[1][j] = fmaf(v[j], cv[j], acc[1][j]);
      }
    }
  }
  if (rv_cta_reduce<2>(acc, gpc, rpi, lane_g, rsub) && live) {
    float* p = partial + static_cast<long long>(blockIdx.x) * 2 * C + cg * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      p[j] = acc[0][j];
      p[C + j] = acc[1][j];
    }
  }
}

#undef MB_ROWS_PROLOGUE

}  // namespace b200
