// Block tails of ShuffleNet v1 (classification/ShuffleNet/models/shufflenetv1.py ResidualBlock:61-82):
//
//   stride 2, forward   y[..., :Cin] = relu(avg_pool3x3/2/p1(x))      (count_include_pad: always / 9)
//                       y[..., Cin:] = relu(c3 * s3 + t3)             the concatenated output, written once
//   backward            conv half  dz = g [y > 0] over y's last Cc channels, stored, with {sum dz, sum dz c3}
//                       pool half  gx[b][ih][iw][c] = sum over the (at most 2x2) pooled outputs whose window reads
//                                  (ih, iw) of g [y > 0], / 9, in (oh, ow) ascending order (c < Cin)
//   stride 1, backward  dz = g [y > 0] with {sum dz, sum dz c3}: bn3's input gradient and the shortcut gradient at once
//   stem, backward      dz = g [c s + t > 0] with {sum dz, sum dz c}: the stem BatchNorm + ReLU behind the max-pool
//
// The stride-1 tail forward is b200_bn_apply (residual + ReLU); the depthwise convolution with bn1 + ReLU applied on load is
// the kDwRelu mode of mbconv.cuh's dw_* kernels.  The reduces use the row geometry of row_passes.cuh over the conv half
// (repvgg_geom(rows, Cc)), so they write b200_repvgg_partial_rows(rows, Cc) partial rows.
//
// The ShuffleNet v2 tails (shufflev2_tail_*) follow below.
#pragma once
#include "row_passes.cuh"

namespace b200 {

// One thread per 8-channel vector of y [B][Ho][Wo][Cin + Cc]; grid-stride.
__global__ void __launch_bounds__(256, 1) shuffle_tail_s2_fwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ c3,
                                                                  const float* __restrict__ scale,
                                                                  const float* __restrict__ shift, uint4* __restrict__ y,
                                                                  int B, int H, int W, int Ho, int Wo, int Cin, int Cc) {
  pdl_wait();
  const int vin = Cin / 8, vc = Cc / 8, vt = vin + vc;
  const long long n = static_cast<long long>(B) * Ho * Wo * vt;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    const int v = static_cast<int>(i % vt);
    const long long r = i / vt;
    float o[8];
    if (v < vin) {
      const int ow = static_cast<int>(r % Wo);
      const long long t = r / Wo;
      const int oh = static_cast<int>(t % Ho);
      const long long b = t / Ho;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = 0.f;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int ih = oh * 2 - 1 + kh;
        if (ih < 0 || ih >= H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int iw = ow * 2 - 1 + kw;
          if (iw < 0 || iw >= W) continue;
          float xv[8];
          unpack8(__ldg(x + ((b * H + ih) * W + iw) * vin + v), xv);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += xv[j];
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaxf(o[j] * (1.f / 9.f), 0.f);
    } else {
      const int cv = v - vin;
      float sc[8], sh[8];
      load8f(scale + cv * 8, sc);
      load8f(shift + cv * 8, sh);
      unpack8(__ldg(c3 + r * vc + cv), o);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaxf(fmaf(o[j], sc[j], sh[j]), 0.f);
    }
    y[i] = pack8(o);
  }
}

// blockIdx.z == 0: the reduce over the conv half, grid (blocks, nchunk) of repvgg_geom(B Ho Wo, Cc).
//   MASK_Y:  dz = g[r][Cin + c] [y[r][Cin + c] > 0] (g and y of row pitch Cin + Cc)
//   else:    dz = g[r][c] [c[r][c] scale + shift > 0] (g of row pitch Cc, Cin == 0)
// blockIdx.z == 1 (POOL only): the pool half, every CTA of the grid striding over the vectors of gx [B][H][W][Cin].
template <bool MASK_Y, bool POOL>
__global__ void __launch_bounds__(256, 2) shuffle_relu_bwd_kernel(
    const uint4* __restrict__ g, const uint4* __restrict__ y, const uint4* __restrict__ c, const float* __restrict__ scale,
    const float* __restrict__ shift, uint4* __restrict__ dz, float* __restrict__ partial, uint4* __restrict__ gx, int B,
    int H, int W, int Ho, int Wo, int Cin, int Cc, int rows_per_block, int gpc) {
  pdl_wait();
  const int vin = Cin / 8, vc = Cc / 8, vt = vin + vc;
  if constexpr (POOL) {
    if (blockIdx.z == 1) {
      const long long n = static_cast<long long>(B) * H * W * vin;
      const long long cta = static_cast<long long>(blockIdx.y) * gridDim.x + blockIdx.x;
      const long long stride = static_cast<long long>(gridDim.x) * gridDim.y * 256;
      for (long long i = cta * 256 + threadIdx.x; i < n; i += stride) {
        const int v = static_cast<int>(i % vin);
        const long long p = i / vin;
        const int iw = static_cast<int>(p % W);
        const long long t = p / W;
        const int ih = static_cast<int>(t % H);
        const long long b = t / H;
        // output oh reads rows 2 oh - 1 .. 2 oh + 1: an even row has one reader, an odd row two
        const int oh0 = (ih + 1) / 2 - ((ih & 1) ? 1 : 0), oh1 = min((ih + 1) / 2, Ho - 1);
        const int ow0 = (iw + 1) / 2 - ((iw & 1) ? 1 : 0), ow1 = min((iw + 1) / 2, Wo - 1);
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = 0.f;
        for (int oh = oh0; oh <= oh1; ++oh)
          for (int ow = ow0; ow <= ow1; ++ow) {
            const long long q = ((b * Ho + oh) * Wo + ow) * vt + v;
            float gv[8], yv[8];
            unpack8(__ldg(g + q), gv);
            unpack8(__ldg(y + q), yv);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] += yv[j] > 0.f ? gv[j] : 0.f;
          }
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] *= 1.f / 9.f;
        gx[i] = pack8(o);
      }
      return;
    }
  }
  const long long rows = static_cast<long long>(B) * Ho * Wo;
  const int cvec = vc, rpi = 256 / gpc;
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;
  const int cg = blockIdx.y * gpc + lane_g;
  const bool live = rsub < rpi && cg < cvec;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  float acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
  if (live) {
    float sc[8], sh[8];
    if constexpr (!MASK_Y) {
      load8f(scale + cg * 8, sc);
      load8f(shift + cg * 8, sh);
    }
    for (long long r = r0 + rsub; r < r1; r += rpi) {
      float v[8], cv[8];
      unpack8(__ldg(c + r * vc + cg), cv);
      unpack8(__ldg(g + r * vt + vin + cg), v);
      if constexpr (MASK_Y) {
        float yv[8];
        unpack8(__ldg(y + r * vt + vin + cg), yv);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = yv[j] > 0.f ? v[j] : 0.f;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaf(cv[j], sc[j], sh[j]) > 0.f ? v[j] : 0.f;
      }
      const uint4 q = pack8(v);
      dz[r * vc + cg] = q;
      unpack8(q, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[0][j] += v[j];
        acc[1][j] = fmaf(v[j], cv[j], acc[1][j]);
      }
    }
  }
  if (rv_cta_reduce<2>(acc, gpc, rpi, lane_g, rsub) && live) {
    float* p = partial + static_cast<long long>(blockIdx.x) * 2 * Cc + cg * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      p[j] = acc[0][j];
      p[Cc + j] = acc[1][j];
    }
  }
}

// ---- ShuffleNet v2 block tails (classification/ShuffleNet/models/shufflenetv2.py InvertedResidual:
//   out = channel_shuffle(cat(u, v), 2),  v = relu(c3 s3 + t3)  (branch2's last BatchNorm + ReLU),
//   u = the passthrough half x1 (stride 1)  or  relu(cu su + tu)  (branch1's BatchNorm + ReLU, stride 2).
// The two-group shuffle of cat(u, v) is an interleave, out[2 i] = u[i], out[2 i + 1] = v[i] (i < b), so
//   joined  out [rows][jp]               channels 0 .. 2b - 1 in reference order, jp - 2b pad channels
//   split   P' [rows][bp] = out[:b],  Q' [rows][bp] = out[b:2b]   (the chunk(2) halves of the next stride-1 block)
// u, c3, cu and the backward outputs are [rows][bp] with pad channels b .. bp - 1.  Every pad channel written is exactly 0.
// Q' starts at source channel b / 2, which need not be a multiple of 4 (b = 58: 29), so its sources are read from any
// element offset.

// four consecutive values from any element offset
__device__ __forceinline__ void ld4_bf16(const __nv_bfloat16* __restrict__ p, float (&f)[4]) {
  if ((reinterpret_cast<uintptr_t>(p) & 7) == 0) {
    const uint2 w = __ldg(reinterpret_cast<const uint2*>(p));
    f[0] = bf16_lo(w.x);
    f[1] = bf16_hi(w.x);
    f[2] = bf16_lo(w.y);
    f[3] = bf16_hi(w.y);
  } else {
    const unsigned short* q = reinterpret_cast<const unsigned short*>(p);
#pragma unroll
    for (int j = 0; j < 4; ++j) f[j] = __uint_as_float(static_cast<uint32_t>(__ldg(q + j)) << 16);
  }
}
__device__ __forceinline__ void ld4_f32(const float* __restrict__ p, float (&f)[4]) {
  if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p));
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) f[j] = __ldg(p + j);
  }
}

// One thread per 8-channel output vector (logical channels k0 .. k0 + 7 of out, reading source channels k0 / 2 .. + 3);
// grid-stride.  SPLIT: vectors [0, bp / 8) of a row are P', the rest Q'.
template <bool BN_U, bool SPLIT>
__global__ void __launch_bounds__(256) shufflev2_tail_fwd_kernel(
    const __nv_bfloat16* __restrict__ u, const float* __restrict__ su, const float* __restrict__ tu,
    const __nv_bfloat16* __restrict__ c3, const float* __restrict__ s3, const float* __restrict__ t3, uint4* __restrict__ y0,
    uint4* __restrict__ y1, long long rows, int b, int bp, int jp) {
  pdl_wait();
  const int vh = bp / 8;
  const int vt = SPLIT ? 2 * vh : jp / 8;
  const long long n = rows * vt;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    const int v = static_cast<int>(i % vt);
    const long long r = i / vt;
    int k0, lim;
    uint4* dst;
    if constexpr (SPLIT) {
      const bool hi = v >= vh;
      const int w = hi ? v - vh : v;
      k0 = (hi ? b : 0) + 8 * w;
      lim = hi ? 2 * b : b;
      dst = (hi ? y1 : y0) + r * vh + w;
    } else {
      k0 = 8 * v;
      lim = 2 * b;
      dst = y0 + r * vt + v;
    }
    float o[8];
    if (k0 >= lim) {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = 0.f;
    } else {
      const int s = k0 / 2;
      float uf[4], cf[4], sc[4], sh[4];
      ld4_bf16(u + r * bp + s, uf);
      ld4_bf16(c3 + r * bp + s, cf);
      ld4_f32(s3 + s, sc);
      ld4_f32(t3 + s, sh);
      if constexpr (BN_U) {
        float a[4], c[4];
        ld4_f32(su + s, a);
        ld4_f32(tu + s, c);
#pragma unroll
        for (int j = 0; j < 4; ++j) uf[j] = fmaxf(fmaf(uf[j], a[j], c[j]), 0.f);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        o[2 * j] = uf[j];
        o[2 * j + 1] = fmaxf(fmaf(cf[j], sc[j], sh[j]), 0.f);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (k0 + j >= lim) o[j] = 0.f;
    }
    *dst = pack8(o);
  }
}

// Backward of shufflev2_tail_fwd over the row geometry of repvgg_geom(rows, bp): a thread owns source channels
// i0 .. i0 + 7 (i0 = 8 cg) and reads the gradient pairs (dL/du[i], dL/dv[i]) = the 32-bit word at logical channel 2 i of the
// output gradient (g0 joined, or g0 = dL/dP', g1 = dL/dQ' split: word 2 i of P' for i < b / 2, else word 2 i - b of Q').
//   dz3 = dL/dv [c3 s3 + t3 > 0] with {sum dz3, sum dz3 c3} -> part3
//   BN_U:  du = dL/du [cu su + tu > 0] with {sum du, sum du cu} -> partu;  else du = dL/du (the passthrough gradient)
template <bool BN_U, bool SPLIT>
__global__ void __launch_bounds__(256, 2) shufflev2_tail_bwd_kernel(
    const __nv_bfloat16* __restrict__ g0, const __nv_bfloat16* __restrict__ g1, const uint4* __restrict__ c3,
    const float* __restrict__ s3, const float* __restrict__ t3, uint4* __restrict__ dz3, float* __restrict__ part3,
    const uint4* __restrict__ cu, const float* __restrict__ su, const float* __restrict__ tu, uint4* __restrict__ du,
    float* __restrict__ partu, long long rows, int b, int bp, int jp, int rows_per_block, int gpc) {
  pdl_wait();
  constexpr int NS = BN_U ? 4 : 2;
  const int cvec = bp / 8, rpi = 256 / gpc;
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;
  const int cg = blockIdx.y * gpc + lane_g;
  const bool live = rsub < rpi && cg < cvec;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  float acc[NS][8];
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[s][j] = 0.f;
  if (live) {
    const int i0 = cg * 8, h = b / 2;
    const long long ld = SPLIT ? bp : jp;
    // all eight words in one tensor at a 16-byte aligned column: two vector loads per row
    const bool in_q = SPLIT && i0 >= h;
    const __nv_bfloat16* fsrc = in_q ? g1 : g0;
    const int fcol = in_q ? 2 * i0 - b : 2 * i0;
    const bool fast = i0 + 8 <= b && (!SPLIT || i0 + 8 <= h || (in_q && (fcol & 7) == 0));
    float sc3[8], sh3[8], scu[8], shu[8];
    load8f(s3 + i0, sc3);
    load8f(t3 + i0, sh3);
    if constexpr (BN_U) {
      load8f(su + i0, scu);
      load8f(tu + i0, shu);
    }
    for (long long r = r0 + rsub; r < r1; r += rpi) {
      uint32_t w[8];
      if (fast) {
        const uint4* p = reinterpret_cast<const uint4*>(fsrc + r * ld + fcol);
        const uint4 a = __ldg(p), c = __ldg(p + 1);
        w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
        w[4] = c.x; w[5] = c.y; w[6] = c.z; w[7] = c.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int i = i0 + j;
          w[j] = 0u;
          if (i < b) {
            const __nv_bfloat16* q = (SPLIT && i >= h) ? g1 + r * ld + (2 * i - b) : g0 + r * ld + 2 * i;
            w[j] = __ldg(reinterpret_cast<const uint32_t*>(q));
          }
        }
      }
      const long long e = r * cvec + cg;
      float cv[8], z[8];
      unpack8(__ldg(c3 + e), cv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        z[j] = fmaf(cv[j], sc3[j], sh3[j]) > 0.f ? bf16_hi(w[j]) : 0.f;
        acc[0][j] += z[j];
        acc[1][j] = fmaf(z[j], cv[j], acc[1][j]);
      }
      dz3[e] = pack8(z);
      if constexpr (BN_U) {
        float uv[8];
        unpack8(__ldg(cu + e), uv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          z[j] = fmaf(uv[j], scu[j], shu[j]) > 0.f ? bf16_lo(w[j]) : 0.f;
          acc[NS - 2][j] += z[j];
          acc[NS - 1][j] = fmaf(z[j], uv[j], acc[NS - 1][j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) z[j] = bf16_lo(w[j]);
      }
      du[e] = pack8(z);
    }
  }
  if (rv_cta_reduce<NS>(acc, gpc, rpi, lane_g, rsub) && live) {
    float* p = part3 + static_cast<long long>(blockIdx.x) * 2 * bp + cg * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      p[j] = acc[0][j];
      p[bp + j] = acc[1][j];
    }
    if constexpr (BN_U) {
      float* q = partu + static_cast<long long>(blockIdx.x) * 2 * bp + cg * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        q[j] = acc[NS - 2][j];
        q[bp + j] = acc[NS - 1][j];
      }
    }
  }
}

}  // namespace b200
