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

}  // namespace b200
