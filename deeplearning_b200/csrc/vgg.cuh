// Passes of the VGG schedule (classification/vggNet/models/network.py) that the convolution GEMMs do not cover:
// 2x2 / stride-2 max-pooling with the ReLU (plain variants) or BatchNorm + ReLU (_bn variants) folded in, its backward with
// the activation mask and the BatchNorm-backward partial sums, AdaptiveAvgPool2d((7, 7)) + torch.flatten, the classifier's
// dropout, and torch.optim.Adam's update (L2 decay added to the gradient, not AdamW's decoupled decay).
//
// Activations are NHWC bf16 moved as 16-byte vectors of 8 channels; sums are fp32 in a fixed order (no atomics).
#pragma once
#include "row_passes.cuh"

namespace b200 {

// MaxPool2d(2, 2) (floor mode) of v = x (plain: x is already relu(conv + b)) or v = relu(x * scale + shift) (BN: x is the
// raw convolution output).  Ties go to the first maximum in row-major window order, as torch's kernels resolve them.
// idx (optional): one byte per element, the window tap 0..3 of the maximum.
template <bool BN>
__global__ void __launch_bounds__(256) vgg_pool_fwd_kernel(const uint4* __restrict__ x, const float* __restrict__ scale,
                                                           const float* __restrict__ shift, uint4* __restrict__ y,
                                                           uint2* __restrict__ idx, int B, int H, int W, int cvec) {
  pdl_wait();
  const int Ho = H / 2, Wo = W / 2;
  const long long n = static_cast<long long>(B) * Ho * Wo * cvec;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % cvec);
    long long t = i / cvec;
    const int ow = static_cast<int>(t % Wo);
    t /= Wo;
    const int oh = static_cast<int>(t % Ho);
    const long long b = t / Ho;
    const long long base = ((b * H + 2 * oh) * W + 2 * ow) * cvec + cg;
    const long long off[4] = {0, cvec, static_cast<long long>(W) * cvec, static_cast<long long>(W + 1) * cvec};
    float sc[8], sh[8];
    if constexpr (BN) {
      load8f(scale + cg * 8, sc);
      load8f(shift + cg * 8, sh);
    }
    float best[8];
    uint32_t bi[2] = {0u, 0u};
#pragma unroll
    for (int tap = 0; tap < 4; ++tap) {
      float f[8];
      unpack8(__ldg(x + base + off[tap]), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if constexpr (BN) f[j] = fmaxf(fmaf(f[j], sc[j], sh[j]), 0.f);
        if (tap == 0) {
          best[j] = f[j];
        } else if (f[j] > best[j]) {
          best[j] = f[j];
          bi[j >> 2] = (bi[j >> 2] & ~(0xFFu << (8 * (j & 3)))) | (static_cast<uint32_t>(tap) << (8 * (j & 3)));
        }
      }
    }
    y[i] = pack8(best);
    if (idx != nullptr) idx[i] = make_uint2(bi[0], bi[1]);
  }
}

// Backward of vgg_pool_fwd over the 2x2 blocks of the input (rows = B * ceil(H/2) * ceil(W/2), the RepVGG row geometry):
// the pooled gradient goes to the arg-max pixel of its window when the activation there was positive, every other pixel
// (including the last row / column of an odd H / W, which no window covers) gets 0.
//   plain: alive iff the pooled output y > 0 (it IS the ReLU output at the arg-max)
//   BN:    alive iff c * scale + shift > 0 at the arg-max; partial [blockIdx.x][2][C] = {sum dz, sum dz c} of the stored bf16
//          dz, the rows b200_bn_bwd_finalize reads
template <bool BN>
__global__ void __launch_bounds__(256) vgg_pool_bwd_kernel(const uint4* __restrict__ g, const uint2* __restrict__ idx,
                                                           const uint4* __restrict__ y, const uint4* __restrict__ c,
                                                           const float* __restrict__ scale, const float* __restrict__ shift,
                                                           uint4* __restrict__ dx, float* __restrict__ partial, int B, int H,
                                                           int W, int C, int rows_per_block, int gpc) {
  pdl_wait();
  const int cvec = C / 8, rpi = 256 / gpc;
  const int lane_g = threadIdx.x % gpc, rsub = threadIdx.x / gpc;
  const int cg = blockIdx.y * gpc + lane_g;
  const bool live = rsub < rpi && cg < cvec;
  const int Ho = H / 2, Wo = W / 2, Hb = (H + 1) / 2, Wb = (W + 1) / 2;
  const long long rows = static_cast<long long>(B) * Hb * Wb;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  float acc[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
  if (live) {
    float sc[8], sh[8];
    if constexpr (BN) {
      load8f(scale + cg * 8, sc);
      load8f(shift + cg * 8, sh);
    }
    for (long long r = r0 + rsub; r < r1; r += rpi) {
      const int bw = static_cast<int>(r % Wb);
      const long long t = r / Wb;
      const int ah = static_cast<int>(t % Hb);
      const long long b = t / Hb;
      const bool win = ah < Ho && bw < Wo;
      float gv[8];
      uint32_t tp[2] = {0xFFFFFFFFu, 0xFFFFFFFFu};   // tap 255: matches no pixel
      if (win) {
        const long long o = ((b * Ho + ah) * Wo + bw) * cvec + cg;
        unpack8(__ldg(g + o), gv);
        const uint2 q = __ldg(idx + o);
        tp[0] = q.x, tp[1] = q.y;
        if constexpr (!BN) {
          const uint4 yv = __ldg(y + o);
          const uint32_t w[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if ((w[k] & 0x7fffu) == 0u) gv[2 * k] = 0.f;
            if ((w[k] & 0x7fff0000u) == 0u) gv[2 * k + 1] = 0.f;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) gv[j] = 0.f;
      }
#pragma unroll
      for (int tap = 0; tap < 4; ++tap) {
        const int ih = 2 * ah + (tap >> 1), iw = 2 * bw + (tap & 1);
        if (ih >= H || iw >= W) continue;
        const long long pix = ((b * H + ih) * W + iw) * cvec + cg;
        float v[8], cv[8];
        if constexpr (BN) unpack8(__ldg(c + pix), cv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const bool hit = ((tp[j >> 2] >> (8 * (j & 3))) & 0xFFu) == static_cast<uint32_t>(tap);
          bool alive = hit;
          if constexpr (BN) alive = alive && fmaf(cv[j], sc[j], sh[j]) > 0.f;
          v[j] = alive ? gv[j] : 0.f;
        }
        const uint4 q = pack8(v);
        dx[pix] = q;
        if constexpr (BN) {
          unpack8(q, v);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            acc[0][j] += v[j];
            acc[1][j] = fmaf(v[j], cv[j], acc[1][j]);
          }
        }
      }
    }
  }
  if constexpr (BN) {
    if (rv_cta_reduce<2>(acc, gpc, rpi, lane_g, rsub) && live) {
      float* p = partial + static_cast<long long>(blockIdx.x) * 2 * C + cg * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        p[j] = acc[0][j];
        p[C + j] = acc[1][j];
      }
    }
  }
}

// AdaptiveAvgPool2d((7, 7)) bins: rows floor(i H / 7) .. ceil((i + 1) H / 7) - 1
__device__ __forceinline__ int vgg_bin_lo(int i, int n) { return (i * n) / 7; }
__device__ __forceinline__ int vgg_bin_hi(int i, int n) { return ((i + 1) * n + 6) / 7; }

constexpr int kVggPoolChans = 64;   // channels per CTA of the adaptive pool: 64 * 49 contiguous outputs

// y bf16 [B][C * 49] with k = c * 49 + i * 7 + j (torch.flatten of the NCHW [B][C][7][7] pool), from x [B][H][W][C].
// grid (B, C / 64); every thread sums the bins of 8 channels with 16-byte loads, the CTA writes its 3136 outputs contiguously.
__global__ void __launch_bounds__(256) vgg_avgpool7_fwd_kernel(const uint4* __restrict__ x, uint32_t* __restrict__ y, int H,
                                                               int W, int C) {
  pdl_wait();
  __shared__ float s[kVggPoolChans * 49];
  const int cvec = C / 8, b = blockIdx.x, cg0 = blockIdx.y * (kVggPoolChans / 8);
  for (int it = threadIdx.x; it < (kVggPoolChans / 8) * 49; it += blockDim.x) {
    const int cgl = it % (kVggPoolChans / 8), bin = it / (kVggPoolChans / 8);
    const int i = bin / 7, j = bin % 7;
    const int h0 = vgg_bin_lo(i, H), h1 = vgg_bin_hi(i, H), w0 = vgg_bin_lo(j, W), w1 = vgg_bin_hi(j, W);
    float a[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) a[q] = 0.f;
    for (int h = h0; h < h1; ++h)
      for (int w = w0; w < w1; ++w) {
        float f[8];
        unpack8(__ldg(x + ((static_cast<long long>(b) * H + h) * W + w) * cvec + cg0 + cgl), f);
#pragma unroll
        for (int q = 0; q < 8; ++q) a[q] += f[q];
      }
    const float cnt = static_cast<float>((h1 - h0) * (w1 - w0));
#pragma unroll
    for (int q = 0; q < 8; ++q) s[(cgl * 8 + q) * 49 + bin] = a[q] / cnt;
  }
  __syncthreads();
  uint32_t* out = y + (static_cast<long long>(b) * C * 49 + static_cast<long long>(blockIdx.y) * kVggPoolChans * 49) / 2;
  for (int k = threadIdx.x; k < kVggPoolChans * 49 / 2; k += blockDim.x) out[k] = pack_bf16x2(s[2 * k], s[2 * k + 1]);
}

// gx [B][H][W][C] = sum over the bins that contain the pixel of gy[b][c * 49 + bin] / |bin|; grid (B, C / 64)
__global__ void __launch_bounds__(256) vgg_avgpool7_bwd_kernel(const uint32_t* __restrict__ gy, uint4* __restrict__ gx,
                                                               int H, int W, int C) {
  pdl_wait();
  __shared__ float s[kVggPoolChans * 49];
  const int cvec = C / 8, b = blockIdx.x, cg0 = blockIdx.y * (kVggPoolChans / 8);
  const uint32_t* in = gy + (static_cast<long long>(b) * C * 49 + static_cast<long long>(blockIdx.y) * kVggPoolChans * 49) / 2;
  for (int k = threadIdx.x; k < kVggPoolChans * 49 / 2; k += blockDim.x) {
    const uint32_t v = __ldg(in + k);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int bin = (2 * k + h) % 49, i = bin / 7, j = bin % 7;
      const float cnt = static_cast<float>((vgg_bin_hi(i, H) - vgg_bin_lo(i, H)) * (vgg_bin_hi(j, W) - vgg_bin_lo(j, W)));
      s[2 * k + h] = (h ? bf16_hi(v) : bf16_lo(v)) / cnt;
    }
  }
  __syncthreads();
  const int items = H * W * (kVggPoolChans / 8);
  for (int it = threadIdx.x; it < items; it += blockDim.x) {
    const int cgl = it % (kVggPoolChans / 8), pix = it / (kVggPoolChans / 8);
    const int h = pix / W, w = pix % W;
    float a[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) a[q] = 0.f;
    for (int i = 0; i < 7; ++i) {
      if (h < vgg_bin_lo(i, H) || h >= vgg_bin_hi(i, H)) continue;
      for (int j = 0; j < 7; ++j) {
        if (w < vgg_bin_lo(j, W) || w >= vgg_bin_hi(j, W)) continue;
#pragma unroll
        for (int q = 0; q < 8; ++q) a[q] += s[(cgl * 8 + q) * 49 + i * 7 + j];
      }
    }
    gx[(static_cast<long long>(b) * H * W + pix) * cvec + cg0 + cgl] = pack8(a);
  }
}

// Classifier dropout: y = x * mask (mask fp32, 0 or 1 / (1 - p), as F.dropout draws it)
__global__ void __launch_bounds__(256) vgg_dropout_fwd_kernel(const uint4* __restrict__ x, const float* __restrict__ mask,
                                                              uint4* __restrict__ y, long long nvec) {
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float f[8], m[8];
    unpack8(__ldg(x + i), f);
    load8f(mask + i * 8, m);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= m[j];
    y[i] = pack8(f);
  }
}

// Backward of h = dropout(relu(pre)) from the stored h alone: h > 0 exactly where both the ReLU and the mask let the value
// through, and the mask's value there is 1 / (1 - p), so dpre = h > 0 ? dh * scale : 0
__global__ void __launch_bounds__(256) vgg_dropout_bwd_kernel(const uint4* __restrict__ g, const uint4* __restrict__ h,
                                                              float scale, uint4* __restrict__ dx, long long nvec) {
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float f[8];
    unpack8(__ldg(g + i), f);
    const uint4 hv = __ldg(h + i);
    const uint32_t w[4] = {hv.x, hv.y, hv.z, hv.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      f[2 * k] = (w[k] & 0x7fffu) != 0u && (w[k] & 0x8000u) == 0u ? f[2 * k] * scale : 0.f;
      f[2 * k + 1] = (w[k] & 0x7fff0000u) != 0u && (w[k] & 0x80000000u) == 0u ? f[2 * k + 1] * scale : 0.f;
    }
    dx[i] = pack8(f);
  }
}

// torch.optim.Adam with L2 weight decay (coupled):  g' = g gscale [clip] + wd p;  m = b1 m + (1 - b1) g';
// v = b2 v + (1 - b2) g'^2;  p -= lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps);  hyper as b200_adamw's (b200_adamw_tick)
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, long long n, const float* __restrict__ hyper,
                                                   float beta1, float beta2, float eps, float wd, float gscale,
                                                   const float* __restrict__ clip) {
  pdl_wait();
  if (clip != nullptr) gscale *= __ldg(clip);
  const float lr = __ldg(hyper), bc1 = __ldg(hyper + 1), bc2 = __ldg(hyper + 2);
  const float step = lr / bc1, rsq = rsqrtf(bc2);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float pi = p[i];
    const float gi = fmaf(wd, pi, g[i] * gscale);
    const float mi = fmaf(beta1, m[i], (1.0f - beta1) * gi);
    const float vi = fmaf(beta2, v[i], (1.0f - beta2) * gi * gi);
    m[i] = mi;
    v[i] = vi;
    pi -= step * mi / (sqrtf(vi) * rsq + eps);
    p[i] = pi;
  }
}

}  // namespace b200
