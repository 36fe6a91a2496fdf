// Masked-autoencoder passes (self-supervised/MAE/models/MAE.py MAE.forward): the per-sample patch shuffle, the masked
// patchify, the decoder-input assembly and its backward, the masked-row gather / scatter around the pixel head, and the
// masked-pixel MSE loss.
//
// Index convention, per sample b of P patches with Nm masked ones:
//   ids[b][s]    patch shown at shuffle slot s = the stable argsort of the sample's P keys (ties -> lower patch index);
//                slots [0, Nm) are the reference's mask_indices, [Nm, P) its unmask_indices
//   slot[b][n]   inverse permutation: the shuffle slot of patch n
// A patch vector is ordered (p1, p2, c), channels last, as x.view(b,c,H/p,p,W/p,p).permute(0,2,4,3,5,1) lays it out.
//
// Every output element is written by exactly one thread and every sum runs over a fixed order (no atomics), so results
// are bitwise reproducible and every pass is capturable in a CUDA graph.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int kMaeMaxP = 1024;        // patches per sample the shuffle CTA holds
constexpr int kMaeMseBlocks = 264;    // fixed grid of the MSE pass: the partial sums do not depend on the device

// One CTA per sample: rank counting over the keys held in shared memory.
__global__ void __launch_bounds__(256) mae_shuffle_kernel(const float* __restrict__ keys, int P, int* __restrict__ ids,
                                                          int* __restrict__ slot) {
  pdl_wait();
  __shared__ float k[kMaeMaxP];
  const long long base = static_cast<long long>(blockIdx.x) * P;
  for (int i = threadIdx.x; i < P; i += blockDim.x) k[i] = keys[base + i];
  __syncthreads();
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const float ki = k[i];
    int r = 0;
    for (int j = 0; j < P; ++j) {
      const float kj = k[j];
      r += (kj < ki || (kj == ki && j < i)) ? 1 : 0;
    }
    ids[base + r] = i;
    slot[base + i] = r;
  }
}

// x fp32 [B][C][H][W] -> vis bf16 [B * (P - Nm)][K] (slots Nm..P-1) and tgt fp32 [B * Nm][K] (slots 0..Nm-1), K = p p C.
__global__ void __launch_bounds__(256) mae_patchify_kernel(const float* __restrict__ x, const int* __restrict__ ids, int B,
                                                           int C, int H, int W, int p, int Nm,
                                                           __nv_bfloat16* __restrict__ vis, float* __restrict__ tgt) {
  pdl_wait();
  const int Wp = W / p, P = (H / p) * Wp, K = p * p * C, Nv = P - Nm;
  const long long n = static_cast<long long>(B) * P * K;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    const int k = static_cast<int>(i % K);
    const long long r = i / K;
    const int s = static_cast<int>(r % P);
    const int b = static_cast<int>(r / P);
    const int c = k % C, t = k / C, pj = t % p, pi = t / p;
    const int pn = ids[static_cast<long long>(b) * P + s];
    const int ph = pn / Wp, pw = pn % Wp;
    const float v = x[((static_cast<long long>(b) * C + c) * H + ph * p + pi) * W + pw * p + pj];
    if (s < Nm)
      tgt[(static_cast<long long>(b) * Nm + s) * K + k] = v;
    else
      vis[(static_cast<long long>(b) * Nv + (s - Nm)) * K + k] = __float2bfloat16(v);
  }
}

// dst[b * n + j][:] = src[b * src_b + ids[b][s0 + j] + off][:] (fp32 rows of width D; src_b = 0: one table for all samples)
template <typename TO>
__global__ void __launch_bounds__(256) mae_gather_rows_kernel(const float* __restrict__ src, long long src_b, int off,
                                                              const int* __restrict__ ids, int B, int P, int s0, int n, int D,
                                                              TO* __restrict__ dst) {
  pdl_wait();
  const long long total = static_cast<long long>(B) * n * D;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * 256) {
    const int d = static_cast<int>(i % D);
    const long long r = i / D;
    const int j = static_cast<int>(r % n);
    const long long b = r / n;
    const long long row = b * src_b + ids[b * P + s0 + j] + off;
    dst[i] = static_cast<TO>(src[row * D + d]);
  }
}

// dec fp32 [B][P][D]: patch n of a sample is mask_embed + dpos[n] when masked, else its encoder row enc[b * Nv + slot - Nm]
__global__ void __launch_bounds__(256) mae_assemble_fwd_kernel(const float* __restrict__ enc, const float* __restrict__ mask,
                                                               const float* __restrict__ dpos, const int* __restrict__ slot,
                                                               int B, int P, int Nm, int D, float* __restrict__ dec) {
  pdl_wait();
  const int Nv = P - Nm;
  const long long total = static_cast<long long>(B) * P * D;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * 256) {
    const int d = static_cast<int>(i % D);
    const long long r = i / D;
    const int pn = static_cast<int>(r % P);
    const long long b = r / P;
    const int s = slot[r];
    dec[i] = s < Nm ? mask[d] + dpos[static_cast<long long>(pn) * D + d] : enc[(b * Nv + (s - Nm)) * D + d];
  }
}

// One CTA per patch position n, threads over the width: the visible rows of g bf16 [B][P][D] go to genc bf16
// [B * Nv][D] at their slot; ddpos[n][:] = sum over b (ascending) of g[b][n][:] where patch n of sample b is masked.
__global__ void __launch_bounds__(256) mae_assemble_bwd_kernel(const __nv_bfloat16* __restrict__ g, const int* __restrict__ slot,
                                                               int B, int P, int Nm, int D, __nv_bfloat16* __restrict__ genc,
                                                               float* __restrict__ ddpos) {
  pdl_wait();
  const int pn = blockIdx.x, Nv = P - Nm;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) {
      const long long r = static_cast<long long>(b) * P + pn;
      const int s = slot[r];
      const __nv_bfloat16 v = g[r * D + d];
      if (s < Nm)
        acc += __bfloat162float(v);
      else
        genc[(static_cast<long long>(b) * Nv + (s - Nm)) * D + d] = v;
    }
    ddpos[static_cast<long long>(pn) * D + d] = acc;
  }
}

// One CTA per pos_embed row q in [0, P]: dpos[q][:] = sum over b (ascending) of the encoder-input gradient row of patch
// q - 1 when that patch is visible (g bf16 [B * Nv][D]); row 0 (the class-token slot) is 0.
__global__ void __launch_bounds__(256) mae_pos_grad_kernel(const __nv_bfloat16* __restrict__ g, const int* __restrict__ slot,
                                                           int B, int P, int Nm, int D, float* __restrict__ dpos) {
  pdl_wait();
  const int q = blockIdx.x, Nv = P - Nm;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    if (q > 0) {
      for (int b = 0; b < B; ++b) {
        const int s = slot[static_cast<long long>(b) * P + q - 1];
        if (s >= Nm) acc += __bfloat162float(g[(static_cast<long long>(b) * Nv + (s - Nm)) * D + d]);
      }
    }
    dpos[static_cast<long long>(q) * D + d] = acc;
  }
}

// g bf16 [B][P][D]: the row of masked patch n is dh[b * Nm + slot][:] (bf16 [B * Nm][D]), every visible row is 0.
__global__ void __launch_bounds__(256) mae_scatter_masked_kernel(const __nv_bfloat16* __restrict__ dh,
                                                                 const int* __restrict__ slot, int B, int P, int Nm, int D,
                                                                 __nv_bfloat16* __restrict__ g) {
  pdl_wait();
  const long long total = static_cast<long long>(B) * P * D;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * 256) {
    const int d = static_cast<int>(i % D);
    const long long r = i / D;
    const long long b = r / P;
    const int s = slot[r];
    g[i] = s < Nm ? dh[(b * Nm + s) * D + d] : __float2bfloat16(0.f);
  }
}

// grad = gscale (pred - t) in bf16; partial[blockIdx.x] = this CTA's sum of (pred - t)^2 (grid kMaeMseBlocks x 256).
__global__ void __launch_bounds__(256) mae_mse_kernel(const float* __restrict__ pred, const float* __restrict__ t, long long n,
                                                      float gscale, __nv_bfloat16* __restrict__ grad,
                                                      float* __restrict__ partial) {
  pdl_wait();
  __shared__ float red[8];
  float acc = 0.f;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    const float e = pred[i] - t[i];
    acc = fmaf(e, e, acc);
    grad[i] = __float2bfloat16(gscale * e);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w];
    partial[blockIdx.x] = s;
  }
}

// loss[0] = (sum of the partials, in index order) / n
__global__ void mae_mse_finish_kernel(const float* __restrict__ partial, int nb, double inv_n, float* __restrict__ loss) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  double s = 0.0;
  for (int i = 0; i < nb; ++i) s += partial[i];
  loss[0] = static_cast<float>(s * inv_n);
}

}  // namespace b200
