// Shared device-side primitives for the sm_90a kernels: mbarrier, TMA, wgmma and the shared-memory accumulator image.
// Everything here is inline PTX for Hopper (compile with -gencode arch=compute_90a,code=sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include "wgmma.cuh"

namespace b200 {

constexpr int kNumSMs = 132;

// ---- Programmatic dependent launch.  Every kernel of the library is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization (host_utils.h launch_pdl): the next kernel of the stream is scheduled
// when the CTAs of its predecessor have finished, without waiting for the grid's completion / memory flush to be processed
// by the launch path; its CTAs run their prologue (barrier init, descriptor prefetch) and then block in
// pdl_wait() until the PREVIOUS kernel has completed and its memory is visible.  Every kernel executes the wait before it
// touches global memory (and before it can exit), so completion stays transitive along the stream: the data dependencies
// are exactly those of plain stream order, only launch latency and prologues overlap the predecessor's end.
// No kernel triggers its dependents explicitly (griddepcontrol.launch_dependents), neither at kernel entry nor right after
// the wait: dependents scheduled early pile onto the SMs that drain first and unbalance the next grid.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}\n" ::"r"(addr),
      "r"(parity)
      : "memory");
}

// Same wait with exponential-free constant back-off: used by the single-lane producer / MMA-issuer roles so that their
// spinning does not steal issue slots from the epilogue warps sharing the SM sub-partition.
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE_%=;\n\t"
      "nanosleep.u32 40;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}\n" ::"r"(addr),
      "r"(parity)
      : "memory");
}

// ---------------------------------------------------------------- shared-memory accessors with 32-bit shared addresses
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
// fp32x2 values in one 64-bit register: the arithmetic is per lane (the same IEEE fp32 results as two scalar operations)
__device__ __forceinline__ uint64_t f2_pack(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void f2_unpack(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t f2_add(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  return f2_pack(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t f2_mul(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  return f2_pack(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t f2_bcast(float c) { return f2_pack(c, c); }
__device__ __forceinline__ uint64_t f2_fma(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  f2_unpack(c, c0, c1);
  return f2_pack(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

// ---------------------------------------------------------------- proxies / fences
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA)
// Every tensor-core kernel of the library follows one scheme: a warpgroup (128 threads, warps 4k .. 4k+3) issues
// wgmma.mma_async for 64 rows of the tile (Wgmma<N, TA, TB>::mma of wgmma.cuh) with the fp32 accumulators in its registers.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Register split of the warp-specialised kernels (384 threads: a TMA producer warpgroup and two consumer warpgroups): the
// producer gives registers back, the consumers, which hold the accumulators, take them.
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// the registers of an accumulator written by wgmma may only be read once wgmma_wait has retired it
template <int R>
__device__ __forceinline__ void wgmma_reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor for a 128B-swizzled tile (rows of 128 bytes, 8-row swizzle atoms of 1024 B).
//   K-major  : rows = M/N index, 128 B of K per row.   SBO = 1024 (next 8 rows), LBO unused.
//   MN-major : rows = K index, 128 B (64 bf16) of M/N per row. SBO = 1024 (next 8 K rows),
//              LBO = byte distance to the next 64-wide M/N atom.
// Bits: [0,14) addr>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout (1 = SWIZZLE_128B). Tiles are 1024-byte aligned, so
// the base-offset field stays 0; a K step of 16 bf16 (32 B) inside the atom adds 2 to the address field.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ---------------------------------------------------------------- accumulator image in shared memory
// The epilogues own one tile row per thread (32 consecutive columns at a time). A warpgroup hands its accumulator fragment
// to them through a row-major fp32 image whose 16-byte chunks are XOR-swizzled by (row & 7) inside each 32-column group:
// the 128-bit row reads of a warp are conflict-free, the 64-bit fragment stores cost two passes.
__device__ __forceinline__ uint32_t img_addr(uint32_t img, int ld, int row, int col) {
  return img + static_cast<uint32_t>(row * ld + (col & 3)) * 4u +
         (static_cast<uint32_t>((col >> 2) ^ (row & 7)) << 4);
}
// fragment of an m64nN accumulator (wgmma.cuh layout) -> image rows row0 .. row0 + 63, columns col0 .. col0 + N - 1
template <int N>
__device__ __forceinline__ void acc_to_img(const float (&d)[N / 2], uint32_t img, int ld, int row0, int col0) {
  const int t = threadIdx.x & 127;
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2);
  const int c = col0 + 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(img_addr(img, ld, r + 8 * h, c + 8 * j)),
                   "f"(d[4 * j + 2 * h]), "f"(d[4 * j + 2 * h + 1])
                   : "memory");
  }
}
// one row, columns col .. col + 4 * CH - 1 (col a multiple of 32 for CH = 8, of 16 for CH = 4) -> v[]
template <int CH>
__device__ __forceinline__ void img_ld(uint32_t img, int ld, int row, int col, uint32_t (&v)[4 * CH]) {
#pragma unroll
  for (int c = 0; c < CH; ++c)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v[4 * c]), "=r"(v[4 * c + 1]), "=r"(v[4 * c + 2]), "=r"(v[4 * c + 3])
                 : "r"(img_addr(img, ld, row, col + 4 * c))
                 : "memory");
}
__device__ __forceinline__ void img_ld32(uint32_t img, int ld, int row, int col, uint32_t (&v)[32]) { img_ld<8>(img, ld, row, col, v); }
__device__ __forceinline__ void img_ld16(uint32_t img, int ld, int row, int col, uint32_t (&v)[16]) { img_ld<4>(img, ld, row, col, v); }

// ---------------------------------------------------------------- misc
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x);
  f[1] = bf16_hi(u.x);
  f[2] = bf16_lo(u.y);
  f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z);
  f[5] = bf16_hi(u.z);
  f[6] = bf16_lo(u.w);
  f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]);
  u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]);
  u.w = pack_bf16x2(f[6], f[7]);
  return u;
}
__device__ __forceinline__ void load8f(const float* __restrict__ p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace b200
