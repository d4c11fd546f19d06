// sdw_ptx.cuh — inline-PTX wrappers for the Hopper (sm_90a) primitives the latent-walk kernels are built from:
// mbarrier, TMA (cp.async.bulk.tensor, including the cluster multicast form), thread-block clusters, and the
// warpgroup-MMA (wgmma) fences and shared-memory matrix descriptors.  The wgmma instructions themselves are in
// sdw_wgmma.cuh.
//
// Everything here is device-side plumbing; the kernels live in sdw_gemm.cu (implicit-GEMM conv / linear) and
// sdw_attn.cu (flash attention).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "sdw_wgmma.cuh"

namespace sdw {

// ----------------------------------------------------------------------------
// shared-memory addresses
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  // make generic-proxy smem writes visible to the async proxy (TMA stores read them)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------
// named barriers (ids 1..15; id 0 is __syncthreads) over `count` threads, a multiple of 32.  bar.arrive counts the
// calling warp towards the barrier without waiting; bar.sync counts it and waits until `count` threads have arrived.
// ----------------------------------------------------------------------------
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ----------------------------------------------------------------------------
// per-warpgroup register budget (all 128 threads of the warpgroup execute it): a warp-specialised kernel launched at
// R registers per thread moves registers from its producer warpgroup (dec) to its consumer warpgroups (inc).  N is a
// multiple of 8 in [24, 256]; inc waits until the registers are free.
// ----------------------------------------------------------------------------
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ----------------------------------------------------------------------------
// TMA tiled loads (global -> shared, completion on an mbarrier)
// ----------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(const void* map, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}
// the same box written to the same shared-memory offset of every CTA in `mask` (cluster multicast); each destination
// CTA's barrier at the offset of `bar` receives the completion bytes of its copy
__device__ __forceinline__ void tma_load_4d_mc(const void* map, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3,
                                               uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, "
      "%4, %5, %6}], [%2], %7;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "h"(mask)
      : "memory");
}

// TMA store (shared::cta -> global through a tensor map; rows / columns outside the tensor are clipped) and its
// bulk-group bookkeeping (issued and waited on by the same thread)
__device__ __forceinline__ void tma_store_4d(const void* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {  // <= N groups still READING shared memory
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------
// thread-block clusters
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cta address of this CTA -> shared::cluster address of the same offset in CTA `rank`
__device__ __forceinline__ uint32_t mapa_rank(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
// remote arrive with the default (CTA-scope) release: the only accesses to order before it are this warpgroup's wgmma
// reads of the stage, already waited on; a cluster-scope release would add a GPU-wide memory fence per K block
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}

// ----------------------------------------------------------------------------
// warpgroup MMA plumbing
// ----------------------------------------------------------------------------
// before the first wgmma of a batch: orders earlier register / shared-memory accesses of the accumulators and operands
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {  // <= N committed groups still in flight
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int K>
__device__ __forceinline__ void reg_fence(float (&d)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major operand tile in shared memory written by TMA with SWIZZLE_128B: rows of 64 fp16 (128 B), 8-row swizzle atoms
// of 1024 B (the atom base must be 1024-byte aligned).  Start address and stride byte offset are encoded >> 4; the
// leading byte offset is unused for swizzled K-major tiles.  Advancing K by 16 elements inside the 128-byte row is
// +32 B, i.e. +2 on the descriptor.
__device__ __forceinline__ uint64_t make_desc_k_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);  // [0,14)  start address
  d |= static_cast<uint64_t>(1) << 16;                 // [16,30) LBO (unused)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;         // [32,46) SBO = 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;                 // [62,64) layout: SWIZZLE_128B
  return d;
}

// ----------------------------------------------------------------------------
// programmatic dependent launch: a kernel launched with the PDL attribute may start while its predecessor drains;
// everything before pdl_wait() (barrier init, descriptor prefetch) overlaps the predecessor's tail, nothing after it
// runs until the predecessor grid has completed and its writes are visible.
// ----------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------------------
// small math helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ float silu_f(float x) { return x / (1.f + __expf(-x)); }
__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// a * gelu(g) with the exact-erf GELU through Abramowitz-Stegun 7.1.26 (|erf error| < 1.5e-7, branch-free:
// 1 rcp + 1 ex2 + ~10 FMA), rearranged so that no sign handling is left:
//   g * (1 + erf(g / sqrt2)) = g + |g| * erf(|g| / sqrt2),  erf(z) = 1 - q(t) e^{-z^2},  t = 1 / (1 + p z)
__device__ __forceinline__ float geglu_f(float a, float g) {
  const float z = fabsf(g);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(z, 0.3275911f * 0.70710678118654752f, 1.f)));
  float q = fmaf(1.061405429f, t, -1.453152027f);
  q = fmaf(q, t, 1.421413741f);
  q = fmaf(q, t, -0.284496736f);
  q = fmaf(q, t, 0.254829592f);
  q *= t;
  const float e = ex2f(z * z * (-0.5f * 1.4426950408889634f));  // e^{-z^2/2}
  const float erf_abs = fmaf(-q, e, 1.f);
  return 0.5f * a * fmaf(z, erf_abs, g);
}
// fp32 pairs (a float2 in one 64-bit register pair) for the GroupNorm / small-conv kernels
__device__ __forceinline__ uint64_t pk2(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void upk2(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  upk2(c, c0, c1);
  return pk2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  return pk2(a0 + b0, a1 + b1);
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  return pk2(a0 * b0, a1 * b1);
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace sdw
