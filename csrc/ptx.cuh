// Thin inline-PTX wrappers for the Hopper (sm_90a) features the kernels in this
// directory are built on: mbarrier, TMA (cp.async.bulk.tensor), clusters, wgmma
// descriptors (the MMA wrappers are in wgmma.cuh), named barriers, cross-GPU
// memory-model primitives. Hand-written — no CUTLASS/CuTe dependency in product code.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
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
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------- proxies / barriers
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// four 8x8 b16 matrices to shared memory: lane l gives the 16-byte row address of matrix l / 8, row l % 8; register k holds
// this lane's two elements (row lane / 4, columns 2 * (lane % 4) + {0, 1}) of matrix k - the wgmma accumulator fragment
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
               : "memory");
}
__device__ __forceinline__ float2 ld_shared_f32x2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ int2 ld_shared_s32x2(uint32_t addr) {
  int2 v;
  asm volatile("ld.shared.v2.s32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_u16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// multicast variant: the tile lands at the same smem offset of every CTA in `cta_mask` and performs
// complete_tx on the mbarrier at the same offset in each of them
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// plain (non-tensor) bulk copy of `bytes` (a multiple of 16, both addresses 16-byte aligned) that completes on `bar`
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------- clusters
// arrive on the barrier at this smem offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 remAddr32;\n\t"
      "mapa.shared::cluster.u32 remAddr32, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [remAddr32];\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// register budget of a warpgroup (producer warpgroups give registers to the MMA warpgroups)
template <int R>
__device__ __forceinline__ void regs_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void regs_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ---------------------------------------------------------------- wgmma shared-memory descriptors (sm_90)
// 128-byte swizzle (layout type 1 in bits [62,64)), tiles written by TMA with CU_TENSOR_MAP_SWIZZLE_128B and 1024-byte aligned.
//   K-major  tile [rows][128 B of K]: 8-row groups 1024 B apart (SBO); LBO unused. A k-step adds its byte offset inside the
//            128-byte row to the start address.
//   MN-major tile [k rows][128 B of MN]: 8-k-row groups 1024 B apart (SBO), the next 128-byte-wide MN chunk `lbo_bytes`
//            further (LBO); a k-step of 16 rows adds 2048 B.
__device__ __forceinline__ uint64_t desc_sw128(const void* smem_ptr, uint32_t lbo_bytes) {
  const uint32_t a = smem_u32(smem_ptr);
  uint64_t d = 0;
  d |= static_cast<uint64_t>((a & 0x3FFFF) >> 4);               // [0,14)  start address >> 4
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;  // [16,30) leading byte offset >> 4
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                  // [32,46) stride byte offset >> 4
  d |= static_cast<uint64_t>(1) << 62;                          // [62,64) SWIZZLE_128B
  return d;
}
// byte offset added to a descriptor's start-address field
__device__ __forceinline__ uint64_t desc_add(uint64_t d, uint32_t bytes) { return d + (bytes >> 4); }

// ---------------------------------------------------------------- fp8 packing (saturating, round-to-nearest-even)
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));   // first source -> upper byte
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return uint32_t(lo) | (uint32_t(hi) << 16);
}
__device__ __forceinline__ uint32_t pack_e5m2x4(float a, float b, float c, float d) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
  asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return uint32_t(lo) | (uint32_t(hi) << 16);
}
// two consecutive fp32 (8-byte aligned) added in global memory by one vector reduction
__device__ __forceinline__ void red_add_f32x2(float* p, float a, float b) {
  asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffff, v, o));
  return v;
}
// running maximum of NON-NEGATIVE floats: their bit patterns order like unsigned integers
__device__ __forceinline__ void atomic_max_pos_f32(float* p, float v) {
  if (__float_as_uint(v) > *reinterpret_cast<volatile unsigned int*>(p)) atomicMax(reinterpret_cast<unsigned int*>(p), __float_as_uint(v));
}

// ---------------------------------------------------------------- misc math / packing
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t v) {
  return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&v));
}
// Exact-erf GELU pieces via Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7, far below bf16 resolution).
// One MUFU.RCP + one MUFU.EX2 per element; the exp(-x^2/2) term is shared between the CDF (erf) and the PDF.
__device__ __forceinline__ void gelu_cdf_pdf(float x, float& cdf, float& pdf) {
  const float ax = fabsf(x) * 0.70710678118f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  const float p = fmaf(fmaf(fmaf(fmaf(1.061405429f, t, -1.453152027f), t, 1.421413741f), t, -0.284496736f), t, 0.254829592f);
  const float e = exp2f(-1.4426950408889634f * ax * ax);   // exp(-x^2/2)
  const float half_erfc = 0.5f * p * t * e;                // 0.5 * erfc(|x|/sqrt2)
  cdf = x >= 0.f ? 1.0f - half_erfc : half_erfc;
  pdf = 0.3989422804f * e;
}
__device__ __forceinline__ float gelu_exact(float x) {
  float c, d;
  gelu_cdf_pdf(x, c, d);
  return x * c;
}
__device__ __forceinline__ float gelu_grad(float x) {
  float c, d;
  gelu_cdf_pdf(x, c, d);
  return fmaf(x, d, c);
}
// silu(x) = x * s and silu'(x) = s * (1 + x * (1 - s)), s = sigmoid(x): one exp for both
__device__ __forceinline__ float silu_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float silu_grad_from(float x, float s) { return s * fmaf(x, 1.0f - s, 1.0f); }

// ---------------------------------------------------------------- cross-GPU flags (sys scope)
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_add_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
__device__ __forceinline__ float4 ld_nc_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
// peer loads must not use the non-coherent path: data is produced by another GPU this launch
__device__ __forceinline__ float4 ld_peer_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.relaxed.sys.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
// NVLS (NVLink SHARP): `p` is an address in a MULTICAST mapping bound to the same buffer on every GPU of the group.
// ld_reduce returns the element-wise sum over all GPUs, computed inside the NVSwitch; st writes all GPUs at once.
__device__ __forceinline__ float4 mm_ld_reduce_add_f4(const float4* p) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void mm_st_f4(float4* p, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void mm_st_u2(uint2* p, uint2 v) {   // 8 bytes of packed bf16, moved as two 32-bit lanes
  asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)) : "memory");
}
__device__ __forceinline__ void st_peer_f4(float4* p, float4 v) {
  asm volatile("st.global.relaxed.sys.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_peer_u2(uint2* p, uint2 v) {
  asm volatile("st.global.relaxed.sys.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}

}  // namespace pb
