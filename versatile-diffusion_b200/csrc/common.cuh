// Common sm_90a device helpers for the vdb200 kernels: mbarrier, TMA
// (cp.async.bulk.tensor), wgmma wrappers and small math utils.
// Everything here is inline PTX; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vdb {

#define VDB_DEVINL __device__ __forceinline__

// ----------------------------------------------------------------------------
// status codes of the C ABI (include/vdb200.h mirrors these)
// ----------------------------------------------------------------------------
enum : int {
  VDB_OK = 0,
  VDB_ERR_INVALID = 1,     // bad argument (shape/alignment/null)
  VDB_ERR_CUDA = 2,        // CUDA runtime / driver error (see vdb_last_error)
  VDB_ERR_UNSUPPORTED = 3, // shape outside what the kernels implement
};

// 16-byte shared-memory load through a 32-bit shared address (a pointer derived from the aligned dynamic window has lost its
// address space: the compiler emits generic LD.E instead of LDS)
VDB_DEVINL float4 lds_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}

VDB_DEVINL float2 lds_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
// stmatrix: four 8x8 b16 matrices from the mma accumulator-fragment layout to shared memory.  Register i of lane l holds
// row l / 4, columns 2 (l % 4) and 2 (l % 4) + 1 of matrix i; lanes 8i .. 8i + 7 give the 16-byte row addresses of matrix i.
VDB_DEVINL void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
               : "memory");
}

VDB_DEVINL uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

VDB_DEVINL uint32_t lane_id() {
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}

VDB_DEVINL bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
VDB_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
VDB_DEVINL void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
VDB_DEVINL void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
VDB_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
VDB_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
VDB_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
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
VDB_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------
// TMA tiled loads (global -> shared), completion on an mbarrier
// ----------------------------------------------------------------------------
VDB_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
VDB_DEVINL void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
VDB_DEVINL void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// TMA tiled store (shared -> global), bulk-group completion.  The issuing thread must have ordered the generic-proxy
// shared-memory writes of the tile before it (fence.proxy.async by every writer, then a barrier).
VDB_DEVINL void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
VDB_DEVINL void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
VDB_DEVINL void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
VDB_DEVINL void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// ----------------------------------------------------------------------------
// thread-block clusters: distributed shared memory and remote mbarrier arrivals
// ----------------------------------------------------------------------------
VDB_DEVINL uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
VDB_DEVINL void cluster_sync_all() {   // every thread of every CTA of the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of the same shared-memory offset in CTA `rank` of the cluster
VDB_DEVINL uint32_t mapa_u32(uint32_t local_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
  return r;
}
VDB_DEVINL void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}

// ----------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): the four warps of a warpgroup issue together, the accumulator lives in registers.
// ----------------------------------------------------------------------------
// K-major, 128-byte-swizzled shared-memory operand descriptor.
// Tile = rows of 128 B (64 bf16 along K), 8-row groups 1024 B apart (SBO), base 1024-B aligned.
// Bits: [0,14) addr>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout=1 (SWIZZLE_128B).
// Advancing 16 bf16 (32 B) along K inside the swizzle atom is +2 on the descriptor.
VDB_DEVINL uint64_t make_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;            // LBO (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;    // SBO
  d |= static_cast<uint64_t>(1) << 62;            // SWIZZLE_128B
  return d;
}
VDB_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
VDB_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
VDB_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins accumulator registers behind the preceding wgmma_wait: the asynchronous MMA writes them after the issuing asm
// statement, so no use may be scheduled between the issue and the wait.
template <int R>
VDB_DEVINL void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// nanosecond wall clock shared by all SMs (debug timelines, watchdogs)
VDB_DEVINL unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ----------------------------------------------------------------------------
// programmatic dependent launch: a kernel launched with the PDL attribute may start while its predecessor
// drains; it must not touch dependent global memory before pdl_wait(). No-ops for ordinary launches.
// ----------------------------------------------------------------------------
VDB_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
VDB_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------------------
// small math / packing helpers
// ----------------------------------------------------------------------------
VDB_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
VDB_DEVINL float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
// 2^x on the MUFU pipe (one SFU op)
VDB_DEVINL float ex2_mufu(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 2^x on the FMA/ALU pipes: round-to-nearest split x = n + f, cubic minimax of 2^f on [-0.5, 0.5]
// (max rel. error 7.7e-5, far below bf16's 4e-3), exponent add through the integer pipe.
VDB_DEVINL float ex2_poly(float x) {
  x = fmaxf(x, -126.0f);
  const float r = x + 12582912.0f;          // 1.5 * 2^23: low mantissa bits now hold rint(x)
  const float f = x - (r - 12582912.0f);
  float p = fmaf(0.0550886838f, f, 0.242604051f);
  p = fmaf(p, f, 0.693276242f);
  p = fmaf(p, f, 0.99992894f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(r) << 23));
}
VDB_DEVINL float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// SiLU for bf16 outputs: x * sigmoid(x) = 0.5x * (1 + tanh(x/2)) with ONE MUFU op (tanh.approx, rel. error < 5e-4,
// below bf16 rounding); the exp+rcp form needs two and made GroupNorm-apply MUFU-bound.
VDB_DEVINL float silu_bf16_f(float x) {
  float th;
  asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(0.5f * x));
  const float hx = 0.5f * x;
  return fmaf(hx, th, hx);
}
VDB_DEVINL float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
// exact-erf GELU through Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7): 2 MUFU + ~10 FMA instead of erff()
VDB_DEVINL float gelu_as_f(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float erf_abs = 1.0f - poly * t * __expf(-z * z);
  return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}
// GELU for bf16 outputs (GEGLU epilogue): x * Phi(x) with Phi through one tanh.approx MUFU op.  The tanh form
// differs from the erf form by < 3e-4 absolute in Phi and tanh.approx adds < 5e-4 relative — both below the
// 2^-9 relative rounding of the bf16 value this feeds, so results match the exact-erf GELU to within one bf16 ulp.
VDB_DEVINL float gelu_fast_f(float x) {
  const float u = x * fmaf(0.0356774081f, x * x, 0.7978845608f);
  float th;
  asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(u));
  const float hx = 0.5f * x;
  return fmaf(hx, th, hx);
}
VDB_DEVINL float quick_gelu_f(float x) { return __fdividef(x, 1.0f + __expf(-1.702f * x)); }

}  // namespace vdb

#include "wgmma.cuh"
