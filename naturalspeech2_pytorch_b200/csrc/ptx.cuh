// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor) and the GMMA shared-memory
// descriptors (the wgmma instructions themselves are in wgmma.cuh).
// Everything here is device-side plumbing shared by gemm.cu, attn.cu, attn_bwd.cu, wgrad.cu and rvq.cu.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma.cuh"

namespace ns2 {

// ---------------------------------------------------------------------------------------------
// generic helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}
// Bounded wait: a pipeline bug must surface as a trapped launch (an error the host sees), never as a
// hung GPU.  ~2e9 SM cycles is about a second; no legitimate wait in these kernels is near that.
// A timeout shows up only as a failed launch (cudaErrorLaunchFailure / illegal instruction on the next
// synchronising call), with no device-side message: any function call here, printf included, makes ptxas
// serialize every wgmma of the calling kernel (warning C7510), so the branch holds nothing but the trap.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t it = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++it) & 0xfff) == 0 && (clock64() - t0) > 2000000000LL) __trap();
  }
}

// Same bounded wait for service warps that idle through long phases of their CTA: sleeping between polls leaves the
// issue slots of their SM sub-partition to the compute warps (+2 % on the RVQ kernel).
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity, unsigned ns) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t it = 0;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(ns);
    if (((++it) & 0xfff) == 0 && (clock64() - t0) > 2000000000LL) __trap();
  }
}

// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// TMA stores (smem -> global, bulk async-group completion).  OOB parts of the box are clipped by the TMA unit.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// global[tile] += smem[tile] (element-wise fp32 add performed at L2): the residual-stream update
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// plain 1-D bulk copy global -> shared (16-byte aligned, size % 16 == 0), completion on an mbarrier like the tensor loads
__device__ __forceinline__ void bulk_load_1d(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(mbar)
               : "memory");
}

// 16-byte global -> shared copy (LDGSTS, cached in L2 only): no register round trip; cp_async_wait_all completes it
__device__ __forceinline__ void cp_async_16(uint32_t dst_smem, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(src))
               : "memory");
}
// 4-byte global -> shared copy (LDGSTS through L1): small per-launch tables such as per-batch lengths
__device__ __forceinline__ void cp_async_4(uint32_t dst_smem, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst_smem), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {  // smem of all but the N newest groups may be reused
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// GMMA (wgmma) shared-memory matrix descriptors
// ---------------------------------------------------------------------------------------------
// 128-byte swizzle.  Both majors use the same encoding for our tiles:
//   K-major  (rows of 64 x 16-bit = 128 B, TMA box {64, rows}): SBO = 1024 B between 8-row groups.
//   MN-major (64 MN elements = 128 B contiguous per K row):     SBO = 1024 B between 8-K-row groups,
//             LBO = stride between 64-element MN atoms (unused when the MN extent is 64).
// start address / LBO / SBO are stored without their 4 LSBs; bits [62,64) = layout type (1 = SWIZZLE_128B).
// Tiles must be 1024-byte aligned (base_offset = 0).  Advancing 16 K elements inside a K-major atom is +32 bytes,
// i.e. +2 on the descriptor.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Un-swizzled ("interleave") K-major operand: 8-row x 16-byte core matrices, LBO = distance between the two K halves of a
// 16-element K step, SBO = distance between consecutive 8-row groups (cute: ((8,m),(T,2)):((1T,SBO),(1,LBO))).
__device__ __forceinline__ uint64_t gmma_desc_plain(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

// stmatrix.x4: four 8x8 b16 matrices; register k of lane l = row l/4, columns 2(l%4)+{0,1} of matrix k (the wgmma
// accumulator fragment layout), lane l gives the shared address of row l%8 of matrix l/8
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_shared_v2_f32(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// named barrier over the 128 threads of one warpgroup (ids 8..11 are reserved for this)
__device__ __forceinline__ void warpgroup_bar(int wg) {
  asm volatile("bar.sync %0, 128;" ::"r"(8 + wg) : "memory");
}
// named barrier `id` over `count` threads (a multiple of 32); id 0 is __syncthreads
__device__ __forceinline__ void named_bar(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---------------------------------------------------------------------------------------------
// small numeric helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// MUFU-based variants for the fused GEMM epilogues (relative error ~2^-11, below the bf16 rounding of the
// value that is stored): tanh.approx, sigmoid(x) = 0.5 tanh(x/2) + 0.5.
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigmoid_fast(float x) { return fmaf(tanh_fast(0.5f * x), 0.5f, 0.5f); }
// exact-erf GELU with erf from Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7; < 6e-7 as evaluated here in fp32, the
// most near x = 0 where 1 - poly e cancels): one MUFU.EX2, one MUFU.RCP, 8 FMA.  The GEGLU GEMM epilogue uses it.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-z * z * 1.4426950408889634f));
  const float erf_abs = fmaf(-poly, e, 1.0f);      // erf(|x|/sqrt2)
  const float erf_v = copysignf(erf_abs, x);
  return 0.5f * x * (1.0f + erf_v);
}

}  // namespace ns2
