// Host-side helpers shared by the C-ABI entry points: error reporting, launch accounting and TMA tensor-map encoding.
// The driver API is reached through cudaGetDriverEntryPoint so the library has no link-time dependency
// on libcuda (it must load, and export its symbols, on a box without a GPU driver).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdarg.h>
#include <atomic>
#include <stdio.h>

namespace ns2 {

enum : int {
  kOk = 0,
  kErrInvalidArg = -1,
  kErrCuda = -2,
  kErrUnsupported = -3,
};

int set_error(int code, const char* fmt, ...);
const char* last_error_cstr();

// Encode a tiled tensor map over a 16-bit-element tensor (bf16 / fp16 share the encoding apart from
// the data-type enum, which only matters for OOB-NaN fill that we do not use).
// dims/strides are innermost-first; strides are in BYTES for dims 1..rank-1 (dim 0 is contiguous).
// Swizzle is always 128 B (inner box = 64 elements = 128 bytes), OOB elements read as zero.
int make_tmap_16bit(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box);
// Same for fp32 tensors (TMA stores / reduce-adds of the fp32 residual stream): inner box = 32 elements.
int make_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                  const uint64_t* strides_bytes, const uint32_t* box);

#define NS2_CUDA_CHECK(expr)                                                                  \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return ns2::set_error(ns2::kErrCuda, "%s failed: %s (%s:%d)", #expr,                    \
                            cudaGetErrorString(_e), __FILE__, __LINE__);                      \
  } while (0)

#define NS2_REQUIRE(cond, ...)                                                                \
  do {                                                                                        \
    if (!(cond)) return ns2::set_error(ns2::kErrInvalidArg, __VA_ARGS__);                     \
  } while (0)

// Kernel launches issued through the library since load (ns2_launch_count).
extern std::atomic<long long> g_launches;

// How every entry point ends: count the k kernels it launched, then report a launch that failed.
inline int launched(int k) {
  g_launches.fetch_add(k, std::memory_order_relaxed);
  NS2_CUDA_CHECK(cudaGetLastError());
  return kOk;
}

// SM count of the CURRENT device (cached per device ordinal).
int num_sms();

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): the attribute is per device, so a
// process that drives several GPUs must opt in on each of them.
cudaError_t set_max_smem_once_impl(const void* kernel, int bytes);
template <typename K>
inline cudaError_t set_max_smem_once(K kernel, int bytes) {
  return set_max_smem_once_impl(reinterpret_cast<const void*>(kernel), bytes);
}

}  // namespace ns2
