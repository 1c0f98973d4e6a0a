#include "host_common.h"
#include "../../include/ns2_b200.h"

#include <cudaTypedefs.h>
#include <atomic>
#include <mutex>
#include <string.h>
#include <utility>
#include <vector>

namespace ns2 {

std::atomic<long long> g_launches{0};

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
const char* last_error_cstr() { return g_err; }

static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
static std::once_flag g_encode_once;

static void resolve_encode() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess)
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
}

static int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank,
                     const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  std::call_once(g_encode_once, resolve_encode);
  if (!g_encode) return set_error(kErrCuda, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return set_error(kErrInvalidArg, "TMA base pointer %p is not 16-byte aligned", base);
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i];
      if (strides_bytes[i] % 16 != 0)
        return set_error(kErrInvalidArg, "TMA stride %llu (dim %d) is not a multiple of 16 bytes",
                         (unsigned long long)strides_bytes[i], i);
    }
  }
  CUresult r = g_encode(out, dtype, rank, const_cast<void*>(base), gdim,
                        gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return set_error(kErrCuda,
                     "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu] box [%u %u %u]",
                     (int)r, rank, (unsigned long long)dims[0],
                     (unsigned long long)(rank > 1 ? dims[1] : 0),
                     (unsigned long long)(rank > 2 ? dims[2] : 0), box[0], rank > 1 ? box[1] : 0,
                     rank > 2 ? box[2] : 0);
  }
  return kOk;
}

int make_tmap_16bit(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box);
}
int make_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                  const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, rank, dims, strides_bytes, box);
}

constexpr int kMaxDevices = 64;

static std::atomic<int> g_sm_limit{0};   // ns2_set_sm_limit: 0 = use every SM

int num_sms() {
  static std::atomic<int> cache[kMaxDevices];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 148;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  const int lim = g_sm_limit.load(std::memory_order_relaxed);
  return (lim > 0 && lim < n) ? lim : n;
}

cudaError_t set_max_smem_once_impl(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::vector<std::pair<const void*, int>> done;  // (kernel, device) pairs already configured
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  for (const auto& d : done)
    if (d.first == kernel && d.second == dev) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done.emplace_back(kernel, dev);
  return e;
}

}  // namespace ns2

extern "C" {
const char* ns2_last_error(void) { return ns2::last_error_cstr(); }
int ns2_abi_version(void) { return NS2_ABI_VERSION; }
int ns2_set_sm_limit(int sms) {
  const int prev = ns2::g_sm_limit.exchange(sms < 0 ? 0 : (sms & ~1), std::memory_order_relaxed);
  return prev;
}
int64_t ns2_launch_count(void) { return ns2::g_launches.load(std::memory_order_relaxed); }
}
