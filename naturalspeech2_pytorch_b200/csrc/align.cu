// Monotonic alignment search (`maximum_path`, aligner.py:88-122 of the reference) as two kernels.
//
// The reference runs the Viterbi recursion as a Python loop over the t_y mel frames (~10 PyTorch launches per
// frame) and a second Python loop for the backtrack.  Here one CTA owns one batch element:
//   * warp 0 keeps the running score column v[0..t_x) in registers (R consecutive text positions per lane, the
//     neighbour across the lane boundary comes from one shuffle per frame) and walks the frames; the 1-bit
//     decisions of a frame leave as one coalesced 128-byte store (32 lanes x R <= 32 bits);
//   * warps 1..7 are producers: they stream value*mask tiles (t_x rows x CW frames) from HBM with coalesced
//     loads and stage them transposed in shared memory (ring of STAGES tiles, named-barrier full/empty
//     hand-off), so the serial warp never waits on HBM;
//   * the backtrack re-reads the decision words in 32-frame chunks (coalesced, prefetched one chunk ahead) and
//     lane 0 walks them in shared memory; it emits idx[b, j] = the text position aligned to frame j.
// A second, grid-wide kernel expands idx into the dense 0/1 path (times the mask) with 128-bit stores: that is
// the only part with real HBM traffic (read mask + write path).
//
// Arithmetic is restated operation for operation (fp32 multiply by the mask, fp32 add, >= compares, ties to
// "stay"), with __fmul_rn/__fadd_rn so the compiler cannot contract them: the result is bit-identical to the
// reference on the same inputs.
#include "host_common.h"
#include "../../include/ns2_b200.h"

namespace ns2 {

namespace {

constexpr int kDpThreads = 256;                    // warp 0 = recursion, warps 1..7 = producers
constexpr int kProducers = kDpThreads - 32;
constexpr int kStages = 3;

__device__ __forceinline__ void bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

template <int R>
struct MasCfg {
  static constexpr int CW = (R >= 32) ? 16 : 32;  // frames per staged tile
  static constexpr int CS = R * 32 + 1;           // padded column stride (floats): conflict-free transposed writes
  static constexpr int TILE_FLOATS = CW * CS;
  static constexpr int MZ_WORDS = 32 * (CW + 1);  // "mask is zero" bits, one word per (lane, frame), padded rows
  static constexpr size_t SMEM = static_cast<size_t>(kStages) * (TILE_FLOATS + MZ_WORDS) * 4 + 32 * 32 * 4;
};

// value/mask: (b, t_x, t_y) f32 contiguous.  dirw: (b, t_y, 32) u32 scratch.  idx_out: (b, t_y) i32.
template <int R>
__global__ void __launch_bounds__(kDpThreads, 1)
mas_dp_kernel(const float* __restrict__ value, const float* __restrict__ mask, int t_x, int t_y, float neg_const,
              uint32_t* __restrict__ dirw, int32_t* __restrict__ idx_out) {
  using Cfg = MasCfg<R>;
  constexpr int CW = Cfg::CW, CS = Cfg::CS;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* tiles = reinterpret_cast<float*>(smem_raw);
  uint32_t* mz = reinterpret_cast<uint32_t*>(tiles + kStages * Cfg::TILE_FLOATS);
  uint32_t* bt = mz + kStages * Cfg::MZ_WORDS;  // backtrack chunk: 32 frames x 32 words

  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* vb = value + static_cast<size_t>(b) * t_x * t_y;
  const float* mb = mask + static_cast<size_t>(b) * t_x * t_y;
  uint32_t* db = dirw + static_cast<size_t>(b) * t_y * 32;
  const int nchunks = (t_y + CW - 1) / CW;

  if (warp != 0) {
    // ---------------- producers ----------------
    // One task = (lane group gi of the recursion warp, frame c): the R text positions gi*R..gi*R+R-1 of one frame.
    // Consecutive threads take consecutive frames (coalesced 128-byte rows); the loads of a task are issued as one
    // batch of up to 2*RB independent requests so HBM latency overlaps; the "mask is zero" bits of the task are
    // assembled in a register (no atomics).
    constexpr int RB = (R < 8) ? R : 8;
    const int p = threadIdx.x - 32;
    for (int k = 0; k < nchunks; ++k) {
      const int s = k % kStages;
      if (k >= kStages) bar_sync(4 + s, kDpThreads);  // tile s drained by the recursion warp
      float* tile = tiles + s * Cfg::TILE_FLOATS;
      uint32_t* mzs = mz + s * Cfg::MZ_WORDS;
      const int j0 = k * CW;
      for (int task = p; task < 32 * CW; task += kProducers) {
        const int c = task % CW, gi = task / CW;
        const int j = j0 + c;
        uint32_t zbits = 0u;
#pragma unroll
        for (int r0 = 0; r0 < R; r0 += RB) {
          float vv[RB], mm[RB];
#pragma unroll
          for (int u = 0; u < RB; ++u) {
            const int i = gi * R + r0 + u;
            const bool ok = (i < t_x) && (j < t_y);
            const size_t off = ok ? static_cast<size_t>(i) * t_y + j : 0;
            vv[u] = ok ? __ldg(vb + off) : 0.f;
            mm[u] = ok ? __ldg(mb + off) : 1.f;
          }
#pragma unroll
          for (int u = 0; u < RB; ++u) {
            tile[c * CS + (r0 + u) * 32 + gi] = __fmul_rn(vv[u], mm[u]);   // value = value * mask  (aligner.py:93)
            zbits |= static_cast<uint32_t>(mm[u] == 0.f) << (r0 + u);       // direction := 1 where ~mask (aligner.py:110)
          }
        }
        mzs[gi * (CW + 1) + c] = zbits;
      }
      __threadfence_block();
      bar_arrive(1 + s, kDpThreads);
    }
    return;
  }

  // ---------------- recursion warp ----------------
  float v[R];
#pragma unroll
  for (int r = 0; r < R; ++r) v[r] = 0.f;          // v = zeros(b, t_x)       (aligner.py:97)
  for (int k = 0; k < nchunks; ++k) {
    const int s = k % kStages;
    bar_sync(1 + s, kDpThreads);
    const float* tile = tiles + s * Cfg::TILE_FLOATS;
    const uint32_t* mzs = mz + s * Cfg::MZ_WORDS;
    const int j0 = k * CW;
    const int cn = min(CW, t_y - j0);
#pragma unroll 4
    for (int c = 0; c < cn; ++c) {
      const int j = j0 + c;
      float val[R];
#pragma unroll
      for (int r = 0; r < R; ++r) val[r] = tile[c * CS + r * 32 + lane];
      float prev = __shfl_up_sync(0xffffffffu, v[R - 1], 1);
      if (lane == 0) prev = neg_const;              // v0 = pad(v, const)[:, :-1] (aligner.py:101)
      uint32_t bits = mzs[lane * (CW + 1) + c];
#pragma unroll
      for (int r = R - 1; r >= 0; --r) {
        const float v0 = (r == 0) ? prev : v[r - 1];
        const float v1 = v[r];
        const bool stay = v1 >= v0;                 // max_mask                  (aligner.py:103)
        const float vmax = stay ? v1 : v0;
        v[r] = (lane * R + r <= j) ? __fadd_rn(vmax, val[r]) : neg_const;  // (aligner.py:107-108)
        bits |= static_cast<uint32_t>(stay) << r;
      }
      db[static_cast<size_t>(j) * 32 + lane] = bits;
    }
    if (k + kStages < nchunks) bar_arrive(4 + s, kDpThreads);
  }

  // index = mask[:, :, 0].sum(1).long() - 1   (aligner.py:113)
  float msum = 0.f;
  for (int i = lane; i < t_x; i += 32) msum += __ldg(mb + static_cast<size_t>(i) * t_y);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) msum += __shfl_xor_sync(0xffffffffu, msum, o);
  int idx = static_cast<int>(static_cast<long long>(msum)) - 1;

  __threadfence_block();
  __syncwarp();
  // ---------------- backtrack (aligner.py:116-118) ----------------
  const int nbt = (t_y + 31) / 32;
  uint32_t pre[32];
  auto load_chunk = [&](int q) {
    const int j0 = q * 32;
#pragma unroll
    for (int c = 0; c < 32; ++c) pre[c] = (j0 + c < t_y) ? db[static_cast<size_t>(j0 + c) * 32 + lane] : 0u;
  };
  load_chunk(nbt - 1);
  for (int q = nbt - 1; q >= 0; --q) {
#pragma unroll
    for (int c = 0; c < 32; ++c) bt[c * 32 + lane] = pre[c];
    __syncwarp();
    if (q > 0) load_chunk(q - 1);                   // in flight while lane 0 walks this chunk
    if (lane == 0) {
      const int j0 = q * 32;
      for (int c = min(31, t_y - 1 - j0); c >= 0; --c) {
        int eff = idx < 0 ? idx + t_x : idx;        // Python index wrap of path[b, index, j]
        eff = max(0, min(eff, t_x - 1));
        idx_out[static_cast<size_t>(b) * t_y + j0 + c] = eff;
        const uint32_t w = bt[c * 32 + eff / R];
        idx = idx + static_cast<int>((w >> (eff % R)) & 1u) - 1;  // index += direction - 1
      }
    }
    __syncwarp();
  }
}

// path[b, i, j] = (idx[b, j] == i) * mask[b, i, j]      (aligner.py:117, 120)
template <int VEC>
__global__ void __launch_bounds__(256)
mas_expand_kernel(const int32_t* __restrict__ idx, const float* __restrict__ mask, int t_x, int t_y, long long total,
                  float* __restrict__ path) {
  const long long nvec = total / VEC;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < nvec;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long flat = e * VEC;
    const int j = static_cast<int>(flat % t_y);
    const long long bi = flat / t_y;
    const int i = static_cast<int>(bi % t_x);
    const long long b = bi / t_x;
    if constexpr (VEC == 4) {
      const int4 id = __ldg(reinterpret_cast<const int4*>(idx + b * t_y + j));
      const float4 m = __ldg(reinterpret_cast<const float4*>(mask + flat));
      float4 o;
      o.x = __fmul_rn(id.x == i ? 1.f : 0.f, m.x);
      o.y = __fmul_rn(id.y == i ? 1.f : 0.f, m.y);
      o.z = __fmul_rn(id.z == i ? 1.f : 0.f, m.z);
      o.w = __fmul_rn(id.w == i ? 1.f : 0.f, m.w);
      *reinterpret_cast<float4*>(path + flat) = o;
    } else {
      path[flat] = __fmul_rn(__ldg(idx + b * t_y + j) == i ? 1.f : 0.f, __ldg(mask + flat));
    }
  }
}

template <int R>
int launch_dp(const float* value, const float* mask, int b, int t_x, int t_y, float neg_const, uint32_t* dirw,
              int32_t* idx, cudaStream_t st) {
  NS2_CUDA_CHECK(set_max_smem_once(mas_dp_kernel<R>, static_cast<int>(MasCfg<R>::SMEM)));
  mas_dp_kernel<R><<<b, kDpThreads, MasCfg<R>::SMEM, st>>>(value, mask, t_x, t_y, neg_const, dirw, idx);
  NS2_CUDA_CHECK(cudaGetLastError());
  return kOk;
}

}  // namespace
}  // namespace ns2

using namespace ns2;

extern "C" {

int64_t ns2_maximum_path_workspace_bytes(int32_t batch, int32_t t_x, int32_t t_y) {
  (void)t_x;
  if (batch <= 0 || t_y <= 0) return 0;
  return static_cast<int64_t>(batch) * t_y * 32 * 4;
}

int ns2_maximum_path(const float* value, const float* mask, int32_t batch, int32_t t_x, int32_t t_y, float neg_const,
                     void* workspace, int64_t workspace_bytes, int32_t* idx, float* path, ns2_stream_t stream) {
  NS2_REQUIRE(batch >= 0 && t_x >= 0 && t_y >= 0, "maximum_path: negative size");
  if (batch == 0 || t_x == 0 || t_y == 0) return kOk;
  NS2_REQUIRE(t_x <= 1024, "maximum_path: t_x = %d > 1024 text positions is not supported", t_x);
  NS2_REQUIRE(value && mask && idx && workspace, "maximum_path: null pointer");
  NS2_REQUIRE(workspace_bytes >= ns2_maximum_path_workspace_bytes(batch, t_x, t_y),
              "maximum_path: workspace too small (%lld bytes)", static_cast<long long>(workspace_bytes));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t* dirw = static_cast<uint32_t*>(workspace);
  int rc;
  if (t_x <= 32) rc = launch_dp<1>(value, mask, batch, t_x, t_y, neg_const, dirw, idx, st);
  else if (t_x <= 64) rc = launch_dp<2>(value, mask, batch, t_x, t_y, neg_const, dirw, idx, st);
  else if (t_x <= 128) rc = launch_dp<4>(value, mask, batch, t_x, t_y, neg_const, dirw, idx, st);
  else if (t_x <= 256) rc = launch_dp<8>(value, mask, batch, t_x, t_y, neg_const, dirw, idx, st);
  else if (t_x <= 512) rc = launch_dp<16>(value, mask, batch, t_x, t_y, neg_const, dirw, idx, st);
  else rc = launch_dp<32>(value, mask, batch, t_x, t_y, neg_const, dirw, idx, st);
  if (rc != kOk) return rc;
  if (path != nullptr) {
    const long long total = static_cast<long long>(batch) * t_x * t_y;
    const bool vec = (t_y % 4 == 0) && ((reinterpret_cast<uintptr_t>(mask) | reinterpret_cast<uintptr_t>(path) |
                                         reinterpret_cast<uintptr_t>(idx)) % 16 == 0);
    const long long nvec = vec ? total / 4 : total;
    long long grid = (nvec + 255) / 256;
    const long long cap = static_cast<long long>(num_sms()) * 8;
    if (grid > cap) grid = cap;
    if (vec) mas_expand_kernel<4><<<static_cast<unsigned>(grid), 256, 0, st>>>(idx, mask, t_x, t_y, total, path);
    else mas_expand_kernel<1><<<static_cast<unsigned>(grid), 256, 0, st>>>(idx, mask, t_x, t_y, total, path);
  }
  return launched(path != nullptr ? 2 : 1);
}

}  // extern "C"
