// HBM-bound kernels of the denoiser step: RMSNorm(+FiLM), conditioning-vector layers, casts/layout,
// and the diffusion element-wise updates.  All are coalesced 128-bit load/store kernels with warp-shuffle
// row reductions; none of them belongs on tensor cores.  See include/ns2_b200.h sections 3-6 for the
// reference lines each one replaces.
#include "ptx.cuh"
#include "host_common.h"
#include "../../include/ns2_b200.h"

namespace ns2 {

// CTAs per SM of the streaming RMSNorm grid: 76 registers -> 3 resident
// (19.5 us vs 20.1 at 3, 20.5 at 4, 23.3 for one CTA per 8 rows; 32768 x 512 rows, profiles/r02j_rmsnorm_stream.txt)
constexpr int kRmsnormCtasPerSm = 6;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One row of RMSNorm(+gamma)(+FiLM) held in a warp's registers: reduction, scale, store.  Shared by both kernels below
// with the floating-point operation order pinned by explicit fmaf (no compiler-chosen contraction), so a row's result
// does not depend on which kernel variant - i.e. on the problem size - produced it.
template <int VEC, bool OUT_BF16>
__device__ __forceinline__ void rmsnorm_row(const float4 (&v)[VEC], long long row, int lane, int dim, float sqrt_dim,
                                            int rows_per_batch, const float* __restrict__ gamma,
                                            const float* __restrict__ film, long long film_bs,
                                            void* __restrict__ out, long long out_rs) {
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) ss = fmaf(v[i].x, v[i].x, fmaf(v[i].y, v[i].y, fmaf(v[i].z, v[i].z, fmaf(v[i].w, v[i].w, ss))));
  ss = warp_sum(ss);
  // F.normalize: x / max(||x||, eps), eps = 1e-12; then * sqrt(dim)   (ns2.py:738)
  const float inv = __fdiv_rn(sqrt_dim, fmaxf(sqrtf(ss), 1e-12f));
  const float* fg = nullptr;
  if (film != nullptr) fg = film + (row / rows_per_batch) * film_bs;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c4 = i * 32 + lane;
    float4 o = make_float4(__fmul_rn(v[i].x, inv), __fmul_rn(v[i].y, inv), __fmul_rn(v[i].z, inv), __fmul_rn(v[i].w, inv));
    if (gamma != nullptr) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + c4);
      o.x = __fmul_rn(o.x, g.x); o.y = __fmul_rn(o.y, g.y); o.z = __fmul_rn(o.z, g.z); o.w = __fmul_rn(o.w, g.w);
    }
    if (fg != nullptr) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(fg) + c4);
      const float4 b = __ldg(reinterpret_cast<const float4*>(fg + dim) + c4);
      o.x = fmaf(o.x, g.x, b.x); o.y = fmaf(o.y, g.y, b.y); o.z = fmaf(o.z, g.z, b.z); o.w = fmaf(o.w, g.w, b.w);
    }
    if constexpr (OUT_BF16) {
      uint2 w;
      w.x = pack_bf16x2(o.x, o.y);
      w.y = pack_bf16x2(o.z, o.w);
      reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + row * out_rs)[c4] = w;
    } else {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + row * out_rs)[c4] = o;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// RMSNorm (+gamma) (+FiLM): one warp per row, the row stays in registers between the reduction and the
// scaled write (single HBM read of x, single write of the result).  DIM = 32 * 4 * VEC.
// ------------------------------------------------------------------------------------------------
// LENS (lens != NULL): row r of batch b = r / rows_per_batch is live iff r % rows_per_batch < lens[b] (clamped to
// [1, rows_per_batch]); rows that are not live are neither read nor written.
__device__ __forceinline__ bool rmsnorm_row_live(long long row, int rows_per_batch, const int* __restrict__ lens) {
  const long long b = row / rows_per_batch;
  return row - b * rows_per_batch < min(max(__ldg(lens + b), 1), rows_per_batch);
}

template <int VEC, bool OUT_BF16, bool LENS = false>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const float* __restrict__ x, long long x_rs,
                                                      long long rows, int dim, int rows_per_batch,
                                                      const float* __restrict__ gamma,
                                                      const float* __restrict__ film, long long film_bs,
                                                      void* __restrict__ out, long long out_rs,
                                                      const int* __restrict__ lens) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * 8 + warp;
  if (row >= rows) return;
  if (LENS && !rmsnorm_row_live(row, rows_per_batch, lens)) return;
  const float4* xp = reinterpret_cast<const float4*>(x + row * x_rs);
  float4 v[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) v[i] = __ldg(xp + i * 32 + lane);
  rmsnorm_row<VEC, OUT_BF16>(v, row, lane, dim, sqrtf(static_cast<float>(dim)), rows_per_batch, gamma, film, film_bs, out,
                             out_rs);
}

// Streaming variant for large row counts: a resident grid (a few CTAs per SM), every warp walks rows
// warp, warp + #warps, ... and issues the loads of its NEXT row before reducing / scaling / storing the current one, so
// each warp always has one row (dim * 4 bytes) in flight.  The one-row-per-warp kernel above leaves the memory
// pipe idle while a warp reduces, fetches its FiLM vectors and stores, and between CTA generations: ncu showed
// 2.9 TB/s of DRAM reads at 53 % active warps (profiles/r02g_rmsnorm_ncu.txt).
template <int VEC, bool OUT_BF16, bool LENS = false>
__global__ void __launch_bounds__(256) rmsnorm_stream_kernel(const float* __restrict__ x, long long x_rs,
                                                             long long rows, int dim, int rows_per_batch,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ film, long long film_bs,
                                                             void* __restrict__ out, long long out_rs,
                                                             const int* __restrict__ lens) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long nwarps = static_cast<long long>(gridDim.x) * 8;
  long long row = static_cast<long long>(blockIdx.x) * 8 + warp;
  if (row >= rows) return;
  float4 cur[VEC], nxt[VEC];
  bool live = !LENS || rmsnorm_row_live(row, rows_per_batch, lens);
  if (live) {
    const float4* xp = reinterpret_cast<const float4*>(x + row * x_rs);
#pragma unroll
    for (int i = 0; i < VEC; ++i) cur[i] = __ldg(xp + i * 32 + lane);
  }
  const float sqrt_dim = sqrtf(static_cast<float>(dim));
  while (true) {
    const long long nrow = row + nwarps;
    const bool has_next = nrow < rows;
    const bool next_live = has_next && (!LENS || rmsnorm_row_live(nrow, rows_per_batch, lens));
    if (next_live) {
      const float4* xp = reinterpret_cast<const float4*>(x + nrow * x_rs);
#pragma unroll
      for (int i = 0; i < VEC; ++i) nxt[i] = __ldg(xp + i * 32 + lane);
    }
    if (live) rmsnorm_row<VEC, OUT_BF16>(cur, row, lane, dim, sqrt_dim, rows_per_batch, gamma, film, film_bs, out, out_rs);
    if (!has_next) break;
#pragma unroll
    for (int i = 0; i < VEC; ++i) cur[i] = nxt[i];
    row = nrow;
    live = next_live;
  }
}

template <bool OUT_BF16>
static int launch_rmsnorm(const float* x, long long x_rs, long long rows, int dim, int rows_per_batch,
                          const float* gamma, const float* film, long long film_bs, void* out,
                          long long out_rs, cudaStream_t stream, const int* lens = nullptr) {
  NS2_REQUIRE(x && out && rows > 0, "rmsnorm: NULL or empty input");
  NS2_REQUIRE(dim % 128 == 0 && dim <= 1024, "rmsnorm: dim=%d must be a multiple of 128, <= 1024", dim);
  NS2_REQUIRE(x_rs % 4 == 0 && out_rs % 4 == 0 && film_bs % 4 == 0, "rmsnorm: strides must be 16B-aligned");
  const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
  // large problems: a few CTAs per SM, every warp walks >= 4 rows with next-row prefetch
  unsigned sgrid = static_cast<unsigned>(num_sms() * kRmsnormCtasPerSm);
  if (sgrid > grid / 4) sgrid = grid / 4;
  const bool stream_variant = grid >= static_cast<unsigned>(8 * num_sms());
#define NS2_RMS_LAUNCH(V, L)                                                                                       \
  if (stream_variant)                                                                                              \
    rmsnorm_stream_kernel<V, OUT_BF16, L><<<sgrid, 256, 0, stream>>>(x, x_rs, rows, dim, rows_per_batch, gamma, film, \
                                                                     film_bs, out, out_rs, lens);                  \
  else                                                                                                             \
    rmsnorm_kernel<V, OUT_BF16, L><<<grid, 256, 0, stream>>>(x, x_rs, rows, dim, rows_per_batch, gamma, film,        \
                                                             film_bs, out, out_rs, lens);
#define NS2_RMS_CASE(V)                                                                                            \
  case V:                                                                                                          \
    if (lens != nullptr) {                                                                                         \
      NS2_RMS_LAUNCH(V, true)                                                                                      \
    } else {                                                                                                       \
      NS2_RMS_LAUNCH(V, false)                                                                                     \
    }                                                                                                              \
    break;
  switch (dim / 128) {
    NS2_RMS_CASE(1) NS2_RMS_CASE(2) NS2_RMS_CASE(3) NS2_RMS_CASE(4) NS2_RMS_CASE(5) NS2_RMS_CASE(6)
    NS2_RMS_CASE(7) NS2_RMS_CASE(8)
  }
#undef NS2_RMS_CASE
#undef NS2_RMS_LAUNCH
  return launched(1);
}

// ------------------------------------------------------------------------------------------------
// small dense layers on the conditioning vector: one warp per output feature, all (<= 64) batch rows at
// once so the weight row is read exactly once.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxSmallBatch = 64;

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }

// If `freqs` is non-NULL the input row is the learned-sinusoidal embedding of x[b] (a scalar time):
// [t, sin(2 pi t w_0..half-1), cos(2 pi t w_0..half-1)], k = 2*half + 1   (ns2.py:108-120).
__global__ void __launch_bounds__(1024) small_linear_kernel(const float* __restrict__ x, long long x_rs,
                                                           int batch, int k,
                                                           const float* __restrict__ freqs,
                                                           const float* __restrict__ W,
                                                           const float* __restrict__ bias, int n_out,
                                                           int act, float* __restrict__ out,
                                                           long long out_rs) {
  extern __shared__ float xs[];  // (batch, k)
  if (freqs == nullptr) {
    for (int i = threadIdx.x; i < batch * k; i += blockDim.x) xs[i] = x[(i / k) * x_rs + (i % k)];
  } else {
    const int half = (k - 1) / 2;
    for (int i = threadIdx.x; i < batch * k; i += blockDim.x) {
      const int b = i / k, c = i % k;
      const float t = x[b];
      float v = t;
      if (c > 0) {
        // same association order as the reference: ((t * w) * 2) * pi   (ns2.py:117)
        const float fr = t * freqs[(c - 1) % half] * 2.0f * 3.14159265358979323846f;
        v = (c - 1 < half) ? sinf(fr) : cosf(fr);
      }
      xs[i] = v;
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * (blockDim.x >> 5) + warp;   // one warp per output feature
  if (j >= n_out) return;
  const float* w = W + static_cast<long long>(j) * k;
  for (int b0 = 0; b0 < batch; b0 += 8) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int kk = lane; kk < k; kk += 32) {
      const float wv = __ldg(w + kk);
#pragma unroll
      for (int b = 0; b < 8; ++b)
        if (b0 + b < batch) acc[b] += wv * xs[(b0 + b) * k + kk];
    }
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const float s = warp_sum(acc[b]);
      if (lane == 0 && b0 + b < batch) {
        float r = s + (bias ? bias[j] : 0.f);
        if (act == 1) r = silu_f(r);
        out[(b0 + b) * out_rs + j] = r;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// casts and layout
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cast_bf16_kernel(const float4* __restrict__ x,
                                                        const float4* __restrict__ add, long long n4,
                                                        uint2* __restrict__ out) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float4 v = __ldg(x + i);
    if (add != nullptr) {
      const float4 a = __ldg(add + i);
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    uint2 w;
    w.x = pack_bf16x2(v.x, v.y);
    w.y = pack_bf16x2(v.z, v.w);
    out[i] = w;
  }
}

// out[b, n, :] = bf16(x[b, n, :] + c) with c = 0 for n >= L (zero padding of pad_or_curtail_to_length, ns2.py:70-77),
// null_cond[:] for a dropped sample, else cproj[b, n, :]   (torch.where(cond_drop_mask, null_cond, cond) + x, ns2.py:982-992).
// cond_lens (optional): sample b's condition ends at min(L, cond_lens[b]) — the zero padding of a sample run alone.
__global__ void __launch_bounds__(256) cond_inject_kernel(const float4* __restrict__ x, const float4* __restrict__ cproj,
                                                          const uint8_t* __restrict__ drop, const float4* __restrict__ null4,
                                                          int n, int L, const int* __restrict__ cond_lens, int d4,
                                                          uint2* __restrict__ out) {
  const int b = blockIdx.y;
  const int Lb = cond_lens != nullptr ? min(L, max(__ldg(cond_lens + b), 0)) : L;
  const bool dropped = drop != nullptr && drop[b] != 0;
  const long long per = static_cast<long long>(n) * d4;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < per;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pos = static_cast<int>(i / d4), c = static_cast<int>(i - static_cast<long long>(pos) * d4);
    float4 v = __ldg(x + b * per + i);
    if (pos < Lb) {
      const float4 a = dropped ? __ldg(null4 + c) : __ldg(cproj + (static_cast<long long>(b) * L + pos) * d4 + c);
      v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    }
    uint2 w;
    w.x = pack_bf16x2(v.x, v.y);
    w.y = pack_bf16x2(v.z, v.w);
    out[b * per + i] = w;
  }
}

// out[b, :] = drop[b] ? null_row[:] : src[b, :]   (fp32 or bf16 output; torch.where of ns2.py:954-968)
__global__ void __launch_bounds__(256) select_rows_kernel(const uint8_t* __restrict__ drop, const float* __restrict__ null_row,
                                                          const float* __restrict__ src, long long src_rs, int row_len,
                                                          void* __restrict__ out, long long out_rs, int out_bf16) {
  const int b = blockIdx.y;
  const bool dropped = drop[b] != 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < row_len; i += gridDim.x * blockDim.x) {
    const float v = dropped ? __ldg(null_row + i) : __ldg(src + b * src_rs + i);
    if (out_bf16) reinterpret_cast<__nv_bfloat16*>(out)[b * out_rs + i] = __float2bfloat16_rn(v);
    else reinterpret_cast<float*>(out)[b * out_rs + i] = v;
  }
}

// lens (optional): mean over rows [0, lens[b]) (clamped to [1, n]), summed in the same order as over n rows
__global__ void __launch_bounds__(256) mean_rows_kernel(const float* __restrict__ x, int n, int dim,
                                                        const int* __restrict__ lens, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= dim) return;
  const int nb = lens != nullptr ? min(max(__ldg(lens + b), 1), n) : n;
  const float* p = x + static_cast<long long>(b) * n * dim + d;
  float s = 0.f;
  for (int i = 0; i < nb; ++i) s += p[static_cast<long long>(i) * dim];
  out[static_cast<long long>(b) * dim + d] = s / static_cast<float>(nb);
}

// x[b, r, 0:cols] = 0 for r in [lens[b], rows) (lens clamped to [0, rows]); T = float or __nv_bfloat16
template <typename T>
__global__ void __launch_bounds__(256) mask_rows_kernel(T* __restrict__ x, long long rs, long long bs, int rows, int cols,
                                                        const int* __restrict__ lens) {
  const int b = blockIdx.y;
  const int len = min(max(__ldg(lens + b), 0), rows);
  const long long total = static_cast<long long>(rows - len) * cols;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = len + i / cols, c = i % cols;
    x[b * bs + r * rs + c] = T(0.0f);
  }
}

// out[b, r, :] = a[b, r, :] for r < La, bsrc[b, r - La, :] for La <= r < La + Lb, else 0 (bf16, 4 columns per thread);
// La = a_lens[b] clamped to [0, a_rows], Lb likewise
__global__ void __launch_bounds__(256) pack_rows_kernel(const uint2* __restrict__ a, long long a_rs, long long a_bs,
                                                        int a_rows, const int* __restrict__ a_lens,
                                                        const uint2* __restrict__ bsrc, long long b_rs, long long b_bs,
                                                        int b_rows, const int* __restrict__ b_lens, int c4,
                                                        uint2* __restrict__ out, long long o_rs, long long o_bs,
                                                        int out_rows) {
  const int b = blockIdx.y;
  const int La = min(max(__ldg(a_lens + b), 0), a_rows), Lb = min(max(__ldg(b_lens + b), 0), b_rows);
  const long long total = static_cast<long long>(out_rows) * c4;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / c4), c = static_cast<int>(i % c4);
    uint2 v = make_uint2(0u, 0u);
    if (r < La) v = __ldg(a + b * a_bs + r * a_rs + c);
    else if (r < La + Lb) v = __ldg(bsrc + b * b_bs + static_cast<long long>(r - La) * b_rs + c);
    out[b * o_bs + r * o_rs + c] = v;
  }
}

// (B, C, L) f32 -> (B, L, C) bf16 through a 32x32 shared tile (coalesced on both sides)
__global__ void __launch_bounds__(256) transpose_cast_kernel(const float* __restrict__ x, int C, int L,
                                                             __nv_bfloat16* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const float* xb = x + static_cast<long long>(b) * C * L;
  __nv_bfloat16* ob = out + static_cast<long long>(b) * C * L;
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, l = l0 + tx;
    tile[j][tx] = (c < C && l < L) ? xb[static_cast<long long>(c) * L + l] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int l = l0 + j, c = c0 + tx;
    if (c < C && l < L) ob[static_cast<long long>(l) * C + c] = __float2bfloat16_rn(tile[tx][j]);
  }
}

// ------------------------------------------------------------------------------------------------
// diffusion element-wise steps
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) q_sample_kernel(const float4* __restrict__ x0,
                                                       const float4* __restrict__ noise,
                                                       const float* __restrict__ alpha,
                                                       const float* __restrict__ sigma,
                                                       long long per4, float4* __restrict__ xt,
                                                       float4* __restrict__ target, int objective) {
  const int b = blockIdx.y;
  const float a = alpha[b], s = sigma[b];
  const long long base = static_cast<long long>(b) * per4;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < per4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 x = __ldg(x0 + base + i), e = __ldg(noise + base + i);
    xt[base + i] = make_float4(a * x.x + s * e.x, a * x.y + s * e.y, a * x.z + s * e.z, a * x.w + s * e.w);
    if (target != nullptr) {  // ns2.py:1637-1644
      if (objective == NS2_OBJ_V)
        target[base + i] =
            make_float4(a * e.x - s * x.x, a * e.y - s * x.y, a * e.z - s * x.z, a * e.w - s * x.w);
      else
        target[base + i] = (objective == NS2_OBJ_EPS) ? e : x;
    }
  }
}

// per-sample mean squared error; deterministic two-level reduction (fixed grid, no atomics on floats).
// With lens, sample b covers its first lens[b] rows of row4 float4s: the same grid-stride walk over those elements as a
// call on the unpadded sample, so the partial sums and the mean are bit-identical to it.
constexpr int kMseBlocks = 64;
__device__ __forceinline__ long long mse_count4(const int* __restrict__ lens, int b, long long row4, int rows,
                                                long long per4) {
  return lens == nullptr ? per4 : static_cast<long long>(min(max(__ldg(lens + b), 1), rows)) * row4;
}
__global__ void __launch_bounds__(256) mse_partial_kernel(const float4* __restrict__ pred,
                                                          const float4* __restrict__ target,
                                                          long long per4, float* __restrict__ partial,
                                                          const int* __restrict__ lens, long long row4, int rows) {
  const int b = blockIdx.y;
  const long long base = static_cast<long long>(b) * per4;
  const long long n4 = mse_count4(lens, b, row4, rows, per4);
  float s = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 p = __ldg(pred + base + i), t = __ldg(target + base + i);
    const float dx = p.x - t.x, dy = p.y - t.y, dz = p.z - t.z, dw = p.w - t.w;
    s += dx * dx + dy * dy + dz * dz + dw * dw;
  }
  __shared__ float red[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) partial[b * kMseBlocks + blockIdx.x] = v;
  }
}
__global__ void mse_final_kernel(const float* __restrict__ partial, long long per_sample,
                                 float* __restrict__ out, const int* __restrict__ lens, long long row4, int rows) {
  const int b = blockIdx.x;
  if (lens != nullptr) per_sample = 4 * mse_count4(lens, b, row4, rows, per_sample / 4);
  float v = threadIdx.x < kMseBlocks ? partial[b * kMseBlocks + threadIdx.x] : 0.f;
  __shared__ float red[2];
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) out[b] = (red[0] + red[1]) / static_cast<float>(per_sample);
}

// mean of `n` per-sample values (one block; fixed summation order => deterministic)
__global__ void __launch_bounds__(256) batch_mean_kernel(const float* __restrict__ v, int n, float* __restrict__ out) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) s += v[i];
  __shared__ float red[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) out[0] = t / static_cast<float>(n);
  }
}

__global__ void __launch_bounds__(256) ddim_step_kernel(float4* __restrict__ x,
                                                        const float4* __restrict__ v,
                                                        const float* __restrict__ alpha,
                                                        const float* __restrict__ sigma,
                                                        const float* __restrict__ alpha_next,
                                                        const float* __restrict__ sigma_next,
                                                        long long per4, int objective) {
  const int b = blockIdx.y;
  const float a = alpha[b], s = sigma[b], an = alpha_next[b], sn = sigma_next[b];
  const float s_safe = fmaxf(s, 1e-10f);  // safe_div (ns2.py:1122-1123)
  const float a_safe = fmaxf(a, 1e-10f);
  const long long base = static_cast<long long>(b) * per4;
  auto upd = [&](float xv, float vv) {
    // x_start from the model output (ns2.py:1412-1421): v / eps / x0 parameterisation
    const float x0 = objective == NS2_OBJ_V ? a * xv - s * vv
                                            : (objective == NS2_OBJ_EPS ? (xv - s * vv) / a_safe : vv);
    const float eps = (xv - a * x0) / s_safe;   // ns2.py:1425
    return x0 * an + eps * sn;                  // ns2.py:1429
  };
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < per4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 xv = x[base + i], vv = __ldg(v + base + i);
    x[base + i] = make_float4(upd(xv.x, vv.x), upd(xv.y, vv.y), upd(xv.z, vv.z), upd(xv.w, vv.w));
  }
}

// x_start implied by a model output under the chosen parameterisation (ns2.py:1673-1680)
__global__ void __launch_bounds__(256) x_start_kernel(const float4* __restrict__ x, const float4* __restrict__ pred,
                                                      const float* __restrict__ alpha, const float* __restrict__ sigma,
                                                      long long per4, float4* __restrict__ out, int objective) {
  const int b = blockIdx.y;
  const float a = alpha[b], s = sigma[b];
  const float a_safe = fmaxf(a, 1e-10f);
  const long long base = static_cast<long long>(b) * per4;
  auto f = [&](float xv, float pv) {
    return objective == NS2_OBJ_V ? a * xv - s * pv : (objective == NS2_OBJ_EPS ? (xv - s * pv) / a_safe : pv);
  };
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < per4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 xv = __ldg(x + base + i), pv = __ldg(pred + base + i);
    out[base + i] = make_float4(f(xv.x, pv.x), f(xv.y, pv.y), f(xv.z, pv.z), f(xv.w, pv.w));
  }
}

__global__ void __launch_bounds__(256) cfg_combine_kernel(const float4* __restrict__ c,
                                                          const float4* __restrict__ n, float scale,
                                                          long long n4, float4* __restrict__ out) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 a = __ldg(c + i), b = __ldg(n + i);
    out[i] = make_float4(b.x + (a.x - b.x) * scale, b.y + (a.y - b.y) * scale,
                         b.z + (a.z - b.z) * scale, b.w + (a.w - b.w) * scale);
  }
}

// token embedding lookup -> bf16 rows (nn.Embedding of PhonemeEncoder, ns2.py:253, 279-282): negative ids are padding
// and read row `pad_id`
__global__ void __launch_bounds__(256) embedding_bf16_kernel(const long long* __restrict__ ids, long long rows,
                                                             const float* __restrict__ table, int dim, int num_rows,
                                                             int pad_id, __nv_bfloat16* __restrict__ out) {
  const int per_row = dim / 4;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < rows * per_row;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = e / per_row;
    const int c4 = static_cast<int>(e % per_row);
    long long id = __ldg(ids + r);
    if (id < 0) id = pad_id;
    id = id < num_rows ? id : num_rows - 1;
    const float4 v = __ldg(reinterpret_cast<const float4*>(table + id * dim) + c4);
    uint2 w;
    w.x = pack_bf16x2(v.x, v.y);
    w.y = pack_bf16x2(v.z, v.w);
    reinterpret_cast<uint2*>(out + r * dim)[c4] = w;
  }
}

// ------------------------------------------------------------------------------------------------
// GroupNorm + SiLU (+ residual) on token-major activations: Block.forward of the duration / pitch predictor
// (ns2.py:345-365: Conv1d -> nn.GroupNorm(groups, C) -> SiLU) and the ResnetBlock residual (ns2.py:399-401).
// One CTA per (group, batch element): statistics over rows x (C/groups) values in three passes over data that
// stays in L1/L2 (mean, centred variance, apply) - the biased variance and eps placement of nn.GroupNorm.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < 8) ? red[lane] : 0.f;
  t = warp_sum(t);
  return t;
}

// RAGGED: sample b has lens[b] rows (clamped to [1, rows]): the statistics walk those rows exactly as the plain kernel
// walks a tensor of that many rows, and rows at or past the length are written as zeros (the residual is not read)
template <bool RAGGED>
__global__ void __launch_bounds__(256) groupnorm_silu_kernel(const float* __restrict__ x, int rows, int channels,
                                                             int cpg, const float* __restrict__ weight,
                                                             const float* __restrict__ bias, float eps,
                                                             const float* __restrict__ resid,
                                                             float* __restrict__ out_f32,
                                                             __nv_bfloat16* __restrict__ out_bf16,
                                                             const int* __restrict__ lens) {
  __shared__ float red[8];
  const int g = blockIdx.x, b = blockIdx.y;
  const int v4 = cpg / 4;                       // float4 per row of this group
  const long long base = (static_cast<long long>(b) * rows) * channels + g * cpg;
  const int len = RAGGED ? min(max(__ldg(lens + b), 1), rows) : rows;
  const int total = len * v4;
  float s = 0.f;
  for (int e = threadIdx.x; e < total; e += 256) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + base + static_cast<long long>(e / v4) * channels) + e % v4);
    s += (v.x + v.y) + (v.z + v.w);
  }
  const float n = static_cast<float>(len) * cpg;
  const float mean = block_sum_256(s, red) / n;
  float q = 0.f;
  for (int e = threadIdx.x; e < total; e += 256) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + base + static_cast<long long>(e / v4) * channels) + e % v4);
    const float a = v.x - mean, c = v.y - mean, d = v.z - mean, f = v.w - mean;
    q += (a * a + c * c) + (d * d + f * f);
  }
  const float rstd = rsqrtf(block_sum_256(q, red) / n + eps);
  for (int e = threadIdx.x; e < total; e += 256) {
    const int r = e / v4, c4 = e % v4;
    const long long off = base + static_cast<long long>(r) * channels + c4 * 4;
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + off));
    const float4 w = __ldg(reinterpret_cast<const float4*>(weight + g * cpg) + c4);
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + g * cpg) + c4);
    float y[4] = {(v.x - mean) * rstd * w.x + bb.x, (v.y - mean) * rstd * w.y + bb.y,
                  (v.z - mean) * rstd * w.z + bb.z, (v.w - mean) * rstd * w.w + bb.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) y[i] = y[i] / (1.0f + __expf(-y[i]));   // SiLU
    if (resid != nullptr) {
      const float4 rr = __ldg(reinterpret_cast<const float4*>(resid + off));
      y[0] += rr.x; y[1] += rr.y; y[2] += rr.z; y[3] += rr.w;
    }
    if (out_f32 != nullptr) *reinterpret_cast<float4*>(out_f32 + off) = make_float4(y[0], y[1], y[2], y[3]);
    if (out_bf16 != nullptr) {
      uint2 pk;
      pk.x = pack_bf16x2(y[0], y[1]);
      pk.y = pack_bf16x2(y[2], y[3]);
      *reinterpret_cast<uint2*>(out_bf16 + off) = pk;
    }
  }
  if constexpr (RAGGED) {   // rows [len, rows): exact zeros
    for (int e = total + threadIdx.x; e < rows * v4; e += 256) {
      const long long off = base + static_cast<long long>(e / v4) * channels + (e % v4) * 4;
      if (out_f32 != nullptr) *reinterpret_cast<float4*>(out_f32 + off) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (out_bf16 != nullptr) *reinterpret_cast<uint2*>(out_bf16 + off) = make_uint2(0u, 0u);
    }
  }
}

// out[r] = act(dot(x[r, :], w) + bias[0]): the Linear(dim, 1) + ReLU heads of the duration / pitch predictor
// (ns2.py:452-456).  One warp per row.
__global__ void __launch_bounds__(256) rowdot_kernel(const float* __restrict__ x, long long rows, int dim,
                                                     const float* __restrict__ w, const float* __restrict__ bias,
                                                     int relu, float* __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * 8 + warp;
  if (r >= rows) return;
  float s = 0.f;
  for (int c = lane; c < dim / 4; c += 32) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(x + r * dim) + c);
    const float4 b = __ldg(reinterpret_cast<const float4*>(w) + c);
    s += (a.x * b.x + a.y * b.y) + (a.z * b.z + a.w * b.w);
  }
  s = warp_sum(s);
  if (lane == 0) {
    s += (bias != nullptr) ? __ldg(bias) : 0.f;
    out[r] = relu ? fmaxf(s, 0.f) : s;
  }
}

// Length regulation of the conditional path: expand_encodings (ns2.py:1449-1455) with the 0/1 alignment given as one
// text index per frame.  out[b, d, n] = phon[b, m, d] + pitch_table[coarse[b, m], d] with m = idx[b, n]; 0 where
// idx < 0 (frames past the sample's length).  Output is channel-first (B, D, L) like the reference's `cond`;
// 32 x 32 tiles go through shared memory so both the gathers (along d) and the stores (along n) are coalesced.
__global__ void __launch_bounds__(256) expand_encodings_kernel(const float* __restrict__ phon,
                                                               const int* __restrict__ coarse,
                                                               const float* __restrict__ table, int table_rows,
                                                               const int* __restrict__ idx, int T, int D, int L,
                                                               float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, n0 = blockIdx.x * 32, d0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int n = n0 + r, d = d0 + tx;
    float v = 0.f;
    if (n < L && d < D) {
      const int m = __ldg(idx + static_cast<long long>(b) * L + n);
      if (m >= 0 && m < T) {
        int c = __ldg(coarse + static_cast<long long>(b) * T + m);
        c = c < 0 ? 0 : (c >= table_rows ? table_rows - 1 : c);
        v = __fadd_rn(__ldg(phon + (static_cast<long long>(b) * T + m) * D + d),
                      __ldg(table + static_cast<long long>(c) * D + d));
      }
    }
    tile[r][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int d = d0 + r, n = n0 + tx;
    if (d < D && n < L) out[(static_cast<long long>(b) * D + d) * L + n] = tile[tx][r];
  }
}

static cudaError_t configure_small_linear() { return set_max_smem_once(small_linear_kernel, 200 * 1024); }

static unsigned grid_for(long long n4) {
  long long g = (n4 + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  return static_cast<unsigned>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace ns2

using namespace ns2;

extern "C" {

int ns2_groupnorm_silu(const float* x, int32_t batch, int32_t rows, int32_t channels, int32_t groups,
                       const float* weight, const float* bias, float eps, const float* resid, float* out_f32,
                       void* out_bf16, const int32_t* lens, ns2_stream_t stream_) {
  NS2_REQUIRE(batch >= 0 && rows >= 0 && channels > 0 && groups > 0 && channels % groups == 0,
              "groupnorm_silu: bad sizes");
  NS2_REQUIRE((channels / groups) % 4 == 0, "groupnorm_silu: channels per group (%d) must be a multiple of 4",
              channels / groups);
  NS2_REQUIRE(batch <= 65535, "groupnorm_silu: batch %d > 65535", batch);
  if (batch == 0 || rows == 0) return kOk;
  NS2_REQUIRE(x && weight && bias && (out_f32 || out_bf16), "groupnorm_silu: null pointer");
  NS2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(weight) | reinterpret_cast<uintptr_t>(bias) |
                reinterpret_cast<uintptr_t>(resid) | reinterpret_cast<uintptr_t>(out_f32)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(out_bf16) & 7) == 0,
              "groupnorm_silu: pointers must be 16-byte aligned");
  const dim3 grid(groups, batch);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (lens != nullptr)
    groupnorm_silu_kernel<true><<<grid, 256, 0, stream>>>(x, rows, channels, channels / groups, weight, bias, eps, resid,
                                                          out_f32, static_cast<__nv_bfloat16*>(out_bf16), lens);
  else
    groupnorm_silu_kernel<false><<<grid, 256, 0, stream>>>(x, rows, channels, channels / groups, weight, bias, eps,
                                                           resid, out_f32, static_cast<__nv_bfloat16*>(out_bf16),
                                                           nullptr);
  return launched(1);
}

int ns2_mask_rows(void* x, int32_t f32, int64_t row_stride, int64_t batch_stride, int32_t batch, int32_t rows,
                  int32_t cols, const int32_t* lens, ns2_stream_t stream) {
  NS2_REQUIRE(batch >= 0 && rows >= 0 && cols >= 0 && row_stride >= cols && batch_stride >= 0, "mask_rows: bad sizes");
  NS2_REQUIRE(batch <= 65535, "mask_rows: batch %d > 65535", batch);
  if (batch == 0 || rows == 0 || cols == 0) return kOk;
  NS2_REQUIRE(x && lens, "mask_rows: null pointer");
  const dim3 grid(grid_for((static_cast<long long>(rows) * cols + 3) / 4) / (batch > 8 ? 4 : 1) + 1, batch);
  if (f32)
    mask_rows_kernel<float><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<float*>(x), row_stride, batch_stride, rows, cols, lens);
  else
    mask_rows_kernel<__nv_bfloat16><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<__nv_bfloat16*>(x), row_stride, batch_stride, rows, cols, lens);
  return launched(1);
}

int ns2_pack_rows(const void* a, int64_t a_row_stride, int64_t a_batch_stride, int32_t a_rows, const int32_t* a_lens,
                  const void* b, int64_t b_row_stride, int64_t b_batch_stride, int32_t b_rows, const int32_t* b_lens,
                  int32_t batch, int32_t cols, void* out, int64_t out_row_stride, int64_t out_batch_stride,
                  int32_t out_rows, ns2_stream_t stream) {
  NS2_REQUIRE(batch >= 0 && a_rows >= 0 && b_rows >= 0 && cols > 0 && out_rows >= 0, "pack_rows: bad sizes");
  NS2_REQUIRE(out_rows >= a_rows + b_rows, "pack_rows: out_rows %d < %d + %d", out_rows, a_rows, b_rows);
  NS2_REQUIRE(batch <= 65535, "pack_rows: batch %d > 65535", batch);
  if (batch == 0 || out_rows == 0) return kOk;
  NS2_REQUIRE(a && b && a_lens && b_lens && out, "pack_rows: null pointer");
  NS2_REQUIRE(cols % 4 == 0 && a_row_stride % 4 == 0 && a_batch_stride % 4 == 0 && b_row_stride % 4 == 0 &&
                  b_batch_stride % 4 == 0 && out_row_stride % 4 == 0 && out_batch_stride % 4 == 0 &&
                  ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) |
                    reinterpret_cast<uintptr_t>(out)) & 7) == 0,
              "pack_rows: columns and strides must be multiples of 4, pointers 8-byte aligned");
  const int c4 = cols / 4;
  const dim3 grid(grid_for(static_cast<long long>(out_rows) * c4) / (batch > 8 ? 4 : 1) + 1, batch);
  pack_rows_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint2*>(a), a_row_stride / 4, a_batch_stride / 4, a_rows, a_lens, static_cast<const uint2*>(b),
      b_row_stride / 4, b_batch_stride / 4, b_rows, b_lens, c4, static_cast<uint2*>(out), out_row_stride / 4,
      out_batch_stride / 4, out_rows);
  return launched(1);
}

int ns2_rowdot(const float* x, int64_t rows, int32_t dim, const float* w, const float* bias, int32_t relu, float* out,
               ns2_stream_t stream) {
  NS2_REQUIRE(rows >= 0 && dim > 0 && dim % 4 == 0, "rowdot: bad sizes");
  if (rows == 0) return kOk;
  NS2_REQUIRE(x && w && out, "rowdot: null pointer");
  NS2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w)) & 15) == 0, "rowdot: x and w must be 16-byte aligned");
  rowdot_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, rows, dim, w, bias,
                                                                                                  relu, out);
  return launched(1);
}

int ns2_expand_encodings(const float* phon, const int32_t* coarse, const float* pitch_table, int32_t table_rows,
                         const int32_t* idx, int32_t batch, int32_t t_text, int32_t dim, int32_t length, float* out,
                         ns2_stream_t stream) {
  NS2_REQUIRE(batch >= 0 && t_text > 0 && dim > 0 && length >= 0 && table_rows > 0, "expand_encodings: bad sizes");
  NS2_REQUIRE(batch <= 65535, "expand_encodings: batch %d > 65535", batch);
  if (batch == 0 || length == 0) return kOk;
  NS2_REQUIRE(phon && coarse && pitch_table && idx && out, "expand_encodings: null pointer");
  const dim3 grid((length + 31) / 32, (dim + 31) / 32, batch);
  NS2_REQUIRE(grid.y <= 65535, "expand_encodings: dim too large");
  expand_encodings_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(phon, coarse, pitch_table, table_rows, idx,
                                                                              t_text, dim, length, out);
  return launched(1);
}

int ns2_embedding_bf16(const int64_t* ids, int64_t rows, const float* table, int32_t num_rows, int32_t dim,
                       int32_t pad_id, void* out_bf16, ns2_stream_t stream) {
  NS2_REQUIRE(rows >= 0 && num_rows > 0 && dim > 0 && dim % 4 == 0, "embedding_bf16: bad sizes");
  NS2_REQUIRE(pad_id >= 0 && pad_id < num_rows, "embedding_bf16: pad_id %d outside the table", pad_id);
  if (rows == 0) return kOk;
  NS2_REQUIRE(ids && table && out_bf16, "embedding_bf16: null pointer");
  NS2_REQUIRE((reinterpret_cast<uintptr_t>(table) & 15) == 0 && (reinterpret_cast<uintptr_t>(out_bf16) & 7) == 0,
              "embedding_bf16: table must be 16-byte and out 8-byte aligned");
  embedding_bf16_kernel<<<grid_for(rows * (dim / 4)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), rows, table, dim, num_rows, pad_id,
      static_cast<__nv_bfloat16*>(out_bf16));
  return launched(1);
}

int ns2_rmsnorm_film(const float* x, int64_t x_row_stride, int64_t rows, int32_t dim, int32_t rows_per_batch,
                     const float* gamma, const float* film, int64_t film_batch_stride, void* out_bf16,
                     int64_t out_row_stride, const int32_t* lens, ns2_stream_t stream) {
  NS2_REQUIRE(rows_per_batch > 0, "rmsnorm_film: rows_per_batch must be positive");
  NS2_REQUIRE(lens == nullptr || rows % rows_per_batch == 0,
              "rmsnorm_film: rows=%lld is not a whole number of batches of %d rows", static_cast<long long>(rows),
              rows_per_batch);
  return launch_rmsnorm<true>(x, x_row_stride, rows, dim, rows_per_batch, gamma, film,
                              film_batch_stride, out_bf16, out_row_stride,
                              static_cast<cudaStream_t>(stream), lens);
}

int ns2_rmsnorm_f32(const float* x, int64_t x_row_stride, int64_t rows, int32_t dim,
                    const float* gamma, float* out, int64_t out_row_stride, ns2_stream_t stream) {
  return launch_rmsnorm<false>(x, x_row_stride, rows, dim, 1, gamma, nullptr, 0, out, out_row_stride,
                               static_cast<cudaStream_t>(stream));
}

int ns2_small_linear(const float* x, int64_t x_row_stride, int32_t batch, int32_t k, const float* W,
                     const float* bias, int32_t n_out, int32_t act, float* out,
                     int64_t out_row_stride, ns2_stream_t stream) {
  NS2_REQUIRE(x && W && out, "small_linear: NULL pointer");
  NS2_REQUIRE(batch > 0 && batch <= kMaxSmallBatch, "small_linear: batch=%d must be in [1,%d]", batch,
              kMaxSmallBatch);
  const size_t smem = static_cast<size_t>(batch) * k * sizeof(float);
  NS2_REQUIRE(smem <= 200 * 1024, "small_linear: batch*k=%d too large for shared memory", batch * k);
  NS2_CUDA_CHECK(configure_small_linear());
  small_linear_kernel<<<(n_out + 7) / 8, 256, smem, static_cast<cudaStream_t>(stream)>>>(
      x, x_row_stride, batch, k, nullptr, W, bias, n_out, act, out, out_row_stride);
  return launched(1);
}

int ns2_time_cond(const float* times, int32_t batch, const float* freqs, int32_t half_dim,
                  const float* W, const float* bias, int32_t n_out, float* out,
                  int64_t out_row_stride, ns2_stream_t stream) {
  NS2_REQUIRE(times && freqs && W && out, "time_cond: NULL pointer");
  NS2_REQUIRE(batch > 0 && batch <= kMaxSmallBatch, "time_cond: batch=%d must be in [1,%d]", batch,
              kMaxSmallBatch);
  const int k = 2 * half_dim + 1;
  const size_t smem = static_cast<size_t>(batch) * k * sizeof(float);
  NS2_REQUIRE(smem <= 200 * 1024, "time_cond: batch*k=%d too large for shared memory", batch * k);
  NS2_CUDA_CHECK(configure_small_linear());
  // every CTA rebuilds the (batch, k) sinusoidal embedding in shared memory (precise sinf / cosf): 32 output features
  // per 1024-thread CTA = one wave of 64 CTAs at n_out = 2048 instead of two waves of 8-feature CTAs (77 -> ~20 us)
  small_linear_kernel<<<(n_out + 31) / 32, 1024, smem, static_cast<cudaStream_t>(stream)>>>(
      times, 1, batch, k, freqs, W, bias, n_out, /*SiLU*/ 1, out, out_row_stride);
  return launched(1);
}

int ns2_cast_bf16(const float* x, const float* add, int64_t count, void* out_bf16,
                  ns2_stream_t stream) {
  NS2_REQUIRE(x && out_bf16 && count > 0 && count % 4 == 0, "cast_bf16: count must be a multiple of 4");
  const long long n4 = count / 4;
  cast_bf16_kernel<<<grid_for(n4), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(add), n4,
      reinterpret_cast<uint2*>(out_bf16));
  return launched(1);
}

int ns2_cond_inject(const float* x, const float* cproj, const uint8_t* drop_mask, const float* null_cond,
                    int32_t batch, int32_t n, int32_t cond_len, int32_t dim, void* out_bf16, const int32_t* cond_lens,
                    ns2_stream_t stream) {
  NS2_REQUIRE(x && cproj && out_bf16 && batch > 0 && n > 0 && cond_len > 0 && dim > 0 && dim % 4 == 0,
              "cond_inject: bad arguments");
  NS2_REQUIRE(drop_mask == nullptr || null_cond != nullptr, "cond_inject: a drop mask needs null_cond");
  NS2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(cproj) |
                reinterpret_cast<uintptr_t>(null_cond)) & 15) == 0, "cond_inject: pointers must be 16-byte aligned");
  const long long per4 = static_cast<long long>(n) * (dim / 4);
  dim3 grid(static_cast<unsigned>((per4 + 255) / 256 > 512 ? 512 : (per4 + 255) / 256), batch);
  cond_inject_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(cproj), drop_mask,
      reinterpret_cast<const float4*>(null_cond), n, cond_len, cond_lens, dim / 4, reinterpret_cast<uint2*>(out_bf16));
  return launched(1);
}

int ns2_select_rows(const uint8_t* drop_mask, const float* null_row, const float* src, int64_t src_row_stride,
                    int32_t batch, int32_t row_len, void* out, int64_t out_row_stride, int32_t out_bf16,
                    ns2_stream_t stream) {
  NS2_REQUIRE(drop_mask && null_row && src && out && batch > 0 && row_len > 0, "select_rows: bad arguments");
  dim3 grid((row_len + 255) / 256 > 64 ? 64 : (row_len + 255) / 256, batch);
  select_rows_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(drop_mask, null_row, src, src_row_stride,
                                                                          row_len, out, out_row_stride, out_bf16);
  return launched(1);
}

int ns2_mean_rows(const float* x, int32_t batch, int32_t n, int32_t dim, float* out, const int32_t* lens,
                  ns2_stream_t stream) {
  NS2_REQUIRE(x && out && batch > 0 && n > 0 && dim > 0, "mean_rows: bad arguments");
  dim3 grid((dim + 255) / 256, batch);
  mean_rows_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, n, dim, lens, out);
  return launched(1);
}

int ns2_transpose_cast(const float* x, int32_t batch, int32_t channels, int32_t length,
                       void* out_bf16, ns2_stream_t stream) {
  NS2_REQUIRE(x && out_bf16 && batch > 0 && channels > 0 && length > 0, "transpose_cast: bad arguments");
  dim3 grid((length + 31) / 32, (channels + 31) / 32, batch);
  transpose_cast_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, channels, length, reinterpret_cast<__nv_bfloat16*>(out_bf16));
  return launched(1);
}

int ns2_q_sample(const float* x0, const float* noise, const float* alpha, const float* sigma,
                 int32_t batch, int64_t per_sample, float* x_t, float* target, int32_t objective,
                 ns2_stream_t stream) {
  NS2_REQUIRE(x0 && noise && alpha && sigma && x_t, "q_sample: NULL pointer");
  NS2_REQUIRE(objective >= NS2_OBJ_V && objective <= NS2_OBJ_X0, "q_sample: unknown objective %d", objective);
  NS2_REQUIRE(per_sample % 4 == 0 && batch > 0, "q_sample: per_sample must be a multiple of 4");
  dim3 grid(grid_for(per_sample / 4) / (batch > 8 ? 4 : 1) + 1, batch);
  q_sample_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(x0), reinterpret_cast<const float4*>(noise), alpha, sigma,
      per_sample / 4, reinterpret_cast<float4*>(x_t), reinterpret_cast<float4*>(target), objective);
  return launched(1);
}

int ns2_mse_rows(const float* pred, const float* target, int32_t batch, int64_t per_sample, float* partial,
                 float* out, float* mean_out, int64_t row_elems, const int32_t* lens, ns2_stream_t stream) {
  NS2_REQUIRE(pred && target && out && partial, "mse_rows: NULL pointer");
  NS2_REQUIRE(per_sample % 4 == 0 && batch > 0, "mse_rows: bad sizes");
  NS2_REQUIRE(lens == nullptr || (row_elems > 0 && row_elems % 4 == 0 && per_sample % row_elems == 0),
              "mse_rows: row_elems=%lld must be a positive multiple of 4 dividing per_sample=%lld",
              static_cast<long long>(row_elems), static_cast<long long>(per_sample));
  const long long row4 = lens == nullptr ? 0 : row_elems / 4;
  const int rows = lens == nullptr ? 0 : static_cast<int>(per_sample / row_elems);
  dim3 grid(kMseBlocks, batch);
  mse_partial_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(pred), reinterpret_cast<const float4*>(target), per_sample / 4,
      partial, lens, row4, rows);
  mse_final_kernel<<<batch, 64, 0, static_cast<cudaStream_t>(stream)>>>(partial, per_sample, out, lens, row4, rows);
  if (mean_out != nullptr) batch_mean_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(out, batch, mean_out);
  return launched(mean_out != nullptr ? 3 : 2);
}

int ns2_ddim_step(float* x, const float* v, const float* alpha, const float* sigma,
                  const float* alpha_next, const float* sigma_next, int32_t batch,
                  int64_t per_sample, int32_t objective, ns2_stream_t stream) {
  NS2_REQUIRE(x && v && alpha && sigma && alpha_next && sigma_next, "ddim_step: NULL pointer");
  NS2_REQUIRE(objective >= NS2_OBJ_V && objective <= NS2_OBJ_X0, "ddim_step: unknown objective %d", objective);
  NS2_REQUIRE(per_sample % 4 == 0 && batch > 0, "ddim_step: per_sample must be a multiple of 4");
  dim3 grid(grid_for(per_sample / 4) / (batch > 8 ? 4 : 1) + 1, batch);
  ddim_step_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(v), alpha, sigma, alpha_next,
      sigma_next, per_sample / 4, objective);
  return launched(1);
}

int ns2_x_start(const float* x, const float* pred, const float* alpha, const float* sigma, int32_t batch,
                int64_t per_sample, float* out, int32_t objective, ns2_stream_t stream) {
  NS2_REQUIRE(x && pred && alpha && sigma && out, "x_start: NULL pointer");
  NS2_REQUIRE(per_sample % 4 == 0 && batch > 0, "x_start: per_sample must be a multiple of 4");
  NS2_REQUIRE(objective >= NS2_OBJ_V && objective <= NS2_OBJ_X0, "x_start: unknown objective %d", objective);
  dim3 grid(grid_for(per_sample / 4) / (batch > 8 ? 4 : 1) + 1, batch);
  x_start_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(pred), alpha, sigma, per_sample / 4,
      reinterpret_cast<float4*>(out), objective);
  return launched(1);
}

int ns2_cfg_combine(const float* cond, const float* null_, float scale, int64_t count, float* out,
                    ns2_stream_t stream) {
  NS2_REQUIRE(cond && null_ && out && count % 4 == 0, "cfg_combine: bad arguments");
  cfg_combine_kernel<<<grid_for(count / 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(cond), reinterpret_cast<const float4*>(null_), scale, count / 4,
      reinterpret_cast<float4*>(out));
  return launched(1);
}

}  // extern "C"
