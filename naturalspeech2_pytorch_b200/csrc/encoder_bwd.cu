// Element-wise / scatter kernels of the conditioning front end's backward pass: what autograd runs for the reference's
// `loss.backward()` (ns2.py:1886) below `Model(prompt=..., cond=...)`.  The diffusion loss is the only gradient path into
// the encoders (SURVEY T11), through
//   prompt_enc = SpeechPromptEncoder(prompt)                              (ns2.py:1538, 289-341)
//   cond       = expand_encodings(PhonemeEncoder(text), aln_mask, pitch)  (ns2.py:1539, 1581-1583, 1449-1455)
// The matrix products are ns2_gemm (dgrad on transposed packs) and ns2_wgrad; this file holds the pieces between them:
//   silu_bwd               backward of the SiLU after every k=9 conv of both encoders (ns2.py:255-257, 316-320)
//   embedding_bwd          nn.Embedding's scatter-add into the phoneme token table (ns2.py:253, 279-282)
//   expand_encodings_bwd   the transpose of length regulation: segmented sums over each phoneme's frames, scattered to
//                          the phoneme encodings and the coarse-pitch table (ns2.py:1449-1455)
//   add_rows_bcast         d prompt of the prompt FiLM vector's mean-pool (Reduce 'b n d -> b d' mean, ns2.py:858-862)
//   dropout_f32            the phoneme encoder's conv dropout (nn.Dropout after the causal conv's SiLU, ns2.py:258) on
//                          the forward activation and, with the same mask, on its gradient (philox.cuh element stream)
// All HBM-bound.  The scatters accumulate with fp32 atomics, so their summation order is not fixed.
#include "host_common.h"
#include "philox.cuh"
#include "../../include/ns2_b200.h"

#include <atomic>
#include <cuda_bf16.h>
#include <math.h>

namespace ns2 {

extern std::atomic<long long> g_launches;

namespace {

__device__ __forceinline__ float2 bf2_f2(uint32_t u) {
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_bf2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// d pre = d out * s * (1 + pre * (1 - s)), s = sigmoid(pre).  For pre -> -inf s underflows to 0 and the product is 0;
// for pre -> +inf s = 1 and d pre = d out.  `dpre` may alias `pre` (each pair is read before it is written).
__device__ __forceinline__ float silu_grad(float x, float dy) {
  const float s = 1.0f / (1.0f + __expf(-x));
  return dy * s * (1.0f + x * (1.0f - s));
}

__global__ void __launch_bounds__(256) silu_bwd_kernel(const uint32_t* pre, const uint32_t* __restrict__ dout,
                                                       long long pairs, uint32_t* dpre) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < pairs;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 x = bf2_f2(pre[i]), d = bf2_f2(__ldg(dout + i));
    dpre[i] = f2_bf2(silu_grad(x.x, d.x), silu_grad(x.y, d.y));
  }
}

// dtable[id(r), c] += de[r, c], id(r) = ids[r] < 0 ? pad_id : ids[r] (clamped like the forward gather)
__global__ void __launch_bounds__(256) embedding_bwd_kernel(const long long* __restrict__ ids, long long rows,
                                                            const float* __restrict__ de, int dim, int num_rows,
                                                            int pad_id, float* __restrict__ dtable) {
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < rows * dim;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = e / dim;
    const int c = static_cast<int>(e - r * dim);
    long long id = __ldg(ids + r);
    if (id < 0) id = pad_id;
    id = id < num_rows ? id : num_rows - 1;
    atomicAdd(dtable + id * dim + c, __ldg(de + e));
  }
}

// One CTA = 32 consecutive frames x 128 channels of one sample.  The frames of one phoneme are contiguous (monotonic
// hard alignment), so each thread walks its channel down the 32 frames, sums the run of equal idx and adds the run sum
// once to dphon[b, m] and to dtable[coarse[b, m]] (a run cut by a CTA boundary is added in two parts).  Reads are
// token-major: one warp reads 32 consecutive channels of a frame.
__global__ void __launch_bounds__(128) expand_encodings_bwd_kernel(const float* __restrict__ dcond, long long row_stride,
                                                                   long long batch_stride, const int* __restrict__ coarse,
                                                                   int table_rows, const int* __restrict__ idx, int T,
                                                                   int D, int L, float* __restrict__ dphon,
                                                                   float* __restrict__ dtable) {
  __shared__ int sidx[32];
  const int b = blockIdx.z, n0 = blockIdx.x * 32, d = blockIdx.y * 128 + threadIdx.x;
  if (threadIdx.x < 32) {
    const int n = n0 + threadIdx.x;
    const int m = n < L ? __ldg(idx + static_cast<long long>(b) * L + n) : -1;
    sidx[threadIdx.x] = (m >= 0 && m < T) ? m : -1;
  }
  __syncthreads();
  if (d >= D) return;
  const float* src = dcond + b * batch_stride + d;
  auto flush = [&](int m, float acc) {
    if (m < 0) return;
    if (dphon) atomicAdd(dphon + (static_cast<long long>(b) * T + m) * D + d, acc);
    if (dtable) {
      int c = __ldg(coarse + static_cast<long long>(b) * T + m);
      c = c < 0 ? 0 : (c >= table_rows ? table_rows - 1 : c);
      atomicAdd(dtable + static_cast<long long>(c) * D + d, acc);
    }
  };
  int cur = -1;
  float acc = 0.f;
  for (int r = 0; r < 32; ++r) {
    const int m = sidx[r];
    if (m != cur) {
      flush(cur, acc);
      cur = m;
      acc = 0.f;
    }
    if (m >= 0) acc += __ldg(src + static_cast<long long>(n0 + r) * row_stride);
  }
  flush(cur, acc);
}

__global__ void __launch_bounds__(256) add_rows_bcast_kernel(float* __restrict__ x, int rows, int dim,
                                                             const float* __restrict__ v, float scale, long long total) {
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = e / (static_cast<long long>(rows) * dim);
    const int c = static_cast<int>(e % dim);
    x[e] += scale * __ldg(v + b * dim + c);
  }
}

// x[i] *= keep(i) ? scale : 0; one Philox block per 4 consecutive elements (the last group may be partial).
__global__ void __launch_bounds__(256) dropout_f32_kernel(float* __restrict__ x, long long n, DropoutDev d) {
  const long long groups = (n + 3) >> 2;
  for (long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; g < groups;
       g += static_cast<long long>(gridDim.x) * blockDim.x) {
    const Philox4 r = philox4x32_10(static_cast<uint32_t>(g), static_cast<uint32_t>(g >> 32), 0xffffffffu, d.site,
                                    d.key0, d.key1);
    const float f0 = r.x >= d.threshold ? d.scale : 0.f, f1 = r.y >= d.threshold ? d.scale : 0.f;
    const float f2 = r.z >= d.threshold ? d.scale : 0.f, f3 = r.w >= d.threshold ? d.scale : 0.f;
    if (4 * g + 4 <= n) {
      float4* p4 = reinterpret_cast<float4*>(x) + g;
      float4 v = *p4;
      v.x *= f0;
      v.y *= f1;
      v.z *= f2;
      v.w *= f3;
      *p4 = v;
    } else {
      const float f[3] = {f0, f1, f2};
      for (long long i = 4 * g; i < n; ++i) x[i] *= f[i - 4 * g];
    }
  }
}

unsigned grid_cap(long long n) {
  long long g = (n + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  return static_cast<unsigned>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace
}  // namespace ns2

using namespace ns2;

extern "C" int ns2_silu_bwd(const void* pre_bf16, const void* dout_bf16, int64_t count, void* dpre_bf16,
                            ns2_stream_t stream) {
  NS2_REQUIRE(count >= 0 && count % 2 == 0, "silu_bwd: count %lld must be even", static_cast<long long>(count));
  if (count == 0) return kOk;
  NS2_REQUIRE(pre_bf16 && dout_bf16 && dpre_bf16, "silu_bwd: null pointer");
  NS2_REQUIRE(((reinterpret_cast<uintptr_t>(pre_bf16) | reinterpret_cast<uintptr_t>(dout_bf16) |
                reinterpret_cast<uintptr_t>(dpre_bf16)) & 3) == 0, "silu_bwd: pointers must be 4-byte aligned");
  silu_bwd_kernel<<<grid_cap(count / 2), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint32_t*>(pre_bf16), static_cast<const uint32_t*>(dout_bf16), count / 2,
      static_cast<uint32_t*>(dpre_bf16));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  NS2_CUDA_CHECK(cudaGetLastError());
  return kOk;
}

extern "C" int ns2_embedding_bwd(const int64_t* ids, int64_t rows, const float* de, int32_t num_rows, int32_t dim,
                                 int32_t pad_id, float* dtable, ns2_stream_t stream) {
  NS2_REQUIRE(rows >= 0 && num_rows > 0 && dim > 0, "embedding_bwd: bad sizes");
  NS2_REQUIRE(pad_id >= 0 && pad_id < num_rows, "embedding_bwd: pad_id %d outside the table", pad_id);
  if (rows == 0) return kOk;
  NS2_REQUIRE(ids && de && dtable, "embedding_bwd: null pointer");
  embedding_bwd_kernel<<<grid_cap(rows * dim), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), rows, de, dim, num_rows, pad_id, dtable);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  NS2_CUDA_CHECK(cudaGetLastError());
  return kOk;
}

extern "C" int ns2_expand_encodings_bwd(const float* dcond, int64_t dcond_row_stride, const int32_t* coarse,
                                        int32_t table_rows, const int32_t* idx, int32_t batch, int32_t t_text,
                                        int32_t dim, int32_t length, float* dphon, float* dtable, ns2_stream_t stream) {
  NS2_REQUIRE(batch >= 0 && t_text > 0 && dim > 0 && length >= 0 && table_rows > 0 && dcond_row_stride >= dim,
              "expand_encodings_bwd: bad sizes");
  NS2_REQUIRE(batch <= 65535, "expand_encodings_bwd: batch %d > 65535", batch);
  if (batch == 0 || length == 0 || (!dphon && !dtable)) return kOk;
  NS2_REQUIRE(dcond && idx && (coarse || !dtable), "expand_encodings_bwd: null pointer");
  const dim3 grid((length + 31) / 32, (dim + 127) / 128, batch);
  NS2_REQUIRE(grid.y <= 65535, "expand_encodings_bwd: dim too large");
  expand_encodings_bwd_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      dcond, dcond_row_stride, dcond_row_stride * length, coarse, table_rows, idx, t_text, dim, length, dphon, dtable);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  NS2_CUDA_CHECK(cudaGetLastError());
  return kOk;
}

extern "C" int ns2_add_rows_bcast(float* x, int32_t batch, int32_t rows, int32_t dim, const float* v, float scale,
                                  ns2_stream_t stream) {
  NS2_REQUIRE(batch >= 0 && rows >= 0 && dim > 0, "add_rows_bcast: bad sizes");
  const long long total = static_cast<long long>(batch) * rows * dim;
  if (total == 0) return kOk;
  NS2_REQUIRE(x && v, "add_rows_bcast: null pointer");
  add_rows_bcast_kernel<<<grid_cap(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, rows, dim, v, scale, total);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  NS2_CUDA_CHECK(cudaGetLastError());
  return kOk;
}

extern "C" int ns2_dropout_f32(float* x, int64_t n, const ns2_dropout* dropout, ns2_stream_t stream) {
  NS2_REQUIRE(dropout != nullptr, "dropout_f32: NULL dropout parameters");
  DropoutDev d;
  NS2_REQUIRE(make_dropout_dev(dropout->seed, dropout->site, dropout->p, &d), "dropout_f32: p=%g is not in [0, 1)",
              static_cast<double>(dropout->p));
  NS2_REQUIRE(n >= 0, "dropout_f32: negative size");
  if (n == 0 || dropout->p == 0.0f) return kOk;
  NS2_REQUIRE(x != nullptr, "dropout_f32: null pointer");
  NS2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "dropout_f32: x must be 16-byte aligned");
  dropout_f32_kernel<<<grid_cap((n + 3) / 4), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, n, d);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  NS2_CUDA_CHECK(cudaGetLastError());
  return kOk;
}
