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
// and those of the duration / pitch predictor (ns2.py:345-527), trained through its L1 losses (ns2.py:1579-1590):
//   groupnorm_silu_bwd     Block's GroupNorm + SiLU (ns2.py:345-365); the ResnetBlock residual (399-401) is the caller's
//   rowdot_bwd             the Linear(dim, 1) + ReLU heads (ns2.py:451-455)
// All HBM-bound.  The scatters accumulate with fp32 atomics, so their summation order is not fixed; the predictor's
// parameter sums go through per-CTA partials and a fixed-order second pass, so they are.
#include "host_common.h"
#include "philox.cuh"
#include "../../include/ns2_b200.h"

#include <cuda_bf16.h>
#include <math.h>

namespace ns2 {

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

// ---- duration / pitch predictor (ns2.py:345-527) ----
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The 256-thread block sum of groupnorm_silu_kernel (elementwise.cu), so that the recomputed statistics are the
// forward's bit for bit.
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

// d z of y = silu(z), z = xh * w + b, and d xh = d z * w (fp32; __expf like the forward).
__device__ __forceinline__ float gn_silu_dz(float xh, float w, float b, float dy) {
  const float z = xh * w + b;
  const float s = 1.0f / (1.0f + __expf(-z));
  return dy * s * (1.0f + z * (1.0f - s));
}

// Backward of groupnorm_silu_kernel.  One CTA per (group, batch element), like the forward:
//   passes 1-2  mean and rstd, the forward's code and summation order
//   pass 3      each thread owns one channel quad (c4 = tid % v4) and walks rows r0, r0 + rstep, ...: per-channel
//               sums of dz * xh and dz (d gamma / d beta of this sample) and the group sums of dxh and dxh * xh
//   pass 4      dx = rstd * (dxh - mean(dxh) - xh * mean(dxh * xh)), written as bf16
// The per-channel sums of the CTA's threads are added in a fixed order through shared memory and written to
// partial[b][0 / 1][channel]; sum_parts_kernel reduces them over the batch.  No atomics anywhere.
__global__ void __launch_bounds__(256) groupnorm_silu_bwd_kernel(const float* __restrict__ x, int rows, int channels,
                                                                 int cpg, const float* __restrict__ weight,
                                                                 const float* __restrict__ bias, float eps,
                                                                 const float* __restrict__ dy,
                                                                 __nv_bfloat16* __restrict__ dx,
                                                                 float* __restrict__ partial) {
  __shared__ float red[8];
  __shared__ float4 s_dg[256], s_db[256];
  const int g = blockIdx.x, b = blockIdx.y;
  const int v4 = cpg / 4;
  const long long base = (static_cast<long long>(b) * rows) * channels + g * cpg;
  const int total = rows * v4;
  float s = 0.f;
  for (int e = threadIdx.x; e < total; e += 256) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + base + static_cast<long long>(e / v4) * channels) + e % v4);
    s += (v.x + v.y) + (v.z + v.w);
  }
  const float n = static_cast<float>(rows) * cpg;
  const float mean = block_sum_256(s, red) / n;
  float q = 0.f;
  for (int e = threadIdx.x; e < total; e += 256) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + base + static_cast<long long>(e / v4) * channels) + e % v4);
    const float a = v.x - mean, c = v.y - mean, d = v.z - mean, f = v.w - mean;
    q += (a * a + c * c) + (d * d + f * f);
  }
  const float rstd = rsqrtf(block_sum_256(q, red) / n + eps);

  const int rstep = 256 / v4;                  // v4 <= 256 (checked on the host)
  const int c4 = threadIdx.x % v4, r0 = threadIdx.x / v4;
  float4 dg = make_float4(0.f, 0.f, 0.f, 0.f), db = dg;
  float s1 = 0.f, s2 = 0.f;
  if (r0 < rstep) {
    const float4 w = __ldg(reinterpret_cast<const float4*>(weight + g * cpg) + c4);
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + g * cpg) + c4);
    for (int r = r0; r < rows; r += rstep) {
      const long long off = base + static_cast<long long>(r) * channels + c4 * 4;
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + off));
      const float4 d = __ldg(reinterpret_cast<const float4*>(dy + off));
      const float h0 = (v.x - mean) * rstd, h1 = (v.y - mean) * rstd, h2 = (v.z - mean) * rstd, h3 = (v.w - mean) * rstd;
      const float z0 = gn_silu_dz(h0, w.x, bb.x, d.x), z1 = gn_silu_dz(h1, w.y, bb.y, d.y);
      const float z2 = gn_silu_dz(h2, w.z, bb.z, d.z), z3 = gn_silu_dz(h3, w.w, bb.w, d.w);
      dg.x += z0 * h0; dg.y += z1 * h1; dg.z += z2 * h2; dg.w += z3 * h3;
      db.x += z0; db.y += z1; db.z += z2; db.w += z3;
      const float e0 = z0 * w.x, e1 = z1 * w.y, e2 = z2 * w.z, e3 = z3 * w.w;
      s1 += (e0 + e1) + (e2 + e3);
      s2 += (e0 * h0 + e1 * h1) + (e2 * h2 + e3 * h3);
    }
  }
  s_dg[threadIdx.x] = dg;
  s_db[threadIdx.x] = db;
  const float m1 = block_sum_256(s1, red) / n;   // its __syncthreads also publishes s_dg / s_db
  const float m2 = block_sum_256(s2, red) / n;
  if (threadIdx.x < v4) {
    float4 tg = s_dg[threadIdx.x], tb = s_db[threadIdx.x];
    for (int j = 1; j < rstep; ++j) {
      const float4 ug = s_dg[j * v4 + threadIdx.x], ub = s_db[j * v4 + threadIdx.x];
      tg.x += ug.x; tg.y += ug.y; tg.z += ug.z; tg.w += ug.w;
      tb.x += ub.x; tb.y += ub.y; tb.z += ub.z; tb.w += ub.w;
    }
    const long long p = static_cast<long long>(b) * 2 * channels + g * cpg + threadIdx.x * 4;
    *reinterpret_cast<float4*>(partial + p) = tg;
    *reinterpret_cast<float4*>(partial + p + channels) = tb;
  }

  for (int e = threadIdx.x; e < total; e += 256) {
    const int r = e / v4, k4 = e % v4;
    const long long off = base + static_cast<long long>(r) * channels + k4 * 4;
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + off));
    const float4 d = __ldg(reinterpret_cast<const float4*>(dy + off));
    const float4 w = __ldg(reinterpret_cast<const float4*>(weight + g * cpg) + k4);
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + g * cpg) + k4);
    const float h0 = (v.x - mean) * rstd, h1 = (v.y - mean) * rstd, h2 = (v.z - mean) * rstd, h3 = (v.w - mean) * rstd;
    const float o0 = rstd * (gn_silu_dz(h0, w.x, bb.x, d.x) * w.x - m1 - h0 * m2);
    const float o1 = rstd * (gn_silu_dz(h1, w.y, bb.y, d.y) * w.y - m1 - h1 * m2);
    const float o2 = rstd * (gn_silu_dz(h2, w.z, bb.z, d.z) * w.z - m1 - h2 * m2);
    const float o3 = rstd * (gn_silu_dz(h3, w.w, bb.w, d.w) * w.w - m1 - h3 * m2);
    uint2 pk;
    pk.x = f2_bf2(o0, o1);
    pk.y = f2_bf2(o2, o3);
    *reinterpret_cast<uint2*>(dx + off) = pk;
  }
}

// out[i] = sum over j = 0 .. parts-1 of partial[j * stride + i], in that order (the fixed-order second level of the
// predictor's deterministic reductions).  Columns [0, split) go to out0, [split, cols) to out1.
__global__ void __launch_bounds__(256) sum_parts_kernel(const float* __restrict__ partial, long long parts,
                                                        long long stride, int cols, int split, float* __restrict__ out0,
                                                        float* __restrict__ out1) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= cols) return;
  float s = 0.f;
  for (long long j = 0; j < parts; ++j) s += __ldg(partial + j * stride + i);
  if (i < split) out0[i] = s;
  else out1[i - split] = s;
}

// Backward of rowdot_kernel with ReLU: dpre[r] = pred[r] > 0 ? dpred[r] : 0 (0 at an exact zero, as torch's
// threshold_backward).  One CTA per NS2_ROWDOT_BWD_ROWS rows: dx[r, :] += dpre[r] * w, and this chunk's
// sum_r dpre[r] * x[r, :] and sum_r dpre[r] (rows in order) to partial[chunk, 0 .. dim] (rows of dim + 4 floats, so
// that every row starts 16-byte aligned).
__global__ void __launch_bounds__(256) rowdot_bwd_kernel(const float* __restrict__ x, long long rows, int dim,
                                                         const float* __restrict__ w, const float* __restrict__ pred,
                                                         const float* __restrict__ dpred, float* __restrict__ dx,
                                                         float* __restrict__ partial) {
  __shared__ float s_d[NS2_ROWDOT_BWD_ROWS];
  const long long r0 = static_cast<long long>(blockIdx.x) * NS2_ROWDOT_BWD_ROWS;
  const int nr = static_cast<int>(rows - r0 < NS2_ROWDOT_BWD_ROWS ? rows - r0 : NS2_ROWDOT_BWD_ROWS);
  if (threadIdx.x < NS2_ROWDOT_BWD_ROWS) {
    float d = 0.f;
    if (threadIdx.x < nr) {
      const long long r = r0 + threadIdx.x;
      d = __ldg(pred + r) > 0.f ? __ldg(dpred + r) : 0.f;
    }
    s_d[threadIdx.x] = d;
  }
  __syncthreads();
  float* prow = partial + static_cast<long long>(blockIdx.x) * (dim + 4);
  for (int c4 = threadIdx.x; c4 < dim / 4; c4 += 256) {
    const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + c4);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = 0; i < nr; ++i) {
      const float d = s_d[i];
      const long long off = (r0 + i) * dim + c4 * 4;
      const float4 xv = __ldg(reinterpret_cast<const float4*>(x + off));
      acc.x += d * xv.x; acc.y += d * xv.y; acc.z += d * xv.z; acc.w += d * xv.w;
      float4 o = *reinterpret_cast<float4*>(dx + off);
      o.x += d * wv.x; o.y += d * wv.y; o.z += d * wv.z; o.w += d * wv.w;
      *reinterpret_cast<float4*>(dx + off) = o;
    }
    *reinterpret_cast<float4*>(prow + c4 * 4) = acc;
  }
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < nr; ++i) s += s_d[i];
    prow[dim] = s;
  }
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
  return launched(1);
}

extern "C" int ns2_embedding_bwd(const int64_t* ids, int64_t rows, const float* de, int32_t num_rows, int32_t dim,
                                 int32_t pad_id, float* dtable, ns2_stream_t stream) {
  NS2_REQUIRE(rows >= 0 && num_rows > 0 && dim > 0, "embedding_bwd: bad sizes");
  NS2_REQUIRE(pad_id >= 0 && pad_id < num_rows, "embedding_bwd: pad_id %d outside the table", pad_id);
  if (rows == 0) return kOk;
  NS2_REQUIRE(ids && de && dtable, "embedding_bwd: null pointer");
  embedding_bwd_kernel<<<grid_cap(rows * dim), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), rows, de, dim, num_rows, pad_id, dtable);
  return launched(1);
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
  return launched(1);
}

extern "C" int ns2_add_rows_bcast(float* x, int32_t batch, int32_t rows, int32_t dim, const float* v, float scale,
                                  ns2_stream_t stream) {
  NS2_REQUIRE(batch >= 0 && rows >= 0 && dim > 0, "add_rows_bcast: bad sizes");
  const long long total = static_cast<long long>(batch) * rows * dim;
  if (total == 0) return kOk;
  NS2_REQUIRE(x && v, "add_rows_bcast: null pointer");
  add_rows_bcast_kernel<<<grid_cap(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, rows, dim, v, scale, total);
  return launched(1);
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
  return launched(1);
}

extern "C" int ns2_groupnorm_silu_bwd(const float* x, int32_t batch, int32_t rows, int32_t channels, int32_t groups,
                                      const float* weight, const float* bias, float eps, const float* dy, void* dx_bf16,
                                      float* partial, float* dweight, float* dbias, ns2_stream_t stream) {
  NS2_REQUIRE(batch >= 0 && rows >= 0 && channels > 0 && groups > 0 && channels % groups == 0,
              "groupnorm_silu_bwd: bad sizes");
  NS2_REQUIRE((channels / groups) % 4 == 0 && channels / groups <= 1024,
              "groupnorm_silu_bwd: channels per group (%d) must be a multiple of 4 and <= 1024", channels / groups);
  NS2_REQUIRE(batch <= 65535, "groupnorm_silu_bwd: batch %d > 65535", batch);
  NS2_REQUIRE(dweight && dbias, "groupnorm_silu_bwd: null pointer");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (batch == 0 || rows == 0) {   // no element: zero parameter gradients
    NS2_CUDA_CHECK(cudaMemsetAsync(dweight, 0, sizeof(float) * channels, st));
    NS2_CUDA_CHECK(cudaMemsetAsync(dbias, 0, sizeof(float) * channels, st));
    return kOk;
  }
  NS2_REQUIRE(x && weight && bias && dy && dx_bf16 && partial, "groupnorm_silu_bwd: null pointer");
  NS2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(weight) | reinterpret_cast<uintptr_t>(bias) |
                reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(partial)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(dx_bf16) & 7) == 0,
              "groupnorm_silu_bwd: pointers must be 16-byte aligned (dx 8-byte)");
  groupnorm_silu_bwd_kernel<<<dim3(groups, batch), 256, 0, st>>>(x, rows, channels, channels / groups, weight, bias, eps,
                                                                 dy, static_cast<__nv_bfloat16*>(dx_bf16), partial);
  NS2_CUDA_CHECK(cudaGetLastError());
  sum_parts_kernel<<<(2 * channels + 255) / 256, 256, 0, st>>>(partial, batch, 2LL * channels, 2 * channels, channels,
                                                               dweight, dbias);
  return launched(2);
}

extern "C" int ns2_rowdot_bwd(const float* x, int64_t rows, int32_t dim, const float* w, const float* pred,
                              const float* dpred, float* dx, float* partial, float* dw, float* db, ns2_stream_t stream) {
  NS2_REQUIRE(rows >= 0 && dim > 0 && dim % 4 == 0, "rowdot_bwd: bad sizes");
  NS2_REQUIRE(dw && db, "rowdot_bwd: null pointer");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (rows == 0) {
    NS2_CUDA_CHECK(cudaMemsetAsync(dw, 0, sizeof(float) * dim, st));
    NS2_CUDA_CHECK(cudaMemsetAsync(db, 0, sizeof(float), st));
    return kOk;
  }
  NS2_REQUIRE(x && w && pred && dpred && dx && partial, "rowdot_bwd: null pointer");
  NS2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(dx) |
                reinterpret_cast<uintptr_t>(partial)) & 15) == 0,
              "rowdot_bwd: x, w, dx and partial must be 16-byte aligned");
  const long long chunks = (rows + NS2_ROWDOT_BWD_ROWS - 1) / NS2_ROWDOT_BWD_ROWS;
  NS2_REQUIRE(chunks <= 0x7fffffffLL, "rowdot_bwd: too many rows");
  rowdot_bwd_kernel<<<static_cast<unsigned>(chunks), 256, 0, st>>>(x, rows, dim, w, pred, dpred, dx, partial);
  NS2_CUDA_CHECK(cudaGetLastError());
  sum_parts_kernel<<<(dim + 1 + 255) / 256, 256, 0, st>>>(partial, chunks, dim + 4LL, dim + 1, dim, dw, db);
  return launched(2);
}
