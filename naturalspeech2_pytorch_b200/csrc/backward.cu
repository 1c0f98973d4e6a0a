// Element-wise / reduction kernels of the backward pass (SURVEY rows a18 / f1: what autograd runs for the reference's
// `loss.backward()`, README.md:63, ns2.py:1886).  The matrix products of the backward pass are ns2_gemm (dgrad, with
// transposed weight packs) and ns2_wgrad; this file holds what sits between them: the backward of RMSNorm(+FiLM)
// (ns2.py:736-746), of GEGLU (1004-1007), of the Wavenet gate tanh(z)sigmoid(z) with FiLM (625-630), bias gradients
// (column sums), the FiLM table gradient, the MSE loss gradient (1646-1666) and small helpers.  All HBM-bound.
#include "host_common.h"
#include "../../include/ns2_b200.h"

#include <cuda_bf16.h>
#include <math.h>

namespace ns2 {

__device__ __forceinline__ float bwd_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float2 bf2_to_f2(uint32_t u) {
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ------------------------------------------------------------------------------------------------
// RMSNorm (+learned gamma) (+FiLM) backward.  Forward: u = x * sqrt(D) / max(||x||, eps); h = u * gamma * fg + fb.
//   du = dh * gamma * fg;  dx = s * (du - u * (u . du) / D)  with s = sqrt(D) / ||x||
//   d fg[b, c] += sum_rows dh * u * gamma;  d fb[b, c] += sum_rows dh;  d gamma[c] += sum_rows dh * u * fg
// One CTA = 64 consecutive rows of one batch (8 warps x 8 rows); column partials are combined in shared memory and
// added to the global gradient tables with one atomicAdd per column per CTA.
// dxr (fp32 residual-stream gradient) is updated IN PLACE (+= dx) and its bf16 copy is written for the next GEMMs.
// ------------------------------------------------------------------------------------------------
template <int VEC>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const float* __restrict__ x, const uint2* __restrict__ dh,
                                                          int rows_per_batch, int dim, const float* __restrict__ gamma,
                                                          const float* __restrict__ film, long long film_bs,
                                                          float* __restrict__ dfilm, long long dfilm_bs,
                                                          float* __restrict__ dgamma, float* __restrict__ dxr,
                                                          uint2* __restrict__ dxr_bf) {
  __shared__ float red[8][VEC * 128];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunks = (rows_per_batch + 63) / 64;
  const int b = blockIdx.x / chunks;
  const int r0 = (blockIdx.x - b * chunks) * 64;
  const float* fg = film ? film + b * film_bs : nullptr;
  float4 acc_g[VEC], acc_b[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc_g[i] = acc_b[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int rr = warp; rr < 64; rr += 8) {
    const int r = r0 + rr;
    if (r >= rows_per_batch) break;
    const long long row = static_cast<long long>(b) * rows_per_batch + r;
    const float4* xp = reinterpret_cast<const float4*>(x + row * dim);
    float4 xv[VEC], du[VEC];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      xv[i] = __ldg(xp + i * 32 + lane);
      ss += xv[i].x * xv[i].x + xv[i].y * xv[i].y + xv[i].z * xv[i].z + xv[i].w * xv[i].w;
    }
    ss = bwd_warp_sum(ss);
    const float s = sqrtf(static_cast<float>(dim)) / fmaxf(sqrtf(ss), 1e-12f);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const int c4 = i * 32 + lane;
      const uint2 d2 = __ldg(dh + row * (dim / 4) + c4);
      const float2 d01 = bf2_to_f2(d2.x), d23 = bf2_to_f2(d2.y);
      const float d[4] = {d01.x, d01.y, d23.x, d23.y};
      float g[4] = {1.f, 1.f, 1.f, 1.f}, f[4] = {1.f, 1.f, 1.f, 1.f};
      if (gamma) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(gamma) + c4);
        g[0] = t.x; g[1] = t.y; g[2] = t.z; g[3] = t.w;
      }
      if (fg) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(fg) + c4);
        f[0] = t.x; f[1] = t.y; f[2] = t.z; f[3] = t.w;
      }
      const float u[4] = {xv[i].x * s, xv[i].y * s, xv[i].z * s, xv[i].w * s};
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        o[j] = d[j] * g[j] * f[j];
        dot += u[j] * o[j];
      }
      du[i] = make_float4(o[0], o[1], o[2], o[3]);
      // column partials: d(film gamma) uses dh*u*gamma, d(learned gamma) uses dh*u*fg; only one of the two tables is
      // accumulated per call site (FiLM norms have no learned gamma and vice versa), so one accumulator serves both
      acc_g[i].x += d[0] * u[0] * (fg ? g[0] : f[0]);
      acc_g[i].y += d[1] * u[1] * (fg ? g[1] : f[1]);
      acc_g[i].z += d[2] * u[2] * (fg ? g[2] : f[2]);
      acc_g[i].w += d[3] * u[3] * (fg ? g[3] : f[3]);
      acc_b[i].x += d[0]; acc_b[i].y += d[1]; acc_b[i].z += d[2]; acc_b[i].w += d[3];
      xv[i] = make_float4(u[0], u[1], u[2], u[3]);
    }
    dot = bwd_warp_sum(dot) / static_cast<float>(dim);
    float4* dp = reinterpret_cast<float4*>(dxr + row * dim);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const int c4 = i * 32 + lane;
      float4 cur = dp[c4];
      cur.x += s * (du[i].x - xv[i].x * dot);
      cur.y += s * (du[i].y - xv[i].y * dot);
      cur.z += s * (du[i].z - xv[i].z * dot);
      cur.w += s * (du[i].w - xv[i].w * dot);
      dp[c4] = cur;
      dxr_bf[row * (dim / 4) + c4] = make_uint2(f2_to_bf2(cur.x, cur.y), f2_to_bf2(cur.z, cur.w));
    }
  }
  // combine the 8 warps' column partials, then one atomic per column
  for (int pass = 0; pass < 2; ++pass) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float4 v = pass == 0 ? acc_g[i] : acc_b[i];
      float* dst = &red[warp][(i * 32 + lane) * 4];
      dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < dim; c += 256) {
      float sum = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) sum += red[w][c];
      if (pass == 0) {
        if (fg) atomicAdd(dfilm + b * dfilm_bs + c, sum);
        else if (dgamma) atomicAdd(dgamma + c, sum);
      } else if (fg) {
        atomicAdd(dfilm + b * dfilm_bs + dim + c, sum);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// GEGLU backward on the packed pre-activation layout (tiles of 256 columns = 128 value | 128 gate, model.py _pack_ff):
//   out = val * gelu(gate)  =>  d val = dg * gelu(gate);  d gate = dg * val * (Phi(gate) + gate * phi(gate))
// `pre` is overwritten with the gradient (same layout).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) geglu_bwd_kernel(uint32_t* __restrict__ pre, const uint32_t* __restrict__ dg,
                                                        long long rows, int dp) {
  const int pairs_per_row = dp / 2;  // bf16x2 words of dg per row
  const long long total = rows * pairs_per_row;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / pairs_per_row;
    const int c = static_cast<int>(i - r * pairs_per_row) * 2;      // output column (even)
    const int tile = c >> 7, in = c & 127;
    uint32_t* vp = pre + (r * (2 * dp) + tile * 256 + in) / 2;
    uint32_t* gp = vp + 64;                                          // +128 columns
    const float2 v = bf2_to_f2(*vp), g = bf2_to_f2(*gp), d = bf2_to_f2(__ldg(dg + i));
    auto f = [](float val, float gate, float dd, float& dval, float& dgate) {
      const float cdf = 0.5f * (1.0f + erff(gate * 0.70710678118654752440f));
      const float pdf = 0.3989422804014327f * expf(-0.5f * gate * gate);
      dval = dd * gate * cdf;
      dgate = dd * val * (cdf + gate * pdf);
    };
    float dv0, dg0, dv1, dg1;
    f(v.x, g.x, d.x, dv0, dg0);
    f(v.y, g.y, d.y, dv1, dg1);
    *vp = f2_to_bf2(dv0, dv1);
    *gp = f2_to_bf2(dg0, dg1);
  }
}

// ------------------------------------------------------------------------------------------------
// Wavenet gate backward.  Forward (per dilation column g): z = c * fg + fb, y = tanh(z) sigmoid(z) + res.
//   dz = dy * [(1 - tanh^2) sigmoid + tanh sigmoid (1 - sigmoid)];  dc = dz * fg;  d fg += sum_rows dz * c;  d fb += sum_rows dz
// c: conv output incl. bias (recomputed), (B, N, G*D) bf16; dy: (B, N, G*D) bf16 view (row stride dy_rs);
// dc written to (B, N, G*D) bf16 view (row stride dc_rs).  film / dfilm: per batch, group g at g*film_gs: [gamma | beta].
// One CTA = 64 rows of one batch x one group (two rows of every warp in flight at once).
// ------------------------------------------------------------------------------------------------
// Thread layout: a thread owns ONE quad of channels and walks the rows of its row lane (256 / (dim/4) row lanes per
// CTA), four rows in flight at a time - few registers, many CTAs per SM, so enough loads are outstanding to stream
// the three (B, N, G*D) bf16 tensors near HBM speed (the previous one-row-per-warp layout reached 2 TB/s).
__global__ void __launch_bounds__(256) wavenet_gate_bwd_kernel(const uint2* __restrict__ c, long long c_rs4,
                                                               const uint2* __restrict__ dy, long long dy_rs4,
                                                               uint2* __restrict__ dc, long long dc_rs4, int rows_per_batch,
                                                               int dim, int groups, const float* __restrict__ film,
                                                               long long film_bs, int film_gs, float* __restrict__ dfilm,
                                                               long long dfilm_bs) {
  extern __shared__ __align__(16) float gate_red[];   // [row lanes][dim]
  const int Q = dim / 4, RL = 256 / Q;
  const int q = threadIdx.x % Q, rl = threadIdx.x / Q;
  const int chunks = (rows_per_batch + 63) / 64;
  int idx = blockIdx.x;
  const int g = idx % groups;
  idx /= groups;
  const int b = idx / chunks;
  const int r0 = (idx - b * chunks) * 64;
  const int nrows = min(64, rows_per_batch - r0);
  const float* fgp = film + b * film_bs + g * film_gs;
  const float4 fg4 = __ldg(reinterpret_cast<const float4*>(fgp) + q);
  const float4 fb4 = __ldg(reinterpret_cast<const float4*>(fgp + dim) + q);
  const float ga[4] = {fg4.x, fg4.y, fg4.z, fg4.w}, be[4] = {fb4.x, fb4.y, fb4.z, fb4.w};
  float acc_g[4] = {0.f, 0.f, 0.f, 0.f}, acc_b[4] = {0.f, 0.f, 0.f, 0.f};
  const int c4 = g * Q + q;
  if (rl < RL) {
#pragma unroll 4
    for (int rr = rl; rr < nrows; rr += RL) {
      const long long row = static_cast<long long>(b) * rows_per_batch + r0 + rr;
      const uint2 cw = __ldg(c + row * c_rs4 + c4), dw = __ldg(dy + row * dy_rs4 + c4);
      const float2 c01 = bf2_to_f2(cw.x), c23 = bf2_to_f2(cw.y), d01 = bf2_to_f2(dw.x), d23 = bf2_to_f2(dw.y);
      const float cv[4] = {c01.x, c01.y, c23.x, c23.y}, dv[4] = {d01.x, d01.y, d23.x, d23.y};
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        // one exponential per element: u = e^-z, sigmoid = 1/(1+u), tanh = (1-u^2)/(1+u^2); |z| clamped where both
        // have saturated to fp32 precision
        const float z = fminf(fmaxf(fmaf(cv[j], ga[j], be[j]), -20.0f), 20.0f);
        const float u = __expf(-z), u2 = u * u;
        const float sg = __fdividef(1.0f, 1.0f + u);
        const float th = (1.0f - u2) * __fdividef(1.0f, 1.0f + u2);
        const float dz = dv[j] * ((1.0f - th * th) * sg + th * sg * (1.0f - sg));
        o[j] = dz * ga[j];
        acc_g[j] = fmaf(dz, cv[j], acc_g[j]);
        acc_b[j] += dz;
      }
      dc[row * dc_rs4 + c4] = make_uint2(f2_to_bf2(o[0], o[1]), f2_to_bf2(o[2], o[3]));
    }
  }
  for (int pass = 0; pass < 2; ++pass) {
    __syncthreads();
    if (rl < RL) {
      const float* v = pass == 0 ? acc_g : acc_b;
      *reinterpret_cast<float4*>(gate_red + rl * dim + 4 * q) = make_float4(v[0], v[1], v[2], v[3]);
    }
    __syncthreads();
    for (int cc = threadIdx.x; cc < dim; cc += 256) {
      float sum = 0.f;
      for (int w = 0; w < RL; ++w) sum += gate_red[w * dim + cc];
      atomicAdd(dfilm + b * dfilm_bs + g * film_gs + pass * dim + cc, sum);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Column sums (bias gradients): out[c] += sum over rows of t[r, c]; t bf16 (rows, cols) with row stride rs (elements).
// grid = (col chunks of 256 (bf16x2 per thread -> 128 threads... ), row chunks); 128 rows per CTA then one atomic per col.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const uint32_t* __restrict__ t, long long rows, int cols,
                                                          long long rs2, float* __restrict__ out) {
  const int c2 = blockIdx.x * 256 + threadIdx.x;   // bf16x2 column index
  if (c2 * 2 >= cols) return;
  const long long r0 = static_cast<long long>(blockIdx.y) * 256;
  const long long r1 = r0 + 256 < rows ? r0 + 256 : rows;
  float a0 = 0.f, a1 = 0.f;
  for (long long r = r0; r < r1; ++r) {
    const float2 v = bf2_to_f2(__ldg(t + r * rs2 + c2));
    a0 += v.x;
    a1 += v.y;
  }
  atomicAdd(out + 2 * c2, a0);
  atomicAdd(out + 2 * c2 + 1, a1);
}

// sum over groups: out[r, c] = sum_g t[r, g*dim + c]   (gradient of an input broadcast to all dilation columns)
__global__ void __launch_bounds__(256) group_sum_kernel(const uint32_t* __restrict__ t, long long rows, int dim2,
                                                        int groups, uint32_t* __restrict__ out) {
  const long long total = rows * dim2;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / dim2;
    const int c = static_cast<int>(i - r * dim2);
    float a0 = 0.f, a1 = 0.f;
    for (int g = 0; g < groups; ++g) {
      const float2 v = bf2_to_f2(__ldg(t + (r * groups + g) * dim2 + c));
      a0 += v.x;
      a1 += v.y;
    }
    out[i] = f2_to_bf2(a0, a1);
  }
}

// d pred = coef[b] * (pred - target) -> fp32 residual-stream gradient seed and its bf16 copy  (MSE backward, ns2.py:1646-1666)
// With lens: elements past sample b's first lens[b] rows of row4 float4s are written as exact zeros
// (pred / target are not read there).
__global__ void __launch_bounds__(256) mse_bwd_kernel(const float4* __restrict__ pred, const float4* __restrict__ target,
                                                      const float* __restrict__ coef, long long per4,
                                                      uint2* __restrict__ out_bf, float4* __restrict__ out_f32,
                                                      const int* __restrict__ lens, long long row4, int rows) {
  const int b = blockIdx.y;
  const float cf = coef[b];
  const long long base = static_cast<long long>(b) * per4;
  const long long n4 = lens == nullptr ? per4 : static_cast<long long>(min(max(__ldg(lens + b), 1), rows)) * row4;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < per4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < n4) {
      const float4 p = __ldg(pred + base + i), t = __ldg(target + base + i);
      d = make_float4(cf * (p.x - t.x), cf * (p.y - t.y), cf * (p.z - t.z), cf * (p.w - t.w));
    }
    if (out_bf != nullptr) out_bf[base + i] = make_uint2(f2_to_bf2(d.x, d.y), f2_to_bf2(d.z, d.w));
    if (out_f32 != nullptr) out_f32[base + i] = d;
  }
}

// acc (fp32) += t (bf16); acc_bf = bf16(acc): joins a branch gradient into a residual-stream gradient
__global__ void __launch_bounds__(256) accum_bf16_kernel(float4* __restrict__ acc, const uint2* __restrict__ t, long long n4,
                                                         uint2* __restrict__ acc_bf) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float4 a = acc[i];
    const uint2 w = __ldg(t + i);
    const float2 lo = bf2_to_f2(w.x), hi = bf2_to_f2(w.y);
    a.x += lo.x; a.y += lo.y; a.z += hi.x; a.w += hi.y;
    acc[i] = a;
    if (acc_bf != nullptr) acc_bf[i] = make_uint2(f2_to_bf2(a.x, a.y), f2_to_bf2(a.z, a.w));
  }
}

// dW[r, c] (+)= sum_b dfilm[b, r] * t[b, c]   (FiLM projection weights, contraction over the batch only).
// HBM-bound on the dW stream (rows x cols fp32, > 1 GB at cfg3): one CTA owns a 64-row x 256-column tile, both operand
// slices sit in shared memory, every thread keeps 16 rows x 4 columns of accumulators (5 shared loads per 64 FMAs) and
// writes 128-bit rows.  ACCUM = 0 writes dW without reading it (fresh gradient buffer: one pass over dW instead of
// zero-fill + read + write).
template <bool ACCUM>
__global__ void __launch_bounds__(256) film_wgrad_kernel(const float* __restrict__ dfilm, long long dfilm_bs,
                                                         const float* __restrict__ t, int batch, long long rows, int cols,
                                                         float* __restrict__ dw) {
  extern __shared__ __align__(16) float fw_smem[];
  float* ts = fw_smem;                 // [batch][256] slice of t
  float* ds = fw_smem + batch * 256;   // [batch][64]  slice of dfilm
  const int c0 = blockIdx.x * 256;
  const long long r0 = static_cast<long long>(blockIdx.y) * 64;
  for (int i = threadIdx.x; i < batch * 256; i += 256) {
    const int b = i >> 8, c = i & 255;
    ts[i] = (c0 + c < cols) ? __ldg(t + static_cast<long long>(b) * cols + c0 + c) : 0.f;
  }
  for (int i = threadIdx.x; i < batch * 64; i += 256) {
    const int b = i >> 6, r = i & 63;
    ds[i] = (r0 + r < rows) ? __ldg(dfilm + b * dfilm_bs + r0 + r) : 0.f;
  }
  __syncthreads();
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;   // 4 columns at 4*tx, 16 rows at 16*ty
  float acc[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int b = 0; b < batch; ++b) {
    const float4 tv = *reinterpret_cast<const float4*>(ts + b * 256 + 4 * tx);
    float dv[16];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 d4 = *reinterpret_cast<const float4*>(ds + b * 64 + ty * 16 + 4 * q);
      dv[4 * q] = d4.x; dv[4 * q + 1] = d4.y; dv[4 * q + 2] = d4.z; dv[4 * q + 3] = d4.w;
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      acc[i][0] = fmaf(dv[i], tv.x, acc[i][0]);
      acc[i][1] = fmaf(dv[i], tv.y, acc[i][1]);
      acc[i][2] = fmaf(dv[i], tv.z, acc[i][2]);
      acc[i][3] = fmaf(dv[i], tv.w, acc[i][3]);
    }
  }
  const int c = c0 + 4 * tx;
  const bool vec = (c + 3 < cols) && (cols % 4 == 0);
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const long long r = r0 + ty * 16 + i;
    if (r >= rows) break;
    float* o = dw + r * cols + c;
    if (vec) {
      float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      if (ACCUM) {
        const float4 old = *reinterpret_cast<const float4*>(o);
        v.x += old.x; v.y += old.y; v.z += old.z; v.w += old.w;
      }
      *reinterpret_cast<float4*>(o) = v;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (c + j < cols) o[j] = ACCUM ? o[j] + acc[i][j] : acc[i][j];
    }
  }
}

static unsigned grid_1d(long long n, int cap = 148 * 16) {
  long long g = (n + 255) / 256;
  return static_cast<unsigned>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace ns2

using namespace ns2;

extern "C" int ns2_rmsnorm_film_bwd(const float* x, const void* dh_bf16, int64_t rows, int32_t dim, int32_t rows_per_batch,
                                    const float* gamma, const float* film, int64_t film_batch_stride, float* dfilm,
                                    int64_t dfilm_batch_stride, float* dgamma, float* dxr, void* dxr_bf16,
                                    ns2_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NS2_REQUIRE(x && dh_bf16 && dxr && dxr_bf16 && rows > 0 && rows_per_batch > 0 && rows % rows_per_batch == 0,
              "rmsnorm_film_bwd: bad arguments");
  NS2_REQUIRE(dim % 128 == 0 && dim <= 1024, "rmsnorm_film_bwd: dim=%d must be a multiple of 128, <= 1024", dim);
  NS2_REQUIRE(!(film && gamma), "rmsnorm_film_bwd: a norm has either FiLM or a learned gamma");
  NS2_REQUIRE(!film || dfilm, "rmsnorm_film_bwd: film needs dfilm");
  const int batches = static_cast<int>(rows / rows_per_batch);
  const unsigned grid = batches * ((rows_per_batch + 63) / 64);
#define NS2_CASE(V)                                                                                              \
  case V:                                                                                                        \
    rmsnorm_bwd_kernel<V><<<grid, 256, 0, stream>>>(x, reinterpret_cast<const uint2*>(dh_bf16), rows_per_batch, dim, \
                                                    gamma, film, film_batch_stride, dfilm, dfilm_batch_stride,   \
                                                    dgamma, dxr, reinterpret_cast<uint2*>(dxr_bf16));            \
    break;
  switch (dim / 128) {
    NS2_CASE(1) NS2_CASE(2) NS2_CASE(3) NS2_CASE(4) NS2_CASE(5) NS2_CASE(6) NS2_CASE(7) NS2_CASE(8)
    default: return set_error(kErrInvalidArg, "rmsnorm_film_bwd: unsupported dim %d", dim);
  }
#undef NS2_CASE
  return launched(1);
}

extern "C" int ns2_geglu_bwd(void* pre_bf16, const void* dg_bf16, int64_t rows, int32_t dp, ns2_stream_t stream_) {
  NS2_REQUIRE(pre_bf16 && dg_bf16 && rows > 0 && dp > 0 && dp % 128 == 0, "geglu_bwd: bad arguments");
  geglu_bwd_kernel<<<grid_1d(rows * (dp / 2)), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<uint32_t*>(pre_bf16), reinterpret_cast<const uint32_t*>(dg_bf16), rows, dp);
  return launched(1);
}

extern "C" int ns2_wavenet_gate_bwd(const void* c_bf16, int64_t c_row_stride, const void* dy_bf16, int64_t dy_row_stride,
                                    void* dc_bf16, int64_t dc_row_stride, int32_t batches, int32_t rows_per_batch,
                                    int32_t dim, int32_t groups, const float* film, int64_t film_batch_stride,
                                    int32_t film_group_stride, float* dfilm, int64_t dfilm_batch_stride,
                                    ns2_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NS2_REQUIRE(c_bf16 && dy_bf16 && dc_bf16 && film && dfilm && batches > 0 && rows_per_batch > 0 && groups > 0,
              "wavenet_gate_bwd: bad arguments");
  NS2_REQUIRE(dim % 128 == 0 && dim <= 1024 && c_row_stride % 4 == 0 && dy_row_stride % 4 == 0 && dc_row_stride % 4 == 0,
              "wavenet_gate_bwd: dim must be a multiple of 128 (<= 1024), strides multiples of 4");
  const unsigned grid = batches * ((rows_per_batch + 63) / 64) * groups;
  const int row_lanes = 256 / (dim / 4);
  wavenet_gate_bwd_kernel<<<grid, 256, static_cast<size_t>(row_lanes) * dim * sizeof(float), stream>>>(
      reinterpret_cast<const uint2*>(c_bf16), c_row_stride / 4, reinterpret_cast<const uint2*>(dy_bf16), dy_row_stride / 4,
      reinterpret_cast<uint2*>(dc_bf16), dc_row_stride / 4, rows_per_batch, dim, groups, film, film_batch_stride,
      film_group_stride, dfilm, dfilm_batch_stride);
  return launched(1);
}

extern "C" int ns2_colsum_bf16(const void* t_bf16, int64_t rows, int32_t cols, int64_t row_stride, float* out,
                               ns2_stream_t stream_) {
  NS2_REQUIRE(t_bf16 && out && rows > 0 && cols > 0 && cols % 2 == 0 && row_stride % 2 == 0, "colsum_bf16: bad arguments");
  dim3 grid((cols / 2 + 255) / 256, static_cast<unsigned>((rows + 255) / 256));
  colsum_bf16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(reinterpret_cast<const uint32_t*>(t_bf16), rows,
                                                                          cols, row_stride / 2, out);
  return launched(1);
}

extern "C" int ns2_group_sum_bf16(const void* t_bf16, int64_t rows, int32_t dim, int32_t groups, void* out_bf16,
                                  ns2_stream_t stream_) {
  NS2_REQUIRE(t_bf16 && out_bf16 && rows > 0 && dim > 0 && dim % 2 == 0 && groups > 0, "group_sum_bf16: bad arguments");
  group_sum_kernel<<<grid_1d(rows * (dim / 2)), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const uint32_t*>(t_bf16), rows, dim / 2, groups, reinterpret_cast<uint32_t*>(out_bf16));
  return launched(1);
}

extern "C" int ns2_mse_bwd(const float* pred, const float* target, const float* coef, int32_t batch, int64_t per_sample,
                           void* out_bf16, float* out_f32, int64_t row_elems, const int32_t* lens, ns2_stream_t stream_) {
  NS2_REQUIRE(pred && target && coef && (out_bf16 || out_f32) && batch > 0 && per_sample % 4 == 0, "mse_bwd: bad arguments");
  NS2_REQUIRE(lens == nullptr || (row_elems > 0 && row_elems % 4 == 0 && per_sample % row_elems == 0),
              "mse_bwd: row_elems=%lld must be a positive multiple of 4 dividing per_sample=%lld",
              static_cast<long long>(row_elems), static_cast<long long>(per_sample));
  const long long row4 = lens == nullptr ? 0 : row_elems / 4;
  const int rows = lens == nullptr ? 0 : static_cast<int>(per_sample / row_elems);
  dim3 grid(grid_1d(per_sample / 4, 64), batch);
  mse_bwd_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(reinterpret_cast<const float4*>(pred),
                                                                      reinterpret_cast<const float4*>(target), coef,
                                                                      per_sample / 4, reinterpret_cast<uint2*>(out_bf16),
                                                                      reinterpret_cast<float4*>(out_f32), lens, row4,
                                                                      rows);
  return launched(1);
}

extern "C" int ns2_accum_bf16(float* acc, const void* t_bf16, int64_t count, void* acc_bf16, ns2_stream_t stream_) {
  NS2_REQUIRE(acc && t_bf16 && count > 0 && count % 4 == 0, "accum_bf16: bad arguments");
  accum_bf16_kernel<<<grid_1d(count / 4), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<float4*>(acc), reinterpret_cast<const uint2*>(t_bf16), count / 4, reinterpret_cast<uint2*>(acc_bf16));
  return launched(1);
}

extern "C" int ns2_film_wgrad(const float* dfilm, int64_t dfilm_batch_stride, const float* t, int32_t batch, int64_t rows,
                              int32_t cols, float* dw, int32_t accumulate, ns2_stream_t stream_) {
  NS2_REQUIRE(dfilm && t && dw && batch > 0 && batch <= 32 && rows > 0 && cols > 0, "film_wgrad: bad arguments (batch <= 32)");
  NS2_REQUIRE((reinterpret_cast<uintptr_t>(dw) & 15) == 0, "film_wgrad: dw must be 16-byte aligned");
  NS2_REQUIRE(dfilm_batch_stride >= rows, "film_wgrad: dfilm_batch_stride %lld < rows", static_cast<long long>(dfilm_batch_stride));
  dim3 grid((cols + 255) / 256, static_cast<unsigned>((rows + 63) / 64));
  const size_t smem = static_cast<size_t>(batch) * (256 + 64) * sizeof(float);
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (accumulate) film_wgrad_kernel<true><<<grid, 256, smem, st>>>(dfilm, dfilm_batch_stride, t, batch, rows, cols, dw);
  else film_wgrad_kernel<false><<<grid, 256, smem, st>>>(dfilm, dfilm_batch_stride, t, batch, rows, cols, dw);
  return launched(1);
}
