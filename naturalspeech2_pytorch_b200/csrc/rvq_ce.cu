// Cross-entropy head of the residual VQ (`codec.rq(x_start, codes)`, ns2.py:1670-1684; vector-quantize-pytorch
// ResidualVQ.forward(x, indices=codes)): per stage q the logits over the K codewords are the NEGATIVE EUCLIDEAN
// DISTANCES -||r_q - c_k|| (cdist), the loss is cross_entropy(logits, codes[:, q]) averaged over the frames whose
// target is not -1, summed over the stages; the residual chain follows the codec's OWN nearest codewords
// (r_{q+1} = r_q - C_q[own_q]), which ns2_rvq_encode supplies bit-exactly.
//
// fp32 CUDA-core kernel (this head is off by default in the reference — rvq_cross_entropy_loss_weight = 0 — so it is
// built for exactness and simplicity, not for the tensor cores): one CTA per 32 frames, 256 threads as an 8 x 32 grid of
// 4-frame x 4-code register tiles, codebook streamed through shared memory in chunks of 128 codes, online
// log-sum-exp per frame.  The backward (ns2_rvq_ce_bwd) uses the same layout and recomputes the distances in one pass
// over the codebook per stage, so the forward saves nothing for it.
#include "host_common.h"
#include "../../include/ns2_b200.h"

#include <math.h>

namespace ns2 {

namespace rvqce {
constexpr int D = 128;
constexpr int FT = 32;    // frames per CTA
constexpr int KC = 128;   // codes per shared-memory chunk
constexpr int RS = D + 4; // padded row strides (floats): conflict-free 4-row register tiles
constexpr int SMEM_BYTES = (FT * RS + KC * RS) * 4 + FT * 8 * 4;
}  // namespace rvqce

__global__ void __launch_bounds__(256) rvq_ce_kernel(const float* __restrict__ frames, long long num_frames,
                                                     const float* __restrict__ codebooks,
                                                     const float* __restrict__ cn2, int Q, int K,
                                                     const long long* __restrict__ own_codes,
                                                     const long long* __restrict__ target_codes,
                                                     float* __restrict__ ce) {
  using namespace rvqce;
  extern __shared__ float sm[];
  float* r_s = sm;                       // [FT][RS] residuals
  float* c_s = sm + FT * RS;             // [KC][RS] codeword chunk
  float* red = c_s + KC * RS;            // [FT][8]: per-frame scratch (max / sum / target-logit partials)
  const int tid = threadIdx.x;
  const int fg = tid >> 5;               // frame group 0..7 -> frames 4*fg .. 4*fg+3
  const int cg = tid & 31;               // code group 0..31 -> codes cg, cg+32, cg+64, cg+96 of the chunk
  const long long f0 = static_cast<long long>(blockIdx.x) * FT;

  for (int i = tid; i < FT * D; i += 256) {
    const int f = i / D, d = i - f * D;
    r_s[f * RS + d] = (f0 + f < num_frames) ? frames[(f0 + f) * D + d] : 0.f;
  }
  __syncthreads();

  for (int q = 0; q < Q; ++q) {
    // ||r||^2 of my 4 frames (every thread of the frame group computes it: cheap, avoids a barrier)
    float rn2[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float s = 0.f;
      const float* rr = r_s + (4 * fg + a) * RS;
      for (int d = 0; d < D; ++d) s = fmaf(rr[d], rr[d], s);
      rn2[a] = s;
    }
    long long tgt[4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
      tgt[a] = (f0 + 4 * fg + a < num_frames) ? target_codes[(f0 + 4 * fg + a) * Q + q] : -1;
    float m_run[4], s_run[4], t_logit[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      m_run[a] = -INFINITY;
      s_run[a] = 0.f;
      t_logit[a] = -INFINITY;
    }
    for (int k0 = 0; k0 < K; k0 += KC) {
      __syncthreads();   // previous chunk fully consumed
      for (int i = tid; i < KC * D; i += 256) {
        const int c = i / D, d = i - c * D;
        c_s[c * RS + d] = (k0 + c < K) ? codebooks[(static_cast<long long>(q) * K + k0 + c) * D + d] : 0.f;
      }
      __syncthreads();
      float acc[4][4];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
      for (int d = 0; d < D; d += 4) {
        float4 rv[4], cv[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) rv[a] = *reinterpret_cast<const float4*>(r_s + (4 * fg + a) * RS + d);
#pragma unroll
        for (int b = 0; b < 4; ++b) cv[b] = *reinterpret_cast<const float4*>(c_s + (cg + 32 * b) * RS + d);
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            acc[a][b] = fmaf(rv[a].x, cv[b].x, acc[a][b]);
            acc[a][b] = fmaf(rv[a].y, cv[b].y, acc[a][b]);
            acc[a][b] = fmaf(rv[a].z, cv[b].z, acc[a][b]);
            acc[a][b] = fmaf(rv[a].w, cv[b].w, acc[a][b]);
          }
      }
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int code = k0 + cg + 32 * b;
        if (code >= K) continue;
        const float c2 = __ldg(cn2 + static_cast<long long>(q) * K + code);
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const float d2 = fmaxf(rn2[a] - 2.f * acc[a][b] + c2, 0.f);
          const float logit = -sqrtf(d2);
          if (code == tgt[a]) t_logit[a] = logit;
          if (logit > m_run[a]) {
            s_run[a] = s_run[a] * expf(m_run[a] - logit) + 1.f;
            m_run[a] = logit;
          } else {
            s_run[a] += expf(logit - m_run[a]);
          }
        }
      }
    }
    // combine the 32 code groups of each frame: warp shuffles (a frame group is exactly one warp)
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float m = m_run[a], s = s_run[a], t = t_logit[a];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, off);
        const float s2 = __shfl_xor_sync(0xffffffffu, s, off);
        const float t2 = __shfl_xor_sync(0xffffffffu, t, off);
        const float mn = fmaxf(m, m2);
        s = s * expf(m - mn) + s2 * expf(m2 - mn);
        m = mn;
        t = fmaxf(t, t2);
      }
      const long long f = f0 + 4 * fg + a;
      if (cg == 0 && f < num_frames)
        ce[f * Q + q] = (tgt[a] < 0) ? 0.f : (m + logf(s)) - t;   // logsumexp - logit[target]
    }
    // residual update with the codec's own code of this stage (exact fp32, same as the encoder's chain)
    __syncthreads();
    for (int i = tid; i < FT * D; i += 256) {
      const int f = i / D, d = i - f * D;
      if (f0 + f < num_frames) {
        const long long own = own_codes[(f0 + f) * Q + q];
        r_s[f * RS + d] -= codebooks[(static_cast<long long>(q) * K + own) * D + d];
      }
    }
    __syncthreads();
  }
  (void)red;
}

// loss = sum_q mean_{f : target[f,q] != -1} ce[f,q]   (F.cross_entropy(..., ignore_index=-1) per stage, summed)
__global__ void __launch_bounds__(256) rvq_ce_reduce_kernel(const float* __restrict__ ce,
                                                            const long long* __restrict__ target_codes,
                                                            long long num_frames, int Q, float* __restrict__ loss) {
  __shared__ float ssum[8];
  __shared__ float scnt[8];
  float total = 0.f;
  for (int q = 0; q < Q; ++q) {
    float s = 0.f, c = 0.f;
    for (long long f = threadIdx.x; f < num_frames; f += 256) {
      if (target_codes[f * Q + q] >= 0) {
        s += ce[f * Q + q];
        c += 1.f;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, off);
      c += __shfl_xor_sync(0xffffffffu, c, off);
    }
    if ((threadIdx.x & 31) == 0) {
      ssum[threadIdx.x >> 5] = s;
      scnt[threadIdx.x >> 5] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float S = 0.f, Cn = 0.f;
      for (int i = 0; i < 8; ++i) {
        S += ssum[i];
        Cn += scnt[i];
      }
      total += S / Cn;   // 0/0 = NaN when every target of a stage is ignored, as in torch
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = total;
}

// ---- backward (ns2.py:1682 differentiated through x_start) ----
//
// d CE_q / d r_q for one frame with target t:  (u_t - sum_k p_k u_k) / count_q,  u_k = (r_q - c_k) / d_k,
// p = softmax(-d).  The subtracted codewords are detached, so d r_q / d x = I and d loss / d x = sum_q of the above.
// u_k = 0 where d_k == 0 (torch.cdist's backward convention).  Frames whose target is -1 get nothing from that stage.
//
// stage_coef[q] = d_loss / count_q (0 when every target of the stage is -1: torch's nll_loss backward gives zeros there).
__global__ void __launch_bounds__(256) rvq_ce_bwd_coef_kernel(const long long* __restrict__ target_codes,
                                                              long long num_frames, int Q, const float* __restrict__ d_loss,
                                                              float* __restrict__ stage_coef) {
  __shared__ long long scnt[8];
  for (int q = 0; q < Q; ++q) {
    long long c = 0;
    for (long long f = threadIdx.x; f < num_frames; f += 256) c += (target_codes[f * Q + q] >= 0);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
    if ((threadIdx.x & 31) == 0) scnt[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      long long n = 0;
      for (int i = 0; i < 8; ++i) n += scnt[i];
      stage_coef[q] = n > 0 ? d_loss[0] / static_cast<float>(n) : 0.f;
    }
    __syncthreads();
  }
}

// One CTA per 32 frames, the forward's 8 x 32 thread grid.  Per 128-code chunk a thread recomputes the distances of its
// 4 frames x 4 codes with the forward's formula, then the warp (= one frame group) keeps a flash-style online softmax
// per frame: running max m, S = sum e^{l-m}, W = sum e^{l-m}/d and A = sum (e^{l-m}/d) c_k, where A (128 wide) is a
// second small GEMM over the chunk (thread tile: 4 frames x 4 consecutive dims) fed by the weights staged in shared
// memory.  sum_k p_k u_k = (W r - A) / S.  The gradient of all stages accumulates in registers and is written once.
namespace rvqce {
constexpr int WS = FT + 4;   // padded stride of the [KC][FT] weight tile: conflict-free float4 stores
constexpr int SMEM_BWD_BYTES = (FT * RS + KC * RS + KC * WS) * 4;
}  // namespace rvqce

__global__ void __launch_bounds__(256) rvq_ce_bwd_kernel(const float* __restrict__ frames, long long num_frames,
                                                         const float* __restrict__ codebooks,
                                                         const float* __restrict__ cn2, int Q, int K,
                                                         const long long* __restrict__ own_codes,
                                                         const long long* __restrict__ target_codes,
                                                         const float* __restrict__ stage_coef,
                                                         const float* __restrict__ row_scale, long long rows_per_sample,
                                                         float* __restrict__ d_frames, long long out_stride) {
  using namespace rvqce;
  extern __shared__ float sm[];
  float* r_s = sm;                       // [FT][RS] residuals
  float* c_s = sm + FT * RS;             // [KC][RS] codeword chunk
  float* w_s = c_s + KC * RS;            // [KC][WS] e^{l-m}/d of the chunk, code-major
  const int tid = threadIdx.x;
  const int fg = tid >> 5;               // frame group (= warp) -> frames 4*fg .. 4*fg+3
  const int cg = tid & 31;               // distance phase: codes cg + 32*b;  gradient phase: dims 4*cg .. 4*cg+3
  const long long f0 = static_cast<long long>(blockIdx.x) * FT;

  for (int i = tid; i < FT * D; i += 256) {
    const int f = i / D, d = i - f * D;
    r_s[f * RS + d] = (f0 + f < num_frames) ? frames[(f0 + f) * D + d] : 0.f;
  }
  __syncthreads();

  float g[4][4];   // d loss / d frame, frames 4*fg+a, dims 4*cg+j
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int j = 0; j < 4; ++j) g[a][j] = 0.f;

  for (int q = 0; q < Q; ++q) {
    float rn2[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float s = 0.f;
      const float* rr = r_s + (4 * fg + a) * RS;
      for (int d = 0; d < D; ++d) s = fmaf(rr[d], rr[d], s);
      rn2[a] = s;
    }
    float m_run[4], s_run[4], w_run[4], A[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      m_run[a] = -INFINITY;
      s_run[a] = 0.f;
      w_run[a] = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) A[a][j] = 0.f;
    }
    for (int k0 = 0; k0 < K; k0 += KC) {
      __syncthreads();   // previous chunk (codewords and weights) fully consumed
      for (int i = tid; i < KC * D; i += 256) {
        const int c = i / D, d = i - c * D;
        c_s[c * RS + d] = (k0 + c < K) ? codebooks[(static_cast<long long>(q) * K + k0 + c) * D + d] : 0.f;
      }
      __syncthreads();
      float acc[4][4];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
      for (int d = 0; d < D; d += 4) {
        float4 rv[4], cv[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) rv[a] = *reinterpret_cast<const float4*>(r_s + (4 * fg + a) * RS + d);
#pragma unroll
        for (int b = 0; b < 4; ++b) cv[b] = *reinterpret_cast<const float4*>(c_s + (cg + 32 * b) * RS + d);
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            acc[a][b] = fmaf(rv[a].x, cv[b].x, acc[a][b]);
            acc[a][b] = fmaf(rv[a].y, cv[b].y, acc[a][b]);
            acc[a][b] = fmaf(rv[a].z, cv[b].z, acc[a][b]);
            acc[a][b] = fmaf(rv[a].w, cv[b].w, acc[a][b]);
          }
      }
      // logits and distances (the forward's formula), chunk max per frame over the warp
      float dist[4][4], cmax[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) cmax[a] = -INFINITY;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int code = k0 + cg + 32 * b;
        const float c2 = code < K ? __ldg(cn2 + static_cast<long long>(q) * K + code) : 0.f;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          dist[a][b] = code < K ? sqrtf(fmaxf(rn2[a] - 2.f * acc[a][b] + c2, 0.f)) : INFINITY;
          cmax[a] = fmaxf(cmax[a], -dist[a][b]);
        }
      }
#pragma unroll
      for (int a = 0; a < 4; ++a) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) cmax[a] = fmaxf(cmax[a], __shfl_xor_sync(0xffffffffu, cmax[a], off));
        if (cmax[a] > m_run[a]) {   // warp-uniform: rescale the running sums once per chunk
          const float sc = expf(m_run[a] - cmax[a]);
          s_run[a] *= sc;
          w_run[a] *= sc;
#pragma unroll
          for (int j = 0; j < 4; ++j) A[a][j] *= sc;
          m_run[a] = cmax[a];
        }
      }
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        float4 wv;
        float* wp = &wv.x;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const float dd = dist[a][b];
          const float e = expf(-dd - m_run[a]);   // 0 for the padding codes (dd = inf)
          const float w = dd > 0.f ? e / dd : 0.f;
          s_run[a] += e;
          w_run[a] += w;
          wp[a] = w;
        }
        *reinterpret_cast<float4*>(w_s + (cg + 32 * b) * WS + 4 * fg) = wv;
      }
      __syncwarp();   // a warp reads only the weights of its own frames
      for (int c = 0; c < KC; ++c) {
        const float4 wv = *reinterpret_cast<const float4*>(w_s + c * WS + 4 * fg);
        const float4 cv = *reinterpret_cast<const float4*>(c_s + c * RS + 4 * cg);
        const float wa[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          A[a][0] = fmaf(wa[a], cv.x, A[a][0]);
          A[a][1] = fmaf(wa[a], cv.y, A[a][1]);
          A[a][2] = fmaf(wa[a], cv.z, A[a][2]);
          A[a][3] = fmaf(wa[a], cv.w, A[a][3]);
        }
      }
    }
    const float coef = __ldg(stage_coef + q);
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float S = s_run[a], W = w_run[a];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        S += __shfl_xor_sync(0xffffffffu, S, off);
        W += __shfl_xor_sync(0xffffffffu, W, off);
      }
      const long long f = f0 + 4 * fg + a;
      const long long t = f < num_frames ? target_codes[f * Q + q] : -1;   // warp-uniform
      const float4 rv = *reinterpret_cast<const float4*>(r_s + (4 * fg + a) * RS + 4 * cg);
      const float r[4] = {rv.x, rv.y, rv.z, rv.w};
      float diff[4] = {0.f, 0.f, 0.f, 0.f};
      if (t >= 0) {
        const float4 ct = __ldg(reinterpret_cast<const float4*>(codebooks + (static_cast<long long>(q) * K + t) * D) + cg);
        diff[0] = r[0] - ct.x;
        diff[1] = r[1] - ct.y;
        diff[2] = r[2] - ct.z;
        diff[3] = r[3] - ct.w;
      }
      float dt2 = diff[0] * diff[0] + diff[1] * diff[1] + diff[2] * diff[2] + diff[3] * diff[3];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) dt2 += __shfl_xor_sync(0xffffffffu, dt2, off);
      if (t >= 0) {
        const float dt = sqrtf(dt2);
        const float inv_t = dt > 0.f ? 1.f / dt : 0.f;
        const float inv_s = 1.f / S;
#pragma unroll
        for (int j = 0; j < 4; ++j) g[a][j] += coef * (diff[j] * inv_t - (W * r[j] - A[a][j]) * inv_s);
      }
    }
    // residual update with the codec's own code of this stage (same as the forward)
    __syncthreads();
    for (int i = tid; i < FT * D; i += 256) {
      const int f = i / D, d = i - f * D;
      if (f0 + f < num_frames) {
        const long long own = own_codes[(f0 + f) * Q + q];
        r_s[f * RS + d] -= codebooks[(static_cast<long long>(q) * K + own) * D + d];
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const long long f = f0 + 4 * fg + a;
    if (f >= num_frames) continue;
    const float sc = row_scale ? __ldg(row_scale + f / rows_per_sample) : 1.f;
    *reinterpret_cast<float4*>(d_frames + f * out_stride + 4 * cg) =
        make_float4(sc * g[a][0], sc * g[a][1], sc * g[a][2], sc * g[a][3]);
  }
}

}  // namespace ns2

extern "C" int ns2_rvq_ce(const float* frames, int64_t num_frames, int32_t d, const float* codebooks,
                          const float* cb_norm2, int32_t q, int32_t k, const int64_t* own_codes,
                          const int64_t* target_codes, float* ce_scratch, float* loss, ns2_stream_t stream_) {
  using namespace ns2;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NS2_REQUIRE(frames && codebooks && cb_norm2 && own_codes && target_codes && ce_scratch && loss,
              "rvq_ce: NULL pointer");
  NS2_REQUIRE(d == rvqce::D && q > 0 && k >= 32 && num_frames > 0,
              "rvq_ce: d must be 128, k >= 32, q and frames positive");
  NS2_CUDA_CHECK(set_max_smem_once(rvq_ce_kernel, rvqce::SMEM_BYTES));
  const long long grid = (num_frames + rvqce::FT - 1) / rvqce::FT;
  NS2_REQUIRE(grid <= 0x7fffffffLL, "rvq_ce: too many frames");
  rvq_ce_kernel<<<static_cast<unsigned>(grid), 256, rvqce::SMEM_BYTES, stream>>>(
      frames, num_frames, codebooks, cb_norm2, q, k, reinterpret_cast<const long long*>(own_codes),
      reinterpret_cast<const long long*>(target_codes), ce_scratch);
  rvq_ce_reduce_kernel<<<1, 256, 0, stream>>>(ce_scratch, reinterpret_cast<const long long*>(target_codes),
                                             num_frames, q, loss);
  return launched(2);
}

extern "C" int ns2_rvq_ce_bwd(const float* frames, int64_t num_frames, int32_t d, const float* codebooks,
                              const float* cb_norm2, int32_t q, int32_t k, const int64_t* own_codes,
                              const int64_t* target_codes, const float* d_loss, const float* row_scale,
                              int64_t rows_per_sample, float* coef_scratch, float* d_frames, int64_t out_stride,
                              ns2_stream_t stream_) {
  using namespace ns2;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NS2_REQUIRE(frames && codebooks && cb_norm2 && own_codes && target_codes && d_loss && coef_scratch && d_frames,
              "rvq_ce_bwd: NULL pointer");
  NS2_REQUIRE(d == rvqce::D && q > 0 && k >= 32 && num_frames > 0,
              "rvq_ce_bwd: d must be 128, k >= 32, q and frames positive");
  NS2_REQUIRE(out_stride >= d && out_stride % 4 == 0, "rvq_ce_bwd: out_stride must be >= 128 and a multiple of 4");
  NS2_REQUIRE((reinterpret_cast<uintptr_t>(d_frames) & 15) == 0 && (reinterpret_cast<uintptr_t>(codebooks) & 15) == 0,
              "rvq_ce_bwd: d_frames and codebooks must be 16-byte aligned");
  NS2_REQUIRE(row_scale == nullptr || rows_per_sample > 0, "rvq_ce_bwd: rows_per_sample must be positive");
  NS2_CUDA_CHECK(set_max_smem_once(rvq_ce_bwd_kernel, rvqce::SMEM_BWD_BYTES));
  const long long grid = (num_frames + rvqce::FT - 1) / rvqce::FT;
  NS2_REQUIRE(grid <= 0x7fffffffLL, "rvq_ce_bwd: too many frames");
  rvq_ce_bwd_coef_kernel<<<1, 256, 0, stream>>>(reinterpret_cast<const long long*>(target_codes), num_frames, q, d_loss,
                                               coef_scratch);
  rvq_ce_bwd_kernel<<<static_cast<unsigned>(grid), 256, rvqce::SMEM_BWD_BYTES, stream>>>(
      frames, num_frames, codebooks, cb_norm2, q, k, reinterpret_cast<const long long*>(own_codes),
      reinterpret_cast<const long long*>(target_codes), coef_scratch, row_scale, rows_per_sample, d_frames, out_stride);
  return launched(2);
}
