// Folds a conv and the Linear after it into one conv pack: the transformer feed-forward's CausalConv1d and output
// projection (ns2.py:1019-1024), which have nothing between them.  Runs once per parameter version for every layer
// (Model._pack), i.e. after every optimizer step in training, so it is a batched fp32 SIMT GEMM of the project's
// own: 128 x 128 tiles of (output channel o) x (conv column n = i * T + t), 8 x 8 per thread, 16-deep k stages in two
// cp.async shared-memory buffers, two CTAs per SM, fp32 FMA accumulation (no TF32), one rounding to bf16 on the way
// into the tap-major pack.  The conv bias rides along as column n = I * T,
// so the folded bias W2 bc + b2 comes out of the same tiles.  See include/ns2_b200.h section 1c.
#include "host_common.h"
#include "../../include/ns2_b200.h"

#include <cuda_bf16.h>

namespace ns2 {

namespace {

constexpr int FOLD_BM = 128;   // output channels per tile
constexpr int FOLD_BN = 128;   // conv columns per tile
constexpr int FOLD_BK = 16;    // contraction (conv output channels) per shared-memory stage
constexpr int FOLD_PAD = 4;    // A rows stay 16-byte aligned, and the transposing stores hit 2-way bank conflicts at most

// 4-byte global -> shared copy; `valid` false writes a zero (src-size 0) and reads nothing
__device__ __forceinline__ void cp_async_4(float* dst, const float* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))),
               "l"(src), "r"(valid ? 4 : 0)
               : "memory");
}

__global__ void __launch_bounds__(256, 2) fold_conv_linear_kernel(const float* __restrict__ w2,
                                                               const float* __restrict__ wc,
                                                               const float* __restrict__ bc,
                                                               const float* __restrict__ b2, __nv_bfloat16* __restrict__ out,
                                                               float* __restrict__ bias_out, int O, int K, int I, int T,
                                                               int i_pad) {
  __shared__ __align__(16) float As[2][FOLD_BK][FOLD_BM + FOLD_PAD];   // W2 tile, [stage][k][o]
  __shared__ __align__(16) float Bs[2][FOLD_BK][FOLD_BN];              // [Wc | bc] tile, [stage][k][n]
  const int l = blockIdx.z;
  const long long NW = static_cast<long long>(I) * T;   // conv weight columns; column NW is the conv bias
  w2 += static_cast<size_t>(l) * O * K;
  wc += static_cast<size_t>(l) * K * NW;
  bc += static_cast<size_t>(l) * K;
  b2 += static_cast<size_t>(l) * O;
  out += static_cast<size_t>(l) * O * T * i_pad;
  bias_out += static_cast<size_t>(l) * O;
  const int m0 = blockIdx.y * FOLD_BM;
  const long long n0 = static_cast<long long>(blockIdx.x) * FOLD_BN;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  // two shared-memory stages: the next stage's cp.async copies (zero-filled past the edges) land under this stage's FMAs
  const int ma = threadIdx.x / FOLD_BK, ka = threadIdx.x % FOLD_BK;   // A: rows ma + 16 r, column ka (16 k of a W2 row)
  const int kb = threadIdx.x / FOLD_BN, nb = threadIdx.x % FOLD_BN;   // B: rows kb + 2 r, column nb
  const long long gn = n0 + nb;
  auto issue = [&](int stage, int k0) {
#pragma unroll 1
    for (int r = 0; r < FOLD_BK * FOLD_BM / 256; ++r) {
      const int gm = m0 + ma + 16 * r, gka = k0 + ka;
      const bool oka = gm < O && gka < K;
      cp_async_4(&As[stage][ka][ma + 16 * r], oka ? w2 + static_cast<size_t>(gm) * K + gka : w2, oka);
      const int gkb = k0 + kb + 2 * r;
      const bool okb = gkb < K && gn <= NW;
      cp_async_4(&Bs[stage][kb + 2 * r][nb], !okb ? wc : gn < NW ? wc + static_cast<size_t>(gkb) * NW + gn : bc + gkb, okb);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  issue(0, 0);
  for (int k0 = 0, s = 0; k0 < K; k0 += FOLD_BK, s ^= 1) {
    if (k0 + FOLD_BK < K) {
      issue(s ^ 1, k0 + FOLD_BK);   // its stage was last read before the previous iteration's closing barrier
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < FOLD_BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[s][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[s][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[s][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[s][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
    if (gm >= O) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const long long gn = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4);
      if (gn < NW) {
        const int ci = static_cast<int>(gn / T), t = static_cast<int>(gn % T);
        out[static_cast<size_t>(gm) * T * i_pad + static_cast<size_t>(t) * i_pad + ci] = __float2bfloat16_rn(acc[i][j]);
      } else if (gn == NW) {
        bias_out[gm] = acc[i][j] + b2[gm];
      }
    }
  }
}

}  // namespace
}  // namespace ns2

extern "C" int ns2_fold_conv_linear(const float* w2, const float* wc, const float* bc, const float* b2, int32_t layers,
                                    int32_t o, int32_t k, int32_t i, int32_t taps, int32_t i_pad, void* out_bf16,
                                    float* bias_out, ns2_stream_t stream_) {
  using namespace ns2;
  NS2_REQUIRE(w2 && wc && bc && b2 && out_bf16 && bias_out, "fold_conv_linear: NULL pointer");
  NS2_REQUIRE(layers > 0 && layers <= 65535 && o > 0 && k > 0 && i > 0 && taps > 0 && i_pad >= i,
              "fold_conv_linear: bad sizes (layers=%d o=%d k=%d i=%d taps=%d i_pad=%d)", layers, o, k, i, taps, i_pad);
  const long long cols = static_cast<long long>(i) * taps + 1;
  NS2_REQUIRE((cols + FOLD_BN - 1) / FOLD_BN <= 0x7fffffff && (o + FOLD_BM - 1) / FOLD_BM <= 65535,
              "fold_conv_linear: too large");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // the pack's padding columns [t * i_pad + i, (t + 1) * i_pad) must be exact zeros: the kernel writes only the others
  if (i_pad > i)
    NS2_CUDA_CHECK(cudaMemsetAsync(out_bf16, 0, static_cast<size_t>(layers) * o * taps * i_pad * 2, stream));
  dim3 grid(static_cast<unsigned>((cols + FOLD_BN - 1) / FOLD_BN), static_cast<unsigned>((o + FOLD_BM - 1) / FOLD_BM),
            static_cast<unsigned>(layers));
  fold_conv_linear_kernel<<<grid, 256, 0, stream>>>(w2, wc, bc, b2, reinterpret_cast<__nv_bfloat16*>(out_bf16), bias_out,
                                                    o, k, i, taps, i_pad);
  return launched(1);
}
