// Kernels of Encodec's SEANet decoder and encoder (24 kHz model) that the segmented GEMM does not cover
// (include/ns2_b200.h, section 10):
//   lstm_seq_kernel   one layer of the decoder's 2-layer LSTM(512), the whole sequence in one launch: a 16-CTA cluster
//                     per group of <= 64 batch rows, CTA c owning hidden units [32c, 32c + 32) of all four gates with
//                     its 128 rows of W_hh resident in shared memory; h_t is exchanged through distributed shared memory
//   elu_pad_kernel    ELU + causal reflect left padding + bf16 cast: the A operand of every conv GEMM
//   seanet_tail_kernel the 32-channel stage at the full sample rate (last ResnetBlock, ELU, 32 -> 1 k7 conv), fp32
//   seanet_head_kernel the encoder's 32-channel stage at the full sample rate (1 -> 32 k7 conv, ResnetBlock, ELU),
//                      fp32, writing the bf16 A operand of the encoder's first strided conv
// Convolutions with >= 64 channels, the transposed and strided convolutions and the LSTM input projections run on
// ns2_gemm.
#include "ptx.cuh"
#include "host_common.h"
#include "../../include/ns2_b200.h"

namespace ns2 {

// ------------------------------------------------------------------------------------------------
// cluster / distributed shared memory plumbing
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_v4(uint32_t addr, uint4 v) {
  asm volatile("st.shared::cluster.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
// generic-proxy shared-memory writes (local or remote) -> visible to wgmma operand reads
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// wgmma m64n32k16 (SS), same conventions as the generated wrappers in wgmma.cuh
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_ss_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, "
      "%13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int NB>
__device__ __forceinline__ void wgmma_lstm(float (&d)[NB / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (NB == 64) wgmma_bf16_ss_n64<0, 0>(d, da, db, scale_d);
  else wgmma_bf16_ss_n32<0, 0>(d, da, db, scale_d);
}

__device__ __forceinline__ float elu_f(float v) { return v > 0.f ? v : expm1f(v); }
__device__ __forceinline__ float sigmoid_acc(float v) { return 1.0f / (1.0f + __expf(-v)); }

// Source row of position t under a causal reflect left pad: rows [-pad, 0) mirror about row 0.  False where the row
// reads as zero: beyond the pad, or at or past `length` (a reflected row of an input shorter than the pad is the
// reflection of its zero extension).
__device__ __forceinline__ bool reflect_src(int& t, int length, int pad) {
  if (t < -pad) return false;
  if (t < 0) t = -t;
  return t < length;
}

// acc[o] += w[o] * v over a row of N weights: one float4 broadcast feeds four outputs
template <int N>
__device__ __forceinline__ void fma_row(float (&acc)[N], const float* w, float v) {
  const float4* wr = reinterpret_cast<const float4*>(w);
#pragma unroll
  for (int o4 = 0; o4 < N / 4; ++o4) {
    const float4 wv = wr[o4];
    acc[4 * o4] = fmaf(wv.x, v, acc[4 * o4]);
    acc[4 * o4 + 1] = fmaf(wv.y, v, acc[4 * o4 + 1]);
    acc[4 * o4 + 2] = fmaf(wv.z, v, acc[4 * o4 + 2]);
    acc[4 * o4 + 3] = fmaf(wv.w, v, acc[4 * o4 + 3]);
  }
}

// ------------------------------------------------------------------------------------------------
// 1. LSTM layer (nn.LSTM gate order i, f, g, o; zero initial state)
//
// CTA c of a cluster holds 128 rows of W_hh, packed on the host so that CTA-local row R = 64 hf + 16 w + 8 i + q is
// gate 2 hf + i of hidden unit 32 c + 8 w + q.  One warpgroup issues two m64nNBk16 wgmma chains (hf = 0: gates i, f;
// hf = 1: gates g, o) against h_{t-1} (NB batch rows x 512, bf16): thread (warp w, lane l) then holds all four gate
// pre-activations of unit 8 w + l/4 for its NB/4 batch columns, so the cell state stays in registers.
// Shared memory: W slice 128 KB + h 8 x NB x 128 B (K-major, 128-byte swizzle) + a NB x 64 B staging slice.  h is
// single-buffered (a second 64-row buffer would not fit beside W): each step splits one cluster barrier around the
// gate math (arrive once the MMAs have read h_{t-1}, wait before h_t overwrites it in the other CTAs) and closes with
// a full cluster barrier after the distributed-shared-memory writes.
// ------------------------------------------------------------------------------------------------
constexpr int kLstmHidden = 512;
constexpr int kLstmCluster = 16;
constexpr int kLstmWBytes = 128 * kLstmHidden * 2;

struct LstmDev {
  const float* xproj;
  long long xp_rs, xp_bs;
  const __nv_bfloat16* w;
  const float* skip;
  long long sk_rs, sk_bs;
  float* out;
  long long out_rs, out_bs;
  __nv_bfloat16* out_bf;
  long long ob_rs, ob_bs;
  int batch, steps;
};

constexpr int lstm_smem_bytes(int nb) { return 1024 + kLstmWBytes + 8 * nb * 128 + nb * 64; }

template <int NB>
__global__ void __launch_bounds__(128, 1) lstm_seq_kernel(const LstmDev p) {
  extern __shared__ uint8_t lstm_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(lstm_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* hbuf = smem + kLstmWBytes;
  uint8_t* stage = hbuf + 8 * NB * 128;
  const uint32_t sw = smem_u32(smem), sh = smem_u32(hbuf);
  constexpr int NC = NB / 4;  // batch columns per thread

  const int c = static_cast<int>(cluster_ctarank());
  const int b0 = (blockIdx.x / kLstmCluster) * NB;
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31, q = lane >> 2;
  const int unit = 8 * w + q;  // CTA-local hidden unit

  // W slice -> shared memory (row r, 16-byte piece kc*8 + s at chunk kc, swizzled position s ^ (r % 8))
  const uint4* wsrc = reinterpret_cast<const uint4*>(p.w + static_cast<size_t>(c) * 128 * kLstmHidden);
  for (int i = tid; i < 128 * 64; i += 128) {
    const int r = i >> 6, kc = (i >> 3) & 7, s = i & 7;
    *reinterpret_cast<uint4*>(smem + kc * 16384 + r * 128 + ((s ^ (r & 7)) << 4)) = __ldg(wsrc + i);
  }
  for (int i = tid; i < 8 * NB * 8; i += 128) reinterpret_cast<uint4*>(hbuf)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_all();
  __syncthreads();
  cluster_arrive();
  cluster_wait();

  float cst[NC];
#pragma unroll
  for (int i = 0; i < NC; ++i) cst[i] = 0.f;
  float acc0[NB / 2], acc1[NB / 2];

  for (int t = 0; t < p.steps; ++t) {
    // this step's input projection (issued before the MMAs so the loads overlap them)
    float xp[4][NC];
#pragma unroll
    for (int j = 0; j < NB / 8; ++j) {
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int b = b0 + 8 * j + 2 * (lane & 3) + k;
        const int idx = 2 * j + k;
        if (b < p.batch) {
          const float* src = p.xproj + b * p.xp_bs + t * p.xp_rs + 128 * c + 16 * w + q;
          xp[0][idx] = __ldg(src);
          xp[1][idx] = __ldg(src + 8);
          xp[2][idx] = __ldg(src + 64);
          xp[3][idx] = __ldg(src + 72);
        } else {
          xp[0][idx] = xp[1][idx] = xp[2][idx] = xp[3][idx] = 0.f;
        }
      }
    }
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
      const uint64_t da0 = gmma_desc_sw128(sw + kc * 16384, 16, 1024);
      const uint64_t da1 = gmma_desc_sw128(sw + kc * 16384 + 8192, 16, 1024);
      const uint64_t db = gmma_desc_sw128(sh + kc * NB * 128, 16, 1024);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t scale = (kc | kk) ? 1u : 0u;
        wgmma_lstm<NB>(acc0, da0 + 2 * kk, db + 2 * kk, scale);
        wgmma_lstm<NB>(acc1, da1 + 2 * kk, db + 2 * kk, scale);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(acc0);
    wgmma_hold(acc1);
    cluster_arrive();  // this CTA no longer reads h_{t-1}

#pragma unroll
    for (int j = 0; j < NB / 8; ++j) {
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int bl = 8 * j + 2 * (lane & 3) + k;
        const int idx = 2 * j + k;
        const float ig = sigmoid_acc(acc0[4 * j + k] + xp[0][idx]);
        const float fg = sigmoid_acc(acc0[4 * j + 2 + k] + xp[1][idx]);
        const float gg = tanhf(acc1[4 * j + k] + xp[2][idx]);
        const float og = sigmoid_acc(acc1[4 * j + 2 + k] + xp[3][idx]);
        cst[idx] = fg * cst[idx] + ig * gg;
        const float hv = og * tanhf(cst[idx]);
        const __nv_bfloat16 hb = __float2bfloat16_rn(hv);
        reinterpret_cast<__nv_bfloat16*>(stage)[bl * 32 + unit] = hb;
        const int b = b0 + bl;
        if (b < p.batch) {
          const int col = 32 * c + unit;
          float v = hv;
          if (p.skip != nullptr) v += p.skip[b * p.sk_bs + t * p.sk_rs + col];
          if (p.out != nullptr) p.out[b * p.out_bs + t * p.out_rs + col] = v;
          if (p.out_bf != nullptr) p.out_bf[b * p.ob_bs + t * p.ob_rs + col] = __float2bfloat16_rn(v);
        }
      }
    }
    __syncthreads();  // staging slice complete
    cluster_wait();   // every CTA of the cluster has read h_{t-1}
    // h_t slice (NB rows x 32 units) -> columns [32c, 32c + 32) of every CTA's h buffer
    for (int i = tid; i < kLstmCluster * NB * 4; i += 128) {
      const int r = i / (NB * 4), rem = i - r * (NB * 4), b = rem >> 2, pc = rem & 3;
      const uint4 v = *reinterpret_cast<const uint4*>(stage + b * 64 + pc * 16);
      const int piece = 4 * (c & 1) + pc;
      const uint32_t local = sh + (c >> 1) * NB * 128 + b * 128 + ((piece ^ (b & 7)) << 4);
      st_cluster_v4(mapa_shared(local, static_cast<uint32_t>(r)), v);
    }
    fence_proxy_async_all();
    cluster_arrive();
    cluster_wait();
    fence_proxy_async_all();
  }
}

template <int NB>
static int launch_lstm(const LstmDev& p, int groups, cudaStream_t stream) {
  auto kern = lstm_seq_kernel<NB>;
  constexpr int smem = lstm_smem_bytes(NB);
  NS2_CUDA_CHECK(set_max_smem_once(kern, smem));
  NS2_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kLstmCluster * groups, 1, 1);
  cfg.blockDim = dim3(128, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kLstmCluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int clusters = 0;
  NS2_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&clusters, kern, &cfg));
  if (clusters == 0)
    return set_error(kErrUnsupported,
                     "ns2_lstm_seq: no %d-CTA cluster with %d bytes of shared memory per CTA fits on this device",
                     kLstmCluster, smem);
  NS2_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, p));
  return launched(1);
}

// ------------------------------------------------------------------------------------------------
// 2. ELU + causal reflect pad + bf16 cast.  Thread = (batch, output row, 4 channels).
// ------------------------------------------------------------------------------------------------
__global__ void elu_pad_kernel(const float* __restrict__ x, long long x_rs, long long x_bs, int batch, int length,
                               int channels, int pad, int flags, __nv_bfloat16* __restrict__ out, long long o_rs,
                               long long o_bs) {
  const int c4 = channels >> 2;
  const int rows = pad + length;
  const long long total = static_cast<long long>(batch) * rows * c4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cc = static_cast<int>(i % c4);
    const long long rest = i / c4;
    const int r = static_cast<int>(rest % rows);
    const int b = static_cast<int>(rest / rows);
    int t = r - pad;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (reflect_src(t, length, pad)) v = *reinterpret_cast<const float4*>(x + b * x_bs + t * x_rs + 4 * cc);
    __nv_bfloat16* o = out + b * o_bs + r * o_rs + 4 * cc;
    float4 e = v;
    if (flags & NS2_ELU_PAD_ELU) e = make_float4(elu_f(v.x), elu_f(v.y), elu_f(v.z), elu_f(v.w));
    *reinterpret_cast<uint2*>(o) = make_uint2(pack_bf16x2(e.x, e.y), pack_bf16x2(e.z, e.w));
    if (flags & NS2_ELU_PAD_RAW)
      *reinterpret_cast<uint2*>(o + channels) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
}

// ------------------------------------------------------------------------------------------------
// 3. ResnetBlock(32, hidden 16) of the tail and head kernels, one position per thread, fp32:
//      out = shortcut(x) + conv1(ELU(conv3(ELU(x))))
// Parameters (kBlkFloats floats from the block's base, packed input-major for fma_row):
//   w3 [3][32][16] (tap, in, out)  b3 [16]   wsc [32][32] (in, out)  wc1 [16][32] (in, out)  b2 [32] = b_sc + b_c1
// Each accumulator takes its bias first, then taps and input channels ascending, the shortcut before the conv1x1.
// ------------------------------------------------------------------------------------------------
constexpr int kBlkW3 = 0, kBlkB3 = 1536, kBlkWsc = 1552, kBlkWc1 = 2576, kBlkB2 = 3088, kBlkFloats = 3120;

// h = b3 + conv3 over the three rows of ELU(x) (row stride 33) that start at xe
__device__ __forceinline__ void resblock32_hidden(float (&h)[16], const float* blk, const float* xe) {
#pragma unroll
  for (int o = 0; o < 16; ++o) h[o] = blk[kBlkB3 + o];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const float* xr = xe + j * 33;
#pragma unroll 8
    for (int ci = 0; ci < 32; ++ci) fma_row(h, blk + kBlkW3 + (j * 32 + ci) * 16, xr[ci]);
  }
}

// acc = b2 + shortcut(row x) + conv1(row eh = ELU(h)).  eh lives in shared memory in the tail (kUnrollH = 4) and in
// registers in the head, where only the fully unrolled loop (kUnrollH = 16) keeps it there.
template <int kUnrollH>
__device__ __forceinline__ void resblock32_out(float (&acc)[32], const float* blk, const float* x, const float* eh) {
#pragma unroll
  for (int o = 0; o < 32; ++o) acc[o] = blk[kBlkB2 + o];
#pragma unroll 4
  for (int ci = 0; ci < 32; ++ci) fma_row(acc, blk + kBlkWsc + ci * 32, x[ci]);
#pragma unroll kUnrollH
  for (int hc = 0; hc < 16; ++hc) fma_row(acc, blk + kBlkWc1 + hc * 32, eh[hc]);
}

// ------------------------------------------------------------------------------------------------
// 4. 32-channel tail: z = ResnetBlock(x), y = conv7(ELU(z)), all causal with reflect padding.
// One CTA = one batch element x kTailOut output samples; 128 threads, one window row each.  Window rows of z (and h)
// cover t0 - 6 .. t0 + kTailOut - 1, x rows t0 - 8 .. t0 + kTailOut - 1.  Parameters (NS2_SEANET_TAIL_PARAMS floats):
//   the ResnetBlock's (section 3)  wf [7][32] (tap, in)  bf [4] (bf[0] = the final bias)
// ------------------------------------------------------------------------------------------------
constexpr int kTailThreads = 128;
constexpr int kTailOut = kTailThreads - 6;
constexpr int kTailXRows = kTailOut + 8;
constexpr int kTailBlk = 0, kTailWf = kTailBlk + kBlkFloats, kTailBf = kTailWf + 7 * 32;
static_assert(kTailBf + 4 == NS2_SEANET_TAIL_PARAMS, "tail parameter layout");
constexpr int kTailSmemFloats = NS2_SEANET_TAIL_PARAMS + 2 * kTailXRows * 33 + kTailThreads * 17 + kTailThreads * 33;

__global__ void __launch_bounds__(kTailThreads) seanet_tail_kernel(const float* __restrict__ x, long long x_rs,
                                                                  long long x_bs, int length,
                                                                  const float* __restrict__ prm, float* __restrict__ y,
                                                                  long long y_bs) {
  extern __shared__ float4 tail_smem4[];
  float* sp = reinterpret_cast<float*>(tail_smem4);
  float* sx = sp + NS2_SEANET_TAIL_PARAMS;   // raw x       [kTailXRows][33]
  float* sxe = sx + kTailXRows * 33;          // ELU(x)      [kTailXRows][33]
  float* sh = sxe + kTailXRows * 33;          // ELU(h)      [128][17]
  float* sz = sh + kTailThreads * 17;         // ELU(z)      [128][33]
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * kTailOut;
  const float* xb = x + b * x_bs;

  for (int i = tid; i < NS2_SEANET_TAIL_PARAMS / 4; i += kTailThreads)
    tail_smem4[i] = __ldg(reinterpret_cast<const float4*>(prm) + i);
  for (int i = tid; i < kTailXRows * 8; i += kTailThreads) {
    const int r = i >> 3, c4 = (i & 7) * 4;
    int t = t0 - 8 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (reflect_src(t, length, 2))  // the k3 conv's reflect pad
      v = __ldg(reinterpret_cast<const float4*>(xb + t * x_rs + c4));
    float* d = sx + r * 33 + c4;
    float* e = sxe + r * 33 + c4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    e[0] = elu_f(v.x); e[1] = elu_f(v.y); e[2] = elu_f(v.z); e[3] = elu_f(v.w);
  }
  __syncthreads();

  const int hr = tid;                 // window row: t = t0 - 6 + hr
  const int t = t0 - 6 + hr;
  const bool live = t >= 0 && t < length;
  const float* blk = sp + kTailBlk;
  {  // h = conv3(ELU(x)) (32 -> 16), stored as ELU(h)
    float acc[16];
    resblock32_hidden(acc, blk, sxe + hr * 33);
#pragma unroll
    for (int o = 0; o < 16; ++o) sh[hr * 17 + o] = elu_f(acc[o]);
  }
  __syncthreads();
  {  // z = shortcut(x) + conv1(ELU(h)) (32 -> 32, 16 -> 32), stored as ELU(z); zero outside [0, length)
    float acc[32];
    resblock32_out<4>(acc, blk, sx + (hr + 2) * 33, sh + hr * 17);
#pragma unroll
    for (int o = 0; o < 32; ++o) sz[hr * 33 + o] = live ? elu_f(acc[o]) : 0.f;
  }
  __syncthreads();
  if (t0 == 0) {  // the k7 conv's reflect pad (6) of ELU(z): rows t = -6..-1 take z_ext[-t]
    for (int i = tid; i < 6 * 32; i += kTailThreads) {
      const int r = i >> 5, o = i & 31;  // window row r holds t = r - 6
      const int src = 6 - r;             // -t
      sz[r * 33 + o] = src < length ? sz[(src + 6) * 33 + o] : 0.f;
    }
    __syncthreads();
  }
  if (tid < kTailOut && t0 + tid < length) {  // y = conv7(ELU(z)) (32 -> 1)
    float acc = sp[kTailBf];
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      const float* zr = sz + (tid + j) * 33;
#pragma unroll 8
      for (int ci = 0; ci < 32; ++ci) acc = fmaf(sp[kTailWf + j * 32 + ci], zr[ci], acc);
    }
    y[b * y_bs + t0 + tid] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
// 5. Encoder head, the 32-channel stage at the full sample rate, fp32:
//      z0 = conv7(x) (1 -> 32),  z1 = shortcut(z0) + conv1(ELU(conv3(ELU(z0)))),  out = bf16(ELU(z1)) reflect-padded
//      by 2 (the A operand of the first strided conv's GEMM), every conv causal with reflect left padding.
// One CTA = one batch element x kHeadOut positions t0 .. t0 + kHeadOut - 1 of z1; 128 threads.  Phase 1: thread r
// computes z0 at window row r (position t0 - 2 + r); the conv3's reflected rows -1, -2 (first tile only) are computed
// directly at their source positions 1, 2.  Phase 2: thread i < kHeadOut computes h and z1 at t0 + i from z0 rows
// i .. i + 2 and writes output row t0 + i + 2; threads 1 and 2 of the first tile also write the reflected rows 1, 0.
// x window: positions t0 - 8 .. t0 + kHeadOut - 1.  Parameters (NS2_SEANET_HEAD_PARAMS floats, input-major):
//   w0 [7][32] (tap, out)  b0 [32]  the ResnetBlock's (section 3)
// ------------------------------------------------------------------------------------------------
constexpr int kHeadThreads = 128;
constexpr int kHeadOut = kHeadThreads - 2;
constexpr int kHeadXRows = kHeadOut + 8;
constexpr int kHeadW0 = 0, kHeadB0 = kHeadW0 + 7 * 32, kHeadBlk = kHeadB0 + 32;
static_assert(kHeadBlk + kBlkFloats == NS2_SEANET_HEAD_PARAMS, "head parameter layout");
constexpr int kHeadSmemFloats = NS2_SEANET_HEAD_PARAMS + ((kHeadXRows + 3) & ~3) + 2 * kHeadThreads * 33;

__global__ void __launch_bounds__(kHeadThreads) seanet_head_kernel(const float* __restrict__ x, long long x_bs,
                                                                  int length, const float* __restrict__ prm,
                                                                  __nv_bfloat16* __restrict__ out, long long o_rs,
                                                                  long long o_bs) {
  extern __shared__ float4 head_smem4[];
  float* sp = reinterpret_cast<float*>(head_smem4);
  float* sx = sp + NS2_SEANET_HEAD_PARAMS;           // x            [kHeadXRows]
  float* sz = sx + ((kHeadXRows + 3) & ~3);          // z0           [128][33]
  float* sze = sz + kHeadThreads * 33;               // ELU(z0)      [128][33]
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * kHeadOut;
  const float* xb = x + b * x_bs;

  for (int i = tid; i < NS2_SEANET_HEAD_PARAMS / 4; i += kHeadThreads)
    head_smem4[i] = __ldg(reinterpret_cast<const float4*>(prm) + i);
  for (int i = tid; i < kHeadXRows; i += kHeadThreads) {
    int t = t0 - 8 + i;
    sx[i] = reflect_src(t, length, 6) ? __ldg(xb + t) : 0.f;  // the k7 conv's reflect pad
  }
  __syncthreads();

  {  // z0 = conv7(x) at window row tid
    int src = t0 - 2 + tid;
    if (src < 0) src = -src;  // the conv3's reflect pad (2) of z0
    float acc[32];
    if (src < length) {
#pragma unroll
      for (int o = 0; o < 32; ++o) acc[o] = sp[kHeadB0 + o];
      const float* xr = sx + src - t0 + 2;
#pragma unroll
      for (int j = 0; j < 7; ++j) fma_row(acc, sp + kHeadW0 + j * 32, xr[j]);
    } else {  // past the end, or a reflected row of an input shorter than the pad (zero-extended)
#pragma unroll
      for (int o = 0; o < 32; ++o) acc[o] = 0.f;
    }
#pragma unroll
    for (int o = 0; o < 32; ++o) {
      sz[tid * 33 + o] = acc[o];
      sze[tid * 33 + o] = elu_f(acc[o]);
    }
  }
  __syncthreads();

  if (tid >= kHeadOut) return;
  const int t = t0 + tid;
  __nv_bfloat16* ob = out + b * o_bs;
  if (t >= length) {  // the reflected output rows of an input shorter than 3 samples are zero-extended
    if (t0 == 0 && (tid == 1 || tid == 2)) {
      uint4* o = reinterpret_cast<uint4*>(ob + (2 - tid) * o_rs);
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = make_uint4(0, 0, 0, 0);
    }
    return;
  }
  const float* blk = sp + kHeadBlk;
  float hv[16];  // h = conv3(ELU(z0)) (32 -> 16), then ELU
  resblock32_hidden(hv, blk, sze + tid * 33);
#pragma unroll
  for (int o = 0; o < 16; ++o) hv[o] = elu_f(hv[o]);
  float acc[32];  // z1 = shortcut(z0) + conv1(ELU(h)) (32 -> 32, 16 -> 32)
  resblock32_out<16>(acc, blk, sz + (tid + 2) * 33, hv);
  uint4 pk[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    pk[i] = make_uint4(pack_bf16x2(elu_f(acc[8 * i]), elu_f(acc[8 * i + 1])),
                       pack_bf16x2(elu_f(acc[8 * i + 2]), elu_f(acc[8 * i + 3])),
                       pack_bf16x2(elu_f(acc[8 * i + 4]), elu_f(acc[8 * i + 5])),
                       pack_bf16x2(elu_f(acc[8 * i + 6]), elu_f(acc[8 * i + 7])));
  uint4* o = reinterpret_cast<uint4*>(ob + (t + 2) * o_rs);
#pragma unroll
  for (int i = 0; i < 4; ++i) o[i] = pk[i];
  if (t == 1 || t == 2) {  // the next conv's reflect pad (2): output rows 1, 0 repeat z1 rows 1, 2
    uint4* r = reinterpret_cast<uint4*>(ob + (2 - t) * o_rs);
#pragma unroll
    for (int i = 0; i < 4; ++i) r[i] = pk[i];
  }
}

}  // namespace ns2

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" int ns2_lstm_seq(const float* xproj, int64_t xp_row_stride, int64_t xp_batch_stride, const void* w_hh,
                            int32_t batch, int32_t steps, int32_t hidden, const float* skip, int64_t skip_row_stride,
                            int64_t skip_batch_stride, float* out, int64_t out_row_stride, int64_t out_batch_stride,
                            void* out_bf16, int64_t outbf_row_stride, int64_t outbf_batch_stride,
                            ns2_stream_t stream) {
  using namespace ns2;
  NS2_REQUIRE(hidden == kLstmHidden, "ns2_lstm_seq: hidden=%d (only 512 is supported: 16 CTAs x 32 units)", hidden);
  NS2_REQUIRE(batch >= 0 && steps >= 0, "ns2_lstm_seq: negative batch or steps");
  if (batch == 0 || steps == 0) return kOk;
  NS2_REQUIRE(xproj != nullptr && w_hh != nullptr, "ns2_lstm_seq: xproj and w_hh must be non-NULL");
  NS2_REQUIRE(out != nullptr || out_bf16 != nullptr, "ns2_lstm_seq: needs out and/or out_bf16");
  NS2_REQUIRE((reinterpret_cast<uintptr_t>(w_hh) & 15) == 0, "ns2_lstm_seq: w_hh must be 16-byte aligned");
  NS2_REQUIRE(xp_row_stride >= 4 * hidden && xp_batch_stride >= 0,
              "ns2_lstm_seq: xproj rows hold the 4*hidden gate pre-activations (row stride %lld)",
              (long long)xp_row_stride);
  LstmDev p;
  p.xproj = xproj;
  p.xp_rs = xp_row_stride;
  p.xp_bs = xp_batch_stride;
  p.w = static_cast<const __nv_bfloat16*>(w_hh);
  p.skip = skip;
  p.sk_rs = skip_row_stride;
  p.sk_bs = skip_batch_stride;
  p.out = out;
  p.out_rs = out_row_stride;
  p.out_bs = out_batch_stride;
  p.out_bf = static_cast<__nv_bfloat16*>(out_bf16);
  p.ob_rs = outbf_row_stride;
  p.ob_bs = outbf_batch_stride;
  p.batch = batch;
  p.steps = steps;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (batch <= 32) return launch_lstm<32>(p, 1, s);
  return launch_lstm<64>(p, (batch + 63) / 64, s);
}

extern "C" int ns2_elu_pad(const float* x, int64_t x_row_stride, int64_t x_batch_stride, int32_t batch, int32_t length,
                           int32_t channels, int32_t pad, int32_t flags, void* out_bf16, int64_t out_row_stride,
                           int64_t out_batch_stride, ns2_stream_t stream) {
  using namespace ns2;
  NS2_REQUIRE(batch >= 0 && length >= 0 && pad >= 0, "ns2_elu_pad: negative size");
  NS2_REQUIRE((flags & ~(NS2_ELU_PAD_ELU | NS2_ELU_PAD_RAW)) == 0, "ns2_elu_pad: unknown flags 0x%x", flags);
  NS2_REQUIRE(channels > 0 && channels % 4 == 0, "ns2_elu_pad: channels=%d must be a positive multiple of 4", channels);
  if (batch == 0 || length == 0) return kOk;
  NS2_REQUIRE(x != nullptr && out_bf16 != nullptr, "ns2_elu_pad: x and out must be non-NULL");
  NS2_REQUIRE(x_row_stride % 4 == 0 && x_batch_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0,
              "ns2_elu_pad: x must be 16-byte aligned with strides multiple of 4");
  NS2_REQUIRE(out_row_stride % 4 == 0 && out_batch_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(out_bf16) & 7) == 0,
              "ns2_elu_pad: out must be 8-byte aligned with strides multiple of 4");
  const long long total = static_cast<long long>(batch) * (pad + length) * (channels / 4);
  long long blocks = (total + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  elu_pad_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, x_row_stride, x_batch_stride, batch, length, channels, pad, flags, static_cast<__nv_bfloat16*>(out_bf16),
      out_row_stride, out_batch_stride);
  return launched(1);
}

extern "C" int ns2_seanet_tail(const float* x, int64_t x_row_stride, int64_t x_batch_stride, int32_t batch,
                               int32_t length, const float* params, float* out, int64_t out_batch_stride,
                               ns2_stream_t stream) {
  using namespace ns2;
  NS2_REQUIRE(batch >= 0 && length >= 0, "ns2_seanet_tail: negative size");
  if (batch == 0 || length == 0) return kOk;
  NS2_REQUIRE(batch <= 65535, "ns2_seanet_tail: batch=%d above 65535", batch);
  NS2_REQUIRE(x != nullptr && params != nullptr && out != nullptr, "ns2_seanet_tail: NULL pointer");
  NS2_REQUIRE(x_row_stride >= 32 && x_row_stride % 4 == 0 && x_batch_stride % 4 == 0 &&
                  (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(params) & 15) == 0,
              "ns2_seanet_tail: x (32 channels) and params must be 16-byte aligned with strides multiple of 4");
  const int smem = kTailSmemFloats * 4;
  NS2_CUDA_CHECK(set_max_smem_once(seanet_tail_kernel, smem));
  const dim3 grid((length + kTailOut - 1) / kTailOut, batch);
  seanet_tail_kernel<<<grid, kTailThreads, smem, static_cast<cudaStream_t>(stream)>>>(x, x_row_stride, x_batch_stride,
                                                                                      length, params, out,
                                                                                      out_batch_stride);
  return launched(1);
}

extern "C" int ns2_seanet_head(const float* x, int64_t x_batch_stride, int32_t batch, int32_t length,
                               const float* params, void* out_bf16, int64_t out_row_stride, int64_t out_batch_stride,
                               ns2_stream_t stream) {
  using namespace ns2;
  NS2_REQUIRE(batch >= 0 && length >= 0, "ns2_seanet_head: negative size");
  if (batch == 0 || length == 0) return kOk;
  NS2_REQUIRE(batch <= 65535, "ns2_seanet_head: batch=%d above 65535", batch);
  NS2_REQUIRE(x != nullptr && params != nullptr && out_bf16 != nullptr, "ns2_seanet_head: NULL pointer");
  NS2_REQUIRE(batch == 1 || x_batch_stride >= length, "ns2_seanet_head: x batch stride %lld below length %d",
              (long long)x_batch_stride, length);
  NS2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 3) == 0 && (reinterpret_cast<uintptr_t>(params) & 15) == 0,
              "ns2_seanet_head: x must be 4-byte and params 16-byte aligned");
  NS2_REQUIRE(out_row_stride >= 32 && out_row_stride % 8 == 0 && out_batch_stride % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0,
              "ns2_seanet_head: out (32 channels) must be 16-byte aligned with strides multiple of 8");
  NS2_REQUIRE(batch == 1 || out_batch_stride >= (length + 2LL) * out_row_stride,
              "ns2_seanet_head: out batch stride %lld below (length + 2) rows", (long long)out_batch_stride);
  const int smem = kHeadSmemFloats * 4;
  NS2_CUDA_CHECK(set_max_smem_once(seanet_head_kernel, smem));
  const dim3 grid((length + kHeadOut - 1) / kHeadOut, batch);
  seanet_head_kernel<<<grid, kHeadThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      x, x_batch_stride, length, params, static_cast<__nv_bfloat16*>(out_bf16), out_row_stride, out_batch_stride);
  return launched(1);
}
