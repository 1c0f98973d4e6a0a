// Flash-attention backward on wgmma for sm_90a (non-causal, unmasked, dim_head = 64) — the backward of
// Attend.forward / F.scaled_dot_product_attention (attend.py:77-155) that autograd runs for the reference's
// loss.backward() (README.md:63, ns2.py:1886).
//
//   P = exp(S*scale - L)      S = Q K^T, L = row log-sum-exp saved by the forward kernel
//   dV = P^T dO               dP = dO V^T               D = rowsum(dO * O)   (ns2_attn_bwd_delta)
//   dS = P * (dP - D) * scale dQ = dS K                 dK = dS^T Q
//
// One CTA per (batch, head, 128-key tile j); it walks over the 64-query tiles i.  384 threads:
//   warpgroup 0     TMA producer (warp 0): K_j, V_j once; Q_i, dO_i through a 2-stage ring
//   warpgroups 1-2  warpgroup w owns keys [64 (w-1), 64 w) of the tile.  S^T = K Q_i^T and dP^T = V dO_i^T come out of
//                   wgmma with the keys as accumulator rows, so P^T and dS^T are formed in registers and feed
//                   dV += P^T dO_i and dK += dS^T Q_i directly as register A operands (dO_i, Q_i are MN-major B
//                   operands: nothing is ever transposed).  dS^T also goes to 128B-swizzled shared memory, from where
//                   dQ_i (partial over this warpgroup's keys) = dS K is computed with dS as the MN-major A operand and
//                   added into the fp32 dQ accumulator with global reductions (every key tile contributes to every
//                   query row).  dK_j / dV_j stay in registers over all query tiles and are stored once at the end.
//
// attn_bwd_kernel<true> is the backward of attn_fwd_kernel<true> (attention dropout, mask M, s = 1 / (1 - p)).  It
// regenerates M from (seed, site, b, h, q, k) with Philox (philox.cuh) while the S^T / dP^T wgmma run:
//   dV = (P * M)^T dO s (s applied when dV is stored)    dP = (dO V^T) * M s    dS = P * (dP - D) * scale
// with D = rowsum(dO * O) of the dropped output O, so attn_delta_kernel is unchanged.
//
// attn_bwd_kernel<false, true> is the backward of attn_fwd_kernel<false, true> (key padding: sample b attends to keys
// [0, kv_lens[b]) only).  A CTA whose key tile starts at or past kv_lens[b] writes its dK / dV rows as exact zeros and
// exits: no TMA, nothing added to dQ.  The last valid tile masks P and dS^T to 0 for the keys past kv_lens[b], exactly
// as keys past kv_len are masked; those K / V rows hold finite data (not the TMA zero fill), and forcing dS^T to 0
// keeps junk in them out of dK, while their dK / dV rows come out as exact zeros.  The forward's lse covers only the
// valid keys, so sample b's dK / dV are bit-identical to the plain kernel called on its keys alone.
#include "ptx.cuh"
#include "philox.cuh"
#include "host_common.h"
#include "../../include/ns2_b200.h"

namespace ns2 {

namespace ab {
constexpr int BQ = 64, BKV = 128, DH = 64;
constexpr int KV_BYTES = BKV * DH * 2;      // 16 KB: a [128 keys][64 x bf16] tile
constexpr int QT_BYTES = BQ * DH * 2;       // 8 KB: a [64 queries][64 x bf16] tile
constexpr int OFF_K = 0, OFF_V = KV_BYTES;
constexpr int OFF_Q = 2 * KV_BYTES;                 // [2 stages]
constexpr int OFF_DO = OFF_Q + 2 * QT_BYTES;        // [2 stages]
constexpr int OFF_DS = OFF_DO + 2 * QT_BYTES;       // dS^T: [128 keys][64 queries] bf16, 128B-swizzled rows
constexpr int OFF_BAR = OFF_DS + BKV * BQ * 2;
constexpr int SMEM_BYTES = OFF_BAR + 256;           // 80.25 KB
constexpr int OFF_KEEP = SMEM_BYTES;                // attn_bwd_kernel<true>: one keep-bit word per gradient thread
constexpr int SMEM_BYTES_DROPOUT = OFF_KEEP + 256 * 4;
constexpr int THREADS = 384;
}  // namespace ab

struct AttnBwdDev {
  CUtensorMap tmQ, tmK, tmV, tmDO;
  const float* lse;     // (batches, heads, q_len): log2-domain log-sum-exp of the scaled scores
  const float* delta;   // (batches, heads, q_len): rowsum(dO * O)
  float* dq;            // (batches, q_len, heads * 64) fp32 accumulator
  __nv_bfloat16* dk;
  __nv_bfloat16* dv;
  long long dk_rs, dk_bs, dv_rs, dv_bs;
  int q_len, kv_len, heads;
  float scale, scale_log2e;
  DropoutDev drop;      // attn_bwd_kernel<true, false> only
  const int* kv_lens;   // attn_bwd_kernel<false, true> only: (batches) key counts, clamped to [1, kv_len]
};

__device__ __forceinline__ float ab_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float ab_keep_if(float x, uint32_t bits, int n) { return (bits >> n) & 1u ? x : 0.f; }

template <bool DROPOUT, bool RAGGED>
__global__ void __launch_bounds__(ab::THREADS, 1) attn_bwd_kernel(const __grid_constant__ AttnBwdDev p) {
  static_assert(!(DROPOUT && RAGGED), "no dropout variant of the key-padding kernel");
  using namespace ab;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* kv_full = bars + 0;
  uint64_t* q_full = bars + 1;     // [2]
  uint64_t* q_empty = bars + 3;    // [2] one arrive per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int TQ = (p.q_len + BQ - 1) / BQ;
  // keys of this sample; the plain kernels read p.kv_len where they use it, which keeps their code as it was
  const int kv_len_b = RAGGED ? min(max(__ldg(p.kv_lens + b), 1), p.kv_len) : 0;
#define NS2_ATTN_BWD_KV_LEN (RAGGED ? kv_len_b : p.kv_len)
  if constexpr (RAGGED) {
    if (j * BKV >= kv_len_b) {   // every key of the tile is padding: dK = dV = 0, nothing else to do
      const int rows = min(BKV, p.kv_len - j * BKV);
      for (int idx = threadIdx.x; idx < rows * (DH / 2); idx += THREADS) {
        const long long key = j * BKV + idx / (DH / 2);
        const int col = head * DH + 2 * (idx % (DH / 2));
        *reinterpret_cast<uint32_t*>(p.dk + b * p.dk_bs + key * p.dk_rs + col) = 0u;
        *reinterpret_cast<uint32_t*>(p.dv + b * p.dv_bs + key * p.dv_rs + col) = 0u;
      }
      return;
    }
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    tma_prefetch_desc(&p.tmDO);
    mbar_init(smem_u32(kv_full), 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(smem_u32(&q_full[i]), 1);
      mbar_init(smem_u32(&q_empty[i]), 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    // ================================ TMA producer ================================
    if (warp == 0) {
      if (elect_one()) {
        mbar_arrive_expect_tx(smem_u32(kv_full), 2 * KV_BYTES);
        tma_load_3d(smem_u32(smem + OFF_K), &p.tmK, smem_u32(kv_full), head * DH, j * BKV, b);
        tma_load_3d(smem_u32(smem + OFF_V), &p.tmV, smem_u32(kv_full), head * DH, j * BKV, b);
      }
      __syncwarp();
      for (int i = 0; i < TQ; ++i) {
        const int st = i & 1;
        mbar_wait(smem_u32(&q_empty[st]), ((i >> 1) & 1) ^ 1);
        if (elect_one()) {
          const uint32_t fb = smem_u32(&q_full[st]);
          mbar_arrive_expect_tx(fb, 2 * QT_BYTES);
          tma_load_3d(smem_u32(smem + OFF_Q + st * QT_BYTES), &p.tmQ, fb, head * DH, i * BQ, b);
          tma_load_3d(smem_u32(smem + OFF_DO + st * QT_BYTES), &p.tmDO, fb, head * DH, i * BQ, b);
        }
        __syncwarp();
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ================================ gradient warpgroups ===============================
    const int w = (warp >> 2) - 1;
    const int kr0 = 64 * w + 16 * (warp & 3) + (lane >> 2);   // this thread's key rows (in the tile): kr0, kr0 + 8
    const int c2 = 2 * (lane & 3);
    const int valid = NS2_ATTN_BWD_KV_LEN - j * BKV;   // keys of this tile that exist (or are not past kv_lens[b])
    const uint32_t k_s = smem_u32(smem + OFF_K) + w * (64 * 128), v_s = smem_u32(smem + OFF_V) + w * (64 * 128);
    const uint32_t ds_s = smem_u32(smem + OFF_DS) + w * (64 * 128);
    uint8_t* ds_rows = smem + OFF_DS;
    const long long inner = static_cast<long long>(p.heads) * DH;
    float dv_acc[DH / 2], dk_acc[DH / 2];
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) {
      dv_acc[i] = 0.f;
      dk_acc[i] = 0.f;
    }
    mbar_wait(smem_u32(kv_full), 0);
    for (int i = 0; i < TQ; ++i) {
      const int st = i & 1;
      mbar_wait(smem_u32(&q_full[st]), (i >> 1) & 1);
      const uint32_t q_s = smem_u32(smem + OFF_Q + st * QT_BYTES), do_s = smem_u32(smem + OFF_DO + st * QT_BYTES);
      // DROPOUT: keep bit of fragment element n = 4 jj + e (key row kr0 + 8 (e >> 1), query 8 jj + c2 + (e & 1)) is bit n
      // of this thread's word at keep_s.  Drawn before the S^T / dP^T wgmma are issued (their accumulators are not live
      // yet) and parked in shared memory, re-read per fragment column: a register held across the P^T / dS^T loop spills.
      const uint32_t keep_s = smem_u32(smem + OFF_KEEP) + 4 * (threadIdx.x - 128);
      if constexpr (DROPOUT) {   // one Philox block per (16-query group g >> 1, column g & 1): keys kr0, kr0 + 8 x queries q, q + 8
        const uint32_t ck = philox_attn_index(j * BKV + kr0), cbh = b * p.heads + head, th = p.drop.threshold;
        uint32_t keep = 0u;
#pragma unroll 1   // one block at a time: unrolled, the Philox rounds would spill the accumulators
        for (int g = 0; g < BQ / 8; ++g) {
          const int qq = g >> 1, t = g & 1;
          const Philox4 r = philox4x32_10(ck, philox_attn_index(i * BQ + 16 * qq + c2 + t), cbh, p.drop.site,
                                          p.drop.key0, p.drop.key1);
          const int n = 8 * qq + t;   // element 4 (2 qq) + t; +2: key + 8; +4: query + 8
          keep |= (r.x >= th ? 1u : 0u) << n | (r.y >= th ? 1u : 0u) << (n + 2) | (r.z >= th ? 1u : 0u) << (n + 4) |
                  (r.w >= th ? 1u : 0u) << (n + 6);
        }
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(keep_s), "r"(keep));
      }
      // S^T = K Q_i^T, dP^T = V dO_i^T (keys x queries; both operands K-major)
      float s[BQ / 2], dp[BQ / 2];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < DH / 16; ++k)
        wgmma_bf16_ss_n64<0, 0>(s, gmma_desc_sw128(k_s, 16, 1024) + 2 * k, gmma_desc_sw128(q_s, 16, 1024) + 2 * k,
                                k > 0 ? 1u : 0u);
#pragma unroll
      for (int k = 0; k < DH / 16; ++k)
        wgmma_bf16_ss_n64<0, 0>(dp, gmma_desc_sw128(v_s, 16, 1024) + 2 * k, gmma_desc_sw128(do_s, 16, 1024) + 2 * k,
                                k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(s);
      wgmma_hold(dp);
      // P^T, dS^T -> bf16 register A fragments (16 queries per k-step) and dS^T -> shared memory
      uint32_t pa[BQ / 16][4], da[BQ / 16][4];
#pragma unroll
      for (int jj = 0; jj < BQ / 8; ++jj) {
        const int qc = 8 * jj + c2;   // query column (in the tile) of elements e = 0, 1
        float L[2], Dl[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int q = i * BQ + qc + e;
          const bool q_ok = q < p.q_len;
          const long long sidx = (static_cast<long long>(b) * p.heads + head) * p.q_len + q;
          L[e] = q_ok ? __ldg(p.lse + sidx) : INFINITY;
          Dl[e] = q_ok ? __ldg(p.delta + sidx) : 0.f;
        }
        float pv[4], dv[4];
        uint32_t keep = 0u;
        if constexpr (DROPOUT) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(keep) : "r"(keep_s));
#pragma unroll
        for (int e = 0; e < 4; ++e) {   // e = 2 r + t: key row kr0 + 8 r, query column qc + t
          const int r = e >> 1, t = e & 1;
          float pp = ab_ex2(fmaf(s[4 * jj + e], p.scale_log2e, -L[t]));
          const bool pad_key = kr0 + 8 * r >= valid;
          if (pad_key) pp = 0.f;
          if constexpr (DROPOUT) {
            pv[e] = ab_keep_if(pp, keep, 4 * jj + e);
            dv[e] = pp * (ab_keep_if(dp[4 * jj + e], keep, 4 * jj + e) * p.drop.scale - Dl[t]) * p.scale;
          } else {
            pv[e] = pp;
            dv[e] = pp * (dp[4 * jj + e] - Dl[t]) * p.scale;
          }
          // a softmax over one key is the constant 1: dS = 0 exactly, not the rounding left of dP - D (dP and
          // D = rowsum(dO * O) are summed in different orders), so dQ and dK come out as exact zeros
          if (NS2_ATTN_BWD_KV_LEN == 1) dv[e] = 0.f;
          // a padding key's dP is formed from its finite but arbitrary V row: dS = 0 outright, not 0 * dP
          if (RAGGED && pad_key) dv[e] = 0.f;
        }
        pa[jj >> 1][(jj & 1) * 2 + 0] = pack_bf16x2(pv[0], pv[1]);
        pa[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16x2(pv[2], pv[3]);
        const uint32_t d0 = pack_bf16x2(dv[0], dv[1]), d1 = pack_bf16x2(dv[2], dv[3]);
        da[jj >> 1][(jj & 1) * 2 + 0] = d0;
        da[jj >> 1][(jj & 1) * 2 + 1] = d1;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int key = kr0 + 8 * r;
          *reinterpret_cast<uint32_t*>(ds_rows + key * 128 + ((jj ^ (key & 7)) << 4) + c2 * 2) = r ? d1 : d0;
        }
      }
      fence_proxy_async_smem();
      warpgroup_bar(w);
      // dV += P^T dO_i, dK += dS^T Q_i (B operands MN-major: 16 queries = 2048 bytes per step);
      // dQ_i = dS K over this warpgroup's keys (A = dS^T in smem: MN-major; B = K: MN-major; 16 keys per step)
      float dq[DH / 2];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BQ / 16; ++k) wgmma_bf16_rs_n64<1>(dv_acc, pa[k], gmma_desc_sw128(do_s + k * 2048, 1024, 1024), 1u);
#pragma unroll
      for (int k = 0; k < BQ / 16; ++k) wgmma_bf16_rs_n64<1>(dk_acc, da[k], gmma_desc_sw128(q_s + k * 2048, 1024, 1024), 1u);
#pragma unroll
      for (int k = 0; k < 64 / 16; ++k)
        wgmma_bf16_ss_n64<1, 1>(dq, gmma_desc_sw128(ds_s + k * 2048, 1024, 1024),
                                gmma_desc_sw128(k_s + k * 2048, 1024, 1024), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(dv_acc);
      wgmma_hold(dk_acc);
      wgmma_hold(dq);
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&q_empty[st]));   // Q_i / dO_i may be overwritten
      warpgroup_bar(w);                                      // dS^T may be overwritten by the next tile
      // dQ accumulator += this warpgroup's partial (rows = queries 16 ww + lane/4 + 8 r of the tile)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int q = i * BQ + 16 * (warp & 3) + (lane >> 2) + 8 * r;
        if (q >= p.q_len) continue;
        float* dst = p.dq + (static_cast<long long>(b) * p.q_len + q) * inner + head * DH + c2;
#pragma unroll
        for (int jj = 0; jj < DH / 8; ++jj) {
          atomicAdd(dst + 8 * jj, dq[4 * jj + 2 * r]);
          atomicAdd(dst + 8 * jj + 1, dq[4 * jj + 2 * r + 1]);
        }
      }
    }
    // ---- dK_j, dV_j -> bf16 ----
    if constexpr (DROPOUT) {
#pragma unroll
      for (int i = 0; i < DH / 2; ++i) dv_acc[i] *= p.drop.scale;
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int key = j * BKV + kr0 + 8 * r;
      if (key >= p.kv_len) continue;
      __nv_bfloat16* pv = p.dv + static_cast<long long>(b) * p.dv_bs + static_cast<long long>(key) * p.dv_rs + head * DH + c2;
      __nv_bfloat16* pk = p.dk + static_cast<long long>(b) * p.dk_bs + static_cast<long long>(key) * p.dk_rs + head * DH + c2;
#pragma unroll
      for (int jj = 0; jj < DH / 8; ++jj) {
        if (RAGGED && key >= kv_len_b) {   // a padding key: exact zeros (its P and dS were 0 already)
          *reinterpret_cast<uint32_t*>(pv + 8 * jj) = 0u;
          *reinterpret_cast<uint32_t*>(pk + 8 * jj) = 0u;
          continue;
        }
        *reinterpret_cast<uint32_t*>(pv + 8 * jj) = pack_bf16x2(dv_acc[4 * jj + 2 * r], dv_acc[4 * jj + 2 * r + 1]);
        *reinterpret_cast<uint32_t*>(pk + 8 * jj) = pack_bf16x2(dk_acc[4 * jj + 2 * r], dk_acc[4 * jj + 2 * r + 1]);
      }
    }
  }
#undef NS2_ATTN_BWD_KV_LEN
}

// delta[b, h, q] = sum_d dO[b, q, h*64 + d] * O[b, q, h*64 + d]; one warp per (b, q) row, lanes over the heads' columns
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* __restrict__ o, long long o_rs, long long o_bs,
                                                         const __nv_bfloat16* __restrict__ d_o, long long do_rs,
                                                         long long do_bs, int batches, int q_len, int heads,
                                                         float* __restrict__ delta) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rowi = static_cast<long long>(blockIdx.x) * 8 + warp;
  if (rowi >= static_cast<long long>(batches) * q_len) return;
  const int b = static_cast<int>(rowi / q_len), q = static_cast<int>(rowi - static_cast<long long>(b) * q_len);
  const uint32_t* op = reinterpret_cast<const uint32_t*>(o + b * o_bs + q * o_rs);
  const uint32_t* dp = reinterpret_cast<const uint32_t*>(d_o + b * do_bs + q * do_rs);
  for (int h = 0; h < heads; ++h) {
    const uint32_t a = __ldg(op + h * 32 + lane), g = __ldg(dp + h * 32 + lane);
    float s = __uint_as_float(a << 16) * __uint_as_float(g << 16) +
              __uint_as_float(a & 0xffff0000u) * __uint_as_float(g & 0xffff0000u);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) delta[(static_cast<long long>(b) * heads + h) * q_len + q] = s;
  }
}

// attn_bwd_kernel<DROPOUT, RAGGED> over the key tiles; its caller has already launched attn_delta_kernel
template <bool DROPOUT, bool RAGGED>
static int launch(const AttnBwdDev& dev, dim3 grid, cudaStream_t stream) {
  constexpr int smem = DROPOUT ? ab::SMEM_BYTES_DROPOUT : ab::SMEM_BYTES;
  NS2_CUDA_CHECK(set_max_smem_once(attn_bwd_kernel<DROPOUT, RAGGED>, smem));
  attn_bwd_kernel<DROPOUT, RAGGED><<<grid, ab::THREADS, smem, stream>>>(dev);
  return launched(2);
}

}  // namespace ns2

using namespace ns2;

// No dropout (or p = 0) and no kv_lens: the plain kernel; dropout with p > 0: attn_bwd_kernel<true, false>; kv_lens:
// attn_bwd_kernel<false, true> (never both).
extern "C" int ns2_attn_bwd(const ns2_attn_bwd_args* a, ns2_stream_t stream_) {
  NS2_REQUIRE(a != nullptr, "attn_bwd: NULL args");
  const ns2_dropout* d = a->dropout;
  DropoutDev drop;
  NS2_REQUIRE(d == nullptr || make_dropout_dev(d->seed, d->site, d->p, &drop), "attn_bwd: dropout p=%g is not in [0, 1)",
              static_cast<double>(d->p));
  const bool dropout = d != nullptr && d->p != 0.0f;
  NS2_REQUIRE(!(dropout && a->kv_lens), "attn_bwd: kv_lens with dropout p > 0 is not supported");
  NS2_REQUIRE(a->q && a->k && a->v && a->o && a->d_o && a->lse && a->delta && a->dq_accum && a->dk && a->dv,
              "attn_bwd: NULL pointer");
  NS2_REQUIRE(a->dim_head == 64, "attn_bwd: dim_head=%d, only 64 is supported", a->dim_head);
  NS2_REQUIRE(a->batches > 0 && a->heads > 0 && a->q_len > 0 && a->kv_len > 0, "attn_bwd: empty problem");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // 1. delta = rowsum(dO * O)
  {
    const long long rows = static_cast<long long>(a->batches) * a->q_len;
    attn_delta_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(a->o), a->o_row_stride, a->o_batch_stride,
        reinterpret_cast<const __nv_bfloat16*>(a->d_o), a->do_row_stride, a->do_batch_stride, a->batches, a->q_len,
        a->heads, a->delta);
  }
  AttnBwdDev dev;
  memset(&dev, 0, sizeof(dev));
  const uint64_t inner = (uint64_t)a->heads * 64;
  auto map16 = [&](CUtensorMap* m, const void* ptr, int len, int64_t rs, int64_t bs, uint32_t rows) {
    const uint64_t dims[3] = {inner, (uint64_t)len, (uint64_t)a->batches};
    const uint64_t str[3] = {2, (uint64_t)rs * 2, (uint64_t)bs * 2};
    const uint32_t box[3] = {64, rows, 1};
    return make_tmap_16bit(m, ptr, 3, dims, str, box);
  };
  int rc;
  if ((rc = map16(&dev.tmQ, a->q, a->q_len, a->q_row_stride, a->q_batch_stride, ab::BQ)) != kOk) return rc;
  if ((rc = map16(&dev.tmK, a->k, a->kv_len, a->k_row_stride, a->k_batch_stride, ab::BKV)) != kOk) return rc;
  if ((rc = map16(&dev.tmV, a->v, a->kv_len, a->v_row_stride, a->v_batch_stride, ab::BKV)) != kOk) return rc;
  if ((rc = map16(&dev.tmDO, a->d_o, a->q_len, a->do_row_stride, a->do_batch_stride, ab::BQ)) != kOk) return rc;
  dev.dq = a->dq_accum;
  dev.lse = a->lse;
  dev.delta = a->delta;
  dev.dk = reinterpret_cast<__nv_bfloat16*>(a->dk);
  dev.dv = reinterpret_cast<__nv_bfloat16*>(a->dv);
  dev.dk_rs = a->dk_row_stride;
  dev.dk_bs = a->dk_batch_stride;
  dev.dv_rs = a->dv_row_stride;
  dev.dv_bs = a->dv_batch_stride;
  dev.q_len = a->q_len;
  dev.kv_len = a->kv_len;
  dev.heads = a->heads;
  dev.scale = a->scale;
  dev.scale_log2e = a->scale * 1.4426950408889634f;
  dim3 grid((a->kv_len + ab::BKV - 1) / ab::BKV, a->heads, a->batches);
  dev.kv_lens = a->kv_lens;
  if (a->kv_lens != nullptr) return launch<false, true>(dev, grid, stream);
  if (!dropout) return launch<false, false>(dev, grid, stream);
  dev.drop = drop;
  return launch<true, false>(dev, grid, stream);
}
