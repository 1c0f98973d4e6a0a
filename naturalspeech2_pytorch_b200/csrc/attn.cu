// Flash attention forward on wgmma for sm_90a (non-causal, unmasked, dim_head = 64).
// Replaces Attend.forward / F.scaled_dot_product_attention (attend.py:77-155) for the only configuration
// the denoiser uses: mask=None, causal=False, dropout=0 (SURVEY T9).
//
// One CTA per (batch, head, 128-query tile); 384 threads:
//   warpgroup 0     TMA producer (warp 0): Q once, then K_j / V_j tiles (128 keys x 64) through a KVS-stage ring
//   warpgroups 1-2  softmax warpgroups, 64 query rows each: S = Q K_j^T by wgmma (both operands K-major in shared
//                   memory, fp32 accumulator fragments in registers) -> online softmax in fp32 -> P packed to bf16
//                   straight from the S fragments into the A-operand fragments of O += P V_j (register-A wgmma; V is
//                   the MN-major B operand: its rows are keys = the reduction dimension, so V is never transposed)
//
// attn_fwd_kernel<true> adds the attention dropout of Attend (attend.py:106 / 149: dropout on the softmax probabilities
// while training).  The keep bits of a key tile come from Philox (philox.cuh), drawn while the S wgmma runs.  The row
// sums l and the saved log-sum-exp use the undropped probabilities (lse is bit-identical to attn_fwd_kernel<false>'s),
// each P element is multiplied by its keep bit before it becomes an A fragment of O += P V, and 1 / (1 - p) is applied
// once, with 1 / l, when O is stored.
//
// attn_fwd_kernel<false, true> is the key-padding variant of sampling a batch of sequences of different lengths
// (Attend with a key mask, attend.py:123-129 / 140-142, which the reference builds but never reaches, SURVEY T9):
// sample b attends to keys [0, kv_lens[b]).  Both the producer and the softmax warpgroups take the key-tile count from
// that length and the last tile masks the keys past it to -inf, exactly as keys past kv_len are masked; those keys'
// P is 0, so their (finite) V rows add 0 to O.  A sample's output is therefore bit-identical to the plain kernel called
// on its keys [0, kv_lens[b]) alone, whose padding keys are the TMA zero fill.
#include "ptx.cuh"
#include "philox.cuh"
#include "host_common.h"
#include "../../include/ns2_b200.h"

namespace ns2 {

namespace attn {
constexpr int BQ = 128;   // queries per CTA (64 per softmax warpgroup)
constexpr int BKV = 128;  // keys per tile
constexpr int DH = 64;
constexpr int KVS = 3;    // K/V ring depth
constexpr int Q_BYTES = BQ * DH * 2;         // 16 KB
constexpr int KV_BYTES = BKV * DH * 2;       // 16 KB each for K and V
constexpr int OFF_Q = 0;
constexpr int OFF_K = OFF_Q + Q_BYTES;                 // KVS stages
constexpr int OFF_V = OFF_K + KVS * KV_BYTES;          // KVS stages
constexpr int OFF_BAR = OFF_V + KVS * KV_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 256;              // 112.25 KB
constexpr int THREADS = 384;
}  // namespace attn

struct AttnDev {
  CUtensorMap tmQ, tmK, tmV;
  __nv_bfloat16* out;
  long long o_rs, o_bs;
  int q_len, kv_len;
  float scale_log2e;
  float* lse;   // optional (batches, heads, q_len): log2-domain log-sum-exp of the scaled scores, for the backward pass
  DropoutDev drop;   // attn_fwd_kernel<true, false> only
  const int* kv_lens;   // attn_fwd_kernel<false, true> only: (batches) key counts, clamped to [1, kv_len]
  const int* q_lens;    // attn_fwd_kernel<false, *, true> only: (batches) query counts, clamped to [1, q_len]
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float keep_if(float x, uint32_t bits, int n) { return (bits >> n) & 1u ? x : 0.f; }

// attn_fwd_kernel<false, *, true> (ns2_attn_args.q_lens) adds query padding: a CTA whose query tile starts at or past
// q_lens[b] returns before it touches anything, the others run exactly as attn_fwd_kernel<false, RAGGED>.
template <bool DROPOUT, bool RAGGED, bool QLENS = false>
__global__ void __launch_bounds__(attn::THREADS, 1) attn_fwd_kernel(const __grid_constant__ AttnDev p) {
  static_assert(!(DROPOUT && RAGGED), "no dropout variant of the key-padding kernel");
  static_assert(!(DROPOUT && QLENS), "no dropout variant of the query-padding kernel");
  using namespace attn;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;            // [KVS]
  uint64_t* kv_empty = bars + 1 + KVS;     // [KVS] one arrive per softmax warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * BQ;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  if (QLENS && q0 >= min(max(__ldg(p.q_lens + b), 1), p.q_len)) return;   // uniform over the CTA
  // keys of this sample; the plain kernels read p.kv_len where they use it, which keeps their code as it was
  const int kv_len_b = RAGGED ? min(max(__ldg(p.kv_lens + b), 1), p.kv_len) : 0;
#define NS2_ATTN_KV_LEN (RAGGED ? kv_len_b : p.kv_len)
  const int T = (NS2_ATTN_KV_LEN + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // dynamic smem not 1024-byte aligned (no printf: see mbar_wait)
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    mbar_init(smem_u32(q_full), 1);
    for (int i = 0; i < KVS; ++i) {
      mbar_init(smem_u32(&kv_full[i]), 1);
      mbar_init(smem_u32(&kv_empty[i]), 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    // ================================ TMA producer ================================
    if (warp == 0 && lane == 0) {
      mbar_arrive_expect_tx(smem_u32(q_full), Q_BYTES);
      tma_load_3d(smem_u32(smem + OFF_Q), &p.tmQ, smem_u32(q_full), head * DH, q0, b);
      for (int j = 0; j < T; ++j) {
        const int st = j % KVS;
        const uint32_t ph = (j / KVS) & 1;
        mbar_wait(smem_u32(&kv_empty[st]), ph ^ 1);
        const uint32_t fb = smem_u32(&kv_full[st]);
        mbar_arrive_expect_tx(fb, 2 * KV_BYTES);
        tma_load_3d(smem_u32(smem + OFF_K + st * KV_BYTES), &p.tmK, fb, head * DH, j * BKV, b);
        tma_load_3d(smem_u32(smem + OFF_V + st * KV_BYTES), &p.tmV, fb, head * DH, j * BKV, b);
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ================================ softmax warpgroups ===============================
    const int w = (warp >> 2) - 1;              // query rows [64 w, 64 w + 64) of the tile
    const int r0 = 64 * w + 16 * (warp & 3) + (lane >> 2);   // this thread's rows: r0 and r0 + 8
    const int c2 = 2 * (lane & 3);
    const float c = p.scale_log2e;
    float o_acc[DH / 2];
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) o_acc[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: this thread's partial row sums
    const uint64_t dq = gmma_desc_sw128(smem_u32(smem + OFF_Q + w * (64 * 128)), 16, 1024);
    mbar_wait(smem_u32(q_full), 0);

    for (int j = 0; j < T; ++j) {
      const int st = j % KVS;
      mbar_wait(smem_u32(&kv_full[st]), (j / KVS) & 1);
      float s[BKV / 2];
      uint32_t keep[2];   // DROPOUT: keep bit of S fragment element n = 4 jj + e is bit n & 31 of keep[n >> 5]
      {
        const uint64_t dk = gmma_desc_sw128(smem_u32(smem + OFF_K + st * KV_BYTES), 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < DH / 16; ++k) wgmma_bf16_ss_n128<0, 0>(s, dq + 2 * k, dk + 2 * k, k > 0 ? 1u : 0u);
        wgmma_commit();
        if constexpr (DROPOUT) {   // one Philox block per (16-key group kk, column t): rows r0, r0 + 8 x keys k, k + 8
          const uint32_t cq = philox_attn_index(q0 + r0), cbh = b * gridDim.y + head, th = p.drop.threshold;
#pragma unroll
          for (int h = 0; h < 2; ++h) {   // keep[h]: 16-key groups 4 h .. 4 h + 3
            keep[h] = 0u;
#pragma unroll 1   // one group at a time: unrolled, the Philox rounds of all groups would spill the accumulators
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
              for (int t = 0; t < 2; ++t) {
                const Philox4 r = philox4x32_10(philox_attn_index(j * BKV + 16 * (4 * h + kk) + c2 + t), cq, cbh,
                                                p.drop.site, p.drop.key0, p.drop.key1);
                const int n = 8 * kk + t;   // element 4 (2 kk) + t of the word; +4: key + 8; +2: row + 8
                keep[h] |= (r.x >= th ? 1u : 0u) << n | (r.y >= th ? 1u : 0u) << (n + 4) |
                           (r.z >= th ? 1u : 0u) << (n + 2) | (r.w >= th ? 1u : 0u) << (n + 6);
              }
          }
        }
        wgmma_wait<0>();
        wgmma_hold(s);
      }
      const int valid = NS2_ATTN_KV_LEN - j * BKV;  // columns >= valid are padding keys (TMA zero-filled or past kv_lens[b])
      if (valid < BKV) {
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (8 * jj + c2 + (e & 1) >= valid) s[4 * jj + e] = -INFINITY;
      }
      float a[2], m_new[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float m = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj) m = fmaxf(m, fmaxf(s[4 * jj + 2 * i], s[4 * jj + 2 * i + 1]));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));   // the four threads of a quad share the row
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        m_new[i] = fmaxf(m_run[i], m * c);
        a[i] = ex2_approx(m_run[i] - m_new[i]);   // 0 on the first tile (m_run = -inf)
        m_run[i] = m_new[i];
        l_run[i] *= a[i];
      }
#pragma unroll
      for (int jj = 0; jj < DH / 8; ++jj) {
        o_acc[4 * jj + 0] *= a[0];
        o_acc[4 * jj + 1] *= a[0];
        o_acc[4 * jj + 2] *= a[1];
        o_acc[4 * jj + 3] *= a[1];
      }
      // P = exp2(s c - m) -> bf16 A fragments (16 keys per k-step: S fragments 2k and 2k + 1)
      uint32_t pa[BKV / 16][4];
#pragma unroll
      for (int jj = 0; jj < BKV / 8; ++jj) {
        const float p0 = ex2_approx(fmaf(s[4 * jj + 0], c, -m_new[0]));
        const float p1 = ex2_approx(fmaf(s[4 * jj + 1], c, -m_new[0]));
        const float p2 = ex2_approx(fmaf(s[4 * jj + 2], c, -m_new[1]));
        const float p3 = ex2_approx(fmaf(s[4 * jj + 3], c, -m_new[1]));
        l_run[0] += p0 + p1;
        l_run[1] += p2 + p3;
        if constexpr (DROPOUT) {
          const uint32_t kb = keep[jj >> 3];
          const int n = (4 * jj) & 31;
          pa[jj >> 1][(jj & 1) * 2 + 0] = pack_bf16x2(keep_if(p0, kb, n), keep_if(p1, kb, n + 1));
          pa[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16x2(keep_if(p2, kb, n + 2), keep_if(p3, kb, n + 3));
        } else {
          pa[jj >> 1][(jj & 1) * 2 + 0] = pack_bf16x2(p0, p1);
          pa[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16x2(p2, p3);
        }
      }
      {
        const uint32_t vbase = smem_u32(smem + OFF_V + st * KV_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BKV / 16; ++k)   // B = V: MN-major (64 dh contiguous per key row); 16 keys = 2048 bytes
          wgmma_bf16_rs_n64<1>(o_acc, pa[k], gmma_desc_sw128(vbase + k * 2048, 1024, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_hold(o_acc);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&kv_empty[st]));
    }

#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float l = l_run[i];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const int qrow = q0 + r0 + 8 * i;
      if (qrow < p.q_len) {
        const float inv = DROPOUT ? p.drop.scale / l : 1.0f / l;
        if (p.lse != nullptr && (lane & 3) == 0)
          p.lse[(static_cast<long long>(b) * gridDim.y + head) * p.q_len + qrow] = m_run[i] + log2f(l);
        __nv_bfloat16* op = p.out + static_cast<long long>(b) * p.o_bs + static_cast<long long>(qrow) * p.o_rs +
                            head * DH + c2;
#pragma unroll
        for (int jj = 0; jj < DH / 8; ++jj)
          *reinterpret_cast<uint32_t*>(op + 8 * jj) =
              pack_bf16x2(o_acc[4 * jj + 2 * i] * inv, o_acc[4 * jj + 2 * i + 1] * inv);
      }
    }
  }
#undef NS2_ATTN_KV_LEN
}

template <bool DROPOUT, bool RAGGED, bool QLENS>
static int launch(const AttnDev& dev, dim3 grid, cudaStream_t stream) {
  NS2_CUDA_CHECK(set_max_smem_once(attn_fwd_kernel<DROPOUT, RAGGED, QLENS>, attn::SMEM_BYTES));
  attn_fwd_kernel<DROPOUT, RAGGED, QLENS><<<grid, attn::THREADS, attn::SMEM_BYTES, stream>>>(dev);
  return launched(1);
}

}  // namespace ns2

using namespace ns2;

// No dropout (or p = 0) and no lengths: the plain kernel; dropout with p > 0: attn_fwd_kernel<true, false>; kv_lens:
// attn_fwd_kernel<false, true> (never with dropout); q_lens: attn_fwd_kernel<false, kv_lens != NULL, true>.
extern "C" int ns2_attn_fwd(const ns2_attn_args* a, ns2_stream_t stream_) {
  NS2_REQUIRE(a != nullptr, "attn_fwd: NULL args");
  const ns2_dropout* d = a->dropout;
  DropoutDev drop;
  NS2_REQUIRE(d == nullptr || make_dropout_dev(d->seed, d->site, d->p, &drop), "attn_fwd: dropout p=%g is not in [0, 1)",
              static_cast<double>(d->p));
  const bool dropout = d != nullptr && d->p != 0.0f;
  NS2_REQUIRE(!(dropout && a->kv_lens), "attn_fwd: kv_lens with dropout p > 0 is not supported");
  NS2_REQUIRE(!(dropout && a->q_lens), "attn_fwd: q_lens with dropout p > 0 is not supported");
  NS2_REQUIRE(a->q && a->k && a->v && a->out, "attn_fwd: NULL pointer");
  NS2_REQUIRE(a->dim_head == 64, "attn_fwd: dim_head=%d, only 64 is supported", a->dim_head);
  NS2_REQUIRE(a->batches > 0 && a->heads > 0 && a->q_len > 0 && a->kv_len > 0, "attn_fwd: empty problem");
  NS2_REQUIRE(a->o_row_stride % 8 == 0 && a->o_batch_stride % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
              "attn_fwd: out must be 16-byte aligned with strides multiple of 8");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  AttnDev dev;
  memset(&dev, 0, sizeof(dev));
  const uint32_t box[3] = {64, attn::BQ, 1};
  const uint32_t box_kv[3] = {64, attn::BKV, 1};
  {
    const uint64_t dims[3] = {(uint64_t)a->heads * 64, (uint64_t)a->q_len, (uint64_t)a->batches};
    const uint64_t str[3] = {2, (uint64_t)a->q_row_stride * 2, (uint64_t)a->q_batch_stride * 2};
    int rc = make_tmap_16bit(&dev.tmQ, a->q, 3, dims, str, box);
    if (rc != kOk) return rc;
  }
  {
    const uint64_t dims[3] = {(uint64_t)a->heads * 64, (uint64_t)a->kv_len, (uint64_t)a->batches};
    const uint64_t strk[3] = {2, (uint64_t)a->k_row_stride * 2, (uint64_t)a->k_batch_stride * 2};
    const uint64_t strv[3] = {2, (uint64_t)a->v_row_stride * 2, (uint64_t)a->v_batch_stride * 2};
    int rc = make_tmap_16bit(&dev.tmK, a->k, 3, dims, strk, box_kv);
    if (rc != kOk) return rc;
    rc = make_tmap_16bit(&dev.tmV, a->v, 3, dims, strv, box_kv);
    if (rc != kOk) return rc;
  }
  dev.out = reinterpret_cast<__nv_bfloat16*>(a->out);
  dev.o_rs = a->o_row_stride;
  dev.o_bs = a->o_batch_stride;
  dev.q_len = a->q_len;
  dev.kv_len = a->kv_len;
  dev.scale_log2e = a->scale * 1.4426950408889634f;
  dev.lse = a->lse;
  dim3 grid((a->q_len + attn::BQ - 1) / attn::BQ, a->heads, a->batches);
  dev.kv_lens = a->kv_lens;
  dev.q_lens = a->q_lens;
  if (a->q_lens != nullptr)
    return a->kv_lens != nullptr ? launch<false, true, true>(dev, grid, stream)
                                 : launch<false, false, true>(dev, grid, stream);
  if (a->kv_lens != nullptr) return launch<false, true, false>(dev, grid, stream);
  if (!dropout) return launch<false, false, false>(dev, grid, stream);
  dev.drop = drop;
  return launch<true, false, false>(dev, grid, stream);
}
