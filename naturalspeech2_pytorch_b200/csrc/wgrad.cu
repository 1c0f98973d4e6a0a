// Weight-gradient GEMM on wgmma for sm_90a (backward of every Linear / CausalConv1d on the hot path):
//
//     dW[g][n, k] += sum over batches b and positions m of  dY[b, m, g*dy_gcs + n] * X[b, m - shift*dil[g], g*x_gcs + x_col_off + k]
//
// i.e. autograd's  grad_weight = grad_output^T @ input  (torch/nn/functional linear / conv1d backward, reached from
// `loss.backward()` in the reference: README.md:63, ns2.py:1886), with the causal-conv tap shift applied to the INPUT rows.
// The contraction runs over positions, which is the strided dimension of both operands (token-major activations), so
// both MMA operands are MN-major: the TMA boxes are [64 positions][64 channels] and the descriptors carry the
// "transposed" bits — no transpose is ever materialised.  Out-of-range positions of a shifted tap are zero-filled by the
// TMA unit (the 3-D map ends each batch), exactly as in the forward conv.
//
// One CTA per (128 x BN output tile, split of the position range), 384 threads:
//   warpgroup 0     TMA producer (warp 0, converged, elect_one): dY tile (2 swizzle atoms) + X tile (BN/64 atoms) per
//                   64 positions
//   warpgroups 1-2  wgmma m64nBNk16: warpgroup w accumulates dW rows [64 (w-1), 64 w) of the tile in registers, then
//                   adds them into dW with fp32 global reductions
// Partial sums of the position splits meet in L2 through the reductions, which is also what makes the call accumulate
// into an existing gradient (autograd's .grad semantics).
#include "ptx.cuh"
#include "host_common.h"
#include "../../include/ns2_b200.h"

namespace ns2 {

namespace wg {
constexpr int BM = 128;           // dW rows per tile (output channels n)
constexpr int BKP = 64;           // positions per pipeline stage
constexpr int ATOM = 64 * BKP * 2;  // one [64 positions][64 channels] bf16 swizzle atom: 8 KB
constexpr int THREADS = 384;
template <int BN>
struct Cfg {
  static constexpr int A_BYTES = 2 * ATOM;              // 128 n-channels
  static constexpr int B_BYTES = (BN / 64) * ATOM;      // BN k-channels
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : 6;
  static constexpr int OFF_BAR = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
};
}  // namespace wg

struct WgradDev {
  float* dW;
  long long dw_rs;
  int n, k;
  CUtensorMap tmDy, tmX;
  int tiles_n, tiles_k, groups, splits;
  int rows, batches;          // positions per batch, batches
  int blocks_per_batch;       // ceil(rows / 64)
  int dy_gcs, x_gcs, x_col_off, out_grs;
  int shift_units;
  int dil[NS2_GEMM_MAX_GROUPS];
};

template <int BN>
__global__ void __launch_bounds__(wg::THREADS, 1) wgrad_kernel(const __grid_constant__ WgradDev p) {
  using namespace wg;
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + C::STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // tile / split decode
  int tile = blockIdx.x;
  const int g = tile / (p.tiles_n * p.tiles_k);
  tile -= g * p.tiles_n * p.tiles_k;
  const int tn = tile / p.tiles_k, tk = tile - tn * p.tiles_k;
  const int total_blocks = p.batches * p.blocks_per_batch;
  const int per_split = (total_blocks + p.splits - 1) / p.splits;
  const int blk0 = blockIdx.y * per_split;
  const int blk1 = (blk0 + per_split < total_blocks) ? blk0 + per_split : total_blocks;
  const int nblk = blk1 - blk0;
  if (nblk <= 0) return;  // empty split (more splits than position blocks): nothing to add

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmDy);
    tma_prefetch_desc(&p.tmX);
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(smem_u32(&full_bar[i]), 1);
      mbar_init(smem_u32(&empty_bar[i]), 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0) {
      // =============================== TMA producer ===============================
      const int shift = p.shift_units * p.dil[g];
      const int dy_c0 = g * p.dy_gcs + tn * BM;
      const int x_c0 = g * p.x_gcs + p.x_col_off + tk * BN;
      for (int i = 0; i < nblk; ++i) {
        const int blk = blk0 + i;
        const int b = blk / p.blocks_per_batch;
        const int m0 = (blk - b * p.blocks_per_batch) * BKP;
        const uint32_t stage = i % C::STAGES, phase = (i / C::STAGES) & 1;
        mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1);
        if (elect_one()) {
          const uint32_t fb = smem_u32(&full_bar[stage]);
          mbar_arrive_expect_tx(fb, C::STAGE_BYTES);
          const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES);
#pragma unroll
          for (int a = 0; a < 2; ++a) tma_load_3d(sa + a * ATOM, &p.tmDy, fb, dy_c0 + a * 64, m0, b);
#pragma unroll
          for (int a = 0; a < BN / 64; ++a)
            tma_load_3d(sa + C::A_BYTES + a * ATOM, &p.tmX, fb, x_c0 + a * 64, m0 - shift, b);
        }
        __syncwarp();
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // =============================== wgmma consumers ===============================
    const int cw = (warp >> 2) - 1;   // dW rows [64 cw, 64 cw + 64) of the tile = swizzle atom cw of the dY tile
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev_stage = -1;
    for (int i = 0; i < nblk; ++i) {
      const uint32_t stage = i % C::STAGES, phase = (i / C::STAGES) & 1;
      mbar_wait(smem_u32(&full_bar[stage]), phase);
      const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BKP / 16; ++k) {
        // 16 positions = two 8-row groups of 1024 bytes; LBO = distance between 64-channel atoms
        const uint64_t da = gmma_desc_sw128(sa + cw * ATOM + k * 2048, ATOM, 1024);
        const uint64_t db = gmma_desc_sw128(sa + C::A_BYTES + k * 2048, ATOM, 1024);
        if constexpr (BN == 256) wgmma_bf16_ss_n256<1, 1>(acc, da, db, 1u);
        else wgmma_bf16_ss_n128<1, 1>(acc, da, db, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev_stage]));
      prev_stage = static_cast<int>(stage);
    }
    wgmma_wait<0>();
    wgmma_hold(acc);
    // ---- dW += acc (fp32 reductions in L2) ----
    const int row_base = tn * BM + cw * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c2 = 2 * (lane & 3);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int n = row_base + 8 * r;
      if (n >= p.n) continue;
      float* drow = p.dW + (static_cast<long long>(g) * p.out_grs + n) * p.dw_rs;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = tk * BN + 8 * j + c2;
        if (col < p.k) {
          atomicAdd(drow + col, acc[4 * j + 2 * r]);
          atomicAdd(drow + col + 1, acc[4 * j + 2 * r + 1]);
        }
      }
    }
  }
}

}  // namespace ns2

extern "C" int ns2_wgrad(const ns2_wgrad_args* a, ns2_stream_t stream_) {
  using namespace ns2;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NS2_REQUIRE(a != nullptr && a->dY && a->X && a->dW, "ns2_wgrad: NULL pointer");
  NS2_REQUIRE(a->groups >= 1 && a->groups <= NS2_GEMM_MAX_GROUPS, "ns2_wgrad: groups=%d out of range", a->groups);
  NS2_REQUIRE(a->n > 0 && a->k > 0 && a->n % 32 == 0 && a->k % 32 == 0, "ns2_wgrad: n=%d and k=%d must be multiples of 32",
              a->n, a->k);
  NS2_REQUIRE(a->rows > 0 && a->batches > 0, "ns2_wgrad: empty activations");
  NS2_REQUIRE(a->dy_row_stride % 8 == 0 && a->dy_batch_stride % 8 == 0 && a->x_row_stride % 8 == 0 &&
                  a->x_batch_stride % 8 == 0 && a->dw_row_stride % 4 == 0,
              "ns2_wgrad: strides must be multiples of 16 bytes");
  const int bn = (a->k % 256 == 0 || a->k > 1024) ? 256 : 128;
  WgradDev dev;
  memset(&dev, 0, sizeof(dev));
  const uint32_t box[3] = {64, 64, 1};
  {
    const uint64_t dims[3] = {(uint64_t)a->dy_cols, (uint64_t)a->rows, (uint64_t)a->batches};
    const uint64_t str[3] = {2, (uint64_t)a->dy_row_stride * 2, (uint64_t)a->dy_batch_stride * 2};
    int rc = make_tmap_16bit(&dev.tmDy, a->dY, 3, dims, str, box);
    if (rc != kOk) return rc;
  }
  {
    const uint64_t dims[3] = {(uint64_t)a->x_cols, (uint64_t)a->rows, (uint64_t)a->batches};
    const uint64_t str[3] = {2, (uint64_t)a->x_row_stride * 2, (uint64_t)a->x_batch_stride * 2};
    int rc = make_tmap_16bit(&dev.tmX, a->X, 3, dims, str, box);
    if (rc != kOk) return rc;
  }
  dev.dW = a->dW;
  dev.dw_rs = a->dw_row_stride;
  dev.n = a->n;
  dev.k = a->k;
  dev.tiles_n = (a->n + wg::BM - 1) / wg::BM;
  dev.tiles_k = (a->k + bn - 1) / bn;
  dev.groups = a->groups;
  dev.rows = a->rows;
  dev.batches = a->batches;
  dev.blocks_per_batch = (a->rows + wg::BKP - 1) / wg::BKP;
  dev.dy_gcs = a->dy_group_col_stride;
  dev.x_gcs = a->x_group_col_stride;
  dev.x_col_off = a->x_col_off;
  dev.out_grs = a->dw_group_row_stride;
  dev.shift_units = a->shift_units;
  for (int g = 0; g < NS2_GEMM_MAX_GROUPS; ++g) dev.dil[g] = a->dil[g];
  // position splits: enough CTAs to fill the machine ~2x, at least 8 position blocks per split
  const int tiles = dev.tiles_n * dev.tiles_k * dev.groups;
  const int total_blocks = dev.batches * dev.blocks_per_batch;
  int splits = (2 * num_sms() + tiles - 1) / tiles;
  if (splits > total_blocks / 8) splits = total_blocks / 8;
  if (splits < 1) splits = 1;
  if (a->splits > 0) splits = a->splits;
  dev.splits = splits;
  dim3 grid(tiles, splits);
  if (bn == 256) {
    NS2_CUDA_CHECK(set_max_smem_once(wgrad_kernel<256>, wg::Cfg<256>::SMEM_BYTES));
    wgrad_kernel<256><<<grid, wg::THREADS, wg::Cfg<256>::SMEM_BYTES, stream>>>(dev);
  } else {
    NS2_CUDA_CHECK(set_max_smem_once(wgrad_kernel<128>, wg::Cfg<128>::SMEM_BYTES));
    wgrad_kernel<128><<<grid, wg::THREADS, wg::Cfg<128>::SMEM_BYTES, stream>>>(dev);
  }
  return launched(1);
}
