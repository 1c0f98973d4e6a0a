// Segmented wgmma GEMM for sm_90a with fused epilogues (see include/ns2_b200.h, section 1).
//
// gemm_kernel: persistent (one CTA per SM), 384 threads, warp-specialised, 128 positions x BN columns per tile:
//   warpgroup 0    TMA producer (warp 0): A tile (128 positions x 64 channels, 3-D map so that shifted rows of a causal
//                  conv that fall before position 0 are zero-filled by the TMA unit) + B tile (BN rows x 64 channels)
//                  through a smem ring (full / empty mbarriers)
//   warpgroups 1-2 consumers: warpgroup w owns positions [64 (w-1), 64 w) of the tile, issues wgmma m64nBNk16 from the
//                  shared-memory ring into register accumulators, then runs the epilogue (bias / residual / GEGLU /
//                  FiLM + gate) in registers, stages the results in shared memory (two 8 KB boxes per warpgroup)
//                  and writes them with TMA stores; the in-place fp32 residual is added by TMA reduce-add at L2.
//                  The tile's column vectors (bias, FiLM) are copied into shared memory by cp.async while its
//                  mainloop runs, so the epilogue reads them from there instead of waiting on global loads
// Tiles are handed out by a static round robin, n fastest so co-resident CTAs share A rows in L2.
//
// Replaces, in the reference: nn.Linear GEMMs (ns2.py:1021,1024,1051-1053,783,613,731) and
// CausalConv1d (ns2.py:583-595) incl. the WavenetResBlock body (ns2.py:619-636) and GEGLU (1004-1007).
#include "ptx.cuh"
#include "host_common.h"
#include "../../include/ns2_b200.h"

#include <type_traits>

namespace ns2 {

constexpr int BM = 128;
constexpr int BK = 64;

struct GemmDev {
  CUtensorMap tmA;
  CUtensorMap tmB;
  CUtensorMap tmOut;   // TMA store / reduce-add target: (columns, group, position, batch), clipped at n and a_rows
  int tiles_n, tiles_per_batch, tiles_m, num_tiles;
  int a_rows, n, groups;
  int a_gcs, b_grs, out_gcs;
  int dil[NS2_GEMM_MAX_GROUPS];
  int num_segs;
  ns2_gemm_seg segs[NS2_GEMM_MAX_SEGS];
  const float* bias;
  int bias1_off;
  void* out;
  long long out_rs;
  const float* resid;
  long long resid_rs;
  int resid_in_place;  // F32 with resid == out (same row stride): out += acc + bias by TMA reduce-add, resid never read
  const float* film;
  long long film_bs;
  int film_gs;
  int act;            // BF16 / F32 epilogues: 0 = none, 1 = SiLU applied to acc + bias (ns2_gemm_args.flags & NS2_GEMM_FLAG_SILU)
  int skip_epilogue;  // measurement aid (ns2_gemm_args.flags & NS2_GEMM_FLAG_SKIP_EPILOGUE): mainloop-only timing
  // gemm_kernel<..., true> only: per-batch row counts (a_batches <= NS2_GEMM_ROW_LENS_MAX_BATCHES values, each clamped
  // to [1, a_rows]); the fields above keep their offsets, so the plain kernels read their parameters as before
  const int* row_lens;
  int batches;
};

struct TileCoord {
  int g, b, n0, n_tile;
};

__device__ __forceinline__ TileCoord decode_tile(const GemmDev& p, int tile) {
  // every m-tile of every batch: tile = (g, b, m, n_tile) in row-major order, n fastest
  TileCoord t;
  const int per_group = p.tiles_m * p.tiles_n;
  t.g = tile / per_group;
  const int r = tile - t.g * per_group;
  const int m_tile = r / p.tiles_n;
  t.n_tile = r - m_tile * p.tiles_n;
  t.b = m_tile / p.tiles_per_batch;
  t.n0 = (m_tile - t.b * p.tiles_per_batch) * BM;
  return t;
}

// Length-aware schedule: only the m-tiles that start before row_lens[b], numbered densely in the same (g, b, m, n_tile)
// order, so the static round robin hands out computed tiles only and stays balanced.  pre[b] (shared memory) is the
// number of such m-tiles in batches < b, pre[batches] their total per group.
__device__ __forceinline__ TileCoord decode_tile_lens(const GemmDev& p, const int* pre, int tile) {
  TileCoord t;
  const int per_group = pre[p.batches] * p.tiles_n;
  t.g = tile / per_group;
  const int r = tile - t.g * per_group;
  const int m_tile = r / p.tiles_n;
  t.n_tile = r - m_tile * p.tiles_n;
  int lo = 0, hi = p.batches;   // the batch b with pre[b] <= m_tile < pre[b + 1] (every batch has >= 1 m-tile)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (pre[mid] <= m_tile) lo = mid;
    else hi = mid;
  }
  t.b = lo;
  t.n0 = (m_tile - pre[lo]) * BM;
  return t;
}

// ------------------------------------------------------------------------------------------------
// epilogue: accumulator fragments -> finished values in registers -> 128-byte-swizzled shared-memory staging box
// (64 rows x 128 bytes per consumer warpgroup, double-buffered) -> TMA store, or a TMA reduce-add for the in-place
// residual update.  Thread (warp ww of the consumer warpgroup, lane l) holds rows 16 ww + l/4 + 8i of its warpgroup's
// 64 rows, columns 8j + 2(l%4) + k:  acc[4j + 2i + k].
// ------------------------------------------------------------------------------------------------
// The tile's column vectors, fp32 in shared memory (vec), column c of the tile at:
//   BF16 / F32  vec[c]                                    bias (not loaded without one)
//   GEGLU       vec[c] value bias, vec[c + 128] gate bias
//   WAVENET     vec[c] b0, vec[128 + c] b1 (bias1_off), vec[256 + c] FiLM gamma, vec[384 + c] FiLM beta
template <int BN, int EPI>
constexpr int tile_vec_floats() { return EPI == NS2_EPI_WAVENET ? 4 * BN : BN; }

// Issue the copies of the tile's vectors: one 16-byte cp.async per consumer thread (ct in [0, 256)) at most.  Columns
// at or past n are not read (n is a multiple of 32, so a 4-column piece is all in or all out).
template <int BN, int EPI>
__device__ __forceinline__ void load_tile_vectors(const GemmDev& p, const TileCoord& t, uint32_t vec, int ct) {
  constexpr int PIECES = BN / 4;   // 16-byte pieces per vector
  static_assert(tile_vec_floats<BN, EPI>() / 4 <= 256, "one piece per consumer thread");
  const int v = ct / PIECES;
  const int c = 4 * (ct - v * PIECES);
  const int col = t.n_tile * BN + c;
  if (ct >= tile_vec_floats<BN, EPI>() / 4 || col >= p.n) return;
  const float* src;
  if constexpr (EPI == NS2_EPI_WAVENET) {
    src = v < 2 ? p.bias + t.g * p.b_grs + col + (v == 1 ? p.bias1_off : 0)
                : p.film + t.b * p.film_bs + t.g * p.film_gs + col + (v == 3 ? p.n : 0);
  } else {
    if (p.bias == nullptr) return;
    src = p.bias + t.g * p.b_grs + col;
  }
  cp_async_16(vec + 4 * (v * BN + c), src);
}

__device__ __forceinline__ float silu_f(float v) { return __fdividef(v, 1.0f + __expf(-v)); }

// tanh(z) * sigmoid(z) with ONE MUFU: u = tanh(z/2); sigmoid = (1 + u)/2; tanh(z) = 2u / (1 + u^2), the reciprocal of
// w = 1 + u^2 in [1, 2] by a linear seed + two Newton steps on the FMA pipe (rel. err < 2e-5)
__device__ __forceinline__ float wavenet_gate(float z) {
  const float u = tanh_fast(0.5f * z);
  const float w = fmaf(u, u, 1.0f);
  float r = fmaf(-0.47058824f, w, 1.4117647f);     // 24/17 - 8/17 w: |1 - w r| <= 1/17 on [1, 2]
  r = r * fmaf(-w, r, 2.0f);
  r = r * fmaf(-w, r, 2.0f);
  return (u * r) * (1.0f + u);
}

constexpr int STG_BYTES = 64 * 128;   // one staging box: 64 rows x (64 bf16 | 32 fp32) columns

// Column groups jj, jj + 1 (jj even) of a bf16 box, o[2 jj + i] = bf16 pair k = 0, 1 of box row 16 ww + l/4 + 8i,
// columns 8 jj + 2(l%4) + k.  Row r of the box is 128 bytes whose 16-byte piece c sits at c ^ (r % 8) (the TMA
// 128-byte swizzle).  stmatrix writes one 8-row x 16-byte matrix per phase, and the 8 rows land on 8 different pieces:
// no bank conflicts.  Written pair by pair, as soon as computed, so that only 4 packed values are live at a time.
__device__ __forceinline__ void stage_bf16_pair(uint32_t buf, const uint32_t (&o)[16], int jj, int ww, int lane) {
  const int m = lane >> 3;                                  // matrix whose row address this lane supplies
  const uint32_t row_addr = buf + (16 * ww + 8 * (m & 1) + (lane & 7)) * 128;
  const int piece = jj + (m >> 1);
  stmatrix_x4(row_addr + ((piece ^ (lane & 7)) << 4), o[2 * jj], o[2 * jj + 1], o[2 * jj + 2], o[2 * jj + 3]);
}
// Same box layout with one 4-byte store per pair: a warp's 8 rows x 4 lanes land on piece jj ^ (row % 8), word l % 4,
// i.e. 32 different banks.  Used where stmatrix's four-register operands would cost the kernel its wgmma overlap.
__device__ __forceinline__ void stage_bf16_single(uint32_t buf, uint32_t v, int jj, int i, int ww, int lane) {
  const int r = lane >> 2;
  st_shared_b32(buf + (16 * ww + 8 * i + r) * 128 + ((jj ^ r) << 4) + 4 * (lane & 3), v);
}

// fp32, o[4 jj + 2i + k]: 8-byte stores, one half-warp per phase = box rows r = l/4 in 0..3 (or 4..7).  Column group jj is a 32-byte
// piece pair, swizzled to pair jj ^ (r / 2): rows 2s and 2s + 1 would share it.  Lanes on odd rows store group jj ^ 3
// while the others store jj, which puts the 4 rows of a phase on 4 different pairs: no bank conflicts.
__device__ __forceinline__ void stage_f32(uint32_t buf, const float (&o)[16], int ww, int lane) {
  const int r = lane >> 2;
  const bool odd = (r & 1) != 0;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const uint32_t row_addr = buf + (16 * ww + 8 * i + r) * 128 + 8 * (lane & 1);
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int jj = odd ? (s ^ 3) : s;
      const float a = odd ? o[4 * (s ^ 3) + 2 * i] : o[4 * s + 2 * i];
      const float b = odd ? o[4 * (s ^ 3) + 2 * i + 1] : o[4 * s + 2 * i + 1];
      st_shared_v2_f32(row_addr + (((2 * jj + ((lane & 3) >> 1)) ^ r) << 4), a, b);
    }
  }
}

// One tile of one consumer warpgroup.  vec: the tile's column vectors in shared memory; stg: its two staging boxes;
// nbox: boxes it has issued so far.  Only the warpgroup's first thread (`leader`) issues and waits on bulk groups; the
// box written now was last read by the store issued two boxes ago, which the leader waited for before the previous
// box's barrier.  (Waiting for that store only, just before the write, needs a second barrier per box and measured no
// faster on H100; see DESIGN.md section 5.)
template <int BN, int NACC, int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmDev& p, const TileCoord& t, const float (&acc)[NACC][BN / 2],
                                              const float* vec, int cw, int ww, int lane, bool leader, uint32_t stg,
                                              uint32_t& nbox) {
  constexpr int CW = EPI == NS2_EPI_F32 ? 32 : 64;                   // output columns per staging box
  constexpr int OUT_COLS = EPI == NS2_EPI_GEGLU ? 128 : BN;         // output columns of the tile
  // First position of this warpgroup's rows.  When it is past a_rows the stores below are clipped away entirely; the
  // warpgroup still runs the epilogue, because returning early (a divergent path around the accumulator reads) makes
  // ptxas serialize the WAVENET kernel's wgmma (C7520).
  const int row0 = t.n0 + cw * 64;
  const int out_col0 = t.n_tile * OUT_COLS;
  const int out_n = EPI == NS2_EPI_GEGLU ? p.n / 2 : p.n;
  const int c2 = 2 * (lane & 3);
  const int rr = row0 + 16 * ww + (lane >> 2);                      // position of this thread's i = 0 row
#pragma unroll
  for (int q = 0; q < OUT_COLS / CW; ++q) {
    if (out_col0 + q * CW >= out_n) break;   // n is a multiple of 32: a box holds at least 32 valid columns
    // finished values of this box: fp32 o[4 jj + 2i + k], or bf16 pairs o[2 jj + i] (packed at once: fewer live registers)
    using OutT = std::conditional_t<EPI == NS2_EPI_F32, float, uint32_t>;
    OutT o[16];
    const uint32_t buf = stg + (nbox & 1) * STG_BYTES;
    auto put = [&](int jj, int i, float v0, float v1) {
      if constexpr (EPI == NS2_EPI_F32) {
        o[4 * jj + 2 * i] = v0;
        o[4 * jj + 2 * i + 1] = v1;
      } else {
        o[2 * jj + i] = pack_bf16x2(v0, v1);
      }
    };
#pragma unroll
    for (int jj = 0; jj < CW / 8; ++jj) {
      const int j = q * (CW / 8) + jj;        // accumulator column group
      const int col = out_col0 + 8 * j + c2;  // output column of k = 0 (value column for GEGLU)
      const int c = 8 * j + c2;               // its column inside the tile
      if (out_col0 + 8 * j >= out_n) {        // right half of a 64-column box past n: clipped by the TMA store
        put(jj, 0, 0.f, 0.f);
        put(jj, 1, 0.f, 0.f);
        if constexpr (EPI == NS2_EPI_BF16 || EPI == NS2_EPI_GEGLU)
          if (jj & 1) stage_bf16_pair(buf, o, jj - 1, ww, lane);
        continue;
      }
      if constexpr (EPI == NS2_EPI_BF16 || EPI == NS2_EPI_F32) {
        float2 bb = make_float2(0.f, 0.f);
        if (p.bias != nullptr) bb = *reinterpret_cast<const float2*>(vec + c);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float v0 = acc[0][4 * j + 2 * i], v1 = acc[0][4 * j + 2 * i + 1];
          if (p.bias != nullptr) {
            v0 += bb.x;
            v1 += bb.y;
          }
          if (p.act != 0) {
            v0 = silu_f(v0);
            v1 = silu_f(v1);
          }
          if constexpr (EPI == NS2_EPI_F32) {
            // residual held elsewhere: read it here (the in-place residual is added by the TMA reduce-add instead)
            if (p.resid != nullptr && !p.resid_in_place && rr + 8 * i < p.a_rows) {
              const long long grow = static_cast<long long>(t.b) * p.a_rows + rr + 8 * i;
              const float2 r2 = *reinterpret_cast<const float2*>(p.resid + grow * p.resid_rs + t.g * p.out_gcs + col);
              v0 += r2.x;
              v1 += r2.y;
            }
          }
          put(jj, i, v0, v1);
        }
      } else if constexpr (EPI == NS2_EPI_GEGLU) {
        static_assert(EPI != NS2_EPI_GEGLU || BN == 256, "GEGLU tiles pair 128 value + 128 gate rows");
        // value column c, its gate column c + 128 (fragment j + 16)
        const float2 bv = *reinterpret_cast<const float2*>(vec + c);
        const float2 bg = *reinterpret_cast<const float2*>(vec + c + 128);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          put(jj, i, (acc[0][4 * j + 2 * i] + bv.x) * gelu_erf_fast(acc[0][4 * (j + 16) + 2 * i] + bg.x),
              (acc[0][4 * j + 2 * i + 1] + bv.y) * gelu_erf_fast(acc[0][4 * (j + 16) + 2 * i + 1] + bg.y));
        }
      } else {  // NS2_EPI_WAVENET: y = tanh(z) sigmoid(z) + res, z = (conv + b0) * gamma + beta   (ns2.py:619-636)
        static_assert(EPI != NS2_EPI_WAVENET || NACC == 2, "wavenet block needs conv + res accumulators");
        const float2 b0 = *reinterpret_cast<const float2*>(vec + c);
        const float2 b1 = *reinterpret_cast<const float2*>(vec + BN + c);
        const float2 ga = *reinterpret_cast<const float2*>(vec + 2 * BN + c);
        const float2 be = *reinterpret_cast<const float2*>(vec + 3 * BN + c);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float z0 = fmaf(acc[0][4 * j + 2 * i] + b0.x, ga.x, be.x);
          const float z1 = fmaf(acc[0][4 * j + 2 * i + 1] + b0.y, ga.y, be.y);
          stage_bf16_single(buf, pack_bf16x2(wavenet_gate(z0) + (acc[NACC - 1][4 * j + 2 * i] + b1.x),
                                             wavenet_gate(z1) + (acc[NACC - 1][4 * j + 2 * i + 1] + b1.y)),
                            jj, i, ww, lane);
        }
      }
      if constexpr (EPI == NS2_EPI_BF16 || EPI == NS2_EPI_GEGLU)
        if (jj & 1) stage_bf16_pair(buf, o, jj - 1, ww, lane);
    }
    if constexpr (EPI == NS2_EPI_F32) stage_f32(buf, o, ww, lane);
    fence_proxy_async_smem();                   // generic-proxy smem writes -> visible to the TMA unit
    if (leader) tma_store_wait_read<0>();        // the previous box has been read: free for the next one
    warpgroup_bar(cw);
    if (leader) {
      if (EPI == NS2_EPI_F32 && p.resid_in_place) tma_reduce_add_4d(&p.tmOut, buf, out_col0 + q * CW, t.g, row0, t.b);
      else tma_store_4d(&p.tmOut, buf, out_col0 + q * CW, t.g, row0, t.b);
      tma_store_commit();
    }
    ++nbox;
  }
}

// ------------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------------
template <int BN, int NACC>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (192 * 1024) / STAGE_BYTES;   // 4 stages of 48 KB (BN 256), 6 of 32 KB (BN 128)
  static constexpr int THREADS = 384;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int STG_OFF = RING_BYTES;                        // 2 consumer warpgroups x 2 staging boxes
  static constexpr int VEC_OFF = STG_OFF + 4 * STG_BYTES;           // the tile's column vectors (tile_vec_floats)
  static constexpr int BAR_OFF = VEC_OFF + (NACC == 2 ? 4 : 1) * BN * 4;
  static constexpr int SMEM_BYTES = BAR_OFF + 256 /*barriers*/;     // 226.25 KB (WAVENET) of 227
  static_assert(SMEM_BYTES <= 232448, "over the sm_90 per-block shared-memory limit");
  // length-aware kernels: the row counts (cp.async-staged) and their m-tile prefix sums after the barriers
  static constexpr int LENS_OFF = SMEM_BYTES;
  static constexpr int SMEM_BYTES_LENS = LENS_OFF + (2 * NS2_GEMM_ROW_LENS_MAX_BATCHES + 4) * 4;
  static_assert(SMEM_BYTES_LENS <= 232448, "NS2_GEMM_ROW_LENS_MAX_BATCHES does not fit in shared memory");
};

constexpr int CONSUMER_BAR = 1;   // named barrier over the 256 consumer threads (warpgroup_bar uses 8 and 9)

template <int BN>
__device__ __forceinline__ void wgmma_tile_k16(float (&d)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 256) wgmma_bf16_ss_n256<0, 0>(d, da, db, 1);
  else wgmma_bf16_ss_n128<0, 0>(d, da, db, 1);
}

// gemm_kernel<BN, NACC, EPI, true>: ns2_gemm with row_lens.  Before the roles split, the first a_batches threads copy
// row_lens into shared memory by cp.async (the kernels read no global memory through the register path, see
// tests/test_gemm_epilogue_loads_cpu.py) and thread 0 forms the m-tile prefix sums; every role then walks the same
// compacted tile list (decode_tile_lens).  A tile is computed and stored exactly as by the plain kernel.
template <int BN, int NACC, int EPI, bool LENS = false>
__global__ void __launch_bounds__(GemmCfg<BN, NACC>::THREADS, 1) gemm_kernel(const __grid_constant__ GemmDev p) {
  using Cfg = GemmCfg<BN, NACC>;
  static_assert(Cfg::VEC_OFF / 4 + tile_vec_floats<BN, EPI>() <= Cfg::BAR_OFF / 4, "vector area too small");
  extern __shared__ __align__(1024) uint8_t smem[];   // 128-byte swizzled TMA boxes need 1024-byte alignment
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
  uint64_t* full_bar = bars;                 // [STAGES]
  uint64_t* empty_bar = bars + Cfg::STAGES;  // [STAGES] one arrive per consumer warp

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // dynamic smem not 1024-byte aligned (no printf: see mbar_wait)
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    tma_prefetch_desc(&p.tmOut);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(smem_u32(&full_bar[i]), 1);
      mbar_init(smem_u32(&empty_bar[i]), 8);
    }
    fence_barrier_init();
  }
  int num_tiles = p.num_tiles;
  const int* pre = nullptr;
  if constexpr (LENS) {
    int* lens = reinterpret_cast<int*>(smem + Cfg::LENS_OFF);
    int* pre_w = lens + NS2_GEMM_ROW_LENS_MAX_BATCHES;
    if (threadIdx.x < p.batches) cp_async_4(smem_u32(lens + threadIdx.x), p.row_lens + threadIdx.x);
    cp_async_wait_all();
    __syncthreads();
    if (threadIdx.x == 0) {
      int acc = 0;
      for (int b = 0; b < p.batches; ++b) {
        pre_w[b] = acc;
        acc += (min(max(lens[b], 1), p.a_rows) + BM - 1) / BM;
      }
      pre_w[p.batches] = acc;
    }
    __syncthreads();
    pre = pre_w;
    num_tiles = pre[p.batches] * p.tiles_n * p.groups;
  } else {
    __syncthreads();
  }
#define NS2_DECODE_TILE(tile) (LENS ? decode_tile_lens(p, pre, tile) : decode_tile(p, tile))

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0) {
      // =============================== TMA producer (converged, one elected lane issues) ===============================
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileCoord t = NS2_DECODE_TILE(tile);
        const int dil = p.dil[t.g];
        for (int s = 0; s < p.num_segs; ++s) {
          const ns2_gemm_seg sg = p.segs[s];
          const int row0 = t.n0 - sg.shift_units * dil;
          const int a_c0 = t.g * p.a_gcs + sg.a_col_off;
          const int b_r0 = t.g * p.b_grs + t.n_tile * BN;
          const int kblocks = (sg.k_len + BK - 1) / BK;
          for (int kb = 0; kb < kblocks; ++kb, ++it) {
            const uint32_t stage = it % Cfg::STAGES;
            const uint32_t phase = (it / Cfg::STAGES) & 1;
            mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1);
            if (elect_one()) {
              const uint32_t fb = smem_u32(&full_bar[stage]);
              mbar_arrive_expect_tx(fb, Cfg::STAGE_BYTES);
              uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
              tma_load_3d(smem_u32(sa), &p.tmA, fb, a_c0 + kb * BK, row0, t.b);
              tma_load_2d(smem_u32(sa + Cfg::A_BYTES), &p.tmB, fb, sg.b_col_off + kb * BK, b_r0);
            }
            __syncwarp();
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // =============================== consumers: wgmma mainloop + epilogue ===============================
    const int cw = (warp >> 2) - 1;   // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
    const int ww = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;   // issues and waits on this warpgroup's bulk stores
    const uint32_t stg = smem_u32(smem + Cfg::STG_OFF + cw * 2 * STG_BYTES);
    const float* vec = reinterpret_cast<const float*>(smem + Cfg::VEC_OFF);
    // the epilogue reads column vectors (uniform over the grid): copy them in under each tile's mainloop
    const bool tile_vecs = !p.skip_epilogue && (EPI == NS2_EPI_GEGLU || EPI == NS2_EPI_WAVENET || p.bias != nullptr);
    uint32_t nbox = 0;
    float acc[NACC][BN / 2];
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileCoord t = NS2_DECODE_TILE(tile);
      if (tile_vecs) {
        named_bar(CONSUMER_BAR, 256);   // both warpgroups' epilogues of the previous tile are done reading vec
        load_tile_vectors<BN, EPI>(p, t, smem_u32(vec), threadIdx.x - 128);
      }
#pragma unroll
      for (int a = 0; a < NACC; ++a)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[a][i] = 0.f;
      int prev_stage = -1;
      for (int s = 0; s < p.num_segs; ++s) {
        const int sel = p.segs[s].acc;
        const int kblocks = (p.segs[s].k_len + BK - 1) / BK;
        for (int kb = 0; kb < kblocks; ++kb, ++it) {
          const uint32_t stage = it % Cfg::STAGES;
          const uint32_t phase = (it / Cfg::STAGES) & 1;
          mbar_wait(smem_u32(&full_bar[stage]), phase);
          const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
          const uint64_t da = gmma_desc_sw128(sa + cw * (64 * 128), 16, 1024);
          const uint64_t db = gmma_desc_sw128(sa + Cfg::A_BYTES, 16, 1024);
          wgmma_fence();
          if (NACC == 1 || sel == 0) {
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) wgmma_tile_k16<BN>(acc[0], da + 2 * k, db + 2 * k);
          } else {
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) wgmma_tile_k16<BN>(acc[NACC - 1], da + 2 * k, db + 2 * k);
          }
          wgmma_commit();
          // the previous k-block's MMAs have retired: its smem slot goes back to the producer
          wgmma_wait<1>();
          if (prev_stage >= 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev_stage]));
          prev_stage = static_cast<int>(stage);
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int a = 0; a < NACC; ++a) wgmma_hold(acc[a]);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev_stage]));
      if (tile_vecs) {
        cp_async_wait_all();             // this thread's copies have landed
        named_bar(CONSUMER_BAR, 256);   // and every other thread's
      }
      if (!p.skip_epilogue) epilogue_tile<BN, NACC, EPI>(p, t, acc, vec, cw, ww, lane, leader, stg, nbox);
    }
    if (leader) tma_store_wait_all();   // shared memory must outlive the reads of the last stores
  }
#undef NS2_DECODE_TILE
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <int BN, int NACC, int EPI>
static int launch_gemm(const GemmDev& dev, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, NACC>;
  // with row lengths the grid is sized for every tile: the CTAs past the compacted count exit at once
  const int grid = dev.num_tiles < num_sms() ? dev.num_tiles : num_sms();
  if (dev.row_lens != nullptr) {
    auto kern = gemm_kernel<BN, NACC, EPI, true>;
    NS2_CUDA_CHECK(set_max_smem_once(kern, Cfg::SMEM_BYTES_LENS));
    kern<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES_LENS, stream>>>(dev);
  } else {
    auto kern = gemm_kernel<BN, NACC, EPI>;
    NS2_CUDA_CHECK(set_max_smem_once(kern, Cfg::SMEM_BYTES));
    kern<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(dev);
  }
  return launched(1);
}

}  // namespace ns2

extern "C" int ns2_gemm(const ns2_gemm_args* a, ns2_stream_t stream_) {
  using namespace ns2;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NS2_REQUIRE(a != nullptr, "ns2_gemm: args is NULL");
  NS2_REQUIRE(a->row_lens == nullptr || (a->a_batches >= 1 && a->a_batches <= NS2_GEMM_ROW_LENS_MAX_BATCHES),
              "ns2_gemm: a_batches=%d, row lengths take 1 to %d batches", a->a_batches,
              NS2_GEMM_ROW_LENS_MAX_BATCHES);
  NS2_REQUIRE(a->A && a->B && a->out, "ns2_gemm: A, B and out must be non-NULL");
  NS2_REQUIRE(a->groups >= 1 && a->groups <= NS2_GEMM_MAX_GROUPS, "ns2_gemm: groups=%d out of range",
              a->groups);
  NS2_REQUIRE(a->num_segs >= 1 && a->num_segs <= NS2_GEMM_MAX_SEGS, "ns2_gemm: num_segs=%d",
              a->num_segs);
  NS2_REQUIRE(a->n > 0 && a->n % 32 == 0, "ns2_gemm: n=%d must be a positive multiple of 32", a->n);
  NS2_REQUIRE(a->a_rows > 0 && a->a_batches > 0, "ns2_gemm: empty A");
  NS2_REQUIRE(a->a_row_stride % 8 == 0 && a->a_batch_stride % 8 == 0 && a->b_row_stride % 8 == 0,
              "ns2_gemm: strides must be multiples of 8 elements (16 bytes)");
  for (int s = 0; s < a->num_segs; ++s) {
    const ns2_gemm_seg& sg = a->segs[s];
    // negative shift_units = rows AFTER the output position (anti-causal taps: the dgrad of a causal conv)
    NS2_REQUIRE(sg.k_len > 0 && sg.acc >= 0 && sg.acc <= 1, "ns2_gemm: bad segment %d", s);
    const bool ends_at_edge = (sg.b_col_off + sg.k_len == a->b_cols) &&
                              (sg.a_col_off + sg.k_len == a->a_cols) && a->groups == 1;
    NS2_REQUIRE(sg.k_len % BK == 0 || ends_at_edge,
                "ns2_gemm: segment %d k_len=%d is not a multiple of 64 and does not end at the edge", s,
                sg.k_len);
    NS2_REQUIRE(sg.acc == 0 || a->epilogue == NS2_EPI_WAVENET,
                "ns2_gemm: second accumulator only exists for the WAVENET epilogue");
  }
  if (a->epilogue == NS2_EPI_WAVENET)
    NS2_REQUIRE(a->film != nullptr && a->bias != nullptr && a->film_batch_stride % 4 == 0 &&
                    a->film_group_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(a->film) & 15) == 0,
                "ns2_gemm: WAVENET needs bias and a 16-byte aligned film table");
  if (a->epilogue == NS2_EPI_GEGLU)
    NS2_REQUIRE(a->bias != nullptr && a->n % 256 == 0,
                "ns2_gemm: GEGLU needs bias and n %% 256 == 0 (n=%d)", a->n);
  if (a->bias != nullptr)
    NS2_REQUIRE(a->b_group_row_stride % 4 == 0 && a->bias1_off % 4 == 0 &&
                    (reinterpret_cast<uintptr_t>(a->bias) & 15) == 0,
                "ns2_gemm: bias must be 16-byte aligned with group strides multiple of 4");
  NS2_REQUIRE(a->out_row_stride % 8 == 0 && a->out_group_col_stride % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
              "ns2_gemm: out must be 16-byte aligned with strides multiple of 8");
  if (a->resid != nullptr)
    NS2_REQUIRE(a->resid_row_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(a->resid) & 15) == 0,
                "ns2_gemm: resid must be 16-byte aligned");
  NS2_REQUIRE((a->flags & ~(NS2_GEMM_FLAG_SKIP_EPILOGUE | NS2_GEMM_FLAG_SILU)) == 0,
              "ns2_gemm: unknown flags 0x%x (only NS2_GEMM_FLAG_SKIP_EPILOGUE and NS2_GEMM_FLAG_SILU exist)", a->flags);

  // ---- tile selection ----
  int bn;
  if (a->epilogue == NS2_EPI_WAVENET) bn = 128;      // two 64-register accumulator fragments per thread
  else if (a->epilogue == NS2_EPI_GEGLU) bn = 256;   // 128 value + 128 gate columns
  else bn = a->n >= 256 ? 256 : 128;

  GemmDev dev;
  memset(&dev, 0, sizeof(dev));
  {
    const uint64_t dims[3] = {(uint64_t)a->a_cols, (uint64_t)a->a_rows, (uint64_t)a->a_batches};
    const uint64_t strides[3] = {2, (uint64_t)a->a_row_stride * 2, (uint64_t)a->a_batch_stride * 2};
    const uint32_t box[3] = {BK, BM, 1};
    int rc = make_tmap_16bit(&dev.tmA, a->A, 3, dims, strides, box);
    if (rc != kOk) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)a->b_cols, (uint64_t)a->b_rows};
    const uint64_t strides[2] = {2, (uint64_t)a->b_row_stride * 2};
    const uint32_t box[2] = {BK, (uint32_t)bn};
    int rc = make_tmap_16bit(&dev.tmB, a->B, 2, dims, strides, box);
    if (rc != kOk) return rc;
  }
  {
    // (columns, group, position, batch): columns clip at n (n / 2 for GEGLU) inside every group, positions at a_rows,
    // so a partial tile writes nothing into the next group's columns or the next batch's rows.  One box = one
    // consumer warpgroup's 64 positions x 128 bytes.
    const bool f32 = a->epilogue == NS2_EPI_F32;
    const uint64_t esz = f32 ? 4 : 2;
    const uint64_t out_cols = a->epilogue == NS2_EPI_GEGLU ? a->n / 2 : a->n;
    const uint64_t row_bytes = (uint64_t)a->out_row_stride * esz;
    const uint64_t dims[4] = {out_cols, (uint64_t)a->groups, (uint64_t)a->a_rows, (uint64_t)a->a_batches};
    const uint64_t strides[4] = {esz, a->groups > 1 ? (uint64_t)a->out_group_col_stride * esz : row_bytes, row_bytes,
                                 (uint64_t)a->a_rows * row_bytes};
    const uint32_t box[4] = {(uint32_t)(128 / esz), 1, 64, 1};
    int rc = f32 ? make_tmap_f32(&dev.tmOut, a->out, 4, dims, strides, box)
                 : make_tmap_16bit(&dev.tmOut, a->out, 4, dims, strides, box);
    if (rc != kOk) return rc;
  }
  dev.tiles_n = (a->n + bn - 1) / bn;
  dev.tiles_per_batch = (a->a_rows + BM - 1) / BM;
  dev.tiles_m = dev.tiles_per_batch * a->a_batches;
  dev.num_tiles = dev.tiles_m * dev.tiles_n * a->groups;
  dev.a_rows = a->a_rows;
  dev.n = a->n;
  dev.groups = a->groups;
  dev.a_gcs = a->a_group_col_stride;
  dev.b_grs = a->b_group_row_stride;
  dev.out_gcs = a->out_group_col_stride;
  for (int g = 0; g < NS2_GEMM_MAX_GROUPS; ++g) dev.dil[g] = a->dil[g];
  dev.num_segs = a->num_segs;
  for (int s = 0; s < a->num_segs; ++s) dev.segs[s] = a->segs[s];
  dev.bias = a->bias;
  dev.bias1_off = a->bias1_off;
  dev.out = a->out;
  dev.out_rs = a->out_row_stride;
  dev.resid = a->resid;
  dev.resid_rs = a->resid_row_stride;
  dev.resid_in_place = (a->epilogue == NS2_EPI_F32 && a->resid != nullptr && a->resid == a->out &&
                        a->resid_row_stride == a->out_row_stride) ? 1 : 0;
  dev.film = a->film;
  dev.film_bs = a->film_batch_stride;
  dev.film_gs = a->film_group_stride;
  dev.act = (a->flags & NS2_GEMM_FLAG_SILU) ? 1 : 0;
  NS2_REQUIRE(dev.act == 0 || a->epilogue == NS2_EPI_BF16 || a->epilogue == NS2_EPI_F32,
              "ns2_gemm: NS2_GEMM_FLAG_SILU only applies to the BF16 / F32 epilogues");
  dev.skip_epilogue = (a->flags & NS2_GEMM_FLAG_SKIP_EPILOGUE) ? 1 : 0;
  dev.row_lens = a->row_lens;
  dev.batches = a->a_batches;

  switch (a->epilogue) {
    case NS2_EPI_BF16:
      return bn == 256 ? launch_gemm<256, 1, NS2_EPI_BF16>(dev, stream)
                       : launch_gemm<128, 1, NS2_EPI_BF16>(dev, stream);
    case NS2_EPI_F32:
      return bn == 256 ? launch_gemm<256, 1, NS2_EPI_F32>(dev, stream)
                       : launch_gemm<128, 1, NS2_EPI_F32>(dev, stream);
    case NS2_EPI_GEGLU:
      return launch_gemm<256, 1, NS2_EPI_GEGLU>(dev, stream);
    case NS2_EPI_WAVENET:
      return launch_gemm<128, 2, NS2_EPI_WAVENET>(dev, stream);
    default:
      return set_error(kErrInvalidArg, "ns2_gemm: unknown epilogue %d", a->epilogue);
  }
}
