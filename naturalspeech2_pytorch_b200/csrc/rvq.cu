// Residual vector quantisation (Encodec RVQ encode / decode) for sm_90a.
//
// Reference behaviour (third-party code behind audiolm_pytorch.EncodecWrapper, reached from ns2.py:1445,1611;
// restated in oracle/rvq_oracle.py from encodec's EuclideanCodebook.quantize + ResidualVectorQuantization):
//   for q in 0..Q-1:  idx = argmin_k ||r - C_q[k]||^2 (first minimum wins);  r -= C_q[idx]
//
// The distance contraction runs on the tensor cores (wgmma) in fp16 (fp32 accumulate) as a *filter*:
//   s~_k = ||c_k||^2 - 2 r.c_k     with a rigorous bound |s~_k - s_k| <= E = 2 * 1.05 * 2^-10 * ||r|| * max_k ||c_k|| + ...
// The whole score comes out of the tensor core: besides the 128 latent dims the MMA contracts one extra K block that
// carries ||c_k||^2 (split into an fp16 hi/lo pair, prepared once per codebook) against a per-row power of two, so
// the accumulator holds D = s~ * 2^-(e+ex+1) and the scan is pure compare/select work (no FMA, no ||c||^2 table).
// Every code whose approximate score is within 2E of the approximate minimum is a candidate; candidates
// are re-scored exactly in fp64 from the fp32 operands, so the emitted index is the exact argmin
// (ties -> lowest index) — bit-exact against the fp64 oracle — while >99% of the flops stay on tensor cores.
//
// One CTA per 128 frames, 320 threads:
//   warps 0-7  scan threads = two warpgroups; warpgroup w computes D[64 frames x 128 codes] per chunk with 8 + 1
//              wgmma m64n128k16 into registers.  The prepared fp16 codebook stores the codes of every 128-code chunk
//              permuted (see rvq_perm) so that each thread's accumulator columns are one contiguous 32-code block for
//              each of its two frames; it scans them with a branch-free top-2 on packed (score|index) keys.  fp32
//              residuals live in padded shared memory for all Q stages; the same threads build the fp16 A tile,
//              re-score near-ties in fp64 (per lane, or warp-cooperatively for crowded 32-code blocks / bands) and
//              subtract the chosen fp32 codeword
//   warp 8     TMA producer: streams the fp16 codebooks (128 codes x 128 dims + the 4 KB norm block per chunk) through
//              a 3-deep ring
#include "ptx.cuh"
#include "host_common.h"
#include "../../include/ns2_b200.h"

namespace ns2 {

namespace rvq {
constexpr int D = 128;        // latent dimension
constexpr int BF = 128;       // frames per CTA
constexpr int BC = 128;       // codes per chunk
constexpr int A_BYTES = BF * D * 2;   // 32 KB: two 64-dim swizzle atoms
constexpr int B_BYTES = BC * D * 2;   // 32 KB per chunk
constexpr int RING = 3;
constexpr int RSTRIDE = D + 4;        // floats per residual row: +4 keeps per-thread float4 row reads conflict-free
constexpr int MAX_K = 2048;
constexpr int OFF_A = 0;
constexpr int OFF_B = OFF_A + A_BYTES;
constexpr int X_BYTES = 4096;         // norm block of one chunk / of the A tile: [16 row groups][2 K halves][8 rows][8 fp16]
                                      // = the canonical un-swizzled K-major GMMA layout (SBO 256 B, LBO 128 B)
constexpr int OFF_BX = OFF_B + RING * B_BYTES;       // norm blocks of the ring stages
constexpr int OFF_AX = OFF_BX + RING * X_BYTES;      // per-row power of two (K half 0, elements 0 and 1), rest zero
constexpr int OFF_R = OFF_AX + X_BYTES;              // fp32 residuals, row-major padded: 67.6 KB
constexpr int OFF_KEYS = OFF_R + BF * RSTRIDE * 4;   // top-8 keys of each column half: [half][row][8] floats (8 KB)
constexpr int OFF_ROWP = OFF_KEYS + 2 * BF * 8 * 4;  // per-row {scale, unused, error bound in D units, force-exact flag}
constexpr int OFF_CAND = OFF_ROWP + BF * 4 * 4;      // CTA-wide queue of the rows that need the exact re-score
constexpr int OFF_BAR = OFF_CAND + (4 + BF) * 4;     // queue of ambiguous rows: [count, pad x3, BF entries]
constexpr int OFF_META = OFF_BAR + 256;             // per-stage {max ||c||, 2^e} of the first 32 stages
constexpr int SMEM_BYTES = OFF_META + 256;
constexpr int SCAN_THREADS = 256;     // warps 0-7: quarter = warp & 3, column half = warp >> 2 (A tile / residual rows)
}  // namespace rvq

struct RvqDev {
  CUtensorMap tmB;            // fp16 codebooks viewed as (Q*K rows, 128 cols)
  const float* frames;        // (F, 128)
  const float* codebooks;     // (Q, K, 128) fp32
  const __half* cbx;          // (Q, K/128, 2048) fp16 norm blocks (behind the fp16 codebooks in the prepared buffer)
  const float* meta;          // (Q, 2): max ||c||, 2^e_q
  long long* codes;           // (F, Q)
  unsigned long long* stats;  // optional: [0] lookups, [1] near-ties re-scored, [2] full scans, [3] sub-chunk scans
  long long num_frames;
  int Q, K;
};

// Exact squared distance in fp64 between one residual row (shared memory, contiguous) and one fp32 codeword.
// Four independent accumulators (dims i mod 4) break the DFMA dependency chain; the summation order is fixed, so
// equal inputs always give bit-equal results (ties between duplicate codewords resolve by index).
__device__ __forceinline__ double exact_dist(const float* rrow, const float* __restrict__ c) {
  double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
  const float4* c4 = reinterpret_cast<const float4*>(c);
  const float4* r4 = reinterpret_cast<const float4*>(rrow);
#pragma unroll 8
  for (int i = 0; i < rvq::D / 4; ++i) {
    const float4 v = __ldg(c4 + i);
    const float4 r = r4[i];
    const double d0 = static_cast<double>(r.x) - static_cast<double>(v.x);
    const double d1 = static_cast<double>(r.y) - static_cast<double>(v.y);
    const double d2 = static_cast<double>(r.z) - static_cast<double>(v.z);
    const double d3 = static_cast<double>(r.w) - static_cast<double>(v.w);
    a0 = fma(d0, d0, a0);
    a1 = fma(d1, d1, a1);
    a2 = fma(d2, d2, a2);
    a3 = fma(d3, d3, a3);
  }
  return (a0 + a1) + (a2 + a3);
}

// Warp-cooperative variant: lane l owns dims [4l, 4l+4); one coalesced 512-byte load of the codeword (issued by the
// caller so that several are in flight), a fixed butterfly reduction (equal inputs give bit-equal results).
// Every lane returns the full distance.
__device__ __forceinline__ float4 coop_load(const float* __restrict__ c, int lane) {
  return __ldg(reinterpret_cast<const float4*>(c) + lane);
}
__device__ __forceinline__ double coop_reduce(const float4 r, const float4 v) {
  const double d0 = static_cast<double>(r.x) - static_cast<double>(v.x);
  const double d1 = static_cast<double>(r.y) - static_cast<double>(v.y);
  const double d2 = static_cast<double>(r.z) - static_cast<double>(v.z);
  const double d3 = static_cast<double>(r.w) - static_cast<double>(v.w);
  double a = fma(d0, d0, fma(d1, d1, fma(d2, d2, d3 * d3)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  return a;
}

// Half-warp variant: lane hl of a 16-lane half owns dims [8 hl, 8 hl + 8); fixed order, xor-butterfly inside the half
// (equal inputs give bit-equal results); every lane of the half returns the full distance.
__device__ __forceinline__ double half_reduce8(const float4 r0, const float4 r1, const float4 c0, const float4 c1) {
  const double d0 = static_cast<double>(r0.x) - static_cast<double>(c0.x);
  const double d1 = static_cast<double>(r0.y) - static_cast<double>(c0.y);
  const double d2 = static_cast<double>(r0.z) - static_cast<double>(c0.z);
  const double d3 = static_cast<double>(r0.w) - static_cast<double>(c0.w);
  const double d4 = static_cast<double>(r1.x) - static_cast<double>(c1.x);
  const double d5 = static_cast<double>(r1.y) - static_cast<double>(c1.y);
  const double d6 = static_cast<double>(r1.z) - static_cast<double>(c1.z);
  const double d7 = static_cast<double>(r1.w) - static_cast<double>(c1.w);
  double a = fma(d0, d0, fma(d1, d1, fma(d2, d2, d3 * d3)));
  const double b = fma(d4, d4, fma(d5, d5, fma(d6, d6, d7 * d7)));
  a += b;
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  return a;
}

__device__ __forceinline__ void scan_barrier() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// sorted insert of a key into the ascending 4-tuple (g0..g3): 7 min/max, no branches
__device__ __forceinline__ void insert4(float key, float& g0, float& g1, float& g2, float& g3) {
  float t = key, lo;
  lo = fminf(g0, t); t = fmaxf(g0, t); g0 = lo;
  lo = fminf(g1, t); t = fmaxf(g1, t); g1 = lo;
  lo = fminf(g2, t); t = fmaxf(g2, t); g2 = lo;
  g3 = fminf(g3, t);
}

// same for an ascending 8-tuple: 15 min/max
__device__ __forceinline__ void insert8(float key, float (&g)[8]) {
  float t = key;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const float lo = fminf(g[i], t);
    t = fmaxf(g[i], t);
    g[i] = lo;
  }
  g[7] = fminf(g[7], t);
}

// packed key of one score: low 5 mantissa bits replaced by the column index, as ONE LOP3 ((a & b) | c = LUT 0xEA)
__device__ __forceinline__ uint32_t key5(uint32_t score_bits, uint32_t idx) {
  uint32_t k;
  asm("lop3.b32 %0, %1, 0xFFFFFFE0, %2, 0xEA;" : "=r"(k) : "r"(score_bits), "r"(idx));
  return k;
}

// (distance, index) lexicographic minimum across the warp
__device__ __forceinline__ void warp_argmin(double& d, int& k) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, d, o);
    const int ok = __shfl_xor_sync(0xffffffffu, k, o);
    if (od < d || (od == d && ok < k)) { d = od; k = ok; }
  }
}

// Column n of a prepared 128-code chunk holds code rvq_perm(n) of the chunk: accumulator column 8j + 2c + k (fragment
// element 4j + k of the thread with lane % 4 == c) is code 32c + 2j + k, so thread c of a quad sees codes [32c, 32c+32).
__host__ __device__ __forceinline__ int rvq_perm(int n) { return ((n >> 1) & 3) * 32 + (n >> 3) * 2 + (n & 1); }
__host__ __device__ __forceinline__ int rvq_perm_inv(int m) { return ((m & 31) >> 1) * 8 + (m >> 5) * 2 + (m & 1); }

// Approximate scores are carried as "keys": the fp32 score with its low mantissa bits replaced by the code index,
// so that min/max on the keys sorts (score, index) pairs without branches or separate index registers.
// Low 11 bits = index (K <= 2048); the 2^-12 relative truncation is folded into the re-score margin.
__global__ void __launch_bounds__(320, 1) rvq_encode_kernel(const __grid_constant__ RvqDev p) {
  using namespace rvq;
  // declared 1024-byte aligned (checked below) and indexed directly so the compiler keeps every access in the
  // shared state space (LDS/STS instead of generic LD/ST)
  extern __shared__ __align__(1024) uint8_t smem[];
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();   // no printf: see mbar_wait in ptx.cuh
  float* R = reinterpret_cast<float*>(smem + OFF_R);
  float* keys_s = reinterpret_cast<float*>(smem + OFF_KEYS);
  float4* rowp_s = reinterpret_cast<float4*>(smem + OFF_ROWP);
  int* queue_s = reinterpret_cast<int*>(smem + OFF_CAND);   // [0] = count, [1 + i] = row | na << 8 | nb << 12 | force << 16
  float* meta_s = reinterpret_cast<float*>(smem + OFF_META);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* b_full = bars + 0;    // [RING]
  uint64_t* b_empty = bars + 3;   // [RING] one arrive per scan warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long f0 = static_cast<long long>(blockIdx.x) * BF;
  const int chunks = p.K / BC;

  if (warp == 8 && lane == 0) tma_prefetch_desc(&p.tmB);
  if (warp == 9 && lane == 0) {
    for (int i = 0; i < RING; ++i) {
      mbar_init(smem_u32(&b_full[i]), 1);
      mbar_init(smem_u32(&b_empty[i]), 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ================================ TMA producer ================================
    if (lane == 0) {
      uint32_t it = 0;
      for (int q = 0; q < p.Q; ++q) {
        for (int c = 0; c < chunks; ++c, ++it) {
          const uint32_t st = it % RING, ph = (it / RING) & 1;
          mbar_wait_backoff(smem_u32(&b_empty[st]), ph ^ 1, 200);
          const uint32_t fb = smem_u32(&b_full[st]);
          mbar_arrive_expect_tx(fb, B_BYTES + X_BYTES);
          const uint32_t dst = smem_u32(smem + OFF_B + st * B_BYTES);
          const int row0 = q * p.K + c * BC;
          tma_load_2d(dst, &p.tmB, fb, 0, row0);
          tma_load_2d(dst + BC * 128, &p.tmB, fb, 64, row0);
          bulk_load_1d(smem_u32(smem + OFF_BX + st * X_BYTES),
                       p.cbx + (static_cast<long long>(q) * chunks + c) * (X_BYTES / 2), X_BYTES, fb);
        }
      }
    }
  } else if (warp < 8) {
    // ================================ scan threads ================================
    const int quarter = warp & 3, half = warp >> 2;
    const int row = quarter * 32 + lane;       // frame owned (together with the thread of the other half)
    const int wgi = warp >> 2;                 // warpgroup: accumulator rows [64 wgi, 64 wgi + 64)
    const int frow = 64 * wgi + 16 * quarter + (lane >> 2);   // accumulator rows of this thread: frow, frow + 8
    const int qc = lane & 3;                                  // 32-code block of every chunk this thread scans

    float* rrow = R + row * RSTRIDE;
    // cooperative, coalesced load of the 128 frames: warp w fills rows [16w, 16w+16)
    {
#pragma unroll 4
      for (int r = warp * 16; r < warp * 16 + 16; ++r) {
        const long long fr = f0 + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (fr < p.num_frames) v = __ldg(reinterpret_cast<const float4*>(p.frames + fr * D) + lane);
        reinterpret_cast<float4*>(R + r * RSTRIDE)[lane] = v;
      }
      for (int i = threadIdx.x; i < X_BYTES / 16; i += SCAN_THREADS)
        reinterpret_cast<uint4*>(smem + OFF_AX)[i] = make_uint4(0u, 0u, 0u, 0u);
      if (threadIdx.x < 64 && threadIdx.x < 2 * p.Q) meta_s[threadIdx.x] = __ldg(p.meta + threadIdx.x);
    }
    unsigned long long n_ambig = 0, n_full = 0, n_sub = 0;
    uint32_t it = 0;
    for (int q = 0; q < p.Q; ++q) {
      scan_barrier();  // [B1] residuals of this stage are in place
      if (threadIdx.x == 0) queue_s[0] = 0;   // filled after [B2]; the previous stage's last read was before [B1]
      // row scale (exact power of two into fp16 range), |r|^2 and the filter margin; both threads of a row compute
      // them redundantly from the same data in the same order (bit-identical), so no exchange is needed
      float xs_row;
      {
        const float cmax = q < 32 ? meta_s[2 * q] : __ldg(p.meta + 2 * q);
        const float cscale = q < 32 ? meta_s[2 * q + 1] : __ldg(p.meta + 2 * q + 1);
        float amax = 0.f, ss = 0.f;
#pragma unroll 8
        for (int i = 0; i < D / 4; ++i) {
          const float4 v = reinterpret_cast<const float4*>(rrow)[i];
          amax = fmaxf(fmaxf(amax, fabsf(v.x)), fmaxf(fabsf(v.y), fmaxf(fabsf(v.z), fabsf(v.w))));
          ss = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, ss))));
        }
        int ex = 0;
        if (amax > 0.f) (void)frexpf(amax, &ex);          // amax = m * 2^ex, m in [0.5, 1)
        int es = 0;
        (void)frexpf(cscale, &es);                        // cscale = 2^(es-1) exactly
        const int e = es - 1;
        xs_row = ldexpf(1.0f, -ex);
        if (half == 0) {
          // accumulator D = -sum (r xs)(c / 2^e) + ax * (hi + lo) = s~ * kinv,  kinv = 2^-(e+ex+1),  ax = 2^(e-ex+6)
          // (hi + lo = ||c||^2 * 2^-(2e+7)).  ax must be a normal fp16; otherwise (residual 2^9 x smaller or 2^20 x
          // larger than the codebook scale) the row skips the filter and is scanned exactly.
          const int axe = e - ex + 6;
          const bool force = axe < -14 || axe > 15;
          const float ax = force ? 0.f : ldexpf(1.0f, axe);
          const float kinv = ldexpf(1.0f, -(e + ex + 1));
          // |D_k - s_k kinv| <= ED: fp16 operand rounding of the dot (2 * 1.05 * 2^-10 ||r|| max||c||), the hi/lo split
          // of ||c||^2 (2^-23 of its fp16-scaled range = 2^-16 * 4^e), and fp32 accumulation of 9 K blocks (2^-20 of
          // the largest partial sum, 128 + max||c||^2 kinv)
          const float ed = (2.0f * 0.001026f * sqrtf(ss) * 1.001f * cmax + 1.53e-5f * cscale * cscale) * kinv +
                           9.6e-7f * (128.0f + cmax * cmax * kinv);
          rowp_s[row] = make_float4(xs_row, 0.f, ed, force ? 1.f : 0.f);   // read by the classification after [B2]
          const uint32_t axx = static_cast<uint32_t>(__half_as_ushort(__float2half_rn(ax))) * 0x00010001u;
          *reinterpret_cast<uint32_t*>(smem + OFF_AX + (row >> 3) * 256 + (row & 7) * 16) = axx;   // K elements 0, 1
        }
      }
      // ---- fp16 A tile: this thread converts dims [64*half, 64*half + 64) of its row into atom `half` ----
      {
        const float xs = -xs_row;   // the tile holds -r * xs: the accumulator is then an ascending score
        uint8_t* arow = smem + OFF_A + half * (BF * 128) + row * 128;
        const float4* src = reinterpret_cast<const float4*>(rrow + half * 64);
#pragma unroll
        for (int ch = 0; ch < 8; ++ch) {  // 8 chunks of 8 halves
          const float4 v0 = src[2 * ch], v1 = src[2 * ch + 1];
          const __half2 h0 = __floats2half2_rn(v0.x * xs, v0.y * xs), h1 = __floats2half2_rn(v0.z * xs, v0.w * xs);
          const __half2 h2 = __floats2half2_rn(v1.x * xs, v1.y * xs), h3 = __floats2half2_rn(v1.z * xs, v1.w * xs);
          *reinterpret_cast<uint4*>(arow + ((ch ^ (row & 7)) << 4)) =
              make_uint4(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1),
                         *reinterpret_cast<const uint32_t*>(&h2), *reinterpret_cast<const uint32_t*>(&h3));
        }
      }
      fence_proxy_async_smem();
      scan_barrier();  // [B1'] the A tile (written by both warpgroups) is complete

      // ---- scan this thread's 32-code block of every 128-code chunk, for both of its frames: branch-free top-8 on
      // packed keys.  The accumulator already is the (scaled) score, so a key is one LOP3: (bits & ~31) | index. ----
      float ga[8], gb[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        ga[i] = INFINITY;
        gb[i] = INFINITY;
      }
      auto scan32 = [&](const uint32_t (&v)[32], int sub_id, float (&g)[8]) {
        // local top-2 of the 32 scores, index i in the low 5 bits.  A tracker (a0 <= a1) absorbs a PAIR of keys in
        // 5 min/max:  m = min(k0,k1), M = max(k0,k1);  a1' = min3(a1, max(a0, m), M);  a0' = min(a0, m).  Two trackers.
        float a0 = INFINITY, a1 = INFINITY, b0 = INFINITY, b1 = INFINITY;
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          const float k0 = __uint_as_float(key5(v[i], static_cast<uint32_t>(i)));
          const float k1 = __uint_as_float(key5(v[i + 1], static_cast<uint32_t>(i + 1)));
          const float k2 = __uint_as_float(key5(v[i + 2], static_cast<uint32_t>(i + 2)));
          const float k3 = __uint_as_float(key5(v[i + 3], static_cast<uint32_t>(i + 3)));
          const float m0 = fminf(k0, k1), M0 = fmaxf(k0, k1);
          const float m1 = fminf(k2, k3), M1 = fmaxf(k2, k3);
          a1 = fminf(fminf(a1, fmaxf(a0, m0)), M0);
          a0 = fminf(a0, m0);
          b1 = fminf(fminf(b1, fmaxf(b0, m1)), M1);
          b0 = fminf(b0, m1);
        }
        const float l0 = fminf(a0, b0);
        const float l1 = fminf(fmaxf(a0, b0), fminf(a1, b1));
        // widen the index field to 11 bits (block id above the 5 local bits) and merge into the top-8
        const uint32_t blk = static_cast<uint32_t>(sub_id) << 5;
        insert8(__uint_as_float((__float_as_uint(l0) & 0xFFFFF81Fu) | blk), g);
        insert8(__uint_as_float((__float_as_uint(l1) & 0xFFFFF81Fu) | blk), g);
      };
      {
        const uint32_t abase = smem_u32(smem + OFF_A) + wgi * (64 * 128);
        const uint64_t dax = gmma_desc_plain(smem_u32(smem + OFF_AX) + wgi * (8 * 256), 128, 256);
#pragma unroll 1
        for (int c = 0; c < chunks; ++c, ++it) {
          const uint32_t st = it % RING, ph = (it / RING) & 1;
          mbar_wait(smem_u32(&b_full[st]), ph);
          const uint32_t bbase = smem_u32(smem + OFF_B + st * B_BYTES);
          float d[BC / 2];
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < D / 16; ++k) {
            const uint32_t aoff = (k >> 2) * (BF * 128) + (k & 3) * 32;   // atom, 16-dim step inside it
            const uint32_t boff = (k >> 2) * (BC * 128) + (k & 3) * 32;
            wgmma_f16_ss_n128<0, 0>(d, gmma_desc_sw128(abase + aoff, 16, 1024), gmma_desc_sw128(bbase + boff, 16, 1024),
                                    k > 0 ? 1u : 0u);
          }
          // + 2^(e-ex+6) * (hi_k + lo_k) = ||c_k||^2 * 2^-(e+ex+1): the norm term of the score
          wgmma_f16_ss_n128<0, 0>(d, dax, gmma_desc_plain(smem_u32(smem + OFF_BX + st * X_BYTES), 128, 256), 1u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_hold(d);
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(&b_empty[st]));   // the ring slot may be refilled
          uint32_t va[32], vb[32];
#pragma unroll
          for (int l = 0; l < 32; ++l) {
            va[l] = __float_as_uint(d[4 * (l >> 1) + (l & 1)]);       // frame frow,     code 32 qc + l
            vb[l] = __float_as_uint(d[4 * (l >> 1) + 2 + (l & 1)]);   // frame frow + 8, code 32 qc + l
          }
          scan32(va, c * 4 + qc, ga);
          scan32(vb, c * 4 + qc, gb);
        }
      }
      // blocks 4c + {0, 1} form column half 0, 4c + {2, 3} half 1: merge the lists of the lane pair (lane ^ 1)
      {
        float oa[8], ob[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          oa[i] = __shfl_xor_sync(0xffffffffu, ga[i], 1);
          ob[i] = __shfl_xor_sync(0xffffffffu, gb[i], 1);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          insert8(oa[i], ga);
          insert8(ob[i], gb);
        }
        if ((qc & 1) == 0) {
          const int hsel = qc >> 1;
          float4* kd = reinterpret_cast<float4*>(keys_s + (hsel * BF + frow) * 8);
          kd[0] = make_float4(ga[0], ga[1], ga[2], ga[3]);
          kd[1] = make_float4(ga[4], ga[5], ga[6], ga[7]);
          float4* ke = reinterpret_cast<float4*>(keys_s + (hsel * BF + frow + 8) * 8);
          ke[0] = make_float4(gb[0], gb[1], gb[2], gb[3]);
          ke[1] = make_float4(gb[4], gb[5], gb[6], gb[7]);
        }
      }
      scan_barrier();  // [B2] both halves' key lists are published

      // ---- exact decision + residual update ----
      // Candidates = every code whose key is within the error band of the best key.  Each column half keeps its own
      // sorted top-8; a band member can only be missing from the two lists if a list is entirely inside the band
      // (-> exact scan of the whole codebook) or if it was 3rd+ inside its 32-code block, in which case two better
      // band members share that block (-> that block is scanned exactly).
      // Step 1: warp w classifies rows [16w, 16w+16) (lanes 0..15, one row each) and appends the ambiguous ones (~9 %)
      //         to a CTA-wide queue.
      // Step 2: it subtracts the exact fp32 codeword (same op as the reference) from its unambiguous rows, all 16
      //         coalesced 512-byte codeword loads in flight at once.
      // Step 3 (after [B3]): the 8 warps drain the queue round-robin - fp64 re-score, then the subtraction with the
      //         winner's codeword, which is still in registers - so the ambiguous rows cost ceil(n/8) rounds instead of
      //         the worst warp's own count (measured: the slowest warp used to hold the CTA ~6k cycles per stage).
      const float* cbq = p.codebooks + static_cast<long long>(q) * p.K * D;
      {
        const int myrow = warp * 16 + (lane & 15);
        float ka[8], kb[8];
        {
          const float4* k0 = reinterpret_cast<const float4*>(keys_s + myrow * 8);
          const float4* k1 = reinterpret_cast<const float4*>(keys_s + (BF + myrow) * 8);
          const float4 x0 = k0[0], x1 = k0[1], y0 = k1[0], y1 = k1[1];
          ka[0] = x0.x; ka[1] = x0.y; ka[2] = x0.z; ka[3] = x0.w; ka[4] = x1.x; ka[5] = x1.y; ka[6] = x1.z; ka[7] = x1.w;
          kb[0] = y0.x; kb[1] = y0.y; kb[2] = y0.z; kb[3] = y0.w; kb[4] = y1.x; kb[5] = y1.y; kb[6] = y1.z; kb[7] = y1.w;
        }
        const float kmin = fminf(ka[0], kb[0]);
        const float4 rpm = rowp_s[myrow];
        const float e16 = rpm.z;                                                    // filter error bound, key units
        const float etrunc = 0.000244140625f * 1.01f * (fabsf(kmin) + 2.0f * e16);  // 2^-12 key truncation
        const float lim = kmin + 2.0f * (e16 + etrunc);
        const bool force = rpm.w != 0.f;   // the filter was skipped for this row (scale out of fp16 range)
        int na = 0, nb = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          na += (ka[i] <= lim) ? 1 : 0;   // lists are sorted: the band is a prefix
          nb += (kb[i] <= lim) ? 1 : 0;
        }
        const int mysel = __float_as_uint(kmin) & 0x7FF;
        const bool amb = na + nb > 1 || force;
        const unsigned amb_mask = __ballot_sync(0xffffffffu, lane < 16 && amb);
        if (lane < 16 && amb) {
          const int slot = atomicAdd(queue_s, 1);
          queue_s[1 + slot] = myrow | (na << 8) | (nb << 12) | (force ? (1 << 16) : 0);
        }
        // step 2
        float4 cw[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) {
          const int sel = __shfl_sync(0xffffffffu, mysel, u);
          cw[u] = coop_load(cbq + static_cast<long long>(sel) * D, lane);
          const int r = warp * 16 + u;
          if (lane == 0 && !((amb_mask >> u) & 1u) && f0 + r < p.num_frames) p.codes[(f0 + r) * p.Q + q] = sel;
        }
#pragma unroll
        for (int u = 0; u < 16; ++u) {
          if ((amb_mask >> u) & 1u) continue;   // warp-uniform
          float4* dst = reinterpret_cast<float4*>(R + (warp * 16 + u) * RSTRIDE) + lane;
          float4 v = *dst;
          v.x -= cw[u].x; v.y -= cw[u].y; v.z -= cw[u].z; v.w -= cw[u].w;
          *dst = v;
        }
      }
      scan_barrier();  // [B3] the queue of ambiguous rows is complete
      // One row per HALF-warp (lane hl of a half owns dims [8 hl, 8 hl + 8)), so a warp resolves two queue rows per
      // round in one instruction stream; the rare rows (crowded block / full scan / filter skipped) are redone by the
      // whole warp with the general routine.
      auto resolve_row_fullwarp = [&](int ent) {
        const int r = ent & 0xFF, ca = (ent >> 8) & 0xF, cb = (ent >> 12) & 0xF;
        // lane l < 8 holds entry l of list a, lanes 8..15 entry l-8 of list b (code index in the low 11 key bits)
        int mycand = 0;
        if (lane < 16) mycand = __float_as_uint(keys_s[((lane >> 3) * BF + r) * 8 + (lane & 7)]) & 0x7FF;
        const bool member = (lane < ca) || (lane >= 8 && lane < 8 + cb);
        float4* rdst = reinterpret_cast<float4*>(R + r * RSTRIDE) + lane;
        const float4 rv = *rdst;
        double dbest = INFINITY;
        int best = 0x7fffffff;
        float4 cbest = make_float4(0.f, 0.f, 0.f, 0.f);   // this lane's 4 dims of the best codeword so far
        // crowded 32-code block: two band members with the same block id (a block never spans the column halves)
        const unsigned same = __match_any_sync(0xffffffffu, member ? (mycand >> 5) : (0x10000 + lane));
        const unsigned crowded = __ballot_sync(0xffffffffu, member && __popc(same) > 1);
        int blk = -1;
        bool full = (ca >= 8) || (cb >= 8) || ((ent >> 16) & 1);
        if (crowded) {
          blk = __shfl_sync(0xffffffffu, mycand >> 5, __ffs(crowded) - 1);
          // two different crowded blocks (astronomically rare): exact scan of the whole codebook
          full = full || __ballot_sync(0xffffffffu, ((crowded >> lane) & 1u) && (mycand >> 5) != blk) != 0u;
        }
        if (full) {
          ++n_full;
#pragma unroll 1
          for (int k0 = 0; k0 < p.K; k0 += 8) {
            float4 cv[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) cv[u] = coop_load(cbq + static_cast<long long>(k0 + u) * D, lane);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const double dk = coop_reduce(rv, cv[u]);
              if (dk < dbest) { dbest = dk; best = k0 + u; cbest = cv[u]; }
            }
          }
        } else {
          // band members of both lists, four codewords in flight at a time
          const int total = ca + cb;
#pragma unroll 1
          for (int u0 = 0; u0 < total; u0 += 4) {
            float4 cv[4];
            int kx[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int t = u0 + u;
              const int src = (t < total) ? (t < ca ? t : 8 + (t - ca)) : 0;
              kx[u] = __shfl_sync(0xffffffffu, mycand, src);
              cv[u] = coop_load(cbq + static_cast<long long>(kx[u]) * D, lane);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const double dk = coop_reduce(rv, cv[u]);
              if (u0 + u < total && (dk < dbest || (dk == dbest && kx[u] < best))) {
                dbest = dk; best = kx[u]; cbest = cv[u];
              }
            }
          }
          if (blk >= 0) {
            ++n_sub;
#pragma unroll 1
            for (int k0 = blk * 32; k0 < blk * 32 + 32; k0 += 16) {   // 16 codewords (8 KB) in flight: 2 L2 round trips
              float4 c8[16];
#pragma unroll
              for (int u = 0; u < 16; ++u) c8[u] = coop_load(cbq + static_cast<long long>(k0 + u) * D, lane);
#pragma unroll
              for (int u = 0; u < 16; ++u) {
                const double dk = coop_reduce(rv, c8[u]);
                if (dk < dbest || (dk == dbest && k0 + u < best)) { dbest = dk; best = k0 + u; cbest = c8[u]; }
              }
            }
          }
        }
        if (lane == 0 && f0 + r < p.num_frames) p.codes[(f0 + r) * p.Q + q] = best;
        *rdst = make_float4(rv.x - cbest.x, rv.y - cbest.y, rv.z - cbest.z, rv.w - cbest.w);
      };
      {
        const int total_rows = queue_s[0];
        const int h = lane >> 4, hl = lane & 15;
#pragma unroll 1
        for (int e0 = warp * 2; e0 < total_rows; e0 += 16) {
          const int e = e0 + h;
          const bool valid = e < total_rows;
          const int ent = valid ? queue_s[1 + e] : 0;
          const int r = ent & 0xFF, ca = (ent >> 8) & 0xF, cb = (ent >> 12) & 0xF;
          // half-lane hl < 8 holds entry hl of list a, 8..15 entry hl-8 of list b (code index in the low 11 key bits)
          const int mycand = valid ? (__float_as_uint(keys_s[((hl >> 3) * BF + r) * 8 + (hl & 7)]) & 0x7FF) : 0;
          const bool member = valid && ((hl < ca) || (hl >= 8 && hl < 8 + cb));
          float4* rdst = reinterpret_cast<float4*>(R + r * RSTRIDE) + 2 * hl;
          const float4 rv0 = rdst[0], rv1 = rdst[1];
          if (lane == 0) n_ambig += 1 + ((e0 + 1 < total_rows) ? 1 : 0);
          // crowded 32-code block: two band members of one row with the same block id
          const unsigned same = __match_any_sync(0xffffffffu, member ? ((h << 12) | (mycand >> 5)) : (0x10000 + lane));
          const unsigned crowded = __ballot_sync(0xffffffffu, member && __popc(same) > 1);
          const bool rare_me = valid && (ca >= 8 || cb >= 8 || ((ent >> 16) & 1) || ((crowded >> (16 * h)) & 0xFFFFu) != 0u);
          const unsigned rare = __ballot_sync(0xffffffffu, rare_me);
          const int total = (valid && !rare_me) ? ca + cb : 0;
          const int tmax = max(__shfl_sync(0xffffffffu, total, 0), __shfl_sync(0xffffffffu, total, 16));
          double dbest = INFINITY;
          int best = 0x7fffffff;
          float4 cb0 = make_float4(0.f, 0.f, 0.f, 0.f), cb1 = cb0;   // this lane's 8 dims of the best codeword so far
#pragma unroll 1
          for (int u0 = 0; u0 < tmax; u0 += 4) {
            float4 c0[4], c1[4];
            int kx[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int t = u0 + u;
              const int src = 16 * h + ((t < total) ? (t < ca ? t : 8 + (t - ca)) : 0);
              kx[u] = __shfl_sync(0xffffffffu, mycand, src);
              const float4* cp = reinterpret_cast<const float4*>(cbq + static_cast<long long>(kx[u]) * D) + 2 * hl;
              c0[u] = __ldg(cp);
              c1[u] = __ldg(cp + 1);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const double dk = half_reduce8(rv0, rv1, c0[u], c1[u]);
              if (u0 + u < total && (dk < dbest || (dk == dbest && kx[u] < best))) {
                dbest = dk; best = kx[u]; cb0 = c0[u]; cb1 = c1[u];
              }
            }
          }
          if (valid && !rare_me) {
            if (hl == 0 && f0 + r < p.num_frames) p.codes[(f0 + r) * p.Q + q] = best;
            rdst[0] = make_float4(rv0.x - cb0.x, rv0.y - cb0.y, rv0.z - cb0.z, rv0.w - cb0.w);
            rdst[1] = make_float4(rv1.x - cb1.x, rv1.y - cb1.y, rv1.z - cb1.z, rv1.w - cb1.w);
          }
          __syncwarp();
#pragma unroll 1
          for (int hh = 0; hh < 2; ++hh)
            if ((rare >> (16 * hh)) & 1u) resolve_row_fullwarp(__shfl_sync(0xffffffffu, ent, 16 * hh));
        }
      }
    }
    if (p.stats != nullptr) {
      if (half == 0 && f0 + row < p.num_frames) atomicAdd(p.stats + 0, static_cast<unsigned long long>(p.Q));
      if (lane == 0) {  // the cooperative decision counts per warp
        if (n_ambig) atomicAdd(p.stats + 1, n_ambig);
        if (n_full) atomicAdd(p.stats + 2, n_full);
        if (n_sub) atomicAdd(p.stats + 3, n_sub);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// prepare: fp16 copy (codes permuted inside each 128-code chunk, see rvq_perm) scaled by a per-quantiser power of two, ||c||^2, max ||c||, and the fp16 hi/lo norm blocks the
// encode kernel contracts as a ninth K block (layout: rvq::X_BYTES per 128-code chunk, see OFF_BX)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rvq_prepare_kernel(const float* __restrict__ cb, int K, int D,
                                                          __half* __restrict__ cb16,
                                                          __half* __restrict__ cbx,
                                                          float* __restrict__ cn2,
                                                          float* __restrict__ meta) {
  const int q = blockIdx.x;
  const float* c = cb + static_cast<long long>(q) * K * D;
  __shared__ float red[8];
  __shared__ float s_scale;
  float amax = 0.f;
  for (int i = threadIdx.x; i < K * D; i += blockDim.x) amax = fmaxf(amax, fabsf(c[i]));
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = 0.f;
    for (int i = 0; i < 8; ++i) m = fmaxf(m, red[i]);
    int e = 0;
    if (m > 0.f) (void)frexpf(m, &e);
    s_scale = ldexpf(1.0f, e);  // codes are stored as c * 2^-e, |.| < 1
    meta[2 * q + 1] = s_scale;
  }
  __syncthreads();
  const float inv = 1.0f / s_scale;
  for (int i = threadIdx.x; i < K * D; i += blockDim.x) {   // row n of the fp16 copy holds code rvq_perm(n) of its chunk
    const int n = i / D;
    const int src = ((n & ~127) | rvq_perm(n & 127)) * D + (i - n * D);
    cb16[static_cast<long long>(q) * K * D + i] = __float2half_rn(c[src] * inv);
  }
  // ||c||^2 in fp64, rounded once to fp32; one warp per code
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float nmax = 0.f;
  for (int k = warp; k < K; k += 8) {
    double s = 0.0;
    for (int i = lane; i < D; i += 32) {
      const double v = c[static_cast<long long>(k) * D + i];
      s += v * v;
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) cn2[q * K + k] = static_cast<float>(s);
    // norm block: val = ||c||^2 / scale^2 / 128 in [0, 1] as hi + lo (elements 0, 1 of K half 0), everything else zero
    {
      const float val = static_cast<float>(s) * inv * inv * 0.0078125f;
      const __half hi = __float2half_rn(val);
      const __half lo = __float2half_rn(val - __half2float(hi));
      const int n = rvq_perm_inv(k & 127);   // column of the chunk that holds code k
      __half* blk = cbx + (static_cast<long long>(q) * (K / 128) + k / 128) * 2048 + (n >> 3) * 128 + (n & 7) * 8;
      if (lane < 8) blk[lane] = lane == 0 ? hi : (lane == 1 ? lo : __float2half_rn(0.f));   // K half 0
      else if (lane < 16) blk[64 + lane - 8] = __float2half_rn(0.f);                        // K half 1
    }
    nmax = fmaxf(nmax, static_cast<float>(sqrt(s)) * 1.0001f);
  }
  __syncthreads();
  if (lane == 0) red[warp] = nmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = 0.f;
    for (int i = 0; i < 8; ++i) m = fmaxf(m, red[i]);
    meta[2 * q] = m;
  }
}

// decode: emb = sum_q C_q[codes[:, q]] accumulated in order q = 0..Q-1 (one warp per frame, float4 per lane)
__global__ void __launch_bounds__(256) rvq_decode_kernel(const long long* __restrict__ codes,
                                                         long long F, int Q, int K,
                                                         const float* __restrict__ cb,
                                                         float* __restrict__ emb) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long f = static_cast<long long>(blockIdx.x) * 8 + warp;
  if (f >= F) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int q = 0; q < Q; ++q) {
    long long idx = codes[f * Q + q];
    idx = idx < 0 ? 0 : (idx >= K ? K - 1 : idx);
    const float4 v =
        __ldg(reinterpret_cast<const float4*>(cb + (static_cast<long long>(q) * K + idx) * 128) + lane);
    acc.x += v.x;
    acc.y += v.y;
    acc.z += v.z;
    acc.w += v.w;
  }
  reinterpret_cast<float4*>(emb + f * 128)[lane] = acc;
}

}  // namespace ns2

using namespace ns2;

extern "C" {

int ns2_rvq_prepare(const float* codebooks, int32_t q, int32_t k, int32_t d, void* cb_f16,
                    float* cb_norm2, float* cb_meta, ns2_stream_t stream) {
  NS2_REQUIRE(codebooks && cb_f16 && cb_norm2 && cb_meta, "rvq_prepare: NULL pointer");
  NS2_REQUIRE(q > 0 && k > 0 && d == 128, "rvq_prepare: d must be 128 (got %d)", d);
  NS2_REQUIRE(k % 128 == 0, "rvq_prepare: codebook size %d must be a multiple of 128", k);
  __half* cb16 = reinterpret_cast<__half*>(cb_f16);
  rvq_prepare_kernel<<<q, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      codebooks, k, d, cb16, cb16 + static_cast<long long>(q) * k * d, cb_norm2, cb_meta);
  return launched(1);
}

int ns2_rvq_encode(const float* frames, int64_t num_frames, int32_t d, const float* codebooks,
                   const void* cb_f16, const float* cb_norm2, const float* cb_meta, int32_t q,
                   int32_t k, int64_t* codes, int64_t* stats, ns2_stream_t stream) {
  NS2_REQUIRE(frames && codebooks && cb_f16 && cb_norm2 && cb_meta && codes, "rvq_encode: NULL pointer");
  NS2_REQUIRE(d == 128, "rvq_encode: d must be 128 (got %d)", d);
  NS2_REQUIRE(k % rvq::BC == 0 && k <= rvq::MAX_K && k > 0,
              "rvq_encode: codebook size %d must be a multiple of 128, <= %d", k, rvq::MAX_K);
  NS2_REQUIRE(q > 0 && num_frames > 0, "rvq_encode: empty problem");
  NS2_REQUIRE((reinterpret_cast<uintptr_t>(frames) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(codebooks) & 15) == 0,
              "rvq_encode: frames and codebooks must be 16-byte aligned");
  RvqDev dev;
  memset(&dev, 0, sizeof(dev));
  const uint64_t dims[2] = {128, (uint64_t)q * k};
  const uint64_t str[2] = {2, 256};
  const uint32_t box[2] = {64, rvq::BC};
  int rc = make_tmap_16bit(&dev.tmB, cb_f16, 2, dims, str, box);
  if (rc != kOk) return rc;
  dev.frames = frames;
  dev.codebooks = codebooks;
  dev.cbx = reinterpret_cast<const __half*>(cb_f16) + static_cast<long long>(q) * k * d;
  dev.meta = cb_meta;
  dev.codes = reinterpret_cast<long long*>(codes);
  dev.stats = reinterpret_cast<unsigned long long*>(stats);
  dev.num_frames = num_frames;
  dev.Q = q;
  dev.K = k;
  const long long grid = (num_frames + rvq::BF - 1) / rvq::BF;
  NS2_REQUIRE(grid <= 0x7fffffffLL, "rvq_encode: too many frames");
  NS2_CUDA_CHECK(set_max_smem_once(rvq_encode_kernel, rvq::SMEM_BYTES));
  rvq_encode_kernel<<<static_cast<unsigned>(grid), 320, rvq::SMEM_BYTES, static_cast<cudaStream_t>(stream)>>>(dev);
  return launched(1);
}

int ns2_rvq_decode(const int64_t* codes, int64_t num_frames, int32_t q, int32_t k, int32_t d,
                   const float* codebooks, float* emb, ns2_stream_t stream) {
  NS2_REQUIRE(codes && codebooks && emb, "rvq_decode: NULL pointer");
  NS2_REQUIRE(d == 128 && q > 0 && k > 0 && num_frames > 0, "rvq_decode: d must be 128");
  const long long grid = (num_frames + 7) / 8;
  rvq_decode_kernel<<<static_cast<unsigned>(grid), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(codes), num_frames, q, k, codebooks, emb);
  return launched(1);
}

}  // extern "C"
