// Counter-based random numbers for dropout: Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2,
// 3", SC 2011) and the keep rule shared by every dropout site of the library.  tests/dropout_oracle.py restates all of
// it in numpy.
//
//   key      (seed & 0xffffffff, seed >> 32), one 64-bit seed per module forward call
//   keep     word >= t, t = min(floor(p 2^32 + 0.5), 2^32 - 1); kept values are scaled by float(1 / (1 - p))
//   counters attention element (b, h, q, k), q' = q & ~8, k' = k & ~8:
//              c0 = (k' >> 4) 8 + (k' & 7), c1 = (q' >> 4) 8 + (q' & 7), c2 = b heads + h, c3 = site;
//              the four words belong to (q', k'), (q', k' + 8), (q' + 8, k'), (q' + 8, k' + 8)
//            element-wise element i: c0 = (i >> 2) & 0xffffffff, c1 = i >> 34, c2 = 0xffffffff, c3 = site; word i & 3
//            (no attention stream has c2 = 0xffffffff: that would need 2^32 (batch, head) pairs)
// The attention layout gives each thread of the flash kernels whole 2 x 2 blocks: the forward's S fragments hold query
// rows {r, r + 8} x key columns {c, c + 8} (over neighbouring 8-column fragments), the backward's S^T fragments key rows
// {r, r + 8} x query columns {c, c + 8}; so the forward and the backward draw the same words for the same elements and
// no word is wasted.  The backward regenerates the forward's mask from (seed, site, b, h, q, k) instead of storing it.
//
// Everything here is __forceinline__ straight-line code: a function call inside a wgmma kernel makes ptxas serialise
// its wgmma (tests/test_ptxas_cpu.py).
#pragma once
#include <math.h>
#include <stdint.h>

namespace ns2 {

struct Philox4 {
  uint32_t x, y, z, w;
};

__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                 uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
    const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0;
    c1 = lo1;
    c2 = n2;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return {c0, c1, c2, c3};
}

// Counter word of attention row / column index x (bit 3 is the word's position inside the 2 x 2 block).
__host__ __device__ __forceinline__ uint32_t philox_attn_index(uint32_t x) { return ((x >> 4) << 3) | (x & 7u); }

// Parameters of one dropout site as the kernels take them.
struct DropoutDev {
  uint32_t key0, key1;   // Philox key = the seed's low / high half
  uint32_t site;
  uint32_t threshold;    // keep iff word >= threshold
  float scale;           // 1 / (1 - p), rounded to fp32
};

// Host side: validated kernel parameters of ns2_dropout {seed, site, p}.  Returns false when p is not in [0, 1).
inline bool make_dropout_dev(uint64_t seed, uint32_t site, float p, DropoutDev* d) {
  if (!(p >= 0.0f && p < 1.0f)) return false;   // also rejects NaN
  const double t = floor(static_cast<double>(p) * 4294967296.0 + 0.5);
  d->key0 = static_cast<uint32_t>(seed & 0xffffffffu);
  d->key1 = static_cast<uint32_t>(seed >> 32);
  d->site = site;
  d->threshold = t >= 4294967295.0 ? 0xffffffffu : static_cast<uint32_t>(t);
  d->scale = static_cast<float>(1.0 / (1.0 - static_cast<double>(p)));
  return true;
}

}  // namespace ns2
