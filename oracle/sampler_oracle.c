/*
 * sampler_oracle.c — plain C restatement of the seeded sampler of the seeded RANSAC and covariance calls
 * (include/covins_b200.h, "Seeded samples"; covins_b200/csrc/ransac_common.cuh, seeded_sample).  TEST INFRASTRUCTURE ONLY.
 *
 *   Philox4x64-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC'11): ten rounds of
 *   (c0, c1, c2, c3) <- (hi(M1 c2) ^ c1 ^ k0, lo(M1 c2), hi(M0 c0) ^ c3 ^ k1, lo(M0 c0)), the key bumped by the Weyl constants
 *   (W0, W1) between rounds.
 *   Sample s of key (seed, stream), k indices of [0, m): u_0, u_1, ... are the 32-bit halves, low first, of the four words of
 *   the blocks with counters (s, 0, 0, 0), (s, 1, 0, 0), ...; a partial Fisher-Yates shuffle of the identity permutation,
 *   j = i + (u_i (m - i)) >> 32, swap perm[i] and perm[j], sample[i] = perm[i].  The permutation is kept as the list of
 *   positions written so far (the latest entry of a position holds its value).
 * Integer arithmetic only.
 */
#include <stdint.h>

#define API __attribute__((visibility("default")))

static const uint64_t M0 = 0xD2E7470EE14C6C93ull, M1 = 0xCA5A826395121157ull;
static const uint64_t W0 = 0x9E3779B97F4A7C15ull, W1 = 0xBB67AE8584CAA73Bull;

/* out = Philox4x64-10(counter ctr, key key) */
API void ora_philox4x64_10(const uint64_t* ctr, const uint64_t* key, uint64_t* out) {
  uint64_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3], k0 = key[0], k1 = key[1];
  for (int r = 0; r < 10; r++) {
    if (r > 0) { k0 += W0; k1 += W1; }
    const unsigned __int128 p0 = (unsigned __int128)M0 * c0, p1 = (unsigned __int128)M1 * c2;
    const uint64_t n0 = (uint64_t)(p1 >> 64) ^ c1 ^ k0, n1 = (uint64_t)p1, n2 = (uint64_t)(p0 >> 64) ^ c3 ^ k1, n3 = (uint64_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

/* samples s0 .. s0 + n - 1 of key (seed, stream): out [n][k], k <= 64, k <= m */
API void ora_seeded_samples(uint64_t seed, uint64_t stream, uint32_t m, int k, int64_t s0, int n, int32_t* out) {
  const uint64_t key[2] = {seed, stream};
  for (int t = 0; t < n; t++) {
    uint32_t pos[64], val[64];
    uint64_t blk[4] = {0, 0, 0, 0};
    for (int i = 0; i < k; i++) {
      if (i % 8 == 0) {
        const uint64_t ctr[4] = {(uint64_t)(s0 + t), (uint64_t)(i / 8), 0, 0};
        ora_philox4x64_10(ctr, key, blk);
      }
      const uint64_t w = blk[(i % 8) / 2];
      const uint32_t u = (i % 2) ? (uint32_t)(w >> 32) : (uint32_t)w;
      const uint32_t j = (uint32_t)i + (uint32_t)(((uint64_t)u * (uint64_t)(m - (uint32_t)i)) >> 32);
      uint32_t vi = (uint32_t)i, vj = j;
      for (int e = 0; e < i; e++) {
        if (pos[e] == (uint32_t)i) vi = val[e];
        if (pos[e] == j) vj = val[e];
      }
      out[(int64_t)t * k + i] = (int32_t)vj;
      pos[i] = j; val[i] = vi;
    }
  }
}
