// tc_match.cu — descriptor k-NN on the Hopper tensor cores (wgmma.mma_async, integer kinds, accumulators in registers).
//
// Same contract as scan_kernel in match_kernels.cu (K1 Hamming / K2 L2 / K3 DenseMatcher lists), different bound.
// The POPC formulation is bound by the integer pipe.  Here the pairwise term is a u8 x u8 -> s32 GEMM:
//     Hamming(a,b) = popc(a) + popc(b) - 2 <bits(a), bits(b)>      (bits expanded to 0/1 bytes in shared memory)
//     |a-b|^2      = |a|^2 + |b|^2 - 2 <a, b>                      (u8 SIFT, exact in s32)
// issued as wgmma.mma_async.m64n128k32.s32.u8.u8 by a warpgroup (64 queries x 128 train rows, K = 32 bytes per
// instruction) with both operands in shared memory.  A thread of the warpgroup holds two query rows x 32 columns of the
// accumulator (rows 16 w + lane / 4 and + 8, columns 8 i + 2 (lane % 4) + {0, 1}); it sees its columns in ascending order,
// keeps per-row k-lists with the sequential OpenCV / DenseMatcher rule, and the four threads of a quad merge their lists
// by (key, index) at the end of a segment — so the result is bit-identical to the scalar kernel.
//
// Warp-specialised, persistent CTA (one per SM), 4-stage ring:
//   warps 0-7   consumers  (two warpgroups, query rows [0, 64) and [64, 128)): wait full[s] → K/32 x wgmma → wait →
//                          empty[s] → epilogue d = pt[j] - 2 acc (+ pq) → k-lists
//   warps 8-15  producers  wait empty[s] → read packed rows from HBM (coalesced 16-B loads) → expand / copy into the
//                          canonical K-major no-swizzle layout → fence.proxy.async → full[s]
// A CTA owns one block of 128 queries (expanded once into shared memory) and streams a contiguous range of candidate
// segments.
#include <float.h>
#include <limits.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "cvb_internal.cuh"
#include "tc_match.cuh"

namespace cvb_tc {

constexpr int TM = 128;       // queries per CTA (two warpgroups of 64)
constexpr int TN = 128;       // train rows per tile (wgmma N)
constexpr int STAGES = 4;        // shared-memory ring of expanded train tiles
constexpr int NORM_RING = 8;
constexpr int kInf = 0x3FFFFFFF;   // list sentinel; rows that must never enter carry this as their norm term

// ---- mbarrier / wgmma wrappers ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(cvb_smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

#define CVB_D8(b) "+r"(d[b]), "+r"(d[b + 1]), "+r"(d[b + 2]), "+r"(d[b + 3]), "+r"(d[b + 4]), "+r"(d[b + 5]), "+r"(d[b + 6]), "+r"(d[b + 7])
#define CVB_D64 CVB_D8(0), CVB_D8(8), CVB_D8(16), CVB_D8(24), CVB_D8(32), CVB_D8(40), CVB_D8(48), CVB_D8(56)
#define CVB_R64                                                                                                         \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
  "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"
// D[64 x 128] (+)= A[64 x 32] B[128 x 32]^T, both operands K-major in shared memory; B_SIGNED selects B = s8 (else u8)
template <bool B_SIGNED>
__device__ __forceinline__ void wg_mma_i8(uint32_t (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  if constexpr (B_SIGNED) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.s8 " CVB_R64 ", %64, %65, p;\n}\n"
        : CVB_D64 : "l"(adesc), "l"(bdesc), "r"(acc));
  } else {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 " CVB_R64 ", %64, %65, p;\n}\n"
        : CVB_D64 : "l"(adesc), "l"(bdesc), "r"(acc));
  }
}
// the accumulator registers are written asynchronously: keep the compiler from moving their uses across the fence / wait
__device__ __forceinline__ void wg_fence_operands(uint32_t (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; i++) asm volatile("" : "+r"(d[i])::"memory");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit_wait() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// NSLICE instructions of K = 32 over operands whose K chunks of 16 B lie 128 B apart (+256 B = +16 in the address field
// per instruction); the accumulator is overwritten by the first
template <bool B_SIGNED, int NSLICE>
__device__ __forceinline__ void wg_gemm(uint32_t (&d)[64], uint64_t adesc0, uint64_t bdesc0) {
  wg_fence_operands(d);
  wg_fence();
#pragma unroll
  for (int k = 0; k < NSLICE; k++) wg_mma_i8<B_SIGNED>(d, adesc0 + (uint64_t)(k * 16), bdesc0 + (uint64_t)(k * 16), k > 0 ? 1u : 0u);
  wg_commit_wait();
  wg_fence_operands(d);
}

// shared-memory matrix descriptor: K-major, no swizzle (core matrices of 8 rows x 16 B; LBO = stride between the two
// core matrices of one K = 32 instruction, SBO = stride between 8-row groups); layout type 0 (interleave)
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

__device__ __forceinline__ uint4 ldg_nc(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

template <int S>
__device__ __forceinline__ uint32_t shl(uint32_t w) {
  if constexpr (S >= 0) return w << S; else return w >> (-S);
}

// ---- metrics: how a packed row becomes a K-major operand row, and its additive norm term ----------------------
// A row is handled by TWO threads (half = 0/1), each loading kLoads 16-byte pieces of the packed row (so that the loads
// of several tiles can be kept in flight in registers) and writing its share of the operand chunks.
struct TcHamming {
  static constexpr int kRowBytes = 32;    // packed bytes in HBM
  static constexpr int kKBytes = 256;     // operand bytes (one byte per bit)
  static constexpr int kLoads = 1;        // uint4 per half row
  static constexpr int kPrefetch = 3;     // tiles in flight per producer thread
  static constexpr bool kIsL2 = false;
  static __device__ __forceinline__ void load_half(const uint8_t* __restrict__ row, int half, uint4 (&v)[kLoads]) {
    v[0] = ldg_nc(row + 16 * half);
  }
  // writes operand chunks 8 half .. 8 half + 7 of the row and returns the partial popcount.  A set bit becomes the byte
  // 1 << BIT: 0x40 (u8 64) in the train operand of tc_scan_kernel, 0x80 (s8 -128) in the resident tiles.
  template <int BIT = 6>
  static __device__ __forceinline__ int store_half(const uint4 (&v)[kLoads], int half, uint8_t* dst_row0) {
    const uint32_t w[4] = {v[0].x, v[0].y, v[0].z, v[0].w};
    constexpr uint32_t M = 0x01010101u << BIT;
    int pc = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      pc += __popc(w[i]);
      // byte j of output word k is 1 << BIT if bit (k + 8 j) of w[i] is set, else 0 (the same permutation on both operands)
      uint4 lo, hi;
      lo.x = shl<BIT>(w[i]) & M; lo.y = shl<BIT - 1>(w[i]) & M; lo.z = shl<BIT - 2>(w[i]) & M; lo.w = shl<BIT - 3>(w[i]) & M;
      hi.x = shl<BIT - 4>(w[i]) & M; hi.y = shl<BIT - 5>(w[i]) & M; hi.z = shl<BIT - 6>(w[i]) & M; hi.w = shl<BIT - 7>(w[i]) & M;
      *reinterpret_cast<uint4*>(dst_row0 + (8 * half + 2 * i) * 128) = lo;
      *reinterpret_cast<uint4*>(dst_row0 + (8 * half + 2 * i + 1) * 128) = hi;
    }
    return pc;
  }
  // query side (one thread per row): the same K permutation with 0/1 bytes, so that accumulator = 64 popc(a & b) =
  // (2 popc(a & b)) << 5, which is what the packed 16-bit keys of the epilogue subtract.  Packed word i of the row becomes
  // operand bytes [32 i, 32 i + 32) = one K = 32 instruction.
  static constexpr int kQWords = 8;
  static __device__ __forceinline__ int load_q(const uint8_t* __restrict__ row, uint32_t (&w)[8]) {
    const uint4 a = ldg_nc(row), b = ldg_nc(row + 16);
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
    int pc = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) pc += __popc(w[i]);
    return pc;
  }
  static __device__ __forceinline__ void expand_q(const uint32_t (&w)[8], int i, uint32_t (&r)[8]) {
#pragma unroll
    for (int b = 0; b < 8; b++) r[b] = (w[i] >> b) & 0x01010101u;
  }
};
struct TcL2 {
  static constexpr int kRowBytes = 128;
  static constexpr int kKBytes = 128;
  static constexpr int kLoads = 4;
  static constexpr int kPrefetch = 2;
  static constexpr bool kIsL2 = true;
  static __device__ __forceinline__ void load_half(const uint8_t* __restrict__ row, int half, uint4 (&v)[kLoads]) {
#pragma unroll
    for (int c = 0; c < 4; c++) v[c] = ldg_nc(row + 64 * half + 16 * c);
  }
  static __device__ __forceinline__ int store_half(const uint4 (&v)[kLoads], int half, uint8_t* dst_row0) {
    unsigned n2 = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
      n2 = __dp4a(v[c].x, v[c].x, n2); n2 = __dp4a(v[c].y, v[c].y, n2); n2 = __dp4a(v[c].z, v[c].z, n2); n2 = __dp4a(v[c].w, v[c].w, n2);
      *reinterpret_cast<uint4*>(dst_row0 + (4 * half + c) * 128) = v[c];
    }
    return (int)n2;
  }
  static constexpr int kQWords = 4;   // 128 operand bytes per row = 4 groups of 32
  static __device__ __forceinline__ int load_q(const uint8_t* __restrict__ row, uint32_t (&w)[32]) {
    unsigned n2 = 0;
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const uint4 v = ldg_nc(row + 16 * c);
      w[4 * c] = v.x; w[4 * c + 1] = v.y; w[4 * c + 2] = v.z; w[4 * c + 3] = v.w;
      n2 = __dp4a(v.x, v.x, n2); n2 = __dp4a(v.y, v.y, n2); n2 = __dp4a(v.z, v.z, n2); n2 = __dp4a(v.w, v.w, n2);
    }
    return (int)n2;
  }
  static __device__ __forceinline__ void expand_q(const uint32_t (&w)[32], int i, uint32_t (&r)[8]) {
#pragma unroll
    for (int b = 0; b < 8; b++) r[b] = w[8 * i + b];
  }
};

// k-list of (key, idx) kept sorted ascending by (key, idx); OpenCV rule for a stream with ascending idx:
// enter iff key < worst key; placed after all entries with key <= new key.
template <int K>
__device__ __forceinline__ void insert_key(int (&wk)[K], int (&wi)[K], int key, int idx) {
  if (!(key < wk[K - 1])) return;
  bool placed = false;
#pragma unroll
  for (int p = K - 1; p >= 1; --p) {
    if (!placed) {
      if (key < wk[p - 1]) { wk[p] = wk[p - 1]; wi[p] = wi[p - 1]; }
      else { wk[p] = key; wi[p] = idx; placed = true; }
    }
  }
  if (!placed) { wk[0] = key; wi[0] = idx; }
}
// merge rule for partial lists of disjoint row subsets: k smallest by (key, idx)
template <int K>
__device__ __forceinline__ void insert_lex(int (&wk)[K], int (&wi)[K], int key, int idx) {
  auto lt = [](int k1, int i1, int k2, int i2) { return k1 < k2 || (k1 == k2 && (unsigned)i1 < (unsigned)i2); };
  if (!lt(key, idx, wk[K - 1], wi[K - 1])) return;
  bool placed = false;
#pragma unroll
  for (int p = K - 1; p >= 1; --p) {
    if (!placed) {
      if (lt(key, idx, wk[p - 1], wi[p - 1])) { wk[p] = wk[p - 1]; wi[p] = wi[p - 1]; }
      else { wk[p] = key; wi[p] = idx; placed = true; }
    }
  }
  if (!placed) { wk[0] = key; wi[0] = idx; }
}
// sorted-list insertion of a packed int key (min/max network)
template <int K>
__device__ __forceinline__ void insert_packed(int (&wk)[K], int x) {
#pragma unroll
  for (int c = 0; c < K; c++) {
    const int lo = min(wk[c], x);
    x = max(wk[c], x);
    wk[c] = lo;
  }
}
template <int K>
__device__ __forceinline__ void insert_packed16(unsigned (&pk)[K], unsigned x) {
#pragma unroll
  for (int c = 0; c < K; c++) {
    const unsigned lo = __vminu2(pk[c], x);
    x = __vmaxu2(pk[c], x);
    pk[c] = lo;
  }
}
// the four threads of a quad hold the lists of the same two rows over disjoint columns: after this all four hold the merge
template <int K>
__device__ __forceinline__ void quad_merge_packed(int (&wk)[K]) {
#pragma unroll
  for (int m = 1; m <= 2; m <<= 1) {
    int o[K];
#pragma unroll
    for (int c = 0; c < K; c++) o[c] = __shfl_xor_sync(0xffffffffu, wk[c], m);
#pragma unroll
    for (int c = 0; c < K; c++) insert_packed<K>(wk, o[c]);
  }
}
template <int K>
__device__ __forceinline__ void quad_merge_lex(int (&wk)[K], int (&wi)[K]) {
#pragma unroll
  for (int m = 1; m <= 2; m <<= 1) {
    int ok[K], oi[K];
#pragma unroll
    for (int c = 0; c < K; c++) { ok[c] = __shfl_xor_sync(0xffffffffu, wk[c], m); oi[c] = __shfl_xor_sync(0xffffffffu, wi[c], m); }
#pragma unroll
    for (int c = 0; c < K; c++)
      if (oi[c] >= 0) insert_lex<K>(wk, wi, ok[c], oi[c]);
  }
}

// keys: Hamming → the distance; L2 → the bit pattern of sqrtf(d2) (non-negative floats order like their bits), which
// is what OpenCV compares.  kInfKey is larger than any real key of either kind.
constexpr int kInfKey = 0x7F000000;

// one query's final list → outputs (filter: best match if it passes the threshold and the ratio test; else the k-list).
// `writer` threads own one query row each; every lane of the warp must call this (ballot).
template <int K, bool IS_L2>
__device__ __forceinline__ void write_list(const TcParams& p, int seg, int q, bool writer, const int (&wk)[K], const int (&wi)[K],
                                           const float (&fd)[K], int lane) {
  const bool valid = writer && q < p.nq;
  if (p.filter) {
    bool ok = false;
    if (K >= 2 && valid) {
      const float dm = fd[0], dn = fd[K >= 2 ? 1 : 0];
      ok = wi[0] >= 0 && wi[K >= 2 ? 1 : 0] >= 0 && dm <= p.thr && dm < __fmul_rn(p.ratio, dn);
      const size_t o = (size_t)seg * p.nq + q;
      p.match_train[o] = ok ? wi[0] : -1;
      p.match_dist[o] = ok ? dm : FLT_MAX;
    }
    const unsigned b = __ballot_sync(0xffffffffu, ok);
    if (lane == 0 && b) atomicAdd(&p.n_matches[seg], __popc(b));
  } else if (valid) {
    const size_t o = ((size_t)seg * p.nq + q) * K;
#pragma unroll
    for (int c = 0; c < K; c++) {
      p.out_idx[o + c] = wi[c];
      if (IS_L2) reinterpret_cast<float*>(p.out_dist)[o + c] = wi[c] >= 0 ? fd[c] : FLT_MAX;
      else reinterpret_cast<int32_t*>(p.out_dist)[o + c] = wi[c] >= 0 ? wk[c] : INT_MAX;
    }
  }
}

constexpr int CONS_THREADS = 2 * 128;           // two consumer warpgroups
constexpr int PROD_WARP0 = CONS_THREADS / 32;   // producer warps 8..15 (two threads per train row)
constexpr int PROD_THREADS = 256;
constexpr int NUM_THREADS = CONS_THREADS + PROD_THREADS;

template <class M>
constexpr size_t smem_bytes() {
  return (size_t)(STAGES + 1) * TN * M::kKBytes + (size_t)NORM_RING * TN * sizeof(int) + 64 * sizeof(uint64_t);
}

// operand row r of a tile with KB operand bytes per row: byte offset of its chunk 0
template <int KB>
__device__ __forceinline__ uint32_t row_offset(int r) {
  return (uint32_t)(r >> 3) * (KB * 8) + (uint32_t)(r & 7) * 16;
}

template <class M, int K>
__global__ void __launch_bounds__(NUM_THREADS, 1) tc_scan_kernel(const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int KB = M::kKBytes;
  uint8_t* sA = smem;                                        // the query block [TM][KB]
  uint8_t* sB = sA + (size_t)TM * KB;                        // [STAGES][TN][KB]
  int* sNorm = reinterpret_cast<int*>(sB + (size_t)STAGES * TN * KB);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sNorm + NORM_RING * TN);
  uint64_t* full = bars;                 // [STAGES] producers → consumers (one arrival per producer warp)
  uint64_t* empty = bars + STAGES;       // [STAGES] consumers' MMAs done → producers (one arrival per consumer warp)
  __shared__ int sQNorm[TM];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qb = blockIdx.x % p.nqb, part = blockIdx.x / p.nqb;
  const int seg0 = (int)((long)part * p.n_seg / p.parts), seg1 = (int)((long)(part + 1) * p.n_seg / p.parts);

  // ---- one-time setup: barriers, the query operand ----
  if (tid == 0) {
    for (int s = 0; s < STAGES; s++) {
      cvb_mbar_init(&full[s], PROD_THREADS / 32);
      cvb_mbar_init(&empty[s], CONS_THREADS / 32);
    }
    cvb_fence_mbar_init();
  }
  if (tid < TM) {
    const int q = qb * TM + tid;
    uint32_t w[M::kIsL2 ? 32 : 8];
    int nrm = 0;
    if (q < p.nq) {
      nrm = M::load_q(p.q + (size_t)q * M::kRowBytes, w);
    } else {
#pragma unroll
      for (int i = 0; i < (M::kIsL2 ? 32 : 8); i++) w[i] = 0;
    }
    sQNorm[tid] = nrm;
    uint8_t* dst = sA + row_offset<KB>(tid);
#pragma unroll
    for (int i = 0; i < KB / 32; i++) {
      uint32_t r[8];
      M::expand_q(w, i, r);
      *reinterpret_cast<uint4*>(dst + (2 * i) * 128) = make_uint4(r[0], r[1], r[2], r[3]);
      *reinterpret_cast<uint4*>(dst + (2 * i + 1) * 128) = make_uint4(r[4], r[5], r[6], r[7]);
    }
    fence_proxy_async();
  }
  __syncthreads();

  if (warp >= PROD_WARP0) {
    // =================================== producers ===================================
    // Two threads per train row; the packed rows of the next kPrefetch tiles are held in registers so that the HBM
    // latency (~1 us) of a tile overlaps the expansion of the previous ones.
    const int pt = tid - PROD_WARP0 * 32;   // 0..255
    const int prow = (pt & 7) | ((pt >> 4) << 3), half = (pt >> 3) & 1;
    struct TileIt {
      int seg, r0, s_begin, len, seg1;
      const int32_t* sp;
      bool done;
      __device__ void next_seg() {
        do {
          seg++;
          if (seg >= seg1) { done = true; return; }
          s_begin = sp[seg];
          len = sp[seg + 1] - s_begin;
        } while (len == 0);
        r0 = 0;
      }
      __device__ void advance() { r0 += TN; if (r0 >= len) next_seg(); }
    };
    TileIt it{seg0 - 1, 0, 0, 0, seg1, p.seg_ptr, false}, ld = it;
    it.next_seg();
    ld.next_seg();
    constexpr int PF = M::kPrefetch;
    uint4 pf[PF][M::kLoads];
    auto issue_load = [&](uint4 (&v)[M::kLoads]) {
      if (!ld.done) {
        const int row = ld.r0 + prow;
        if (row < ld.len) M::load_half(p.t + (size_t)(ld.s_begin + row) * M::kRowBytes, half, v);
        ld.advance();
      }
    };
#pragma unroll
    for (int u = 0; u < PF; u++) issue_load(pf[u]);
    int n = 0;
    while (!it.done) {
#pragma unroll
      for (int u = 0; u < PF; u++) {
        if (it.done) break;
        uint4 cur[M::kLoads];
#pragma unroll
        for (int c = 0; c < M::kLoads; c++) cur[c] = pf[u][c];
        issue_load(pf[u]);   // refill this register slot with the tile PF steps ahead
        const int s = n % STAGES;
        if (n >= STAGES) cvb_mbar_wait(&empty[s], ((n / STAGES) - 1) & 1);
        uint8_t* dst = sB + (size_t)s * TN * KB + row_offset<KB>(prow);
        const bool rv = it.r0 + prow < it.len;
        int part = 0;
        if (rv) {
          part = M::store_half(cur, half, dst);
        } else {
          for (int c = 0; c < KB / 32; c++) *reinterpret_cast<uint4*>(dst + (half * (KB / 32) + c) * 128) = make_uint4(0, 0, 0, 0);
        }
        part += __shfl_xor_sync(0xffffffffu, part, 8);   // the two halves of a row sit 8 lanes apart
        if (M::kIsL2) {
          if (half == 0) sNorm[(n % NORM_RING) * TN + prow] = rv ? part : kInf;
        } else if (half == 0) {
          // Hamming: 16-bit column term ((popc(row) + 256) << 5 | slot), slot = 2 (column / 8) + column % 2 — the position
          // of the column among the 32 columns one consumer thread holds; 0xFFFF = no row
          reinterpret_cast<uint16_t*>(sNorm)[(n % NORM_RING) * TN + prow] =
              rv ? (uint16_t)(((part + 256) << 5) | ((prow >> 3) << 1) | (prow & 1)) : (uint16_t)0xFFFFu;
        }
        // every lane makes its own stores visible to the async proxy; ONE arrival per warp
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[s]);
        it.advance();
        n++;
      }
    }
  } else {
    // =================================== consumers: warpgroup h = query rows [64 h, 64 h + 64) ===================================
    const int h = warp >> 2;
    const int quad = lane & 3;
    const int row0 = 64 * h + 16 * (warp & 3) + (lane >> 2);   // this thread's rows: row0 and row0 + 8
    const bool valid0 = qb * TM + row0 < p.nq, valid1 = qb * TM + row0 + 8 < p.nq;
    const int qn0 = sQNorm[row0], qn1 = sQNorm[row0 + 8];
    const uint64_t a_desc = make_desc(cvb_smem_addr(sA + (size_t)h * 64 * KB), 128, KB * 8);
    const uint32_t b_addr0 = cvb_smem_addr(sB);
    int wk0[K], wi0[K], wd0[K], wk1[K], wi1[K], wd1[K];   // key, index, raw integer distance (pre-test only) per row
    int n = 0;
    for (int seg = seg0; seg < seg1; seg++) {
      const int len = p.seg_ptr[seg + 1] - p.seg_ptr[seg];
#pragma unroll
      for (int c = 0; c < K; c++) {
        wk0[c] = wk1[c] = M::kIsL2 ? kInfKey : INT_MAX;
        wi0[c] = wi1[c] = -1;
        wd0[c] = wd1[c] = kInf;
      }
      for (int r0 = 0; r0 < len; r0 += TN, n++) {
        const int s = n % STAGES;
        cvb_mbar_wait(&full[s], (n / STAGES) & 1);
        uint32_t acc[64];
        wg_gemm<false, KB / 32>(acc, a_desc, make_desc(b_addr0 + (uint32_t)s * (TN * KB), 128, KB * 8));
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);   // operands consumed: the producers may refill this stage
        if (!M::kIsL2) {
          // Two columns per instruction: 16-bit keys ((popc(t) - 2 popc(q & t) + 256) << 5 | slot) packed pairwise
          // (even column low, odd column high), k-lists kept per half with packed 16-bit min/max, merged into the 32-bit
          // (distance, index) lists once per tile — and only if the tile holds a candidate that beats the current k-th
          // entry (later tiles have larger indices, so "beats" is a strict distance comparison).
          const uint32_t* nrm2 = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(sNorm) + (n % NORM_RING) * TN);
          unsigned pk0[K], pk1[K];
#pragma unroll
          for (int c = 0; c < K; c++) pk0[c] = pk1[c] = 0xFFFFFFFFu;
#pragma unroll
          for (int i = 0; i < 16; i++) {
            const unsigned nv = nrm2[4 * i + quad];   // columns 8 i + 2 quad (low half) and + 1 (high half)
            insert_packed16<K>(pk0, nv - __byte_perm(acc[4 * i], acc[4 * i + 1], 0x5410));
            insert_packed16<K>(pk1, nv - __byte_perm(acc[4 * i + 2], acc[4 * i + 3], 0x5410));
          }
#pragma unroll
          for (int rr = 0; rr < 2; rr++) {
            unsigned (&pk)[K] = rr ? pk1 : pk0;
            int (&wk)[K] = rr ? wk1 : wk0;
            const unsigned best16 = min(pk[0] & 0xFFFFu, pk[0] >> 16);
            const int worst_v = wk[K - 1] == INT_MAX ? 1024 : (wk[K - 1] >> kIdxBits) + 256;   // arithmetic shift: t-domain value
            if ((int)(best16 >> 5) < worst_v) {
#pragma unroll
              for (int c = 0; c < K; c++)
#pragma unroll
                for (int hh = 0; hh < 2; hh++) {
                  const unsigned k16 = hh ? (pk[c] >> 16) : (pk[c] & 0xFFFFu);
                  const int col = 8 * (int)((k16 & 31u) >> 1) + 2 * quad + (int)(k16 & 1u);
                  insert_packed<K>(wk, k16 == 0xFFFFu ? INT_MAX
                                                      : (int)((((unsigned)(k16 >> 5) - 256u) << kIdxBits) + (unsigned)(r0 + col)));
                }
            }
          }
        } else {
          const int* nrm = sNorm + (n % NORM_RING) * TN;
#pragma unroll
          for (int i = 0; i < 16; i++) {
            const int2 nn = *reinterpret_cast<const int2*>(nrm + 8 * i + 2 * quad);
#pragma unroll
            for (int e = 0; e < 4; e++) {
              const int j = 8 * i + 2 * quad + (e & 1);
              const int tn = (e & 1) ? nn.y : nn.x;
              int (&wk)[K] = e < 2 ? wk0 : wk1;
              int (&wi)[K] = e < 2 ? wi0 : wi1;
              int (&wd)[K] = e < 2 ? wd0 : wd1;
              const int d = (e < 2 ? qn0 : qn1) + tn - 2 * (int)acc[4 * i + e];
              if (d < wd[K - 1]) {
                const int key = __float_as_int(__fsqrt_rn((float)d));
                if (key < wk[K - 1]) {
                  insert_key<K>(wk, wi, key, r0 + j);
                  const float f = __int_as_float(wk[K - 1]);   // raw-distance bound of the worst entry (pre-test)
                  wd[K - 1] = wk[K - 1] == kInfKey ? kInf : (int)ceilf(f * f * 1.000001f) + 1;
                }
              }
            }
          }
        }
      }
      // ---- segment finished: merge the quad's lists; lane quad 0 writes row0, quad 1 writes row0 + 8 ----
      const bool second = quad == 1;
      int wk[K], wi[K];
      float fd[K];
      if (!M::kIsL2) {
        quad_merge_packed<K>(wk0);
        quad_merge_packed<K>(wk1);
        const int qq = (second ? qn1 : qn0) << kIdxBits;
#pragma unroll
        for (int c = 0; c < K; c++) {
          const int x = second ? wk1[c] : wk0[c];
          wi[c] = x == INT_MAX ? -1 : (x & ((1 << kIdxBits) - 1));
          wk[c] = x == INT_MAX ? INT_MAX : ((x + qq) >> kIdxBits);
          fd[c] = (float)wk[c];
        }
      } else {
        quad_merge_lex<K>(wk0, wi0);
        quad_merge_lex<K>(wk1, wi1);
#pragma unroll
        for (int c = 0; c < K; c++) {
          wk[c] = second ? wk1[c] : wk0[c];
          wi[c] = second ? wi1[c] : wi0[c];
          fd[c] = __int_as_float(wk[c]);
        }
      }
      write_list<K, M::kIsL2>(p, seg, qb * TM + row0 + (second ? 8 : 0), quad < 2 && (second ? valid1 : valid0), wk, wi, fd, lane);
    }
  }
}


// ===================================================================================================================
// Hamming k-NN on PRE-EXPANDED operand tiles.
//
// The kernel above spends its issue slots on ALU work: producers turn every packed bit into a byte (>= 64 logic
// operations per row and tile) and the epilogue rebuilds the distance from the accumulator and a per-column term read
// from shared memory.  Both disappear when the operand the tensor core reads is stored once and reused by every query:
//
//   * cvb_tc::expand_tiles writes, per keyframe, ceil(rows / 128) tiles of 128 rows x 288 operand bytes in exactly the
//     shared-memory image wgmma wants (K-major, no swizzle, 8-row groups of 2304 B): 256 data bytes (0x80 = -128
//     as s8 for a set bit) + a 32-byte KEY slice.  A tile is 36 KB and contiguous, so the producer is ONE thread issuing
//     cp.async.bulk copies (TMA engine) — no register path, no expansion in the matching kernel.  The map database
//     (map_db.cu) keeps these tiles resident next to the packed rows; 9 bytes of HBM per descriptor byte.
//   * the key slice folds the whole distance into the GEMM: with query bytes 0/2 (u8) and
//         A key bytes = [1, 128, 128, 128, c4, c5, c6, 0...]   c4 + c5 + c6 = 2 popc(q)      (per query row)
//         B key bytes = [col, p1, p2, p3, 64, 64, 64, 0...]    p1 + p2 + p3 = popc(t)        (per train row)
//     the s32 accumulator is  (popc(q) + popc(t) - 2 popc(q & t)) << 7 | col  =  Hamming << 7 | row-in-tile: the sort key
//     itself, <= 32895, so the epilogue packs two adjacent columns into one register and runs nothing but the packed
//     min/max network.  Rows past a keyframe's end carry B key bytes [127,127,127,127,0...] → key 48895, which never
//     enters a list.
//   * NGRP segment STREAMS: consumer warpgroups (h, g) own query rows [64 h, 64 h + 64) and every NGRP-th keyframe of the
//     CTA's range starting at g; the producer interleaves the streams' tiles, so while one stream's warpgroups run
//     their epilogue the other's keep the tensor cores busy.  A (query, keyframe) list lives in one quad's registers
//     from the first tile to the output — no shared-memory lists, no CTA barrier per keyframe.
namespace xt {
constexpr int KX = 288;                       // operand bytes per row
constexpr int NSLICE = KX / 32;               // 9 instructions of K = 32 per tile
constexpr int TILE_BYTES = TN * KX;           // 36864
constexpr int XSTAGES = 5;                    // shared-memory ring (180 KB) — more than NGRP (phase parity of full[])
constexpr int NGRP = 2;                       // streams
constexpr int CONS_WARPS = 4 * 2 * NGRP;      // warpgroups (h, g), h = query half
constexpr int TMA_WARP = CONS_WARPS;
constexpr int XTHREADS = (TMA_WARP + 1) * 32;
constexpr int kKeyInvalid = 32896;            // keys >= this are "no row"
constexpr size_t kSmemBytes = (size_t)(XSTAGES + 1) * TILE_BYTES + 1024;   // query block + ring + barriers

__device__ __forceinline__ uint32_t xrow_off(int r) { return (uint32_t)(r >> 3) * (KX * 8) + (uint32_t)(r & 7) * 16; }

// ---- one-time expansion (also the append path of the map database) ----
__global__ void __launch_bounds__(256) expand_tiles_kernel(const uint8_t* __restrict__ t, const int32_t* __restrict__ seg_ptr,
                                                           const int32_t* __restrict__ seg_tile, int seg_lo, int seg_hi,
                                                           int tile_lo, uint8_t* __restrict__ out) {
  const int tile = tile_lo + blockIdx.x;
  int lo = seg_lo, hi = seg_hi - 1;             // the last segment whose first tile is <= tile (skips empty segments)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seg_tile[mid] <= tile) lo = mid; else hi = mid - 1;
  }
  const int s_begin = seg_ptr[lo], len = seg_ptr[lo + 1] - s_begin, r0 = (tile - seg_tile[lo]) * TN;
  const int pt = threadIdx.x, prow = (pt & 7) | ((pt >> 4) << 3), half = (pt >> 3) & 1;
  const bool rv = r0 + prow < len;
  uint8_t* dst = out + (size_t)tile * TILE_BYTES + xrow_off(prow);
  int part = 0;
  if (rv) {
    uint4 v[1];
    TcHamming::load_half(t + (size_t)(s_begin + r0 + prow) * 32, half, v);
    part = TcHamming::store_half<7>(v, half, dst);
  } else {
#pragma unroll
    for (int c = 0; c < 8; c++) *reinterpret_cast<uint4*>(dst + (8 * half + c) * 128) = make_uint4(0, 0, 0, 0);
  }
  part += __shfl_xor_sync(0xffffffffu, part, 8);
  if (half == 0) {
    uint4 key = make_uint4(0x7F7F7F7Fu, 0, 0, 0);
    if (rv) {
      const int p1 = min(part, 127), p2 = min(part - p1, 127), p3 = part - p1 - p2;
      key.x = (uint32_t)prow | ((uint32_t)p1 << 8) | ((uint32_t)p2 << 16) | ((uint32_t)p3 << 24);
      key.y = 0x00404040u;
    }
    *reinterpret_cast<uint4*>(dst + 16 * 128) = key;
  } else {
    *reinterpret_cast<uint4*>(dst + 17 * 128) = make_uint4(0, 0, 0, 0);
  }
}

// the interleaved tile sequence of a CTA: stream g walks keyframes seg0 + g, seg0 + g + NGRP, ... ; round-robin over the
// streams that still have tiles.  Producer and consumers generate the same sequence.
struct Streams {
  int seg[NGRP], t[NGRP], nt[NGRP], tile0[NGRP];
  int seg1;
  const int32_t* seg_tile;
  __device__ void load(int g) {          // position stream g on its next non-empty keyframe (or past the end)
    while (seg[g] < seg1) {
      tile0[g] = seg_tile[seg[g]];
      nt[g] = seg_tile[seg[g] + 1] - tile0[g];
      if (nt[g] > 0) break;
      seg[g] += NGRP;
    }
    t[g] = 0;
  }
  __device__ void init(int seg0, int seg1_, const int32_t* st) {
    seg1 = seg1_; seg_tile = st;
#pragma unroll
    for (int g = 0; g < NGRP; g++) { seg[g] = seg0 + g; nt[g] = 0; tile0[g] = 0; load(g); }
  }
  __device__ bool active(int g) const { return seg[g] < seg1; }
  __device__ bool any() const {
    bool a = false;
#pragma unroll
    for (int g = 0; g < NGRP; g++) a |= seg[g] < seg1;
    return a;
  }
  __device__ void advance(int g) {
    if (++t[g] >= nt[g]) { seg[g] += NGRP; load(g); }
  }
};

template <int K>
__global__ void __launch_bounds__(XTHREADS, 1) tc_xt_kernel(const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;                                  // the query block, one tile image [TM][KX]
  uint8_t* sB = smem + TILE_BYTES;                     // [XSTAGES] tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)(XSTAGES + 1) * TILE_BYTES);
  uint64_t* full = bars;                  // [XSTAGES] TMA bytes landed (expect_tx)
  uint64_t* empty = bars + XSTAGES;       // [XSTAGES] the stage's two warpgroups finished their MMAs (one arrival per warp)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qb = blockIdx.x % p.nqb, part = blockIdx.x / p.nqb;
  const int seg0 = (int)((long)part * p.n_seg / p.parts), seg1 = (int)((long)(part + 1) * p.n_seg / p.parts);

  if (tid == 0) {
    for (int s = 0; s < XSTAGES; s++) { cvb_mbar_init(&full[s], 1); cvb_mbar_init(&empty[s], 8); }
    cvb_fence_mbar_init();
  }
  if (tid < TM) {
    // query block → shared memory (thread = row): data bytes 0/2, then the key slice
    const int q = qb * TM + tid;
    uint32_t w[8];
    int pq = 0;
    if (q < p.nq) {
      pq = TcHamming::load_q(p.q + (size_t)q * 32, w);
    } else {
#pragma unroll
      for (int i = 0; i < 8; i++) w[i] = 0;
    }
    uint8_t* dst = sA + xrow_off(tid);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint32_t r[8];
#pragma unroll
      for (int b = 0; b < 8; b++) r[b] = ((w[i] >> b) & 0x01010101u) * 2u;
      *reinterpret_cast<uint4*>(dst + (2 * i) * 128) = make_uint4(r[0], r[1], r[2], r[3]);
      *reinterpret_cast<uint4*>(dst + (2 * i + 1) * 128) = make_uint4(r[4], r[5], r[6], r[7]);
    }
    {
      const int c4 = min(2 * pq, 255), c5 = min(2 * pq - c4, 255), c6 = 2 * pq - c4 - c5;
      uint4 key = make_uint4(0, 0, 0, 0);
      if (q < p.nq) { key.x = 0x80808001u; key.y = (uint32_t)c4 | ((uint32_t)c5 << 8) | ((uint32_t)c6 << 16); }
      *reinterpret_cast<uint4*>(dst + 16 * 128) = key;
      *reinterpret_cast<uint4*>(dst + 17 * 128) = make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == TMA_WARP) {
    // =================================== producer: one thread, bulk copies ===================================
    if (lane == 0) {
      Streams S;
      S.init(seg0, seg1, p.seg_tile);
      int n = 0;
      while (S.any()) {
#pragma unroll
        for (int g = 0; g < NGRP; g++) {
          if (!S.active(g)) continue;
          const int s = n % XSTAGES;
          if (n >= XSTAGES) cvb_mbar_wait(&empty[s], ((n / XSTAGES) - 1) & 1);
          cvb_mbar_expect_tx(&full[s], TILE_BYTES);
          const uint8_t* src = p.xt + (size_t)(S.tile0[g] + S.t[g]) * TILE_BYTES;
          uint8_t* dst = sB + (size_t)s * TILE_BYTES;
#pragma unroll
          for (int c = 0; c < 4; c++) cvb_bulk_g2s(dst + c * (TILE_BYTES / 4), src + c * (TILE_BYTES / 4), TILE_BYTES / 4, &full[s]);
          S.advance(g);
          n++;
        }
      }
    }
    __syncwarp();
  } else {
    // =================================== consumer warpgroup (h, g): every NGRP-th keyframe, start to finish ===================================
    const int h = (warp >> 2) & 1, g = warp >> 3;
    const int quad = lane & 3;
    const int row0 = 64 * h + 16 * (warp & 3) + (lane >> 2);   // this thread's rows: row0 and row0 + 8
    const uint64_t a_desc = make_desc(cvb_smem_addr(sA + (size_t)h * 8 * (KX * 8)), 128, KX * 8);
    const uint32_t b_addr0 = cvb_smem_addr(sB);
    // empty keyframes of this stream have no tiles: their (empty) lists are written here
    for (int seg = seg0 + g; seg < seg1; seg += NGRP) {
      if (p.seg_tile[seg + 1] != p.seg_tile[seg]) continue;
      int wk[K], wi[K];
      float fd[K];
#pragma unroll
      for (int c = 0; c < K; c++) { wk[c] = INT_MAX; wi[c] = -1; fd[c] = (float)INT_MAX; }
      write_list<K, false>(p, seg, qb * TM + row0 + (quad == 1 ? 8 : 0), quad < 2, wk, wi, fd, lane);
    }
    Streams S;
    S.init(seg0, seg1, p.seg_tile);
    int wk0[K], wk1[K];   // (distance << kIdxBits) + row within the keyframe, ascending — rows row0 and row0 + 8
    int n = 0;
    while (S.any()) {
#pragma unroll
      for (int g2 = 0; g2 < NGRP; g2++) {
        if (!S.active(g2)) continue;
        if (g2 == g) {
          const int t = S.t[g2];
          if (t == 0) {
#pragma unroll
            for (int c = 0; c < K; c++) wk0[c] = wk1[c] = INT_MAX;
          }
          const int s = n % XSTAGES;
          cvb_mbar_wait(&full[s], (n / XSTAGES) & 1);
          uint32_t acc[64];
          wg_gemm<true, NSLICE>(acc, a_desc, make_desc(b_addr0 + (uint32_t)s * TILE_BYTES, 128, KX * 8));
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[s]);   // operands consumed: the producer may refill this stage
          unsigned pk0[K], pk1[K];
#pragma unroll
          for (int c = 0; c < K; c++) pk0[c] = pk1[c] = 0xFFFFFFFFu;
#pragma unroll
          for (int i = 0; i < 16; i++) {   // columns 8 i + 2 quad (low half) and + 1 (high half)
            insert_packed16<K>(pk0, __byte_perm(acc[4 * i], acc[4 * i + 1], 0x5410));
            insert_packed16<K>(pk1, __byte_perm(acc[4 * i + 2], acc[4 * i + 3], 0x5410));
          }
          // later tiles hold larger row indices: a candidate enters only with a strictly smaller distance than the k-th entry
#pragma unroll
          for (int rr = 0; rr < 2; rr++) {
            unsigned (&pk)[K] = rr ? pk1 : pk0;
            int (&wk)[K] = rr ? wk1 : wk0;
            const unsigned best16 = min(pk[0] & 0xFFFFu, pk[0] >> 16);
            const int worst_d = wk[K - 1] == INT_MAX ? 1024 : (wk[K - 1] >> kIdxBits);
            if ((int)(best16 >> 7) < worst_d) {
#pragma unroll
              for (int c = 0; c < K; c++)
#pragma unroll
                for (int hh = 0; hh < 2; hh++) {
                  const unsigned k16 = hh ? (pk[c] >> 16) : (pk[c] & 0xFFFFu);
                  insert_packed<K>(wk, k16 >= (unsigned)kKeyInvalid ? INT_MAX
                                                                   : (int)(((k16 >> 7) << kIdxBits) + (unsigned)(t * TN) + (k16 & 127u)));
                }
            }
          }
          if (t == S.nt[g2] - 1) {
            // ---- keyframe finished: merge the quad's lists; lane quad 0 writes row0, quad 1 writes row0 + 8 ----
            quad_merge_packed<K>(wk0);
            quad_merge_packed<K>(wk1);
            const bool second = quad == 1;
            int wk[K], wi[K];
            float fd[K];
#pragma unroll
            for (int c = 0; c < K; c++) {
              const int x = second ? wk1[c] : wk0[c];
              wi[c] = x == INT_MAX ? -1 : (x & ((1 << kIdxBits) - 1));
              wk[c] = x == INT_MAX ? INT_MAX : (x >> kIdxBits);
              fd[c] = (float)wk[c];
            }
            write_list<K, false>(p, S.seg[g2], qb * TM + row0 + (second ? 8 : 0), quad < 2, wk, wi, fd, lane);
          }
        }
        S.advance(g2);
        n++;
      }
    }
  }
}

template <int K>
int launch_xt(cvb_ctx* ctx, const TcParams& p, cudaStream_t st) {
  static cvb_once_per_device once;
  {
    std::lock_guard<std::mutex> once_lk(once.mtx);
    if (once.first(ctx->device)) {
      CVB_CUDA(ctx, cudaFuncSetAttribute(tc_xt_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
    }
  }
  tc_xt_kernel<K><<<p.nqb * p.parts, XTHREADS, kSmemBytes, st>>>(p);
  CVB_CHECK_LAUNCH(ctx);
  return CVB_OK;
}
}  // namespace xt

int64_t tiles_of(const int32_t* h_seg, int n_seg, std::vector<int32_t>* seg_tile) {
  int64_t total = 0;
  if (seg_tile) seg_tile->assign((size_t)n_seg + 1, 0);
  for (int s = 0; s < n_seg; s++) {
    total += (h_seg[s + 1] - h_seg[s] + TN - 1) / TN;
    if (seg_tile) (*seg_tile)[s + 1] = (int32_t)total;
  }
  return total;
}
size_t tile_bytes() { return xt::TILE_BYTES; }

int expand_tiles(cvb_ctx* ctx, const uint8_t* d_rows, const int32_t* d_seg_ptr, const int32_t* d_seg_tile, int seg_lo, int seg_hi,
                 int tile_lo, int n_tiles, uint8_t* d_xt, cudaStream_t st) {
  if (n_tiles <= 0) return CVB_OK;
  xt::expand_tiles_kernel<<<n_tiles, 256, 0, st>>>(d_rows, d_seg_ptr, d_seg_tile, seg_lo, seg_hi, tile_lo, d_xt);
  CVB_CHECK_LAUNCH(ctx);
  return CVB_OK;
}

template <class M, int K>
int launch_tc(cvb_ctx* ctx, const TcParams& p, cudaStream_t st) {
  static cvb_once_per_device once;
  const size_t smem = smem_bytes<M>();
  {
    std::lock_guard<std::mutex> once_lk(once.mtx);
    if (once.first(ctx->device)) {
      CVB_CUDA(ctx, cudaFuncSetAttribute(tc_scan_kernel<M, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
  }
  tc_scan_kernel<M, K><<<p.nqb * p.parts, NUM_THREADS, smem, st>>>(p);
  CVB_CHECK_LAUNCH(ctx);
  return CVB_OK;
}

bool profitable(const cvb_ctx* ctx, int nq, int n_seg, long total_rows, int max_seg_len) {
  if (max_seg_len >= (1 << kIdxBits)) return false;   // packed (distance, index) keys need < 4 Mi rows per segment
  const char* e = getenv("COVINS_B200_MATCH_KERNEL");
  if (e && !strcmp(e, "popc")) return false;
  if (e && !strcmp(e, "tc")) return n_seg >= 1 && nq >= 1;
  const int nqb = (nq + TM - 1) / TM;
  const int want_parts = ctx->sm_count / nqb > 0 ? ctx->sm_count / nqb : 1;
  return n_seg >= want_parts && (long)nq * total_rows >= (1L << 26);
}

int launch(cvb_ctx* ctx, TcParams p, int metric, int k, cudaStream_t st) {
  p.nqb = (p.nq + TM - 1) / TM;
  int parts = ctx->sm_count / p.nqb;
  if (parts < 1) parts = 1;
  if (parts > p.n_seg) parts = p.n_seg;
  p.parts = parts;
  if (metric == 0 && !(getenv("COVINS_B200_TC_XT") && !strcmp(getenv("COVINS_B200_TC_XT"), "0"))) {
    cvb_block B(ctx, st);
    if (!p.xt) {
      // no resident tile store for this train set (raw-pointer API): expand it into the call's block first (HBM-bound pre-pass)
      CVB_REQUIRE(ctx, p.h_seg != nullptr, "tensor-core Hamming path needs the host copy of the segment table");
      std::vector<int32_t> h_tile;
      const int64_t n_tiles = tiles_of(p.h_seg, p.n_seg, &h_tile);
      int32_t* d_tile;
      uint8_t* d_xt;
      B.tmp(d_tile, (size_t)p.n_seg + 1); B.tmp(d_xt, (size_t)n_tiles * xt::TILE_BYTES);
      if (const int rc = B.place()) return rc;
      CVB_CUDA(ctx, cudaMemcpyAsync(d_tile, h_tile.data(), sizeof(int32_t) * ((size_t)p.n_seg + 1), cudaMemcpyHostToDevice, st));
      CVB_CUDA(ctx, cudaStreamSynchronize(st));   // h_tile goes out of scope
      const int rc = expand_tiles(ctx, p.t, p.seg_ptr, d_tile, 0, p.n_seg, 0, (int)n_tiles, d_xt, st);
      if (rc) return rc;
      p.xt = d_xt;
      p.seg_tile = d_tile;
    }
    switch (k) {
      case 1: return xt::launch_xt<1>(ctx, p, st);
      case 2: return xt::launch_xt<2>(ctx, p, st);
      case 3: return xt::launch_xt<3>(ctx, p, st);
      default: return xt::launch_xt<4>(ctx, p, st);
    }
  }
#define TC_CASE(MM, KK) return launch_tc<MM, KK>(ctx, p, st)
  if (metric == 0) {
    switch (k) { case 1: TC_CASE(TcHamming, 1); case 2: TC_CASE(TcHamming, 2); case 3: TC_CASE(TcHamming, 3); default: TC_CASE(TcHamming, 4); }
  }
  switch (k) { case 1: TC_CASE(TcL2, 1); case 2: TC_CASE(TcL2, 2); case 3: TC_CASE(TcL2, 3); default: TC_CASE(TcL2, 4); }
#undef TC_CASE
}

}  // namespace cvb_tc
