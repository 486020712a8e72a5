// cholesky.cu — dense FP64 Cholesky factorisation + triangular solves of the reduced camera system (K8).
//
// Replaces the CHOLMOD factorisation inside Ceres' SPARSE_SCHUR (optimization_be.cpp:258,561,1025).  The
// reduced camera matrix S (n = 6K or 15K, padded to a multiple of the 128 tile) is stored as a PACKED list of the
// 128x128 tiles of L's structure (lower triangle, symbolic fill included; row-major inside a tile, a tile column's
// tiles contiguous — TilePlan::h_col_base / h_tile_of): memory is proportional to nnz(L) at tile granularity (0.8 GB at
// C3 instead of 7.4 GB dense; C5 fits), every tile is one contiguous 128 KB block, and a panel is one contiguous range.
// At EuRoC scale every keyframe is covisible with hundreds of others (all agents fly the same hall), so the pose part
// of S is ~10 % block-dense before fill and fills in almost completely: a tiled dense-tile factorisation is the right
// shape for the GPU; this is the one BA stage that is a true GEMM and runs on the FP64 tensor cores (DMMA,
// mma.sync.m16n8k16.f64, Hopper's full-rate shape — wgmma has no FP64 kind).
//
// Right-looking, panel width 128:
//   potrf_inv_kernel   1 CTA: factor the 128x128 diagonal tile in shared memory, write L, write L^-1
//   trsm_kernel        row tiles below: A(i,k) <- A(i,k) * Linv^T            (128^3 DMMA GEMM per CTA)
//   tile_update_kernel trailing tiles (i >= j > k): A(i,j) -= A(i,k) A(j,k)^T (one 128x128 tile per CTA, 128^3 DMMA GEMM
//                      per panel; in blocks of kPanelBlock columns, all of a block's panels per visit to a tile — see
//                      factor()); syrk_kernel does the same for the chain's diagonal pair, spread over 4 CTAs for latency
// Solves use the stored tile inverses: forward L y = b, backward L^T x = y, one launch per tile column.
// All reductions have a fixed order → bit-reproducible run to run.
#include "cholesky.cuh"

#include <stdlib.h>

#include <algorithm>

namespace cvb_chol {

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(cvb_smem_addr(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// D = C + A B^T on one 16 x 8 x 16 block (SASS DMMA.16x8x16).  Fragments, g = lane / 4, t = lane % 4:
//   a[i] = A(g + 8 (i % 2), t + 4 (i / 2)),  b[i] = B(g, t + 4 i),  c[i] = C(g + 8 (i / 2), 2 t + i % 2).
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
               "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                 "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// acc(64 x BN) = A(64 x T) * B(BN x T)^T, both operands row-major with K contiguous (leading dims lda, ldb).
// 2 x BN/32 warps, 32x32 per warp = 2 (m16) x 4 (n8) m16n8k16 blocks, acc[i][j] = rows 16 i.., columns 8 j.. of the warp
// tile in the C-fragment order of dmma16816.  m16n8k16 is Hopper's full-rate FP64 MMA shape: on an H100 SXM (400 W limit)
// a register-only probe sustained 64 TFLOP/s with it (~128 FMA/clk/SM) and 34 TFLOP/s with the Ampere m8n8k4 shape, and
// its results were bit-identical to four chained m8n8k4 over the same 16-wide K chunk.  K is staged in chunks of 16 (one
// MMA per block and chunk) through a STAGES-deep cp.async ring (one barrier per chunk).  Row stride 20 doubles (≡ 8 words
// mod 32): the fragment loads of a half-warp (rows g = 0..3, columns t = 0..3) hit words 8g + 2t, conflict-free.  The CTA
// is deliberately small (64 x 64 x 128 for syrk_kernel: 128 threads, 60 KB): three to four CTAs share an SM, so one CTA's
// fixed costs — index fetch, pipeline fill, the C round trip of the epilogue, barrier bubbles — overlap the others' main
// loops.  The throughput path of the trailing update (tile_update_kernel) takes the whole 128x128 tile per CTA instead:
// it halves the operand bytes per FMA and keeps C in shared memory, so it has no per-panel C round trip to hide.
constexpr int KC = 16;
constexpr int LDS = KC + 4;
constexpr int GEMM_STAGES = 3;

template <int BN>
__device__ __forceinline__ void gemm_abt_64(const double* __restrict__ A, size_t lda, const double* __restrict__ B,
                                            size_t ldb, double (&acc)[2][4][4], double* smem) {
  constexpr int WN = BN / 32, THREADS = 2 * WN * 32, STAGE = (64 + BN) * LDS, NCH = T / KC, UPR = KC / 2;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp / WN, wn = warp % WN;
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[i][j][e] = 0.0;
  // a thread copies the same 16-byte segment of rows r0, r0 + RSTEP, ...: one base address per operand
  constexpr int RSTEP = THREADS / UPR;
  const int r0 = tid / UPR, seg = tid % UPR;
  const double* ga = A + (size_t)r0 * lda + seg * 2;
  const double* gb = B + (size_t)r0 * ldb + seg * 2;
  const int so = r0 * LDS + seg * 2;
  auto load_chunk = [&](int kc) {
    if (kc < NCH) {
      double* As = smem + (kc % GEMM_STAGES) * STAGE + so;
      double* Bs = As + 64 * LDS;
#pragma unroll
      for (int it = 0; it < 64 / RSTEP; it++) cp_async16(As + it * RSTEP * LDS, ga + (size_t)it * RSTEP * lda + kc * KC);
#pragma unroll
      for (int it = 0; it < BN / RSTEP; it++) cp_async16(Bs + it * RSTEP * LDS, gb + (size_t)it * RSTEP * ldb + kc * KC);
    }
    cp_async_commit();   // always commit (possibly empty) so the wait count below is uniform
  };
#pragma unroll
  for (int c = 0; c < GEMM_STAGES - 1; c++) load_chunk(c);
#pragma unroll 1   // unrolled, both instantiations exceed their register budgets and spill
  for (int kc = 0; kc < NCH; kc++) {
    cp_async_wait<GEMM_STAGES - 2>();   // chunk kc has landed
    __syncthreads();                    // ... for every thread, and chunk kc-1's stage is free again
    load_chunk(kc + GEMM_STAGES - 1);
    const double* As = smem + (kc % GEMM_STAGES) * STAGE;
    const double* a_base = As + (wm * 32 + (lane >> 2)) * LDS + (lane & 3);
    const double* b_base = As + 64 * LDS + (wn * 32 + (lane >> 2)) * LDS + (lane & 3);
    double a[2][8];
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
      for (int e = 0; e < 8; e++) a[i][e] = a_base[(i * 16 + 8 * (e & 1)) * LDS + 4 * (e >> 1)];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      double b[4];
#pragma unroll
      for (int e = 0; e < 4; e++) b[e] = b_base[j * 8 * LDS + 4 * e];
#pragma unroll
      for (int i = 0; i < 2; i++) dmma16816(acc[i][j], a[i], b);
    }
  }
}

constexpr int TRSM_THREADS = 256, SYRK_THREADS = 128;
constexpr size_t TT = (size_t)T * T;   // doubles per tile
constexpr size_t kTrsmSmem = (size_t)GEMM_STAGES * (64 + 128) * LDS * sizeof(double);   //  92160 B → 2 CTAs / SM
constexpr size_t kSyrkSmem = (size_t)GEMM_STAGES * (64 + 64) * LDS * sizeof(double);    //  61440 B → 3 CTAs / SM

// A(i,k) <- A(i,k) * Linv_k^T for the structurally non-zero row tiles i of tile column k (rows[]).  Two CTAs per tile,
// each owns 64 full rows (it has consumed all of them as the A operand before it overwrites them).
// `panel` = first row tile of the column (the column's row tiles are contiguous in the packed array).
__global__ void __launch_bounds__(TRSM_THREADS, 2) trsm_kernel(double* __restrict__ panel,
                                                                const double* __restrict__ linv_k) {
  extern __shared__ __align__(16) double smem_d[];
  constexpr size_t ld = T;
  const int half = blockIdx.x & 1;
  double* At = panel + (size_t)(blockIdx.x >> 1) * TT + (size_t)half * 64 * T;
  double acc[2][4][4];
  gemm_abt_64<128>(At, ld, linv_k, T, acc, smem_d);
  __syncthreads();   // every warp is done reading this CTA's rows (they were all staged through shared memory)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wm = warp >> 2, wn = warp & 3;
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int r = wm * 32 + a * 16 + h * 8 + (lane >> 2), c = wn * 32 + b * 8 + (lane & 3) * 2;
        *reinterpret_cast<double2*>(At + (size_t)r * ld + c) = make_double2(acc[a][b][2 * h], acc[a][b][2 * h + 1]);
      }
}

// The two small products of the critical chain (see factor(): "chain column"), one 128x128 tile each:
//   MODE 0:  C = P Q^T            (solve of the first panel tile: P = C = S(k+1,k) in place, Q = L(k,k)^-1)
//   MODE 1:  C -= P Q^T, j <= i   (update of the next diagonal tile: P = Q = L(k+1,k), C = S(k+1,k+1))
// The throughput kernels above give a tile to 2-4 CTAs (8.7 us of DMMA each); on the chain only latency counts, so the tile
// is spread over 64 CTAs x 2 rows: a CTA stages Q (128 KB, L2-resident, 8-byte cp.async, row stride 129 doubles) and its own
// two rows of P, then every thread owns one output column (plain FP64 FMAs: 2 x 128 per thread).  ~3 us per launch.
constexpr int CHAIN_ROWS = 2;
constexpr int CHAIN_LDQ = T + 1;
constexpr size_t kChainSmem = ((size_t)T * CHAIN_LDQ + (size_t)CHAIN_ROWS * T) * sizeof(double);
__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(cvb_smem_addr(smem)), "l"(gmem) : "memory");
}
template <int MODE>
__global__ void __launch_bounds__(T, 1) chain_gemm_kernel(double* __restrict__ C, const double* P, const double* Q) {
  extern __shared__ __align__(16) double smem_d[];
  double* Qs = smem_d;                          // [T][CHAIN_LDQ]
  double* Ps = smem_d + (size_t)T * CHAIN_LDQ;  // [CHAIN_ROWS][T]
  const int j = threadIdx.x, i0 = blockIdx.x * CHAIN_ROWS;
#pragma unroll 16
  for (int r = 0; r < T; r++) cp_async8(Qs + (size_t)r * CHAIN_LDQ + j, Q + (size_t)r * T + j);
#pragma unroll
  for (int r = 0; r < CHAIN_ROWS; r++) cp_async8(Ps + r * T + j, P + (size_t)(i0 + r) * T + j);
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  double acc[CHAIN_ROWS];
#pragma unroll
  for (int r = 0; r < CHAIN_ROWS; r++) acc[r] = 0.0;
  const double* qrow = Qs + (size_t)j * CHAIN_LDQ;
#pragma unroll 8
  for (int c = 0; c < T; c++) {
    const double qv = qrow[c];
#pragma unroll
    for (int r = 0; r < CHAIN_ROWS; r++) acc[r] = fma(Ps[r * T + c], qv, acc[r]);
  }
#pragma unroll
  for (int r = 0; r < CHAIN_ROWS; r++) {
    double* dst = C + (size_t)(i0 + r) * T + j;
    if (MODE == 0) *dst = acc[r];
    else if (j <= i0 + r) *dst -= acc[r];
  }
}

// A(i,j) -= A(i,k) A(j,k)^T for the tile pairs (i >= j) pi[]/pj[] and the panels k = k0 + q of the bits q of pmask[]
// (TilePlan::h_pair_mask), in increasing k, each panel's product subtracted on its own.  Used for the chain's diagonal pair
// (factor()), where one tile is updated alone and latency counts: four CTAs per pair, one 64x64
// quadrant each (consecutive CTAs share the pair's operands in L2); the quadrant above the diagonal of a diagonal tile is
// skipped.  The quadrant (32 KB) is fetched into L2 at the start, so the first epilogue does not wait on HBM, and stays
// there for the read-modify-write of the later panels: several panels per visit make one HBM round trip of C.
__global__ void __launch_bounds__(SYRK_THREADS, 3) syrk_kernel(double* __restrict__ S, const int* __restrict__ tile_of, int nt,
                                                                int k0, const int* __restrict__ pi, const int* __restrict__ pj,
                                                                const int* __restrict__ pmask) {
  extern __shared__ __align__(16) double smem_d[];
  constexpr size_t ld = T;
  const int p = blockIdx.x >> 2, qr = (blockIdx.x >> 1) & 1, qc = blockIdx.x & 1;
  const int i = pi[p], j = pj[p];
  if (i == j && qc > qr) return;
  double* C = S + (size_t)tile_of[(size_t)i * nt + j] * TT + (size_t)qr * 64 * T + qc * 64;
#pragma unroll
  for (int u = threadIdx.x; u < 64 * 4; u += SYRK_THREADS)   // 64 rows x 4 lines of 128 B
    asm volatile("prefetch.global.L2 [%0];" ::"l"(C + (size_t)(u >> 2) * ld + (u & 3) * 16));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wm = warp >> 1, wn = warp & 1;
  unsigned mask = (unsigned)pmask[p];
#pragma unroll 1
  for (int k = k0; mask != 0; k++, mask >>= 1) {
    if (!(mask & 1u)) continue;
    const double* Ai = S + (size_t)tile_of[(size_t)i * nt + k] * TT + (size_t)qr * 64 * T;
    const double* Aj = S + (size_t)tile_of[(size_t)j * nt + k] * TT + (size_t)qc * 64 * T;
    double acc[2][4][4];
    __syncthreads();   // every warp is done with the previous panel's last stages before the prologue refills them
    gemm_abt_64<64>(Ai, ld, Aj, ld, acc, smem_d);
#pragma unroll
    for (int a = 0; a < 2; a++)
#pragma unroll
      for (int b = 0; b < 4; b++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int r = wm * 32 + a * 16 + h * 8 + (lane >> 2), c = wn * 32 + b * 8 + (lane & 3) * 2;
          double2* q = reinterpret_cast<double2*>(C + (size_t)r * ld + c);
          double2 v = *q;
          v.x -= acc[a][b][2 * h];
          v.y -= acc[a][b][2 * h + 1];
          *q = v;
        }
  }
}

// The same update, one CTA per pair and the whole 128x128 tile per CTA: the throughput path (every update list except the
// chain's diagonal pair, see factor()).  Per 16-wide K chunk a CTA stages 128 rows of each operand for 128x128x16 FMA —
// half the operand bytes per FMA of the 64x64 quadrants above, whose L2→SM traffic bounded them.  8 warps of 64x32
// (4 m16 x 4 n8 blocks; a thread holds 128 accumulator doubles, the four B fragments of a chunk and one m16 row of A
// fragments at a time): 221 registers, 1 CTA/SM.  The operands come through a 3-stage cp.async ring that runs on across
// the panels of the pair's mask (a chunk's stage is refilled with the next panel's chunks while the epilogue runs).
// C lives in shared memory for the whole visit: it is copied in during the first chunks, each panel's product
// (accumulated from zero over the K chunks in order) is subtracted from it on its own, in increasing panel order, and it
// is written back once.  So the results are bit-identical to syrk_kernel's, with one C read and one C write per visit
// instead of an L2 read-modify-write per panel.  Ring rows are 128 B, unpadded: segment s of a row r sits at
// s ^ 2 (r & 3), which makes the fragment loads conflict-free; C rows are 1 KB, 16-byte segment s of row r at s ^ 4 (r & 1),
// which makes the epilogue's double2 accesses conflict-free.  Shared memory: 128 KB of C + 3 x 32 KB ring (+ 512 B).
constexpr int TILE_THREADS = 256;
constexpr int TILE_STAGES = 3;
constexpr int TILE_STAGE = 2 * T * KC;   // doubles per ring stage: 128 rows of A(i,k), then 128 rows of A(j,k)
constexpr size_t kTileSmem = (TT + (size_t)TILE_STAGES * TILE_STAGE) * sizeof(double);   // 229376 B → 1 CTA / SM

__global__ void __launch_bounds__(TILE_THREADS, 1) tile_update_kernel(double* __restrict__ S, const int* __restrict__ tile_of,
                                                                      int nt, int k0, const int* __restrict__ pi,
                                                                      const int* __restrict__ pj,
                                                                      const int* __restrict__ pmask) {
  extern __shared__ __align__(128) double smem_d[];
  __shared__ const double* s_ai[32];   // operand tiles A(i,k), A(j,k) of the pair's panels, in increasing k
  __shared__ const double* s_aj[32];
  constexpr int NCH = T / KC;
  double* Cs = smem_d;            // [T][T], swizzled
  double* ring = smem_d + TT;     // [TILE_STAGES][2 T][KC], swizzled
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int i = pi[blockIdx.x], j = pj[blockIdx.x];
  const bool diag = i == j;
  const unsigned mask = (unsigned)pmask[blockIdx.x];
  double* C = S + (size_t)tile_of[(size_t)i * nt + j] * TT;
  if (tid < 32 && ((mask >> tid) & 1u)) {
    const int q = __popc(mask & ((1u << tid) - 1u));
    s_ai[q] = S + (size_t)tile_of[(size_t)i * nt + k0 + tid] * TT;
    s_aj[q] = S + (size_t)tile_of[(size_t)j * nt + k0 + tid] * TT;
  }
  __syncthreads();
  const int nch = __popc(mask) * NCH;   // chunk c = K chunk c % NCH of the pair's panel c / NCH
  // a thread copies 16-byte segment `seg` of rows r0, r0 + 32, ... of both operands (r0 & 3 fixes the swizzle)
  const int r0 = tid >> 3, seg = tid & 7;
  const int so = r0 * KC + ((seg ^ ((r0 & 3) << 1)) << 1);
  auto load_chunk = [&](int c) {
    if (c < nch) {
      const size_t go = (size_t)r0 * T + (c % NCH) * KC + seg * 2;
      const double* ga = s_ai[c / NCH] + go;
      const double* gb = s_aj[c / NCH] + go;
      double* As = ring + (c % TILE_STAGES) * TILE_STAGE + so;
#pragma unroll
      for (int it = 0; it < T / 32; it++) cp_async16(As + it * 32 * KC, ga + (size_t)it * 32 * T);
#pragma unroll
      for (int it = 0; it < T / 32; it++) cp_async16(As + T * KC + it * 32 * KC, gb + (size_t)it * 32 * T);
    }
    cp_async_commit();   // always commit (possibly empty) so the wait count below is uniform
  };
  // rows 32 part .. 32 part + 31 of C join the group of chunk part + 2 (part < 4): all of C has landed at chunk 5, before
  // the first epilogue, and the copy overlaps the first chunks.  The quadrant above the diagonal of a diagonal tile is
  // neither read nor written.
  auto load_c = [&](int part) {
#pragma unroll
    for (int it = 0; it < 8; it++) {
      const int u = tid + it * TILE_THREADS, r = part * 32 + (u >> 6), s = u & 63;
      if (!(diag && r < 64 && s >= 32)) cp_async16(Cs + r * T + ((s ^ ((r & 1) << 2)) << 1), C + (size_t)r * T + s * 2);
    }
  };
  const int g = lane >> 2, t = lane & 3, wm = warp >> 2, wn = warp & 3;   // warp tile: rows 64 wm.., columns 32 wn..
  const bool idle = diag && wm == 0 && wn >= 2;                             // above the diagonal of a diagonal tile
  int cq[4];   // ring column of fragment K index t + 4 q (rows g + 8 n: the swizzle depends on g & 3 only)
#pragma unroll
  for (int q = 0; q < 4; q++) cq[q] = t + 4 * (q ^ (g & 3));
  double acc[4][4][4];
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[a][b][e] = 0.0;
#pragma unroll
  for (int c = 0; c < TILE_STAGES - 1; c++) load_chunk(c);
#pragma unroll 1
  for (int c = 0; c < nch; c++) {
    cp_async_wait<TILE_STAGES - 2>();   // chunk c has landed
    __syncthreads();                    // ... for every thread, and chunk c-1's stage is free again
    if (c < 4) load_c(c);
    load_chunk(c + TILE_STAGES - 1);
    if (idle) continue;
    const double* As = ring + (c % TILE_STAGES) * TILE_STAGE + (wm * 64 + g) * KC;
    const double* Bs = ring + (c % TILE_STAGES) * TILE_STAGE + T * KC + (wn * 32 + g) * KC;
    double b[4][4];
#pragma unroll
    for (int bj = 0; bj < 4; bj++)
#pragma unroll
      for (int e = 0; e < 4; e++) b[bj][e] = Bs[bj * 8 * KC + cq[e]];
#pragma unroll
    for (int ai = 0; ai < 4; ai++) {
      double a[8];
#pragma unroll
      for (int e = 0; e < 8; e++) a[e] = As[(ai * 16 + 8 * (e & 1)) * KC + cq[e >> 1]];
#pragma unroll
      for (int bj = 0; bj < 4; bj++) dmma16816(acc[ai][bj], a, b[bj]);
    }
    if (c % NCH == NCH - 1) {   // the panel is complete: subtract it, start the next one from zero
#pragma unroll
      for (int ai = 0; ai < 4; ai++)
#pragma unroll
        for (int bj = 0; bj < 4; bj++)
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const int r = wm * 64 + ai * 16 + h * 8 + g, s = wn * 16 + bj * 4 + t;
            double2* q = reinterpret_cast<double2*>(Cs + r * T + ((s ^ ((r & 1) << 2)) << 1));
            double2 v = *q;
            v.x -= acc[ai][bj][2 * h];
            v.y -= acc[ai][bj][2 * h + 1];
            *q = v;
            acc[ai][bj][2 * h] = 0.0;
            acc[ai][bj][2 * h + 1] = 0.0;
          }
    }
  }
  __syncthreads();   // every warp's last epilogue is in Cs
#pragma unroll 8
  for (int it = 0; it < (int)(TT / 2 / TILE_THREADS); it++) {
    const int u = tid + it * TILE_THREADS, r = u >> 6, s = u & 63;
    if (!(diag && r < 64 && s >= 32))
      *reinterpret_cast<double2*>(C + (size_t)r * T + s * 2) =
          *reinterpret_cast<const double2*>(Cs + r * T + ((s ^ ((r & 1) << 2)) << 1));
  }
}

// Factor the diagonal tile k in shared memory and invert the factor, one CTA of 512 threads.  This kernel is the serial
// chain of the whole factorisation (one launch per tile column, nothing else can run before its panel is solved), so it
// is organised around dependent-operation latency (DFMA, SHFL, STS→LDS and rsqrt latencies on the critical chain):
//   Cholesky: blocked right-looking, 16-wide block columns.  Per block column
//     (a) warp 0 factors the 16x16 diagonal block register-resident (lane = 2*row + half).  Per pivot the *unscaled*
//         column goes through 128 B of shared memory and the update uses a_rj * a_cj / pivot, so the chain per pivot is
//         STS → LDS → reciprocal → DMUL → DFMA (≈ 100 cycles); rsqrt and the L values are computed off the chain;
//     (b) one thread per row below solves its 16 unknowns by substitution against the block (in place, no scratch);
//     (c) the trailing sub-matrix gets its rank-16 update with 4x4 register tiles whose rows are interleaved with stride
//         n/4 (conflict-free shared-memory operand loads); one thread owns the product of row sets {tr+i*S} x {tc+j*S}
//         and scatters it to both triangles' canonical (row >= col) positions;
//     meanwhile warp 15 inverts the 16x16 diagonal block (needed only by the inverse phase) off the critical path.
//   Inverse: in place by recursive doubling (16 → 32 → 64 → 128): X21 = -C^-1 (B A^-1), 4x4 register tiles with
//   interleaved columns, a padded scratch tile; the 16x16 diagonal inverses come from the factorisation.
// L is written back to S, the inverse (row-major 128x128, zeros above the diagonal) to linv_k.  flag[0] |= 1 on a
// non-positive pivot (matrix not positive definite → the caller raises mu, as Ceres does on LINEAR_SOLVER_FAILURE).
constexpr int LDP = T + 1;
constexpr int PB = 16;
constexpr int POTRF_THREADS = 512;
constexpr int POTRF_WORKERS = POTRF_THREADS - 32;   // warp 15 inverts the diagonal blocks
constexpr int TMP_DOUBLES = 64 * 65;
constexpr size_t kPotrfSmem = ((size_t)T * LDP + (size_t)TMP_DOUBLES + (size_t)(T / PB) * PB * PB + 5 * PB) * sizeof(double);

#define POTRF_MARK(i)                                     \
  do {                                                    \
    if (prof != nullptr && tid == 0) prof[i] = clock64(); \
  } while (0)

__global__ void __launch_bounds__(POTRF_THREADS, 1) potrf_inv_kernel(double* __restrict__ S, size_t ld, int k,
                                                                     double* __restrict__ linv_k, int* __restrict__ flag,
                                                                     long long* __restrict__ prof, int prof_fine) {
  extern __shared__ __align__(16) double smem_d[];
  double* a = smem_d;                     // [T][LDP]
  double* tmp = smem_d + T * LDP;         // scratch of the inverse phase
  double* binv = tmp + TMP_DOUBLES;       // [8][16][16] inverses of the diagonal 16x16 blocks of L
  double* colbuf = binv + (T / PB) * PB * PB;   // [2][2*PB] pivot-column exchange (second half: dummy slots)
  double* rdbuf = colbuf + 4 * PB;              // [PB] reciprocal diagonal of the current diagonal block
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* At = S + (size_t)k * T * ld + (size_t)k * T;
  POTRF_MARK(0);
  {
    // all 16 16-byte loads of a thread are in flight before the first use (one L2/HBM round trip for the tile)
    double2 buf[T * T / 2 / POTRF_THREADS];
#pragma unroll
    for (int it = 0; it < T * T / 2 / POTRF_THREADS; it++) {
      const int u = tid + it * POTRF_THREADS, r = u / (T / 2), c = (u % (T / 2)) * 2;
      buf[it] = (c <= r) ? *reinterpret_cast<const double2*>(At + (size_t)r * ld + c) : make_double2(0.0, 0.0);
    }
#pragma unroll
    for (int it = 0; it < T * T / 2 / POTRF_THREADS; it++) {
      const int u = tid + it * POTRF_THREADS, r = u / (T / 2), c = (u % (T / 2)) * 2;
      a[r * LDP + c] = buf[it].x;
      a[r * LDP + c + 1] = (c + 1 <= r) ? buf[it].y : 0.0;
    }
  }
  __syncthreads();
  POTRF_MARK(1);
  // ---------------- Cholesky ----------------
  long long t_a = 0, acc_a = 0, acc_ab = 0, acc_b = 0, acc_c = 0;   // fine profile (thread 0 only), kept in registers
  for (int jb = 0; jb < T / PB; jb++) {
    const int c0 = jb * PB, nbelow = T - c0 - PB;
    if (prof_fine && tid == 0) t_a = clock64();
    if (warp == 0) {
      // (a) the 16x16 diagonal block.  Branch-free pivot loop: every lane stores one value per step (lanes of the other
      // column half into a dummy slot), readers mask by row index; a non-positive pivot only sets a flag bit.
      const int r = lane >> 1, hf = lane & 1;
      double v[8];
#pragma unroll
      for (int c = 0; c < 8; c++) {
        const int cc = hf * 8 + c;
        v[c] = (cc <= r) ? a[(c0 + r) * LDP + c0 + cc] : a[(c0 + cc) * LDP + c0 + r];
      }
      int bad = 0;
#pragma unroll
      for (int j = 0; j < PB; j++) {
        const int jh = j >> 3, jc = j & 7;
        double* cbuf = colbuf + (j & 1) * 2 * PB;
        cbuf[(hf == jh) ? r : PB + r] = v[jc];          // column j (unscaled, incl. the pivot at row j); dummy half
        __syncwarp();
        const double pv = cbuf[j];
        const double own_raw = cbuf[r];
        const double2* cb = reinterpret_cast<const double2*>(cbuf + hf * 8);
        double2 l01 = cb[0], l23 = cb[1], l45 = cb[2], l67 = cb[3];
        bad |= !(pv > 0.0);
        const double piv = (pv > 0.0) ? pv : 1.0;
        const double rinv = rsqrt(piv);                 // the chain: LDS → rsqrt → 2 DMUL → DFMA → STS
        const double own = (r > j) ? own_raw : 0.0;
        const double t = (own * rinv) * rinv;
        // rows of the column at or above the pivot must not contribute: zero them (off the chain, parallel to rsqrt)
        const int cbase = hf * 8;
        l01.x = (cbase + 0 > j) ? l01.x : 0.0; l01.y = (cbase + 1 > j) ? l01.y : 0.0;
        l23.x = (cbase + 2 > j) ? l23.x : 0.0; l23.y = (cbase + 3 > j) ? l23.y : 0.0;
        l45.x = (cbase + 4 > j) ? l45.x : 0.0; l45.y = (cbase + 5 > j) ? l45.y : 0.0;
        l67.x = (cbase + 6 > j) ? l67.x : 0.0; l67.y = (cbase + 7 > j) ? l67.y : 0.0;
        v[0] -= t * l01.x; v[1] -= t * l01.y; v[2] -= t * l23.x; v[3] -= t * l23.y;
        v[4] -= t * l45.x; v[5] -= t * l45.y; v[6] -= t * l67.x; v[7] -= t * l67.y;
        const double lval = (r > j) ? own * rinv : ((r == j) ? piv * rinv : 0.0);   // column j of L
        v[jc] = (hf == jh) ? lval : v[jc];
        if (lane == 0) rdbuf[j] = rinv;
      }
      if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(flag, 1);
#pragma unroll
      for (int c = 0; c < 8; c++) a[(c0 + r) * LDP + c0 + hf * 8 + c] = (hf * 8 + c <= r) ? v[c] : 0.0;
      if (prof_fine && tid == 0) acc_a += clock64() - t_a;
    }
    __syncthreads();
    if (prof_fine && tid == 0) { const long long tt = clock64(); acc_ab += tt - t_a; t_a = tt; }
    if (warp == POTRF_THREADS / 32 - 1) {
      // inverse of the diagonal block, off the critical path: lane j (< 16) builds column j of Ljj^-1 by forward
      // substitution in axpy form (16 dependent steps, the row updates of a step are independent)
      if (lane < PB) {
        const int j = lane;
        double res[PB];
#pragma unroll
        for (int q = 0; q < PB; q++) res[q] = (q == j) ? 1.0 : 0.0;
#pragma unroll
        for (int m = 0; m < PB; m++) {
          const double xm = res[m] * rdbuf[m];       // rows m < j stay exactly zero
          res[m] = xm;
#pragma unroll
          for (int q = m + 1; q < PB; q++) res[q] -= a[(c0 + q) * LDP + c0 + m] * xm;
        }
#pragma unroll
        for (int q = 0; q < PB; q++) binv[(jb * PB + q) * PB + j] = res[q];   // Linv_block[q][j]
      }
    } else if (nbelow > 0) {
      // (b) panel: row r of X solves X Ljj^T = A(r, block), one thread per row, in place
      if (tid < nbelow) {
        const int r = c0 + PB + tid;
        double x[PB];
#pragma unroll
        for (int m = 0; m < PB; m++) x[m] = a[r * LDP + c0 + m];
#pragma unroll
        for (int m = 0; m < PB; m++) {
          const double xm = x[m] * rdbuf[m];
          x[m] = xm;
#pragma unroll
          for (int q = m + 1; q < PB; q++) x[q] -= a[(c0 + q) * LDP + c0 + m] * xm;
        }
#pragma unroll
        for (int m = 0; m < PB; m++) a[r * LDP + c0 + m] = x[m];
      }
    }
    __syncthreads();   // (the last block column has no panel; warp 15 still finishes its inverse before the barrier)
    if (prof_fine && tid == 0) { const long long tt = clock64(); acc_b += tt - t_a; t_a = tt; }
    if (nbelow > 0) {
      // (c) trailing update A[r][c] -= sum_{m<16} L[r][c0+m] L[c][c0+m] for r >= c >= c0+16
      const int Sx = nbelow / 4, ntiles = Sx * (Sx + 1) / 2, base = c0 + PB;
      if (tid < POTRF_WORKERS)
        for (int u = tid; u < ntiles; u += POTRF_WORKERS) {
          int tr = (int)((sqrtf(8.0f * (float)u + 1.0f) - 1.0f) * 0.5f);
          while ((tr + 1) * (tr + 2) / 2 <= u) tr++;
          while (tr * (tr + 1) / 2 > u) tr--;
          const int tc = u - tr * (tr + 1) / 2;   // tc <= tr
          const double* P = a + (base + tr) * LDP + c0;
          const double* Q = a + (base + tc) * LDP + c0;
          double g[4][4];
#pragma unroll
          for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) g[i][j] = 0.0;
#pragma unroll 4
          for (int m = 0; m < PB; m++) {
            double pv[4], qv[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { pv[i] = P[i * Sx * LDP + m]; qv[i] = Q[i * Sx * LDP + m]; }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
              for (int j = 0; j < 4; j++) g[i][j] += pv[i] * qv[j];
          }
          // g[i][j] = <row tr+i*Sx, row tc+j*Sx>: canonical position is (larger row index, smaller row index)
#pragma unroll
          for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) {
              const int ri = base + tr + i * Sx, cj = base + tc + j * Sx;
              if (j <= i) a[ri * LDP + cj] -= g[i][j];
              else if (tr != tc) a[cj * LDP + ri] -= g[i][j];
            }
        }
      __syncthreads();
      if (prof_fine && tid == 0) acc_c += clock64() - t_a;
    }
  }
  POTRF_MARK(2);
  if (prof_fine && tid == 0) { prof[6] = acc_a; prof[7] = acc_ab; prof[8] = acc_b; prof[9] = acc_c; }
  for (int u = tid; u < T * T / 2; u += POTRF_THREADS) {
    const int r = u / (T / 2), c = (u % (T / 2)) * 2;
    if (c + 1 <= r)
      *reinterpret_cast<double2*>(At + (size_t)r * ld + c) = make_double2(a[r * LDP + c], a[r * LDP + c + 1]);
    else if (c <= r)
      At[(size_t)r * ld + c] = a[r * LDP + c];
  }
  __syncthreads();
  POTRF_MARK(3);
  // ---------------- inverse of L, in place ----------------
  // level 0: the diagonal 16x16 blocks were inverted during the factorisation
  for (int u = tid; u < (T / PB) * PB * PB; u += POTRF_THREADS) {
    const int blk = u / (PB * PB), r = (u / PB) % PB, c = u % PB;
    a[(blk * PB + r) * LDP + blk * PB + c] = binv[u];
  }
  __syncthreads();
  // levels h = 16, 32, 64: for each pair (A = inv at [p,p], C = inv at [p+h,p+h], B at [p+h,p]):
  //   tmp = B * A  (A lower triangular),  B <- -C * tmp  (C lower triangular).  A thread owns rows r0..r0+3 and the
  //   interleaved columns {ct + j*h/4}: lanes run along ct → conflict-free operand loads.
  for (int h = PB; h < T; h *= 2) {
    const int npairs = T / (2 * h), h4 = h / 4, ldt = h + 1;
    for (int u = tid; u < npairs * h4 * h4; u += POTRF_THREADS) {
      const int pr = u / (h4 * h4), r0 = 4 * ((u / h4) % h4), ct = u % h4;
      const int p0 = pr * 2 * h;
      double c4[4][4];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) c4[i][j] = 0.0;
      // (B A)[r][c] = sum_m B[r][m] A[m][c]; A[m][c] = 0 for m < c, the smallest column of the thread is ct
      const double* Bp = a + (p0 + h + r0) * LDP + p0;
      const double* Ap = a + p0 * LDP + p0 + ct;
      for (int m = ct; m < h; m++) {
        double bv[4], av[4];
#pragma unroll
        for (int i = 0; i < 4; i++) { bv[i] = Bp[i * LDP + m]; av[i] = Ap[m * LDP + i * h4]; }
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) c4[i][j] += bv[i] * av[j];
      }
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) tmp[pr * h * ldt + (r0 + i) * ldt + ct + j * h4] = c4[i][j];
    }
    __syncthreads();
    for (int u = tid; u < npairs * h4 * h4; u += POTRF_THREADS) {
      const int pr = u / (h4 * h4), r0 = 4 * ((u / h4) % h4), ct = u % h4;
      const int p0 = pr * 2 * h;
      double c4[4][4];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) c4[i][j] = 0.0;
      // (C tmp)[r][c] = sum_{m <= r} C[r][m] tmp[m][c]   (C[r][m] = 0 above the diagonal)
      const double* Cp = a + (p0 + h + r0) * LDP + p0 + h;
      const double* Tp = tmp + pr * h * ldt + ct;
      for (int m = 0; m < r0 + 4; m++) {
        double cv[4], tv[4];
#pragma unroll
        for (int i = 0; i < 4; i++) { cv[i] = Cp[i * LDP + m]; tv[i] = Tp[m * ldt + i * h4]; }
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) c4[i][j] += cv[i] * tv[j];
      }
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) a[(p0 + h + r0 + i) * LDP + p0 + ct + j * h4] = -c4[i][j];
    }
    __syncthreads();
  }
  POTRF_MARK(4);
  for (int u = tid; u < T * T / 2; u += POTRF_THREADS) {
    const int r = u / (T / 2), c = (u % (T / 2)) * 2;
    reinterpret_cast<double2*>(linv_k)[u] =
        make_double2((c <= r) ? a[r * LDP + c] : 0.0, (c + 1 <= r) ? a[r * LDP + c + 1] : 0.0);
  }
  POTRF_MARK(5);
}

// Triangular solves.  One launch per tile column; every CTA recomputes the tiny diagonal product (128x128 mat-vec with
// the stored tile inverse) and then updates its own off-diagonal tile.  512 threads, all loads of a mat-vec are issued
// before the first use (32 independent coalesced loads per thread) — these kernels are latency-, not bandwidth-bound.
constexpr int SOLVE_THREADS = 512;

// out[r] = sum_c A[r][c] x[c]   (A row-major 128x128 with leading dimension lda; lanes run along c)
__device__ __forceinline__ void matvec_rows(const double* __restrict__ A, size_t lda, const double* x, double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;   // 16 warps x 8 rows
  double v[8][4];
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) v[i][j] = A[(size_t)(warp * 8 + i) * lda + lane + 32 * j];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    double s = (v[i][0] * x[lane] + v[i][1] * x[lane + 32]) + (v[i][2] * x[lane + 64] + v[i][3] * x[lane + 96]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[warp * 8 + i] = s;
  }
}
// out[c] = sum_m A[m][c] x[m]   (threads run along c; 4 groups of 128 threads split m, partials combined in order)
__device__ __forceinline__ void matvec_cols(const double* __restrict__ A, size_t lda, const double* x, double* out,
                                            double* part /*[4][128]*/) {
  const int c = threadIdx.x & 127, g = threadIdx.x >> 7;
  double v[32];
#pragma unroll
  for (int i = 0; i < 32; i++) v[i] = A[(size_t)(g * 32 + i) * lda + c];
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 32; i++) s += v[i] * x[g * 32 + i];
  part[g * T + c] = s;
  __syncthreads();
  if (threadIdx.x < T) out[c] = (part[c] + part[T + c]) + (part[2 * T + c] + part[3 * T + c]);
  __syncthreads();
}

// forward step k: y_k = Linv_k b_k (written by CTA 0), b_i -= L(i,k) y_k for the non-zero row tiles i > k (rows[])
// `panel` = first row tile of column k (row tiles contiguous)
__global__ void __launch_bounds__(SOLVE_THREADS) fwd_kernel(const double* __restrict__ panel, int k,
                                                            const double* __restrict__ linv, double* __restrict__ b,
                                                            double* __restrict__ y, const int* __restrict__ rows) {
  constexpr size_t ld = T;
  __shared__ double bk[T], yk[T], upd[T];
  const int tid = threadIdx.x;
  if (tid < T) bk[tid] = b[(size_t)k * T + tid];
  __syncthreads();
  matvec_rows(linv + (size_t)k * T * T, T, bk, yk);   // Linv is stored with zeros above the diagonal
  __syncthreads();
  if (blockIdx.x == 0) {
    if (tid < T) y[(size_t)k * T + tid] = yk[tid];
    return;
  }
  const int i = rows[blockIdx.x - 1];
  matvec_rows(panel + (size_t)(blockIdx.x - 1) * TT, ld, yk, upd);
  __syncthreads();
  if (tid < T) b[(size_t)i * T + tid] -= upd[tid];
}

// backward step k: x_k = Linv_k^T y_k (CTA 0), y_i -= L(k,i)^T x_k for the non-zero column tiles i < k of row k (cols[])
__global__ void __launch_bounds__(SOLVE_THREADS) bwd_kernel(const double* __restrict__ L, const int* __restrict__ tile_of, int nt,
                                                            int k, const double* __restrict__ linv, double* __restrict__ y,
                                                            double* __restrict__ x, const int* __restrict__ cols) {
  constexpr size_t ld = T;
  __shared__ double ykk[T], xk[T], upd[T], part[4 * T];
  const int tid = threadIdx.x;
  if (tid < T) ykk[tid] = y[(size_t)k * T + tid];
  __syncthreads();
  matvec_cols(linv + (size_t)k * T * T, T, ykk, xk, part);
  if (blockIdx.x == 0) {
    if (tid < T) x[(size_t)k * T + tid] = xk[tid];
    return;
  }
  const int i = cols[blockIdx.x - 1];
  matvec_cols(L + (size_t)tile_of[(size_t)k * nt + i] * TT, ld, xk, upd, part);
  if (tid < T) y[(size_t)i * T + tid] -= upd[tid];
}

// Symbolic phase (host): tile-level structure of L from the tile-level structure of S (lower, nt x nt, row-major
// bools, diagonal forced).  Right-looking elimination: the non-zero rows of column k become a clique.
void TilePlan::build(int nt_, std::vector<uint8_t> mask, std::vector<int> col_group, const std::vector<int>* owner, int rank) {
  nt = nt_;
  my_rank = rank;
  h_col_group = std::move(col_group);
  h_owner.clear();
  if (owner) h_owner = *owner;
  const bool dist = !h_owner.empty();
  h_col_ptr.assign(1, 0); h_row_idx.clear();
  for (int k = 0; k < nt; k++) mask[(size_t)k * nt + k] = 1;
  // Distributed: the structure (fill) is the global one, but a rank executes only the updates of the columns it owns.
  double n_trsm = 0.0, n_upd = 0.0;
  for (int k = 0; k < nt; k++) {
    std::vector<int> rows;
    for (int i = k + 1; i < nt; i++)
      if (mask[(size_t)i * nt + k]) rows.push_back(i);
    if (!dist || h_owner[k] == rank) n_trsm += (double)rows.size();
    for (size_t a = 0; a < rows.size(); a++)
      for (size_t b = 0; b <= a; b++) {
        mask[(size_t)rows[a] * nt + rows[b]] = 1;
        if (!dist || h_owner[rows[b]] == rank) n_upd += 1.0;
      }
    h_row_idx.insert(h_row_idx.end(), rows.begin(), rows.end());
    h_col_ptr.push_back((int)h_row_idx.size());
  }
  // Blocks: runs of up to kPanelBlock consecutive main-sequence columns.  Width 1 for the column groups (pure latency
  // chains with tiny updates: nothing to amortise, and their updates stay off the bulk stream) and for the distributed
  // factorisation (its owner map, flags and peer copies hand over one column at a time).
  const auto in_group = [&](int k) { return !h_col_group.empty() && h_col_group[k] >= 0; };
  h_blk_end.assign(nt, 0);
  for (int k0 = 0; k0 < nt;) {
    int k1 = k0 + 1;
    if (!dist && !in_group(k0))
      while (k1 < nt && k1 - k0 < kPanelBlock && !in_group(k1)) k1++;
    for (int k = k0; k < k1; k++) h_blk_end[k] = k1;
    k0 = k1;
  }
  // Launch lists.  Per target column: the next block's columns go on the work stream (the first of them first: the next
  // panel solve needs it), the rest on the bulk stream; the column groups put all their updates on the work stream.
  h_pair_ptr.assign(1, 0); h_pair_i.clear(); h_pair_j.clear(); h_pair_mask.clear(); h_pair_k0.clear(); h_pair_split.clear();
  const auto tile = [&](int i, int j) { return mask[(size_t)i * nt + j] != 0; };
  for (int k = 0; k < nt; k++) {
    // panels [p_lo, k] onto the target columns [j_lo, nt) at a block's last column, panel k onto (k, k1) inside a block
    const int k1 = h_blk_end[k];
    const bool last = k1 == k + 1;
    int p_lo = k;
    if (last)
      while (p_lo > 0 && h_blk_end[p_lo - 1] == k1) p_lo--;
    const int j_lo = last ? k1 : k + 1, j_end = last ? nt : k1;
    const int j_work = in_group(k) ? nt : (last && k1 < nt ? h_blk_end[k1] : k1);   // target columns < j_work: work stream
    std::vector<int> rows;   // rows >= j_lo of the panels: the targets' rows and columns
    for (int p = p_lo; p <= k; p++)
      for (int q = h_col_ptr[p]; q < h_col_ptr[p + 1]; q++)
        if (h_row_idx[q] >= j_lo && h_row_idx[q] < nt) rows.push_back(h_row_idx[q]);
    std::sort(rows.begin(), rows.end());
    rows.erase(std::unique(rows.begin(), rows.end()), rows.end());
    int n_work = 0;
    for (size_t b = 0; b < rows.size(); b++) {   // target column j = rows[b] (ascending: the first work column first)
      const int j = rows[b];
      if (j >= j_end || (dist && h_owner[j] != rank)) continue;
      for (size_t a = b; a < rows.size(); a++) {
        const int i = rows[a];
        int m = 0;
        for (int p = p_lo; p <= k; p++)   // (p+1, p+1) with panel p is the chain's product
          if (tile(i, p) && tile(j, p) && !(i == p + 1 && j == p + 1)) m |= 1 << (p - p_lo);
        if (!m) continue;
        h_pair_i.push_back(i);
        h_pair_j.push_back(j);
        h_pair_mask.push_back(m);
        if (j < j_work) n_work++;
      }
    }
    h_pair_k0.push_back(p_lo);
    h_pair_split.push_back(n_work);
    h_pair_ptr.push_back((int)h_pair_i.size());
  }
  h_rowc_ptr.assign(1, 0); h_rowc_idx.clear();
  for (int k = 0; k < nt; k++) {
    for (int i = 0; i < k; i++)
      if (mask[(size_t)k * nt + i]) h_rowc_idx.push_back(i);
    h_rowc_ptr.push_back((int)h_rowc_idx.size());
  }
  n_tiles_L = (long)h_row_idx.size() + nt;
  // packed layout: column by column, diagonal tile first
  h_col_base.assign(nt, 0);
  h_tile_of.assign((size_t)nt * nt, -1);
  int next = 0;
  for (int k = 0; k < nt; k++) {
    h_col_base[k] = next;
    h_tile_of[(size_t)k * nt + k] = next++;
    for (int q = h_col_ptr[k]; q < h_col_ptr[k + 1]; q++) h_tile_of[(size_t)h_row_idx[q] * nt + k] = next++;
  }
  // flops this rank executes: one 128^3 GEMM (2 flop per MAC) per trsm tile and per (target tile, panel) update
  flops = 2.0 * T * T * T * (n_trsm + n_upd);
}

int TilePlan::upload(cvb_ctx* ctx, cudaStream_t st) {
  release();
  auto up = [&](int** d, const std::vector<int>& h) -> int {
    const size_t n = h.size() ? h.size() : 1;
    CVB_CUDA(ctx, cudaMalloc(d, n * sizeof(int)));
    if (h.size()) CVB_CUDA(ctx, cudaMemcpyAsync(*d, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    return CVB_OK;
  };
  int rc;
  if ((rc = up(&d_row_idx, h_row_idx)) || (rc = up(&d_pair_i, h_pair_i)) || (rc = up(&d_pair_j, h_pair_j)) ||
      (rc = up(&d_pair_mask, h_pair_mask)) || (rc = up(&d_rowc_idx, h_rowc_idx)) || (rc = up(&d_tile_of, h_tile_of)))
    return rc;
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  return CVB_OK;
}

void TilePlan::release() {
  if (d_row_idx) cudaFree(d_row_idx);
  if (d_pair_i) cudaFree(d_pair_i);
  if (d_pair_j) cudaFree(d_pair_j);
  if (d_pair_mask) cudaFree(d_pair_mask);
  if (d_rowc_idx) cudaFree(d_rowc_idx);
  if (d_tile_of) cudaFree(d_tile_of);
  d_row_idx = d_pair_i = d_pair_j = d_pair_mask = d_rowc_idx = d_tile_of = nullptr;
}

int FactorStreams::create(cvb_ctx* ctx, int nt) {
  int lo = 0, hi = 0;   // lo = numerically greatest = lowest priority
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  CVB_CUDA(ctx, cudaStreamCreateWithPriority(&bulk, cudaStreamNonBlocking, lo));
  ev.assign((size_t)5 * nt, nullptr);
  for (auto& e : ev) CVB_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  CVB_CUDA(ctx, cudaStreamCreateWithPriority(&fast, cudaStreamNonBlocking, hi));
  CVB_CUDA(ctx, cudaEventCreateWithFlags(&fork_fast, cudaEventDisableTiming));
  for (int g = 0; g < n_group; g++) {
    CVB_CUDA(ctx, cudaStreamCreateWithPriority(&group_aux[g], cudaStreamNonBlocking, hi));
    CVB_CUDA(ctx, cudaEventCreateWithFlags(&join_aux[g], cudaEventDisableTiming));
  }
  for (int g = 0; g < n_group; g++) {
    CVB_CUDA(ctx, cudaStreamCreateWithPriority(&group[g], cudaStreamNonBlocking, hi));
    CVB_CUDA(ctx, cudaEventCreateWithFlags(&join[g], cudaEventDisableTiming));
  }
  CVB_CUDA(ctx, cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
  return CVB_OK;
}

void FactorStreams::destroy() {
  for (auto& e : ev) if (e) cudaEventDestroy(e);
  ev.clear();
  if (bulk) cudaStreamDestroy(bulk);
  if (fast) cudaStreamDestroy(fast);
  if (fork_fast) cudaEventDestroy(fork_fast);
  for (int g = 0; g < n_group; g++) {
    if (group_aux[g]) cudaStreamDestroy(group_aux[g]);
    if (join_aux[g]) cudaEventDestroy(join_aux[g]);
    if (group[g]) cudaStreamDestroy(group[g]);
    if (join[g]) cudaEventDestroy(join[g]);
    group_aux[g] = group[g] = nullptr;
    join_aux[g] = join[g] = nullptr;
  }
  if (fork) cudaEventDestroy(fork);
  bulk = fast = nullptr;
  fork_fast = fork = nullptr;
}

// ---- cross-GPU hand-over of a finished panel (distributed factorisation) -------------------------------------------
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__global__ void bump_epoch_kernel(int* epoch) { *epoch += 1; }
// owner: all writes of the preceding kernels on this stream (the panel, the tile inverse) are ordered before the
// system-scope release store of the flag into every peer's memory (NVLink store)
__global__ void signal_panel_kernel(int* const* __restrict__ peer_flag, int k, const int* __restrict__ epoch, int world, int rank) {
  const int g = threadIdx.x;
  if (g < world && g != rank) {
    __threadfence_system();
    st_release_sys(peer_flag[g] + k, *epoch);
  }
}
// peer: spin on the LOCAL flag (one thread, one CTA: nothing else of this GPU is held up)
// A peer that never signals (crashed rank) must not wedge this GPU: after kWaitPanelNs the factorisation is flagged failed.
constexpr unsigned long long kWaitPanelNs = 20ull * 1000 * 1000 * 1000;
__global__ void wait_panel_kernel(const int* __restrict__ flag, const int* __restrict__ epoch, int* __restrict__ fail) {
  const int e = *epoch;
  unsigned long long t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  while (ld_acquire_sys(flag) < e) {
    __nanosleep(200);
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (t - t0 > kWaitPanelNs) { atomicExch(fail, 1); return; }
  }
}

int factor(cvb_ctx* ctx, double* S, double* linv, int* d_flag, const TilePlan& plan, cudaStream_t st,
           const FactorStreams& fs, const DistView* dv) {
  static cvb_once_per_device once;
  if (once.first(ctx->device)) {
    CVB_CUDA(ctx, cudaFuncSetAttribute(trsm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrsmSmem));
    CVB_CUDA(ctx, cudaFuncSetAttribute(syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSyrkSmem));
    CVB_CUDA(ctx, cudaFuncSetAttribute(tile_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTileSmem));
    CVB_CUDA(ctx, cudaFuncSetAttribute(potrf_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPotrfSmem));
    CVB_CUDA(ctx, cudaFuncSetAttribute(chain_gemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kChainSmem));
    CVB_CUDA(ctx, cudaFuncSetAttribute(chain_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kChainSmem));
  }
  const int nt = plan.nt;
  const bool dist = dv != nullptr && dv->world > 1 && !plan.h_owner.empty();
  CVB_REQUIRE(ctx, plan.d_tile_of != nullptr && (int)plan.h_col_base.size() == nt, "tile plan not built / uploaded");
  CVB_REQUIRE(ctx, fs.ev.size() >= (size_t)5 * nt, "factor streams not created for this plan");
  CVB_CUDA(ctx, cudaMemsetAsync(d_flag, 0, sizeof(int), st));
  if (dist) {
    bump_epoch_kernel<<<1, 1, 0, st>>>(dv->d_epoch);
    CVB_CHECK_LAUNCH(ctx);
  }
  cudaStream_t st2 = fs.bulk;
  const std::vector<cudaEvent_t>& ev = fs.ev;
  const int n_gs = plan.h_col_group.empty() ? 0 : fs.n_group;
  // Blocked trailing update (TilePlan::h_blk_end): inside a block of kPanelBlock main-sequence columns each panel updates
  // only the block's own columns; after the block's last panel one pass applies all of its panels to every tile past the
  // block.  Lookahead (depth 1 block): the next block's steps only need the part of that pass on the next block's columns
  // (the work stream; the first of them first); the bulk of the pass runs on the second (low-priority) stream
  // concurrently.  The bulk writes the tiles past the next block only, so the one thing that waits for it is the first
  // use of those tiles: the next block's own pass and its last chain step.  ev[5k] = panel of step k available,
  // ev[5k+1] = bulk update of step k done.
  // Independent column groups (the IMU chains of different agents, see TilePlan::h_col_group) run on their own
  // streams: their tile columns are pure latency chains (diagonal tile → panel → tiny update) that do not share tiles.
  // Distributed: "panel available" = factored here (owner) or pulled from the owner's memory (everyone else).
  // Development trace (COVINS_B200_FACTOR_TRACE=<csv path>): per-column timeline of the first non-captured call.
  static bool traced = false;
  const char* trace_path = getenv("COVINS_B200_FACTOR_TRACE");
  cudaStreamCaptureStatus cap_status = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cap_status);
  const bool tr = trace_path && !traced && cap_status == cudaStreamCaptureStatusNone;
  std::vector<cudaEvent_t> tev;
  if (tr) {
    traced = true;
    tev.resize((size_t)nt * 5 + 1);
    for (auto& e : tev) cudaEventCreate(&e);
    cudaEventRecord(tev[(size_t)nt * 5], st);
  }
  int last_bulk = -1;
  bool forked = false;
  std::vector<char> used(n_gs > 0 ? n_gs : 1, 0);
  // Critical-chain stream (fs.fast, highest priority).  Step k+1's diagonal tile needs from step k only ONE tile of the
  // panel, L(k+1,k), and ONE update, S(k+1,k+1) -= L(k+1,k) L(k+1,k)^T.  So the chain
  //     potrf(k) -> solve tile (k+1,k) -> update tile (k+1,k+1) -> potrf(k+1) -> ...
  // runs on its own stream while the rest of panel k (main stream) and the rest of its updates (main: tile column k+1,
  // bulk stream: everything else) proceed beside it.  Distributed, the hand-over to the next column's owner moves one
  // 128 KB tile (flag A) instead of waiting for the whole panel (flag B).
  cudaStream_t sf = fs.fast;
  bool sf_live = false;          // sf has been forked off the main stream
  int prev_chain = -1;           // previous column handled by the chain (its evA is what step C waits for)
  // The column groups (IMU chains) are pure chains: the same split with the group's stream as the chain stream and a second
  // stream per group for the rest of the panel and all of its (small) updates.
  int prev_chain_g[FactorStreams::n_group] = {-1, -1, -1, -1, -1, -1, -1, -1};
  int rc_join = 0;
  auto join_groups = [&]() -> int {
    for (int g = 0; g < n_gs; g++)
      if (used[g]) {
        CVB_CUDA(ctx, cudaEventRecord(fs.join_aux[g], fs.group_aux[g]));
        CVB_CUDA(ctx, cudaStreamWaitEvent(fs.group[g], fs.join_aux[g], 0));
        CVB_CUDA(ctx, cudaEventRecord(fs.join[g], fs.group[g]));
        CVB_CUDA(ctx, cudaStreamWaitEvent(st, fs.join[g], 0));
        used[g] = 0;
      }
    return CVB_OK;
  };
  for (int k = 0; k < nt; k++) {
    const int grp = n_gs > 0 ? plan.h_col_group[k] : -1;
    cudaStream_t s = st;
    if (grp >= 0) {
      if (!forked) {
        CVB_CUDA(ctx, cudaEventRecord(fs.fork, st));
        forked = true;
      }
      s = fs.group[grp % n_gs];
      if (!used[grp % n_gs]) {
        CVB_CUDA(ctx, cudaStreamWaitEvent(s, fs.fork, 0));
        CVB_CUDA(ctx, cudaStreamWaitEvent(fs.group_aux[grp % n_gs], fs.fork, 0));
        used[grp % n_gs] = 1;
      }
    } else if (forked) {   // first column after the grouped ones: join
      if ((rc_join = join_groups())) return rc_join;
      forked = false;
    }
    if (tr) cudaEventRecord(tev[(size_t)k * 5 + 0], s);
    const int m = plan.h_col_ptr[k + 1] - plan.h_col_ptr[k];
    double* diag = S + (size_t)plan.h_col_base[k] * TT;
    double* linv_k = linv + (size_t)k * TT;
    const bool mine = !dist || plan.h_owner[k] == dv->rank;
    const int p0 = plan.h_pair_ptr[k], np = plan.h_pair_ptr[k + 1] - p0;
    // ------------------------------------ chain column ------------------------------------
    cudaEvent_t evPanel = ev[5 * k], evBulk = ev[5 * k + 1], evP = ev[5 * k + 2], evD = ev[5 * k + 3], evA = ev[5 * k + 4];
    const bool is_grp = grp >= 0;
    const int gi = is_grp ? grp % n_gs : 0;
    if (!is_grp && !sf_live) {   // everything before this column (the column groups) is on the main stream
      CVB_CUDA(ctx, cudaEventRecord(fs.fork_fast, st));
      CVB_CUDA(ctx, cudaStreamWaitEvent(sf, fs.fork_fast, 0));
      sf_live = true;
    }
    cudaStream_t cs = is_grp ? fs.group[gi] : sf;        // chain stream of this column
    cudaStream_t ws = is_grp ? fs.group_aux[gi] : st;    // its work stream (rest of the panel, tile column k+1)
    int& pc = is_grp ? prev_chain_g[gi] : prev_chain;     // previous chain column of this sequence
    // the bulk is waited for at a block's last column only (column groups have no bulk stream: all their updates are small)
    const bool blk_last = plan.h_blk_end[k] == k + 1;
    const int lb = is_grp || !blk_last ? -1 : last_bulk;
    const bool has_next = m > 0 && plan.h_row_idx[plan.h_col_ptr[k]] == k + 1;
    // tile (k+1,k+1) gets panel k from the chain when this rank applies the updates of column k+1
    const bool mine_n = has_next && (!dist || plan.h_owner[k + 1] == dv->rank);
    const int na = plan.h_pair_split[k];
    const int k0 = plan.h_pair_k0[k];
    // a list that starts with (k+1,k+1) (at a block's last column) holds the block's earlier panels for it: they go on the
    // chain stream, before the chain's own product and potrf(k+1)
    const bool diag_pair = np > 0 && plan.h_pair_i[p0] == k + 1 && plan.h_pair_j[p0] == k + 1;
    // A. tile (k,k) is final: column k-1's contribution came with the chain, the others were waited for by the previous
    //    chain step (below) — nothing to wait for here
    if (mine) {
      potrf_inv_kernel<<<1, POTRF_THREADS, kPotrfSmem, cs>>>(diag, (size_t)T, 0, linv_k, d_flag, nullptr, 0);
      CVB_CHECK_LAUNCH(ctx);
    }
    CVB_CUDA(ctx, cudaEventRecord(evP, cs));
    if (tr) cudaEventRecord(tev[(size_t)k * 5 + 1], cs);
    // C. tile (k+1,k): final once column k-1's updates of tile column k are done (evA of the previous chain column).
    //    Inside a block the work stream also updates tile (k+1,k+1) (panels before k): the same wait orders potrf(k+1)
    //    after those.
    if (pc >= 0) CVB_CUDA(ctx, cudaStreamWaitEvent(cs, ev[5 * pc + 4], 0));
    if (has_next) {
      if (mine) {
        chain_gemm_kernel<0><<<T / CHAIN_ROWS, T, kChainSmem, cs>>>(diag + TT, diag + TT, linv_k);
        CVB_CHECK_LAUNCH(ctx);
        if (dist && !is_grp) {     // (a column group stays on one rank: nobody waits for its flag A)
          signal_panel_kernel<<<1, 32, 0, cs>>>(dv->d_peer_flag, k, dv->d_epoch, dv->world, dv->rank);          // flag A
          CVB_CHECK_LAUNCH(ctx);
        }
      } else if (mine_n) {
        wait_panel_kernel<<<1, 1, 0, cs>>>(dv->peer_flag[dv->rank] + k, dv->d_epoch, d_flag);
        CVB_CHECK_LAUNCH(ctx);
        CVB_CUDA(ctx, cudaMemcpyAsync(diag + TT, dv->peer_S[plan.h_owner[k]] + ((size_t)plan.h_col_base[k] + 1) * TT, TT * sizeof(double),
                                      cudaMemcpyDeviceToDevice, cs));
      }
    }
    // at a block's last column, the previous block's bulk update also writes tile (k+1,k+1) (and everything the next
    // chain step reads): it has to be complete before the diagonal pair is applied / before potrf(k+1) — the depth-1
    // lookahead rule
    if (lb >= 0) CVB_CUDA(ctx, cudaStreamWaitEvent(cs, ev[5 * lb + 1], 0));
    if (diag_pair) {
      syrk_kernel<<<4, SYRK_THREADS, kSyrkSmem, cs>>>(S, plan.d_tile_of, nt, k0, plan.d_pair_i + p0, plan.d_pair_j + p0,
                                                       plan.d_pair_mask + p0);
      CVB_CHECK_LAUNCH(ctx);
    }
    if (mine_n) {
      chain_gemm_kernel<1><<<T / CHAIN_ROWS, T, kChainSmem, cs>>>(S + (size_t)plan.h_col_base[k + 1] * TT, diag + TT, diag + TT);
      CVB_CHECK_LAUNCH(ctx);
    }
    CVB_CUDA(ctx, cudaEventRecord(evD, cs));
    if (tr) cudaEventRecord(tev[(size_t)k * 5 + 2], cs);
    // D. the rest of the panel on the work stream
    const bool early_tile = has_next && (mine || mine_n);     // tile (k+1,k) was produced / fetched by the chain
    if (mine) {
      CVB_CUDA(ctx, cudaStreamWaitEvent(ws, evP, 0));
      const int first = has_next ? 1 : 0;
      if (m - first > 0) {
        trsm_kernel<<<2 * (m - first), TRSM_THREADS, kTrsmSmem, ws>>>(diag + (size_t)(1 + first) * TT, linv_k);
        CVB_CHECK_LAUNCH(ctx);
      }
      CVB_CUDA(ctx, cudaStreamWaitEvent(ws, evD, 0));
      if (dist) {
        signal_panel_kernel<<<1, 32, 0, ws>>>(dv->d_peer_flag, nt + k, dv->d_epoch, dv->world, dv->rank);       // flag B
        CVB_CHECK_LAUNCH(ctx);
      }
    } else {
      const int o = plan.h_owner[k];
      wait_panel_kernel<<<1, 1, 0, ws>>>(dv->peer_flag[dv->rank] + nt + k, dv->d_epoch, d_flag);
      CVB_CHECK_LAUNCH(ctx);
      const double* src = dv->peer_S[o] + (size_t)plan.h_col_base[k] * TT;
      if (early_tile) {   // the chain owns tile (k+1,k): copy around it
        CVB_CUDA(ctx, cudaMemcpyAsync(diag, src, TT * sizeof(double), cudaMemcpyDeviceToDevice, ws));
        if (m > 1) CVB_CUDA(ctx, cudaMemcpyAsync(diag + 2 * (size_t)TT, src + 2 * (size_t)TT, (size_t)(m - 1) * TT * sizeof(double), cudaMemcpyDeviceToDevice, ws));
      } else {
        CVB_CUDA(ctx, cudaMemcpyAsync(diag, src, (size_t)(1 + m) * TT * sizeof(double), cudaMemcpyDeviceToDevice, ws));
      }
      CVB_CUDA(ctx, cudaMemcpyAsync(linv_k, dv->peer_linv[o] + (size_t)k * TT, TT * sizeof(double), cudaMemcpyDeviceToDevice, ws));
      CVB_CUDA(ctx, cudaStreamWaitEvent(ws, evD, 0));
    }
    // E. the work stream's part of the update list (the next block's columns, minus the diagonal pair), then "panel k
    //    available" for the bulk stream.  (At a block's last column the list holds all of the block's panels, so it can
    //    be non-empty for a column without rows.)
    if (np > 0) {
      CVB_CUDA(ctx, cudaEventRecord(evPanel, ws));
      if (lb >= 0) CVB_CUDA(ctx, cudaStreamWaitEvent(ws, ev[5 * lb + 1], 0));
      const int a0 = diag_pair ? 1 : 0;
      if (na - a0 > 0) {
        tile_update_kernel<<<na - a0, TILE_THREADS, kTileSmem, ws>>>(S, plan.d_tile_of, nt, k0, plan.d_pair_i + p0 + a0,
                                                                     plan.d_pair_j + p0 + a0, plan.d_pair_mask + p0 + a0);
        CVB_CHECK_LAUNCH(ctx);
      }
      if (tr) cudaEventRecord(tev[(size_t)k * 5 + 3], ws);
      if (np - na > 0) {
        CVB_CUDA(ctx, cudaStreamWaitEvent(st2, evPanel, 0));
        tile_update_kernel<<<np - na, TILE_THREADS, kTileSmem, st2>>>(S, plan.d_tile_of, nt, k0, plan.d_pair_i + p0 + na,
                                                                       plan.d_pair_j + p0 + na, plan.d_pair_mask + p0 + na);
        CVB_CHECK_LAUNCH(ctx);
        CVB_CUDA(ctx, cudaEventRecord(evBulk, st2));
        if (tr) cudaEventRecord(tev[(size_t)k * 5 + 4], st2);
        last_bulk = k;
      }
    }
    CVB_CUDA(ctx, cudaEventRecord(evA, ws));
    pc = k;
  }
  if (sf_live) {   // join the chain stream
    CVB_CUDA(ctx, cudaEventRecord(fs.fork_fast, sf));
    CVB_CUDA(ctx, cudaStreamWaitEvent(st, fs.fork_fast, 0));
  }
  if (forked && (rc_join = join_groups())) return rc_join;
  if (last_bulk >= 0) CVB_CUDA(ctx, cudaStreamWaitEvent(st, ev[5 * last_bulk + 1], 0));   // join
  if (tr) {
    cudaStreamSynchronize(st);
    FILE* f = fopen(trace_path, "w");
    if (f) {
      // n_pairs / n_work_pairs: pairs of column k's update list / of its work-stream part; t_bulk_us: end of the bulk
      // update launched at column k (a block's last column), -1 if none
      fprintf(f, "k,group,owner,n_rows,n_pairs,n_work_pairs,t_start_us,t_panel_ready_us,t_trsm_us,t_syrk_a_us,t_bulk_us\n");
      for (int k = 0; k < nt; k++) {
        float t[5];
        for (int e = 0; e < 5; e++) {
          t[e] = -1.f;
          if (cudaEventQuery(tev[(size_t)k * 5 + e]) == cudaSuccess) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, tev[(size_t)nt * 5], tev[(size_t)k * 5 + e]) == cudaSuccess) t[e] = ms * 1e3f;
          }
        }
        fprintf(f, "%d,%d,%d,%d,%d,%d,%.1f,%.1f,%.1f,%.1f,%.1f\n", k, plan.h_col_group.empty() ? -1 : plan.h_col_group[k],
                plan.h_owner.empty() ? 0 : plan.h_owner[k], plan.h_col_ptr[k + 1] - plan.h_col_ptr[k],
                plan.h_pair_ptr[k + 1] - plan.h_pair_ptr[k], plan.h_pair_split[k], t[0], t[1], t[2], t[3], t[4]);
      }
      fclose(f);
    }
    for (auto& e : tev) cudaEventDestroy(e);
    cudaGetLastError();   // queries of never-recorded events leave a sticky-looking error code behind
  }
  return CVB_OK;
}

// solves L L^T x = b; b is destroyed, tmp is scratch (n_pad), result in x
int solve(cvb_ctx* ctx, const double* L, const double* linv, double* b, double* tmp, double* x,
          const TilePlan& plan, cudaStream_t st, const FactorStreams& fs) {
  const int nt = plan.nt;
  // The leading tile columns that belong to independent column groups (IMU chains, TilePlan::h_col_group) touch only
  // their own chain's rows of b / y, so the chains' substitution steps — pure launch-latency chains — run concurrently
  // on the group streams, forward before and backward after the sequential part.
  const int n_gs = plan.h_col_group.empty() ? 0 : fs.n_group;
  int n_grouped = 0;
  while (n_gs > 0 && n_grouped < nt && plan.h_col_group[n_grouped] >= 0) n_grouped++;
  for (int k = n_grouped; k < nt; k++)
    if (n_gs > 0 && plan.h_col_group[k] >= 0) { n_grouped = 0; break; }   // groups must be a prefix; else run sequentially
  std::vector<char> used(n_gs > 0 ? n_gs : 1, 0);
  auto fork = [&]() -> int {
    CVB_CUDA(ctx, cudaEventRecord(fs.fork, st));
    std::fill(used.begin(), used.end(), 0);
    return CVB_OK;
  };
  auto stream_of = [&](int k, cudaStream_t* s) -> int {
    const int g = plan.h_col_group[k] % n_gs;
    if (!used[g]) {
      CVB_CUDA(ctx, cudaStreamWaitEvent(fs.group[g], fs.fork, 0));
      used[g] = 1;
    }
    *s = fs.group[g];
    return CVB_OK;
  };
  auto join = [&]() -> int {
    for (int g = 0; g < n_gs; g++)
      if (used[g]) {
        CVB_CUDA(ctx, cudaEventRecord(fs.join[g], fs.group[g]));
        CVB_CUDA(ctx, cudaStreamWaitEvent(st, fs.join[g], 0));
      }
    return CVB_OK;
  };
  int rc;
  if (n_grouped > 0 && (rc = fork())) return rc;
  for (int k = 0; k < nt; k++) {
    cudaStream_t s = st;
    if (k < n_grouped && (rc = stream_of(k, &s))) return rc;
    if (k == n_grouped && n_grouped > 0 && (rc = join())) return rc;
    const int m = plan.h_col_ptr[k + 1] - plan.h_col_ptr[k];
    fwd_kernel<<<1 + m, SOLVE_THREADS, 0, s>>>(L + (size_t)(plan.h_col_base[k] + 1) * TT, k, linv, b, tmp,
                                               plan.d_row_idx + plan.h_col_ptr[k]);
    CVB_CHECK_LAUNCH(ctx);
  }
  if (n_grouped == nt && n_grouped > 0 && (rc = join())) return rc;
  for (int k = nt - 1; k >= 0; k--) {
    cudaStream_t s = st;
    if (k == n_grouped - 1 && (rc = fork())) return rc;
    if (k < n_grouped && (rc = stream_of(k, &s))) return rc;
    const int m = plan.h_rowc_ptr[k + 1] - plan.h_rowc_ptr[k];
    bwd_kernel<<<1 + m, SOLVE_THREADS, 0, s>>>(L, plan.d_tile_of, nt, k, linv, tmp, x, plan.d_rowc_idx + plan.h_rowc_ptr[k]);
    CVB_CHECK_LAUNCH(ctx);
  }
  if (n_grouped > 0 && (rc = join())) return rc;
  return CVB_OK;
}

}  // namespace cvb_chol

// ---- test/diagnostic entry: solve A x = b for a host SPD matrix (row-major n x n) with the BA factorisation ----
// Latency of the diagonal-tile kernel (the serial chain of the tiled factorisation): factors `reps` copies of a synthetic
// SPD tile back to back; us_per_tile = average launch-to-launch time; phase_cycles[0..5] = clock64 marks of the last
// launch relative to its start (loaded, factored, L stored, inverted, Linv stored); summed over the 8 block columns:
// [6] = inside the 16x16 diagonal-block step, [7] = the same incl. the closing barrier, [8] = panel, [9] = trailing update.
extern "C" int cvb_microbench_potrf(cvb_ctx* ctx, int reps, double* us_per_tile, int64_t* phase_cycles) {
  if (!ctx || reps < 1 || !us_per_tile) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  using namespace cvb_chol;
  CVB_CUDA(ctx, cudaFuncSetAttribute(potrf_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPotrfSmem));
  const int nt = 8;
  std::vector<double> h((size_t)nt * T * T);
  for (int t = 0; t < nt; t++)
    for (int r = 0; r < T; r++)
      for (int c = 0; c < T; c++)
        h[((size_t)t * T + r) * T + c] = (r == c ? 4.0 + 0.01 * t : 0.0) + 1.0 / (1.0 + (r > c ? r - c : c - r));
  double *d_a = nullptr, *d_w = nullptr, *d_inv = nullptr;
  int* d_flag = nullptr;
  long long* d_prof = nullptr;
  CVB_CUDA(ctx, cudaMalloc(&d_a, h.size() * 8));
  CVB_CUDA(ctx, cudaMalloc(&d_w, h.size() * 8));
  CVB_CUDA(ctx, cudaMalloc(&d_inv, h.size() * 8));
  CVB_CUDA(ctx, cudaMalloc(&d_flag, 4));
  CVB_CUDA(ctx, cudaMalloc(&d_prof, 16 * sizeof(long long)));
  CVB_CUDA(ctx, cudaMemcpy(d_a, h.data(), h.size() * 8, cudaMemcpyHostToDevice));
  CVB_CUDA(ctx, cudaMemset(d_flag, 0, 4));
  cudaStream_t st = ctx->stream;
  cudaEvent_t e0, e1;
  CVB_CUDA(ctx, cudaEventCreate(&e0));
  CVB_CUDA(ctx, cudaEventCreate(&e1));
  float ms = 0.f;
  for (int pass = 0; pass < 2; pass++) {   // pass 0 = warm-up
    CVB_CUDA(ctx, cudaMemcpyAsync(d_w, d_a, h.size() * 8, cudaMemcpyDeviceToDevice, st));
    const int n = pass == 0 ? nt : reps;
    CVB_CUDA(ctx, cudaEventRecord(e0, st));
    for (int i = 0; i < n; i++) {
      if (i % nt == 0 && i) CVB_CUDA(ctx, cudaMemcpyAsync(d_w, d_a, h.size() * 8, cudaMemcpyDeviceToDevice, st));
      // each tile is its own 128 x 128 matrix (ld = T, k = 0)
      potrf_inv_kernel<<<1, POTRF_THREADS, kPotrfSmem, st>>>(d_w + (size_t)(i % nt) * T * T, (size_t)T, 0,
                                                             d_inv + (size_t)(i % nt) * T * T, d_flag, nullptr, 0);
      CVB_CHECK_LAUNCH(ctx);
    }
    CVB_CUDA(ctx, cudaEventRecord(e1, st));
    CVB_CUDA(ctx, cudaStreamSynchronize(st));
    CVB_CUDA(ctx, cudaEventElapsedTime(&ms, e0, e1));
  }
  *us_per_tile = (double)ms * 1e3 / reps;
  if (phase_cycles) {
    long long hp[16], hq[16];
    for (int fine = 0; fine < 2; fine++) {
      for (int rep = 0; rep < 4; rep++) {   // the last (warm instruction cache) launch is reported
        CVB_CUDA(ctx, cudaMemcpyAsync(d_w, d_a, (size_t)T * T * 8, cudaMemcpyDeviceToDevice, st));
        CVB_CUDA(ctx, cudaMemsetAsync(d_prof, 0, 16 * sizeof(long long), st));
        potrf_inv_kernel<<<1, POTRF_THREADS, kPotrfSmem, st>>>(d_w, (size_t)T, 0, d_inv, d_flag, d_prof, fine);
        CVB_CHECK_LAUNCH(ctx);
      }
      CVB_CUDA(ctx, cudaMemcpyAsync(fine ? hq : hp, d_prof, sizeof(hp), cudaMemcpyDeviceToHost, st));
      CVB_CUDA(ctx, cudaStreamSynchronize(st));
    }
    for (int i = 6; i < 10; i++) hp[i] = hq[i];   // marks from the coarse run, in-loop sums from the fine run
    for (int i = 0; i < 6; i++) phase_cycles[i] = (int64_t)(hp[i] - hp[0]);
    for (int i = 6; i < 10; i++) phase_cycles[i] = (int64_t)hp[i];
  }
  int hflag = 0;
  CVB_CUDA(ctx, cudaMemcpy(&hflag, d_flag, 4, cudaMemcpyDeviceToHost));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(d_a); cudaFree(d_w); cudaFree(d_inv); cudaFree(d_flag); cudaFree(d_prof);
  if (hflag) return cvb_fail(ctx, CVB_ERR_NUMERIC, "microbench tile not positive definite");
  return CVB_OK;
}

extern "C" int cvb_dense_cholesky_solve(cvb_ctx* ctx, const double* A, int n, const double* b, double* x,
                                        double* factor_ms) {
  if (!ctx || !A || !b || !x || n <= 0) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  using namespace cvb_chol;
  const int np = ((n + T - 1) / T) * T;
  cudaStream_t st = ctx->stream;
  const int nt = np / T;
  // tile structure of the input (zero tiles are skipped) → symbolic fill → packed tiles
  std::vector<uint8_t> mask((size_t)nt * nt, 0);
  for (int i = 0; i < n; i++)
    for (int j = 0; j <= i; j++)
      if (A[(size_t)i * n + j] != 0.0) mask[(size_t)(i / T) * nt + (j / T)] = 1;
  TilePlan plan;
  plan.build(nt, mask);
  std::vector<double> hs((size_t)plan.n_tiles_L * TT, 0.0), hb(np, 0.0);
  for (int i = 0; i < n; i++)
    for (int j = 0; j <= i; j++)
      if (A[(size_t)i * n + j] != 0.0) hs[plan.tile_index(i / T, j / T) * TT + (size_t)(i % T) * T + (j % T)] = A[(size_t)i * n + j];
  for (int i = n; i < np; i++) hs[plan.tile_index(i / T, i / T) * TT + (size_t)(i % T) * T + (i % T)] = 1.0;
  for (int i = 0; i < n; i++) hb[i] = b[i];
  double* dS = (double*)cvb_ws(ctx, WS_T, hs.size() * sizeof(double));
  double* dl = (double*)cvb_ws(ctx, WS_Q, (size_t)np * T * sizeof(double));
  double* dv = (double*)cvb_ws(ctx, WS_OUT0, (size_t)np * 3 * sizeof(double));
  int* dflag = (int*)cvb_ws(ctx, WS_FLAG, 16);
  if (!dS || !dl || !dv || !dflag) return CVB_ERR_CUDA;
  CVB_CUDA(ctx, cudaMemcpyAsync(dS, hs.data(), hs.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  CVB_CUDA(ctx, cudaMemcpyAsync(dv, hb.data(), np * sizeof(double), cudaMemcpyHostToDevice, st));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  int rc = plan.upload(ctx, st);
  if (rc) return rc;
  FactorStreams fs;
  if ((rc = fs.create(ctx, nt))) return rc;
  cudaEventRecord(e0, st);
  rc = factor(ctx, dS, dl, dflag, plan, st, fs);
  cudaEventRecord(e1, st);
  if (rc) return rc;
  rc = solve(ctx, dS, dl, dv, dv + np, dv + 2 * np, plan, st, fs);
  if (rc) return rc;
  int flag = 0;
  CVB_CUDA(ctx, cudaMemcpyAsync(&flag, dflag, sizeof(int), cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaMemcpyAsync(hb.data(), dv + 2 * np, np * sizeof(double), cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (factor_ms) *factor_ms = ms;
  plan.release();
  if (flag) return cvb_fail(ctx, CVB_ERR_NUMERIC, "matrix is not positive definite");
  for (int i = 0; i < n; i++) x[i] = hb[i];
  return CVB_OK;
}
