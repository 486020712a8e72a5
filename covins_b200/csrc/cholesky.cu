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
// Solves use the stored tile inverses: forward L y = b, backward L^T x = y, one persistent launch per direction.
// All reductions have a fixed order → bit-reproducible run to run.
#include "cholesky.cuh"

#include <stdlib.h>

#include <algorithm>
#include <map>

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

// acc(64 x BN) = A(64 x T) * B(BN x T)^T, both operands row-major with K contiguous (leading dims lda, ldb); with
// FROM_ACC the product is accumulated onto acc as it stands, K chunk by K chunk in increasing order.
// 2 x BN/32 warps, 32x32 per warp = 2 (m16) x 4 (n8) m16n8k16 blocks, acc[i][j] = rows 16 i.., columns 8 j.. of the warp
// tile in the C-fragment order of dmma16816.  m16n8k16 is Hopper's full-rate FP64 MMA shape: on an H100 SXM (400 W limit)
// a register-only probe sustained 64 TFLOP/s with it (~128 FMA/clk/SM) and 34 TFLOP/s with the Ampere m8n8k4 shape, and
// its results were bit-identical to four chained m8n8k4 over the same 16-wide K chunk.  K is staged in chunks of 16 (one
// MMA per block and chunk) through a STAGES-deep cp.async ring (one barrier per chunk).  Row stride 20 doubles (≡ 8 words
// mod 32): the fragment loads of a half-warp (rows g = 0..3, columns t = 0..3) hit words 8g + 2t, conflict-free.  The CTA
// is deliberately small (64 x 64 x 128 for syrk_kernel: 128 threads, 60 KB): three to four CTAs share an SM, so one CTA's
// fixed costs — index fetch, pipeline fill, the C load and store, barrier bubbles — overlap the others' main loops.  The
// throughput path of the trailing update (tile_update_kernel) takes the whole 128x128 tile per CTA instead: it halves
// the operand bytes per FMA.
constexpr int KC = 16;
constexpr int LDS = KC + 4;
constexpr int GEMM_STAGES = 3;

template <int BN, bool FROM_ACC = false>
__device__ __forceinline__ void gemm_abt_64(const double* __restrict__ A, size_t lda, const double* __restrict__ B,
                                            size_t ldb, double (&acc)[2][4][4], double* smem) {
  constexpr int WN = BN / 32, THREADS = 2 * WN * 32, STAGE = (64 + BN) * LDS, NCH = T / KC, UPR = KC / 2;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp / WN, wn = warp % WN;
  if (!FROM_ACC)
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
__device__ __forceinline__ void trsm_tile(double* __restrict__ tile, const double* __restrict__ linv_k) {
  extern __shared__ __align__(16) double smem_d[];
  constexpr size_t ld = T;
  const int half = blockIdx.x & 1;
  double* At = tile + (size_t)half * 64 * T;
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
__global__ void __launch_bounds__(TRSM_THREADS, 2) trsm_kernel(double* __restrict__ panel,
                                                                const double* __restrict__ linv_k) {
  trsm_tile(panel + (size_t)(blockIdx.x >> 1) * TT, linv_k);
}
// The same for the panel tiles of a level (TilePlan::h_lvl_trsm_*): two CTAs per packed tile tiles[t], each tile with the
// inverse of its own column cols[t].
__global__ void __launch_bounds__(TRSM_THREADS, 2) trsm_level_kernel(double* __restrict__ S, const double* __restrict__ linv,
                                                                      const int* __restrict__ tiles,
                                                                      const int* __restrict__ cols) {
  const int t = blockIdx.x >> 1;
  trsm_tile(S + (size_t)tiles[t] * TT, linv + (size_t)cols[t] * TT);
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
  double acc[CHAIN_ROWS];   // MODE 1: -C (see tile_update), so the products are added and 0 - acc is stored
#pragma unroll
  for (int r = 0; r < CHAIN_ROWS; r++) acc[r] = MODE == 1 && j <= i0 + r ? -C[(size_t)(i0 + r) * T + j] : 0.0;
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
    else if (j <= i0 + r) *dst = 0.0 - acc[r];
  }
}

// A(i,j) += (-A(i,k)) A(j,k)^T for the tile pairs (i >= j) pi[]/pj[] and the panels k = k0 + q of the bits q of pmask[]
// (TilePlan::h_pair_mask), in increasing k, the K chunks of each panel in increasing order, in the accumulators that hold
// the target for the whole visit (the convention of tile_update below, which gives the same bits).  Used for the chain's
// diagonal pair (factor()), where one tile is updated alone and latency counts: four CTAs per pair, one 64x64 quadrant
// each (consecutive CTAs share the pair's operands in L2); the quadrant above the diagonal of a diagonal tile is skipped.
// The quadrant is read once at the start and written once at the end.
__global__ void __launch_bounds__(SYRK_THREADS, 3) syrk_kernel(double* __restrict__ S, const int* __restrict__ tile_of, int nt,
                                                                int k0, const int* __restrict__ pi, const int* __restrict__ pj,
                                                                const int* __restrict__ pmask) {
  extern __shared__ __align__(16) double smem_d[];
  constexpr size_t ld = T;
  const int p = blockIdx.x >> 2, qr = (blockIdx.x >> 1) & 1, qc = blockIdx.x & 1;
  const int i = pi[p], j = pj[p];
  if (i == j && qc > qr) return;
  double* C = S + (size_t)tile_of[(size_t)i * nt + j] * TT + (size_t)qr * 64 * T + qc * 64;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wm = warp >> 1, wn = warp & 1;
  double* Cw = C + (size_t)(wm * 32 + (lane >> 2)) * ld + wn * 32 + (lane & 3) * 2;   // + (16 a + 8 h) ld + 8 b
  double acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const double2 v = *reinterpret_cast<const double2*>(Cw + (size_t)(a * 16 + h * 8) * ld + b * 8);
        acc[a][b][2 * h] = -v.x;
        acc[a][b][2 * h + 1] = -v.y;
      }
  unsigned mask = (unsigned)pmask[p];
#pragma unroll 1
  for (int k = k0; mask != 0; k++, mask >>= 1) {
    if (!(mask & 1u)) continue;
    const double* Ai = S + (size_t)tile_of[(size_t)i * nt + k] * TT + (size_t)qr * 64 * T;
    const double* Aj = S + (size_t)tile_of[(size_t)j * nt + k] * TT + (size_t)qc * 64 * T;
    __syncthreads();   // every warp is done with the previous panel's last stages before the prologue refills them
    gemm_abt_64<64, true>(Ai, ld, Aj, ld, acc, smem_d);
  }
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
      for (int h = 0; h < 2; h++)
        *reinterpret_cast<double2*>(Cw + (size_t)(a * 16 + h * 8) * ld + b * 8) =
            make_double2(0.0 - acc[a][b][2 * h], 0.0 - acc[a][b][2 * h + 1]);
}

// The trailing update's pipeline (tile_update below) uses the mbarrier helpers of cvb_internal.cuh and these two arrivals.
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(cvb_smem_addr(bar)) : "memory");
}
// arrives on `bar` once every cp.async this thread issued before has landed (the arrival counts against the init count)
__device__ __forceinline__ void mbar_arrive_cp_async(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(cvb_smem_addr(bar)) : "memory");
}

// The same update, one CTA per pair and the whole 128x128 tile per CTA: the throughput path (every update list except the
// chain's diagonal pair, see factor()).  Per 16-wide K chunk a CTA stages 128 rows of each operand for 128x128x16 FMA —
// half the operand bytes per FMA of the 64x64 quadrants above, whose L2→SM traffic bounded them.  The operands come
// through a TILE_STAGES-deep ring that runs on across the panels of the pair's mask, fed by a warp-specialised pipeline
// with no CTA barrier after the set-up:
//   producer   warpgroup 2 (4 warps, 24 registers after setmaxnreg) issues each chunk's cp.asyncs (16 per thread) into a
//              stage once the stage's `empty` barrier has completed, and arrives on its `full` barrier through
//              cp.async.mbarrier.arrive.noinc, which fires when the thread's copies have landed;
//   consumers  warpgroups 0 and 1 (8 warps of 64x32: 4 m16 x 4 n8 blocks, 240 registers after setmaxnreg) wait on `full`,
//              load the whole chunk's fragments (32 A + 16 B doubles beside the 64 accumulator doubles), release the stage
//              on `empty` (one arrival per warp) and only then issue the chunk's 16 DMMAs.  So the stage is refilled
//              while the DMMAs run, and the warps drift apart instead of meeting at a barrier every chunk.
// The CTA is launched with 168 registers per thread (384 threads, 1 CTA/SM), and 24 x 128 + 240 x 256 = 168 x 384: the
// consumers take exactly what the producer gives back.
// The target lives in the accumulators for the whole visit.  Arithmetic convention of every trailing-update kernel
// (this one, syrk_kernel, chain_gemm_kernel<1>): C <- C + (-A(i,k)) A(j,k)^T, the accumulator starting at C, the panels in
// increasing k and the K chunks in increasing order inside each panel, no separate product per panel.  It is computed as
// -C + A(i,k) A(j,k)^T and stored as 0 - acc: round-to-nearest is symmetric under negation, so every rounding is the
// mirror image of the convention's and a non-zero result has its bits, at no cost inside the K loop; a zero is stored as
// +0 (a +0 entry that receives only zero products stays +0).  Since the accumulation starts from the stored target,
// applying a pair's panels in one visit or over several visits gives the same bits, which keeps the blocked,
// column-by-column and column-group schedules bit-identical.  The convention costs accuracy: the sum is recursive, every
// rounding at the magnitude of the running target, where a product per panel summed from zero and then subtracted
// rounded mostly at the product's magnitude.  That product cannot be kept beside the target: the two take 128 registers
// per thread each, more than the consumers' 240 (built that way, ptxas spills 712 B).  Each consumer warp loads
// its 64x32 slice of -C from global memory before its first `full` wait, so the load overlaps the ring fill, and stores
// it once at the end; the warps of a diagonal tile's upper quadrant stay idle, so that quadrant is neither read nor
// written.  Ring rows are 128 B, unpadded: segment s of a row r sits at s ^ 2 (r & 3), which makes the fragment loads
// conflict-free.  Shared memory: TILE_STAGES x 32 KB ring (+ 640 B), 1 CTA/SM.
constexpr int TILE_CONSUMERS = 256;                   // warpgroups 0 and 1
constexpr int TILE_PRODUCERS = 128;                   // warpgroup 2
constexpr int TILE_THREADS = TILE_CONSUMERS + TILE_PRODUCERS;
constexpr int TILE_STAGES = 4;
constexpr int TILE_STAGE = 2 * T * KC;   // doubles per ring stage: 128 rows of A(i,k), then 128 rows of A(j,k)
constexpr size_t kTileSmem = (size_t)TILE_STAGES * TILE_STAGE * sizeof(double);

__device__ __forceinline__ void tile_update(double* __restrict__ S, const int* __restrict__ tile_of, int nt, int k0,
                                            const int* __restrict__ pi, const int* __restrict__ pj,
                                            const int* __restrict__ pmask) {
  extern __shared__ __align__(128) double ring[];   // [TILE_STAGES][2 T][KC], swizzled
  __shared__ const double* s_ai[32];   // operand tiles A(i,k), A(j,k) of the pair's panels, in increasing k
  __shared__ const double* s_aj[32];
  __shared__ uint64_t full[TILE_STAGES], empty[TILE_STAGES];
  __shared__ int s_nch;   // chunks of the visit, read by each role after the set-up barrier (a register would spill)
  constexpr int NCH = T / KC;
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
  // the two warps of 64x32 above the diagonal of a diagonal tile are idle: they never touch the ring
  const int g = lane >> 2, t = lane & 3, wm = warp >> 2, wn = warp & 3;   // warp tile: rows 64 wm.., columns 32 wn..
  const bool idle = diag && wm == 0 && wn >= 2;
  if (tid == 0) s_nch = __popc(mask) * NCH;   // chunk c = K chunk c % NCH of the pair's panel c / NCH
  if (tid < TILE_STAGES) {
    cvb_mbar_init(&full[tid], TILE_PRODUCERS);
    cvb_mbar_init(&empty[tid], diag ? TILE_CONSUMERS / 32 - 2 : TILE_CONSUMERS / 32);
    cvb_fence_mbar_init();
  }
  __syncthreads();

  if (tid >= TILE_CONSUMERS) {   // ---- producer warpgroup
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    const int nch = s_nch;
    const int pt = tid - TILE_CONSUMERS;
    // a thread copies 16-byte segment `seg` of rows r0, r0 + 16, ... of both operands (r0 & 3 fixes the swizzle)
    const int r0 = pt >> 3, seg = pt & 7;
    const int so = r0 * KC + ((seg ^ ((r0 & 3) << 1)) << 1);
#pragma unroll 1
    for (int c = 0; c < nch; c++) {
      const int st = c % TILE_STAGES;
      if (c >= TILE_STAGES) cvb_mbar_wait(&empty[st], (c / TILE_STAGES - 1) & 1);   // chunk c - TILE_STAGES has left
      const size_t go = (size_t)r0 * T + (c % NCH) * KC + seg * 2;
      const double* ga = s_ai[c / NCH] + go;
      const double* gb = s_aj[c / NCH] + go;
      double* As = ring + st * TILE_STAGE + so;
#pragma unroll
      for (int it = 0; it < T / 16; it++) cp_async16(As + it * 16 * KC, ga + (size_t)it * 16 * T);
#pragma unroll
      for (int it = 0; it < T / 16; it++) cp_async16(As + T * KC + it * 16 * KC, gb + (size_t)it * 16 * T);
      mbar_arrive_cp_async(&full[st]);
    }
    asm volatile("cp.async.wait_all;" ::: "memory");   // no copy outlives its issuing thread
    return;
  }

  // ---- consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");
  if (idle) return;
  const int nch = s_nch;
  int cq[4];   // ring column of fragment K index t + 4 q (rows g + 8 n: the swizzle depends on g & 3 only)
#pragma unroll
  for (int q = 0; q < 4; q++) cq[q] = t + 4 * (q ^ (g & 3));
  // the warp's slice of -C in the C-fragment order of dmma16816: acc[ai][bj][2 h + x] = -C(r0 + 16 ai + 8 h,
  // c0 + 8 bj + x), row r0 = 64 wm + g, column c0 = 32 wn + 2 t
  double* Cw = C + (size_t)(wm * 64 + g) * T + wn * 32 + 2 * t;
  double acc[4][4][4];
#pragma unroll
  for (int ai = 0; ai < 4; ai++)
#pragma unroll
    for (int bj = 0; bj < 4; bj++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const double2 v = *reinterpret_cast<const double2*>(Cw + (size_t)(ai * 16 + h * 8) * T + bj * 8);
        acc[ai][bj][2 * h] = -v.x;
        acc[ai][bj][2 * h + 1] = -v.y;
      }
#pragma unroll 1
  for (int c = 0; c < nch; c++) {
    const int st = c % TILE_STAGES;
    cvb_mbar_wait(&full[st], (c / TILE_STAGES) & 1);   // chunk c has landed
    const double* As = ring + st * TILE_STAGE + (wm * 64 + g) * KC;
    const double* Bs = ring + st * TILE_STAGE + T * KC + (wn * 32 + g) * KC;
    double a[4][8], b[4][4];
#pragma unroll
    for (int bj = 0; bj < 4; bj++)
#pragma unroll
      for (int e = 0; e < 4; e++) b[bj][e] = Bs[bj * 8 * KC + cq[e]];
#pragma unroll
    for (int ai = 0; ai < 4; ai++)
#pragma unroll
      for (int e = 0; e < 8; e++) a[ai][e] = As[(ai * 16 + 8 * (e & 1)) * KC + cq[e >> 1]];
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);   // the warp's fragments are in registers: the stage may be refilled
#pragma unroll
    for (int ai = 0; ai < 4; ai++)
#pragma unroll
      for (int bj = 0; bj < 4; bj++) dmma16816(acc[ai][bj], a[ai], b[bj]);
  }
#pragma unroll
  for (int ai = 0; ai < 4; ai++)
#pragma unroll
    for (int bj = 0; bj < 4; bj++)
#pragma unroll
      for (int h = 0; h < 2; h++)
        *reinterpret_cast<double2*>(Cw + (size_t)(ai * 16 + h * 8) * T + bj * 8) =
            make_double2(0.0 - acc[ai][bj][2 * h], 0.0 - acc[ai][bj][2 * h + 1]);
}
__global__ void __launch_bounds__(TILE_THREADS, 1) tile_update_kernel(double* __restrict__ S, const int* __restrict__ tile_of,
                                                                      int nt, int k0, const int* __restrict__ pi,
                                                                      const int* __restrict__ pj,
                                                                      const int* __restrict__ pmask) {
  tile_update(S, tile_of, nt, k0, pi, pj, pmask);
}
// The same for a level's merged update list (TilePlan::h_lvl_pair_*): each pair with its own first panel pk0[].
__global__ void __launch_bounds__(TILE_THREADS, 1) tile_update_level_kernel(double* __restrict__ S,
                                                                            const int* __restrict__ tile_of, int nt,
                                                                            const int* __restrict__ pk0,
                                                                            const int* __restrict__ pi,
                                                                            const int* __restrict__ pj,
                                                                            const int* __restrict__ pmask) {
  tile_update(S, tile_of, nt, pk0[blockIdx.x], pi, pj, pmask);
}

// Factor the diagonal tile k in shared memory and invert the factor, one CTA of 512 threads.  This kernel is the serial
// chain of the whole factorisation (one launch per tile column, nothing else can run before its panel is solved), so it
// is organised around the latency of that chain: the eight 16x16 diagonal blocks, each factored by one warp, with
// everything that does not feed the next diagonal block done beside it.  Blocked right-looking Cholesky over the 16-wide
// block columns jb, two CTA barriers per block column:
//   step 1  warp 0 factors the diagonal block (jb, jb) register-resident (lane = 2*row + half).  Per pivot the *unscaled*
//           column goes through 128 B of shared memory and the update uses a_rj * a_cj / pivot, so the chain per pivot is
//           STS → LDS → rsqrt → DMUL → DFMA (rsqrt and the L values are computed off the chain).  Meanwhile the 12
//           warps that do not share warp 0's scheduler (warp w runs on sub-partition w % 4) apply block column jb-1's
//           rank-16 update to the trailing blocks (look-ahead: the diagonal block itself got it at the end of the previous
//           step 2) and finish block row jb-1 of the inverse;
//   step 2  one thread per row below solves its 16 unknowns by substitution against the diagonal block, and warp 0,
//           which owns the rows of the next diagonal block, applies their update to that block at once.  Meanwhile warp
//           15 inverts the diagonal block and 8 warps form P_jb = L[jb,:jb] X[:jb,:jb] for the inverse.
// The inverse X = L^-1 is built behind the factor by the block-row recurrence X[j,:j] = -X[j,j] P_j, which follows from
// XL = I and keeps the left residual |XL - I| small; X[j,j] comes from warp 15.  When the last diagonal block is factored
// only block row 7 of X is left.  Every 16x16x16 product (trailing update, P_j, X[j,j] P_j) is two mma.sync.m16n8k16.f64
// on one warp.  Results go to global memory as soon as they are final, off the chain: X's blocks from the registers that
// formed them, L's block column jb-1 by the step-1 warps of block column jb.  L lives in the lower triangle of the tile `a`, the off-diagonal blocks of X
// transposed in its upper triangle (X[j,c] as block (c,j)), the X[j,j] in `binv`.  Row strides ≡ 4 doubles mod 16 make
// the fragment loads of a half-warp (rows g = 0..3, columns t = 0..3, or the transpose) hit 16 different banks.
// L is written back to S, the inverse (row-major 128x128, zeros above the diagonal) to linv_k.  flag[0] |= 1 on a
// non-positive pivot (matrix not positive definite → the caller raises mu, as Ceres does on LINEAR_SOLVER_FAILURE).
constexpr int PB = 16;
constexpr int NB = T / PB;      // block columns of the tile
constexpr int LDP = T + 4;      // row stride of the tile in shared memory
constexpr int BLD = PB + 4;     // row stride of binv and of the P_j scratch
constexpr int POTRF_THREADS = 512;
constexpr int POTRF_WARPS = POTRF_THREADS / 32;
constexpr size_t kPotrfSmem =
    ((size_t)T * LDP + (size_t)NB * PB * BLD + (size_t)(T - PB) * BLD + 5 * PB) * sizeof(double);   // 174208 B

// c[h] += A B^T over one 16x16x16 block, as two m16n8k16 (c[h] = columns 8h.. of the output, in dmma16816's C-fragment
// order).  A(r,k) = A[r lda + k] (negated when NEG: exact); B(n,k) = B[n ldb + k], or B[k ldb + n] when BT.
template <bool NEG, bool BT>
__device__ __forceinline__ void mma16(double (&c)[2][4], const double* A, int lda, const double* B, int ldb) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  double a[8];
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const double v = A[(g + 8 * (e & 1)) * lda + t + 4 * (e >> 1)];
    a[e] = NEG ? -v : v;
  }
#pragma unroll
  for (int h = 0; h < 2; h++) {
    double b[4];
#pragma unroll
    for (int e = 0; e < 4; e++) b[e] = BT ? B[(t + 4 * e) * ldb + 8 * h + g] : B[(8 * h + g) * ldb + t + 4 * e];
    dmma16816(c[h], a, b);
  }
}
// offset of element c[h][e] of mma16's output in a 16x16 block with row stride ld (TR: the block stored transposed)
template <bool TR>
__device__ __forceinline__ int frag_off(int h, int e, int ld) {
  const int lane = threadIdx.x & 31, r = (lane >> 2) + 8 * (e >> 1), c = 8 * h + 2 * (lane & 3) + (e & 1);
  return TR ? c * ld + r : r * ld + c;
}

#define POTRF_MARK(i)                                     \
  do {                                                    \
    if (prof != nullptr && tid == 0) prof[i] = clock64(); \
  } while (0)

__device__ __forceinline__ void potrf_inv(double* __restrict__ S, size_t ld, int k, double* __restrict__ linv_k,
                                          int* __restrict__ flag, long long* __restrict__ prof, int prof_fine) {
  extern __shared__ __align__(16) double smem_d[];
  double* a = smem_d;                          // [T][LDP]: L on and below the diagonal, X^T above it
  double* binv = a + T * LDP;                  // [NB][PB][BLD]: X[j,j] = L[j,j]^-1
  double* pt = binv + NB * PB * BLD;           // [T - PB][BLD]: P_j^T
  double* colbuf = pt + (T - PB) * BLD;        // [2][2*PB] pivot-column exchange (second half: dummy slots)
  double* rdbuf = colbuf + 4 * PB;             // [PB] reciprocal diagonal of the current diagonal block
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* At = S + (size_t)k * T * ld + (size_t)k * T;
  auto blk = [&](int i, int j) { return a + i * PB * LDP + j * PB; };
  // A(i,m) -= L(i,jb) L(m,jb)^T on one 16x16 block (one warp)
  auto update_block = [&](int i, int m, int jb) {
    double* C = blk(i, m);
    double c[2][4];
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 4; e++) c[h][e] = C[frag_off<false>(h, e, LDP)];
    mma16<true, false>(c, blk(i, jb), LDP, blk(m, jb), LDP);
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 4; e++) C[frag_off<false>(h, e, LDP)] = c[h][e];
  };
  // L's block column jb (rows >= 16 jb, on and below the diagonal) from shared memory to S
  auto store_l = [&](int jb, int u0, int nthr) {
    const int c0 = jb * PB;
    for (int u = u0; u < (T - c0) * (PB / 2); u += nthr) {
      const int r = c0 + u / (PB / 2), c = c0 + 2 * (u % (PB / 2));
      if (c + 1 <= r)
        *reinterpret_cast<double2*>(At + (size_t)r * ld + c) = make_double2(a[r * LDP + c], a[r * LDP + c + 1]);
      else if (c <= r)
        At[(size_t)r * ld + c] = a[r * LDP + c];
    }
  };
  // X[j,c] = -X[j,j] P_j[:,c] (one warp): kept transposed as block (c,j) for the later P's, and written to linv_k
  auto finish_x = [&](int j, int c) {
    double x[2][4] = {};
    mma16<true, false>(x, binv + j * PB * BLD, BLD, pt + c * PB * BLD, BLD);
    double* D = blk(c, j);
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 4; e++) D[frag_off<true>(h, e, LDP)] = x[h][e];
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 4; e += 2)
        *reinterpret_cast<double2*>(linv_k + (size_t)(j * PB) * T + c * PB + frag_off<false>(h, e, T)) =
            make_double2(x[h][e], x[h][e + 1]);
  };
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
  long long t_a = 0, acc_a = 0, acc_1 = 0, acc_2 = 0;   // fine profile (thread 0 only), kept in registers
  for (int jb = 0; jb < NB; jb++) {
    const int c0 = jb * PB, nbelow = T - c0 - PB;
    if (prof_fine && tid == 0) t_a = clock64();
    // ---------------- step 1 ----------------
    if (warp == 0) {
      // the 16x16 diagonal block.  Branch-free pivot loop: every lane stores one value per step (lanes of the other
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
    } else if ((warp & 3) != 0) {
      // The 12 warps that do not share warp 0's scheduler (warps 4, 8, 12 stay idle: they would take issue slots from
      // the pivot chain): block column jb-1's update of the trailing blocks (i, m), jb <= m <= i, (jb, jb) excepted
      // (numbered row by row), then the blocks X[jb-1, c], c < jb-1, of the inverse, then L's block column jb-1.
      // In block column 0 they write the zeros of X right of its diagonal blocks instead.
      const int w = warp - (warp >> 2) - 1, nw = POTRF_WARPS * 3 / 4;
      if (jb == 0) {
        for (int u = w * 32 + lane; u < T * T / 2; u += nw * 32) {
          const int r = u / (T / 2), c = (u % (T / 2)) * 2;
          if (c >= (r | (PB - 1)) + 1) reinterpret_cast<double2*>(linv_k)[u] = make_double2(0.0, 0.0);
        }
      } else {
        const int nt = NB - jb, nupd = nt * (nt + 1) / 2 - 1;
#pragma unroll 1
        for (int u = w; u < nupd + jb - 1; u += nw) {
          if (u < nupd) {
            int i = 0;
            while ((i + 1) * (i + 2) / 2 <= u + 1) i++;
            update_block(jb + i, jb + (u + 1 - i * (i + 1) / 2), jb - 1);
          } else {
            finish_x(jb - 1, u - nupd);
          }
        }
        store_l(jb - 1, w * 32 + lane, nw * 32);
      }
    }
    __syncthreads();
    if (prof_fine && tid == 0) { const long long tt = clock64(); acc_1 += tt - t_a; t_a = tt; }
    // ---------------- step 2 ----------------
    if (warp == POTRF_WARPS - 1) {
      // inverse of the diagonal block: lane j (< 16) builds column j of Ljj^-1 by forward substitution in axpy form
      // (16 dependent steps, the row updates of a step are independent)
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
        for (int q = 0; q < PB; q++) {
          binv[(jb * PB + q) * BLD + j] = res[q];   // Linv_block[q][j]
          linv_k[(size_t)(c0 + q) * T + c0 + j] = (q >= j) ? res[q] : 0.0;
        }
      }
    } else if (warp >= 4 && (warp & 3) != 0) {
      // P_jb^T: P_jb[:, c] = sum_{m = c..jb-1} L(jb,m) X(m,c) for c < jb, in increasing m (on the 8 warps 5-7, 9-11,
      // 13-14: not beside warp 0 on its scheduler)
      for (int c = warp - 4 - (warp >> 2); c < jb; c += 8) {
        double p[2][4] = {};
        mma16<false, true>(p, blk(jb, c), LDP, binv + c * PB * BLD, BLD);
        for (int m = c + 1; m < jb; m++) mma16<false, false>(p, blk(jb, m), LDP, blk(c, m), LDP);
        double* D = pt + c * PB * BLD;
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
          for (int e = 0; e < 4; e++) D[frag_off<true>(h, e, BLD)] = p[h][e];
      }
    } else if (tid < nbelow) {
      // panel: row r of X solves X Ljj^T = A(r, block), one thread per row, in place
      const int r = c0 + PB + tid;
      double x[PB];
#pragma unroll
      for (int m = 0; m < PB; m += 2) {
        const double2 v = *reinterpret_cast<const double2*>(a + r * LDP + c0 + m);
        x[m] = v.x;
        x[m + 1] = v.y;
      }
#pragma unroll
      for (int m = 0; m < PB; m++) {
        const double xm = x[m] * rdbuf[m];
        x[m] = xm;
#pragma unroll
        for (int q = m + 1; q < PB; q++) x[q] -= a[(c0 + q) * LDP + c0 + m] * xm;
      }
#pragma unroll
      for (int m = 0; m < PB; m += 2) *reinterpret_cast<double2*>(a + r * LDP + c0 + m) = make_double2(x[m], x[m + 1]);
    }
    if (warp == 0 && nbelow > 0) {   // the next diagonal block gets this block column's update now (its rows are warp 0's)
      __syncwarp();
      update_block(jb + 1, jb + 1, jb);
    }
    __syncthreads();
    if (prof_fine && tid == 0) { const long long tt = clock64(); acc_2 += tt - t_a; t_a = tt; }
    if (jb == NB / 2 - 1) POTRF_MARK(2);
    if (jb == NB - 3) POTRF_MARK(3);
  }
  POTRF_MARK(4);
  // block row NB-1 of the inverse, the last diagonal block of L
  if (warp < NB - 1) finish_x(NB - 1, warp);
  else store_l(NB - 1, tid - (NB - 1) * 32, POTRF_THREADS - (NB - 1) * 32);
  if (prof != nullptr) {
    __syncthreads();
    POTRF_MARK(5);
    if (prof_fine && tid == 0) { prof[6] = acc_a; prof[7] = acc_1; prof[8] = acc_2; prof[9] = clock64() - t_a; }
  }
}
__global__ void __launch_bounds__(POTRF_THREADS, 1) potrf_inv_kernel(double* __restrict__ S, size_t ld, int k,
                                                                     double* __restrict__ linv_k, int* __restrict__ flag,
                                                                     long long* __restrict__ prof, int prof_fine) {
  potrf_inv(S, ld, k, linv_k, flag, prof, prof_fine);
}
// The diagonal tiles of the columns c0 .. c0 + gridDim.x - 1 of a level (packed storage), one CTA each.
__global__ void __launch_bounds__(POTRF_THREADS, 1) potrf_inv_level_kernel(double* __restrict__ S,
                                                                           const int* __restrict__ tile_of, int nt, int c0,
                                                                           double* __restrict__ linv, int* __restrict__ flag) {
  const int k = c0 + blockIdx.x;
  potrf_inv(S + (size_t)tile_of[(size_t)k * nt + k] * TT, (size_t)T, 0, linv + (size_t)k * TT, flag, nullptr, 0);
}

// Triangular solves: one persistent kernel per direction, subst_kernel<true> for L y = b and subst_kernel<false> for
// L^T x = y.  A CTA takes the next tile row from a global ticket (increasing row index forward, decreasing backward) and
// forms it completely:
//   forward  row i: r = b_i; r -= L(i,k) y_k for the non-zero tiles (i,k), k < i, in increasing k; y_i = Linv_i r;
//   backward row k: r = y_k; r -= L(i,k)^T x_i for the non-zero tiles (i,k), i > k, in decreasing i; x_k = Linv_k^T r;
// then publishes its result through a per-row flag.  Row r only waits for rows that the ticket handed out before r, to
// CTAs that are already running and never wait for r, so the kernel cannot deadlock whatever the grid size or residency.
// The subtractions are those of a column-by-column solve (one launch per tile column), in the same order and with the
// same products (tile_dot), so the result is bit-identical to it and does not depend on the grid.  A row's tile inverse
// goes to shared memory (cp.async) and each tile to registers before the row waits for the operand, and the next tile is
// fetched into L2 meanwhile: once the operand is published the row reads 128 doubles and does on-chip work only.
// A wait that exceeds kSolveWaitNs (a broken dependency, never a slow one) gives up: the row's result is written as NaN
// and still published, so a fault shows up as a non-finite solution instead of a hang.
constexpr int SOLVE_THREADS = 512;
constexpr size_t kSolveSmem = TT * sizeof(double);   // the row's tile inverse: 128 KB → 1 CTA / SM
constexpr unsigned long long kSolveWaitNs = 4ull * 1000 * 1000 * 1000;

// FWD: out = A x, row r of A by the 32 lanes of a warp (16 warps x 8 rows), lanes along the columns.  Backward:
// out = A^T x, threads along the columns, 4 groups of 128 threads split the rows, partials combined in order.  A is a
// row-major 128x128 tile.  tile_load fetches this thread's 32 elements, tile_dot forms the products; out is complete for
// every thread when tile_dot returns.
template <bool FWD>
__device__ __forceinline__ void tile_load(const double* __restrict__ A, double (&v)[32]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c = threadIdx.x & 127, g = threadIdx.x >> 7;
#pragma unroll
  for (int i = 0; i < 32; i++) v[i] = FWD ? A[(size_t)(warp * 8 + i / 4) * T + lane + 32 * (i % 4)] : A[(size_t)(g * 32 + i) * T + c];
}
template <bool FWD>
__device__ __forceinline__ void tile_dot(const double (&v)[32], const double* x, double* out, double* part /*[4][128]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c = threadIdx.x & 127, g = threadIdx.x >> 7;
  if (FWD) {
    double s[8];
#pragma unroll
    for (int i = 0; i < 8; i++)
      s[i] = (v[4 * i] * x[lane] + v[4 * i + 1] * x[lane + 32]) + (v[4 * i + 2] * x[lane + 64] + v[4 * i + 3] * x[lane + 96]);
    // Each row is summed over the lanes by the butterfly s += (s of lane ^ o), o = 16, 8, 4, 2, 1, as lane 0 sees it.  At
    // the first three steps the partners split the rows instead of both summing all of them (lane 16 h1 + 8 h2 + 4 h3 ends
    // with row 4 h1 + 2 h2 + h3): 9 shuffles instead of 40, and as IEEE addition commutes, the same bits.
    const int h1 = (lane >> 4) & 1, h2 = (lane >> 3) & 1, h3 = (lane >> 2) & 1;
    double t[4], u[2];
#pragma unroll
    for (int j = 0; j < 4; j++) t[j] = (h1 ? s[4 + j] : s[j]) + __shfl_xor_sync(0xffffffffu, h1 ? s[j] : s[4 + j], 16);
#pragma unroll
    for (int j = 0; j < 2; j++) u[j] = (h2 ? t[2 + j] : t[j]) + __shfl_xor_sync(0xffffffffu, h2 ? t[j] : t[2 + j], 8);
    double w = (h3 ? u[1] : u[0]) + __shfl_xor_sync(0xffffffffu, h3 ? u[0] : u[1], 4);
    w += __shfl_xor_sync(0xffffffffu, w, 2);
    w += __shfl_xor_sync(0xffffffffu, w, 1);
    if ((lane & 3) == 0) out[warp * 8 + 4 * h1 + 2 * h2 + h3] = w;
    __syncthreads();
  } else {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 32; i++) s += v[i] * x[g * 32 + i];
    part[g * T + c] = s;
    __syncthreads();
    if (threadIdx.x < T) out[c] = (part[c] + part[T + c]) + (part[2 * T + c] + part[3 * T + c]);
    __syncthreads();
  }
}
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Rows r of the direction: operands / results in out (row r at out + r T), the rows' input in `in`.  ptr / idx: the
// non-zero tiles of row r — forward, the column tiles k < r of tile row r (TilePlan::h_rowc_*, packed index from
// tile_of); backward, the row tiles i > r of tile column r (TilePlan::h_col_ptr / h_row_idx, packed contiguously after
// the diagonal tile: index r + 1 + q).  sync[0] = ticket, sync[1 + r] = row r published; zero at launch.
template <bool FWD>
__global__ void __launch_bounds__(SOLVE_THREADS, 1) subst_kernel(const double* __restrict__ L, const double* __restrict__ linv,
                                                                 const int* __restrict__ ptr, const int* __restrict__ idx,
                                                                 const int* __restrict__ tile_of, int nt, const double* in,
                                                                 double* out, int* sync) {
  extern __shared__ __align__(16) double linv_s[];   // [T][T]
  __shared__ double xs[T], upd[T], part[4 * T];
  __shared__ int s_ticket, s_fail;
  const int tid = threadIdx.x;
  for (;;) {
    if (tid == 0) {
      s_ticket = atomicAdd(sync, 1);
      s_fail = 0;
    }
    __syncthreads();
    if (s_ticket >= nt) return;
    const int r = FWD ? s_ticket : nt - 1 - s_ticket;
#pragma unroll
    for (int it = 0; it < (int)(TT / 2 / SOLVE_THREADS); it++) {
      const int u = 2 * (tid + it * SOLVE_THREADS);
      cp_async16(linv_s + u, linv + (size_t)r * TT + u);
    }
    cp_async_commit();
    double acc = tid < T ? in[(size_t)r * T + tid] : 0.0;
    const int q0 = ptr[r], n = ptr[r + 1] - q0;
    auto tile = [&](int s) {   // s-th product of the row
      const int q = FWD ? q0 + s : q0 + n - 1 - s;
      return L + (size_t)(FWD ? tile_of[(size_t)r * nt + idx[q]] : r + 1 + q) * TT;
    };
    for (int s = 0; s < n; s++) {
      const int k = idx[FWD ? q0 + s : q0 + n - 1 - s];
      double v[32];
      tile_load<FWD>(tile(s), v);
      if (s + 1 < n) {
        const double* nx = tile(s + 1);
#pragma unroll
        for (int it = 0; it < (int)(TT / 16 / SOLVE_THREADS); it++)   // the tile's 128-byte lines
          asm volatile("prefetch.global.L2 [%0];" ::"l"(nx + (size_t)(tid + it * SOLVE_THREADS) * 16));
      }
      if (tid == 0 && !s_fail && !ld_acquire_gpu(sync + 1 + k)) {
        const unsigned long long t0 = globaltimer_ns();
        while (!ld_acquire_gpu(sync + 1 + k))
          if (globaltimer_ns() - t0 > kSolveWaitNs) {
            s_fail = 1;
            break;
          }
      }
      __syncthreads();
      if (tid < T) xs[tid] = __ldcg(out + (size_t)k * T + tid);
      __syncthreads();
      tile_dot<FWD>(v, xs, upd, part);
      if (tid < T) acc -= upd[tid];
    }
    if (tid < T) xs[tid] = acc;
    cp_async_wait<0>();
    __syncthreads();
    double v[32];
    tile_load<FWD>(linv_s, v);   // stored with zeros above the diagonal
    tile_dot<FWD>(v, xs, upd, part);
    if (tid < T) out[(size_t)r * T + tid] = s_fail ? __longlong_as_double(0x7ff8000000000000ll) : upd[tid];
    __syncthreads();
    if (tid == 0) st_release_gpu(sync + 1 + r, 1);
  }
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
  // Levels: a group column joins the run of the previous column when that is a group column too, no column of the run has
  // row tile k, and every row tile i of k first appeared in the run less than 32 columns before k (a target (i, j) then
  // receives panels from at most 32 consecutive columns).
  h_lvl_ptr.assign(1, 0);
  {
    std::vector<int> first(nt, -1);   // per row tile: first column of the current run that has it
    int c0 = 0;
    for (int k = 0; k < nt; k++) {
      bool join = k > c0 && in_group(k) && in_group(c0);
      for (int c = c0; join && c < k; c++) join = !tile(k, c);
      for (int q = h_col_ptr[k]; join && q < h_col_ptr[k + 1]; q++)
        join = first[h_row_idx[q]] < 0 || k - first[h_row_idx[q]] < 32;
      if (!join && k > 0) {
        h_lvl_ptr.push_back(k);
        for (int c = c0; c < k; c++)
          for (int q = h_col_ptr[c]; q < h_col_ptr[c + 1]; q++) first[h_row_idx[q]] = -1;
        c0 = k;
      }
      for (int q = h_col_ptr[k]; q < h_col_ptr[k + 1]; q++)
        if (first[h_row_idx[q]] < 0) first[h_row_idx[q]] = k;
    }
    if (nt > 0) h_lvl_ptr.push_back(nt);
  }
  const int n_lvl = (int)h_lvl_ptr.size() - 1;
  h_lvl_pair_ptr.assign(1, 0); h_lvl_pair_i.clear(); h_lvl_pair_j.clear(); h_lvl_pair_k0.clear(); h_lvl_pair_mask.clear();
  h_lvl_trsm_ptr.assign(1, 0); h_lvl_trsm_tile.clear(); h_lvl_trsm_col.clear();
  h_lvl_fwd_ptr.assign(1, 0); h_lvl_fwd_idx.clear(); h_lvl_bwd_ptr.assign(1, 0); h_lvl_bwd_idx.clear();
  for (int l = 0; l < n_lvl; l++) {
    const int c0 = h_lvl_ptr[l], c1 = in_group(c0) ? h_lvl_ptr[l + 1] : c0;   // lists for the group levels only
    // merged update list: the group columns' width-1 lists (panel k alone), targets in their order (column j, then row i)
    std::map<std::pair<int, int>, std::pair<int, int>> pairs;   // (j, i) -> (first panel, mask)
    for (int k = c0; k < c1; k++)
      for (int p = h_pair_ptr[k]; p < h_pair_ptr[k + 1]; p++) {
        auto it = pairs.find({h_pair_j[p], h_pair_i[p]});
        if (it == pairs.end()) pairs[{h_pair_j[p], h_pair_i[p]}] = {k, 1};
        else it->second.second = (int)((unsigned)it->second.second | 1u << (k - it->second.first));
      }
    for (const auto& e : pairs) {
      h_lvl_pair_j.push_back(e.first.first);
      h_lvl_pair_i.push_back(e.first.second);
      h_lvl_pair_k0.push_back(e.second.first);
      h_lvl_pair_mask.push_back(e.second.second);
    }
    h_lvl_pair_ptr.push_back((int)h_lvl_pair_i.size());
    std::vector<int> fwd, bwd;
    for (int k = c0; k < c1; k++) {
      const bool has_next = h_col_ptr[k + 1] > h_col_ptr[k] && h_row_idx[h_col_ptr[k]] == k + 1;
      for (int q = h_col_ptr[k]; q < h_col_ptr[k + 1]; q++) {
        fwd.push_back(h_row_idx[q]);
        if (has_next && q == h_col_ptr[k]) continue;
        h_lvl_trsm_tile.push_back(h_col_base[k] + 1 + (q - h_col_ptr[k]));
        h_lvl_trsm_col.push_back(k);
      }
      bwd.insert(bwd.end(), h_rowc_idx.begin() + h_rowc_ptr[k], h_rowc_idx.begin() + h_rowc_ptr[k + 1]);
    }
    h_lvl_trsm_ptr.push_back((int)h_lvl_trsm_tile.size());
    for (std::vector<int>* v : {&fwd, &bwd}) {
      std::sort(v->begin(), v->end());
      v->erase(std::unique(v->begin(), v->end()), v->end());
    }
    h_lvl_fwd_idx.insert(h_lvl_fwd_idx.end(), fwd.begin(), fwd.end());
    h_lvl_fwd_ptr.push_back((int)h_lvl_fwd_idx.size());
    h_lvl_bwd_idx.insert(h_lvl_bwd_idx.end(), bwd.begin(), bwd.end());
    h_lvl_bwd_ptr.push_back((int)h_lvl_bwd_idx.size());
  }
}

int nd_layout(const std::vector<std::vector<int>>& members, int bw, std::vector<int>& off, std::vector<int>& group_of_tile) {
  const int per = T / bw;
  const auto level = [](int p) { return __builtin_ctz(~(unsigned)p); };
  int n_level = 0;
  for (const auto& m : members)
    for (int p = 0; p * per < (int)m.size(); p++) n_level = std::max(n_level, level(p) + 1);
  group_of_tile.clear();
  for (int lv = 0; lv < n_level; lv++)
    for (size_t g = 0; g < members.size(); g++)
      for (int p = 0; p * per < (int)members[g].size(); p++) {
        if (level(p) != lv) continue;
        const int tile = (int)group_of_tile.size();
        for (int q = p * per; q < std::min((p + 1) * per, (int)members[g].size()); q++)
          off[members[g][q]] = tile * T + (q - p * per) * bw;
        group_of_tile.push_back((int)g);
      }
  return (int)group_of_tile.size();
}

int TilePlan::upload(cvb_ctx* ctx, cudaStream_t st) {
  auto up = [&](cvb_dev_arr<int>& d, const std::vector<int>& h) -> int {
    CVB_CUDA(ctx, d.alloc(h.size(), st));
    if (h.size()) CVB_CUDA(ctx, cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    return CVB_OK;
  };
  int rc;
  if ((rc = up(d_row_idx, h_row_idx)) || (rc = up(d_pair_i, h_pair_i)) || (rc = up(d_pair_j, h_pair_j)) ||
      (rc = up(d_pair_mask, h_pair_mask)) || (rc = up(d_rowc_idx, h_rowc_idx)) || (rc = up(d_tile_of, h_tile_of)) ||
      (rc = up(d_lvl_pair_i, h_lvl_pair_i)) || (rc = up(d_lvl_pair_j, h_lvl_pair_j)) ||
      (rc = up(d_lvl_pair_k0, h_lvl_pair_k0)) || (rc = up(d_lvl_pair_mask, h_lvl_pair_mask)) ||
      (rc = up(d_lvl_trsm_tile, h_lvl_trsm_tile)) || (rc = up(d_lvl_trsm_col, h_lvl_trsm_col)) ||
      (rc = up(d_col_ptr, h_col_ptr)) || (rc = up(d_rowc_ptr, h_rowc_ptr)))
    return rc;
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  return CVB_OK;
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
  CVB_CUDA(ctx, cudaMalloc(&d_solve_sync, (size_t)2 * (nt + 1) * sizeof(int)));
  solve_nt = nt;
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
  if (d_solve_sync) cudaFree(d_solve_sync);
  d_solve_sync = nullptr;
  solve_nt = 0;
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
  {
    std::lock_guard<std::mutex> once_lk(once.mtx);
    if (once.first(ctx->device)) {
      CVB_CUDA(ctx, cudaFuncSetAttribute(trsm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrsmSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSyrkSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(tile_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTileSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(potrf_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPotrfSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(chain_gemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kChainSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(chain_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kChainSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(trsm_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrsmSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(tile_update_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTileSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(potrf_inv_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPotrfSmem));
    }
  }
  const int nt = plan.nt;
  const bool dist = dv != nullptr && dv->world > 1 && !plan.h_owner.empty();
  CVB_REQUIRE(ctx, plan.d_tile_of.p != nullptr && (int)plan.h_col_base.size() == nt, "tile plan not built / uploaded");
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
  // Level schedule of the column groups (single GPU and replicated plans; TilePlan::h_lvl_ptr): the columns of a level are
  // independent, so each level is three batched launches on the main stream — every diagonal tile, every panel tile, the
  // merged update list — instead of a chain step per column.  Per tile the kernels and the order of the products are those
  // of the column-by-column schedule, so the results are bit-identical to it.  The one product the column-by-column
  // schedule leaves to the chain, S(k+1,k+1) -= L(k+1,k) L(k+1,k)^T when the level's last column k has row tile k+1, is
  // made the chain's way too (chain_gemm_kernel), after the merged list, as is the solve of tile (k+1,k).
  auto run_level = [&](int l) -> int {
    const int c0 = plan.h_lvl_ptr[l], nc = plan.h_lvl_ptr[l + 1] - c0, kl = c0 + nc - 1;
    if (sf_live) {   // the main sequence's chain and bulk streams join the main stream
      CVB_CUDA(ctx, cudaEventRecord(fs.fork_fast, sf));
      CVB_CUDA(ctx, cudaStreamWaitEvent(st, fs.fork_fast, 0));
      sf_live = false;
    }
    if (last_bulk >= 0) CVB_CUDA(ctx, cudaStreamWaitEvent(st, ev[5 * last_bulk + 1], 0));
    last_bulk = prev_chain = -1;
    auto mark = [&](int e) {   // one event per stage of the level (the trace gives it to each of the level's columns)
      if (tr) cudaEventRecord(tev[(size_t)c0 * 5 + e], st);
    };
    mark(0);
    potrf_inv_level_kernel<<<nc, POTRF_THREADS, kPotrfSmem, st>>>(S, plan.d_tile_of.p, nt, c0, linv, d_flag);
    CVB_CHECK_LAUNCH(ctx);
    mark(1);
    double* diag = S + (size_t)plan.h_col_base[kl] * TT;
    const bool has_next = plan.h_col_ptr[kl + 1] > plan.h_col_ptr[kl] && plan.h_row_idx[plan.h_col_ptr[kl]] == kl + 1;
    if (has_next) {
      chain_gemm_kernel<0><<<T / CHAIN_ROWS, T, kChainSmem, st>>>(diag + TT, diag + TT, linv + (size_t)kl * TT);
      CVB_CHECK_LAUNCH(ctx);
    }
    const int t0 = plan.h_lvl_trsm_ptr[l], ntr = plan.h_lvl_trsm_ptr[l + 1] - t0;
    if (ntr > 0) {
      trsm_level_kernel<<<2 * ntr, TRSM_THREADS, kTrsmSmem, st>>>(S, linv, plan.d_lvl_trsm_tile.p + t0, plan.d_lvl_trsm_col.p + t0);
      CVB_CHECK_LAUNCH(ctx);
    }
    mark(2);
    const int p0 = plan.h_lvl_pair_ptr[l], np = plan.h_lvl_pair_ptr[l + 1] - p0;
    if (np > 0) {
      tile_update_level_kernel<<<np, TILE_THREADS, kTileSmem, st>>>(S, plan.d_tile_of.p, nt, plan.d_lvl_pair_k0.p + p0,
                                                                    plan.d_lvl_pair_i.p + p0, plan.d_lvl_pair_j.p + p0,
                                                                    plan.d_lvl_pair_mask.p + p0);
      CVB_CHECK_LAUNCH(ctx);
    }
    if (has_next) {
      chain_gemm_kernel<1><<<T / CHAIN_ROWS, T, kChainSmem, st>>>(S + (size_t)plan.h_col_base[kl + 1] * TT, diag + TT, diag + TT);
      CVB_CHECK_LAUNCH(ctx);
    }
    mark(3);
    return CVB_OK;
  };
  int lvl = 0;
  for (int k = 0; k < nt; k++) {
    while (plan.h_lvl_ptr[lvl + 1] <= k) lvl++;
    if (!dist && plan.level_is_group(lvl)) {
      if ((rc_join = run_level(lvl))) return rc_join;
      k = plan.h_lvl_ptr[lvl + 1] - 1;
      continue;
    }
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
    // A. tile (k,k) is final: when the previous chain column is k-1, its contribution came with the chain and the others
    //    were waited for by its chain step (below).  Otherwise (a column group in nested-dissection order: the group's
    //    previous column is a lower level and may have row tile k) that column's updates of tile (k,k) ran on the work
    //    stream as ordinary list pairs, so they are waited for here.
    if (pc >= 0 && pc != k - 1) CVB_CUDA(ctx, cudaStreamWaitEvent(cs, ev[5 * pc + 4], 0));
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
      syrk_kernel<<<4, SYRK_THREADS, kSyrkSmem, cs>>>(S, plan.d_tile_of.p, nt, k0, plan.d_pair_i.p + p0, plan.d_pair_j.p + p0,
                                                       plan.d_pair_mask.p + p0);
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
        tile_update_kernel<<<na - a0, TILE_THREADS, kTileSmem, ws>>>(S, plan.d_tile_of.p, nt, k0, plan.d_pair_i.p + p0 + a0,
                                                                     plan.d_pair_j.p + p0 + a0, plan.d_pair_mask.p + p0 + a0);
        CVB_CHECK_LAUNCH(ctx);
      }
      if (tr) cudaEventRecord(tev[(size_t)k * 5 + 3], ws);
      if (np - na > 0) {
        CVB_CUDA(ctx, cudaStreamWaitEvent(st2, evPanel, 0));
        tile_update_kernel<<<np - na, TILE_THREADS, kTileSmem, st2>>>(S, plan.d_tile_of.p, nt, k0, plan.d_pair_i.p + p0 + na,
                                                                       plan.d_pair_j.p + p0 + na, plan.d_pair_mask.p + p0 + na);
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
      for (int k = 0, l = 0; k < nt; k++) {
        while (plan.h_lvl_ptr[l + 1] <= k) l++;
        const int ke = !dist && plan.level_is_group(l) ? plan.h_lvl_ptr[l] : k;   // column whose events time column k
        float t[5];
        for (int e = 0; e < 5; e++) {
          t[e] = -1.f;
          if (cudaEventQuery(tev[(size_t)ke * 5 + e]) == cudaSuccess) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, tev[(size_t)nt * 5], tev[(size_t)ke * 5 + e]) == cudaSuccess) t[e] = ms * 1e3f;
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

// solves L L^T x = b; tmp is scratch (n_pad), result in x.  grid = CTAs per direction, 0 = as many as fit on the device
// at once (solve()); the result does not depend on it.
int solve_grid(cvb_ctx* ctx, const double* L, const double* linv, const double* b, double* tmp, double* x,
               const TilePlan& plan, cudaStream_t st, const FactorStreams& fs, int grid) {
  static cvb_once_per_device once;
  {
    std::lock_guard<std::mutex> once_lk(once.mtx);
    if (once.first(ctx->device)) {
      CVB_CUDA(ctx, cudaFuncSetAttribute(subst_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSolveSmem));
      CVB_CUDA(ctx, cudaFuncSetAttribute(subst_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSolveSmem));
    }
  }
  const int nt = plan.nt;
  CVB_REQUIRE(ctx, plan.d_rowc_ptr.p != nullptr && plan.d_col_ptr.p != nullptr, "tile plan not built / uploaded");
  CVB_REQUIRE(ctx, fs.d_solve_sync != nullptr && fs.solve_nt >= nt, "factor streams not created for this plan");
  if (nt == 0) return CVB_OK;
  if (grid <= 0) {
    int per_sm = 0, n_sm = 0;
    CVB_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, subst_kernel<true>, SOLVE_THREADS, kSolveSmem));
    CVB_CUDA(ctx, cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, ctx->device));
    grid = per_sm * n_sm;
  }
  grid = std::max(1, std::min(grid, nt));
  int* fsync = fs.d_solve_sync;   // forward: [0, nt], backward: [nt + 1, 2 nt + 1]
  CVB_CUDA(ctx, cudaMemsetAsync(fsync, 0, (size_t)2 * (nt + 1) * sizeof(int), st));
  subst_kernel<true><<<grid, SOLVE_THREADS, kSolveSmem, st>>>(L, linv, plan.d_rowc_ptr.p, plan.d_rowc_idx.p, plan.d_tile_of.p,
                                                              nt, b, tmp, fsync);
  CVB_CHECK_LAUNCH(ctx);
  subst_kernel<false><<<grid, SOLVE_THREADS, kSolveSmem, st>>>(L, linv, plan.d_col_ptr.p, plan.d_row_idx.p, nullptr, nt, tmp,
                                                               x, fsync + nt + 1);
  CVB_CHECK_LAUNCH(ctx);
  return CVB_OK;
}
int solve(cvb_ctx* ctx, const double* L, const double* linv, double* b, double* tmp, double* x,
          const TilePlan& plan, cudaStream_t st, const FactorStreams& fs) {
  return solve_grid(ctx, L, linv, b, tmp, x, plan, st, fs, 0);
}

}  // namespace cvb_chol

// ---- test/diagnostic entry: solve A x = b for a host SPD matrix (row-major n x n) with the BA factorisation ----
// Latency of the diagonal-tile kernel (the serial chain of the tiled factorisation): factors `reps` copies of a synthetic
// SPD tile back to back; us_per_tile = average launch-to-launch time; phase_cycles[0..5] = clock64 marks of the last
// launch relative to its start (loaded, 4 and 6 of the 8 block columns factored, factored, inverted); summed over the 8
// block columns: [6] = the 16x16 diagonal-block factorisations, [7] = step 1 (diagonal block beside the trailing update)
// incl. its barrier, [8] = step 2 (panel beside the inverse's products) incl. its barrier; [9] = the inverse's last block
// row after the last block column.
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
  cvb_block B(ctx, st);
  double *dS, *db, *dl, *dy, *dx;
  int* dflag;
  B.in(dS, hs.data(), hs.size()); B.in(db, hb.data(), np);
  B.tmp(dl, (size_t)np * T); B.tmp(dy, np);
  B.out_host(dflag, 1); B.out_host(dx, np);
  int rc;
  if ((rc = B.place()) || (rc = B.upload())) return rc;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  if ((rc = plan.upload(ctx, st))) return rc;
  FactorStreams fs;
  if ((rc = fs.create(ctx, nt))) return rc;
  cudaEventRecord(e0, st);
  rc = factor(ctx, dS, dl, dflag, plan, st, fs);
  cudaEventRecord(e1, st);
  if (rc) return rc;
  rc = solve(ctx, dS, dl, db, dy, dx, plan, st, fs);
  if (rc) return rc;
  if ((rc = B.download())) return rc;
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (factor_ms) *factor_ms = ms;
  if (*B.host(dflag)) return cvb_fail(ctx, CVB_ERR_NUMERIC, "matrix is not positive definite");
  memcpy(x, B.host(dx), (size_t)n * sizeof(double));
  return CVB_OK;
}
