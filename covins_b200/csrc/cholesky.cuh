// cholesky.cuh — interface of the tiled FP64 Cholesky (cholesky.cu) used by the BA engine.
#pragma once
#include <vector>

#include "cvb_internal.cuh"

namespace cvb_chol {

constexpr int T = 128;  // tile edge
// Width of the outer block of the main sequence: the trailing update of the tiles past a block applies all of the block's
// panels in one visit to each tile (one C round trip to HBM per block instead of per panel).  4 was the fastest of 2, 3
// and 4 at C3 with the whole-tile update kernel (DESIGN.md §9).
constexpr int kPanelBlock = 4;

// Tile-level structure of the factor: which 128x128 tiles of L are structurally non-zero, as launch lists.
struct TilePlan {
  int nt = 0;
  std::vector<int> h_col_ptr, h_row_idx;           // per tile column k: non-zero row tiles i > k
  // Trailing-update launch lists, issued after the panel of tile column k is solved: pairs (i >= j) of target tiles with
  // the panels each one receives, bit q of h_pair_mask = panel h_pair_k0[k] + q (the panel tiles (i,k') and (j,k') both
  // exist).  Width 1 (h_blk_end[k] == k + 1 and h_pair_k0[k] == k): the pairs of panel k.  Inside a block of
  // kPanelBlock columns: panel k alone, on the targets inside the block.  At a block's last column: all of the block's
  // panels on every target past the block.  The product S(k+1,k+1) -= L(k+1,k) L(k+1,k)^T is never listed: the chain
  // (factor()) computes it.
  std::vector<int> h_pair_ptr, h_pair_i, h_pair_j, h_pair_mask;
  std::vector<int> h_pair_k0;                      // per tile column k: panel of mask bit 0
  std::vector<int> h_pair_split;                   // per tile column k: how many of its pairs (listed first) go on the work
                                                   // stream (the next block's columns); the rest go on the bulk stream
  std::vector<int> h_blk_end;                      // per tile column k: one past the last column of its block
  std::vector<int> h_rowc_ptr, h_rowc_idx;         // per tile row k: non-zero column tiles i < k (backward solve)
  std::vector<int> h_col_group;                    // optional, per tile column: id (>= 0) of an independent column group
                                                   // (its columns share no tile with other groups), -1 = main sequence
  // Packed tile storage: only the tiles of L's structure exist.  Column k's tiles are contiguous — the diagonal tile at
  // h_col_base[k], then its row tiles in h_row_idx order — so a panel is one contiguous block (one peer copy when the
  // factorisation is distributed).  h_tile_of[i * nt + j] = packed index of tile (i >= j) or -1.
  std::vector<int> h_col_base, h_tile_of;
  // Distributed factorisation: h_owner[k] = rank that factors tile column k and applies every update to it (empty =
  // single GPU).  With an owner map the pair lists hold only the pairs whose TARGET column this rank owns.
  std::vector<int> h_owner;
  int my_rank = 0;
  int *d_row_idx = nullptr, *d_pair_i = nullptr, *d_pair_j = nullptr, *d_pair_mask = nullptr, *d_rowc_idx = nullptr,
      *d_tile_of = nullptr;
  long n_tiles_L = 0;
  double flops = 0.0;   // flops of one numeric factorisation with this plan
  // col_group (optional, nt entries): h_col_group.  owner (optional, nt entries) + rank: distributed plan.  flops = the
  // tile GEMMs this rank executes.
  void build(int nt, std::vector<uint8_t> lower_mask, std::vector<int> col_group = {}, const std::vector<int>* owner = nullptr,
             int rank = 0);
  size_t tile_index(int i, int j) const { return (size_t)h_tile_of[(size_t)i * nt + j]; }
  int upload(cvb_ctx* ctx, cudaStream_t st);
  void release();
};

// Extra streams/events of a factorisation (all events with timing disabled), made by create() for a plan of nt tile
// columns and released by destroy() or the destructor.
struct FactorStreams {
  FactorStreams() = default;
  FactorStreams(const FactorStreams&) = delete;
  FactorStreams& operator=(const FactorStreams&) = delete;
  ~FactorStreams() { destroy(); }
  static constexpr int n_group = 8;
  cudaStream_t bulk = nullptr;       // low-priority stream of the bulk trailing updates (depth-1 lookahead)
  cudaStream_t fast = nullptr;       // highest-priority stream of the critical chain (diagonal tile -> first panel tile -> next diagonal tile)
  cudaEvent_t fork_fast = nullptr;
  std::vector<cudaEvent_t> ev;       // 5 * nt events: panel available, bulk done, diagonal tile done, chain step done, tile column k+1 updated
  cudaStream_t group[n_group] = {};  // streams of the independent column groups (their chain streams)
  cudaStream_t group_aux[n_group] = {};   // second stream per group: rest of the panel + updates, beside the group's chain
  cudaEvent_t join_aux[n_group] = {};
  cudaEvent_t fork = nullptr, join[n_group] = {};
  int create(cvb_ctx* ctx, int nt);
  void destroy();
};
// Peer view of a distributed factorisation (one process per GPU, buffers mapped with CUDA IPC over NVLink):
// every rank owns the tile columns h_owner says; after trsm of column k the owner raises flag[k] = epoch in every
// peer's flag array, the peers wait on their LOCAL flag and pull the panel (and the tile inverse) out of the owner's
// memory straight into the same place of their own packed array — so every rank ends up with the complete factor.
struct DistView {
  int rank = 0, world = 1;
  double* peer_S[16] = {};       // packed tile arrays of all ranks (own entry = local pointer)
  double* peer_linv[16] = {};
  int* peer_flag[16] = {};       // [2 nt] per rank: [k] = first panel tile of column k ready (chain), [nt + k] = whole panel ready
  int* d_epoch = nullptr;        // local factorisation counter (device)
  int** d_peer_flag = nullptr;   // device copy of peer_flag[]
};
// S: packed tiles (plan.h_col_base / h_tile_of), linv: nt tile inverses
int factor(cvb_ctx* ctx, double* S, double* linv, int* d_flag, const TilePlan& plan, cudaStream_t st,
           const FactorStreams& fs, const DistView* dv = nullptr);
int solve(cvb_ctx* ctx, const double* L, const double* linv, double* b, double* tmp, double* x,
          const TilePlan& plan, cudaStream_t st, const FactorStreams& fs);

}  // namespace cvb_chol
