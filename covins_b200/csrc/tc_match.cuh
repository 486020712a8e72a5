// tc_match.cuh — interface of the wgmma (tensor-core) matching kernel and of the matcher's kernel choice, see tc_match.cu
#pragma once
#include <vector>

#include "cvb_internal.cuh"

namespace cvb_tc {

constexpr int kIdxBits = 22;   // Hamming packed key: distance << 22 | segment-local train index (segments < 4 Mi rows)

struct TcParams {
  const uint8_t* q;
  int nq;
  const uint8_t* t;
  const int32_t* seg_ptr;
  int n_seg;
  int nqb, parts;           // filled by launch()
  int32_t* out_idx;
  void* out_dist;
  int filter;
  float thr, ratio;
  int32_t* match_train;
  float* match_dist;
  int32_t* n_matches;
  // the operand tiles of the train set (expand_tiles, the metric's tile image) and the first tile of every segment
  // [n_seg + 1]; xt == nullptr → launch() expands into the call's device block (needs h_seg, the host copy of seg_ptr)
  const uint8_t* xt;
  const int32_t* seg_tile;
  const int32_t* h_seg;
};

// metric 0 = Hamming (32-byte rows), 1 = L2 on u8 (128-byte rows); OpenCV k-NN rule (the DenseMatcher list rule is
// order dependent and stays on the scalar kernel)
int launch(cvb_ctx* ctx, TcParams p, int metric, int k, cudaStream_t st);

// operand tile store of the tensor-core path: 128-row tiles per segment, tile_bytes(metric) each, in the shared-memory image the
// metric's wgmma reads (Hamming: expanded bits + key slice; L2: u8 rows + |t|^2 per row)
int64_t tiles_of(const int32_t* h_seg, int n_seg, std::vector<int32_t>* seg_tile);   // total tiles; optional prefix [n_seg + 1]
size_t tile_bytes(int metric);
int expand_tiles(cvb_ctx* ctx, int metric, const uint8_t* d_rows, const int32_t* d_seg_ptr, const int32_t* d_seg_tile, int seg_lo,
                 int seg_hi, int tile_lo, int n_tiles, uint8_t* d_xt, cudaStream_t st);

// The formulation that matches nq >= 1 queries against n_seg segments of `total` rows, the longest max_len rows (filter: the
// fused ratio filter of k = 2).  kTensor: launch() on the segments, when there are enough of them per query block to fill
// the SMs.  kTensorChunks: one long segment cut into `chunk`-row segments for launch(), whose lists the caller merges by
// (distance, index).  kScalar: the POPC / DP4A scan of match_kernels.cu.  COVINS_B200_MATCH_KERNEL=popc forces the scalar
// scan; =tc forces the tensor cores wherever the packed keys can index every segment.
enum class Kernel { kScalar, kTensor, kTensorChunks };
struct Choice {
  Kernel kernel;
  int64_t chunk;   // kTensorChunks: rows per chunk, a multiple of 128 below 2^kIdxBits
};
Choice choose(const cvb_ctx* ctx, int nq, int n_seg, int64_t total, int max_len, bool filter);

}  // namespace cvb_tc
