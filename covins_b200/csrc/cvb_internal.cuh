// cvb_internal.cuh — ctx, error plumbing and small device helpers shared by all translation units of
// libcovins_b200.so.  Not part of the public boundary (that is include/covins_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/covins_b200.h"

struct cvb_buf {
  void* p = nullptr;
  size_t cap = 0;
};

struct cvb_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  int sm_count = 132;
  int64_t launches = 0;
  std::string err;
  // grow-only device workspaces (named slots so independent stages never alias)
  cvb_buf ws[27];   // one per WS_* slot below
  // pinned host staging
  void* h_pin = nullptr;
  size_t h_pin_cap = 0;
  void* ba = nullptr;  // BA state (owned by ba_*.cu)
  // resident operand tiles of a train set (set by the map database around its matching call, see tc_match.cu): when the
  // matcher is handed the packed rows `xt_for`, their pre-expanded tiles are at `xt` / `xt_seg_tile`
  const uint8_t* xt_for = nullptr;
  const uint8_t* xt = nullptr;
  const int32_t* xt_seg_tile = nullptr;
  // every extern "C" entry point holds this lock for its duration (cvb_device_guard): a ctx may be shared between host
  // threads — calls on one ctx are serialised, concurrency comes from one ctx per thread
  mutable std::recursive_mutex mtx;
};

enum { WS_Q = 0, WS_T, WS_SEG, WS_OUT0, WS_OUT1, WS_OUT2, WS_PART_I, WS_PART_D, WS_LIST_I, WS_LIST_D, WS_SKIPA,
       WS_SKIPB, WS_TMP0, WS_TMP1, WS_FLAG, WS_MISC, WS_CHUNK_PS, WS_CHUNK_OFF, WS_GS0, WS_GS1, WS_GS2, WS_GS3, WS_GS4, WS_GS5, WS_GS6, WS_XT, WS_XT_TILE };
static_assert(WS_XT_TILE < (int)(sizeof(cvb_ctx::ws) / sizeof(cvb_buf)), "cvb_ctx::ws has a buffer per workspace slot");

// cudaFuncSetAttribute applies to the CURRENT device: one flag per (call site, device), so that a process that opens contexts
// on several GPUs raises the dynamic shared-memory limit on each of them
struct cvb_once_per_device {
  std::atomic<bool> done[64];
  cvb_once_per_device() { for (auto& d : done) d.store(false); }
  bool first(int device) {
    if (device < 0 || device >= 64) return true;
    return !done[device].exchange(true);
  }
};

int cvb_fail(cvb_ctx* ctx, int code, const char* fmt, ...);
void* cvb_ws(cvb_ctx* ctx, int slot, size_t bytes);          // returns nullptr on failure (ctx->err set)
void* cvb_pinned(cvb_ctx* ctx, size_t bytes);

// match_kernels.cu: the fused 2-NN + ratio filter of cvb_match_hamming_batch for n_pairs pairs of keyframes of one device
// descriptor table d_desc in one launch on ctx->stream.  d_pairs [n_pairs][5] = (query row0, query rows, train row0, train rows,
// output offset); pair s writes match_train / match_dist [offset + query] and n_matches [s]; max_nq: the largest query count.
// cvb_match_l2_pairs_dev: the same for cvb_match_l2_batch on the u8 SIFT layout, d_desc [rows][128] (16-byte aligned).
int cvb_match_hamming_pairs_dev(cvb_ctx* ctx, const uint8_t* d_desc, const int32_t* d_pairs, int n_pairs, int max_nq, float thr, float ratio,
                                int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches);
int cvb_match_l2_pairs_dev(cvb_ctx* ctx, const uint8_t* d_desc, const int32_t* d_pairs, int n_pairs, int max_nq, float thr, float ratio,
                           int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches);

// ransac_abs.cu: the seeded GP3P RANSAC of cvb_ransac_absolute_pose_seeded_batch on device inputs and outputs (one CTA per
// problem on ctx->stream).  d_cam [n_prob][12] = camera offset (3) then rotation (9, row-major); d_inlier_mask nullable.
int cvb_abs_ransac_seeded_dev(cvb_ctx* ctx, int n_prob, const int32_t* d_prob_ptr, const double* d_pts, const double* d_f, const double* d_sigma,
                              const double* d_cam, const uint64_t* d_seed, double threshold, int max_iterations, double probability,
                              int32_t* d_best_sample, double* d_best_model, int32_t* d_best_count, int32_t* d_iterations, int32_t* d_consumed,
                              uint8_t* d_inlier_mask);

// relpose.cu: one problem of cvb_optimize_relative_pose in device memory (all pointers device).  pose_in [7]; removed [n];
// out [27] = T12_out [7], n_inliers, the two solves' iterations, the cost-history length and the history [16].
struct cvb_relcam {
  double intr[4], dist[4];
  int cam, dm;
  double xi;
};
struct cvb_relpose_dev {
  int n;
  const double* pA; const double* pB; const float* kpA; const float* kpB; const double* sA; const double* sB;
  cvb_relcam camA, camB;
  const double* pose_in; uint8_t* removed; double* out;
};
constexpr int CVB_RELPOSE_OUT = 27;
// refines the n_prob problems d_probs [n_prob] (device) in one launch on ctx->stream, one CTA each; a problem with n < 12 gets
// cvb_optimize_relative_pose's early result (T12_out = pose_in, nothing removed, zero counts)
int cvb_relpose_batch_dev(cvb_ctx* ctx, const cvb_relpose_dev* d_probs, int n_prob, double th_outlier_align);

#define CVB_CUDA(ctx, call)                                                                         \
  do {                                                                                              \
    cudaError_t e_ = (call);                                                                        \
    if (e_ != cudaSuccess)                                                                          \
      return cvb_fail((ctx), CVB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_),  \
                      __FILE__, __LINE__);                                                          \
  } while (0)

#define CVB_CHECK_LAUNCH(ctx)                                                                       \
  do {                                                                                              \
    (ctx)->launches++;                                                                              \
    cudaError_t e_ = cudaGetLastError();                                                            \
    if (e_ != cudaSuccess)                                                                          \
      return cvb_fail((ctx), CVB_ERR_CUDA, "kernel launch failed: %s (%s:%d)",                      \
                      cudaGetErrorString(e_), __FILE__, __LINE__);                                  \
  } while (0)

#define CVB_REQUIRE(ctx, cond, ...)                                      \
  do {                                                                   \
    if (!(cond)) return cvb_fail((ctx), CVB_ERR_INVALID, __VA_ARGS__);   \
  } while (0)

static inline cudaStream_t cvb_stream(cvb_ctx* ctx, void* s) { return s ? (cudaStream_t)s : ctx->stream; }

// Scoped guard of every extern "C" entry point: takes the ctx's lock (calls on one ctx are serialised, so a ctx may be
// shared between host threads) and makes the ctx's device current for the calling thread (a new host thread defaults to
// device 0; two ctxs on different GPUs may be driven from one thread), restoring the previous device on exit.
struct cvb_device_guard {
  int prev = -1;
  bool switched = false;
  const cvb_ctx* ctx = nullptr;
  explicit cvb_device_guard(const cvb_ctx* c) : ctx(c) {
    if (c) c->mtx.lock();
    if (c && cudaGetDevice(&prev) == cudaSuccess && prev != c->device) switched = cudaSetDevice(c->device) == cudaSuccess;
  }
  ~cvb_device_guard() {
    if (switched) cudaSetDevice(prev);
    if (ctx) ctx->mtx.unlock();
  }
  cvb_device_guard(const cvb_device_guard&) = delete;
  cvb_device_guard& operator=(const cvb_device_guard&) = delete;
};
#define CVB_GUARD(ctx) cvb_device_guard cvb_guard_((ctx))

// ---------------------------------------------------------------------------------------------
// Device helpers: mbarrier + 1-D bulk TMA (cp.async.bulk → SASS UBLKCP), used to stage descriptor
// tiles into shared memory.
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t cvb_smem_addr(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void cvb_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(cvb_smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void cvb_fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void cvb_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(cvb_smem_addr(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void cvb_mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(cvb_smem_addr(bar)),
      "r"(parity)
      : "memory");
}
// global → shared bulk copy (bytes % 16 == 0, both addresses 16-B aligned), completion on `bar`.
__device__ __forceinline__ void cvb_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          cvb_smem_addr(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(cvb_smem_addr(bar))
      : "memory");
}
#endif
