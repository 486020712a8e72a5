// cvb_internal.cuh — ctx, error plumbing and small device helpers shared by all translation units of
// libcovins_b200.so.  Not part of the public boundary (that is include/covins_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/covins_b200.h"

struct cvb_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  int sm_count = 132;
  int64_t launches = 0;
  std::string err;
  // pinned host staging (grow-only), used by one cvb_block at a time (pin_busy)
  void* h_pin = nullptr;
  size_t h_pin_cap = 0;
  bool pin_busy = false;
  void* ba = nullptr;  // BA state (owned by ba_*.cu)
  // every extern "C" entry point holds this lock for its duration (cvb_device_guard): a ctx may be shared between host
  // threads — calls on one ctx are serialised, concurrency comes from one ctx per thread
  mutable std::recursive_mutex mtx;
};

// cudaFuncSetAttribute applies to the CURRENT device: one flag per (call site, device), so that a process that opens contexts
// on several GPUs raises the dynamic shared-memory limit on each of them
// Call sites hold `mtx` around first() and the attribute set-up, so that a concurrent first call on the
// same device (several contexts of one device driven from their own threads) waits until the attributes are set instead of
// launching before them.
struct cvb_once_per_device {
  std::mutex mtx;
  std::atomic<bool> done[64];
  cvb_once_per_device() { for (auto& d : done) d.store(false); }
  bool first(int device) {
    if (device < 0 || device >= 64) return true;
    return !done[device].exchange(true);
  }
};

int cvb_fail(cvb_ctx* ctx, int code, const char* fmt, ...);

// One call's device memory: one allocation from the device's stream-ordered pool on the stream the call's work runs on
// (st), freed there when the block goes out of scope, early returns included.  So the scratch of a nested call, or of a
// _dev call on a caller's stream, is never shared with another call.  Arrays are bound to pointer variables, which place()
// sets: the inputs, then the scratch, then the outputs, each in declaration order, every array on a 256-byte boundary.
//   in(p, src, n)          uploaded by upload(); src == nullptr: filled through host(p) between place() and upload()
//   tmp(p, n)              device only
//   out(p, dst, n)         downloaded by download() and copied to dst; dst == nullptr: left on the device
//   out_host(p, n, want)   downloaded (when want) for the call to read through host(p) after download()
// download() moves one range, from the first output to the end of the last one wanted: optional outputs are declared last.
// Nothing is zeroed; pool memory holds whatever an earlier user left.  Inputs and downloaded outputs are staged in the ctx's
// pinned buffer, which one block holds at a time: a second staging block on the same ctx is refused.  A direct block
// (staged = false) instead copies each input from its src and each output to its dst, one copy per array and no host copy:
// for calls whose arrays are large (rows of descriptors, possibly in the caller's pinned memory); it has no host().
struct cvb_block {
  cvb_block(cvb_ctx* c, cudaStream_t s, bool staged = true) : ctx(c), st(s), staged(staged) {}
  ~cvb_block() {
    if (d) cudaFreeAsync(d, st);
    if (h) ctx->pin_busy = false;
  }
  cvb_block(const cvb_block&) = delete;
  cvb_block& operator=(const cvb_block&) = delete;

  template <class T> void in(T*& p, const void* src, size_t n) { arrs.push_back({(void**)&p, n * sizeof(T), kIn, src, nullptr, true}); }
  template <class T> void tmp(T*& p, size_t n) { arrs.push_back({(void**)&p, n * sizeof(T), kTmp, nullptr, nullptr, false}); }
  template <class T> void out(T*& p, void* dst, size_t n) { arrs.push_back({(void**)&p, n * sizeof(T), kOut, nullptr, dst, dst != nullptr}); }
  template <class T> void out_host(T*& p, size_t n, bool want = true) { arrs.push_back({(void**)&p, n * sizeof(T), kOut, nullptr, nullptr, want}); }

  int place();      // the allocation; sets every bound pointer and copies the inputs' src into the pinned buffer
  int upload();     // one H2D copy of the inputs
  int download();   // one D2H copy of the wanted outputs, a synchronisation of st, the copies into the callers' arrays
  // the pinned copy of bound input or output p
  template <class T> T* host(const T* p) const {
    const size_t o = (const unsigned char*)p - d;
    return (T*)(o < out_lo ? h + o : h + in_hi + (o - out_lo));
  }

 private:
  enum { kIn, kTmp, kOut };
  struct Arr {
    void** p;
    size_t bytes;
    int kind;
    const void* src;
    void* dst;
    bool want;
    size_t off;
  };
  cvb_ctx* ctx;
  cudaStream_t st;
  bool staged;
  std::vector<Arr> arrs;
  unsigned char* d = nullptr;   // device block
  unsigned char* h = nullptr;   // pinned: [0, in_hi) the inputs, then [out_lo, out_hi) of the outputs
  size_t in_hi = 0, out_lo = 0, out_hi = 0;
};

// match_kernels.cu: the fused 2-NN + ratio filter of cvb_match_hamming_batch for n_pairs pairs of keyframes of one device
// descriptor table d_desc in one launch on ctx->stream.  d_pairs [n_pairs][5] = (query row0, query rows, train row0, train rows,
// output offset); pair s writes match_train / match_dist [offset + query] and n_matches [s]; max_nq: the largest query count.
// cvb_match_l2_pairs_dev: the same for cvb_match_l2_batch on the u8 SIFT layout, d_desc [rows][128] (16-byte aligned).
int cvb_match_hamming_pairs_dev(cvb_ctx* ctx, const uint8_t* d_desc, const int32_t* d_pairs, int n_pairs, int max_nq, float thr, float ratio,
                                int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches);
int cvb_match_l2_pairs_dev(cvb_ctx* ctx, const uint8_t* d_desc, const int32_t* d_pairs, int n_pairs, int max_nq, float thr, float ratio,
                           int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches);
// cvb_match_dev: the fused 2-NN + ratio filter of cvb_match_{hamming,l2}_batch on device rows, metric 0 = Hamming (32-byte
// rows), 1 = L2 (the u8 SIFT layout cvb_knn_l2_u8_batch_dev takes); outputs as cvb_match_hamming_batch_dev, on st.  d_xt /
// d_seg_tile: the train rows' resident operand tiles (cvb_tc::expand_tiles), or nullptr when they have none.  The map
// database matches its keyframes through it.
int cvb_match_dev(cvb_ctx* ctx, int metric, const uint8_t* d_q, int nq, const uint8_t* d_t, const int32_t* d_seg_ptr,
                  const int32_t* h_seg_ptr, int n_seg, const uint8_t* d_xt, const int32_t* d_seg_tile, float thr, float ratio,
                  int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches, cudaStream_t st);

// ransac_rel.cu: SIFT rows (CV_32F) to the u8 layout of the L2 kernels on the host; false if a value is not an integer in [0, 255]
bool cvb_quantize_sift(const float* src, size_t n, uint8_t* dst);

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

// map_graph.cu: cvb_covisibility with the pair budget as an argument.  The shared-landmark pairs are expanded, sorted and
// counted at most `pair_budget` at a time and the partial counts merged by key; the result does not depend on the budget
// (tests force several chunks at small size through this argument; the public entry point passes the default).
int cvb_covisibility_budgeted(cvb_ctx* ctx, int K, int L, const int32_t* lm_obs_ptr, const int32_t* obs_kf, const uint8_t* obs_skip,
                              const uint8_t* lm_valid, int min_weight, int32_t* nbr_ptr, int32_t* nbr_kf, int32_t* nbr_w, int64_t cap,
                              int64_t* n_total, int64_t pair_budget);

// Every keyframe's camera as the reprojection kernels read it (bam::reproj): the extr [K][7], intr [K][4] and
// dist [K][4] of its calibration cam_of_kf[k], model = camera | distortion << 8, xi (0 for a pinhole camera).  The bundle
// adjustment and cvb_landmark_outliers stage it here, so both project through the same numbers.  CVB_ERR_INVALID for a
// calibration index out of range, CVB_ERR_UNSUPPORTED (the reference's messages) for an unknown camera or distortion model.
struct cvb_kf_cameras {
  std::vector<double> extr, intr, dist, xi;
  std::vector<int> model;
};

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

// The context's pinned staging buffer, grown to at least `bytes` (nullptr on failure, ctx->err set).  It and the block's
// functions are defined here, in the header, so that a translation unit built without ctx.cu (the Cholesky test
// harnesses) needs only cvb_fail.
inline void* cvb_pinned(cvb_ctx* ctx, size_t bytes) {
  if (bytes <= ctx->h_pin_cap && ctx->h_pin) return ctx->h_pin;
  if (ctx->h_pin) {
    cudaStreamSynchronize(ctx->stream);
    cudaFreeHost(ctx->h_pin);
    ctx->h_pin = nullptr;
    ctx->h_pin_cap = 0;
  }
  size_t want = bytes < 4096 ? 4096 : bytes + bytes / 4;
  cudaError_t e = cudaMallocHost(&ctx->h_pin, want);
  if (e != cudaSuccess) {
    cvb_fail(ctx, CVB_ERR_CUDA, "cudaMallocHost(%zu) failed: %s", want, cudaGetErrorString(e));
    ctx->h_pin = nullptr;
    return nullptr;
  }
  ctx->h_pin_cap = want;
  return ctx->h_pin;
}

inline int cvb_block::place() {
  const auto align = [](size_t o) { return (o + 255) & ~size_t(255); };
  size_t top = 0;
  for (int kind : {kIn, kTmp, kOut}) {
    if (kind == kOut) out_lo = out_hi = top = align(top);
    for (Arr& a : arrs) {
      if (a.kind != kind) continue;
      a.off = align(top);
      top = a.off + a.bytes;
      if (kind == kIn) in_hi = top;
      if (kind == kOut && a.want) out_hi = top;
    }
  }
  if (staged && (in_hi || out_hi > out_lo)) {
    if (ctx->pin_busy) return cvb_fail(ctx, CVB_ERR_INVALID, "host staging nested in another call's host staging on the same ctx");
    if (!(h = (unsigned char*)cvb_pinned(ctx, in_hi + (out_hi - out_lo)))) return CVB_ERR_CUDA;
    ctx->pin_busy = true;
    for (const Arr& a : arrs)
      if (a.kind == kIn && a.src && a.bytes) memcpy(h + a.off, a.src, a.bytes);
  }
  const cudaError_t e = cudaMallocAsync((void**)&d, top > 256 ? top : 256, st);
  if (e != cudaSuccess) {
    d = nullptr;
    return cvb_fail(ctx, CVB_ERR_CUDA, "cudaMallocAsync(%zu) failed: %s", top, cudaGetErrorString(e));
  }
  for (const Arr& a : arrs) *a.p = d + a.off;
  return CVB_OK;
}

inline int cvb_block::upload() {
  if (staged) {
    if (in_hi) CVB_CUDA(ctx, cudaMemcpyAsync(d, h, in_hi, cudaMemcpyHostToDevice, st));
    return CVB_OK;
  }
  for (const Arr& a : arrs)
    if (a.kind == kIn && a.src && a.bytes) CVB_CUDA(ctx, cudaMemcpyAsync(d + a.off, a.src, a.bytes, cudaMemcpyHostToDevice, st));
  return CVB_OK;
}

inline int cvb_block::download() {
  if (!staged) {
    for (const Arr& a : arrs)
      if (a.kind == kOut && a.dst && a.bytes) CVB_CUDA(ctx, cudaMemcpyAsync(a.dst, d + a.off, a.bytes, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaStreamSynchronize(st));
    return CVB_OK;
  }
  if (out_hi > out_lo) CVB_CUDA(ctx, cudaMemcpyAsync(h + in_hi, d + out_lo, out_hi - out_lo, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  for (const Arr& a : arrs)
    if (a.kind == kOut && a.dst && a.bytes) memcpy(a.dst, h + in_hi + (a.off - out_lo), a.bytes);
  return CVB_OK;
}

inline int cvb_stage_kf_cameras(cvb_ctx* ctx, const cvb_ba_problem* p, cvb_kf_cameras& out) {
  const int K = p->K;
  out.extr.assign((size_t)7 * K, 0.0); out.intr.assign((size_t)4 * K, 0.0); out.dist.assign((size_t)4 * K, 0.0);
  out.xi.assign(K, 0.0); out.model.assign(K, 0);
  for (int k = 0; k < K; k++) {
    const int c = p->cam_of_kf ? p->cam_of_kf[k] : 0;
    CVB_REQUIRE(ctx, c >= 0 && c < p->n_cam, "cam_of_kf out of range");
    const int cam = p->cam_model ? p->cam_model[c] : 0, dm = p->dist_model ? p->dist_model[c] : 0;
    // optimization_be.cpp:186-231: "Unknown projection type" / "Unknown distortion type" → exit(-1) in the reference
    if (cam < 0 || cam > 1) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown projection type (%d) for camera %d", cam, c);
    if (dm < 0 || dm > 2) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown distortion type (%d) for camera %d", dm, c);
    CVB_REQUIRE(ctx, cam == 0 || p->cam_xi, "unified projection camera needs cam_xi");
    out.model[k] = cam | (dm << 8);
    out.xi[k] = (cam == 1) ? p->cam_xi[c] : 0.0;
    memcpy(&out.extr[7 * (size_t)k], p->extr + 7 * (size_t)c, 7 * sizeof(double));
    memcpy(&out.intr[4 * (size_t)k], p->intr + 4 * (size_t)c, 4 * sizeof(double));
    memcpy(&out.dist[4 * (size_t)k], p->dist + 4 * (size_t)c, 4 * sizeof(double));
  }
  return CVB_OK;
}

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
