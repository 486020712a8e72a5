// ransac_common.cuh — the RANSAC shared by ransac_abs.cu (GP3P) and ransac_rel.cu (17-point and 5-point): on the device, everything
// of a problem's CTA from the selection state to the inlier mask (ransac_cta); on the host, the argument checks (check_ransac)
// and the staging, upload, launch, download and copy-out of a call (run_ransac).  The kernels supply only what differs: their
// per-problem setup, how a wave of samples is solved, the preparation of a hypothesis for scoring and the per-correspondence
// score.
#pragma once
#include <float.h>
#include <math.h>

#include "cvb_internal.cuh"
#include "geom_common.cuh"

namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32, kWave = 64;
constexpr unsigned kFull = 0xffffffffu;

// the selection parameters and the outputs of a RANSAC call (device pointers)
struct RansacOut {
  int n_samples, max_iterations;
  double threshold, log_p;
  int* best_sample; double* best_model; int* best_count; int* iterations; int* consumed;
  uint8_t* inlier_mask;                                             // nullable
  double* sample_model; uint8_t* sample_valid; int* sample_count;   // nullable together
};

// The RANSAC of problem blockIdx.x (n correspondences from off, kS indices per sample) after the kernel's per-problem setup.
// Samples are taken in waves of kWave: Pb.solve_wave(base, w_model, w_valid) writes the models (zero if invalid) and valid flags
// of samples base .. base + kWave - 1; every warp scores the wave's valid hypotheses against all correspondences (Pb.scorer(M),
// called by every lane of the warp, prepares hypothesis M and returns the score of correspondence i under it; warp-shuffle
// integer counts); thread 0 replays
// opengv's Ransac::computeModel over the wave in sample order, and the CTA stops as soon as the adaptive bound ends the selection
// (unless the per-sample outputs are requested), so the early stop saves the solver and scoring work of the samples it never
// reads.  The CTA then writes the result and the selected model's inlier mask.
template <int kS, class Problem>
__device__ __forceinline__ void ransac_cta(const RansacOut& D, Problem& Pb, int off, int n) {
  const int pi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool all = D.sample_model != nullptr;
  __shared__ double w_model[kWave][12];
  __shared__ int w_valid[kWave], w_count[kWave];
  __shared__ double best_model[12], k_bound;
  __shared__ int best, best_n, it, used, running;
  __shared__ long long skipped;
  if (tid == 0) {
    best = -1; best_n = 0; it = 0; used = 0; skipped = 0; k_bound = (double)D.max_iterations;
    running = D.max_iterations > 0;
    for (int i = 0; i < 12; i++) best_model[i] = 0.0;
  }
  __syncthreads();
  const long long max_skip = 10LL * D.max_iterations;
  for (int base = 0; base < D.n_samples && (running || all); base += kWave) {
    Pb.solve_wave(base, w_model, w_valid);
    __syncthreads();
    for (int h = warp; h < kWave; h += kWarps) {
      int cnt = 0;
      if (w_valid[h]) {
        const auto score = Pb.scorer(w_model[h]);
        for (int i = lane; i < n; i += 32) cnt += score(i) < D.threshold;
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(kFull, cnt, o);   // integer: order-independent
        __syncwarp();
      }
      if (lane == 0) w_count[h] = cnt;
    }
    __syncthreads();
    if (all && tid < kWave && base + tid < D.n_samples) {
      const size_t g = (size_t)pi * D.n_samples + base + tid;
      for (int i = 0; i < 12; i++) D.sample_model[12 * g + i] = w_model[tid][i];
      D.sample_valid[g] = (uint8_t)w_valid[tid]; D.sample_count[g] = w_count[tid];
    }
    if (tid == 0) {   // placerec.ransac_select over the valid samples, opengv's skipped_count for the invalid ones
      for (int h = 0; h < kWave && base + h < D.n_samples; h++) {
        running = it < D.max_iterations && (double)it < k_bound && skipped < max_skip;
        if (!running) break;
        used++;
        if (!w_valid[h]) { skipped++; continue; }
        const int c = w_count[h];
        if (c > best_n) {
          best_n = c; best = base + h;
          for (int i = 0; i < 12; i++) best_model[i] = w_model[h][i];
          const double w = __ddiv_rn((double)c, (double)n);
          double wp = w;   // w^kS, multiplied left to right
          for (int e = 1; e < kS; e++) wp = mul(wp, w);
          double pno = sub(1.0, wp);
          pno = pno > DBL_EPSILON ? pno : DBL_EPSILON;
          pno = pno < 1.0 - DBL_EPSILON ? pno : 1.0 - DBL_EPSILON;
          k_bound = __ddiv_rn(D.log_p, log(pno));
        }
        it++;
      }
      running = it < D.max_iterations && (double)it < k_bound && skipped < max_skip;
    }
    __syncthreads();
  }
  if (tid == 0) {
    D.best_sample[pi] = best; D.best_count[pi] = best_n; D.iterations[pi] = it; D.consumed[pi] = used;
    for (int i = 0; i < 12; i++) D.best_model[12 * (size_t)pi + i] = best_model[i];
  }
  if (D.inlier_mask) {
    if (best >= 0) {
      const auto score = Pb.scorer(best_model);
      for (int i = tid; i < n; i += kThreads) D.inlier_mask[off + i] = score(i) < D.threshold;
    } else {
      for (int i = tid; i < n; i += kThreads) D.inlier_mask[off + i] = 0;
    }
  }
}

bool ptr_ok(const int32_t* p, int n) {
  if (p[0] != 0) return false;
  for (int i = 0; i < n; i++)
    if (p[i + 1] < p[i]) return false;
  return true;
}

// every sample index of a problem with at least k correspondences in [0, n); the samples of smaller problems, and of problems
// flagged in skip (nullable), are not read
int check_samples(cvb_ctx* ctx, const char* name, const int32_t* samples, const int32_t* prob_ptr, int n_prob, int ns, int k,
                  const uint8_t* skip = nullptr) {
  for (int i = 0; i < n_prob; i++) {
    const int n = prob_ptr[i + 1] - prob_ptr[i];
    if (n < k || (skip && skip[i])) continue;
    const int32_t* s = samples + k * (size_t)i * ns;
    for (size_t j = 0; j < k * (size_t)ns; j++)
      CVB_REQUIRE(ctx, s[j] >= 0 && s[j] < n, "%s: sample index %d out of range [0, %d) in problem %d", name, s[j], n, i);
  }
  return CVB_OK;
}

// The argument checks of a RANSAC call that do not depend on its problem type: the sizes, the result pointers, prob_ptr and the
// samples (k indices each).  With n_prob = 0 only the sizes are checked.
template <class Problems, class Result>
int check_ransac(cvb_ctx* ctx, const char* name, const Problems* p, int max_iterations, const Result* r, int k) {
  CVB_REQUIRE(ctx, p && r && p->n_prob >= 0 && p->n_samples >= 0 && max_iterations >= 0, "%s: bad arguments", name);
  CVB_REQUIRE(ctx, max_iterations <= INT32_MAX / 10, "%s: max_iterations too large", name);
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  CVB_REQUIRE(ctx, p->prob_ptr && r->best_sample && r->best_model && r->best_count && r->iterations && r->consumed, "%s: null required pointer", name);
  CVB_REQUIRE(ctx, (r->sample_model != nullptr) == (r->sample_valid != nullptr) && (r->sample_model != nullptr) == (r->sample_count != nullptr),
              "%s: sample_model / sample_valid / sample_count are requested together", name);
  CVB_REQUIRE(ctx, ptr_ok(p->prob_ptr, n_prob), "%s: prob_ptr does not start at 0 or decreases", name);
  CVB_REQUIRE(ctx, ns == 0 || p->samples, "%s: null samples", name);
  return check_samples(ctx, name, p->samples, p->prob_ptr, n_prob, ns, k);
}

// The rest of a RANSAC call whose inputs are staged in St: its outputs staged after them, one upload into workspace slot
// ws_slot, one launch of kernel (one CTA per problem, smem bytes of dynamic shared memory) with the device struct
// inputs(device block) and its common part filled here, one download, the copy-out into r.
template <class Dev, class Result, class Inputs>
int run_ransac(cvb_ctx* ctx, int ws_slot, void (*kernel)(Dev), size_t smem, Stager& St, const Inputs& inputs, int n_prob, int ns, size_t N,
               double threshold, int max_iterations, double probability, Result* r) {
  const size_t S_all = (size_t)n_prob * ns;
  const bool all = r->sample_model != nullptr;
  const size_t in_bytes = St.h.size();
  const size_t o_bm = St.reserve((size_t)n_prob * 96), o_bs = St.reserve((size_t)n_prob * 4), o_bc = St.reserve((size_t)n_prob * 4),
               o_it = St.reserve((size_t)n_prob * 4), o_us = St.reserve((size_t)n_prob * 4), o_mask = r->inlier_mask ? St.reserve(N) : 0,
               o_sm = all ? St.reserve(S_all * 96) : 0, o_sv = all ? St.reserve(S_all) : 0, o_sc = all ? St.reserve(S_all * 4) : 0;
  const size_t total = St.h.size();
  unsigned char* d = (unsigned char*)cvb_ws(ctx, ws_slot, total);
  unsigned char* hpin = (unsigned char*)cvb_pinned(ctx, total);
  if (!d || !hpin) return CVB_ERR_CUDA;
  memcpy(hpin, St.h.data(), in_bytes);
  Dev D = inputs(d);
  RansacOut& O = D.o;
  O.n_samples = ns; O.max_iterations = max_iterations; O.threshold = threshold; O.log_p = log(1.0 - probability);
  O.best_sample = (int*)(d + o_bs); O.best_model = (double*)(d + o_bm); O.best_count = (int*)(d + o_bc); O.iterations = (int*)(d + o_it);
  O.consumed = (int*)(d + o_us); O.inlier_mask = r->inlier_mask ? d + o_mask : nullptr;
  if (all) { O.sample_model = (double*)(d + o_sm); O.sample_valid = d + o_sv; O.sample_count = (int*)(d + o_sc); }
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemcpyAsync(d, hpin, in_bytes, cudaMemcpyHostToDevice, st));
  kernel<<<n_prob, kThreads, smem, st>>>(D);
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaMemcpyAsync(hpin + o_bm, d + o_bm, total - o_bm, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(r->best_model, hpin + o_bm, (size_t)n_prob * 96); memcpy(r->best_sample, hpin + o_bs, (size_t)n_prob * 4);
  memcpy(r->best_count, hpin + o_bc, (size_t)n_prob * 4); memcpy(r->iterations, hpin + o_it, (size_t)n_prob * 4);
  memcpy(r->consumed, hpin + o_us, (size_t)n_prob * 4);
  if (r->inlier_mask) memcpy(r->inlier_mask, hpin + o_mask, N);
  if (all) {
    memcpy(r->sample_model, hpin + o_sm, S_all * 96); memcpy(r->sample_valid, hpin + o_sv, S_all); memcpy(r->sample_count, hpin + o_sc, S_all * 4);
  }
  return CVB_OK;
}

}  // namespace
