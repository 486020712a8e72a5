// ransac_common.cuh — the RANSAC shared by ransac_abs.cu (GP3P) and ransac_rel.cu (17-point and 5-point): on the device, everything
// of a problem's CTA from the selection state to the inlier mask (ransac_cta) and the two sources of samples it reads
// (SuppliedSamples: the caller's, SeededSamples: drawn per wave from the problem's seed by seeded_sample); on the host, the
// argument checks (check_ransac) and the staging, upload, launch, download and copy-out of a call (run_ransac).  The kernels
// supply only what differs: their per-problem setup, how a wave of samples is solved, the preparation of a hypothesis for
// scoring and the per-correspondence score.
#pragma once
#include <float.h>
#include <math.h>

#include <cub/block/block_scan.cuh>

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
  const unsigned long long* seed; int* drawn;                       // seeded calls: [n_prob], [n_prob][n_samples][kS] (nullable)
};

// ---- the seeded sampler (include/covins_b200.h, "Seeded samples"; oracle/sampler_oracle.c restates it) ----
// Philox4x64-10 (Salmon et al., SC'11; Random123's philox4x64 and numpy.random.Philox): counter c, key (k0, k1)
__device__ __forceinline__ void philox4x64_10(unsigned long long* c, unsigned long long k0, unsigned long long k1) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    if (r > 0) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
    const unsigned long long m0 = 0xD2E7470EE14C6C93ull, m1 = 0xCA5A826395121157ull;
    const unsigned long long hi0 = __umul64hi(m0, c[0]), lo0 = m0 * c[0], hi1 = __umul64hi(m1, c[2]), lo1 = m1 * c[2];
    const unsigned long long c1 = c[1], c3 = c[3];
    c[0] = hi1 ^ c1 ^ k0; c[1] = lo1; c[2] = hi0 ^ c3 ^ k1; c[3] = lo0;
  }
}

// Sample s of key (seed, stream): the ordered kS-subset of [0, m) (m >= kS) by a partial Fisher-Yates shuffle of the identity,
// j = i + (u_i (m - i)) >> 32, u_0, u_1, ... the 32-bit halves (low first) of the words of Philox blocks (s, 0, 0, 0),
// (s, 1, 0, 0), ...  Instead of an m-sized permutation, the kS positions written so far are kept as (position, value) pairs
// in registers; the last pair of a position holds its value.
template <int kS>
__device__ __forceinline__ void seeded_sample(unsigned long long seed, unsigned long long stream, unsigned m, unsigned long long s, int* out) {
  unsigned pos[kS], val[kS];
  unsigned long long blk[4];
#pragma unroll
  for (int i = 0; i < kS; i++) {
    if (i % 8 == 0) {
      blk[0] = s; blk[1] = (unsigned long long)(i / 8); blk[2] = 0; blk[3] = 0;
      philox4x64_10(blk, seed, stream);
    }
    const unsigned long long w = blk[(i % 8) / 2];
    const unsigned u = i % 2 ? (unsigned)(w >> 32) : (unsigned)w;
    const unsigned j = (unsigned)i + (unsigned)(((unsigned long long)u * (m - (unsigned)i)) >> 32);
    unsigned vi = (unsigned)i, vj = j;
#pragma unroll
    for (int e = 0; e < i; e++) {
      if (pos[e] == (unsigned)i) vi = val[e];
      if (pos[e] == j) vj = val[e];
    }
    out[i] = (int)vj;                  // perm[i] <-> perm[j]; position i is never read again
    pos[i] = j; val[i] = vi;
  }
}

// The caller's samples of a problem ([n_samples][kS], read from global memory)
template <int kS>
struct SuppliedSamples {
  static constexpr bool kSeeded = false;
  static constexpr int kSize = kS;
  const int* samples;
  int n_samples;
  __device__ void draw(int) const {}
  __device__ bool has(int s) const { return s < n_samples; }
  __device__ const int* sample(int s) const { return samples + kS * (size_t)s; }
};

// Samples drawn on the device: before a wave is solved, thread t < kWave draws sample base + t of the problem (stream 0, m = n)
// into shared memory, and copies it to drawn[s] for s < n_samples.  A problem with fewer than kS correspondences has none.
template <int kS>
struct SeededSamples {
  static constexpr bool kSeeded = true;
  static constexpr int kSize = kS;
  int (*w_smp)[kS];
  unsigned long long seed;
  int n, n_samples;
  int* drawn;   // this problem's [n_samples][kS], nullable
  __device__ void draw(int base) const {
    const int t = threadIdx.x, s = base + t;
    if (t >= kWave || n < kS) return;
    seeded_sample<kS>(seed, 0, (unsigned)n, (unsigned long long)s, w_smp[t]);
    if (drawn && s < n_samples)
      for (int i = 0; i < kS; i++) drawn[kS * (size_t)s + i] = w_smp[t][i];
  }
  __device__ bool has(int) const { return n >= kS; }
  __device__ const int* sample(int s) const { return w_smp[s % kWave]; }
};

// the sample source Src of problem pi (n correspondences) of a RANSAC call; samples: the problem's supplied samples
template <class Src>
__device__ __forceinline__ Src sample_source(const RansacOut& D, const int* samples, int pi, int n) {
  if constexpr (Src::kSeeded) {
    __shared__ int w_smp[kWave][Src::kSize];
    return Src{w_smp, D.seed[pi], n, D.n_samples, D.drawn ? D.drawn + (size_t)Src::kSize * pi * D.n_samples : nullptr};
  } else {
    return Src{samples, D.n_samples};
  }
}

// The RANSAC of problem blockIdx.x (n correspondences from off, kS indices per sample) after the kernel's per-problem setup.
// Samples are taken in waves of kWave: src.draw(base) prepares them (seeded: draws them), Pb.solve_wave(src, base, w_model,
// w_valid) writes the models (zero if invalid) and valid flags of samples base .. base + kWave - 1; every warp scores the wave's
// valid hypotheses against all correspondences (Pb.scorer(M), called by every lane of the warp, prepares hypothesis M and returns
// the score of correspondence i under it; warp-shuffle integer counts); thread 0 replays
// opengv's Ransac::computeModel over the wave in sample order, and the CTA stops as soon as the adaptive bound ends the selection
// (unless the per-sample outputs are requested), so the early stop saves the solver and scoring work of the samples it never
// reads.  Supplied samples also end the selection when they run out; seeded ones never do (a problem with fewer than kS
// correspondences draws none and selects nothing).  The CTA then writes the result and the selected model's inlier mask.
template <int kS, class Src, class Problem>
__device__ __forceinline__ void ransac_cta(const RansacOut& D, Problem& Pb, const Src& src, int off, int n) {
  const int pi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool all = D.sample_model != nullptr;
  __shared__ double w_model[kWave][12];
  __shared__ int w_valid[kWave], w_count[kWave];
  __shared__ double best_model[12], k_bound;
  __shared__ int best, best_n, it, used, running;
  __shared__ long long skipped;
  if (tid == 0) {
    best = -1; best_n = 0; it = 0; used = 0; skipped = 0; k_bound = (double)D.max_iterations;
    running = D.max_iterations > 0 && (!Src::kSeeded || n >= kS);
    for (int i = 0; i < 12; i++) best_model[i] = 0.0;
  }
  __syncthreads();
  const long long max_skip = 10LL * D.max_iterations;
  for (int base = 0; Src::kSeeded ? running || (all && base < D.n_samples) : base < D.n_samples && (running || all); base += kWave) {
    if constexpr (Src::kSeeded) {
      src.draw(base);
      __syncthreads();
    }
    Pb.solve_wave(src, base, w_model, w_valid);
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
      for (int h = 0; h < kWave && src.has(base + h); h++) {
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
      // (a seeded problem with fewer than kS correspondences never starts: it would draw forever)
      running = (!Src::kSeeded || n >= kS) && it < D.max_iterations && (double)it < k_bound && skipped < max_skip;
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

// ---- the glue kernels of the fused verification calls (ransac_rel.cu, geom_kernels.cu): one CTA of kGlueThreads per unit ----
constexpr int kGlueThreads = 256;
using GlueScan = cub::BlockScan<int, kGlueThreads>;

// emit(i, rank) for every i < n with flag(i), rank = the number of flagged indices before i (a CTA-wide scan in chunks of
// kGlueThreads); returns the number of flagged indices to every thread
template <class Flag, class Emit>
__device__ int scan_emit(int n, const Flag& flag, const Emit& emit) {
  __shared__ typename GlueScan::TempStorage tmp;
  __shared__ int carry;
  __syncthreads();
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int b = 0; b < n; b += kGlueThreads) {
    const int i = b + threadIdx.x;
    const int f = i < n && flag(i);
    int rank, total;
    GlueScan(tmp).ExclusiveSum(f, rank, total);
    if (f) emit(i, carry + rank);
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
  return carry;
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
// samples (k indices each).  With n_prob = 0 only the sizes are checked.  A seeded call (seeded) instead takes no samples and
// one seed per problem.
template <class Problems, class Result>
int check_ransac(cvb_ctx* ctx, const char* name, const Problems* p, int max_iterations, const Result* r, int k, bool seeded = false,
                 const uint64_t* seed = nullptr) {
  CVB_REQUIRE(ctx, p && r && p->n_prob >= 0 && p->n_samples >= 0 && max_iterations >= 0, "%s: bad arguments", name);
  CVB_REQUIRE(ctx, max_iterations <= INT32_MAX / 10, "%s: max_iterations too large", name);
  CVB_REQUIRE(ctx, !seeded || !p->samples, "%s: samples must be NULL (the samples are drawn from the seeds)", name);
  CVB_REQUIRE(ctx, !seeded || max_iterations <= (INT32_MAX - kWave) / 11, "%s: max_iterations too large", name);   // sample numbers fit an int
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  CVB_REQUIRE(ctx, p->prob_ptr && r->best_sample && r->best_model && r->best_count && r->iterations && r->consumed, "%s: null required pointer", name);
  CVB_REQUIRE(ctx, (r->sample_model != nullptr) == (r->sample_valid != nullptr) && (r->sample_model != nullptr) == (r->sample_count != nullptr),
              "%s: sample_model / sample_valid / sample_count are requested together", name);
  CVB_REQUIRE(ctx, ptr_ok(p->prob_ptr, n_prob), "%s: prob_ptr does not start at 0 or decreases", name);
  if (seeded) {
    CVB_REQUIRE(ctx, seed, "%s: null seed", name);
    return CVB_OK;
  }
  CVB_REQUIRE(ctx, ns == 0 || p->samples, "%s: null samples", name);
  return check_samples(ctx, name, p->samples, p->prob_ptr, n_prob, ns, k);
}

// the selection parameters of a RANSAC call
inline void set_selection(RansacOut& O, int ns, int max_iterations, double threshold, double probability) {
  O.n_samples = ns; O.max_iterations = max_iterations; O.threshold = threshold; O.log_p = log(1.0 - probability);
}

// the selection parameters and the result pointers (device) of a RANSAC call; inlier_mask nullable
inline void set_outputs(RansacOut& O, int ns, int max_iterations, double threshold, double probability, int* best_sample, double* best_model,
                        int* best_count, int* iterations, int* consumed, uint8_t* inlier_mask) {
  set_selection(O, ns, max_iterations, threshold, probability);
  O.best_sample = best_sample; O.best_model = best_model; O.best_count = best_count; O.iterations = iterations; O.consumed = consumed;
  O.inlier_mask = inlier_mask;
}

// The launcher: kernel on device inputs and outputs D (one CTA per problem, smem bytes of dynamic shared memory) on ctx's stream.
template <class Dev>
int launch_ransac(cvb_ctx* ctx, void (*kernel)(Dev), size_t smem, const Dev& D, int n_prob) {
  kernel<<<n_prob, kThreads, smem, ctx->stream>>>(D);
  CVB_CHECK_LAUNCH(ctx);
  return CVB_OK;
}

// cameras as the kernels read them: each one's offset (3) directly followed by its rotation (9, row-major)
inline std::vector<double> pack_cams(const double* off, const double* rot, size_t n) {
  std::vector<double> c(n * 12);
  for (size_t j = 0; j < n; j++) {
    memcpy(&c[12 * j], off + 3 * j, 24);
    memcpy(&c[12 * j + 3], rot + 9 * j, 72);
  }
  return c;
}

// The rest of a RANSAC call whose inputs are bound in B (to D's pointers): its outputs bound after them, one upload,
// launch_ransac of kernel with D and its common part filled here, one download into r.  A seeded call may also ask for its
// drawn samples (drawn, k indices each, -1 where not drawn).
template <class Dev, class Result>
int run_ransac(cvb_ctx* ctx, cvb_block& B, void (*kernel)(Dev), size_t smem, Dev& D, int n_prob, int ns, size_t N, double threshold,
               int max_iterations, double probability, Result* r, int32_t* drawn = nullptr, int k = 0) {
  const size_t S_all = (size_t)n_prob * ns;
  RansacOut& O = D.o;
  set_selection(O, ns, max_iterations, threshold, probability);
  B.out(O.best_model, r->best_model, (size_t)n_prob * 12); B.out(O.best_sample, r->best_sample, n_prob); B.out(O.best_count, r->best_count, n_prob);
  B.out(O.iterations, r->iterations, n_prob); B.out(O.consumed, r->consumed, n_prob);
  if (r->inlier_mask) B.out(O.inlier_mask, r->inlier_mask, N);
  if (r->sample_model) { B.out(O.sample_model, r->sample_model, S_all * 12); B.out(O.sample_valid, r->sample_valid, S_all); B.out(O.sample_count, r->sample_count, S_all); }
  if (drawn) B.out(O.drawn, drawn, S_all * k);
  if (const int rc = B.place()) return rc;
  if (const int rc = B.upload()) return rc;
  if (drawn) CVB_CUDA(ctx, cudaMemsetAsync(O.drawn, 0xff, S_all * k * 4, ctx->stream));
  if (const int rc = launch_ransac(ctx, kernel, smem, D, n_prob)) return rc;
  return B.download();
}

}  // namespace
