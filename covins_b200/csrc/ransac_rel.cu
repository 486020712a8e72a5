// ransac_rel.cu — the non-central relative-pose RANSAC of RelNonCentralPosSolver::computeNonCentralRelPose (17-point,
// RelNonCentralPosSolver.cpp:146-173; the COVINS_G verification of a place-recognition candidate, each side a rig of a
// keyframe and its neighbours) on the GPU from caller-supplied samples: the 17-point solve per sample, scoring per camera pair
// and the sequential model selection of opengv's Ransac::computeModel, for a batch of problems (candidates) in one launch.
//
// One CTA per problem, both rigs staged in shared memory.  Samples are taken in waves of kWave: each warp solves one sample at
// a time (lane k owns column k of A^T in its warp's shared-memory area, every norm and dot product is a sequential sum inside
// one lane), then every warp scores the wave's hypotheses against all correspondences (camera-pair models in the warp's area,
// warp-shuffle integer counts), thread 0 replays the selection over the wave in sample order, and the CTA stops as soon as the
// adaptive bound ends the selection.  The CTA then writes the selected model's inlier mask.
//
// Only + - * / and sqrt as explicit non-fused intrinsics, fixed iteration counts: the results are bit-identical to the plain
// IEEE restatement compiled with -ffp-contract=off (oracle/ransac_rel_oracle.c, whose header states the problem and its assumptions;
// so does include/covins_b200.h).
#include <float.h>
#include <math.h>

#include "cvb_internal.cuh"
#include "geom_common.cuh"

namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32, kWave = 64, kSample = 17, kMaxCams = CVB_REL_MAX_CAMS;
constexpr int kPolarIters = 12;
constexpr double kRankTol = 1e-10;
// per-warp shared-memory area (doubles): the solver's arrays, or the camera-pair models (12 each) while scoring
constexpr int kLd = 19;   // leading dimension of A^T's columns (17 lanes hit distinct banks)
constexpr int oAt = 0, oDm = oAt + kSample * kLd, oX = oDm + kSample * 12, oAl = oX + 18, oVt = oAl + kSample, oGh = oVt + kSample,
              oR = oGh + kSample * 4, kSolveArea = oR + 9;
constexpr int kPairArea = 12;
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ void cross3(const double* a, const double* b, double* o) {
  o[0] = sub(mul(a[1], b[2]), mul(a[2], b[1]));
  o[1] = sub(mul(a[2], b[0]), mul(a[0], b[2]));
  o[2] = sub(mul(a[0], b[1]), mul(a[1], b[0]));
}

// d = Rc f, m = c x d; cam = offset (3) then Rc (9, row-major)
__device__ __forceinline__ void plucker(const double* cam, const double* f, double* d, double* m) {
  const double* cr = cam + 3;
#pragma unroll
  for (int r = 0; r < 3; r++) d[r] = dot3(cr[3 * r], cr[3 * r + 1], cr[3 * r + 2], f);
  cross3(cam, d, m);
}

// camera-pair model [R_p|t_p] of the rig-frame model M: R_p = Rc1^T R Rc2, t_p = Rc1^T (R c2 + t - c1)
__device__ void pair_model(const double* M, const double* cam1, const double* cam2, double* P) {
  const double *co1 = cam1, *cr1 = cam1 + 3, *co2 = cam2, *cr2 = cam2 + 3;
  double RR[9], u[3];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) RR[3 * r + c] = add(add(mul(M[4 * r], cr2[c]), mul(M[4 * r + 1], cr2[3 + c])), mul(M[4 * r + 2], cr2[6 + c]));
  for (int r = 0; r < 3; r++) u[r] = sub(add(dot3(M[4 * r], M[4 * r + 1], M[4 * r + 2], co2), M[4 * r + 3]), co1[r]);
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) P[4 * r + c] = add(add(mul(cr1[r], RR[c]), mul(cr1[3 + r], RR[3 + c])), mul(cr1[6 + r], RR[6 + c]));
    P[4 * r + 3] = dot3(cr1[r], cr1[3 + r], cr1[6 + r], u);
  }
}

__device__ __forceinline__ bool finite3(const double* v) { return isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]); }

// the hypothesis of sample s (17 problem-local indices), solved by one warp in its area W; lane 0 writes the model.  Returns the
// (warp-uniform) valid flag.
__device__ bool rel17(const int* s, int n, const double* F1, const double* F2, const int* C1, const int* C2, const double* rig1,
                      const double* rig2, bool rigs_finite, double* W, double* model, int lane) {
  if (n < kSample || !rigs_finite) return false;
  const int idx = lane < kSample ? s[lane] : 0;
  bool ok = true;
  if (lane < kSample) {
    for (int j = 0; j < kSample; j++) ok &= j == lane || s[j] != idx;
    ok &= finite3(F1 + 3 * (size_t)idx) && finite3(F2 + 3 * (size_t)idx);
  }
  if (!__all_sync(kFull, ok)) return false;
  double *At = W + oAt, *dm = W + oDm, *x = W + oX, *al = W + oAl, *vt = W + oVt, *gh = W + oGh, *Rm = W + oR;
  if (lane < kSample) {   // row `lane` of A = column `lane` of A^T
    double* q = dm + 12 * lane;
    plucker(rig1 + 12 * C1[idx], F1 + 3 * (size_t)idx, q, q + 3);
    plucker(rig2 + 12 * C2[idx], F2 + 3 * (size_t)idx, q + 6, q + 9);
    double* col = At + kLd * lane;
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) {
        col[3 * a + b] = mul(q[a], q[6 + b]);
        col[9 + 3 * a + b] = add(mul(q[a], q[9 + b]), mul(q[3 + a], q[6 + b]));
      }
  }
  __syncwarp();
  // Householder QR of A^T: step k reflects rows k..17; v_k overwrites column k from row k, r_kk = al[k], |v_k|^2 = vt[k]
  for (int k = 0; k < kSample; k++) {
    if (lane == k) {
      double* col = At + kLd * k;
      double ss = 0.0;
      for (int i = k; i < 18; i++) ss = i == k ? mul(col[i], col[i]) : add(ss, mul(col[i], col[i]));
      const double sigma = __dsqrt_rn(ss), ak = col[k];
      const double alpha = ak >= 0.0 ? -sigma : sigma;
      col[k] = sub(ak, alpha);
      al[k] = alpha;
      vt[k] = mul(2.0, add(ss, mul(fabs(ak), sigma)));
    }
    __syncwarp();
    if (lane > k && lane < kSample) {
      const double* v = At + kLd * k;
      double* a = At + kLd * lane;
      double dot = 0.0;
      for (int i = k; i < 18; i++) dot = i == k ? mul(v[i], a[i]) : add(dot, mul(v[i], a[i]));
      const double c = __ddiv_rn(mul(2.0, dot), vt[k]);
      for (int i = k; i < 18; i++) a[i] = sub(a[i], mul(c, v[i]));
    }
    __syncwarp();
  }
  int good = 0;
  if (lane == 0) {   // rank: every |r_kk| >= kRankTol * max |r_kk|
    double rmax = 0.0;
    for (int k = 0; k < kSample; k++) rmax = fabs(al[k]) > rmax ? fabs(al[k]) : rmax;
    good = rmax > 0.0;
    for (int k = 0; k < kSample; k++)
      if (!(fabs(al[k]) >= mul(kRankTol, rmax))) good = 0;
  }
  if (!__shfl_sync(kFull, good, 0)) return false;
  // x = H_0 H_1 ... H_16 e18 (every lane forms the same dot product; lane i updates x[i])
  if (lane < 18) x[lane] = lane == 17 ? 1.0 : 0.0;
  for (int k = kSample - 1; k >= 0; k--) {
    __syncwarp();
    const double* v = At + kLd * k;
    double dot = 0.0;
    for (int i = k; i < 18; i++) dot = i == k ? mul(v[i], x[i]) : add(dot, mul(v[i], x[i]));
    const double c = __ddiv_rn(mul(2.0, dot), vt[k]);
    __syncwarp();
    if (lane >= k && lane < 18) x[lane] = sub(x[lane], mul(c, v[lane]));
  }
  __syncwarp();
  if (lane == 0) {   // R' = x[9:18] with det > 0, its polar factor by Newton from |R'|_F = sqrt(3)
    double X[9], Xi[9];
    for (int i = 0; i < 9; i++) X[i] = x[9 + i];
    const double det = add(add(mul(X[0], sub(mul(X[4], X[8]), mul(X[5], X[7]))), mul(X[1], sub(mul(X[5], X[6]), mul(X[3], X[8])))),
                           mul(X[2], sub(mul(X[3], X[7]), mul(X[4], X[6]))));
    good = det > 0.0 || det < 0.0;
    if (good) {
      double fro = 0.0;
      for (int i = 0; i < 9; i++) fro = i == 0 ? mul(X[i], X[i]) : add(fro, mul(X[i], X[i]));
      const double scale = __dsqrt_rn(__ddiv_rn(3.0, fro));
      for (int i = 0; i < 9; i++) X[i] = det < 0.0 ? -mul(X[i], scale) : mul(X[i], scale);
      for (int it = 0; it < kPolarIters; it++) {
        inv3(X, Xi);
        for (int r = 0; r < 3; r++)
          for (int c = 0; c < 3; c++) X[3 * r + c] = mul(0.5, add(X[3 * r + c], Xi[3 * c + r]));
      }
      for (int i = 0; i < 9; i++) Rm[i] = X[i];
    }
  }
  if (!__shfl_sync(kFull, good, 0)) return false;
  __syncwarp();
  if (lane < kSample) {   // row `lane`: g = R d2 x d1, h = -(d1 . R m2 + m1 . R d2)
    const double *q = dm + 12 * lane, *d1 = q, *m1 = q + 3, *d2 = q + 6, *m2 = q + 9;
    double u[3], w[3];
    for (int r = 0; r < 3; r++) { u[r] = dot3(Rm[3 * r], Rm[3 * r + 1], Rm[3 * r + 2], d2); w[r] = dot3(Rm[3 * r], Rm[3 * r + 1], Rm[3 * r + 2], m2); }
    double* g = gh + 4 * lane;
    cross3(u, d1, g);
    g[3] = -add(dot3(d1[0], d1[1], d1[2], w), dot3(m1[0], m1[1], m1[2], u));
  }
  __syncwarp();
  if (lane == 0) {   // t from the normal equations, summed in sample order
    double N[9], b[3], Ni[9];
    for (int i = 0; i < kSample; i++) {
      const double* g = gh + 4 * i;
      for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) N[3 * r + c] = i == 0 ? mul(g[r], g[c]) : add(N[3 * r + c], mul(g[r], g[c]));
        b[r] = i == 0 ? mul(g[r], g[3]) : add(b[r], mul(g[r], g[3]));
      }
    }
    inv3(N, Ni);
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) model[4 * r + c] = Rm[3 * r + c];
      model[4 * r + 3] = dot3(Ni[3 * r], Ni[3 * r + 1], Ni[3 * r + 2], b);
    }
    for (int i = 0; i < 12; i++) good &= isfinite(model[i]);
  }
  return __shfl_sync(kFull, good, 0);
}

struct RelDev {
  const int* prob_ptr; const double* f1; const double* f2; const double* s1; const double* s2; const int* cam1; const int* cam2;
  const int* cam_ptr1; const int* cam_ptr2; const double* rig1; const double* rig2;   // rigs: [cam][12] offset then Rc
  const int* samples;
  int n_samples, max_iterations, area;   // area: doubles per warp in dynamic shared memory
  double threshold, log_p;
  int* best_sample; double* best_model; int* best_count; int* iterations; int* consumed;
  uint8_t* inlier_mask;                                    // nullable
  double* sample_model; uint8_t* sample_valid; int* sample_count;   // nullable together
};

// the camera-pair models of M for every pair (j1, j2) at P[12 (j1 nc2 + j2)], formed by the lanes of one warp
__device__ __forceinline__ void warp_pair_models(const double* M, const double* rig1, int nc1, const double* rig2, int nc2, double* P, int lane) {
  for (int p = lane; p < nc1 * nc2; p += 32) pair_model(M, rig1 + 12 * (p / nc2), rig2 + 12 * (p % nc2), P + kPairArea * p);
  __syncwarp();
}

__global__ void __launch_bounds__(kThreads) ransac_rel_kernel(RelDev D) {
  extern __shared__ double dyn[];
  const int pi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int off = D.prob_ptr[pi], n = D.prob_ptr[pi + 1] - off;
  const int nc1 = D.cam_ptr1[pi + 1] - D.cam_ptr1[pi], nc2 = D.cam_ptr2[pi + 1] - D.cam_ptr2[pi];
  const double* F1 = D.f1 + 3 * (size_t)off;
  const double* F2 = D.f2 + 3 * (size_t)off;
  const double* S1 = D.s1 + off;
  const double* S2 = D.s2 + off;
  const int* C1 = D.cam1 + off;
  const int* C2 = D.cam2 + off;
  double* W = dyn + (size_t)warp * D.area;
  const bool all = D.sample_model != nullptr;
  __shared__ double rig1[kMaxCams * 12], rig2[kMaxCams * 12];
  __shared__ double w_model[kWave][12];
  __shared__ int w_valid[kWave], w_count[kWave];
  __shared__ double best_model[12], k_bound;
  __shared__ int best, best_n, it, used, running, rigs_finite;
  __shared__ long long skipped;
  for (int i = tid; i < 12 * nc1; i += kThreads) rig1[i] = D.rig1[12 * (size_t)D.cam_ptr1[pi] + i];
  for (int i = tid; i < 12 * nc2; i += kThreads) rig2[i] = D.rig2[12 * (size_t)D.cam_ptr2[pi] + i];
  if (tid == 0) {
    best = -1; best_n = 0; it = 0; used = 0; skipped = 0; k_bound = (double)D.max_iterations;
    running = D.max_iterations > 0;
    for (int i = 0; i < 12; i++) best_model[i] = 0.0;
  }
  __syncthreads();
  if (tid == 0) {
    int fin = 1;
    for (int i = 0; i < 12 * nc1; i++) fin &= isfinite(rig1[i]);
    for (int i = 0; i < 12 * nc2; i++) fin &= isfinite(rig2[i]);
    rigs_finite = fin;
  }
  __syncthreads();
  const long long max_skip = 10LL * D.max_iterations;
  for (int base = 0; base < D.n_samples && (running || all); base += kWave) {
    for (int h = warp; h < kWave; h += kWarps) {
      const int s = base + h;
      bool v = false;
      if (s < D.n_samples)
        v = rel17(D.samples + kSample * ((size_t)pi * D.n_samples + s), n, F1, F2, C1, C2, rig1, rig2, rigs_finite, W, w_model[h], lane);
      __syncwarp();
      if (lane == 0) {
        if (!v)
          for (int i = 0; i < 12; i++) w_model[h][i] = 0.0;
        w_valid[h] = v;
      }
    }
    __syncthreads();
    for (int h = warp; h < kWave; h += kWarps) {
      int cnt = 0;
      if (w_valid[h]) {
        warp_pair_models(w_model[h], rig1, nc1, rig2, nc2, W, lane);
        for (int i = lane; i < n; i += 32) {
          const double* q = W + kPairArea * (C1[i] * nc2 + C2[i]);
          cnt += rel_score(q, F1, F2, S1, S2, i) < D.threshold;
        }
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
          double wp = w;
          for (int e = 1; e < kSample; e++) wp = mul(wp, w);
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
    if (best >= 0) warp_pair_models(best_model, rig1, nc1, rig2, nc2, W, lane);   // every warp its own copy
    for (int i = tid; i < n; i += kThreads) {
      const double* q = W + kPairArea * (C1[i] * nc2 + C2[i]);
      D.inlier_mask[off + i] = best >= 0 && rel_score(q, F1, F2, S1, S2, i) < D.threshold;
    }
  }
}

bool ptr_ok(const int32_t* p, int n) {
  if (p[0] != 0) return false;
  for (int i = 0; i < n; i++)
    if (p[i + 1] < p[i]) return false;
  return true;
}

}  // namespace

extern "C" int cvb_ransac_noncentral_relative_pose_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, double threshold, int max_iterations,
                                                         double probability, cvb_rel_ransac_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, p && r && p->n_prob >= 0 && p->n_samples >= 0 && max_iterations >= 0, "ransac_noncentral_relative_pose: bad arguments");
  CVB_REQUIRE(ctx, max_iterations <= INT32_MAX / 10, "ransac_noncentral_relative_pose: max_iterations too large");
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  CVB_REQUIRE(ctx, p->prob_ptr && p->cam_ptr1 && p->cam_ptr2 && r->best_sample && r->best_model && r->best_count && r->iterations && r->consumed,
              "ransac_noncentral_relative_pose: null required pointer");
  CVB_REQUIRE(ctx, (r->sample_model != nullptr) == (r->sample_valid != nullptr) && (r->sample_model != nullptr) == (r->sample_count != nullptr),
              "ransac_noncentral_relative_pose: sample_model / sample_valid / sample_count are requested together");
  CVB_REQUIRE(ctx, ptr_ok(p->prob_ptr, n_prob), "ransac_noncentral_relative_pose: prob_ptr does not start at 0 or decreases");
  CVB_REQUIRE(ctx, ptr_ok(p->cam_ptr1, n_prob) && ptr_ok(p->cam_ptr2, n_prob), "ransac_noncentral_relative_pose: cam_ptr1 / cam_ptr2 does not start at 0 or decreases");
  int max_pairs = 0;
  for (int i = 0; i < n_prob; i++) {
    const int nc1 = p->cam_ptr1[i + 1] - p->cam_ptr1[i], nc2 = p->cam_ptr2[i + 1] - p->cam_ptr2[i];
    CVB_REQUIRE(ctx, nc1 <= kMaxCams && nc2 <= kMaxCams, "ransac_noncentral_relative_pose: problem %d has a rig of more than %d cameras", i, kMaxCams);
    max_pairs = nc1 * nc2 > max_pairs ? nc1 * nc2 : max_pairs;
  }
  const size_t N = (size_t)p->prob_ptr[n_prob], NC1 = (size_t)p->cam_ptr1[n_prob], NC2 = (size_t)p->cam_ptr2[n_prob];
  CVB_REQUIRE(ctx, N == 0 || (p->f1 && p->f2 && p->sigma1 && p->sigma2 && p->cam1 && p->cam2), "ransac_noncentral_relative_pose: null correspondence arrays");
  CVB_REQUIRE(ctx, (NC1 == 0 || (p->cam_off1 && p->cam_rot1)) && (NC2 == 0 || (p->cam_off2 && p->cam_rot2)), "ransac_noncentral_relative_pose: null rig arrays");
  CVB_REQUIRE(ctx, ns == 0 || p->samples, "ransac_noncentral_relative_pose: null samples");
  for (int i = 0; i < n_prob; i++) {
    const int o = p->prob_ptr[i], n = p->prob_ptr[i + 1] - o;
    const int nc1 = p->cam_ptr1[i + 1] - p->cam_ptr1[i], nc2 = p->cam_ptr2[i + 1] - p->cam_ptr2[i];
    for (int j = o; j < o + n; j++)
      CVB_REQUIRE(ctx, p->cam1[j] >= 0 && p->cam1[j] < nc1 && p->cam2[j] >= 0 && p->cam2[j] < nc2,
                  "ransac_noncentral_relative_pose: correspondence %d of problem %d names camera (%d, %d) outside its rigs (%d, %d cameras)", j - o, i,
                  p->cam1[j], p->cam2[j], nc1, nc2);
    if (n < kSample) continue;   // every sample of such a problem is invalid; its indices are not read
    const int32_t* s = p->samples + kSample * (size_t)i * ns;
    for (size_t j = 0; j < kSample * (size_t)ns; j++)
      CVB_REQUIRE(ctx, s[j] >= 0 && s[j] < n, "ransac_noncentral_relative_pose: sample index %d out of range [0, %d) in problem %d", s[j], n, i);
  }
  const size_t S_all = (size_t)n_prob * ns;
  const bool all = r->sample_model != nullptr;
  Stager St;
  const size_t o_ptr = St.put(p->prob_ptr, ((size_t)n_prob + 1) * 4), o_f1 = St.put(p->f1, N * 24), o_f2 = St.put(p->f2, N * 24),
               o_s1 = St.put(p->sigma1, N * 8), o_s2 = St.put(p->sigma2, N * 8), o_c1 = St.put(p->cam1, N * 4), o_c2 = St.put(p->cam2, N * 4),
               o_cp1 = St.put(p->cam_ptr1, ((size_t)n_prob + 1) * 4), o_cp2 = St.put(p->cam_ptr2, ((size_t)n_prob + 1) * 4),
               o_smp = St.put(p->samples, S_all * kSample * 4);
  const size_t o_rig1 = St.reserve(NC1 * 96), o_rig2 = St.reserve(NC2 * 96);
  for (size_t j = 0; j < NC1; j++) {   // camera: offset (3) directly followed by the rotation (9, row-major)
    memcpy(St.h.data() + o_rig1 + 96 * j, p->cam_off1 + 3 * j, 24);
    memcpy(St.h.data() + o_rig1 + 96 * j + 24, p->cam_rot1 + 9 * j, 72);
  }
  for (size_t j = 0; j < NC2; j++) {
    memcpy(St.h.data() + o_rig2 + 96 * j, p->cam_off2 + 3 * j, 24);
    memcpy(St.h.data() + o_rig2 + 96 * j + 24, p->cam_rot2 + 9 * j, 72);
  }
  const size_t in_bytes = St.h.size();
  const size_t o_bm = St.reserve((size_t)n_prob * 96), o_bs = St.reserve((size_t)n_prob * 4), o_bc = St.reserve((size_t)n_prob * 4),
               o_it = St.reserve((size_t)n_prob * 4), o_us = St.reserve((size_t)n_prob * 4), o_mask = r->inlier_mask ? St.reserve(N) : 0,
               o_sm = all ? St.reserve(S_all * 96) : 0, o_sv = all ? St.reserve(S_all) : 0, o_sc = all ? St.reserve(S_all * 4) : 0;
  const size_t total = St.h.size();
  unsigned char* d = (unsigned char*)cvb_ws(ctx, WS_GS6, total);
  unsigned char* hpin = (unsigned char*)cvb_pinned(ctx, total);
  if (!d || !hpin) return CVB_ERR_CUDA;
  memcpy(hpin, St.h.data(), in_bytes);
  RelDev D{};
  D.prob_ptr = (const int*)(d + o_ptr); D.f1 = (const double*)(d + o_f1); D.f2 = (const double*)(d + o_f2);
  D.s1 = (const double*)(d + o_s1); D.s2 = (const double*)(d + o_s2); D.cam1 = (const int*)(d + o_c1); D.cam2 = (const int*)(d + o_c2);
  D.cam_ptr1 = (const int*)(d + o_cp1); D.cam_ptr2 = (const int*)(d + o_cp2);
  D.rig1 = (const double*)(d + o_rig1); D.rig2 = (const double*)(d + o_rig2); D.samples = (const int*)(d + o_smp);
  D.n_samples = ns; D.max_iterations = max_iterations; D.threshold = threshold; D.log_p = log(1.0 - probability);
  D.area = kSolveArea > kPairArea * max_pairs ? kSolveArea : kPairArea * max_pairs;
  D.best_sample = (int*)(d + o_bs); D.best_model = (double*)(d + o_bm); D.best_count = (int*)(d + o_bc); D.iterations = (int*)(d + o_it);
  D.consumed = (int*)(d + o_us); D.inlier_mask = r->inlier_mask ? d + o_mask : nullptr;
  if (all) { D.sample_model = (double*)(d + o_sm); D.sample_valid = d + o_sv; D.sample_count = (int*)(d + o_sc); }
  constexpr int kMaxArea = kSolveArea > kPairArea * kMaxCams * kMaxCams ? kSolveArea : kPairArea * kMaxCams * kMaxCams;
  static cvb_once_per_device once;
  if (once.first(ctx->device)) {
    CVB_CUDA(ctx, cudaFuncSetAttribute(ransac_rel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kWarps * kMaxArea * sizeof(double))));
  }
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemcpyAsync(d, hpin, in_bytes, cudaMemcpyHostToDevice, st));
  ransac_rel_kernel<<<n_prob, kThreads, (size_t)kWarps * D.area * sizeof(double), st>>>(D);
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
