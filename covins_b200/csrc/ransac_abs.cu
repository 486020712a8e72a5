// ransac_abs.cu — the absolute-pose RANSAC of Se3Solver::projectiveAlignment (GP3P, Se3Solver.cpp:59-110) on the GPU from
// caller-supplied samples: P3P per sample, the fourth-point choice, scoring and the sequential model selection of opengv's
// Ransac::computeModel, for a batch of problems (candidate keyframes) in one launch (SURVEY §8a V1).
//
// One CTA per problem.  Samples are taken in waves of kWave: the first kWave threads solve one sample each, every warp scores
// the wave's hypotheses against all correspondences (warp-shuffle integer counts), thread 0 replays the selection over the
// wave in sample order, and the CTA stops as soon as the adaptive bound ends the selection, so opengv's early stop saves the
// solver and scoring work of the samples it never reads.  The CTA then writes the best model's inlier mask.
//
// P3P is Lambda Twist (Persson & Nordberg, ECCV 2018): Newton iterations for one root of the cubic det(D1 + g D2) = 0, the
// eigen-decomposition of the degenerate conic D1 + g D2 with its known zero eigenvalue, two quadratics, Newton refinement of
// the depths, the pose from a 3x3 inverse.  Only + - * / and sqrt as explicit non-fused intrinsics, fixed iteration counts:
// the results are bit-identical to the plain IEEE restatement compiled with -ffp-contract=off (oracle/ransac_oracle.c).
#include <float.h>
#include <math.h>

#include "cvb_internal.cuh"
#include "geom_common.cuh"

namespace {

constexpr int kThreads = 256, kWave = 64;
constexpr int kCubicNewtonIters = 30, kDepthNewtonIters = 5;

__device__ __forceinline__ double dv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double sq(double a) { return __dsqrt_rn(a); }
__device__ __forceinline__ double dotv(const double* a, const double* b) { return dot3(a[0], a[1], a[2], b); }
__device__ __forceinline__ void cross3(const double* a, const double* b, double* o) {
  o[0] = sub(mul(a[1], b[2]), mul(a[2], b[1]));
  o[1] = sub(mul(a[2], b[0]), mul(a[0], b[2]));
  o[2] = sub(mul(a[0], b[1]), mul(a[1], b[0]));
}

// symmetric 3x3 as (s00, s01, s02, s11, s12, s22) → cofactors in the same layout
__device__ __forceinline__ void sym_cof(const double* s, double* c) {
  c[0] = sub(mul(s[3], s[5]), mul(s[4], s[4]));
  c[1] = sub(mul(s[2], s[4]), mul(s[1], s[5]));
  c[2] = sub(mul(s[1], s[4]), mul(s[2], s[3]));
  c[3] = sub(mul(s[0], s[5]), mul(s[2], s[2]));
  c[4] = sub(mul(s[1], s[2]), mul(s[0], s[4]));
  c[5] = sub(mul(s[0], s[3]), mul(s[1], s[1]));
}
// tr(adj(A) B), adj(A) given by its cofactors
__device__ __forceinline__ double sym_tr(const double* c, const double* b) {
  return add(add(add(mul(c[0], b[0]), mul(c[3], b[3])), mul(c[5], b[5])), mul(2.0, add(add(mul(c[1], b[1]), mul(c[2], b[2])), mul(c[4], b[4]))));
}

// one real root of g^3 + b g^2 + c g + d
__device__ double cubic_root(double b, double c, double d) {
  double r;
  if (mul(b, b) >= mul(3.0, c)) {
    const double v = sq(sub(mul(b, b), mul(3.0, c)));
    const double t1 = dv(sub(-b, v), 3.0);
    const double k1 = add(mul(add(mul(add(t1, b), t1), c), t1), d);
    if (k1 > 0.0) {
      r = sub(t1, sq(dv(-k1, add(mul(3.0, t1), b))));
    } else {
      const double t2 = dv(add(-b, v), 3.0);
      const double k2 = add(mul(add(mul(add(t2, b), t2), c), t2), d);
      r = add(t2, sq(dv(-k2, add(mul(3.0, t2), b))));
    }
  } else {
    r = dv(-b, 3.0);
    if (fabs(add(mul(add(mul(3.0, r), mul(2.0, b)), r), c)) < 1e-4) r = add(r, 1.0);
  }
  for (int it = 0; it < kCubicNewtonIters; it++) {
    const double fx = add(mul(add(mul(add(r, b), r), c), r), d);
    const double fpx = add(mul(add(mul(3.0, r), mul(2.0, b)), r), c);
    if (fpx != 0.0) r = sub(r, dv(fx, fpx));
  }
  return r;
}

// unit eigenvector of symmetric A for eigenvalue e: the largest cross product of two rows of A - eI
__device__ void eigvec(const double* A, double e, double* v) {
  const double r0[3] = {sub(A[0], e), A[1], A[2]}, r1[3] = {A[1], sub(A[3], e), A[4]}, r2[3] = {A[2], A[4], sub(A[5], e)};
  double c0[3], c1[3], c2[3];
  cross3(r0, r1, c0); cross3(r0, r2, c1); cross3(r1, r2, c2);
  const double n0 = dotv(c0, c0), n1 = dotv(c1, c1), n2 = dotv(c2, c2);
  const double* best = c0;
  double bn = n0;
  if (n1 > bn) { bn = n1; best = c1; }
  if (n2 > bn) { bn = n2; best = c2; }
  const double s = sq(bn);
  for (int i = 0; i < 3; i++) v[i] = dv(best[i], s);
}

__device__ __forceinline__ double depth_residual(const double* L, const double* a, const double* b) {
  const double r1 = sub(add(add(mul(L[0], L[0]), mul(L[1], L[1])), mul(mul(b[0], L[0]), L[1])), a[0]);
  const double r2 = sub(add(add(mul(L[0], L[0]), mul(L[2], L[2])), mul(mul(b[1], L[0]), L[2])), a[1]);
  const double r3 = sub(add(add(mul(L[1], L[1]), mul(L[2], L[2])), mul(mul(b[2], L[1]), L[2])), a[2]);
  return add(add(fabs(r1), fabs(r2)), fabs(r3));
}

// Newton on l_i^2 + l_j^2 + b_ij l_i l_j = a_ij; a step is kept only if it does not increase the residual
__device__ void refine_depths(double* L, const double* a, const double* b) {
  for (int it = 0; it < kDepthNewtonIters; it++) {
    const double l1 = L[0], l2 = L[1], l3 = L[2];
    const double r1 = sub(add(add(mul(l1, l1), mul(l2, l2)), mul(mul(b[0], l1), l2)), a[0]);
    const double r2 = sub(add(add(mul(l1, l1), mul(l3, l3)), mul(mul(b[1], l1), l3)), a[1]);
    const double r3 = sub(add(add(mul(l2, l2), mul(l3, l3)), mul(mul(b[2], l2), l3)), a[2]);
    const double v0 = add(mul(2.0, l1), mul(b[0], l2)), v1 = add(mul(2.0, l2), mul(b[0], l1));
    const double v3 = add(mul(2.0, l1), mul(b[1], l3)), v5 = add(mul(2.0, l3), mul(b[1], l1));
    const double v7 = add(mul(2.0, l2), mul(b[2], l3)), v8 = add(mul(2.0, l3), mul(b[2], l2));
    const double det = sub(-mul(mul(v0, v5), v7), mul(mul(v1, v3), v8));
    const double s0 = add(sub(mul(-mul(v5, v7), r1), mul(mul(v1, v8), r2)), mul(mul(v1, v5), r3));
    const double s1 = sub(add(mul(-mul(v3, v8), r1), mul(mul(v0, v8), r2)), mul(mul(v0, v5), r3));
    const double s2 = sub(sub(mul(mul(v3, v7), r1), mul(mul(v0, v7), r2)), mul(mul(v1, v3), r3));
    const double N[3] = {sub(l1, dv(s0, det)), sub(l2, dv(s1, det)), sub(l3, dv(s2, det))};
    const double old_r = add(add(fabs(r1), fabs(r2)), fabs(r3));
    if (depth_residual(N, a, b) <= old_r) { L[0] = N[0]; L[1] = N[1]; L[2] = N[2]; }
  }
}

// P3P: bearings f[3][3] (camera frame), world points x[3][3] → up to 4 poses Rt[k][12], lambda_i f_i = R x_i + t, lambda_i > 0
__device__ int p3p(const double* f, const double* x, double* Rt) {
  double y[3][3];
  for (int i = 0; i < 3; i++) {
    const double n = sq(dotv(f + 3 * i, f + 3 * i));
    for (int r = 0; r < 3; r++) y[i][r] = dv(f[3 * i + r], n);
  }
  const double h12 = -dotv(y[0], y[1]), h13 = -dotv(y[0], y[2]), h23 = -dotv(y[1], y[2]);
  const double b[3] = {mul(2.0, h12), mul(2.0, h13), mul(2.0, h23)};
  double d12[3], d13[3], d23[3];
  for (int r = 0; r < 3; r++) { d12[r] = sub(x[r], x[3 + r]); d13[r] = sub(x[r], x[6 + r]); d23[r] = sub(x[3 + r], x[6 + r]); }
  const double a[3] = {dotv(d12, d12), dotv(d13, d13), dotv(d23, d23)};
  const double a12 = a[0], a13 = a[1], a23 = a[2];
  const double D1[6] = {a23, mul(a23, h12), 0.0, sub(a23, a12), -mul(a12, h23), -a12};
  const double D2[6] = {a23, 0.0, mul(a23, h13), -a13, -mul(a13, h23), sub(a23, a13)};
  double C1[6], C2[6];
  sym_cof(D1, C1); sym_cof(D2, C2);
  const double c3 = add(add(mul(D2[0], C2[0]), mul(D2[1], C2[1])), mul(D2[2], C2[2]));
  const double c0 = add(add(mul(D1[0], C1[0]), mul(D1[1], C1[1])), mul(D1[2], C1[2]));
  const double c1 = sym_tr(C1, D2), c2 = sym_tr(C2, D1);
  const double g = cubic_root(dv(c2, c3), dv(c1, c3), dv(c0, c3));
  double A[6], Ac[6];
  for (int i = 0; i < 6; i++) A[i] = add(D1[i], mul(g, D2[i]));
  sym_cof(A, Ac);
  const double p = -add(add(A[0], A[3]), A[5]), q = add(add(Ac[0], Ac[3]), Ac[5]);
  const double disc = sub(mul(p, p), mul(4.0, q)), sd = disc > 0.0 ? sq(disc) : 0.0;
  double e1, e2;
  if (p < 0.0) { e1 = mul(0.5, add(-p, sd)); e2 = dv(mul(2.0, q), add(-p, sd)); }
  else { e1 = dv(mul(2.0, q), sub(-p, sd)); e2 = mul(0.5, sub(-p, sd)); }
  if (fabs(e1) < fabs(e2)) { const double t = e1; e1 = e2; e2 = t; }
  double v1[3], v2[3];
  eigvec(A, e1, v1); eigvec(A, e2, v2);
  const double ratio = dv(-e2, e1), s = ratio > 0.0 ? sq(ratio) : 0.0;
  double Ls[4][3];
  int ns = 0;
  for (int side = 0; side < 2; side++) {
    const double sg = side == 0 ? s : -s;
    const double den = sub(mul(sg, v2[0]), v1[0]);
    const double w0 = dv(sub(v1[1], mul(sg, v2[1])), den), w1 = dv(sub(v1[2], mul(sg, v2[2])), den);
    const double qa = sub(sub(mul(mul(sub(a13, a12), w1), w1), mul(mul(a12, b[1]), w1)), a12);
    const double qb = sub(sub(mul(mul(a13, b[0]), w1), mul(mul(a12, b[1]), w0)), mul(mul(mul(2.0, w0), w1), sub(a12, a13)));
    const double qc = add(add(mul(mul(sub(a13, a12), w0), w0), mul(mul(a13, b[0]), w0)), a13);
    const double B = dv(qb, qa), C = dv(qc, qa);
    const double dq = sub(mul(B, B), mul(4.0, C));
    if (!(dq >= 0.0)) continue;
    const double yq = sq(dq);
    double tau[2];
    if (B < 0.0) { tau[0] = mul(0.5, add(-B, yq)); tau[1] = dv(mul(2.0, C), add(-B, yq)); }
    else { tau[0] = dv(mul(2.0, C), sub(-B, yq)); tau[1] = mul(0.5, sub(-B, yq)); }
    for (int k = 0; k < 2; k++) {
      if (!(tau[k] > 0.0)) continue;
      const double l2 = sq(dv(a23, add(mul(tau[k], add(b[2], tau[k])), 1.0)));
      const double l3 = mul(tau[k], l2), l1 = add(mul(w0, l2), mul(w1, l3));
      if (!(l1 > 0.0)) continue;
      Ls[ns][0] = l1; Ls[ns][1] = l2; Ls[ns][2] = l3; ns++;
    }
  }
  double X[9], Xi[9], n13[3];
  cross3(d12, d13, n13);
  for (int r = 0; r < 3; r++) { X[3 * r] = d12[r]; X[3 * r + 1] = d13[r]; X[3 * r + 2] = n13[r]; }
  inv3(X, Xi);
  int out = 0;
  for (int k = 0; k < ns; k++) {
    double* L = Ls[k];
    refine_depths(L, a, b);
    if (!(L[0] > 0.0 && L[1] > 0.0 && L[2] > 0.0)) continue;
    double p1[3], yd1[3], yd2[3], yc[3], Y[9];
    for (int r = 0; r < 3; r++) { p1[r] = mul(L[0], y[0][r]); yd1[r] = sub(p1[r], mul(L[1], y[1][r])); yd2[r] = sub(p1[r], mul(L[2], y[2][r])); }
    cross3(yd1, yd2, yc);
    for (int r = 0; r < 3; r++) { Y[3 * r] = yd1[r]; Y[3 * r + 1] = yd2[r]; Y[3 * r + 2] = yc[r]; }
    double* M = Rt + 12 * out;
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) M[4 * r + c] = add(add(mul(Y[3 * r], Xi[c]), mul(Y[3 * r + 1], Xi[3 + c])), mul(Y[3 * r + 2], Xi[6 + c]));
    for (int r = 0; r < 3; r++) M[4 * r + 3] = sub(p1[r], add(add(mul(M[4 * r], x[0]), mul(M[4 * r + 1], x[1])), mul(M[4 * r + 2], x[2])));
    out++;
  }
  return out;
}

// the hypothesis of sample s (problem-local indices) → body-in-world model [R|t]; false = invalid sample
__device__ bool hypothesis(const int* s, int n, const double* pts, const double* f, const double* cam, double* model) {
  if (n < 4) return false;
  for (int i = 0; i < 4; i++)
    for (int j = i + 1; j < 4; j++)
      if (s[i] == s[j]) return false;
  double fb[9], xw[9];
  for (int i = 0; i < 4; i++)
    for (int r = 0; r < 3; r++)
      if (!isfinite(pts[3 * (size_t)s[i] + r]) || !isfinite(f[3 * (size_t)s[i] + r])) return false;
  for (int i = 0; i < 3; i++)
    for (int r = 0; r < 3; r++) { fb[3 * i + r] = f[3 * (size_t)s[i] + r]; xw[3 * i + r] = pts[3 * (size_t)s[i] + r]; }
  double Rt[48];
  const int ns = p3p(fb, xw, Rt);
  const double* co = cam;
  const double* cr = cam + 3;
  const double* p4 = pts + 3 * (size_t)s[3];
  const double* f4 = f + 3 * (size_t)s[3];
  bool found = false;
  double best_score = INFINITY;
  for (int k = 0; k < ns; k++) {
    const double* P = Rt + 12 * k;   // camera from world → body from world: Rbw = Rc Rcw, tbw = Rc tcw + c
    double Rbw[9], tbw[3], M[12];
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) Rbw[3 * r + c] = add(add(mul(cr[3 * r], P[c]), mul(cr[3 * r + 1], P[4 + c])), mul(cr[3 * r + 2], P[8 + c]));
      tbw[r] = add(add(add(mul(cr[3 * r], P[3]), mul(cr[3 * r + 1], P[7])), mul(cr[3 * r + 2], P[11])), co[r]);
    }
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) M[4 * r + c] = Rbw[3 * c + r];
      M[4 * r + 3] = -add(add(mul(Rbw[r], tbw[0]), mul(Rbw[3 + r], tbw[1])), mul(Rbw[6 + r], tbw[2]));
    }
    double Ri[9], ti[3], q[3];
    abs_inverse(M, Ri, ti);
    const double nrm = abs_ray(Ri, ti, p4, cam, q);
    const double score = sub(1.0, add(add(mul(dv(q[0], nrm), f4[0]), mul(dv(q[1], nrm), f4[1])), mul(dv(q[2], nrm), f4[2])));
    if (score < best_score) {
      best_score = score; found = true;
      for (int i = 0; i < 12; i++) model[i] = M[i];
    }
  }
  if (!found) return false;
  for (int i = 0; i < 12; i++)
    if (!isfinite(model[i])) return false;
  return true;
}

struct RansacDev {
  const int* prob_ptr; const double* pts; const double* f; const double* sigma; const double* cam;   // cam: [n_prob][12] offset, Rc
  const int* samples;
  int n_samples, max_iterations;
  double threshold, log_p;
  int* best_sample; double* best_model; int* best_count; int* iterations; int* consumed;
  uint8_t* inlier_mask;                                    // nullable
  double* sample_model; uint8_t* sample_valid; int* sample_count;   // nullable together
};

__global__ void __launch_bounds__(kThreads) ransac_abs_kernel(RansacDev D) {
  const int pi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int off = D.prob_ptr[pi], n = D.prob_ptr[pi + 1] - off;
  const double* P = D.pts + 3 * (size_t)off;
  const double* F = D.f + 3 * (size_t)off;
  const double* S = D.sigma + off;
  const double* cam = D.cam + 12 * (size_t)pi;
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
    if (tid < kWave) {
      const int s = base + tid;
      double M[12];
      for (int i = 0; i < 12; i++) M[i] = 0.0;
      bool v = false;
      if (s < D.n_samples) v = hypothesis(D.samples + 4 * ((size_t)pi * D.n_samples + s), n, P, F, cam, M);
      if (!v)
        for (int i = 0; i < 12; i++) M[i] = 0.0;
      for (int i = 0; i < 12; i++) w_model[tid][i] = M[i];
      w_valid[tid] = v;
    }
    __syncthreads();
    for (int h = warp; h < kWave; h += kThreads / 32) {
      int cnt = 0;
      if (w_valid[h]) {
        double Ri[9], ti[3];
        abs_inverse(w_model[h], Ri, ti);
        for (int i = lane; i < n; i += 32) cnt += abs_score(Ri, ti, P + 3 * (size_t)i, F + 3 * (size_t)i, S[i], cam) < D.threshold;
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);   // integer: order-independent
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
          const double w = dv((double)c, (double)n);
          double pno = sub(1.0, mul(mul(mul(w, w), w), w));
          pno = pno > DBL_EPSILON ? pno : DBL_EPSILON;
          pno = pno < 1.0 - DBL_EPSILON ? pno : 1.0 - DBL_EPSILON;
          k_bound = dv(D.log_p, log(pno));
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
    double Ri[9], ti[3];
    abs_inverse(best_model, Ri, ti);
    for (int i = tid; i < n; i += kThreads)
      D.inlier_mask[off + i] = best >= 0 && abs_score(Ri, ti, P + 3 * (size_t)i, F + 3 * (size_t)i, S[i], cam) < D.threshold;
  }
}

}  // namespace

extern "C" int cvb_ransac_absolute_pose_batch(cvb_ctx* ctx, const cvb_abs_ransac_problems* p, double threshold, int max_iterations,
                                              double probability, cvb_abs_ransac_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, p && r && p->n_prob >= 0 && p->n_samples >= 0 && max_iterations >= 0, "ransac_absolute_pose: bad arguments");
  CVB_REQUIRE(ctx, max_iterations <= INT32_MAX / 10, "ransac_absolute_pose: max_iterations too large");
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  CVB_REQUIRE(ctx, p->prob_ptr && p->cam_off && p->cam_rot && r->best_sample && r->best_model && r->best_count && r->iterations && r->consumed,
              "ransac_absolute_pose: null required pointer");
  CVB_REQUIRE(ctx, (r->sample_model != nullptr) == (r->sample_valid != nullptr) && (r->sample_model != nullptr) == (r->sample_count != nullptr),
              "ransac_absolute_pose: sample_model / sample_valid / sample_count are requested together");
  CVB_REQUIRE(ctx, p->prob_ptr[0] == 0, "ransac_absolute_pose: prob_ptr[0] != 0");
  for (int i = 0; i < n_prob; i++) CVB_REQUIRE(ctx, p->prob_ptr[i + 1] >= p->prob_ptr[i], "ransac_absolute_pose: prob_ptr decreases at %d", i);
  const size_t N = (size_t)p->prob_ptr[n_prob];
  CVB_REQUIRE(ctx, N == 0 || (p->pts && p->f && p->sigma), "ransac_absolute_pose: null correspondence arrays");
  CVB_REQUIRE(ctx, ns == 0 || p->samples, "ransac_absolute_pose: null samples");
  for (int i = 0; i < n_prob; i++) {
    const int n = p->prob_ptr[i + 1] - p->prob_ptr[i];
    if (n < 4) continue;   // every sample of such a problem is invalid; its indices are not read
    const int32_t* s = p->samples + 4 * (size_t)i * ns;
    for (size_t j = 0; j < 4 * (size_t)ns; j++)
      CVB_REQUIRE(ctx, s[j] >= 0 && s[j] < n, "ransac_absolute_pose: sample index %d out of range [0, %d) in problem %d", s[j], n, i);
  }
  const size_t S_all = (size_t)n_prob * ns;
  const bool all = r->sample_model != nullptr;
  Stager St;
  const size_t o_ptr = St.put(p->prob_ptr, ((size_t)n_prob + 1) * 4), o_pts = St.put(p->pts, N * 24), o_f = St.put(p->f, N * 24),
               o_sg = St.put(p->sigma, N * 8), o_smp = St.put(p->samples, S_all * 16);
  const size_t o_cam = St.reserve((size_t)n_prob * 96);
  for (int i = 0; i < n_prob; i++) {   // one camera per problem: offset (3) directly followed by the rotation (9, row-major)
    memcpy(St.h.data() + o_cam + 96 * (size_t)i, p->cam_off + 3 * (size_t)i, 24);
    memcpy(St.h.data() + o_cam + 96 * (size_t)i + 24, p->cam_rot + 9 * (size_t)i, 72);
  }
  const size_t in_bytes = St.h.size();
  const size_t o_bm = St.reserve((size_t)n_prob * 96), o_bs = St.reserve((size_t)n_prob * 4), o_bc = St.reserve((size_t)n_prob * 4),
               o_it = St.reserve((size_t)n_prob * 4), o_us = St.reserve((size_t)n_prob * 4), o_mask = r->inlier_mask ? St.reserve(N) : 0,
               o_sm = all ? St.reserve(S_all * 96) : 0, o_sv = all ? St.reserve(S_all) : 0, o_sc = all ? St.reserve(S_all * 4) : 0;
  const size_t total = St.h.size();
  unsigned char* d = (unsigned char*)cvb_ws(ctx, WS_GS5, total);
  unsigned char* hpin = (unsigned char*)cvb_pinned(ctx, total);
  if (!d || !hpin) return CVB_ERR_CUDA;
  memcpy(hpin, St.h.data(), in_bytes);
  RansacDev D{};
  D.prob_ptr = (const int*)(d + o_ptr); D.pts = (const double*)(d + o_pts); D.f = (const double*)(d + o_f); D.sigma = (const double*)(d + o_sg);
  D.cam = (const double*)(d + o_cam); D.samples = (const int*)(d + o_smp);
  D.n_samples = ns; D.max_iterations = max_iterations; D.threshold = threshold; D.log_p = log(1.0 - probability);
  D.best_sample = (int*)(d + o_bs); D.best_model = (double*)(d + o_bm); D.best_count = (int*)(d + o_bc); D.iterations = (int*)(d + o_it);
  D.consumed = (int*)(d + o_us); D.inlier_mask = r->inlier_mask ? d + o_mask : nullptr;
  if (all) { D.sample_model = (double*)(d + o_sm); D.sample_valid = d + o_sv; D.sample_count = (int*)(d + o_sc); }
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemcpyAsync(d, hpin, in_bytes, cudaMemcpyHostToDevice, st));
  ransac_abs_kernel<<<n_prob, kThreads, 0, st>>>(D);
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
