// ransac_abs.cu — the absolute-pose RANSAC of Se3Solver::projectiveAlignment (GP3P, Se3Solver.cpp:59-110) on the GPU from
// caller-supplied samples: P3P per sample, the fourth-point choice, scoring and the sequential model selection of opengv's
// Ransac::computeModel, for a batch of problems (candidate keyframes) in one launch (SURVEY §8a V1).
//
// One CTA per problem, driven by ransac_cta (ransac_common.cuh, shared with ransac_rel.cu): the waves of kWave samples, the
// scoring, the selection with its early stop and the inlier mask.  This file supplies the solver: in each wave the first kWave
// threads solve one sample each; a hypothesis is scored by its inverse (abs_inverse, abs_score in geom_common.cuh).
//
// P3P is Lambda Twist (Persson & Nordberg, ECCV 2018): Newton iterations for one root of the cubic det(D1 + g D2) = 0, the
// eigen-decomposition of the degenerate conic D1 + g D2 with its known zero eigenvalue, two quadratics, Newton refinement of
// the depths, the pose from a 3x3 inverse.  Only + - * / and sqrt as explicit non-fused intrinsics, fixed iteration counts:
// the results are bit-identical to the plain IEEE restatement compiled with -ffp-contract=off (oracle/ransac_oracle.c).
#include "ransac_common.cuh"

namespace {

constexpr int kCubicNewtonIters = 30, kDepthNewtonIters = 5;

__device__ __forceinline__ double dv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double sq(double a) { return __dsqrt_rn(a); }
__device__ __forceinline__ double dotv(const double* a, const double* b) { return dot3(a[0], a[1], a[2], b); }

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
  const double s = sq(cross_max(r0, r1, r2, v));
  for (int i = 0; i < 3; i++) v[i] = dv(v[i], s);
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
  RansacOut o;
};

// problem blockIdx.x for ransac_cta
struct AbsProblem {
  const double *P, *F, *S, *cam;
  int n;
  __device__ AbsProblem(const RansacDev& D, int pi, int off)
      : P(D.pts + 3 * (size_t)off), F(D.f + 3 * (size_t)off), S(D.sigma + off), cam(D.cam + 12 * (size_t)pi), n(D.prob_ptr[pi + 1] - off) {}
  // the first kWave threads solve one sample each
  template <class Src>
  __device__ void solve_wave(const Src& src, int base, double (*w_model)[12], int* w_valid) const {
    const int tid = threadIdx.x;
    if (tid >= kWave) return;
    const int s = base + tid;
    double M[12];
    for (int i = 0; i < 12; i++) M[i] = 0.0;
    bool v = false;
    if (src.has(s)) v = hypothesis(src.sample(s), n, P, F, cam, M);
    if (!v)
      for (int i = 0; i < 12; i++) M[i] = 0.0;
    for (int i = 0; i < 12; i++) w_model[tid][i] = M[i];
    w_valid[tid] = v;
  }
  // the score of correspondence i under M
  __device__ auto scorer(const double* M) const {
    double Ri[9], ti[3];
    abs_inverse(M, Ri, ti);
    return [=](int i) { return abs_score(Ri, ti, P + 3 * (size_t)i, F + 3 * (size_t)i, S[i], cam); };
  }
};

// Src: SuppliedSamples<4> (cvb_ransac_absolute_pose_batch) or SeededSamples<4> (cvb_ransac_absolute_pose_seeded_batch)
template <class Src>
__global__ void __launch_bounds__(kThreads) ransac_abs_kernel(RansacDev D) {
  const int pi = blockIdx.x, off = D.prob_ptr[pi];
  const int* samples = D.samples + 4 * (size_t)pi * D.o.n_samples;   // supplied: this problem's
  AbsProblem Pb(D, pi, off);
  ransac_cta<4>(D.o, Pb, sample_source<Src>(D.o, samples, pi, Pb.n), off, Pb.n);
}

// cvb_ransac_absolute_pose_batch (seeded = false) and cvb_ransac_absolute_pose_seeded_batch
int abs_ransac(cvb_ctx* ctx, const char* name, const cvb_abs_ransac_problems* p, bool seeded, const uint64_t* seed, double threshold, int max_iterations,
               double probability, cvb_abs_ransac_result* r, int32_t* drawn) {
  if (const int rc = check_ransac(ctx, name, p, max_iterations, r, 4, seeded, seed)) return rc;
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  CVB_REQUIRE(ctx, p->cam_off && p->cam_rot, "%s: null camera arrays", name);
  const size_t N = (size_t)p->prob_ptr[n_prob];
  CVB_REQUIRE(ctx, N == 0 || (p->pts && p->f && p->sigma), "%s: null correspondence arrays", name);
  const std::vector<double> cam = pack_cams(p->cam_off, p->cam_rot, n_prob);   // one camera per problem
  cvb_block B(ctx, ctx->stream);
  RansacDev D{};
  B.in(D.prob_ptr, p->prob_ptr, (size_t)n_prob + 1); B.in(D.pts, p->pts, N * 3); B.in(D.f, p->f, N * 3); B.in(D.sigma, p->sigma, N);
  if (seeded) B.in(D.o.seed, seed, n_prob);
  else B.in(D.samples, p->samples, (size_t)n_prob * ns * 4);
  B.in(D.cam, cam.data(), (size_t)n_prob * 12);
  if (seeded)
    return run_ransac(ctx, B, ransac_abs_kernel<SeededSamples<4>>, 0, D, n_prob, ns, N, threshold, max_iterations, probability, r, drawn, 4);
  return run_ransac(ctx, B, ransac_abs_kernel<SuppliedSamples<4>>, 0, D, n_prob, ns, N, threshold, max_iterations, probability, r);
}

}  // namespace

int cvb_abs_ransac_seeded_dev(cvb_ctx* ctx, int n_prob, const int32_t* d_prob_ptr, const double* d_pts, const double* d_f, const double* d_sigma,
                              const double* d_cam, const uint64_t* d_seed, double threshold, int max_iterations, double probability,
                              int32_t* d_best_sample, double* d_best_model, int32_t* d_best_count, int32_t* d_iterations, int32_t* d_consumed,
                              uint8_t* d_inlier_mask) {
  if (n_prob == 0) return CVB_OK;
  RansacDev D{};
  D.prob_ptr = d_prob_ptr; D.pts = d_pts; D.f = d_f; D.sigma = d_sigma; D.cam = d_cam;
  set_outputs(D.o, 0, max_iterations, threshold, probability, d_best_sample, d_best_model, d_best_count, d_iterations, d_consumed, d_inlier_mask);
  D.o.seed = (const unsigned long long*)d_seed;
  return launch_ransac(ctx, ransac_abs_kernel<SeededSamples<4>>, 0, D, n_prob);
}

extern "C" int cvb_ransac_absolute_pose_batch(cvb_ctx* ctx, const cvb_abs_ransac_problems* p, double threshold, int max_iterations,
                                              double probability, cvb_abs_ransac_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return abs_ransac(ctx, "ransac_absolute_pose", p, false, nullptr, threshold, max_iterations, probability, r, nullptr);
}

extern "C" int cvb_ransac_absolute_pose_seeded_batch(cvb_ctx* ctx, const cvb_abs_ransac_problems* p, const uint64_t* seed, double threshold,
                                                     int max_iterations, double probability, cvb_abs_ransac_result* r, int32_t* drawn) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return abs_ransac(ctx, "ransac_absolute_pose_seeded", p, true, seed, threshold, max_iterations, probability, r, drawn);
}
