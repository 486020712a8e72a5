/* oracle/ransac_oracle.c — CPU restatement of the absolute-pose RANSAC of Se3Solver::projectiveAlignment (GP3P, Se3Solver.cpp:59-110)
 * from caller-supplied samples: P3P per sample, the fourth-point choice, the per-correspondence score and the sequential model
 * selection.  TEST INFRASTRUCTURE ONLY (tests/, tools/); never linked into covins_b200/.  It is the bit-for-bit reference of
 * cvb_ransac_absolute_pose_batch (covins_b200/csrc/ransac_abs.cu); the existing scoring oracle (geom_oracle.c) is left alone.
 *
 * ASSUMPTIONS (opengv is not in the tree, dependencies.rosinstall:43-45):
 *   [S] sample size 4 and the choice among the minimal solutions follow opengv's AbsolutePoseSacProblem (GP3P branch): the
 *       first three correspondences are solved, the solution whose predicted direction of the fourth point has the smallest
 *       1 - cos angle to its bearing is kept (strict <, the first of equal values wins).
 *   [K] a sample without a hypothesis does not consume an iteration (Ransac::computeModel's skipped_count), and at most
 *       10 * max_iterations samples are skipped.
 *   Selection = covins_b200.placerec.ransac_select over the valid samples in order (sample_size 4), w^4 as plain products.
 * P3P: Lambda Twist (Persson & Nordberg, ECCV 2018), restated from the paper: one real root of the cubic det(D1 + g D2) = 0 by
 * Newton iterations, the eigen-decomposition of the degenerate conic D1 + g D2 (known zero eigenvalue), two quadratics, Newton
 * refinement of the three depths, pose from a 3x3 inverse.  A camera with offset c and rotation Rc in the body frame sees the
 * three rays from one centre, so GP3P (one camera per problem) has the solution set of central P3P.
 * Only + - * / and sqrt, fixed iteration counts; plain IEEE double without contraction (compile with -ffp-contract=off): the
 * CUDA path uses explicit non-fused operations in the same order, so results are compared bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define API __attribute__((visibility("default")))

enum { CUBIC_NEWTON_ITERS = 30, DEPTH_NEWTON_ITERS = 5 };

static double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}

/* symmetric 3x3 as (s00, s01, s02, s11, s12, s22): cofactors (c00, c01, c02, c11, c12, c22) */
static void sym_cof(const double* s, double* c) {
  c[0] = s[3] * s[5] - s[4] * s[4];
  c[1] = s[2] * s[4] - s[1] * s[5];
  c[2] = s[1] * s[4] - s[2] * s[3];
  c[3] = s[0] * s[5] - s[2] * s[2];
  c[4] = s[1] * s[2] - s[0] * s[4];
  c[5] = s[0] * s[3] - s[1] * s[1];
}
/* tr(adj(A) B) for symmetric A (given by its cofactors) and B */
static double sym_tr(const double* c, const double* b) {
  return ((c[0] * b[0] + c[3] * b[3]) + c[5] * b[5]) + 2.0 * ((c[1] * b[1] + c[2] * b[2]) + c[4] * b[4]);
}

/* one real root of g^3 + b g^2 + c g + d (Lambda Twist's starting point, then Newton) */
static double cubic_root(double b, double c, double d) {
  double r;
  if (b * b >= 3.0 * c) {
    const double v = sqrt(b * b - 3.0 * c);
    const double t1 = (-b - v) / 3.0;
    const double k1 = ((t1 + b) * t1 + c) * t1 + d;
    if (k1 > 0.0) {
      r = t1 - sqrt(-k1 / (3.0 * t1 + b));
    } else {
      const double t2 = (-b + v) / 3.0;
      const double k2 = ((t2 + b) * t2 + c) * t2 + d;
      r = t2 + sqrt(-k2 / (3.0 * t2 + b));
    }
  } else {
    r = -b / 3.0;
    if (fabs((3.0 * r + 2.0 * b) * r + c) < 1e-4) r = r + 1.0;
  }
  for (int it = 0; it < CUBIC_NEWTON_ITERS; it++) {
    const double fx = ((r + b) * r + c) * r + d;
    const double fpx = (3.0 * r + 2.0 * b) * r + c;
    if (fpx != 0.0) r = r - fx / fpx;
  }
  return r;
}

/* unit eigenvector of symmetric A (6 entries) for eigenvalue e: the largest cross product of two rows of A - eI */
static void eigvec(const double* A, double e, double* v) {
  const double r0[3] = {A[0] - e, A[1], A[2]}, r1[3] = {A[1], A[3] - e, A[4]}, r2[3] = {A[2], A[4], A[5] - e};
  double c[3][3];
  cross3(r0, r1, c[0]); cross3(r0, r2, c[1]); cross3(r1, r2, c[2]);
  int best = 0;
  double bn = dot3(c[0], c[0]);
  for (int i = 1; i < 3; i++) {
    const double n = dot3(c[i], c[i]);
    if (n > bn) { bn = n; best = i; }
  }
  const double s = sqrt(bn);
  for (int i = 0; i < 3; i++) v[i] = c[best][i] / s;
}

static double depth_residual(const double* L, const double* a, const double* b) {
  const double r1 = ((L[0] * L[0] + L[1] * L[1]) + (b[0] * L[0]) * L[1]) - a[0];
  const double r2 = ((L[0] * L[0] + L[2] * L[2]) + (b[1] * L[0]) * L[2]) - a[1];
  const double r3 = ((L[1] * L[1] + L[2] * L[2]) + (b[2] * L[1]) * L[2]) - a[2];
  return (fabs(r1) + fabs(r2)) + fabs(r3);
}

/* Newton on l_i^2 + l_j^2 + b_ij l_i l_j = a_ij (a = a12, a13, a23; b = b12, b13, b23); a step is kept only if it does not
 * increase the residual */
static void refine_depths(double* L, const double* a, const double* b) {
  for (int it = 0; it < DEPTH_NEWTON_ITERS; it++) {
    const double l1 = L[0], l2 = L[1], l3 = L[2];
    const double r1 = ((l1 * l1 + l2 * l2) + (b[0] * l1) * l2) - a[0];
    const double r2 = ((l1 * l1 + l3 * l3) + (b[1] * l1) * l3) - a[1];
    const double r3 = ((l2 * l2 + l3 * l3) + (b[2] * l2) * l3) - a[2];
    const double v0 = 2.0 * l1 + b[0] * l2, v1 = 2.0 * l2 + b[0] * l1;     /* dr1/dl1, dr1/dl2 */
    const double v3 = 2.0 * l1 + b[1] * l3, v5 = 2.0 * l3 + b[1] * l1;     /* dr2/dl1, dr2/dl3 */
    const double v7 = 2.0 * l2 + b[2] * l3, v8 = 2.0 * l3 + b[2] * l2;     /* dr3/dl2, dr3/dl3 */
    const double det = -((v0 * v5) * v7) - (v1 * v3) * v8;
    const double s0 = ((-(v5 * v7)) * r1 - (v1 * v8) * r2) + (v1 * v5) * r3;
    const double s1 = ((-(v3 * v8)) * r1 + (v0 * v8) * r2) - (v0 * v5) * r3;
    const double s2 = ((v3 * v7) * r1 - (v0 * v7) * r2) - (v1 * v3) * r3;
    const double N[3] = {l1 - s0 / det, l2 - s1 / det, l3 - s2 / det};
    const double old_r = (fabs(r1) + fabs(r2)) + fabs(r3);
    if (depth_residual(N, a, b) <= old_r) { L[0] = N[0]; L[1] = N[1]; L[2] = N[2]; }
  }
}

static void inv3(const double* m, double* o) {
  const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
  const double det = (m[0] * c00 + m[1] * c01) + m[2] * c02;
  o[0] = c00 / det; o[1] = (m[2] * m[7] - m[1] * m[8]) / det; o[2] = (m[1] * m[5] - m[2] * m[4]) / det;
  o[3] = c01 / det; o[4] = (m[0] * m[8] - m[2] * m[6]) / det; o[5] = (m[2] * m[3] - m[0] * m[5]) / det;
  o[6] = c02 / det; o[7] = (m[1] * m[6] - m[0] * m[7]) / det; o[8] = (m[0] * m[4] - m[1] * m[3]) / det;
}

/* P3P: bearings f[3][3] (camera frame), world points x[3][3] → up to 4 poses Rt[k][12] = [R|t] row-major with
 * lambda_i f_i = R x_i + t, every lambda_i > 0.  Returns the number of solutions. */
API int ora_p3p(const double* f, const double* x, double* Rt) {
  double y[3][3];
  for (int i = 0; i < 3; i++) {
    const double n = sqrt(dot3(f + 3 * i, f + 3 * i));
    for (int r = 0; r < 3; r++) y[i][r] = f[3 * i + r] / n;
  }
  const double h12 = -dot3(y[0], y[1]), h13 = -dot3(y[0], y[2]), h23 = -dot3(y[1], y[2]);   /* b_ij / 2 */
  const double b[3] = {2.0 * h12, 2.0 * h13, 2.0 * h23};
  double d12[3], d13[3], d23[3];
  for (int r = 0; r < 3; r++) { d12[r] = x[r] - x[3 + r]; d13[r] = x[r] - x[6 + r]; d23[r] = x[3 + r] - x[6 + r]; }
  const double a[3] = {dot3(d12, d12), dot3(d13, d13), dot3(d23, d23)};
  const double a12 = a[0], a13 = a[1], a23 = a[2];
  /* D1 = a23 M12 - a12 M23, D2 = a23 M13 - a13 M23 with L^T M_ij L = l_i^2 + l_j^2 + b_ij l_i l_j */
  const double D1[6] = {a23, a23 * h12, 0.0, a23 - a12, -(a12 * h23), -a12};
  const double D2[6] = {a23, 0.0, a23 * h13, -a13, -(a13 * h23), a23 - a13};
  double C1[6], C2[6];
  sym_cof(D1, C1); sym_cof(D2, C2);
  const double c3 = (D2[0] * C2[0] + D2[1] * C2[1]) + D2[2] * C2[2];
  const double c0 = (D1[0] * C1[0] + D1[1] * C1[1]) + D1[2] * C1[2];
  const double c1 = sym_tr(C1, D2), c2 = sym_tr(C2, D1);
  const double g = cubic_root(c2 / c3, c1 / c3, c0 / c3);
  double A[6];
  for (int i = 0; i < 6; i++) A[i] = D1[i] + g * D2[i];
  /* eigenvalues other than the known 0: e^2 + p e + q = 0 */
  double Ac[6];
  sym_cof(A, Ac);
  const double p = -((A[0] + A[3]) + A[5]), q = (Ac[0] + Ac[3]) + Ac[5];
  const double disc = p * p - 4.0 * q, sd = disc > 0.0 ? sqrt(disc) : 0.0;
  double e1, e2;
  if (p < 0.0) { e1 = 0.5 * (-p + sd); e2 = (2.0 * q) / (-p + sd); }
  else { e1 = (2.0 * q) / (-p - sd); e2 = 0.5 * (-p - sd); }
  if (fabs(e1) < fabs(e2)) { const double t = e1; e1 = e2; e2 = t; }
  double v1[3], v2[3];
  eigvec(A, e1, v1); eigvec(A, e2, v2);
  const double ratio = -e2 / e1, s = ratio > 0.0 ? sqrt(ratio) : 0.0;
  /* A = e1 v1 v1^T + e2 v2 v2^T: the two planes (v1 -+ s v2) . L = 0; on each, l1 = w0 l2 + w1 l3, l3 = tau l2 */
  double Ls[4][3];
  int ns = 0;
  for (int side = 0; side < 2; side++) {
    const double sg = side == 0 ? s : -s;
    const double den = sg * v2[0] - v1[0];
    const double w0 = (v1[1] - sg * v2[1]) / den, w1 = (v1[2] - sg * v2[2]) / den;
    /* a13 (l1^2 + l2^2 + b12 l1 l2) - a12 (l1^2 + l3^2 + b13 l1 l3) = 0 → tau^2 + B tau + C = 0 */
    const double qa = (((a13 - a12) * w1) * w1 - ((a12 * b[1]) * w1)) - a12;
    const double qb = ((a13 * b[0]) * w1 - (a12 * b[1]) * w0) - ((2.0 * w0) * w1) * (a12 - a13);
    const double qc = ((((a13 - a12) * w0) * w0) + (a13 * b[0]) * w0) + a13;
    const double B = qb / qa, C = qc / qa;
    const double dq = B * B - 4.0 * C;
    if (!(dq >= 0.0)) continue;
    const double yq = sqrt(dq);
    double tau[2];
    if (B < 0.0) { tau[0] = 0.5 * (-B + yq); tau[1] = (2.0 * C) / (-B + yq); }
    else { tau[0] = (2.0 * C) / (-B - yq); tau[1] = 0.5 * (-B - yq); }
    for (int k = 0; k < 2; k++) {
      if (!(tau[k] > 0.0)) continue;
      const double l2 = sqrt(a23 / (tau[k] * (b[2] + tau[k]) + 1.0));
      const double l3 = tau[k] * l2, l1 = w0 * l2 + w1 * l3;
      if (!(l1 > 0.0)) continue;
      Ls[ns][0] = l1; Ls[ns][1] = l2; Ls[ns][2] = l3; ns++;
    }
  }
  /* pose: R [d12 d13 d12xd13] = [yd1 yd2 yd1xyd2], yd1 = l1 y1 - l2 y2, yd2 = l1 y1 - l3 y3; t = l1 y1 - R x1 */
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
    for (int r = 0; r < 3; r++) { p1[r] = L[0] * y[0][r]; yd1[r] = p1[r] - L[1] * y[1][r]; yd2[r] = p1[r] - L[2] * y[2][r]; }
    cross3(yd1, yd2, yc);
    for (int r = 0; r < 3; r++) { Y[3 * r] = yd1[r]; Y[3 * r + 1] = yd2[r]; Y[3 * r + 2] = yc[r]; }
    double* M = Rt + 12 * out;
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) M[4 * r + c] = (Y[3 * r] * Xi[c] + Y[3 * r + 1] * Xi[3 + c]) + Y[3 * r + 2] * Xi[6 + c];
    for (int r = 0; r < 3; r++) M[4 * r + 3] = p1[r] - ((M[4 * r] * x[0] + M[4 * r + 1] * x[1]) + M[4 * r + 2] * x[2]);
    out++;
  }
  return out;
}

/* inverseSolution = [R^T | -R^T t] of a body-in-world model [R|t] */
static void abs_inverse(const double* M, double* Ri, double* ti) {
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) Ri[3 * r + c] = M[4 * c + r];
  for (int r = 0; r < 3; r++) ti[r] = -((Ri[3 * r] * M[3] + Ri[3 * r + 1] * M[7]) + Ri[3 * r + 2] * M[11]);
}
/* camera-frame ray q of world point p and its norm (FrameAbsolutePoseSacProblem.h:95-126) */
static double abs_ray(const double* Ri, const double* ti, const double* p, const double* co, const double* cr, double* q) {
  double b[3];
  for (int r = 0; r < 3; r++) b[r] = (((Ri[3 * r] * p[0] + Ri[3 * r + 1] * p[1]) + Ri[3 * r + 2] * p[2]) + ti[r]) - co[r];
  for (int r = 0; r < 3; r++) q[r] = (cr[r] * b[0] + cr[3 + r] * b[1]) + cr[6 + r] * b[2];
  return sqrt((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]);
}
static double abs_score(const double* Ri, const double* ti, const double* p, const double* f, double sigma, const double* co, const double* cr) {
  double q[3], e2 = 0.0;
  const double nrm = abs_ray(Ri, ti, p, co, cr, q);
  for (int r = 0; r < 3; r++) { const double e = q[r] / nrm - f[r]; e2 = r == 0 ? e * e : e2 + e * e; }
  return e2 / sigma;
}

/* the hypothesis of one sample (local indices s[4]) of a problem with n correspondences; 0 = invalid sample */
static int hypothesis(const int32_t* s, int n, const double* pts, const double* f, const double* co, const double* cr, double* model) {
  if (n < 4) return 0;
  for (int i = 0; i < 4; i++)
    for (int j = i + 1; j < 4; j++)
      if (s[i] == s[j]) return 0;
  double fb[9], xw[9];
  for (int i = 0; i < 4; i++)
    for (int r = 0; r < 3; r++)
      if (!isfinite(pts[3 * (size_t)s[i] + r]) || !isfinite(f[3 * (size_t)s[i] + r])) return 0;
  for (int i = 0; i < 3; i++)
    for (int r = 0; r < 3; r++) { fb[3 * i + r] = f[3 * (size_t)s[i] + r]; xw[3 * i + r] = pts[3 * (size_t)s[i] + r]; }
  double Rt[48];
  const int ns = ora_p3p(fb, xw, Rt);
  int best = -1;
  double best_score = INFINITY, cand[12];
  for (int k = 0; k < ns; k++) {
    const double* P = Rt + 12 * k;    /* camera from world: x_c = Rcw x + tcw */
    /* body from world: Rbw = Rc Rcw, tbw = Rc tcw + c;  model = [Rbw^T | -Rbw^T tbw] */
    double Rbw[9], tbw[3];
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) Rbw[3 * r + c] = (cr[3 * r] * P[c] + cr[3 * r + 1] * P[4 + c]) + cr[3 * r + 2] * P[8 + c];
      tbw[r] = ((cr[3 * r] * P[3] + cr[3 * r + 1] * P[7]) + cr[3 * r + 2] * P[11]) + co[r];
    }
    double M[12];
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) M[4 * r + c] = Rbw[3 * c + r];
      M[4 * r + 3] = -((Rbw[r] * tbw[0] + Rbw[3 + r] * tbw[1]) + Rbw[6 + r] * tbw[2]);
    }
    double Ri[9], ti[3], q[3];
    abs_inverse(M, Ri, ti);
    const double nrm = abs_ray(Ri, ti, pts + 3 * (size_t)s[3], co, cr, q);
    const double* f4 = f + 3 * (size_t)s[3];
    const double score = 1.0 - (((q[0] / nrm) * f4[0] + (q[1] / nrm) * f4[1]) + (q[2] / nrm) * f4[2]);
    if (score < best_score) { best_score = score; best = k; memcpy(cand, M, sizeof(cand)); }
  }
  if (best < 0) return 0;
  for (int i = 0; i < 12; i++)
    if (!isfinite(cand[i])) return 0;
  memcpy(model, cand, sizeof(cand));
  return 1;
}

/* hypotheses only (the host half of the two-step path that scores with cvb_score_absolute_pose_batch): models [n_samples][12],
 * valid [n_samples] for the samples of one problem */
API void ora_abs_hypotheses(int n, const double* pts, const double* f, const double* cam_off, const double* cam_rot, const int32_t* samples,
                            int n_samples, double* models, uint8_t* valid) {
  for (int s = 0; s < n_samples; s++) {
    memset(models + 12 * (size_t)s, 0, 96);
    valid[s] = (uint8_t)hypothesis(samples + 4 * (size_t)s, n, pts, f, cam_off, cam_rot, models + 12 * (size_t)s);
  }
}

static int count_inliers(const double* M, int n, const double* pts, const double* f, const double* sigma, const double* co, const double* cr,
                         double threshold, uint8_t* mask) {
  double Ri[9], ti[3];
  abs_inverse(M, Ri, ti);
  int cnt = 0;
  for (int i = 0; i < n; i++) {
    const int in = abs_score(Ri, ti, pts + 3 * (size_t)i, f + 3 * (size_t)i, sigma[i], co, cr) < threshold;
    if (mask) mask[i] = (uint8_t)in;
    cnt += in;
  }
  return cnt;
}

/* Samples [n_prob][n_samples][4] (problem-local indices), correspondences concatenated by prob_ptr[n_prob+1], one camera per
 * problem.  Per problem: best_sample (-1 = none), best_model [12], best_count, iterations, consumed (samples read by the
 * selection).  inlier_mask [N_total] (nullable): the best model's mask, 0 where there is none.  sample_model [..][12],
 * sample_valid, sample_count (nullable together): every sample's hypothesis (zeros when invalid) and inlier count — when
 * requested, every sample is solved, not only the consumed ones. */
API void ora_ransac_absolute_pose(int n_prob, const int32_t* prob_ptr, const double* pts, const double* f, const double* sigma,
                                  const double* cam_off, const double* cam_rot, const int32_t* samples, int n_samples, double threshold,
                                  int max_iterations, double probability, int32_t* best_sample, double* best_model, int32_t* best_count,
                                  int32_t* iterations, int32_t* consumed, uint8_t* inlier_mask, double* sample_model, uint8_t* sample_valid,
                                  int32_t* sample_count) {
  const double log_p = log(1.0 - probability), eps = 2.220446049250313e-16;
  const long long max_skip = 10LL * max_iterations;
#pragma omp parallel for schedule(dynamic, 1)
  for (int pi = 0; pi < n_prob; pi++) {
    const int off = prob_ptr[pi], n = prob_ptr[pi + 1] - prob_ptr[pi];
    const double *P = pts + 3 * (size_t)off, *F = f + 3 * (size_t)off, *S = sigma + off;
    const double *co = cam_off + 3 * (size_t)pi, *cr = cam_rot + 9 * (size_t)pi;
    int best = -1, best_n = 0, it = 0, s_used = 0;
    long long skipped = 0;
    double k = (double)max_iterations, bm[12] = {0};
    for (int s = 0; s < n_samples; s++) {
      const int running = it < max_iterations && (double)it < k && skipped < max_skip;
      if (!running && !sample_model) break;
      double M[12] = {0};
      const int valid = hypothesis(samples + 4 * ((size_t)pi * n_samples + s), n, P, F, co, cr, M);
      const int cnt = valid ? count_inliers(M, n, P, F, S, co, cr, threshold, NULL) : 0;
      if (sample_model) {
        const size_t g = (size_t)pi * n_samples + s;
        memcpy(sample_model + 12 * g, M, sizeof(M)); sample_valid[g] = (uint8_t)valid; sample_count[g] = cnt;
      }
      if (!running) continue;
      s_used++;
      if (!valid) { skipped++; continue; }
      if (cnt > best_n) {
        best_n = cnt; best = s; memcpy(bm, M, sizeof(bm));
        const double w = (double)cnt / (double)n;
        double pno = 1.0 - ((w * w) * w) * w;
        pno = pno > eps ? pno : eps;
        pno = pno < 1.0 - eps ? pno : 1.0 - eps;
        k = log_p / log(pno);
      }
      it++;
    }
    best_sample[pi] = best; best_count[pi] = best_n; iterations[pi] = it; consumed[pi] = s_used;
    memcpy(best_model + 12 * (size_t)pi, bm, sizeof(bm));
    if (inlier_mask) {
      if (best >= 0) count_inliers(bm, n, P, F, S, co, cr, threshold, inlier_mask + off);
      else memset(inlier_mask + off, 0, (size_t)n);
    }
  }
}
