/* oracle/ransac_rel_oracle.c — CPU restatement of the non-central relative-pose (17-point) RANSAC of
 * RelNonCentralPosSolver::computeNonCentralRelPose (RelNonCentralPosSolver.cpp:146-173) from caller-supplied samples.
 * TEST INFRASTRUCTURE ONLY (tests/, tools/); never linked into covins_b200/.  It is the bit-for-bit reference of
 * cvb_ransac_noncentral_relative_pose_batch (covins_b200/csrc/ransac_rel.cu); the absolute-pose restatement
 * (ransac_oracle.c) and the scoring oracle (geom_oracle.c) are left alone.
 * Only + - * / and sqrt, fixed iteration counts; plain IEEE double without contraction (compile with -ffp-contract=off).
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define API __attribute__((visibility("default")))

static double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
/* 3x3 inverse by the adjugate (the same expression as ransac_oracle.c and the device's inv3) */
static void inv3(const double* m, double* o) {
  const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
  const double det = (m[0] * c00 + m[1] * c01) + m[2] * c02;
  o[0] = c00 / det; o[1] = (m[2] * m[7] - m[1] * m[8]) / det; o[2] = (m[1] * m[5] - m[2] * m[4]) / det;
  o[3] = c01 / det; o[4] = (m[0] * m[8] - m[2] * m[6]) / det; o[5] = (m[2] * m[3] - m[0] * m[5]) / det;
  o[6] = c02 / det; o[7] = (m[1] * m[6] - m[0] * m[7]) / det; o[8] = (m[0] * m[4] - m[1] * m[3]) / det;
}

/* ASSUMPTIONS (opengv is not in the tree):
 *   [T] the model's t is the least-squares solution of the sample's 17 generalised epipolar rows with R fixed; opengv's
 *       seventeenpt may recover t from E instead.  On noise-free data both give the same model.
 *   [S] the 17-point RANSAC scores with FrameRelativePoseSacProblem's score (as the 5-point one), applied per camera pair:
 *       R_p = Rc1^T R Rc2, t_p = Rc1^T (R c2 + t - c1).
 *   [K] as the absolute-pose RANSAC: an invalid sample does not consume an iteration, at most 10 * max_iterations skips.
 *   Selection = covins_b200.placerec.ransac_select over the valid samples in order (sample_size 17), w^17 as a left-to-right
 *   product chain.
 * Hypothesis: Plücker lines d = Rc f, m = c x d; row i of A (17x18) = [vec(d1 d2^T), vec(d1 m2^T + m1 d2^T)] (row-major);
 * null vector x = Q e18 of the Householder QR of A^T, invalid if min |r_kk| < REL_RANK_TOL max |r_kk|; R' = x[9:18] with
 * det > 0 (negated if det < 0, invalid if 0); R = polar factor of R' (scaled to |R'|_F = sqrt(3), REL_POLAR_ITERS Newton steps
 * X <- (X + X^-T) / 2); t from the 3x3 normal equations of (R d2 x d1) . t = -(d1^T R m2 + m1^T R d2) summed in sample order.
 * Every sum is sequential, first term first, in the order written here: the CUDA path computes the same sums in the same order.
 */
#define REL_SAMPLE 17
#define REL_MAX_CAMS 8
#define REL_RANK_TOL 1e-10
enum { REL_POLAR_ITERS = 12 };

/* d = Rc f, m = c x d of camera cam (offset (3) at co, rotation (9, row-major) at cr) */
static void plucker(const double* co, const double* cr, const double* f, double* d, double* m) {
  for (int r = 0; r < 3; r++) d[r] = (cr[3 * r] * f[0] + cr[3 * r + 1] * f[1]) + cr[3 * r + 2] * f[2];
  cross3(co, d, m);
}

static int finite_n(const double* v, size_t n) {
  for (size_t i = 0; i < n; i++)
    if (!isfinite(v[i])) return 0;
  return 1;
}

/* camera-pair model [R_p|t_p] of rig-frame model M (X1 = R X2 + t), camera 1 (co1, cr1) of rig 1, camera 2 (co2, cr2) of rig 2 */
static void pair_model(const double* M, const double* co1, const double* cr1, const double* co2, const double* cr2, double* P) {
  double RR[9], u[3];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) RR[3 * r + c] = (M[4 * r] * cr2[c] + M[4 * r + 1] * cr2[3 + c]) + M[4 * r + 2] * cr2[6 + c];
  for (int r = 0; r < 3; r++) u[r] = (((M[4 * r] * co2[0] + M[4 * r + 1] * co2[1]) + M[4 * r + 2] * co2[2]) + M[4 * r + 3]) - co1[r];
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) P[4 * r + c] = (cr1[r] * RR[c] + cr1[3 + r] * RR[3 + c]) + cr1[6 + r] * RR[6 + c];
    P[4 * r + 3] = (cr1[r] * u[0] + cr1[3 + r] * u[1]) + cr1[6 + r] * u[2];
  }
}

/* cvb_score_relative_pose_batch's per-correspondence score (geom_oracle.c:ora_score_relative_pose) under P = [R12|t12],
 * ti = -R12^T t12 */
static double rel_score(const double* M, const double* ti, const double* a, const double* bb, double s1, double s2) {
  const double t[3] = {M[3], M[7], M[11]};
  double u[3];
  for (int r = 0; r < 3; r++) u[r] = (M[4 * r] * bb[0] + M[4 * r + 1] * bb[1]) + M[4 * r + 2] * bb[2];
  const double b0 = (t[0] * a[0] + t[1] * a[1]) + t[2] * a[2], b1 = (t[0] * u[0] + t[1] * u[1]) + t[2] * u[2];
  const double A00 = (a[0] * a[0] + a[1] * a[1]) + a[2] * a[2], A10 = (a[0] * u[0] + a[1] * u[1]) + a[2] * u[2];
  const double A01 = -A10, A11 = -((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]);
  const double det = A00 * A11 - A01 * A10;
  const double l0 = (A11 * b0 - A01 * b1) / det, l1 = (A00 * b1 - A10 * b0) / det;
  double X[3], r2[3];
  for (int r = 0; r < 3; r++) X[r] = (l0 * a[r] + (t[r] + l1 * u[r])) / 2.0;
  for (int r = 0; r < 3; r++) r2[r] = ((M[r] * X[0] + M[4 + r] * X[1]) + M[8 + r] * X[2]) + ti[r];
  const double n1 = sqrt((X[0] * X[0] + X[1] * X[1]) + X[2] * X[2]), n2 = sqrt((r2[0] * r2[0] + r2[1] * r2[1]) + r2[2] * r2[2]);
  double e1 = 0.0, e2 = 0.0;
  for (int r = 0; r < 3; r++) {
    const double d1 = X[r] / n1 - a[r], d2 = r2[r] / n2 - bb[r];
    e1 = r == 0 ? d1 * d1 : e1 + d1 * d1;
    e2 = r == 0 ? d2 * d2 : e2 + d2 * d2;
  }
  return e1 * 0.5 / s1 + e2 * 0.5 / s2;
}

/* One problem's view of the inputs: correspondences and the two rigs (cameras as offset (3) then rotation (9)). */
typedef struct {
  int n, nc1, nc2;
  const double *f1, *f2, *s1, *s2;
  const int32_t *cam1, *cam2;
  double rig1[REL_MAX_CAMS][12], rig2[REL_MAX_CAMS][12];
  int rigs_finite;
} rel_problem;

static void rel_problem_init(rel_problem* P, int n, const double* f1, const double* f2, const double* s1, const double* s2, const int32_t* cam1,
                             const int32_t* cam2, int nc1, const double* co1, const double* cr1, int nc2, const double* co2, const double* cr2) {
  P->n = n; P->nc1 = nc1; P->nc2 = nc2; P->f1 = f1; P->f2 = f2; P->s1 = s1; P->s2 = s2; P->cam1 = cam1; P->cam2 = cam2;
  P->rigs_finite = 1;
  for (int j = 0; j < nc1; j++) {
    memcpy(P->rig1[j], co1 + 3 * (size_t)j, 24); memcpy(P->rig1[j] + 3, cr1 + 9 * (size_t)j, 72);
    P->rigs_finite &= finite_n(P->rig1[j], 12);
  }
  for (int j = 0; j < nc2; j++) {
    memcpy(P->rig2[j], co2 + 3 * (size_t)j, 24); memcpy(P->rig2[j] + 3, cr2 + 9 * (size_t)j, 72);
    P->rigs_finite &= finite_n(P->rig2[j], 12);
  }
}

/* the hypothesis of one sample s[17]; 0 = invalid.  rank_ratio (nullable): min |r_kk| / max |r_kk| of the QR. */
static int rel_hypothesis(const rel_problem* P, const int32_t* s, double* model, double* rank_ratio) {
  if (rank_ratio) *rank_ratio = 0.0;
  if (P->n < REL_SAMPLE) return 0;
  for (int i = 0; i < REL_SAMPLE; i++)
    for (int j = i + 1; j < REL_SAMPLE; j++)
      if (s[i] == s[j]) return 0;
  if (!P->rigs_finite) return 0;
  for (int i = 0; i < REL_SAMPLE; i++)
    if (!finite_n(P->f1 + 3 * (size_t)s[i], 3) || !finite_n(P->f2 + 3 * (size_t)s[i], 3)) return 0;
  /* At[k] = row k of A = column k of A^T; dm[k] = d1, m1, d2, m2 */
  double At[REL_SAMPLE][18], dm[REL_SAMPLE][12];
  for (int i = 0; i < REL_SAMPLE; i++) {
    const double* c1 = P->rig1[P->cam1[s[i]]];
    const double* c2 = P->rig2[P->cam2[s[i]]];
    double *d1 = dm[i], *m1 = dm[i] + 3, *d2 = dm[i] + 6, *m2 = dm[i] + 9;
    plucker(c1, c1 + 3, P->f1 + 3 * (size_t)s[i], d1, m1);
    plucker(c2, c2 + 3, P->f2 + 3 * (size_t)s[i], d2, m2);
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) { At[i][3 * a + b] = d1[a] * d2[b]; At[i][9 + 3 * a + b] = d1[a] * m2[b] + m1[a] * d2[b]; }
  }
  /* Householder QR of A^T: step k reflects rows k..17; v_k overwrites At[k][k..17], r_kk = alpha[k], |v_k|^2 = vtv[k] */
  double alpha[REL_SAMPLE], vtv[REL_SAMPLE];
  for (int k = 0; k < REL_SAMPLE; k++) {
    double* col = At[k];
    double ss = 0.0;
    for (int i = k; i < 18; i++) ss = i == k ? col[i] * col[i] : ss + col[i] * col[i];
    const double sigma = sqrt(ss), ak = col[k];
    alpha[k] = ak >= 0.0 ? -sigma : sigma;
    col[k] = ak - alpha[k];
    vtv[k] = 2.0 * (ss + fabs(ak) * sigma);
    for (int j = k + 1; j < REL_SAMPLE; j++) {
      double dot = 0.0;
      for (int i = k; i < 18; i++) dot = i == k ? col[i] * At[j][i] : dot + col[i] * At[j][i];
      const double c = (2.0 * dot) / vtv[k];
      for (int i = k; i < 18; i++) At[j][i] = At[j][i] - c * col[i];
    }
  }
  double rmax = 0.0;
  for (int k = 0; k < REL_SAMPLE; k++) rmax = fabs(alpha[k]) > rmax ? fabs(alpha[k]) : rmax;
  int full_rank = rmax > 0.0;
  double rmin = rmax;
  for (int k = 0; k < REL_SAMPLE; k++) {
    if (!(fabs(alpha[k]) >= REL_RANK_TOL * rmax)) full_rank = 0;
    rmin = fabs(alpha[k]) < rmin ? fabs(alpha[k]) : rmin;
  }
  if (rank_ratio) *rank_ratio = rmax > 0.0 ? rmin / rmax : 0.0;
  if (!full_rank) return 0;
  /* x = H_0 H_1 ... H_16 e18 */
  double x[18];
  for (int i = 0; i < 18; i++) x[i] = i == 17 ? 1.0 : 0.0;
  for (int k = REL_SAMPLE - 1; k >= 0; k--) {
    double dot = 0.0;
    for (int i = k; i < 18; i++) dot = i == k ? At[k][i] * x[i] : dot + At[k][i] * x[i];
    const double c = (2.0 * dot) / vtv[k];
    for (int i = k; i < 18; i++) x[i] = x[i] - c * At[k][i];
  }
  /* R' = x[9:18], det > 0; polar factor by Newton from |R'|_F = sqrt(3) */
  double X[9], Xi[9];
  for (int i = 0; i < 9; i++) X[i] = x[9 + i];
  const double det = (X[0] * (X[4] * X[8] - X[5] * X[7]) + X[1] * (X[5] * X[6] - X[3] * X[8])) + X[2] * (X[3] * X[7] - X[4] * X[6]);
  if (!(det > 0.0 || det < 0.0)) return 0;
  double fro = 0.0;
  for (int i = 0; i < 9; i++) fro = i == 0 ? X[i] * X[i] : fro + X[i] * X[i];
  const double scale = sqrt(3.0 / fro);
  for (int i = 0; i < 9; i++) X[i] = det < 0.0 ? -(X[i] * scale) : X[i] * scale;
  for (int it = 0; it < REL_POLAR_ITERS; it++) {
    inv3(X, Xi);
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) X[3 * r + c] = 0.5 * (X[3 * r + c] + Xi[3 * c + r]);
  }
  /* t: normal equations N t = b of g_i . t = h_i, g_i = R d2 x d1, h_i = -(d1 . R m2 + m1 . R d2) */
  double N[9], b[3], Ni[9];
  for (int i = 0; i < REL_SAMPLE; i++) {
    const double *d1 = dm[i], *m1 = dm[i] + 3, *d2 = dm[i] + 6, *m2 = dm[i] + 9;
    double u[3], w[3], g[3];
    for (int r = 0; r < 3; r++) {
      u[r] = (X[3 * r] * d2[0] + X[3 * r + 1] * d2[1]) + X[3 * r + 2] * d2[2];
      w[r] = (X[3 * r] * m2[0] + X[3 * r + 1] * m2[1]) + X[3 * r + 2] * m2[2];
    }
    cross3(u, d1, g);
    const double h = -(dot3(d1, w) + dot3(m1, u));
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) N[3 * r + c] = i == 0 ? g[r] * g[c] : N[3 * r + c] + g[r] * g[c];
      b[r] = i == 0 ? g[r] * h : b[r] + g[r] * h;
    }
  }
  inv3(N, Ni);
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) model[4 * r + c] = X[3 * r + c];
    model[4 * r + 3] = (Ni[3 * r] * b[0] + Ni[3 * r + 1] * b[1]) + Ni[3 * r + 2] * b[2];
  }
  return finite_n(model, 12);
}

static int rel_count(const rel_problem* P, const double* M, double threshold, double* scores, uint8_t* mask) {
  double pm[REL_MAX_CAMS * REL_MAX_CAMS][15];   /* per camera pair: [R_p|t_p] then ti = -R_p^T t_p */
  for (int j1 = 0; j1 < P->nc1; j1++)
    for (int j2 = 0; j2 < P->nc2; j2++) {
      double* q = pm[j1 * P->nc2 + j2];
      pair_model(M, P->rig1[j1], P->rig1[j1] + 3, P->rig2[j2], P->rig2[j2] + 3, q);
      for (int r = 0; r < 3; r++) q[12 + r] = -((q[r] * q[3] + q[4 + r] * q[7]) + q[8 + r] * q[11]);
    }
  int cnt = 0;
  for (int i = 0; i < P->n; i++) {
    const double* q = pm[P->cam1[i] * P->nc2 + P->cam2[i]];
    const double s = rel_score(q, q + 12, P->f1 + 3 * (size_t)i, P->f2 + 3 * (size_t)i, P->s1[i], P->s2[i]);
    const int in = s < threshold;
    if (scores) scores[i] = s;
    if (mask) mask[i] = (uint8_t)in;
    cnt += in;
  }
  return cnt;
}

/* one sample: correspondences of one problem (n), its rigs (nc1 / nc2 cameras), the sample's 17 local indices → model [12],
 * rank_ratio (nullable); returns valid */
API int ora_rel17(int n, const double* f1, const double* f2, const int32_t* cam1, const int32_t* cam2, int nc1, const double* cam_off1,
                  const double* cam_rot1, int nc2, const double* cam_off2, const double* cam_rot2, const int32_t* sample, double* model,
                  double* rank_ratio) {
  rel_problem P;
  rel_problem_init(&P, n, f1, f2, NULL, NULL, cam1, cam2, nc1, cam_off1, cam_rot1, nc2, cam_off2, cam_rot2);
  memset(model, 0, 96);
  const int v = rel_hypothesis(&P, sample, model, rank_ratio);
  if (!v) memset(model, 0, 96);
  return v;
}

/* camera-pair model of a rig-frame model: M [12] → P [12] */
API void ora_rel_pair_model(const double* M, const double* cam_off1, const double* cam_rot1, const double* cam_off2, const double* cam_rot2, double* P) {
  pair_model(M, cam_off1, cam_rot1, cam_off2, cam_rot2, P);
}

/* scores / inlier flags / counts of n_hyp rig-frame models over one problem's correspondences (scores, inlier: [n_hyp][n],
 * nullable) */
API void ora_score_noncentral_relative_pose(const double* model, int n_hyp, int n, const double* f1, const double* f2, const double* sigma1,
                                            const double* sigma2, const int32_t* cam1, const int32_t* cam2, int nc1, const double* cam_off1,
                                            const double* cam_rot1, int nc2, const double* cam_off2, const double* cam_rot2, double threshold,
                                            double* scores, uint8_t* inlier, int32_t* n_inliers) {
  rel_problem P;
  rel_problem_init(&P, n, f1, f2, sigma1, sigma2, cam1, cam2, nc1, cam_off1, cam_rot1, nc2, cam_off2, cam_rot2);
  for (int h = 0; h < n_hyp; h++)
    n_inliers[h] = rel_count(&P, model + 12 * (size_t)h, threshold, scores ? scores + (size_t)h * n : NULL, inlier ? inlier + (size_t)h * n : NULL);
}

/* hypotheses only (host 17-point solves): models [n_samples][12], valid [n_samples] for the samples of one problem */
API void ora_rel_hypotheses(int n, const double* f1, const double* f2, const int32_t* cam1, const int32_t* cam2, int nc1, const double* cam_off1,
                            const double* cam_rot1, int nc2, const double* cam_off2, const double* cam_rot2, const int32_t* samples, int n_samples,
                            double* models, uint8_t* valid) {
  rel_problem P;
  rel_problem_init(&P, n, f1, f2, NULL, NULL, cam1, cam2, nc1, cam_off1, cam_rot1, nc2, cam_off2, cam_rot2);
  for (int s = 0; s < n_samples; s++) {
    double* M = models + 12 * (size_t)s;
    memset(M, 0, 96);
    valid[s] = (uint8_t)rel_hypothesis(&P, samples + REL_SAMPLE * (size_t)s, M, NULL);
    if (!valid[s]) memset(M, 0, 96);
  }
}

/* Same arguments and outputs as cvb_ransac_noncentral_relative_pose_batch (flattened), the selection as
 * ora_ransac_absolute_pose with sample size 17. */
API void ora_ransac_noncentral_relative_pose(int n_prob, const int32_t* prob_ptr, const double* f1, const double* f2, const double* sigma1,
                                             const double* sigma2, const int32_t* cam1, const int32_t* cam2, const int32_t* cam_ptr1,
                                             const double* cam_off1, const double* cam_rot1, const int32_t* cam_ptr2, const double* cam_off2,
                                             const double* cam_rot2, const int32_t* samples, int n_samples, double threshold, int max_iterations,
                                             double probability, int32_t* best_sample, double* best_model, int32_t* best_count,
                                             int32_t* iterations, int32_t* consumed, uint8_t* inlier_mask, double* sample_model,
                                             uint8_t* sample_valid, int32_t* sample_count) {
  const double log_p = log(1.0 - probability), eps = 2.220446049250313e-16;
  const long long max_skip = 10LL * max_iterations;
#pragma omp parallel for schedule(dynamic, 1)
  for (int pi = 0; pi < n_prob; pi++) {
    const int off = prob_ptr[pi], n = prob_ptr[pi + 1] - prob_ptr[pi];
    rel_problem P;
    rel_problem_init(&P, n, f1 + 3 * (size_t)off, f2 + 3 * (size_t)off, sigma1 + off, sigma2 + off, cam1 + off, cam2 + off,
                     cam_ptr1[pi + 1] - cam_ptr1[pi], cam_off1 + 3 * (size_t)cam_ptr1[pi], cam_rot1 + 9 * (size_t)cam_ptr1[pi],
                     cam_ptr2[pi + 1] - cam_ptr2[pi], cam_off2 + 3 * (size_t)cam_ptr2[pi], cam_rot2 + 9 * (size_t)cam_ptr2[pi]);
    int best = -1, best_n = 0, it = 0, s_used = 0;
    long long skipped = 0;
    double k = (double)max_iterations, bm[12] = {0};
    for (int s = 0; s < n_samples; s++) {
      const int running = it < max_iterations && (double)it < k && skipped < max_skip;
      if (!running && !sample_model) break;
      double M[12] = {0};
      const int valid = rel_hypothesis(&P, samples + REL_SAMPLE * ((size_t)pi * n_samples + s), M, NULL);
      if (!valid) memset(M, 0, sizeof(M));
      const int cnt = valid ? rel_count(&P, M, threshold, NULL, NULL) : 0;
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
        double wp = w;
        for (int e = 1; e < REL_SAMPLE; e++) wp = wp * w;
        double pno = 1.0 - wp;
        pno = pno > eps ? pno : eps;
        pno = pno < 1.0 - eps ? pno : 1.0 - eps;
        k = log_p / log(pno);
      }
      it++;
    }
    best_sample[pi] = best; best_count[pi] = best_n; iterations[pi] = it; consumed[pi] = s_used;
    memcpy(best_model + 12 * (size_t)pi, bm, sizeof(bm));
    if (inlier_mask) {
      if (best >= 0) rel_count(&P, bm, threshold, NULL, inlier_mask + off);
      else memset(inlier_mask + off, 0, (size_t)n);
    }
  }
}
