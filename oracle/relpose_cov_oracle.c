/* oracle/relpose_cov_oracle.c — CPU restatement of the sampling-based 6x6 covariance of the non-central relative pose
 * (RelNonCentralPosSolver::computeNonCentralRelPose, RelNonCentralPosSolver.cpp:199,236,276-279) from caller-supplied samples.
 * TEST INFRASTRUCTURE ONLY (tests/, tools/); never linked into covins_b200/.  It is the bit-for-bit reference of
 * cvb_noncentral_relative_pose_covariance_batch (covins_b200/csrc/ransac_rel.cu, rel_cov_solve_kernel / rel_cov_reduce_kernel).
 * It includes the 17-point restatement (ransac_rel_oracle.c, unchanged) for rel_hypothesis and the problem view.
 * Only + - * / and sqrt; plain IEEE double without contraction (compile with -ffp-contract=off).
 *
 * ASSUMPTIONS (robopt and opengv are not in the tree):
 *   [D] rotation first, right-side deviation, 2 vec(q) rather than Log: delta = [2 vec(q); t_s - t_ref] with q the quaternion of
 *       R_ref^T R_s, so that cov is in the coordinates of the residual it whitens, the pose-graph between factor
 *       e = [2 vec(q_m^-1 q_hat); t_hat - t_m] (covins_b200/csrc/ba_math.cuh).  robopt's quaternion::Minus may instead be a
 *       left-side Log (SURVEY A.2): the two disagree.
 *   [M] the second moment about the reference, divided by n_valid: the mean is not subtracted, the divisor is not n - 1.
 *   [S] minimal 17-point re-solves (rel_hypothesis), not a non-minimal solver.
 * Per sample: rel_hypothesis; an invalid sample is skipped and not counted.  q by Eigen's matrix-to-quaternion branches
 * (QuaternionBase::operator=(MatrixBase), as covins_b200_shim.hpp's transform_to_pose7): trace > 0, else the largest diagonal
 * entry (the first on ties); q negated if w < 0.  R_ref^T R_s entry (r, c) = (ref_0r s_0c + ref_1r s_1c) + ref_2r s_2c.
 * Per problem: cov_rc = (sum over the valid samples in sample order of delta_r delta_c, from 0.0) / n_valid; 0 if n_valid = 0.
 * A problem whose reference model is all zeros is skipped (n_valid = 0, samples not read).
 */
#include "ransac_rel_oracle.c"

#include <omp.h>
#include <stdlib.h>

/* q = (x, y, z, w) of the row-major rotation m, Eigen's branch for the largest diagonal entry i */
static void rel_quat_diag(const double* m, int i, double* q) {
  const int j = (i + 1) % 3, k = (j + 1) % 3;
  double t = sqrt(((m[4 * i] - m[4 * j]) - m[4 * k]) + 1.0);
  q[i] = 0.5 * t;
  t = 0.5 / t;
  q[3] = (m[3 * k + j] - m[3 * j + k]) * t;
  q[j] = (m[3 * j + i] + m[3 * i + j]) * t;
  q[k] = (m[3 * k + i] + m[3 * i + k]) * t;
}

/* delta [6] of model M against the reference ref (both 3x4 row-major) */
static void rel_deviation(const double* ref, const double* M, double* d) {
  double m[9], q[4];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) m[3 * r + c] = (ref[r] * M[c] + ref[4 + r] * M[4 + c]) + ref[8 + r] * M[8 + c];
  const double tr = (m[0] + m[4]) + m[8];
  if (tr > 0.0) {
    double t = sqrt(tr + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[7] - m[5]) * t; q[1] = (m[2] - m[6]) * t; q[2] = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[4 * i]) i = 2;
    rel_quat_diag(m, i, q);
  }
  const double s = q[3] < 0.0 ? -2.0 : 2.0;
  for (int r = 0; r < 3; r++) {
    d[r] = s * q[r];
    d[3 + r] = M[4 * r + 3] - ref[4 * r + 3];
  }
}

static int rel_model_is_zero(const double* M) {
  for (int i = 0; i < 12; i++)
    if (M[i] != 0.0) return 0;
  return 1;
}

/* the deviation of one model from a reference: ref [12], model [12] → delta [6] */
API void ora_rel_deviation(const double* ref, const double* model, double* delta) { rel_deviation(ref, model, delta); }

/* Same arguments and outputs as cvb_noncentral_relative_pose_covariance_batch (flattened; no sigmas).  The samples of all
 * problems are solved in parallel on n_threads OpenMP threads (0: the OpenMP default); each problem's sum is then taken in
 * sample order. */
API void ora_noncentral_relative_pose_covariance(int n_prob, const int32_t* prob_ptr, const double* f1, const double* f2, const int32_t* cam1,
                                                 const int32_t* cam2, const int32_t* cam_ptr1, const double* cam_off1, const double* cam_rot1,
                                                 const int32_t* cam_ptr2, const double* cam_off2, const double* cam_rot2, const int32_t* samples,
                                                 int n_samples, const double* ref_model, int n_threads, double* cov, int32_t* n_valid,
                                                 double* sample_delta, uint8_t* sample_valid) {
  const size_t S_all = (size_t)n_prob * n_samples;
  double* delta = sample_delta ? sample_delta : malloc((S_all ? S_all : 1) * 6 * sizeof(double));
  uint8_t* valid = sample_valid ? sample_valid : malloc(S_all ? S_all : 1);
  const long long total = (long long)S_all;
#pragma omp parallel for schedule(dynamic, 4) num_threads(n_threads > 0 ? n_threads : omp_get_max_threads())
  for (long long g = 0; g < total; g++) {
    const int pi = (int)(g / n_samples);
    const double* ref = ref_model + 12 * (size_t)pi;
    double* d = delta + 6 * (size_t)g;
    for (int i = 0; i < 6; i++) d[i] = 0.0;
    valid[g] = 0;
    if (rel_model_is_zero(ref)) continue;
    const int off = prob_ptr[pi], n = prob_ptr[pi + 1] - off;
    rel_problem P;
    rel_problem_init(&P, n, f1 + 3 * (size_t)off, f2 + 3 * (size_t)off, NULL, NULL, cam1 + off, cam2 + off, cam_ptr1[pi + 1] - cam_ptr1[pi],
                     cam_off1 + 3 * (size_t)cam_ptr1[pi], cam_rot1 + 9 * (size_t)cam_ptr1[pi], cam_ptr2[pi + 1] - cam_ptr2[pi],
                     cam_off2 + 3 * (size_t)cam_ptr2[pi], cam_rot2 + 9 * (size_t)cam_ptr2[pi]);
    double M[12] = {0};
    if (!rel_hypothesis(&P, samples + REL_SAMPLE * (size_t)g, M, NULL)) continue;
    rel_deviation(ref, M, d);
    valid[g] = 1;
  }
  for (int pi = 0; pi < n_prob; pi++) {
    double acc[36];
    int nv = 0;
    for (int i = 0; i < 36; i++) acc[i] = 0.0;
    for (int s = 0; s < n_samples; s++) {
      const size_t g = (size_t)pi * n_samples + s;
      if (!valid[g]) continue;
      const double* d = delta + 6 * g;
      for (int r = 0; r < 6; r++)
        for (int c = 0; c < 6; c++) acc[6 * r + c] = acc[6 * r + c] + d[r] * d[c];
      nv++;
    }
    for (int i = 0; i < 36; i++) cov[36 * (size_t)pi + i] = nv > 0 ? acc[i] / (double)nv : 0.0;
    n_valid[pi] = nv;
  }
  if (!sample_delta) free(delta);
  if (!sample_valid) free(valid);
}
