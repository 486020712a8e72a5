// ransac_rel.cu — the non-central relative-pose RANSAC of RelNonCentralPosSolver::computeNonCentralRelPose (17-point,
// RelNonCentralPosSolver.cpp:146-173; the COVINS_G verification of a place-recognition candidate, each side a rig of a
// keyframe and its neighbours) on the GPU from caller-supplied samples: the 17-point solve per sample, scoring per camera pair
// and the sequential model selection of opengv's Ransac::computeModel, for a batch of problems (candidates) in one launch.
//
// The same kernel, instantiated with the 5-point solver (rel5), runs the central relative-pose RANSAC of
// RelNonCentralPosSolver::computePose (cvb_ransac_central_relative_pose_batch): a central problem is a non-central one with a
// single identity camera per side.
//
// The 17-point solver also serves the sampling-based 6x6 covariance of computeNonCentralRelPose
// (cvb_noncentral_relative_pose_covariance_batch, rel_cov_solve_kernel / rel_cov_reduce_kernel at the end of the file;
// oracle/relpose_cov_oracle.c restates it).
//
// One CTA per problem, both rigs staged in shared memory, driven by ransac_cta (ransac_common.cuh, shared with ransac_abs.cu):
// the waves of kWave samples, the scoring, the selection with its early stop and the inlier mask.  This file supplies the
// solvers: in each wave a warp solves one sample at a time (lane k owns column k of A^T in its warp's shared-memory area, the
// Householder QR warp_householder serves both solvers, every norm and dot product is a sequential sum inside one lane); a
// hypothesis is scored through its camera-pair models in the warp's area.
//
// Only + - * / and sqrt as explicit non-fused intrinsics, fixed iteration counts: the results are bit-identical to the plain
// IEEE restatement compiled with -ffp-contract=off (oracle/ransac_rel_oracle.c for the 17-point solver,
// oracle/ransac_rel5_oracle.c for the 5-point one; their headers state the problems and their assumptions; so does
// include/covins_b200.h).
#include <algorithm>
#include <type_traits>

#include <cub/block/block_scan.cuh>

#include "ransac_common.cuh"

namespace {

constexpr int kSample = 17, kMaxCams = CVB_REL_MAX_CAMS;
constexpr int kPolarIters = 12;
constexpr double kRankTol = 1e-10;
// per-warp shared-memory area (doubles): the solver's arrays, or the camera-pair models (12 each) while scoring
constexpr int kLd = 19;   // leading dimension of A^T's columns (17 lanes hit distinct banks)
constexpr int oAt = 0, oDm = oAt + kSample * kLd, oX = oDm + kSample * 12, oAl = oX + 18, oVt = oAl + kSample, oGh = oVt + kSample,
              oR = oGh + kSample * 4, kSolveArea = oR + 9;
constexpr int kPairArea = 12;

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

// Householder QR of the kRows x kCols matrix in the warp's shared memory A, lane j owning column j (leading dimension kLd): step
// k reflects rows k .. kRows - 1; v_k overwrites column k from row k, r_kk = al[k], |v_k|^2 = vt[k].  Returns the rank test,
// every |r_kk| >= kRankTol * max |r_kk| and max |r_kk| > 0, which every lane evaluates on the same values (warp-uniform).
template <int kRows, int kCols, int kLd>
__device__ __forceinline__ bool warp_householder(double* A, double* al, double* vt, int lane) {
  for (int k = 0; k < kCols; k++) {
    if (lane == k) {
      double* col = A + kLd * k;
      double ss = 0.0;
      for (int i = k; i < kRows; i++) ss = i == k ? mul(col[i], col[i]) : add(ss, mul(col[i], col[i]));
      const double sigma = __dsqrt_rn(ss), ak = col[k];
      const double alpha = ak >= 0.0 ? -sigma : sigma;
      col[k] = sub(ak, alpha);
      al[k] = alpha;
      vt[k] = mul(2.0, add(ss, mul(fabs(ak), sigma)));
    }
    __syncwarp();
    if (lane > k && lane < kCols) {
      const double* v = A + kLd * k;
      double* a = A + kLd * lane;
      double dot = 0.0;
      for (int i = k; i < kRows; i++) dot = i == k ? mul(v[i], a[i]) : add(dot, mul(v[i], a[i]));
      const double c = __ddiv_rn(mul(2.0, dot), vt[k]);
      for (int i = k; i < kRows; i++) a[i] = sub(a[i], mul(c, v[i]));
    }
    __syncwarp();
  }
  double rmax = 0.0;
  for (int k = 0; k < kCols; k++) rmax = fabs(al[k]) > rmax ? fabs(al[k]) : rmax;
  bool good = rmax > 0.0;
  for (int k = 0; k < kCols; k++)
    if (!(fabs(al[k]) >= mul(kRankTol, rmax))) good = false;
  return good;
}

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
  if (!warp_householder<18, kSample, kLd>(At, al, vt, lane)) return false;   // QR of A^T (18 x 17)
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
  int good = 0;
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

// ---- the 5-point hypothesis of a central problem (oracle/ransac_rel5_oracle.c:rel5_hypothesis states it step by step) ----
constexpr int kSample5 = 5, kBisect = 64, kNewton = 4, kPolish = 6;
constexpr double kPivotTol = 1e-10;
// per-warp area (doubles): Q^T (5 columns of 9), r_kk, |v_k|^2, the null-space basis X Y Z W (4 x 9), E E^T (9 quadratics),
// the 10x20 matrix column-major (lane j owns column j) and row-major unreduced (A0, for the polish), B(z) (9 x 5 coefficients),
// n(z) and its derivatives (11 x 11), the roots, and per root its best quality and model
constexpr int kLdA = 11;
constexpr int o5Qt = 0, o5Al = o5Qt + 45, o5Vt = o5Al + 5, o5Bas = o5Vt + 5, o5S = o5Bas + 36, o5A = o5S + 90, o5A0 = o5A + 20 * kLdA,
              o5Bp = o5A0 + 200, o5D = o5Bp + 45, o5Rt = o5D + 121, o5Q = o5Rt + 10, o5M = o5Q + 10, kSolveArea5 = o5M + 120;

// products of polynomials linear in (x, y, z): (quadratic or linear term i) x (linear term j) lands in out[at(i, j)]; the
// oracle's rel5_qidx / rel5_cidx packed into compile-time constants (4 and 5 bits per entry)
struct QIdx {
  static constexpr unsigned long long kQ = 0x9863875265413210ull;
  __device__ static constexpr int at(int i, int j) { return (int)((kQ >> (4 * (4 * i + j))) & 15); }
};
struct CIdx {
  static constexpr unsigned long long kC0 = 0x18b5250329040ull, kC1 = 0x1ee69cc14a062ull, kC2 = 0x251839a65a904ull, kC3 = 0x2728bdc762d25ull;
  __device__ static constexpr int at(int i, int j) { return (int)(((j == 0 ? kC0 : j == 1 ? kC1 : j == 2 ? kC2 : kC3) >> (5 * i)) & 31); }
};
// minors of a 3x3 (row-major index): M_c = m[a] m[b] - m[c'] m[d']
__device__ __constant__ int c_minor[3][4] = {{4, 8, 5, 7}, {5, 6, 3, 8}, {3, 7, 4, 6}};
// exponents of x, y, z of the cubic terms in Nistér's order, 2 bits per term (oracle: rel5_exp)
constexpr unsigned long long kExpX = 0x1550a63ull, kExpY = 0x5405a09cull, kExpZ = 0x1b18611100ull;
__device__ __forceinline__ constexpr int expo(unsigned long long packed, int i) { return (int)((packed >> (2 * i)) & 3); }

// out += p * l (p: NP terms, l: linear), term i outer, j inner
template <int NP, class Idx>
__device__ __forceinline__ void pmul(const double* p, const double* l, double* out) {
#pragma unroll
  for (int i = 0; i < NP; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) out[Idx::at(i, j)] = add(out[Idx::at(i, j)], mul(p[i], l[j]));
}
// out (ascending powers) += a * b, i outer, j inner
template <int NA, int NB>
__device__ __forceinline__ void upmul(const double* a, const double* b, double* out) {
#pragma unroll
  for (int i = 0; i < NA; i++)
#pragma unroll
    for (int j = 0; j < NB; j++) out[i + j] = add(out[i + j], mul(a[i], b[j]));
}
__device__ __forceinline__ double horner(const double* c, int d, double x) {
  double v = c[d];
  for (int i = d - 1; i >= 0; i--) v = add(mul(v, x), c[i]);
  return v;
}
__device__ __forceinline__ int sgn(double v) { return (v > 0.0) - (v < 0.0); }

// at most kPolish Gauss-Newton steps on the ten cubics A0 m(x, y, z) = 0 (A0 row-major) from v = (x, y, z); the first step that
// does not lower |F|^2 is undone and ends the polish.  The monomials are recomputed per row (the same expressions as the oracle's
// table, so the same values).
__device__ void polish(const double* A0, double* v) {
  double prev[3] = {v[0], v[1], v[2]}, rprev = INFINITY;
  for (int it = 0; it <= kPolish; it++) {
    double pw[3][4];
#pragma unroll
    for (int a = 0; a < 3; a++) {
      pw[a][0] = 1.0;
#pragma unroll
      for (int e = 1; e < 4; e++) pw[a][e] = mul(pw[a][e - 1], v[a]);
    }
    double N[9], g[3], Ni[9], res = 0.0;
    for (int r = 0; r < 10; r++) {
      const double* row = A0 + 20 * r;
      double F[4];
#pragma unroll
      for (int i = 0; i < 20; i++) {
        const int e0 = expo(kExpX, i), e1 = expo(kExpY, i), e2 = expo(kExpZ, i);
        const double m = mul(mul(pw[0][e0], pw[1][e1]), pw[2][e2]);
        const double dx = e0 ? mul(mul(mul((double)e0, pw[0][e0 ? e0 - 1 : 0]), pw[1][e1]), pw[2][e2]) : 0.0;
        const double dy = e1 ? mul(mul(mul((double)e1, pw[0][e0]), pw[1][e1 ? e1 - 1 : 0]), pw[2][e2]) : 0.0;
        const double dz = e2 ? mul(mul(mul((double)e2, pw[0][e0]), pw[1][e1]), pw[2][e2 ? e2 - 1 : 0]) : 0.0;
        const double ai = row[i];
        F[0] = i == 0 ? mul(ai, m) : add(F[0], mul(ai, m));
        F[1] = i == 0 ? mul(ai, dx) : add(F[1], mul(ai, dx));
        F[2] = i == 0 ? mul(ai, dy) : add(F[2], mul(ai, dy));
        F[3] = i == 0 ? mul(ai, dz) : add(F[3], mul(ai, dz));
      }
      res = r == 0 ? mul(F[0], F[0]) : add(res, mul(F[0], F[0]));
#pragma unroll
      for (int a = 0; a < 3; a++) {
#pragma unroll
        for (int b = 0; b < 3; b++) N[3 * a + b] = r == 0 ? mul(F[1 + a], F[1 + b]) : add(N[3 * a + b], mul(F[1 + a], F[1 + b]));
        g[a] = r == 0 ? mul(F[1 + a], F[0]) : add(g[a], mul(F[1 + a], F[0]));
      }
    }
    if (!(res < rprev)) { v[0] = prev[0]; v[1] = prev[1]; v[2] = prev[2]; break; }
    if (it == kPolish) break;
    prev[0] = v[0]; prev[1] = v[1]; prev[2] = v[2];
    rprev = res;
    inv3(N, Ni);
#pragma unroll
    for (int a = 0; a < 3; a++) v[a] = sub(v[a], dot3(Ni[3 * a], Ni[3 * a + 1], Ni[3 * a + 2], g));
  }
}

// the hypothesis of sample s (5 problem-local indices) of a central problem, solved by one warp in its area W; lane 0 writes the
// model.  Returns the (warp-uniform) valid flag.
__device__ bool rel5(const int* s, int n, const double* F1, const double* F2, double* W, double* model, int lane) {
  if (n < kSample5) return false;
  bool ok = true;
  if (lane < kSample5) {
    const int idx = s[lane];
    for (int j = 0; j < kSample5; j++) ok &= j == lane || s[j] != idx;
    ok &= finite3(F1 + 3 * (size_t)idx) && finite3(F2 + 3 * (size_t)idx);
  }
  if (!__all_sync(kFull, ok)) return false;
  double *Qt = W + o5Qt, *al = W + o5Al, *vt = W + o5Vt, *bas = W + o5Bas, *S = W + o5S, *A = W + o5A, *A0 = W + o5A0, *Bp = W + o5Bp,
         *Dp = W + o5D, *rt = W + o5Rt, *qual = W + o5Q, *rm = W + o5M;
  // 1. null space: Householder QR of Q^T (column i = vec(f1_i f2_i^T)), as rel17's
  if (lane < kSample5) {
    const double *a = F1 + 3 * (size_t)s[lane], *b = F2 + 3 * (size_t)s[lane];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) Qt[9 * lane + 3 * r + c] = mul(a[r], b[c]);
  }
  __syncwarp();
  if (!warp_householder<9, kSample5, 9>(Qt, al, vt, lane)) return false;
  if (lane < 4) {   // basis vector `lane` = H_0 ... H_4 e_{5+lane}
    double x[9];
#pragma unroll
    for (int i = 0; i < 9; i++) x[i] = i == kSample5 + lane ? 1.0 : 0.0;
#pragma unroll
    for (int k = kSample5 - 1; k >= 0; k--) {
      const double* v = Qt + 9 * k;
      double dot = 0.0;
#pragma unroll
      for (int i = k; i < 9; i++) dot = i == k ? mul(v[i], x[i]) : add(dot, mul(v[i], x[i]));
      const double c = __ddiv_rn(mul(2.0, dot), vt[k]);
#pragma unroll
      for (int i = k; i < 9; i++) x[i] = sub(x[i], mul(c, v[i]));
    }
    for (int i = 0; i < 9; i++) bas[9 * lane + i] = x[i];
  }
  __syncwarp();
  // 2. the 10x20 matrix; E_i = (X_i, Y_i, Z_i, W_i)
  auto Ei = [&](int i, double* e) { for (int j = 0; j < 4; j++) e[j] = bas[9 * j + i]; };
  if (lane < 9) {   // S_rk = sum_m E_rm E_km, (r, k) = lane
    const int r = lane / 3, k = lane % 3;
    double q[10];
    for (int i = 0; i < 10; i++) q[i] = 0.0;
    for (int m = 0; m < 3; m++) {
      double ea[4], eb[4];
      Ei(3 * r + m, ea); Ei(3 * k + m, eb);
      pmul<4, QIdx>(ea, eb, q);
    }
    for (int i = 0; i < 10; i++) S[10 * lane + i] = q[i];
  }
  __syncwarp();
  if (lane < 10) {
    double row[20], e[4];
#pragma unroll
    for (int m = 0; m < 20; m++) row[m] = 0.0;
    if (lane < 9) {   // entry (r, c) of 2 E E^T E - tr(E E^T) E
      const int r = lane / 3, c = lane % 3;
      double T[20], tr[10];
#pragma unroll
      for (int m = 0; m < 20; m++) T[m] = 0.0;
      for (int k = 0; k < 3; k++) {
        Ei(3 * k + c, e);
        pmul<10, CIdx>(S + 10 * (3 * r + k), e, row);
      }
#pragma unroll
      for (int i = 0; i < 10; i++) tr[i] = add(add(S[i], S[40 + i]), S[80 + i]);
      Ei(3 * r + c, e);
      pmul<10, CIdx>(tr, e, T);
#pragma unroll
      for (int m = 0; m < 20; m++) row[m] = sub(mul(2.0, row[m]), T[m]);
    } else {          // det E by cofactors along row 0
      for (int c = 0; c < 3; c++) {
        double p[10], q[10], Mc[10], ea[4], eb[4];
#pragma unroll
        for (int i = 0; i < 10; i++) { p[i] = 0.0; q[i] = 0.0; }
        Ei(c_minor[c][0], ea); Ei(c_minor[c][1], eb); pmul<4, QIdx>(ea, eb, p);
        Ei(c_minor[c][2], ea); Ei(c_minor[c][3], eb); pmul<4, QIdx>(ea, eb, q);
#pragma unroll
        for (int i = 0; i < 10; i++) Mc[i] = sub(p[i], q[i]);
        Ei(c, e);
        pmul<10, CIdx>(Mc, e, row);
      }
    }
#pragma unroll
    for (int m = 0; m < 20; m++) { A[kLdA * m + lane] = row[m]; A0[20 * lane + m] = row[m]; }
  }
  __syncwarp();
  // 3. Gauss-Jordan on the left 10x10 block; lane j owns column j
  double amax = 0.0;
  if (lane < 20)
    for (int i = 0; i < 10; i++) amax = fabs(A[kLdA * lane + i]) > amax ? fabs(A[kLdA * lane + i]) : amax;
  for (int o = 16; o > 0; o >>= 1) {
    const double other = __shfl_xor_sync(kFull, amax, o);
    amax = other > amax ? other : amax;
  }
  const double tol = mul(kPivotTol, amax);
  for (int k = 0; k < 10; k++) {
    const double* ck = A + kLdA * k;
    int p = k;
    for (int i = k + 1; i < 10; i++)
      if (fabs(ck[i]) > fabs(ck[p])) p = i;
    const double piv = ck[p];
    if (!(fabs(piv) >= tol) || !(amax > 0.0)) return false;   // warp-uniform: every lane reads the same column
    double f[10];
#pragma unroll
    for (int i = 0; i < 10; i++) f[i] = ck[i == k ? p : (i == p ? k : i)];
    __syncwarp();
    if (lane < 20) {
      double* cj = A + kLdA * lane;
      const double t = cj[k];
      cj[k] = cj[p]; cj[p] = t;
      const double akj = __ddiv_rn(cj[k], piv);
      cj[k] = akj;
#pragma unroll
      for (int i = 0; i < 10; i++)
        if (i != k) cj[i] = sub(cj[i], mul(f[i], akj));
    }
    __syncwarp();
  }
  // B(z) rows <e> - z<f>, <g> - z<h>, <i> - z<j>; n(z) = det B(z); its derivatives; the Cauchy bound
  double bnd = 0.0;
  if (lane == 0) {
    for (int r = 0; r < 3; r++) {
      const int ge = 4 + 2 * r, gf = 5 + 2 * r;
      auto g = [&](int m) { return A[kLdA * (10 + m) + ge]; };
      auto h = [&](int m) { return A[kLdA * (10 + m) + gf]; };
      for (int c = 0; c < 2; c++) {
        const int o = 3 * c;
        double* b = Bp + 5 * (3 * r + c);
        b[0] = g(o + 2); b[1] = sub(g(o + 1), h(o + 2)); b[2] = sub(g(o), h(o + 1)); b[3] = -h(o); b[4] = 0.0;
      }
      double* b = Bp + 5 * (3 * r + 2);
      b[0] = g(9); b[1] = sub(g(8), h(9)); b[2] = sub(g(7), h(8)); b[3] = sub(g(6), h(7)); b[4] = -h(6);
    }
    double nz[13];
#pragma unroll
    for (int i = 0; i < 13; i++) nz[i] = 0.0;
    for (int c = 0; c < 3; c++) {
      double p[9], q[9], Mc[9];
#pragma unroll
      for (int i = 0; i < 9; i++) { p[i] = 0.0; q[i] = 0.0; }
      upmul<5, 5>(Bp + 5 * c_minor[c][0], Bp + 5 * c_minor[c][1], p);
      upmul<5, 5>(Bp + 5 * c_minor[c][2], Bp + 5 * c_minor[c][3], q);
#pragma unroll
      for (int i = 0; i < 9; i++) Mc[i] = sub(p[i], q[i]);
      upmul<5, 9>(Bp + 5 * c, Mc, nz);
    }
    for (int i = 0; i <= 10; i++) Dp[110 + i] = nz[i];
    for (int d = 10; d >= 1; d--)
      for (int i = 0; i < d; i++) Dp[11 * (d - 1) + i] = mul(Dp[11 * d + i + 1], (double)(i + 1));
    double bmax = 0.0;
    for (int i = 0; i < 10; i++) {
      const double q = fabs(__ddiv_rn(nz[i], nz[10]));
      bmax = q > bmax ? q : bmax;
    }
    bnd = add(1.0, bmax);
  }
  bnd = __shfl_sync(kFull, bnd, 0);
  if (!(bnd < INFINITY)) return false;
  __syncwarp();
  // real roots: the roots of n^(d) for d = 9, ..., 0 in turn, lane k brackets interval k between the previous level's roots
  int nr = 0;
  for (int d = 1; d <= 10; d++) {
    const double *c = Dp + 11 * d, *dc = Dp + 11 * (d - 1);
    bool found = false;
    double z = 0.0;
    if (lane <= nr) {
      double a = lane == 0 ? -bnd : rt[lane - 1], b = lane == nr ? bnd : rt[lane];
      const int sa = sgn(horner(c, d, a)), sb = sgn(horner(c, d, b));
      found = sa != 0 && sb != sa;
      if (found) {
        for (int it = 0; it < kBisect; it++) {
          const double m = add(mul(0.5, a), mul(0.5, b));
          if (sgn(horner(c, d, m)) == sa) a = m; else b = m;
        }
        z = add(mul(0.5, a), mul(0.5, b));
        for (int it = 0; it < kNewton; it++) {
          const double zn = sub(z, __ddiv_rn(horner(c, d, z), horner(dc, d - 1, z)));
          if (zn >= a && zn <= b) z = zn;
        }
      }
    }
    const unsigned fm = __ballot_sync(kFull, found);
    __syncwarp();
    if (found) rt[__popc(fm & ((1u << lane) - 1))] = z;
    nr = __popc(fm);
    __syncwarp();
  }
  // 4-5. lane k < nr: root k's E, its four decompositions and the best of their qualities
  if (lane < nr) {
    double Bz[9], v[3], xyz[3];
    for (int i = 0; i < 9; i++) Bz[i] = horner(Bp + 5 * i, 4, rt[lane]);
    cross_max(Bz, Bz + 3, Bz + 6, v);
    xyz[0] = __ddiv_rn(v[0], v[2]); xyz[1] = __ddiv_rn(v[1], v[2]); xyz[2] = rt[lane];
    polish(A0, xyz);
    double E[9];
    for (int i = 0; i < 9; i++) E[i] = add(add(add(mul(xyz[0], bas[i]), mul(xyz[1], bas[9 + i])), mul(xyz[2], bas[18 + i])), bas[27 + i]);
    double fro = 0.0;
    for (int i = 0; i < 9; i++) fro = i == 0 ? mul(E[i], E[i]) : add(fro, mul(E[i], E[i]));
    const double sc = __dsqrt_rn(mul(0.5, fro));
    for (int i = 0; i < 9; i++) E[i] = __ddiv_rn(E[i], sc);
    double col[3][3], b[3], cof[9], bx[9];
    for (int j = 0; j < 3; j++)
      for (int i = 0; i < 3; i++) col[j][i] = E[3 * i + j];
    const double bn = __dsqrt_rn(cross_max(col[0], col[1], col[2], b));
    for (int i = 0; i < 3; i++) b[i] = __ddiv_rn(b[i], bn);
    cross3(E + 3, E + 6, cof); cross3(E + 6, E, cof + 3); cross3(E, E + 3, cof + 6);
    for (int j = 0; j < 3; j++) {
      double u[3];
      cross3(b, col[j], u);
      for (int i = 0; i < 3; i++) bx[3 * i + j] = u[i];
    }
    double best = INFINITY;
    for (int c = 0; c < 4; c++) {
      double M[12];
      for (int r = 0; r < 3; r++) {
        for (int j = 0; j < 3; j++) M[4 * r + j] = c < 2 ? sub(cof[3 * r + j], bx[3 * r + j]) : add(cof[3 * r + j], bx[3 * r + j]);
        M[4 * r + 3] = c & 1 ? -b[r] : b[r];
      }
      double q = 0.0;
      for (int i = 0; i < kSample5; i++) {
        const double *pa = F1 + 3 * (size_t)s[i], *pb = F2 + 3 * (size_t)s[i];
        const double a3[3] = {pa[0], pa[1], pa[2]}, b3[3] = {pb[0], pb[1], pb[2]};
        double X[3], r2[3], Xn[3], rn[3];
        rel_triangulate(M, a3, b3, X, r2);
        const double n1 = __dsqrt_rn(add(add(mul(X[0], X[0]), mul(X[1], X[1])), mul(X[2], X[2])));
        const double n2 = __dsqrt_rn(add(add(mul(r2[0], r2[0]), mul(r2[1], r2[1])), mul(r2[2], r2[2])));
        for (int r = 0; r < 3; r++) { Xn[r] = __ddiv_rn(X[r], n1); rn[r] = __ddiv_rn(r2[r], n2); }
        const double term = add(sub(1.0, dot3(a3[0], a3[1], a3[2], Xn)), sub(1.0, dot3(b3[0], b3[1], b3[2], rn)));
        q = i == 0 ? term : add(q, term);
      }
      if (isfinite(q) && q < best) {
        best = q;
        for (int i = 0; i < 12; i++) rm[12 * lane + i] = M[i];
      }
    }
    qual[lane] = best;
  }
  __syncwarp();
  int good = 0;
  if (lane == 0) {   // the strictly lowest finite quality, roots in ascending order
    double best = INFINITY;
    int k = -1;
    for (int r = 0; r < nr; r++)
      if (qual[r] < best) { best = qual[r]; k = r; }
    good = k >= 0;
    if (good) {
      for (int i = 0; i < 12; i++) model[i] = rm[12 * k + i];
      for (int i = 0; i < 12; i++) good &= isfinite(model[i]);
    }
  }
  return __shfl_sync(kFull, good, 0);
}

// one problem's view of the inputs for the per-sample solvers
struct ProbView {
  int n;
  const double *F1, *F2;
  const int *C1, *C2;
  const double *rig1, *rig2;
  bool rigs_finite;
};

// the per-sample solvers the kernel is instantiated with: sample size, per-warp area and whether the problem is central (one
// identity camera per side: no camera arrays, and pair_model with Rc = I, c = 0 reproduces the model bit for bit)
struct Solver17 {
  static constexpr int kSample = 17, kArea = kSolveArea;
  static constexpr bool kCentral = false;
  __device__ static bool solve(const int* s, const ProbView& P, double* W, double* model, int lane) {
    return rel17(s, P.n, P.F1, P.F2, P.C1, P.C2, P.rig1, P.rig2, P.rigs_finite, W, model, lane);
  }
};
struct Solver5 {
  static constexpr int kSample = kSample5, kArea = kSolveArea5;
  static constexpr bool kCentral = true;
  __device__ static bool solve(const int* s, const ProbView& P, double* W, double* model, int lane) {
    return rel5(s, P.n, P.F1, P.F2, W, model, lane);
  }
};

struct RelDev {
  const int* prob_ptr; const double* f1; const double* f2; const double* s1; const double* s2; const int* cam1; const int* cam2;
  const int* cam_ptr1; const int* cam_ptr2; const double* rig1; const double* rig2;   // rigs: [cam][12] offset then Rc
  const int* samples;
  int area;   // doubles per warp in dynamic shared memory
  RansacOut o;
};

// the camera-pair models of M for every pair (j1, j2) at P[12 (j1 nc2 + j2)], formed by the lanes of one warp
__device__ __forceinline__ void warp_pair_models(const double* M, const double* rig1, int nc1, const double* rig2, int nc2, double* P, int lane) {
  for (int p = lane; p < nc1 * nc2; p += 32) pair_model(M, rig1 + 12 * (p / nc2), rig2 + 12 * (p % nc2), P + kPairArea * p);
  __syncwarp();
}

// problem blockIdx.x for ransac_cta: its inputs, the rigs in shared memory and the warp's area W, which holds the solver's arrays
// while a sample is solved and the camera-pair models of the hypothesis being scored
template <class Sv>
struct RelProblem {
  ProbView P;
  const double *S1, *S2;
  int nc1, nc2;
  double* W;
  int warp, lane;
  // each warp solves one sample at a time
  template <class Src>
  __device__ void solve_wave(const Src& src, int base, double (*w_model)[12], int* w_valid) const {
    for (int h = warp; h < kWave; h += kWarps) {
      const int s = base + h;
      bool v = false;
      if (src.has(s)) v = Sv::solve(src.sample(s), P, W, w_model[h], lane);
      __syncwarp();
      if (lane == 0) {
        if (!v)
          for (int i = 0; i < 12; i++) w_model[h][i] = 0.0;
        w_valid[h] = v;
      }
    }
  }
  // the score of correspondence i under M (called by every lane of the warp)
  __device__ auto scorer(const double* M) const {
    warp_pair_models(M, P.rig1, nc1, P.rig2, nc2, W, lane);
    return [this](int i) { return rel_score(W + kPairArea * (Sv::kCentral ? 0 : P.C1[i] * nc2 + P.C2[i]), P.F1, P.F2, S1, S2, i); };
  }
};

// Sv: Solver17 (non-central, rigs and camera indices from D) or Solver5 (central: one identity camera per side); Src:
// SuppliedSamples<Sv::kSample> or SeededSamples<Sv::kSample>
template <class Sv, class Src>
__global__ void __launch_bounds__(kThreads) ransac_rel_kernel(RelDev D) {
  extern __shared__ double dyn[];
  const int pi = blockIdx.x, tid = threadIdx.x;
  const int off = D.prob_ptr[pi], n = D.prob_ptr[pi + 1] - off;
  const int nc1 = Sv::kCentral ? 1 : D.cam_ptr1[pi + 1] - D.cam_ptr1[pi], nc2 = Sv::kCentral ? 1 : D.cam_ptr2[pi + 1] - D.cam_ptr2[pi];
  __shared__ double rig1[kMaxCams * 12], rig2[kMaxCams * 12];
  __shared__ int rigs_finite;
  if (Sv::kCentral) {   // camera: offset 0, rotation I
    for (int i = tid; i < 12; i += kThreads) rig1[i] = rig2[i] = i == 3 || i == 7 || i == 11 ? 1.0 : 0.0;
  } else {
    for (int i = tid; i < 12 * nc1; i += kThreads) rig1[i] = D.rig1[12 * (size_t)D.cam_ptr1[pi] + i];
    for (int i = tid; i < 12 * nc2; i += kThreads) rig2[i] = D.rig2[12 * (size_t)D.cam_ptr2[pi] + i];
  }
  __syncthreads();
  if (tid == 0) {
    int fin = 1;
    for (int i = 0; i < 12 * nc1; i++) fin &= isfinite(rig1[i]);
    for (int i = 0; i < 12 * nc2; i++) fin &= isfinite(rig2[i]);
    rigs_finite = fin;
  }
  __syncthreads();
  RelProblem<Sv> Pb{ProbView{n, D.f1 + 3 * (size_t)off, D.f2 + 3 * (size_t)off, Sv::kCentral ? nullptr : D.cam1 + off,
                             Sv::kCentral ? nullptr : D.cam2 + off, rig1, rig2, rigs_finite != 0},
                    D.s1 + off, D.s2 + off, nc1, nc2, dyn + (size_t)(tid >> 5) * D.area, tid >> 5, tid & 31};
  ransac_cta<Sv::kSample>(D.o, Pb, sample_source<Src>(D.o, D.samples + Sv::kSample * (size_t)pi * D.o.n_samples, pi, n), off, n);
}

// staging offsets of the inputs (camera arrays unused by a central problem)
// the argument checks of a non-central problem batch (n_prob > 0) shared by the RANSAC and the covariance calls, up to the
// samples; with_sigma: sigma1 / sigma2 are read; with_samples: the samples are (the sample-supplied calls).  Sets *max_pairs to the largest rig1 x rig2 camera-pair count.
int check_rel_problems(cvb_ctx* ctx, const char* name, const cvb_rel_ransac_problems* p, bool with_sigma, bool with_samples, int* max_pairs) {
  const int n_prob = p->n_prob;
  CVB_REQUIRE(ctx, ptr_ok(p->prob_ptr, n_prob), "%s: prob_ptr does not start at 0 or decreases", name);
  CVB_REQUIRE(ctx, ptr_ok(p->cam_ptr1, n_prob) && ptr_ok(p->cam_ptr2, n_prob), "%s: cam_ptr1 / cam_ptr2 does not start at 0 or decreases", name);
  *max_pairs = 0;
  for (int i = 0; i < n_prob; i++) {
    const int nc1 = p->cam_ptr1[i + 1] - p->cam_ptr1[i], nc2 = p->cam_ptr2[i + 1] - p->cam_ptr2[i];
    CVB_REQUIRE(ctx, nc1 <= kMaxCams && nc2 <= kMaxCams, "%s: problem %d has a rig of more than %d cameras", name, i, kMaxCams);
    *max_pairs = nc1 * nc2 > *max_pairs ? nc1 * nc2 : *max_pairs;
  }
  const size_t N = (size_t)p->prob_ptr[n_prob], NC1 = (size_t)p->cam_ptr1[n_prob], NC2 = (size_t)p->cam_ptr2[n_prob];
  CVB_REQUIRE(ctx, N == 0 || (p->f1 && p->f2 && (!with_sigma || (p->sigma1 && p->sigma2)) && p->cam1 && p->cam2), "%s: null correspondence arrays", name);
  CVB_REQUIRE(ctx, (NC1 == 0 || (p->cam_off1 && p->cam_rot1)) && (NC2 == 0 || (p->cam_off2 && p->cam_rot2)), "%s: null rig arrays", name);
  CVB_REQUIRE(ctx, !with_samples || p->n_samples == 0 || p->samples, "%s: null samples", name);
  for (int i = 0; i < n_prob; i++) {
    const int o = p->prob_ptr[i], n = p->prob_ptr[i + 1] - o;
    const int nc1 = p->cam_ptr1[i + 1] - p->cam_ptr1[i], nc2 = p->cam_ptr2[i + 1] - p->cam_ptr2[i];
    for (int j = o; j < o + n; j++)
      CVB_REQUIRE(ctx, p->cam1[j] >= 0 && p->cam1[j] < nc1 && p->cam2[j] >= 0 && p->cam2[j] < nc2,
                  "%s: correspondence %d of problem %d names camera (%d, %d) outside its rigs (%d, %d cameras)", name, j - o, i, p->cam1[j],
                  p->cam2[j], nc1, nc2);
  }
  return CVB_OK;
}

// the per-warp area (doubles) of ransac_rel_kernel<Sv, Src> for a batch whose largest camera-pair count is max_pairs; the
// kernel's dynamic shared-memory limit is raised to the largest possible area on first use per device
template <class Sv, class Src>
int rel_ransac_area(cvb_ctx* ctx, int max_pairs, int* area) {
  constexpr int kMaxPairs = Sv::kCentral ? 1 : kMaxCams * kMaxCams;
  constexpr int kMaxArea = Sv::kArea > kPairArea * kMaxPairs ? Sv::kArea : kPairArea * kMaxPairs;
  static cvb_once_per_device once;
  {
    std::lock_guard<std::mutex> once_lk(once.mtx);
    if (once.first(ctx->device)) {
      CVB_CUDA(ctx, cudaFuncSetAttribute(ransac_rel_kernel<Sv, Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kWarps * kMaxArea * sizeof(double))));
    }
  }
  *area = Sv::kArea > kPairArea * max_pairs ? Sv::kArea : kPairArea * max_pairs;
  return CVB_OK;
}

// ransac_rel_kernel<Sv, Src> on the inputs bound in B to D (max_pairs: the largest camera-pair count of a problem; a seeded
// call's drawn samples to drawn)
template <class Sv, class Src>
int run_rel_ransac(cvb_ctx* ctx, cvb_block& B, RelDev& D, int n_prob, int ns, size_t N, int max_pairs, double threshold, int max_iterations,
                   double probability, cvb_rel_ransac_result* r, int32_t* drawn = nullptr) {
  if (const int rc = rel_ransac_area<Sv, Src>(ctx, max_pairs, &D.area)) return rc;
  return run_ransac(ctx, B, ransac_rel_kernel<Sv, Src>, (size_t)kWarps * D.area * sizeof(double), D, n_prob, ns, N, threshold, max_iterations,
                    probability, r, drawn, Sv::kSample);
}

// ---- the sampling-based covariance of a 17-point model (cvb_noncentral_relative_pose_covariance_batch) ----
// Solve: a problem's samples are spread over ceil(n_samples / kCovPerCta) CTAs (one linear grid over all problems), each
// with both rigs and the reference model in shared memory and one warp per sample through rel17; lane 0 writes the sample's
// deviation and valid flag to a scratch array.  Reduce: one CTA per problem, thread (r, c) sums delta_r delta_c over the valid
// samples in sample order.
constexpr int kCovPerCta = 4;   // samples (and warps) per solve CTA, chosen by measurement (DESIGN §9, K11e)
constexpr int kCovReduceThreads = 64, kCovChunk = 256;

struct CovDev {
  const int* prob_ptr; const double* f1; const double* f2; const int* cam1; const int* cam2;
  const int* cam_ptr1; const int* cam_ptr2; const double* rig1; const double* rig2;   // rigs: [cam][12] offset then Rc
  const int* samples; const double* ref_model;
  int n_samples, ctas_per_prob;
  double* delta; uint8_t* valid;   // [n_prob][n_samples][6], [n_prob][n_samples]
  double* cov; int* n_valid;       // [n_prob][36], [n_prob]
};
// the seeded call's solve: the inlier mask [N], the seeds [n_prob] and the drawn samples (nullable) instead of samples
struct CovSeededDev : CovDev {
  const uint8_t* mask; const unsigned long long* seed; int* drawn;
};

// q = (x, y, z, w) of a rotation matrix m (row-major) in Eigen's branch for the largest diagonal entry i
template <int i>
__device__ __forceinline__ void quat_diag_branch(const double* m, double* q) {
  constexpr int j = (i + 1) % 3, k = (j + 1) % 3;
  double t = __dsqrt_rn(add(sub(sub(m[4 * i], m[4 * j]), m[4 * k]), 1.0));
  q[i] = mul(0.5, t);
  t = __ddiv_rn(0.5, t);
  q[3] = mul(sub(m[3 * k + j], m[3 * j + k]), t);
  q[j] = mul(add(m[3 * j + i], m[3 * i + j]), t);
  q[k] = mul(add(m[3 * k + i], m[3 * i + k]), t);
}

// delta = [2 vec(q); t_s - t_ref], q the quaternion of R_ref^T R_s (Eigen's matrix-to-quaternion branches), w >= 0
__device__ void rel_deviation(const double* ref, const double* M, double* d) {
  double m[9], q[4];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) m[3 * r + c] = add(add(mul(ref[r], M[c]), mul(ref[4 + r], M[4 + c])), mul(ref[8 + r], M[8 + c]));
  const double tr = add(add(m[0], m[4]), m[8]);
  if (tr > 0.0) {
    double t = __dsqrt_rn(add(tr, 1.0));
    q[3] = mul(0.5, t);
    t = __ddiv_rn(0.5, t);
    q[0] = mul(sub(m[7], m[5]), t); q[1] = mul(sub(m[2], m[6]), t); q[2] = mul(sub(m[3], m[1]), t);
  } else {
    const int i = m[8] > (m[4] > m[0] ? m[4] : m[0]) ? 2 : (m[4] > m[0] ? 1 : 0);
    if (i == 0) quat_diag_branch<0>(m, q);
    else if (i == 1) quat_diag_branch<1>(m, q);
    else quat_diag_branch<2>(m, q);
  }
  const double s = q[3] < 0.0 ? -2.0 : 2.0;
  for (int r = 0; r < 3; r++) {
    d[r] = mul(s, q[r]);
    d[3 + r] = sub(M[4 * r + 3], ref[4 * r + 3]);
  }
}

// Dev = CovSeededDev: the seeded form (cvb_noncentral_relative_pose_covariance_seeded_batch).  Its CTA counts the problem's
// inliers m in the mask; a problem with m < 17 is skipped like one without a reference model.  For sample s, lane 0 draws the
// ranks (stream 1, [0, m)), and the warp maps each rank j to the j-th inlier in ascending order with one ballot scan of the mask.
template <class Dev>
__global__ void __launch_bounds__(kThreads) rel_cov_solve_kernel(Dev D) {
  constexpr bool kSeeded = !std::is_same<Dev, CovDev>::value;
  extern __shared__ double dyn[];
  const int pi = blockIdx.x / D.ctas_per_prob, chunk = blockIdx.x % D.ctas_per_prob;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int off = D.prob_ptr[pi], n = D.prob_ptr[pi + 1] - off;
  const int nc1 = D.cam_ptr1[pi + 1] - D.cam_ptr1[pi], nc2 = D.cam_ptr2[pi + 1] - D.cam_ptr2[pi];
  __shared__ double rig1[kMaxCams * 12], rig2[kMaxCams * 12], ref[12], w_model[kWarps][12];
  __shared__ int rigs_finite, skip;
  for (int i = tid; i < 12 * nc1; i += blockDim.x) rig1[i] = D.rig1[12 * (size_t)D.cam_ptr1[pi] + i];
  for (int i = tid; i < 12 * nc2; i += blockDim.x) rig2[i] = D.rig2[12 * (size_t)D.cam_ptr2[pi] + i];
  if (tid < 12) ref[tid] = D.ref_model[12 * (size_t)pi + tid];
  [[maybe_unused]] __shared__ int n_inl, w_smp[kSeeded ? kWarps : 1][kSample];
  if constexpr (kSeeded) {
    if (tid == 0) n_inl = 0;
    __syncthreads();
    int c = 0;
    for (int i = tid; i < n; i += blockDim.x) c += D.mask[off + i] != 0;
    atomicAdd(&n_inl, c);   // integer: order-independent
  }
  __syncthreads();
  if (tid == 0) {
    int fin = 1, zero = 1;
    for (int i = 0; i < 12 * nc1; i++) fin &= isfinite(rig1[i]);
    for (int i = 0; i < 12 * nc2; i++) fin &= isfinite(rig2[i]);
    for (int i = 0; i < 12; i++) zero &= ref[i] == 0.0;
    rigs_finite = fin; skip = zero;
    if constexpr (kSeeded) skip |= n_inl < kSample;
  }
  __syncthreads();
  const ProbView P{n, D.f1 + 3 * (size_t)off, D.f2 + 3 * (size_t)off, D.cam1 + off, D.cam2 + off, rig1, rig2, rigs_finite != 0};
  double* W = dyn + (size_t)warp * kSolveArea;
  const int s_end = min((chunk + 1) * kCovPerCta, D.n_samples);
  for (int s = chunk * kCovPerCta + warp; s < s_end; s += nw) {
    const size_t g = (size_t)pi * D.n_samples + s;
    bool v;
    if constexpr (kSeeded) {
      if (!skip) {
        if (lane == 0) seeded_sample<kSample>(D.seed[pi], 1, (unsigned)n_inl, (unsigned long long)s, w_smp[warp]);
        __syncwarp();
        const int r = lane < kSample ? w_smp[warp][lane] : -1;
        int idx = -1;
        for (int b = 0, c = 0; b < n; b += 32) {   // c: inliers before correspondence b
          const unsigned bal = __ballot_sync(kFull, b + lane < n && D.mask[off + b + lane]);
          const int cnt = __popc(bal);
          if (r >= c && r < c + cnt) idx = b + (int)__fns(bal, 0, r - c + 1);
          c += cnt;
        }
        __syncwarp();
        if (lane < kSample) {
          w_smp[warp][lane] = idx;
          if (D.drawn) D.drawn[kSample * g + lane] = idx;
        }
        __syncwarp();
      }
      v = !skip && Solver17::solve(w_smp[warp], P, W, w_model[warp], lane);
    } else {
      v = !skip && Solver17::solve(D.samples + kSample * g, P, W, w_model[warp], lane);   // a skipped problem's samples are not read
    }
    __syncwarp();
    if (lane == 0) {
      double d[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      if (v) rel_deviation(ref, w_model[warp], d);
      for (int i = 0; i < 6; i++) D.delta[6 * g + i] = d[i];
      D.valid[g] = (uint8_t)v;
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kCovReduceThreads) rel_cov_reduce_kernel(CovDev D) {
  const int pi = blockIdx.x, tid = threadIdx.x, r = tid / 6, c = tid % 6;
  __shared__ double sd[kCovChunk * 6];
  __shared__ uint8_t sv[kCovChunk];
  double acc = 0.0;
  int nv = 0;
  for (int base = 0; base < D.n_samples; base += kCovChunk) {
    const int m = min(kCovChunk, D.n_samples - base);
    const size_t g0 = (size_t)pi * D.n_samples + base;
    for (int i = tid; i < 6 * m; i += kCovReduceThreads) sd[i] = D.delta[6 * g0 + i];
    for (int i = tid; i < m; i += kCovReduceThreads) sv[i] = D.valid[g0 + i];
    __syncthreads();
    if (tid < 36)
      for (int i = 0; i < m; i++)
        if (sv[i]) { acc = add(acc, mul(sd[6 * i + r], sd[6 * i + c])); nv++; }
    __syncthreads();
  }
  if (tid < 36) D.cov[36 * (size_t)pi + tid] = nv > 0 ? __ddiv_rn(acc, (double)nv) : 0.0;
  if (tid == 0) D.n_valid[pi] = nv;
}

// cvb_ransac_noncentral_relative_pose_batch (seeded = false) and cvb_ransac_noncentral_relative_pose_seeded_batch
int noncentral_ransac(cvb_ctx* ctx, const char* name, const cvb_rel_ransac_problems* p, bool seeded, const uint64_t* seed, double threshold,
                      int max_iterations, double probability, cvb_rel_ransac_result* r, int32_t* drawn) {
  if (const int rc = check_ransac(ctx, name, p, max_iterations, r, kSample, seeded, seed)) return rc;
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  CVB_REQUIRE(ctx, p->cam_ptr1 && p->cam_ptr2, "%s: null cam_ptr1 / cam_ptr2", name);
  int max_pairs = 0;
  if (const int rc = check_rel_problems(ctx, name, p, true, !seeded, &max_pairs)) return rc;
  const size_t N = (size_t)p->prob_ptr[n_prob], S_all = (size_t)n_prob * ns;
  const std::vector<double> rig1 = pack_cams(p->cam_off1, p->cam_rot1, p->cam_ptr1[n_prob]), rig2 = pack_cams(p->cam_off2, p->cam_rot2, p->cam_ptr2[n_prob]);
  cvb_block B(ctx, ctx->stream);
  RelDev D{};
  B.in(D.prob_ptr, p->prob_ptr, (size_t)n_prob + 1); B.in(D.f1, p->f1, N * 3); B.in(D.f2, p->f2, N * 3); B.in(D.s1, p->sigma1, N);
  B.in(D.s2, p->sigma2, N); B.in(D.cam1, p->cam1, N); B.in(D.cam2, p->cam2, N);
  B.in(D.cam_ptr1, p->cam_ptr1, (size_t)n_prob + 1); B.in(D.cam_ptr2, p->cam_ptr2, (size_t)n_prob + 1);
  if (seeded) B.in(D.o.seed, seed, n_prob);
  else B.in(D.samples, p->samples, S_all * kSample);
  B.in(D.rig1, rig1.data(), rig1.size()); B.in(D.rig2, rig2.data(), rig2.size());
  if (seeded)
    return run_rel_ransac<Solver17, SeededSamples<kSample>>(ctx, B, D, n_prob, ns, N, max_pairs, threshold, max_iterations, probability, r, drawn);
  return run_rel_ransac<Solver17, SuppliedSamples<kSample>>(ctx, B, D, n_prob, ns, N, max_pairs, threshold, max_iterations, probability, r);
}

// cvb_ransac_central_relative_pose_batch (seeded = false) and cvb_ransac_central_relative_pose_seeded_batch
int central_ransac(cvb_ctx* ctx, const char* name, const cvb_central_rel_ransac_problems* p, bool seeded, const uint64_t* seed, double threshold,
                   int max_iterations, double probability, cvb_rel_ransac_result* r, int32_t* drawn) {
  if (const int rc = check_ransac(ctx, name, p, max_iterations, r, kSample5, seeded, seed)) return rc;
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  const size_t N = (size_t)p->prob_ptr[n_prob];
  CVB_REQUIRE(ctx, N == 0 || (p->f1 && p->f2 && p->sigma1 && p->sigma2), "%s: null correspondence arrays", name);
  cvb_block B(ctx, ctx->stream);
  RelDev D{};
  B.in(D.prob_ptr, p->prob_ptr, (size_t)n_prob + 1); B.in(D.f1, p->f1, N * 3); B.in(D.f2, p->f2, N * 3); B.in(D.s1, p->sigma1, N);
  B.in(D.s2, p->sigma2, N);
  if (seeded) B.in(D.o.seed, seed, n_prob);
  else B.in(D.samples, p->samples, (size_t)n_prob * ns * kSample5);
  if (seeded)
    return run_rel_ransac<Solver5, SeededSamples<kSample5>>(ctx, B, D, n_prob, ns, N, 1, threshold, max_iterations, probability, r, drawn);
  return run_rel_ransac<Solver5, SuppliedSamples<kSample5>>(ctx, B, D, n_prob, ns, N, 1, threshold, max_iterations, probability, r);
}

}  // namespace

extern "C" int cvb_ransac_noncentral_relative_pose_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, double threshold, int max_iterations,
                                                         double probability, cvb_rel_ransac_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return noncentral_ransac(ctx, "ransac_noncentral_relative_pose", p, false, nullptr, threshold, max_iterations, probability, r, nullptr);
}

extern "C" int cvb_ransac_noncentral_relative_pose_seeded_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, const uint64_t* seed,
                                                                double threshold, int max_iterations, double probability, cvb_rel_ransac_result* r,
                                                                int32_t* drawn) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return noncentral_ransac(ctx, "ransac_noncentral_relative_pose_seeded", p, true, seed, threshold, max_iterations, probability, r, drawn);
}

extern "C" int cvb_ransac_central_relative_pose_batch(cvb_ctx* ctx, const cvb_central_rel_ransac_problems* p, double threshold, int max_iterations,
                                                      double probability, cvb_rel_ransac_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return central_ransac(ctx, "ransac_central_relative_pose", p, false, nullptr, threshold, max_iterations, probability, r, nullptr);
}

extern "C" int cvb_ransac_central_relative_pose_seeded_batch(cvb_ctx* ctx, const cvb_central_rel_ransac_problems* p, const uint64_t* seed,
                                                             double threshold, int max_iterations, double probability, cvb_rel_ransac_result* r,
                                                             int32_t* drawn) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return central_ransac(ctx, "ransac_central_relative_pose_seeded", p, true, seed, threshold, max_iterations, probability, r, drawn);
}

namespace {

// cvb_noncentral_relative_pose_covariance_batch (seeded = false) and cvb_noncentral_relative_pose_covariance_seeded_batch
int rel_cov(cvb_ctx* ctx, const char* name, const cvb_rel_ransac_problems* p, const double* ref_model, bool seeded, const uint8_t* inlier_mask,
            const uint64_t* seed, cvb_rel_cov_result* r, int32_t* drawn) {
  CVB_REQUIRE(ctx, p && r && p->n_prob >= 0 && p->n_samples >= 0, "%s: bad arguments", name);
  CVB_REQUIRE(ctx, !seeded || !p->samples, "%s: samples must be NULL (the samples are drawn from the seeds)", name);
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  CVB_REQUIRE(ctx, p->prob_ptr && p->cam_ptr1 && p->cam_ptr2 && ref_model && r->cov && r->n_valid, "%s: null required pointer", name);
  CVB_REQUIRE(ctx, !seeded || (inlier_mask && seed), "%s: null inlier_mask / seed", name);
  CVB_REQUIRE(ctx, (r->sample_delta != nullptr) == (r->sample_valid != nullptr), "%s: sample_delta / sample_valid are requested together", name);
  int max_pairs = 0;   // unused: the covariance does not score
  if (const int rc = check_rel_problems(ctx, name, p, false, !seeded, &max_pairs)) return rc;
  // the reference models: all zeros (skipped), or finite with a rotation R
  std::vector<uint8_t> skip(n_prob);
  for (int i = 0; i < n_prob; i++) {
    const double* M = ref_model + 12 * (size_t)i;
    bool zero = true, finite = true;
    for (int k = 0; k < 12; k++) { zero &= M[k] == 0.0; finite &= isfinite(M[k]) != 0; }
    skip[i] = zero;
    if (zero) continue;
    CVB_REQUIRE(ctx, finite, "%s: reference model of problem %d is not finite", name, i);
    double dev = 0.0;
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) {
        const double g = M[a] * M[b] + M[4 + a] * M[4 + b] + M[8 + a] * M[8 + b] - (a == b ? 1.0 : 0.0);
        dev = fabs(g) > dev ? fabs(g) : dev;
      }
    CVB_REQUIRE(ctx, dev <= 1e-6, "%s: R of the reference model of problem %d is not a rotation (max |R^T R - I| = %g)", name, i, dev);
  }
  if (!seeded)
    if (const int rc = check_samples(ctx, name, p->samples, p->prob_ptr, n_prob, ns, kSample, skip.data())) return rc;
  const size_t N = (size_t)p->prob_ptr[n_prob], S_all = (size_t)n_prob * ns;
  const int ctas_per_prob = (ns + kCovPerCta - 1) / kCovPerCta;
  const long long grid = (long long)n_prob * ctas_per_prob;
  CVB_REQUIRE(ctx, grid <= INT32_MAX, "%s: %lld solve CTAs exceed the grid limit", name, grid);
  const std::vector<double> rig1 = pack_cams(p->cam_off1, p->cam_rot1, p->cam_ptr1[n_prob]), rig2 = pack_cams(p->cam_off2, p->cam_rot2, p->cam_ptr2[n_prob]);
  cvb_block B(ctx, ctx->stream);
  CovSeededDev D{};   // the sample-supplied solve and the reduce take its CovDev part
  B.in(D.prob_ptr, p->prob_ptr, (size_t)n_prob + 1); B.in(D.f1, p->f1, N * 3); B.in(D.f2, p->f2, N * 3); B.in(D.cam1, p->cam1, N); B.in(D.cam2, p->cam2, N);
  B.in(D.cam_ptr1, p->cam_ptr1, (size_t)n_prob + 1); B.in(D.cam_ptr2, p->cam_ptr2, (size_t)n_prob + 1);
  if (seeded) {
    B.in(D.seed, seed, n_prob);
    B.in(D.mask, inlier_mask, N);
  } else {
    B.in(D.samples, p->samples, S_all * kSample);
  }
  B.in(D.rig1, rig1.data(), rig1.size()); B.in(D.rig2, rig2.data(), rig2.size()); B.in(D.ref_model, ref_model, (size_t)n_prob * 12);
  B.out(D.cov, r->cov, (size_t)n_prob * 36); B.out(D.n_valid, r->n_valid, n_prob); B.out(D.delta, r->sample_delta, S_all * 6);
  B.out(D.valid, r->sample_valid, S_all);
  if (drawn) B.out(D.drawn, drawn, S_all * kSample);
  if (const int rc = B.place()) return rc;
  if (const int rc = B.upload()) return rc;
  D.n_samples = ns; D.ctas_per_prob = ctas_per_prob;
  cudaStream_t st = ctx->stream;
  if (drawn) CVB_CUDA(ctx, cudaMemsetAsync(D.drawn, 0xff, S_all * kSample * 4, st));
  if (ns > 0) {
    constexpr int kSolveWarps = kCovPerCta < kWarps ? kCovPerCta : kWarps;
    const size_t smem = (size_t)kSolveWarps * kSolveArea * sizeof(double);
    if (seeded) rel_cov_solve_kernel<CovSeededDev><<<(unsigned)grid, 32 * kSolveWarps, smem, st>>>(D);
    else rel_cov_solve_kernel<CovDev><<<(unsigned)grid, 32 * kSolveWarps, smem, st>>>(static_cast<const CovDev&>(D));
    CVB_CHECK_LAUNCH(ctx);
  }
  rel_cov_reduce_kernel<<<n_prob, kCovReduceThreads, 0, st>>>(static_cast<const CovDev&>(D));
  CVB_CHECK_LAUNCH(ctx);
  return B.download();
}

}  // namespace

extern "C" int cvb_noncentral_relative_pose_covariance_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, const double* ref_model,
                                                             cvb_rel_cov_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return rel_cov(ctx, "noncentral_relative_pose_covariance", p, ref_model, false, nullptr, nullptr, r, nullptr);
}

extern "C" int cvb_noncentral_relative_pose_covariance_seeded_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, const double* ref_model,
                                                                    const uint8_t* inlier_mask, const uint64_t* seed, cvb_rel_cov_result* r,
                                                                    int32_t* drawn) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return rel_cov(ctx, "noncentral_relative_pose_covariance_seeded", p, ref_model, true, inlier_mask, seed, r, drawn);
}

// ---- the verification chain of cvb_verify_noncentral_relative_pose_seeded_batch on the device ----
// The matcher's pair-list scan (match_kernels.cu), verify_gather_kernel (matches -> 5-point problems), ransac_rel_kernel<Solver5>,
// verify_merge_kernel (5-point inliers -> 17-point problems), ransac_rel_kernel<Solver17>, rel_cov_solve_kernel / rel_cov_reduce_kernel
// and verify_list_kernel (the correspondence list), all on the arrays of one device block (cvb_block).  The correspondence arrays are sized
// by the host-known bound sum over pairings of rows(kf1); the problems are packed to the front in pairing (candidate) order.
// SIFT rows (CV_32F) to the u8 layout of the L2 scan in one pass; false if a value is not an integer in [0, 255] (NaN and
// +-inf included).  This is quantize_u8_kernel's test rintf(v) == v && 0 <= v <= 255 (checked equal on every float bit
// pattern), written without branches or conversions so that the loop vectorises and runs at copy speed: c = v + 1.5 * 2^23
// rounds v to an integer held in c's low mantissa bits (|v| < 2^22), and c - 1.5 * 2^23 == v holds exactly when v is one.
// Needs IEEE arithmetic (no -ffast-math).
bool cvb_quantize_sift(const float* src, size_t n, uint8_t* dst) {
  int bad = 0;
  for (size_t i = 0; i < n; i++) {
    const float v = src[i];
    const float c = v + 12582912.f;
    int32_t bits;
    memcpy(&bits, &c, 4);
    bad |= (c - 12582912.f != v) | (v < 0.f) | (v > 255.f);
    dst[i] = (uint8_t)(bits - 0x4B400000);   // the bits of 1.5 * 2^23
  }
  return bad == 0;
}

namespace {

struct VerifyDev {
  const double* bearings; const double* sigma;          // keyframe table [R][3], [R]
  const int* pair_rows;                                  // [P][5] the matcher's pair table: query row0, rows, train row0, rows, offset
  const int* pair_cams;                                  // [P][2]
  const int* pair_ptr;                                   // [C+1]
  const int* match_train; const int* n_matches;          // the matcher's outputs
  int* prob_ptr5; double *f1_5, *f2_5, *s1_5, *s2_5; int *row1, *row2;   // 5-point problems [P+1], [N5] ...
  const uint8_t* mask5; const int* count5;
  int* prob_ptr17; double *f1_17, *f2_17, *s1_17, *s2_17; int *cam1_17, *cam2_17;
  int* pos17;                                            // [N5] the 17-point correspondence of a 5-point inlier, -1 otherwise
  const uint8_t* mask17;
  int* corr; int corr_cap;                               // [corr_cap][5] (nullable)
};

// one CTA per pairing: its problem's offset (the matches of the pairings before it), prob_ptr5, and its matches in query order
__global__ void __launch_bounds__(kGlueThreads) verify_gather_kernel(VerifyDev V) {
  const int p = blockIdx.x;
  __shared__ int off;
  if (threadIdx.x == 0) {
    int o = 0;
    for (int q = 0; q < p; q++) o += V.n_matches[q];
    off = o;
    if (p == 0) V.prob_ptr5[0] = 0;
    V.prob_ptr5[p + 1] = o + V.n_matches[p];
  }
  __syncthreads();
  const int* pr = V.pair_rows + 5 * p;
  const int q0 = pr[0], t0 = pr[2], o = off;
  const int* mt = V.match_train + pr[4];
  scan_emit(pr[1], [&](int i) { return mt[i] >= 0; }, [&](int i, int r) {
    const int j = o + r, t = mt[i];
    const size_t a = (size_t)q0 + i, b = (size_t)t0 + t;
    for (int k = 0; k < 3; k++) { V.f1_5[3 * (size_t)j + k] = V.bearings[3 * a + k]; V.f2_5[3 * (size_t)j + k] = V.bearings[3 * b + k]; }
    V.s1_5[j] = V.sigma[a]; V.s2_5[j] = V.sigma[b]; V.row1[j] = i; V.row2[j] = t;
  });
}

// one CTA per candidate: its 17-point problem, the 5-point inliers of its pairings in order.  Its offset sums the 5-point
// best_count of the pairings before it: best_count is the number of set flags in the selected model's inlier mask (ransac_cta
// scores the same model with the same device function for both).
__global__ void __launch_bounds__(kGlueThreads) verify_merge_kernel(VerifyDev V) {
  const int c = blockIdx.x, pb = V.pair_ptr[c], pe = V.pair_ptr[c + 1];
  __shared__ int off;
  if (threadIdx.x == 0) {
    int o = 0, m = 0;
    for (int q = 0; q < pb; q++) o += V.count5[q];
    for (int q = pb; q < pe; q++) m += V.count5[q];
    off = o;
    if (c == 0) V.prob_ptr17[0] = 0;
    V.prob_ptr17[c + 1] = o + m;
  }
  __syncthreads();
  int j0 = off;
  for (int q = pb; q < pe; q++) {
    const int b5 = V.prob_ptr5[q], n5 = V.prob_ptr5[q + 1] - b5, c1 = V.pair_cams[2 * q], c2 = V.pair_cams[2 * q + 1];
    for (int i = threadIdx.x; i < n5; i += kGlueThreads) V.pos17[b5 + i] = -1;
    __syncthreads();
    j0 += scan_emit(n5, [&](int i) { return V.mask5[b5 + i] != 0; }, [&](int i, int r) {
      const size_t j = (size_t)j0 + r, a = (size_t)b5 + i;
      for (int k = 0; k < 3; k++) { V.f1_17[3 * j + k] = V.f1_5[3 * a + k]; V.f2_17[3 * j + k] = V.f2_5[3 * a + k]; }
      V.s1_17[j] = V.s1_5[a]; V.s2_17[j] = V.s2_5[a]; V.cam1_17[j] = c1; V.cam2_17[j] = c2;
      V.pos17[a] = (int)j;
    });
  }
}

// one CTA per pairing: its entries of the correspondence list (those below corr_cap)
__global__ void __launch_bounds__(kGlueThreads) verify_list_kernel(VerifyDev V) {
  const int p = blockIdx.x, b = V.prob_ptr5[p], e = min(V.prob_ptr5[p + 1], V.corr_cap);
  for (int j = b + threadIdx.x; j < e; j += kGlueThreads) {
    int* o = V.corr + 5 * (size_t)j;
    const int k = V.pos17[j];
    o[0] = p; o[1] = V.row1[j]; o[2] = V.row2[j]; o[3] = V.mask5[j]; o[4] = k >= 0 ? V.mask17[k] : 0;
  }
}


// cvb_verify_noncentral_relative_pose{,_sift}_seeded_batch: KF is cvb_verify_keyframes (ORB rows, staged as they are, matched by
// the Hamming pair scan) or cvb_verify_keyframes_sift (SIFT rows, checked and quantised to u8 while staged, matched by the L2 one)
template <class KF>
int verify_noncentral(cvb_ctx* ctx, const KF* kf, const cvb_verify_candidates* cd, const cvb_verify_params* prm, const uint64_t* seed5,
                      const uint64_t* seed, cvb_verify_result* r) {
  constexpr bool kSift = std::is_same<KF, cvb_verify_keyframes_sift>::value;
  const char* name = kSift ? "verify_noncentral_relative_pose_sift_seeded" : "verify_noncentral_relative_pose_seeded";
  constexpr int kMaxIt = (INT32_MAX - kWave) / 11;   // the seeded RANSAC's limit: every sample number fits an int
  CVB_REQUIRE(ctx, kf && cd && prm && r && kf->n_kf >= 0 && cd->n_cand >= 0, "%s: bad arguments", name);
  CVB_REQUIRE(ctx, prm->max_iterations5 >= 0 && prm->max_iterations5 <= kMaxIt && prm->max_iterations17 >= 0 && prm->max_iterations17 <= kMaxIt,
              "%s: max_iterations5 / max_iterations17 outside [0, %d]", name, kMaxIt);
  CVB_REQUIRE(ctx, prm->n_cov_samples >= 0 && r->corr_cap >= 0, "%s: negative n_cov_samples / corr_cap", name);
  const int n_kf = kf->n_kf, C = cd->n_cand;
  r->n_total = 0;
  if (C == 0) return CVB_OK;
  CVB_REQUIRE(ctx, kf->kf_ptr && cd->cam_ptr1 && cd->cam_ptr2 && cd->pair_ptr && seed, "%s: null required pointer", name);
  CVB_REQUIRE(ctx, r->n_matches && r->best_sample5 && r->best_model5 && r->best_count5 && r->iterations5 && r->consumed5 && r->best_sample &&
                   r->best_model && r->best_count && r->iterations && r->consumed && r->cov && r->n_valid, "%s: null result pointer", name);
  CVB_REQUIRE(ctx, ptr_ok(kf->kf_ptr, n_kf), "%s: kf_ptr does not start at 0 or decreases", name);
  CVB_REQUIRE(ctx, ptr_ok(cd->pair_ptr, C), "%s: pair_ptr does not start at 0 or decreases", name);
  CVB_REQUIRE(ctx, ptr_ok(cd->cam_ptr1, C) && ptr_ok(cd->cam_ptr2, C), "%s: cam_ptr1 / cam_ptr2 does not start at 0 or decreases", name);
  const size_t R = (size_t)kf->kf_ptr[n_kf];
  const int P = cd->pair_ptr[C];
  CVB_REQUIRE(ctx, R == 0 || (kf->desc && kf->bearings && kf->sigma), "%s: null keyframe arrays", name);
  CVB_REQUIRE(ctx, P == 0 || (cd->pairs && seed5), "%s: null pairs / seed5", name);
  const size_t NC1 = (size_t)cd->cam_ptr1[C], NC2 = (size_t)cd->cam_ptr2[C];
  CVB_REQUIRE(ctx, (NC1 == 0 || (cd->cam_off1 && cd->cam_rot1)) && (NC2 == 0 || (cd->cam_off2 && cd->cam_rot2)), "%s: null rig arrays", name);
  // the pair table of the matcher and the bound of the correspondence arrays
  std::vector<int32_t> rows((size_t)P * 5), cams((size_t)P * 2);
  size_t B = 0;
  int max_pairs = 0, max_nq = 0;
  for (int c = 0; c < C; c++) {
    const int nc1 = cd->cam_ptr1[c + 1] - cd->cam_ptr1[c], nc2 = cd->cam_ptr2[c + 1] - cd->cam_ptr2[c];
    CVB_REQUIRE(ctx, nc1 <= kMaxCams && nc2 <= kMaxCams, "%s: candidate %d has a rig of more than %d cameras", name, c, kMaxCams);
    max_pairs = nc1 * nc2 > max_pairs ? nc1 * nc2 : max_pairs;
    for (int q = cd->pair_ptr[c]; q < cd->pair_ptr[c + 1]; q++) {
      const int32_t* e = cd->pairs + 4 * (size_t)q;
      CVB_REQUIRE(ctx, e[0] >= 0 && e[0] < n_kf && e[1] >= 0 && e[1] < n_kf, "%s: pairing %d names keyframe (%d, %d) outside [0, %d)", name, q, e[0],
                  e[1], n_kf);
      CVB_REQUIRE(ctx, e[2] >= 0 && e[2] < nc1 && e[3] >= 0 && e[3] < nc2, "%s: pairing %d names camera (%d, %d) outside its rigs (%d, %d cameras)",
                  name, q, e[2], e[3], nc1, nc2);
      const int nq = kf->kf_ptr[e[0] + 1] - kf->kf_ptr[e[0]];
      int32_t* w = rows.data() + 5 * (size_t)q;
      w[0] = kf->kf_ptr[e[0]]; w[1] = nq; w[2] = kf->kf_ptr[e[1]]; w[3] = kf->kf_ptr[e[1] + 1] - kf->kf_ptr[e[1]]; w[4] = (int32_t)B;
      cams[2 * (size_t)q] = e[2]; cams[2 * (size_t)q + 1] = e[3];
      B += (size_t)nq;
      max_nq = nq > max_nq ? nq : max_nq;
    }
  }
  CVB_REQUIRE(ctx, B <= INT32_MAX, "%s: %zu query rows over the pairings exceed the int32 range", name, B);
  const int ns = prm->n_cov_samples, ctas_per_cand = (ns + kCovPerCta - 1) / kCovPerCta;
  CVB_REQUIRE(ctx, (long long)C * ctas_per_cand <= INT32_MAX, "%s: %lld covariance CTAs exceed the grid limit", name, (long long)C * ctas_per_cand);
  const size_t S_all = (size_t)C * ns, L = r->corr ? std::min(B, (size_t)r->corr_cap) : 0;
  std::vector<uint8_t> q8;   // the SIFT rows quantised; their check is an argument check, so it comes before the device block
  if constexpr (kSift) {
    q8.resize(R * 128);
    if (!cvb_quantize_sift(kf->desc, R * 128, q8.data()))
      return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "%s: SIFT descriptors must be integer-valued in [0,255] (cv::xfeatures2d::SIFT output)", name);
  }
  const std::vector<double> rig1 = pack_cams(cd->cam_off1, cd->cam_rot1, NC1), rig2 = pack_cams(cd->cam_off2, cd->cam_rot2, NC2);
  // device block: V, the 5-point RANSAC D5, the 17-point RANSAC D, the covariance Q
  cvb_block blk(ctx, ctx->stream);
  VerifyDev V{};
  RelDev D5{}, D{};
  CovSeededDev Q{};
  const uint8_t* d_desc;
  int *d_mt, *d_nm;
  float* d_md;
  blk.in(d_desc, kSift ? (const void*)q8.data() : (const void*)kf->desc, R * (kSift ? 128 : 32));
  blk.in(V.bearings, kf->bearings, R * 3); blk.in(V.sigma, kf->sigma, R);
  blk.in(V.pair_rows, rows.data(), (size_t)P * 5); blk.in(V.pair_cams, cams.data(), (size_t)P * 2); blk.in(V.pair_ptr, cd->pair_ptr, (size_t)C + 1);
  blk.in(D.cam_ptr1, cd->cam_ptr1, (size_t)C + 1); blk.in(D.cam_ptr2, cd->cam_ptr2, (size_t)C + 1);
  blk.in(D.rig1, rig1.data(), rig1.size()); blk.in(D.rig2, rig2.data(), rig2.size());
  blk.in(D5.o.seed, seed5, P); blk.in(D.o.seed, seed, C);
  blk.tmp(d_mt, B); blk.tmp(d_md, B);
  blk.tmp(V.f1_5, B * 3); blk.tmp(V.f2_5, B * 3); blk.tmp(V.s1_5, B); blk.tmp(V.s2_5, B);
  blk.tmp(V.row1, B); blk.tmp(V.row2, B); blk.tmp(D5.o.inlier_mask, B); blk.tmp(V.pos17, B);
  blk.tmp(V.f1_17, B * 3); blk.tmp(V.f2_17, B * 3); blk.tmp(V.s1_17, B); blk.tmp(V.s2_17, B);
  blk.tmp(V.cam1_17, B); blk.tmp(V.cam2_17, B); blk.tmp(D.o.inlier_mask, B); blk.tmp(V.prob_ptr17, (size_t)C + 1);
  blk.tmp(Q.delta, S_all * 6); blk.tmp(Q.valid, S_all);
  blk.out(d_nm, r->n_matches, P); blk.out_host(V.prob_ptr5, (size_t)P + 1);
  blk.out(D5.o.best_sample, r->best_sample5, P); blk.out(D5.o.best_model, r->best_model5, (size_t)P * 12); blk.out(D5.o.best_count, r->best_count5, P);
  blk.out(D5.o.iterations, r->iterations5, P); blk.out(D5.o.consumed, r->consumed5, P);
  blk.out(D.o.best_sample, r->best_sample, C); blk.out(D.o.best_model, r->best_model, (size_t)C * 12); blk.out(D.o.best_count, r->best_count, C);
  blk.out(D.o.iterations, r->iterations, C); blk.out(D.o.consumed, r->consumed, C);
  blk.out(Q.cov, r->cov, (size_t)C * 36); blk.out(Q.n_valid, r->n_valid, C); blk.out_host(V.corr, L * 5);
  if (const int rc = blk.place()) return rc;
  if (const int rc = blk.upload()) return rc;
  cudaStream_t st = ctx->stream;
  V.match_train = d_mt; V.n_matches = d_nm; V.mask5 = D5.o.inlier_mask; V.count5 = D5.o.best_count; V.mask17 = D.o.inlier_mask; V.corr_cap = (int)L;
  // 1. matches
  const auto match_pairs = kSift ? cvb_match_l2_pairs_dev : cvb_match_hamming_pairs_dev;
  if (const int rc = match_pairs(ctx, d_desc, V.pair_rows, P, max_nq, prm->img_match_thres, prm->ratio_thres, d_mt, d_md, d_nm)) return rc;
  if (P == 0) CVB_CUDA(ctx, cudaMemsetAsync(V.prob_ptr5, 0, 4, st));
  // 2. the 5-point problems and their RANSACs
  if (P > 0) {
    verify_gather_kernel<<<P, kGlueThreads, 0, st>>>(V);
    CVB_CHECK_LAUNCH(ctx);
    D5.prob_ptr = V.prob_ptr5; D5.f1 = V.f1_5; D5.f2 = V.f2_5; D5.s1 = V.s1_5; D5.s2 = V.s2_5;
    set_selection(D5.o, 0, prm->max_iterations5, prm->threshold5, prm->probability);
    if (const int rc = rel_ransac_area<Solver5, SeededSamples<kSample5>>(ctx, 1, &D5.area)) return rc;
    if (const int rc = launch_ransac(ctx, ransac_rel_kernel<Solver5, SeededSamples<kSample5>>, (size_t)kWarps * D5.area * sizeof(double), D5, P)) return rc;
  }
  // 3. the 17-point problems and their RANSACs
  verify_merge_kernel<<<C, kGlueThreads, 0, st>>>(V);
  CVB_CHECK_LAUNCH(ctx);
  D.prob_ptr = V.prob_ptr17; D.f1 = V.f1_17; D.f2 = V.f2_17; D.s1 = V.s1_17; D.s2 = V.s2_17; D.cam1 = V.cam1_17; D.cam2 = V.cam2_17;
  set_selection(D.o, 0, prm->max_iterations17, prm->threshold17, prm->probability);
  if (const int rc = rel_ransac_area<Solver17, SeededSamples<kSample>>(ctx, max_pairs, &D.area)) return rc;
  if (const int rc = launch_ransac(ctx, ransac_rel_kernel<Solver17, SeededSamples<kSample>>, (size_t)kWarps * D.area * sizeof(double), D, C)) return rc;
  // 4. the covariance from the 17-point inlier mask in place
  Q.prob_ptr = V.prob_ptr17; Q.f1 = V.f1_17; Q.f2 = V.f2_17; Q.cam1 = V.cam1_17; Q.cam2 = V.cam2_17;
  Q.cam_ptr1 = D.cam_ptr1; Q.cam_ptr2 = D.cam_ptr2; Q.rig1 = D.rig1; Q.rig2 = D.rig2; Q.ref_model = D.o.best_model;
  Q.n_samples = ns; Q.ctas_per_prob = ctas_per_cand;
  Q.mask = V.mask17; Q.seed = D.o.seed;
  if (ns > 0) {
    constexpr int kSolveWarps = kCovPerCta < kWarps ? kCovPerCta : kWarps;
    rel_cov_solve_kernel<CovSeededDev><<<(unsigned)(C * ctas_per_cand), 32 * kSolveWarps, (size_t)kSolveWarps * kSolveArea * sizeof(double), st>>>(Q);
    CVB_CHECK_LAUNCH(ctx);
  }
  rel_cov_reduce_kernel<<<C, kCovReduceThreads, 0, st>>>(static_cast<const CovDev&>(Q));
  CVB_CHECK_LAUNCH(ctx);
  // 5. the correspondence list
  if (L > 0) {
    verify_list_kernel<<<P, kGlueThreads, 0, st>>>(V);
    CVB_CHECK_LAUNCH(ctx);
  }
  if (const int rc = blk.download()) return rc;
  const int32_t n_total = blk.host(V.prob_ptr5)[P];
  r->n_total = n_total;
  if (r->corr && (size_t)n_total <= L) memcpy(r->corr, blk.host(V.corr), (size_t)n_total * 20);
  return CVB_OK;
}

}  // namespace

extern "C" int cvb_verify_noncentral_relative_pose_seeded_batch(cvb_ctx* ctx, const cvb_verify_keyframes* kf, const cvb_verify_candidates* cand,
                                                                const cvb_verify_params* prm, const uint64_t* seed5, const uint64_t* seed,
                                                                cvb_verify_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return verify_noncentral(ctx, kf, cand, prm, seed5, seed, r);
}

extern "C" int cvb_verify_noncentral_relative_pose_sift_seeded_batch(cvb_ctx* ctx, const cvb_verify_keyframes_sift* kf,
                                                                     const cvb_verify_candidates* cand, const cvb_verify_params* prm,
                                                                     const uint64_t* seed5, const uint64_t* seed, cvb_verify_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return verify_noncentral(ctx, kf, cand, prm, seed5, seed, r);
}
