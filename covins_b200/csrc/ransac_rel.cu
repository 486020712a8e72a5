// ransac_rel.cu — the non-central relative-pose RANSAC of RelNonCentralPosSolver::computeNonCentralRelPose (17-point,
// RelNonCentralPosSolver.cpp:146-173; the COVINS_G verification of a place-recognition candidate, each side a rig of a
// keyframe and its neighbours) on the GPU from caller-supplied samples: the 17-point solve per sample, scoring per camera pair
// and the sequential model selection of opengv's Ransac::computeModel, for a batch of problems (candidates) in one launch.
//
// The same kernel, instantiated with the 5-point solver (rel5), runs the central relative-pose RANSAC of
// RelNonCentralPosSolver::computePose (cvb_ransac_central_relative_pose_batch): a central problem is a non-central one with a
// single identity camera per side.
//
// One CTA per problem, both rigs staged in shared memory.  Samples are taken in waves of kWave: each warp solves one sample at
// a time (lane k owns column k of A^T in its warp's shared-memory area, every norm and dot product is a sequential sum inside
// one lane), then every warp scores the wave's hypotheses against all correspondences (camera-pair models in the warp's area,
// warp-shuffle integer counts), thread 0 replays the selection over the wave in sample order, and the CTA stops as soon as the
// adaptive bound ends the selection.  The CTA then writes the selected model's inlier mask.
//
// Only + - * / and sqrt as explicit non-fused intrinsics, fixed iteration counts: the results are bit-identical to the plain
// IEEE restatement compiled with -ffp-contract=off (oracle/ransac_rel_oracle.c for the 17-point solver,
// oracle/ransac_rel5_oracle.c for the 5-point one; their headers state the problems and their assumptions; so does
// include/covins_b200.h).
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
// the largest of the three cross products r0 x r1, r0 x r2, r1 x r2 (the first on ties) and its squared norm
__device__ __forceinline__ double cross_max(const double* r0, const double* r1, const double* r2, double* v) {
  double c[3][3];
  cross3(r0, r1, c[0]); cross3(r0, r2, c[1]); cross3(r1, r2, c[2]);
  double best = dot3(c[0][0], c[0][1], c[0][2], c[0]);
  v[0] = c[0][0]; v[1] = c[0][1]; v[2] = c[0][2];
#pragma unroll
  for (int j = 1; j < 3; j++) {
    const double nj = dot3(c[j][0], c[j][1], c[j][2], c[j]);
    if (nj > best) { best = nj; v[0] = c[j][0]; v[1] = c[j][1]; v[2] = c[j][2]; }
  }
  return best;
}

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
  for (int k = 0; k < kSample5; k++) {
    if (lane == k) {
      double* col = Qt + 9 * k;
      double ss = 0.0;
      for (int i = k; i < 9; i++) ss = i == k ? mul(col[i], col[i]) : add(ss, mul(col[i], col[i]));
      const double sigma = __dsqrt_rn(ss), ak = col[k];
      const double alpha = ak >= 0.0 ? -sigma : sigma;
      col[k] = sub(ak, alpha);
      al[k] = alpha;
      vt[k] = mul(2.0, add(ss, mul(fabs(ak), sigma)));
    }
    __syncwarp();
    if (lane > k && lane < kSample5) {
      const double* v = Qt + 9 * k;
      double* a = Qt + 9 * lane;
      double dot = 0.0;
      for (int i = k; i < 9; i++) dot = i == k ? mul(v[i], a[i]) : add(dot, mul(v[i], a[i]));
      const double c = __ddiv_rn(mul(2.0, dot), vt[k]);
      for (int i = k; i < 9; i++) a[i] = sub(a[i], mul(c, v[i]));
    }
    __syncwarp();
  }
  int good = 0;
  if (lane == 0) {
    double rmax = 0.0;
    for (int k = 0; k < kSample5; k++) rmax = fabs(al[k]) > rmax ? fabs(al[k]) : rmax;
    good = rmax > 0.0;
    for (int k = 0; k < kSample5; k++)
      if (!(fabs(al[k]) >= mul(kRankTol, rmax))) good = 0;
  }
  if (!__shfl_sync(kFull, good, 0)) return false;
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

// Sv: Solver17 (non-central, rigs and camera indices from D) or Solver5 (central: one identity camera per side)
template <class Sv>
__global__ void __launch_bounds__(kThreads) ransac_rel_kernel(RelDev D) {
  constexpr int kS = Sv::kSample;
  extern __shared__ double dyn[];
  const int pi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int off = D.prob_ptr[pi], n = D.prob_ptr[pi + 1] - off;
  const int nc1 = Sv::kCentral ? 1 : D.cam_ptr1[pi + 1] - D.cam_ptr1[pi], nc2 = Sv::kCentral ? 1 : D.cam_ptr2[pi + 1] - D.cam_ptr2[pi];
  const double* F1 = D.f1 + 3 * (size_t)off;
  const double* F2 = D.f2 + 3 * (size_t)off;
  const double* S1 = D.s1 + off;
  const double* S2 = D.s2 + off;
  const int* C1 = Sv::kCentral ? nullptr : D.cam1 + off;
  const int* C2 = Sv::kCentral ? nullptr : D.cam2 + off;
  double* W = dyn + (size_t)warp * D.area;
  const bool all = D.sample_model != nullptr;
  __shared__ double rig1[kMaxCams * 12], rig2[kMaxCams * 12];
  __shared__ double w_model[kWave][12];
  __shared__ int w_valid[kWave], w_count[kWave];
  __shared__ double best_model[12], k_bound;
  __shared__ int best, best_n, it, used, running, rigs_finite;
  __shared__ long long skipped;
  if (Sv::kCentral) {   // camera: offset 0, rotation I
    for (int i = tid; i < 12; i += kThreads) rig1[i] = rig2[i] = i == 3 || i == 7 || i == 11 ? 1.0 : 0.0;
  } else {
    for (int i = tid; i < 12 * nc1; i += kThreads) rig1[i] = D.rig1[12 * (size_t)D.cam_ptr1[pi] + i];
    for (int i = tid; i < 12 * nc2; i += kThreads) rig2[i] = D.rig2[12 * (size_t)D.cam_ptr2[pi] + i];
  }
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
  const ProbView P{n, F1, F2, C1, C2, rig1, rig2, rigs_finite != 0};
  const long long max_skip = 10LL * D.max_iterations;
  for (int base = 0; base < D.n_samples && (running || all); base += kWave) {
    for (int h = warp; h < kWave; h += kWarps) {
      const int s = base + h;
      bool v = false;
      if (s < D.n_samples)
        v = Sv::solve(D.samples + kS * ((size_t)pi * D.n_samples + s), P, W, w_model[h], lane);
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
          const double* q = W + kPairArea * (Sv::kCentral ? 0 : C1[i] * nc2 + C2[i]);
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
    if (best >= 0) warp_pair_models(best_model, rig1, nc1, rig2, nc2, W, lane);   // every warp its own copy
    for (int i = tid; i < n; i += kThreads) {
      const double* q = W + kPairArea * (Sv::kCentral ? 0 : C1[i] * nc2 + C2[i]);
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

// every sample index of a problem with at least k correspondences in [0, n); the samples of smaller problems are not read
int check_samples(cvb_ctx* ctx, const char* name, const int32_t* samples, const int32_t* prob_ptr, int n_prob, int ns, int k) {
  for (int i = 0; i < n_prob; i++) {
    const int n = prob_ptr[i + 1] - prob_ptr[i];
    if (n < k) continue;
    const int32_t* s = samples + k * (size_t)i * ns;
    for (size_t j = 0; j < k * (size_t)ns; j++)
      CVB_REQUIRE(ctx, s[j] >= 0 && s[j] < n, "%s: sample index %d out of range [0, %d) in problem %d", name, s[j], n, i);
  }
  return CVB_OK;
}

// staging offsets of the inputs (camera arrays unused by a central problem)
struct RelIn { size_t ptr, f1, f2, s1, s2, c1, c2, cp1, cp2, rig1, rig2, smp; };

// the tail shared by both calls: outputs staged after the inputs in St, one upload, one launch of ransac_rel_kernel<Sv>, one
// download
template <class Sv>
int run_rel_ransac(cvb_ctx* ctx, Stager& St, const RelIn& in, int n_prob, int ns, size_t N, int max_pairs, double threshold, int max_iterations,
                   double probability, cvb_rel_ransac_result* r) {
  const size_t S_all = (size_t)n_prob * ns;
  const bool all = r->sample_model != nullptr;
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
  D.prob_ptr = (const int*)(d + in.ptr); D.f1 = (const double*)(d + in.f1); D.f2 = (const double*)(d + in.f2);
  D.s1 = (const double*)(d + in.s1); D.s2 = (const double*)(d + in.s2); D.samples = (const int*)(d + in.smp);
  if (!Sv::kCentral) {
    D.cam1 = (const int*)(d + in.c1); D.cam2 = (const int*)(d + in.c2); D.cam_ptr1 = (const int*)(d + in.cp1); D.cam_ptr2 = (const int*)(d + in.cp2);
    D.rig1 = (const double*)(d + in.rig1); D.rig2 = (const double*)(d + in.rig2);
  }
  D.n_samples = ns; D.max_iterations = max_iterations; D.threshold = threshold; D.log_p = log(1.0 - probability);
  D.area = Sv::kArea > kPairArea * max_pairs ? Sv::kArea : kPairArea * max_pairs;
  D.best_sample = (int*)(d + o_bs); D.best_model = (double*)(d + o_bm); D.best_count = (int*)(d + o_bc); D.iterations = (int*)(d + o_it);
  D.consumed = (int*)(d + o_us); D.inlier_mask = r->inlier_mask ? d + o_mask : nullptr;
  if (all) { D.sample_model = (double*)(d + o_sm); D.sample_valid = d + o_sv; D.sample_count = (int*)(d + o_sc); }
  constexpr int kMaxPairs = Sv::kCentral ? 1 : kMaxCams * kMaxCams;
  constexpr int kMaxArea = Sv::kArea > kPairArea * kMaxPairs ? Sv::kArea : kPairArea * kMaxPairs;
  static cvb_once_per_device once;
  if (once.first(ctx->device)) {
    CVB_CUDA(ctx, cudaFuncSetAttribute(ransac_rel_kernel<Sv>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kWarps * kMaxArea * sizeof(double))));
  }
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemcpyAsync(d, hpin, in_bytes, cudaMemcpyHostToDevice, st));
  ransac_rel_kernel<Sv><<<n_prob, kThreads, (size_t)kWarps * D.area * sizeof(double), st>>>(D);
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
  }
  if (const int rc = check_samples(ctx, "ransac_noncentral_relative_pose", p->samples, p->prob_ptr, n_prob, ns, kSample)) return rc;
  const size_t S_all = (size_t)n_prob * ns;
  Stager St;
  RelIn in{};
  in.ptr = St.put(p->prob_ptr, ((size_t)n_prob + 1) * 4); in.f1 = St.put(p->f1, N * 24); in.f2 = St.put(p->f2, N * 24);
  in.s1 = St.put(p->sigma1, N * 8); in.s2 = St.put(p->sigma2, N * 8); in.c1 = St.put(p->cam1, N * 4); in.c2 = St.put(p->cam2, N * 4);
  in.cp1 = St.put(p->cam_ptr1, ((size_t)n_prob + 1) * 4); in.cp2 = St.put(p->cam_ptr2, ((size_t)n_prob + 1) * 4);
  in.smp = St.put(p->samples, S_all * kSample * 4);
  in.rig1 = St.reserve(NC1 * 96); in.rig2 = St.reserve(NC2 * 96);
  for (size_t j = 0; j < NC1; j++) {   // camera: offset (3) directly followed by the rotation (9, row-major)
    memcpy(St.h.data() + in.rig1 + 96 * j, p->cam_off1 + 3 * j, 24);
    memcpy(St.h.data() + in.rig1 + 96 * j + 24, p->cam_rot1 + 9 * j, 72);
  }
  for (size_t j = 0; j < NC2; j++) {
    memcpy(St.h.data() + in.rig2 + 96 * j, p->cam_off2 + 3 * j, 24);
    memcpy(St.h.data() + in.rig2 + 96 * j + 24, p->cam_rot2 + 9 * j, 72);
  }
  return run_rel_ransac<Solver17>(ctx, St, in, n_prob, ns, N, max_pairs, threshold, max_iterations, probability, r);
}

extern "C" int cvb_ransac_central_relative_pose_batch(cvb_ctx* ctx, const cvb_central_rel_ransac_problems* p, double threshold, int max_iterations,
                                                      double probability, cvb_rel_ransac_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, p && r && p->n_prob >= 0 && p->n_samples >= 0 && max_iterations >= 0, "ransac_central_relative_pose: bad arguments");
  CVB_REQUIRE(ctx, max_iterations <= INT32_MAX / 10, "ransac_central_relative_pose: max_iterations too large");
  const int n_prob = p->n_prob, ns = p->n_samples;
  if (n_prob == 0) return CVB_OK;
  CVB_REQUIRE(ctx, p->prob_ptr && r->best_sample && r->best_model && r->best_count && r->iterations && r->consumed,
              "ransac_central_relative_pose: null required pointer");
  CVB_REQUIRE(ctx, (r->sample_model != nullptr) == (r->sample_valid != nullptr) && (r->sample_model != nullptr) == (r->sample_count != nullptr),
              "ransac_central_relative_pose: sample_model / sample_valid / sample_count are requested together");
  CVB_REQUIRE(ctx, ptr_ok(p->prob_ptr, n_prob), "ransac_central_relative_pose: prob_ptr does not start at 0 or decreases");
  const size_t N = (size_t)p->prob_ptr[n_prob];
  CVB_REQUIRE(ctx, N == 0 || (p->f1 && p->f2 && p->sigma1 && p->sigma2), "ransac_central_relative_pose: null correspondence arrays");
  CVB_REQUIRE(ctx, ns == 0 || p->samples, "ransac_central_relative_pose: null samples");
  if (const int rc = check_samples(ctx, "ransac_central_relative_pose", p->samples, p->prob_ptr, n_prob, ns, kSample5)) return rc;
  Stager St;
  RelIn in{};
  in.ptr = St.put(p->prob_ptr, ((size_t)n_prob + 1) * 4); in.f1 = St.put(p->f1, N * 24); in.f2 = St.put(p->f2, N * 24);
  in.s1 = St.put(p->sigma1, N * 8); in.s2 = St.put(p->sigma2, N * 8); in.smp = St.put(p->samples, (size_t)n_prob * ns * kSample5 * 4);
  return run_rel_ransac<Solver5>(ctx, St, in, n_prob, ns, N, 1, threshold, max_iterations, probability, r);
}
