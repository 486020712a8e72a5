// geom_common.cuh — helpers shared by the geometric-verification translation units (geom_kernels.cu, ransac_abs.cu,
// ransac_rel.cu): the host staging block and the device arithmetic, including the per-correspondence absolute-pose score
// (score_abs_kernel, ransac_abs_kernel), the relative-pose score (score_rel_kernel, ransac_rel_kernel) and the 3x3 inverse of
// both RANSAC solvers.  Every device operation is an explicit round-to-nearest non-fused intrinsic, so results are
// reproducible bit for bit against a plain IEEE evaluation compiled with -ffp-contract=off.
#pragma once
#include <cuda_runtime.h>
#include <string.h>

#include <vector>

namespace {

// host staging: everything of a call goes through ONE pinned block and ONE device block
struct Stager {
  std::vector<unsigned char> h;
  size_t put(const void* p, size_t bytes) {
    const size_t off = (h.size() + 15) & ~size_t(15);
    h.resize(off + bytes);
    if (p && bytes) memcpy(h.data() + off, p, bytes);
    return off;
  }
  size_t reserve(size_t bytes) { return put(nullptr, bytes); }
};

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dot3(double a0, double a1, double a2, const double* p) {
  return add(add(mul(a0, p[0]), mul(a1, p[1])), mul(a2, p[2]));
}

// inverseSolution = [R^T | -R^T t] of a 3x4 [R|t] body-in-world model (row-major)
__device__ __forceinline__ void abs_inverse(const double* M, double Ri[9], double ti[3]) {
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) Ri[3 * r + c] = M[4 * c + r];
  const double t[3] = {M[3], M[7], M[11]};
#pragma unroll
  for (int r = 0; r < 3; r++) ti[r] = -dot3(Ri[3 * r], Ri[3 * r + 1], Ri[3 * r + 2], t);
}

// camera-frame ray q = Rc^T (inverseSolution * p - c) of world point p; returns |q|.  cam = offset (3) then Rc (9, row-major).
__device__ __forceinline__ double abs_ray(const double* Ri, const double* ti, const double* p, const double* cam, double q[3]) {
  double b[3];
#pragma unroll
  for (int r = 0; r < 3; r++) b[r] = sub(add(dot3(Ri[3 * r], Ri[3 * r + 1], Ri[3 * r + 2], p), ti[r]), cam[r]);
  const double* Rc = cam + 3;
#pragma unroll
  for (int r = 0; r < 3; r++) q[r] = dot3(Rc[r], Rc[3 + r], Rc[6 + r], b);
  return __dsqrt_rn(add(add(mul(q[0], q[0]), mul(q[1], q[1])), mul(q[2], q[2])));
}

// per-correspondence score of FrameAbsolutePoseSacProblem (FrameAbsolutePoseSacProblem.h:95-126):
// |normalize(q) - f|^2 / sigma; inlier iff score < threshold
__device__ __forceinline__ double abs_score(const double* Ri, const double* ti, const double* p, const double* f, double sigma, const double* cam) {
  double q[3];
  const double nrm = abs_ray(Ri, ti, p, cam, q);
  double e2 = 0.0;
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const double e = sub(__ddiv_rn(q[r], nrm), f[r]);
    e2 = r == 0 ? mul(e, e) : add(e2, mul(e, e));
  }
  return __ddiv_rn(e2, sigma);
}

// opengv::triangulation::triangulate2 [A] of bearings a (view 1), bb (view 2) under the model M = [R12|t12] (X1 = R12 X2 + t12):
// lambda = A^-1 b, X = (lambda0 a + t12 + lambda1 R12 bb) / 2 in view 1, r2 = R12^T X - R12^T t12 in view 2
__device__ __forceinline__ void rel_triangulate(const double* __restrict__ M, const double* a, const double* bb, double X[3], double r2[3]) {
  const double t[3] = {M[3], M[7], M[11]};
  double Ri[9], ti[3];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) Ri[3 * r + c] = M[4 * c + r];
#pragma unroll
  for (int r = 0; r < 3; r++) ti[r] = -dot3(Ri[3 * r], Ri[3 * r + 1], Ri[3 * r + 2], t);
  double u[3];
#pragma unroll
  for (int r = 0; r < 3; r++) u[r] = dot3(M[4 * r], M[4 * r + 1], M[4 * r + 2], bb);
  const double b0 = dot3(t[0], t[1], t[2], a), b1 = dot3(t[0], t[1], t[2], u);
  const double A00 = dot3(a[0], a[1], a[2], a), A10 = dot3(a[0], a[1], a[2], u), A01 = -A10, A11 = -dot3(u[0], u[1], u[2], u);
  const double det = sub(mul(A00, A11), mul(A01, A10));
  const double l0 = __ddiv_rn(sub(mul(A11, b0), mul(A01, b1)), det), l1 = __ddiv_rn(sub(mul(A00, b1), mul(A10, b0)), det);
#pragma unroll
  for (int r = 0; r < 3; r++) X[r] = __ddiv_rn(add(mul(l0, a[r]), add(t[r], mul(l1, u[r]))), 2.0);
#pragma unroll
  for (int r = 0; r < 3; r++) r2[r] = add(dot3(Ri[3 * r], Ri[3 * r + 1], Ri[3 * r + 2], X), ti[r]);
}

// score of correspondence i (bearings f1 / f2 [.][3], sigma1 / sigma2) of FrameRelativePoseSacProblem
// (frame-relative-pose-sac-problem.hpp:69-104) under the model M = [R12|t12] (X1 = R12 X2 + t12): the triangulation above, then
// 0.5 |normalize(X) - f|^2 / sigma per view; inlier iff score < threshold
__device__ __forceinline__ double rel_score(const double* __restrict__ M, const double* __restrict__ f1, const double* __restrict__ f2,
                                            const double* __restrict__ s1, const double* __restrict__ s2, int i) {
  const double a[3] = {f1[3 * (size_t)i], f1[3 * (size_t)i + 1], f1[3 * (size_t)i + 2]};
  const double bb[3] = {f2[3 * (size_t)i], f2[3 * (size_t)i + 1], f2[3 * (size_t)i + 2]};
  double X[3], r2[3];
  rel_triangulate(M, a, bb, X, r2);
  const double n1 = __dsqrt_rn(add(add(mul(X[0], X[0]), mul(X[1], X[1])), mul(X[2], X[2])));
  const double n2 = __dsqrt_rn(add(add(mul(r2[0], r2[0]), mul(r2[1], r2[1])), mul(r2[2], r2[2])));
  double e1 = 0.0, e2 = 0.0;
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const double d1 = sub(__ddiv_rn(X[r], n1), a[r]), d2 = sub(__ddiv_rn(r2[r], n2), bb[r]);
    e1 = r == 0 ? mul(d1, d1) : add(e1, mul(d1, d1));
    e2 = r == 0 ? mul(d2, d2) : add(e2, mul(d2, d2));
  }
  return add(__ddiv_rn(mul(e1, 0.5), s1[i]), __ddiv_rn(mul(e2, 0.5), s2[i]));
}

// inverse of a 3x3 matrix (row-major) by its adjugate
__device__ void inv3(const double* m, double* o) {
  const double c00 = sub(mul(m[4], m[8]), mul(m[5], m[7])), c01 = sub(mul(m[5], m[6]), mul(m[3], m[8])), c02 = sub(mul(m[3], m[7]), mul(m[4], m[6]));
  const double det = add(add(mul(m[0], c00), mul(m[1], c01)), mul(m[2], c02));
  o[0] = __ddiv_rn(c00, det); o[1] = __ddiv_rn(sub(mul(m[2], m[7]), mul(m[1], m[8])), det); o[2] = __ddiv_rn(sub(mul(m[1], m[5]), mul(m[2], m[4])), det);
  o[3] = __ddiv_rn(c01, det); o[4] = __ddiv_rn(sub(mul(m[0], m[8]), mul(m[2], m[6])), det); o[5] = __ddiv_rn(sub(mul(m[2], m[3]), mul(m[0], m[5])), det);
  o[6] = __ddiv_rn(c02, det); o[7] = __ddiv_rn(sub(mul(m[1], m[6]), mul(m[0], m[7])), det); o[8] = __ddiv_rn(sub(mul(m[0], m[4]), mul(m[1], m[3])), det);
}

}  // namespace
