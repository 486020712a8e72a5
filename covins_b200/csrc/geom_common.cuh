// geom_common.cuh — helpers shared by the geometric-verification translation units (geom_kernels.cu, ransac_abs.cu): the
// host staging block and the device arithmetic, including the per-correspondence absolute-pose score both score_abs_kernel
// and ransac_abs_kernel call.  Every device operation is an explicit round-to-nearest non-fused intrinsic, so results are
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

}  // namespace
