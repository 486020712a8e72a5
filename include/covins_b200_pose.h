/*
 * covins_b200_pose.h — the pose conversions of the pose graph, one implementation for the host shim and the device kernels.
 *
 * Poses are row-major 4x4 [R t; 0 0 0 1] (double[16]) or pose7 = qx, qy, qz, qw, x, y, z.  Every product, sum and
 * difference is rounded on its own, in the order written: device code spells them __dmul_rn / __dadd_rn / __dsub_rn, so
 * ptxas cannot contract them into fused multiply-adds, and host code is plain C++ (the x86-64 baseline has no FMA
 * instruction to contract into).  sqrt and division are the correctly rounded defaults on both sides.  The host shim and
 * the kernels of cvb_pgo therefore give the same bits, and oracle/pgo.py restates the same order in float64.
 */
#ifndef COVINS_B200_POSE_H_
#define COVINS_B200_POSE_H_

#include <math.h>

#if defined(__CUDACC__)
#define CVB_POSE_HD __host__ __device__ __forceinline__
#else
#define CVB_POSE_HD inline
#endif

namespace cvb_pose {

CVB_POSE_HD double mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
CVB_POSE_HD double add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
CVB_POSE_HD double sub(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}

// rotation part → quaternion (x,y,z,w), the convention of Eigen::Quaterniond(R) used at keyframe_base.cpp:490-499 (w >= 0
// branch of Eigen's algorithm); the translation is copied
CVB_POSE_HD void transform_to_pose7(const double* T /*[16]*/, double* out /*[7]*/) {
  const double m00 = T[0], m11 = T[5], m22 = T[10];
  double q[4];  // x y z w
  const double tr = add(add(m00, m11), m22);
  if (tr > 0) {
    double t = sqrt(add(tr, 1.0));
    q[3] = mul(0.5, t);
    t = 0.5 / t;
    q[0] = mul(sub(T[9], T[6]), t);
    q[1] = mul(sub(T[2], T[8]), t);
    q[2] = mul(sub(T[4], T[1]), t);
  } else {
    int i = 0;
    if (m11 > m00) i = 1;
    if (m22 > T[5 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double t = sqrt(add(sub(sub(T[5 * i], T[5 * j]), T[5 * k]), 1.0));
    q[i] = mul(0.5, t);
    t = 0.5 / t;
    q[3] = mul(sub(T[4 * k + j], T[4 * j + k]), t);
    q[j] = mul(add(T[4 * j + i], T[4 * i + j]), t);
    q[k] = mul(add(T[4 * k + i], T[4 * i + k]), t);
  }
  out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3];
  out[4] = T[3]; out[5] = T[7]; out[6] = T[11];
}

// Utils::Ceres2Transform (covins_comm/src/covins_base/utils_base.cpp:28-43): normalised quaternion → 4x4
CVB_POSE_HD void pose7_to_transform(const double* p /*[7]*/, double* T /*[16]*/) {
  double x = p[0], y = p[1], z = p[2], w = p[3];
  const double n = 1.0 / sqrt(add(add(add(mul(x, x), mul(y, y)), mul(z, z)), mul(w, w)));
  x = mul(x, n); y = mul(y, n); z = mul(z, n); w = mul(w, n);
  T[0] = sub(1.0, mul(2.0, add(mul(y, y), mul(z, z))));
  T[1] = mul(2.0, sub(mul(x, y), mul(z, w)));
  T[2] = mul(2.0, add(mul(x, z), mul(y, w)));
  T[4] = mul(2.0, add(mul(x, y), mul(z, w)));
  T[5] = sub(1.0, mul(2.0, add(mul(x, x), mul(z, z))));
  T[6] = mul(2.0, sub(mul(y, z), mul(x, w)));
  T[8] = mul(2.0, sub(mul(x, z), mul(y, w)));
  T[9] = mul(2.0, add(mul(y, z), mul(x, w)));
  T[10] = sub(1.0, mul(2.0, add(mul(x, x), mul(y, y))));
  T[3] = p[4]; T[7] = p[5]; T[11] = p[6];
  T[12] = 0.0; T[13] = 0.0; T[14] = 0.0; T[15] = 1.0;
}

// Ta^-1 * Tb for rigid transforms: R = Ra^T Rb, t = Ra^T (tb - ta), each entry summed from 0 over m = 0, 1, 2
CVB_POSE_HD void rel_transform(const double* Ta, const double* Tb, double* R /*[16]*/) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      double s = 0;
      for (int m = 0; m < 3; m++) s = add(s, mul(Ta[4 * m + r], Tb[4 * m + c]));
      R[4 * r + c] = s;
    }
  for (int r = 0; r < 3; r++) {
    double s = 0;
    for (int m = 0; m < 3; m++) s = add(s, mul(Ta[4 * m + r], sub(Tb[4 * m + 3], Ta[4 * m + 3])));
    R[4 * r + 3] = s;
  }
  R[12] = 0.0; R[13] = 0.0; R[14] = 0.0; R[15] = 1.0;
}

// LLT(cov^-1).matrixL().transpose() of a symmetric 6x6 (optimization_be.cpp:922-923): cov is factored, its factor inverted,
// the inverse formed and factored again.  false when either factorisation meets a pivot that is not > 0 (out untouched).
CVB_POSE_HD bool sqrt_info_from_cov(const double* cov /*[36] row-major*/, double* out /*[36]*/) {
  double L[36] = {0}, X[36] = {0}, P[36];
  for (int c = 0; c < 6; c++)
    for (int r = c; r < 6; r++) {
      double s = cov[6 * r + c];
      for (int m = 0; m < c; m++) s = sub(s, mul(L[6 * r + m], L[6 * c + m]));
      if (r == c) {
        if (!(s > 0)) return false;
        L[6 * c + c] = sqrt(s);
      } else {
        L[6 * r + c] = s / L[6 * c + c];
      }
    }
  for (int c = 0; c < 6; c++)
    for (int r = c; r < 6; r++) {
      double s = (r == c) ? 1.0 : 0.0;
      for (int m = c; m < r; m++) s = sub(s, mul(L[6 * r + m], X[6 * m + c]));
      X[6 * r + c] = s / L[6 * r + r];
    }
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      double s = 0;
      for (int m = (r > c ? r : c); m < 6; m++) s = add(s, mul(X[6 * m + r], X[6 * m + c]));
      P[6 * r + c] = s;
    }
  double M[36] = {0};
  for (int c = 0; c < 6; c++)
    for (int r = c; r < 6; r++) {
      double s = P[6 * r + c];
      for (int m = 0; m < c; m++) s = sub(s, mul(M[6 * r + m], M[6 * c + m]));
      if (r == c) {
        if (!(s > 0)) return false;
        M[6 * c + c] = sqrt(s);
      } else {
        M[6 * r + c] = s / M[6 * c + c];
      }
    }
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) out[6 * r + c] = M[6 * c + r];
  return true;
}

}  // namespace cvb_pose

#endif /* COVINS_B200_POSE_H_ */
