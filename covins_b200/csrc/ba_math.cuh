// ba_math.cuh — FP64 device math for the BA/PGO kernels: SO(3)/quaternion helpers and the three cost
// functions with ANALYTIC Jacobians in the local (tangent) parametrisation.
//
// Restates (assumptions marked [A], see SURVEY.md Appendix A; the arithmetic lives in robopt_open / aslam_cv2,
// which are not in the reference tree):
//   pose block [qx,qy,qz,qw,x,y,z] = T_ws            keyframe_base.cpp:486-499
//   Plus [A]   delta = [dtheta, dp]; q+ = Exp(dtheta) * q (world-side), p+ = p + dp
//              (robopt::local_param::PoseQuaternionLocalParameterization, optimization_be.cpp:69,303,843)
//   reprojection [A]  robopt::reprojection::GlobalEuclideanReprError<Camera,Distortion>, all six instantiations
//                     (optimization_be.cpp:186-231)
//   between [A]       robopt::posegraph::SixDofBetweenError, kImu (optimization_be.cpp:252,554,934,968,1017)
//   IMU [A]           robopt::imu::PreintegrationFactor over VINS-Mono style midpoint preintegration
//                     (optimization_be.cpp:140-143, 396-416)
// The oracle (oracle/ba_oracle.py) gets the same Jacobians from autograd; tests compare the two.
#pragma once
#include <math.h>

namespace bam {

struct V3 {
  double x, y, z;
};
struct M3 {
  double m[9];  // row-major
};

__host__ __device__ inline V3 v3(double x, double y, double z) { return V3{x, y, z}; }
__host__ __device__ inline V3 operator+(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
__host__ __device__ inline V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
__host__ __device__ inline V3 operator*(double s, V3 a) { return V3{s * a.x, s * a.y, s * a.z}; }
__host__ __device__ inline double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__host__ __device__ inline V3 cross(V3 a, V3 b) {
  return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
__host__ __device__ inline V3 mul(const M3& A, V3 v) {
  return V3{A.m[0] * v.x + A.m[1] * v.y + A.m[2] * v.z, A.m[3] * v.x + A.m[4] * v.y + A.m[5] * v.z,
            A.m[6] * v.x + A.m[7] * v.y + A.m[8] * v.z};
}
__host__ __device__ inline V3 mulT(const M3& A, V3 v) {  // A^T v
  return V3{A.m[0] * v.x + A.m[3] * v.y + A.m[6] * v.z, A.m[1] * v.x + A.m[4] * v.y + A.m[7] * v.z,
            A.m[2] * v.x + A.m[5] * v.y + A.m[8] * v.z};
}
__host__ __device__ inline M3 mul(const M3& A, const M3& B) {
  M3 C;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C.m[3 * i + j] = A.m[3 * i] * B.m[j] + A.m[3 * i + 1] * B.m[3 + j] + A.m[3 * i + 2] * B.m[6 + j];
  return C;
}
__host__ __device__ inline M3 transpose(const M3& A) {
  return M3{{A.m[0], A.m[3], A.m[6], A.m[1], A.m[4], A.m[7], A.m[2], A.m[5], A.m[8]}};
}
__host__ __device__ inline M3 mulAtB(const M3& A, const M3& B) { return mul(transpose(A), B); }
__host__ __device__ inline M3 skew(V3 v) { return M3{{0, -v.z, v.y, v.z, 0, -v.x, -v.y, v.x, 0}}; }
__host__ __device__ inline M3 eye3() { return M3{{1, 0, 0, 0, 1, 0, 0, 0, 1}}; }

struct Q4 {
  double x, y, z, w;
};
__host__ __device__ inline Q4 qmul(Q4 a, Q4 b) {
  return Q4{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
            a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
__host__ __device__ inline Q4 qconj(Q4 q) { return Q4{-q.x, -q.y, -q.z, q.w}; }
__host__ __device__ inline Q4 qnormalized(Q4 q) {
  const double n = 1.0 / sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return Q4{q.x * n, q.y * n, q.z * n, q.w * n};
}
__host__ __device__ inline M3 q2R(Q4 q) {
  const double x = q.x, y = q.y, z = q.z, w = q.w;
  return M3{{1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w), 2 * (x * y + z * w),
             1 - 2 * (x * x + z * z), 2 * (y * z - x * w), 2 * (x * z - y * w), 2 * (y * z + x * w),
             1 - 2 * (x * x + y * y)}};
}
// Exp: rotation vector → unit quaternion (series below 1e-6 rad)
__host__ __device__ inline Q4 qexp(V3 p) {
  const double th2 = dot(p, p);
  double k, w;
  if (th2 < 1e-12) {
    k = 0.5 - th2 / 48.0;
    w = 1.0 - th2 / 8.0;
  } else {
    const double th = sqrt(th2);
    k = sin(0.5 * th) / th;
    w = cos(0.5 * th);
  }
  return Q4{k * p.x, k * p.y, k * p.z, w};
}
// right Jacobian of SO(3): Exp(phi + d) ~ Exp(phi) Exp(Jr(phi) d)
__host__ __device__ inline M3 so3_Jr(V3 p) {
  const double th2 = dot(p, p);
  const M3 K = skew(p), K2 = mul(K, K);
  double a, b;
  if (th2 < 1e-10) {
    a = 0.5 - th2 / 24.0;
    b = 1.0 / 6.0 - th2 / 120.0;
  } else {
    const double th = sqrt(th2);
    a = (1.0 - cos(th)) / th2;
    b = (th - sin(th)) / (th2 * th);
  }
  M3 J = eye3();
  for (int i = 0; i < 9; i++) J.m[i] += -a * K.m[i] + b * K2.m[i];
  return J;
}
// d(2 vec(E * Exp(phi)))/dphi at 0 for E = (v, w):  w I + [v]x
__host__ __device__ inline M3 quat_right_jac(Q4 E) {
  M3 J = skew(V3{E.x, E.y, E.z});
  J.m[0] += E.w;
  J.m[4] += E.w;
  J.m[8] += E.w;
  return J;
}

struct Pose {
  Q4 q;
  V3 t;
};
__host__ __device__ inline Pose load_pose(const double* p) { return Pose{Q4{p[0], p[1], p[2], p[3]}, V3{p[4], p[5], p[6]}}; }
__host__ __device__ inline void pose_plus(const double* p, const double* d, double* out) {
  Q4 q = qnormalized(qmul(qexp(V3{d[0], d[1], d[2]}), Q4{p[0], p[1], p[2], p[3]}));
  out[0] = q.x; out[1] = q.y; out[2] = q.z; out[3] = q.w;
  out[4] = p[4] + d[3]; out[5] = p[5] + d[4]; out[6] = p[6] + d[5];
}

// ceres::CauchyLoss(a) + Corrector: rho'' <= 0 → residual and Jacobian scaled by sqrt(rho'); cost = rho/2.
// a2 = a*a; a2 <= 0 means "no loss".
__host__ __device__ inline void cauchy(double s, double a2, double* scale, double* cost) {
  if (a2 <= 0.0) {
    *scale = 1.0;
    *cost = 0.5 * s;
  } else {
    *scale = sqrt(1.0 / (1.0 + s / a2));
    *cost = 0.5 * a2 * log1p(s / a2);
  }
}

// ---- camera models of robopt::reprojection::GlobalEuclideanReprError<Camera, Distortion> (optimization_be.cpp:186-231,
// 480-525): Camera ∈ {aslam::PinholeCamera, aslam::UnifiedProjectionCamera}, Distortion ∈ {RadTan, Equidistant, Fisheye}.
// The formulas are the published aslam_cv2 ones [A] (the library is not in the tree):
//   pinhole   x = X/Z, y = Y/Z
//   unified   x = X/(Z + xi |p|), y = Y/(Z + xi |p|)            (intrinsics [xi, fu, fv, cu, cv])
//   radtan    (k1,k2,p1,p2): xd = x(1+k1 r2+k2 r4) + 2 p1 x y + p2 (r2+2x2),  yd = y(...) + p1 (r2+2y2) + 2 p2 x y
//   equidist  (k1..k4): theta = atan r, thd = theta (1 + k1 th2 + k2 th4 + k3 th6 + k4 th8), (xd,yd) = (thd/r)(x,y)
//   fisheye   FOV model (w): (xd,yd) = atan(2 r tan(w/2)) / (w r) (x,y); w*w < 1e-5 → identity; r*r < 1e-5 → 2 tan(w/2)/w
//   u = fu xd + cu, v = fv yd + cv.
constexpr int CAM_PINHOLE = 0, CAM_UNIFIED = 1;
constexpr int DIST_RADTAN = 0, DIST_EQUI = 1, DIST_FISHEYE = 2;
struct CamModel {
  int cam, dist;
  double xi;
};

// normalised image point (x, y) of a camera-frame point and its 2x3 Jacobian N (row-major); false = not projectable
__host__ __device__ inline bool cam_normalise(const CamModel& cm, V3 pc, double* x, double* y, double N[6], bool want_jac) {
  if (cm.cam == CAM_PINHOLE) {
    if (!(pc.z > 1e-10)) return false;   // aslam::ProjectionResult::POINT_BEHIND_CAMERA [A]
    const double iz = 1.0 / pc.z;
    *x = pc.x * iz; *y = pc.y * iz;
    if (want_jac) { N[0] = iz; N[1] = 0.0; N[2] = -pc.x * iz * iz; N[3] = 0.0; N[4] = iz; N[5] = -pc.y * iz * iz; }
    return true;
  }
  const double d = sqrt(pc.x * pc.x + pc.y * pc.y + pc.z * pc.z);
  const double den = pc.z + cm.xi * d;
  if (!(den > 1e-10) || !(d > 0.0)) return false;   // outside the unified model's field of view [A]
  const double rz = 1.0 / den;
  *x = pc.x * rz; *y = pc.y * rz;
  if (want_jac) {
    const double k = cm.xi / d, rz2 = rz * rz;
    // d den / d pc = (xi X/d, xi Y/d, 1 + xi Z/d)
    const double dx = k * pc.x, dy = k * pc.y, dz = 1.0 + k * pc.z;
    N[0] = rz - pc.x * rz2 * dx; N[1] = -pc.x * rz2 * dy; N[2] = -pc.x * rz2 * dz;
    N[3] = -pc.y * rz2 * dx; N[4] = rz - pc.y * rz2 * dy; N[5] = -pc.y * rz2 * dz;
  }
  return true;
}

// distorted point and its 2x2 Jacobian D (row-major) w.r.t. (x, y)
__host__ __device__ inline void cam_distort(const CamModel& cm, const double* dist, double x, double y, double* xd, double* yd, double D[4],
                                            bool want_jac) {
  const double r2 = x * x + y * y;
  if (cm.dist == DIST_RADTAN) {
    const double k1 = dist[0], k2 = dist[1], p1 = dist[2], p2 = dist[3];
    const double rad = 1.0 + k1 * r2 + k2 * r2 * r2;
    *xd = x * rad + 2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x);
    *yd = y * rad + p1 * (r2 + 2.0 * y * y) + 2.0 * p2 * x * y;
    if (want_jac) {
      const double c = k1 + 2.0 * k2 * r2;
      D[0] = rad + 2.0 * x * x * c + 2.0 * p1 * y + 6.0 * p2 * x;
      D[1] = 2.0 * x * y * c + 2.0 * p1 * x + 2.0 * p2 * y;
      D[2] = D[1];
      D[3] = rad + 2.0 * y * y * c + 6.0 * p1 * y + 2.0 * p2 * x;
    }
    return;
  }
  double s, ds_dr_over_r;   // (xd,yd) = s (x,y);  ds/dr divided by r (finite at r → 0)
  if (cm.dist == DIST_EQUI) {
    const double r = sqrt(r2);
    if (r < 1e-8) { s = 1.0; ds_dr_over_r = 0.0; }
    else {
      const double th = atan(r), t2 = th * th, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
      const double thd = th * (1.0 + dist[0] * t2 + dist[1] * t4 + dist[2] * t6 + dist[3] * t8);
      const double dthd = 1.0 + 3.0 * dist[0] * t2 + 5.0 * dist[1] * t4 + 7.0 * dist[2] * t6 + 9.0 * dist[3] * t8;
      s = thd / r;
      ds_dr_over_r = (dthd / (1.0 + r2) * r - thd) / (r2 * r);
    }
  } else {   // DIST_FISHEYE (FOV)
    const double w = dist[0];
    if (w * w < 1e-5) { s = 1.0; ds_dr_over_r = 0.0; }
    else {
      const double c = 2.0 * tan(0.5 * w);
      if (r2 < 1e-5) { s = c / w; ds_dr_over_r = 0.0; }
      else {
        const double r = sqrt(r2), at = atan(c * r);
        s = at / (w * r);
        ds_dr_over_r = (c * r / (1.0 + c * c * r2) - at) / (w * r2 * r);
      }
    }
  }
  *xd = s * x; *yd = s * y;
  if (want_jac) {
    D[0] = s + x * x * ds_dr_over_r; D[1] = x * y * ds_dr_over_r;
    D[2] = D[1]; D[3] = s + y * y * ds_dr_over_r;
  }
}

// ---- reprojection: r (2), Jl = dr/dp_w (2x3, row-major), Jp = dr/d[dtheta,dp] (2x6).  Returns false if the
// point is not projectable (behind the camera / outside the model's field of view): the residual is then defined as zero
// with zero Jacobian.
__host__ __device__ inline bool reproj(const double* pose, const double* extr, const double* intr, const double* dist, const CamModel& cm,
                                       const double* lm, double u_obs, double v_obs, double sigma, double r[2],
                                       double Jp[12], double Jl[6], bool want_jac) {
  const Pose Pw = load_pose(pose), Ps = load_pose(extr);
  const M3 Rws = q2R(Pw.q), Rsc = q2R(Ps.q);
  const V3 d = V3{lm[0], lm[1], lm[2]} - Pw.t;
  const V3 ps = mulT(Rws, d);
  const V3 pc = mulT(Rsc, ps - Ps.t);
  double x, y, N[6];
  if (!cam_normalise(cm, pc, &x, &y, N, want_jac)) {
    r[0] = r[1] = 0.0;
    if (want_jac) {
      for (int i = 0; i < 12; i++) Jp[i] = 0.0;
      for (int i = 0; i < 6; i++) Jl[i] = 0.0;
    }
    return false;
  }
  double xd, yd, D[4];
  cam_distort(cm, dist, x, y, &xd, &yd, D, want_jac);
  const double is = 1.0 / sigma;
  r[0] = (intr[0] * xd + intr[2] - u_obs) * is;
  r[1] = (intr[1] * yd + intr[3] - v_obs) * is;
  if (!want_jac) return true;
  // d(u,v)/d pc (2x3), already divided by sigma:  diag(fx, fy)/sigma * D * N
  const double fx = intr[0] * is, fy = intr[1] * is;
  const double a00 = fx * (D[0] * N[0] + D[1] * N[3]), a01 = fx * (D[0] * N[1] + D[1] * N[4]), a02 = fx * (D[0] * N[2] + D[1] * N[5]);
  const double a10 = fy * (D[2] * N[0] + D[3] * N[3]), a11 = fy * (D[2] * N[1] + D[3] * N[4]), a12 = fy * (D[2] * N[2] + D[3] * N[5]);
  // B = A * Rsc^T (2x3): derivative w.r.t. p_s
  const double b00 = a00 * Rsc.m[0] + a01 * Rsc.m[1] + a02 * Rsc.m[2], b01 = a00 * Rsc.m[3] + a01 * Rsc.m[4] + a02 * Rsc.m[5],
               b02 = a00 * Rsc.m[6] + a01 * Rsc.m[7] + a02 * Rsc.m[8];
  const double b10 = a10 * Rsc.m[0] + a11 * Rsc.m[1] + a12 * Rsc.m[2], b11 = a10 * Rsc.m[3] + a11 * Rsc.m[4] + a12 * Rsc.m[5],
               b12 = a10 * Rsc.m[6] + a11 * Rsc.m[7] + a12 * Rsc.m[8];
  // Jl = B * Rws^T
  Jl[0] = b00 * Rws.m[0] + b01 * Rws.m[1] + b02 * Rws.m[2];
  Jl[1] = b00 * Rws.m[3] + b01 * Rws.m[4] + b02 * Rws.m[5];
  Jl[2] = b00 * Rws.m[6] + b01 * Rws.m[7] + b02 * Rws.m[8];
  Jl[3] = b10 * Rws.m[0] + b11 * Rws.m[1] + b12 * Rws.m[2];
  Jl[4] = b10 * Rws.m[3] + b11 * Rws.m[4] + b12 * Rws.m[5];
  Jl[5] = b10 * Rws.m[6] + b11 * Rws.m[7] + b12 * Rws.m[8];
  // Jp = [Jl [d]x , -Jl]
  Jp[0] = Jl[1] * d.z - Jl[2] * d.y;
  Jp[1] = Jl[2] * d.x - Jl[0] * d.z;
  Jp[2] = Jl[0] * d.y - Jl[1] * d.x;
  Jp[3] = -Jl[0]; Jp[4] = -Jl[1]; Jp[5] = -Jl[2];
  Jp[6] = Jl[4] * d.z - Jl[5] * d.y;
  Jp[7] = Jl[5] * d.x - Jl[3] * d.z;
  Jp[8] = Jl[3] * d.y - Jl[4] * d.x;
  Jp[9] = -Jl[3]; Jp[10] = -Jl[4]; Jp[11] = -Jl[5];
  return true;
}

// ---- loss-corrected reprojection residual norm of one observation (cvb_ba_reproj_norms, optimization_be.cpp:270-290):
// r from reproj, s = r.r, norm = sqrt(s) * the Cauchy scale (a2 <= 0: |r|); *projectable = reproj's result.  Never inlined:
// ptxas may fuse a multiply and an add differently in different callers, so the kernels that must report the same norm
// bit for bit (the bundle adjustment's reproj_norms_kernel, cvb_landmark_outliers) call this one separately compiled body.
// Device code only: host translation units that include this header for its __host__ __device__ math do not see it.
#ifdef __CUDACC__
__device__ __noinline__ static double corrected_norm(const double* pose, const double* extr, const double* intr, const double* dist,
                                                     const CamModel& cm, const double* lm, double u_obs, double v_obs, double sigma,
                                                     double a2, bool* projectable) {
  double r[2];
  *projectable = reproj(pose, extr, intr, dist, cm, lm, u_obs, v_obs, sigma, r, nullptr, nullptr, false);
  const double s = r[0] * r[0] + r[1] * r[1];
  double sc, c;
  cauchy(s, a2, &sc, &c);
  return sqrt(s) * sc;
}
#endif

// ---- between factor: e = S [2 vec(qm^-1 q1^-1 q2); R1^T (t2 - t1) - tm]   (6), J = [de/dx1 (6x6) | de/dx2 (6x6)]
// stored row-major as 6 x 12.
__host__ __device__ inline void between(const double* pose1, const double* pose2, const double* qm, const double* tm,
                                        const double* S, double e[6], double J[72], bool want_jac) {
  const Pose P1 = load_pose(pose1), P2 = load_pose(pose2);
  const Q4 Qm{qm[0], qm[1], qm[2], qm[3]};
  const Q4 E = qmul(qconj(Qm), qmul(qconj(P1.q), P2.q));
  const M3 R1 = q2R(P1.q), R2 = q2R(P2.q);
  const V3 dt = P2.t - P1.t;
  const V3 et = mulT(R1, dt) - V3{tm[0], tm[1], tm[2]};
  const double raw[6] = {2 * E.x, 2 * E.y, 2 * E.z, et.x, et.y, et.z};
  for (int i = 0; i < 6; i++) {
    double s = 0;
    for (int k = 0; k < 6; k++) s += S[6 * i + k] * raw[k];
    e[i] = s;
  }
  if (!want_jac) return;
  const M3 Gq = quat_right_jac(E);
  const M3 A = mul(Gq, transpose(R2));   // d e_rot / d dtheta2 ; d e_rot / d dtheta1 = -A
  const M3 R1t = transpose(R1);
  const M3 B = mul(R1t, skew(dt));       // d e_t / d dtheta1
  double Jr[72];
  for (int i = 0; i < 72; i++) Jr[i] = 0.0;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      Jr[12 * i + j] = -A.m[3 * i + j];           // rot wrt dtheta1
      Jr[12 * i + 6 + j] = A.m[3 * i + j];        // rot wrt dtheta2
      Jr[12 * (3 + i) + j] = B.m[3 * i + j];      // trans wrt dtheta1
      Jr[12 * (3 + i) + 3 + j] = -R1t.m[3 * i + j];   // trans wrt dp1
      Jr[12 * (3 + i) + 9 + j] = R1t.m[3 * i + j];    // trans wrt dp2
    }
  for (int i = 0; i < 6; i++)
    for (int c = 0; c < 12; c++) {
      double s = 0;
      for (int k = 0; k < 6; k++) s += S[6 * i + k] * Jr[12 * k + c];
      J[12 * i + c] = s;
    }
}

// ---- IMU preintegration factor.  pre: dt_sum, alpha(3), beta(3), gamma(4), ba_lin(3), bg_lin(3), then the five
// bias Jacobian blocks dp_dba, dp_dbg, dq_dbg, dv_dba, dv_dbg (9 each, row-major), then sqrt_info (225).
struct ImuPre {
  double T;
  double alpha[3], beta[3], gamma[4], ba[3], bg[3];
  double dp_dba[9], dp_dbg[9], dq_dbg[9], dv_dba[9], dv_dbg[9];
  double sqrt_info[225];
};

// raw residual r (15) and raw Jacobian Jraw (15 x 30, columns [pose_i 6 | sb_i 9 | pose_j 6 | sb_j 9]); whitening by
// sqrt_info is applied by the caller.
__host__ __device__ inline void imu_raw(const double* pose_i, const double* sb_i, const double* pose_j, const double* sb_j,
                                        const ImuPre& P, double g, double r[15], double* Jraw /*450 or null*/) {
  const Pose Pi = load_pose(pose_i), Pj = load_pose(pose_j);
  const M3 Ri = q2R(Pi.q), Rj = q2R(Pj.q);
  const V3 vi{sb_i[0], sb_i[1], sb_i[2]}, vj{sb_j[0], sb_j[1], sb_j[2]};
  const V3 dba{sb_i[3] - P.ba[0], sb_i[4] - P.ba[1], sb_i[5] - P.ba[2]};
  const V3 dbg{sb_i[6] - P.bg[0], sb_i[7] - P.bg[1], sb_i[8] - P.bg[2]};
  const M3 Jpa{{P.dp_dba[0], P.dp_dba[1], P.dp_dba[2], P.dp_dba[3], P.dp_dba[4], P.dp_dba[5], P.dp_dba[6], P.dp_dba[7], P.dp_dba[8]}};
  const M3 Jpg{{P.dp_dbg[0], P.dp_dbg[1], P.dp_dbg[2], P.dp_dbg[3], P.dp_dbg[4], P.dp_dbg[5], P.dp_dbg[6], P.dp_dbg[7], P.dp_dbg[8]}};
  const M3 Jqg{{P.dq_dbg[0], P.dq_dbg[1], P.dq_dbg[2], P.dq_dbg[3], P.dq_dbg[4], P.dq_dbg[5], P.dq_dbg[6], P.dq_dbg[7], P.dq_dbg[8]}};
  const M3 Jva{{P.dv_dba[0], P.dv_dba[1], P.dv_dba[2], P.dv_dba[3], P.dv_dba[4], P.dv_dba[5], P.dv_dba[6], P.dv_dba[7], P.dv_dba[8]}};
  const M3 Jvg{{P.dv_dbg[0], P.dv_dbg[1], P.dv_dbg[2], P.dv_dbg[3], P.dv_dbg[4], P.dv_dbg[5], P.dv_dbg[6], P.dv_dbg[7], P.dv_dbg[8]}};
  const double T = P.T;
  const V3 gv{0, 0, g};
  const V3 a_hat = V3{P.alpha[0], P.alpha[1], P.alpha[2]} + mul(Jpa, dba) + mul(Jpg, dbg);
  const V3 b_hat = V3{P.beta[0], P.beta[1], P.beta[2]} + mul(Jva, dba) + mul(Jvg, dbg);
  const V3 theta = mul(Jqg, dbg);
  const Q4 gam{P.gamma[0], P.gamma[1], P.gamma[2], P.gamma[3]};
  const Q4 g_hat = qmul(gam, qexp(theta));
  const V3 wp = 0.5 * T * T * gv + Pj.t - Pi.t - T * vi;
  const V3 wv = T * gv + vj - vi;
  const V3 rp = mulT(Ri, wp) - a_hat;
  const Q4 Mq = qmul(qconj(gam), qmul(qconj(Pi.q), Pj.q));   // gamma^-1 qi^-1 qj
  const Q4 E = qmul(qconj(g_hat), qmul(qconj(Pi.q), Pj.q));
  const V3 rv = mulT(Ri, wv) - b_hat;
  r[0] = rp.x; r[1] = rp.y; r[2] = rp.z;
  r[3] = 2 * E.x; r[4] = 2 * E.y; r[5] = 2 * E.z;
  r[6] = rv.x; r[7] = rv.y; r[8] = rv.z;
  for (int k = 0; k < 3; k++) {
    r[9 + k] = sb_j[3 + k] - sb_i[3 + k];
    r[12 + k] = sb_j[6 + k] - sb_i[6 + k];
  }
  if (!Jraw) return;
  for (int i = 0; i < 450; i++) Jraw[i] = 0.0;
  const M3 Rit = transpose(Ri);
  const M3 Gq = quat_right_jac(E);
  const M3 GRjT = mul(Gq, transpose(Rj));
  const M3 dp_th = mul(Rit, skew(wp));
  const M3 dv_th = mul(Rit, skew(wv));
  // d r_q / d bg_i = -Gq * R(M)^T * Jr(-theta) * Jqg
  const V3 mth{-theta.x, -theta.y, -theta.z};
  const M3 dq_bg = mul(mul(Gq, transpose(q2R(Mq))), mul(so3_Jr(mth), Jqg));
  // column offsets: pose_i 0..5 (theta 0-2, p 3-5), sb_i 6..14 (v 6-8, ba 9-11, bg 12-14), pose_j 15..20, sb_j 21..29
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {
      const int ab = 3 * a + b;
      // r_p rows 0..2
      Jraw[30 * a + b] = dp_th.m[ab];
      Jraw[30 * a + 3 + b] = -Rit.m[ab];
      Jraw[30 * a + 6 + b] = -T * Rit.m[ab];
      Jraw[30 * a + 9 + b] = -Jpa.m[ab];
      Jraw[30 * a + 12 + b] = -Jpg.m[ab];
      Jraw[30 * a + 18 + b] = Rit.m[ab];
      // r_q rows 3..5
      Jraw[30 * (3 + a) + b] = -GRjT.m[ab];
      Jraw[30 * (3 + a) + 12 + b] = -dq_bg.m[ab];
      Jraw[30 * (3 + a) + 15 + b] = GRjT.m[ab];
      // r_v rows 6..8
      Jraw[30 * (6 + a) + b] = dv_th.m[ab];
      Jraw[30 * (6 + a) + 6 + b] = -Rit.m[ab];
      Jraw[30 * (6 + a) + 9 + b] = -Jva.m[ab];
      Jraw[30 * (6 + a) + 12 + b] = -Jvg.m[ab];
      Jraw[30 * (6 + a) + 21 + b] = Rit.m[ab];
    }
  for (int a = 0; a < 3; a++) {
    Jraw[30 * (9 + a) + 9 + a] = -1.0;
    Jraw[30 * (9 + a) + 24 + a] = 1.0;
    Jraw[30 * (12 + a) + 12 + a] = -1.0;
    Jraw[30 * (12 + a) + 27 + a] = 1.0;
  }
}

// Column c (0..29) of the raw IMU Jacobian and, optionally, the raw residual — the same quantities as imu_raw(), arranged for
// one-lane-per-column evaluation (lin_imu_kernel: a warp per factor; every lane recomputes the handful of shared 3x3
// products, ~600 flops, and owns one column of the 15x30 Jacobian).
__host__ __device__ inline void imu_raw_column(const double* pose_i, const double* sb_i, const double* pose_j, const double* sb_j,
                                               const ImuPre& P, double g, int c, double col[15], double* r /*15 or null*/) {
  const Pose Pi = load_pose(pose_i), Pj = load_pose(pose_j);
  const M3 Ri = q2R(Pi.q), Rj = q2R(Pj.q);
  const V3 vi{sb_i[0], sb_i[1], sb_i[2]}, vj{sb_j[0], sb_j[1], sb_j[2]};
  const V3 dba{sb_i[3] - P.ba[0], sb_i[4] - P.ba[1], sb_i[5] - P.ba[2]};
  const V3 dbg{sb_i[6] - P.bg[0], sb_i[7] - P.bg[1], sb_i[8] - P.bg[2]};
  M3 Jpa, Jpg, Jqg, Jva, Jvg;
  for (int i = 0; i < 9; i++) { Jpa.m[i] = P.dp_dba[i]; Jpg.m[i] = P.dp_dbg[i]; Jqg.m[i] = P.dq_dbg[i]; Jva.m[i] = P.dv_dba[i]; Jvg.m[i] = P.dv_dbg[i]; }
  const double T = P.T;
  const V3 gv{0, 0, g};
  const V3 theta = mul(Jqg, dbg);
  const Q4 gam{P.gamma[0], P.gamma[1], P.gamma[2], P.gamma[3]};
  const Q4 g_hat = qmul(gam, qexp(theta));
  const V3 wp = 0.5 * T * T * gv + Pj.t - Pi.t - T * vi;
  const V3 wv = T * gv + vj - vi;
  const Q4 qij = qmul(qconj(Pi.q), Pj.q);
  const Q4 E = qmul(qconj(g_hat), qij);
  if (r) {
    const V3 a_hat = V3{P.alpha[0], P.alpha[1], P.alpha[2]} + mul(Jpa, dba) + mul(Jpg, dbg);
    const V3 b_hat = V3{P.beta[0], P.beta[1], P.beta[2]} + mul(Jva, dba) + mul(Jvg, dbg);
    const V3 rp = mulT(Ri, wp) - a_hat, rv = mulT(Ri, wv) - b_hat;
    r[0] = rp.x; r[1] = rp.y; r[2] = rp.z; r[3] = 2 * E.x; r[4] = 2 * E.y; r[5] = 2 * E.z; r[6] = rv.x; r[7] = rv.y; r[8] = rv.z;
    for (int k = 0; k < 3; k++) { r[9 + k] = sb_j[3 + k] - sb_i[3 + k]; r[12 + k] = sb_j[6 + k] - sb_i[6 + k]; }
  }
  if (!col) return;
  for (int a = 0; a < 15; a++) col[a] = 0.0;
  const int cb = c / 3, b = c % 3;
  const M3 Rit = transpose(Ri);
  auto put = [&](int row0, const M3& A, double sgn) { for (int a = 0; a < 3; a++) col[row0 + a] = sgn * A.m[3 * a + b]; };
  switch (cb) {
    case 0: {   // dtheta_i
      const M3 GRjT = mul(quat_right_jac(E), transpose(Rj));
      put(0, mul(Rit, skew(wp)), 1.0); put(3, GRjT, -1.0); put(6, mul(Rit, skew(wv)), 1.0);
    } break;
    case 1: put(0, Rit, -1.0); break;                                   // dp_i
    case 2: put(0, Rit, -T); put(6, Rit, -1.0); break;                  // v_i
    case 3: put(0, Jpa, -1.0); put(6, Jva, -1.0); col[9 + b] = -1.0; break;   // ba_i
    case 4: {   // bg_i
      const Q4 Mq = qmul(qconj(gam), qij);
      const V3 mth{-theta.x, -theta.y, -theta.z};
      const M3 dq_bg = mul(mul(quat_right_jac(E), transpose(q2R(Mq))), mul(so3_Jr(mth), Jqg));
      put(0, Jpg, -1.0); put(3, dq_bg, -1.0); put(6, Jvg, -1.0); col[12 + b] = -1.0;
    } break;
    case 5: put(3, mul(quat_right_jac(E), transpose(Rj)), 1.0); break;  // dtheta_j
    case 6: put(0, Rit, 1.0); break;                                    // dp_j
    case 7: put(6, Rit, 1.0); break;                                    // v_j
    case 8: col[9 + b] = 1.0; break;                                    // ba_j
    default: col[12 + b] = 1.0; break;                                  // bg_j
  }
}

}  // namespace bam
