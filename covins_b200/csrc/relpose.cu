// relpose.cu — Optimization::OptimizeRelativePose on the GPU (SURVEY.md §8a O3).
//
// Replaces, behind include/covins_b200.h, the two ceres::Solve calls and the outlier purge of
//   Optimization::OptimizeRelativePose(kf1, kf2, matches1, T12, th2)      optimization_be.cpp:620-831
// a 6-dof problem (one pose block, T12) with up to 2 N reprojection residuals
//   robopt::reprojection::RelativeEuclideanReprError<Camera, Distortion>  kNormal (camera A sees B's point through T12)
//                                                                         kInverse (camera B sees A's point through T12^-1)
// [A: robopt_open is not in the tree; formulas restated, oracle/relpose_oracle.py], CauchyLoss(1.0), dogleg, 5 + 5
// iterations.  The whole call is ONE kernel launch of ONE CTA (the kernel reads its problem record from blockIdx.x, so
// cvb_relpose_batch_dev refines a batch of problems, one CTA each, in the same launch): every thread linearises a strided share of the
// correspondences, the 6x6 normal equations are reduced in shared memory in a fixed order (bit-reproducible), and thread 0
// runs the Ceres trust-region logic (Jacobi scaling, dogleg, accept/reject — the same restatement as ba_engine.cu) on the
// 6x6 system between the passes; the outlier purge and the second solve follow inside the same launch.  The problem is far
// too small for more than one SM (<= 2000 residuals); what matters is that it costs one launch + one 7-double read-back
// instead of ~25 kernel launches and host round trips.
#include <float.h>

#include "ba_math.cuh"
#include "cvb_internal.cuh"

namespace {

using namespace bam;

using RelCam = cvb_relcam;
using RelDev = cvb_relpose_dev;

constexpr int NT = 256, NW = NT / 32, NACC = 28;   // 21 (J^T J lower) + 6 (J^T r) + 1 (cost)

// residual (2) of one block and, optionally, its 2x6 Jacobian w.r.t. [dtheta, dp] of T12.  inverse = kInverse block.
__device__ __forceinline__ bool rel_residual(const double* pose, const RelCam& c, const double* p_other, float u, float v, double sigma,
                                             bool inverse, double r[2], double J[12], bool want_jac) {
  const Q4 q{pose[0], pose[1], pose[2], pose[3]};
  const M3 R = q2R(q);
  const V3 t{pose[4], pose[5], pose[6]}, po{p_other[0], p_other[1], p_other[2]};
  V3 pc;
  M3 dth;                       // d pc / d dtheta
  if (!inverse) {               // pc = R p + t:  Exp(dth) R p ~ R p + dth x (R p)  →  -[R p]x
    const V3 rp = mul(R, po);
    pc = rp + t;
    dth = skew(rp);
    for (int i = 0; i < 9; i++) dth.m[i] = -dth.m[i];
  } else {                      // pc = R^T (p - t):  R^T Exp(-dth) w ~ R^T w + R^T [w]x dth
    const V3 w = po - t;
    pc = mulT(R, w);
    dth = mul(transpose(R), skew(w));
  }
  const CamModel cm{c.cam, c.dm, c.xi};
  double x, y, N[6];
  if (!cam_normalise(cm, pc, &x, &y, N, want_jac)) {
    r[0] = r[1] = 0.0;
    if (want_jac) for (int i = 0; i < 12; i++) J[i] = 0.0;
    return false;
  }
  double xd, yd, D[4];
  cam_distort(cm, c.dist, x, y, &xd, &yd, D, want_jac);
  const double is = 1.0 / sigma;
  r[0] = (c.intr[0] * xd + c.intr[2] - (double)u) * is;
  r[1] = (c.intr[1] * yd + c.intr[3] - (double)v) * is;
  if (!want_jac) return true;
  const double fx = c.intr[0] * is, fy = c.intr[1] * is;
  const double A[6] = {fx * (D[0] * N[0] + D[1] * N[3]), fx * (D[0] * N[1] + D[1] * N[4]), fx * (D[0] * N[2] + D[1] * N[5]),
                       fy * (D[2] * N[0] + D[3] * N[3]), fy * (D[2] * N[1] + D[3] * N[4]), fy * (D[2] * N[2] + D[3] * N[5])};
  const M3 Rt = transpose(R);
  for (int a = 0; a < 2; a++) {
    for (int b = 0; b < 3; b++) {
      J[6 * a + b] = A[3 * a] * dth.m[b] + A[3 * a + 1] * dth.m[3 + b] + A[3 * a + 2] * dth.m[6 + b];
      // d pc / d dp: I (normal), -R^T (inverse)
      J[6 * a + 3 + b] = inverse ? -(A[3 * a] * Rt.m[b] + A[3 * a + 1] * Rt.m[3 + b] + A[3 * a + 2] * Rt.m[6 + b]) : A[3 * a + b];
    }
  }
  return true;
}

// sum over the active correspondences of this thread's share; acc[0..20] lower J^T J, [21..26] J^T r, [27] cost
__device__ void accumulate(const RelDev& P, const uint8_t* removed, const double* pose, bool jac, double acc[NACC]) {
  for (int i = 0; i < NACC; i++) acc[i] = 0.0;
  for (int i = threadIdx.x; i < P.n; i += NT) {
    if (removed[i]) continue;
    for (int blk = 0; blk < 2; blk++) {
      double r[2], J[12];
      rel_residual(pose, blk ? P.camB : P.camA, blk ? P.pA + 3 * (size_t)i : P.pB + 3 * (size_t)i, blk ? P.kpB[2 * i] : P.kpA[2 * i],
                   blk ? P.kpB[2 * i + 1] : P.kpA[2 * i + 1], blk ? P.sB[i] : P.sA[i], blk == 1, r, J, jac);
      double sc, c;
      cauchy(r[0] * r[0] + r[1] * r[1], 1.0, &sc, &c);
      acc[27] += c;
      if (!jac) continue;
      const double r0 = r[0] * sc, r1 = r[1] * sc;
      int idx = 0;
      for (int a = 0; a < 6; a++) {
        const double ja0 = J[a] * sc, ja1 = J[6 + a] * sc;
        for (int b = 0; b <= a; b++) acc[idx++] += ja0 * (J[b] * sc) + ja1 * (J[6 + b] * sc);
        acc[21 + a] += ja0 * r0 + ja1 * r1;
      }
    }
  }
}

// fixed-order block reduction: lanes by shuffle, warps summed by thread 0 in warp order → out[NACC] (shared)
__device__ void block_reduce(double acc[NACC], double (*wsum)[NACC], double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = 0; i < NACC; i++) {
    double v = acc[i];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) wsum[warp][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < NACC) {
    double s = 0.0;
    for (int w = 0; w < NW; w++) s += wsum[w][threadIdx.x];
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

// 6x6 SPD solve by Cholesky (A lower-packed row-major 6x6 full array); false if not positive definite
__device__ bool chol6_solve(const double* A, const double* b, double* x) {
  double L[36];
  for (int j = 0; j < 6; j++) {
    double d = A[6 * j + j];
    for (int k = 0; k < j; k++) d -= L[6 * j + k] * L[6 * j + k];
    if (!(d > 0.0)) return false;
    d = sqrt(d);
    L[6 * j + j] = d;
    for (int i = j + 1; i < 6; i++) {
      double s = A[6 * i + j];
      for (int k = 0; k < j; k++) s -= L[6 * i + k] * L[6 * j + k];
      L[6 * i + j] = s / d;
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) { double s = b[i]; for (int k = 0; k < i; k++) s -= L[6 * i + k] * y[k]; y[i] = s / L[6 * i + i]; }
  for (int i = 5; i >= 0; i--) { double s = y[i]; for (int k = i + 1; k < 6; k++) s -= L[6 * k + i] * x[k]; x[i] = s / L[6 * i + i]; }
  for (int i = 0; i < 6; i++) if (!isfinite(x[i])) return false;
  return true;
}

struct TrState {   // trust-region state shared by the CTA (thread 0 writes)
  double pose[7], cand[7], scale[6], H[36], g[6], gn[6], grad[6], diag[6];
  double cost, ccost, radius, mu, alpha, gn2, gg, g_gn, x_norm, dogleg_norm, model_change;
  int reuse, invalid_run, iterations, done, have_scale, phase;   // phase: what the CTA does next
  double hist[16];
  int n_hist;
};

// one ceres::Solve (max_iter trust-region iterations) on the active correspondences
__device__ void solve(const RelDev& P, const uint8_t* removed, TrState& S, double (*wsum)[NACC], double* red, int max_iter) {
  const int tid = threadIdx.x;
  double acc[NACC];
  if (tid == 0) { S.radius = 1e4; S.mu = 1e-8; S.reuse = 0; S.invalid_run = 0; S.iterations = 0; S.done = 0; S.have_scale = 0; }
  __syncthreads();
  // iteration 0: linearise (unscaled), fix the Jacobi scaling at x0
  accumulate(P, removed, S.pose, true, acc);
  block_reduce(acc, wsum, red);
  if (tid == 0) {
    int idx = 0;
    for (int a = 0; a < 6; a++) for (int b = 0; b <= a; b++) { S.H[6 * a + b] = red[idx]; S.H[6 * b + a] = red[idx]; idx++; }
    for (int a = 0; a < 6; a++) { S.g[a] = red[21 + a]; S.scale[a] = 1.0 / (1.0 + sqrt(S.H[7 * a])); }
    S.cost = red[27];
    S.hist[S.n_hist < 16 ? S.n_hist++ : 15] = S.cost;
    double xn = 0.0;
    for (int c = 0; c < 7; c++) xn += S.pose[c] * S.pose[c];
    S.x_norm = sqrt(xn);
    double gmax = 0.0;
    for (int a = 0; a < 6; a++) gmax = fmax(gmax, fabs(S.g[a]));
    if (gmax <= 1e-10) S.done = 1;   // gradient tolerance at the start point
  }
  __syncthreads();
  while (!S.done && S.iterations < max_iter) {
    if (tid == 0) {
      S.iterations++;
      bool solver_ok = true;
      if (!S.reuse) {
        S.reuse = 1;
        double Hs[36], gs[6];
        for (int a = 0; a < 6; a++) { gs[a] = S.g[a] * S.scale[a]; for (int b = 0; b < 6; b++) Hs[6 * a + b] = S.H[6 * a + b] * S.scale[a] * S.scale[b]; }
        double sg[6];
        for (int a = 0; a < 6; a++) {
          S.diag[a] = sqrt(fmin(fmax(Hs[7 * a], 1e-6), 1e32));
          S.grad[a] = gs[a] / S.diag[a];
          sg[a] = S.grad[a] / S.diag[a];
        }
        double JgJg = 0.0, gg = 0.0;
        for (int a = 0; a < 6; a++) { gg += S.grad[a] * S.grad[a]; for (int b = 0; b < 6; b++) JgJg += sg[a] * Hs[6 * a + b] * sg[b]; }
        S.gg = gg; S.alpha = gg / JgJg;
        bool solved = false;
        while (S.mu < 1.0) {
          double Ad[36], x[6];
          for (int i = 0; i < 36; i++) Ad[i] = Hs[i];
          for (int a = 0; a < 6; a++) Ad[7 * a] += S.mu * S.diag[a] * S.diag[a];
          if (!chol6_solve(Ad, gs, x)) { S.mu *= 10.0; continue; }
          double gn2 = 0.0, ggn = 0.0;
          for (int a = 0; a < 6; a++) { S.gn[a] = -x[a] * S.diag[a]; gn2 += S.gn[a] * S.gn[a]; ggn += S.grad[a] * S.gn[a]; }
          S.gn2 = gn2; S.g_gn = ggn;
          solved = true;
          break;
        }
        solver_ok = solved;
      }
      S.phase = 0;
      if (solver_ok) {
        const double gn_norm = sqrt(S.gn2), g_norm = sqrt(S.gg);
        double ca, cb;
        if (gn_norm <= S.radius) { ca = 0.0; cb = 1.0; }
        else if (g_norm * S.alpha >= S.radius) { ca = -(S.radius / g_norm); cb = 0.0; }
        else {
          const double b_dot_a = -S.alpha * S.g_gn, a2 = (S.alpha * g_norm) * (S.alpha * g_norm), bma2 = a2 - 2.0 * b_dot_a + gn_norm * gn_norm,
                       c = b_dot_a - a2, d = sqrt(c * c + bma2 * (S.radius * S.radius - a2));
          const double beta = c <= 0 ? (d - c) / bma2 : (S.radius * S.radius - a2) / (d + c);
          ca = -S.alpha * (1.0 - beta); cb = beta;
        }
        double step[6], dl2 = 0.0;
        for (int a = 0; a < 6; a++) { const double dl = ca * S.grad[a] + cb * S.gn[a]; dl2 += dl * dl; step[a] = dl / S.diag[a]; }
        S.dogleg_norm = sqrt(dl2);
        double jvr = 0.0, jv2 = 0.0;   // (J step).r and |J step|^2 in the Jacobi-scaled space
        for (int a = 0; a < 6; a++) {
          jvr += step[a] * S.g[a] * S.scale[a];
          for (int b = 0; b < 6; b++) jv2 += step[a] * S.H[6 * a + b] * S.scale[a] * S.scale[b] * step[b];
        }
        S.model_change = -(jvr + 0.5 * jv2);
        if (S.model_change > 0.0) {
          double delta[6];
          for (int a = 0; a < 6; a++) delta[a] = step[a] * S.scale[a];
          pose_plus(S.pose, delta, S.cand);
          S.phase = 1;   // evaluate the candidate
        }
      }
      if (S.phase == 0) {   // invalid step (solver failure or non-positive model decrease)
        S.invalid_run++;
        S.hist[S.n_hist < 16 ? S.n_hist++ : 15] = S.cost;
        if (S.invalid_run > 5) S.done = 1;
        S.mu *= 10.0; S.reuse = 0;
      }
    }
    __syncthreads();
    if (S.phase == 1) {
      accumulate(P, removed, S.cand, false, acc);
      block_reduce(acc, wsum, red);
      if (tid == 0) {
        S.invalid_run = 0;
        S.ccost = red[27];
        double st2 = 0.0, cx2 = 0.0;
        for (int c = 0; c < 7; c++) { const double d = S.cand[c] - S.pose[c]; st2 += d * d; cx2 += S.cand[c] * S.cand[c]; }
        S.phase = 0;
        if (sqrt(st2) <= 1e-8 * (S.x_norm + 1e-8)) S.done = 1;                          // parameter tolerance
        else if (fabs(S.cost - S.ccost) <= 1e-6 * S.cost) S.done = 1;                  // function tolerance
        else {
          const double rho = (S.cost - S.ccost) / S.model_change;
          if (rho > 1e-3) {
            for (int c = 0; c < 7; c++) S.pose[c] = S.cand[c];
            S.cost = S.ccost; S.x_norm = sqrt(cx2);
            if (rho < 0.25) S.radius *= 0.5;
            if (rho > 0.75) S.radius = fmax(S.radius, 3.0 * S.dogleg_norm);
            S.mu = fmax(1e-8, 2.0 * S.mu / 10.0);
            S.reuse = 0;
            S.phase = 2;   // relinearise at the accepted state
          } else {
            S.radius *= 0.5; S.reuse = 1;
          }
          S.hist[S.n_hist < 16 ? S.n_hist++ : 15] = S.cost;
        }
      }
      __syncthreads();
      if (S.phase == 2) {
        accumulate(P, removed, S.pose, true, acc);
        block_reduce(acc, wsum, red);
        if (tid == 0) {
          int idx = 0;
          for (int a = 0; a < 6; a++) for (int b = 0; b <= a; b++) { S.H[6 * a + b] = red[idx]; S.H[6 * b + a] = red[idx]; idx++; }
          for (int a = 0; a < 6; a++) S.g[a] = red[21 + a];
        }
        __syncthreads();
      }
    }
  }
  __syncthreads();
}

// problem blockIdx.x of probs; out: pose[7], n_inliers, it1, it2, n_hist, hist[16]
__global__ void __launch_bounds__(NT, 1) relpose_kernel(const RelDev* __restrict__ probs, double th_outlier) {
  __shared__ TrState S;
  __shared__ double wsum[NW][NACC];
  __shared__ double red[NACC];
  __shared__ int n_bad;
  const RelDev& P = probs[blockIdx.x];   // read-only for the whole launch
  const int tid = threadIdx.x;
  const double* __restrict__ pose_in = P.pose_in;
  uint8_t* __restrict__ removed = P.removed;
  double* __restrict__ out = P.out;
  if (P.n < 12) {   // cvb_optimize_relative_pose's early result: fewer than 12 correspondences can never pass :821
    for (int i = tid; i < P.n; i += NT) removed[i] = 0;
    for (int i = tid; i < CVB_RELPOSE_OUT; i += NT) out[i] = i < 7 ? pose_in[i] : 0.0;
    return;
  }
  if (tid == 0) { for (int c = 0; c < 7; c++) S.pose[c] = pose_in[c]; S.n_hist = 0; n_bad = 0; }
  for (int i = tid; i < P.n; i += NT) removed[i] = 0;
  __syncthreads();
  solve(P, removed, S, wsum, red, 5);                                              // :787-794
  const int it1 = S.iterations;
  // outlier purge on the loss-corrected residual norms of either block (:798-818)
  int bad = 0;
  for (int i = tid; i < P.n; i += NT) {
    double nrm[2];
    for (int blk = 0; blk < 2; blk++) {
      double r[2];
      rel_residual(S.pose, blk ? P.camB : P.camA, blk ? P.pA + 3 * (size_t)i : P.pB + 3 * (size_t)i, blk ? P.kpB[2 * i] : P.kpA[2 * i],
                   blk ? P.kpB[2 * i + 1] : P.kpA[2 * i + 1], blk ? P.sB[i] : P.sA[i], blk == 1, r, nullptr, false);
      const double s = r[0] * r[0] + r[1] * r[1];
      double sc, c;
      cauchy(s, 1.0, &sc, &c);
      nrm[blk] = sqrt(s) * sc;
    }
    if (nrm[0] > th_outlier || nrm[1] > th_outlier) { removed[i] = 1; bad++; }
  }
  for (int o = 16; o > 0; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
  if ((tid & 31) == 0 && bad) atomicAdd(&n_bad, bad);
  __syncthreads();
  const int left = P.n - n_bad;
  int it2 = 0;
  if (left >= 12) {                                                                 // :821-823
    solve(P, removed, S, wsum, red, 5);
    it2 = S.iterations;
  }
  if (tid == 0) {
    if (left >= 12) {
      const Q4 q = qnormalized(Q4{S.pose[0], S.pose[1], S.pose[2], S.pose[3]});     // Utils::Ceres2Transform (utils_base.cpp:38-40)
      out[0] = q.x; out[1] = q.y; out[2] = q.z; out[3] = q.w;
      for (int c = 4; c < 7; c++) out[c] = S.pose[c];
      out[7] = (double)left;
    } else {
      for (int c = 0; c < 7; c++) out[c] = pose_in[c];                             // T12 untouched, return 0
      out[7] = 0.0;
    }
    out[8] = (double)it1; out[9] = (double)it2; out[10] = (double)S.n_hist;
    for (int i = 0; i < 16; i++) out[11 + i] = i < S.n_hist ? S.hist[i] : 0.0;
  }
}

}  // namespace

extern "C" int cvb_optimize_relative_pose(cvb_ctx* ctx, const cvb_relpose_problem* p, double th_outlier_align, double* T12_out,
                                          uint8_t* removed, int32_t* n_inliers, double* info /* nullable, 19 doubles */) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, p && T12_out && n_inliers && p->n >= 0, "optimize_relative_pose: bad arguments");
  CVB_REQUIRE(ctx, p->n == 0 || (p->pA_c && p->pB_c && p->kpA && p->kpB && p->sigmaA && p->sigmaB), "optimize_relative_pose: null arrays");
  for (int s = 0; s < 2; s++) {
    const int cam = s ? p->cam_model_B : p->cam_model_A, dm = s ? p->dist_model_B : p->dist_model_A;
    if (cam < 0 || cam > 1) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown projection type.");       // :705-707
    if (dm < 0 || dm > 2) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown distortion type.");          // :684-688
  }
  const int n = p->n;
  if (n < 12) {   // fewer than 12 correspondences can never pass :821 — same outcome without touching the GPU
    for (int c = 0; c < 7; c++) T12_out[c] = p->T12[c];
    *n_inliers = 0;
    if (removed) for (int i = 0; i < n; i++) removed[i] = 0;
    if (info) for (int i = 0; i < 19; i++) info[i] = 0.0;
    return CVB_OK;
  }
  cvb_block B(ctx, ctx->stream);
  RelDev D{};
  RelDev* d_rec;
  B.in(D.pA, p->pA_c, (size_t)n * 3); B.in(D.pB, p->pB_c, (size_t)n * 3); B.in(D.sA, p->sigmaA, n); B.in(D.sB, p->sigmaB, n);
  B.in(D.kpA, p->kpA, (size_t)n * 2); B.in(D.kpB, p->kpB, (size_t)n * 2); B.in(D.pose_in, p->T12, 7); B.in(d_rec, nullptr, 1);
  B.out_host(D.out, CVB_RELPOSE_OUT); B.out(D.removed, removed, n);
  if (const int rc = B.place()) return rc;
  D.n = n;
  for (int c = 0; c < 4; c++) { D.camA.intr[c] = p->intrA[c]; D.camA.dist[c] = p->distA[c]; D.camB.intr[c] = p->intrB[c]; D.camB.dist[c] = p->distB[c]; }
  D.camA.cam = p->cam_model_A; D.camA.dm = p->dist_model_A; D.camA.xi = p->xiA;
  D.camB.cam = p->cam_model_B; D.camB.dm = p->dist_model_B; D.camB.xi = p->xiB;
  *B.host(d_rec) = D;
  if (const int rc = B.upload()) return rc;
  relpose_kernel<<<1, NT, 0, ctx->stream>>>(d_rec, th_outlier_align);
  CVB_CHECK_LAUNCH(ctx);
  if (const int rc = B.download()) return rc;
  const double* out = B.host(D.out);
  for (int c = 0; c < 7; c++) T12_out[c] = out[c];
  *n_inliers = (int32_t)out[7];
  if (info) for (int i = 0; i < 19; i++) info[i] = out[8 + i];
  return CVB_OK;
}

int cvb_relpose_batch_dev(cvb_ctx* ctx, const cvb_relpose_dev* d_probs, int n_prob, double th_outlier_align) {
  if (n_prob == 0) return CVB_OK;
  relpose_kernel<<<n_prob, NT, 0, ctx->stream>>>(d_probs, th_outlier_align);
  CVB_CHECK_LAUNCH(ctx);
  return CVB_OK;
}
