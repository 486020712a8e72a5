// pgo.cu — cvb_pgo: Optimization::PoseGraphOptimization (optimization_be.cpp:833-1086) on a flattened map in one call
// (include/covins_b200.h states the rule).
//
// The host checks the input and builds the edge topology: which pairs, in which order, with which weight class.  That part
// is a walk over predecessor links and a de-duplication, and the engine's tile plan needs it on the host anyway.  Everything
// that is arithmetic runs on the device, through the one implementation of the conversions in include/covins_b200_pose.h:
//   K17a pgo_edges_kernel, one thread per keyframe and per edge: the start poses as pose7 and each edge's measurement and
//        sqrt_info, written straight into the solver's arrays (cvb_ba_solve_dev_edges);
//   the solve: the bundle adjustment engine with PGO's options;
//   K17b pgo_writeback_kernel, a grid-stride over K + L: pose7_to_transform of the solved poses, the velocity rotation, and
//        the landmark re-anchoring and erase flags, reading the solved poses where the solver left them.
// All outputs come back in one download.
#include <algorithm>
#include <cmath>
#include <unordered_set>
#include <vector>

#include "../../include/covins_b200_pose.h"
#include "cvb_internal.cuh"

namespace {

constexpr int PGO_THREADS = 256;

struct PgoWeights {
  double diag[3][6];   // S1, S23, S45 diagonals (the matrices are diagonal)
};

enum : int32_t { EDGE_LOOP = 0, EDGE_S1 = 1, EDGE_S23 = 2, EDGE_S45 = 3 };

__device__ __forceinline__ void load16(const double* __restrict__ src, double* T) {
  const double2* s = reinterpret_cast<const double2*>(src);
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const double2 v = s[j];
    T[2 * j] = v.x;
    T[2 * j + 1] = v.y;
  }
}

// kept out of line: its four 6x6 work arrays would otherwise be unrolled into the kernel's registers for the few loop edges
__device__ __noinline__ bool loop_sqrt_info(const double* cov, double* S) { return cvb_pose::sqrt_info_from_cov(cov, S); }

// K17a: item i < K is keyframe i's start pose, item K + e is edge e.  Loops come first in the edge list, so loop e is edge e.
__global__ void __launch_bounds__(PGO_THREADS) pgo_edges_kernel(const __grid_constant__ PgoWeights W, int K, int n_edge,
                                                                const double* __restrict__ T_init, const double* __restrict__ T_vio,
                                                                const int32_t* __restrict__ einfo, const double* __restrict__ loop_q,
                                                                const double* __restrict__ loop_t, const double* __restrict__ loop_cov,
                                                                double* __restrict__ pose, double* __restrict__ pose0,
                                                                double* __restrict__ eq, double* __restrict__ et, double* __restrict__ eS) {
  const int64_t n = (int64_t)K + n_edge;
  for (int64_t i = (int64_t)blockIdx.x * PGO_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * PGO_THREADS) {
    double T[16], p7[7];
    if (i < K) {
      load16(T_init + 16 * i, T);
      cvb_pose::transform_to_pose7(T, p7);
#pragma unroll
      for (int c = 0; c < 7; c++) {
        pose[7 * i + c] = p7[c];
        pose0[7 * i + c] = p7[c];
      }
      continue;
    }
    const int64_t e = i - K;
    const int a = einfo[3 * e], b = einfo[3 * e + 1], kind = einfo[3 * e + 2];
    double* S = eS + 36 * e;
    bool diag = true;
    if (kind == EDGE_LOOP) {
#pragma unroll
      for (int c = 0; c < 4; c++) p7[c] = loop_q[4 * e + c];
#pragma unroll
      for (int c = 0; c < 3; c++) p7[4 + c] = loop_t[3 * e + c];
      if (loop_cov) {
        loop_sqrt_info(loop_cov + 36 * e, S);   // positive definite: the host checked it with the same function
        diag = false;
      }
    } else {
      double Ta[16], R[16];
      load16(T_vio + 16 * (int64_t)a, Ta);
      load16(T_vio + 16 * (int64_t)b, T);
      cvb_pose::rel_transform(Ta, T, R);
      cvb_pose::transform_to_pose7(R, p7);
    }
    if (diag) {
      const int w = kind == EDGE_LOOP ? 0 : kind - 1;
      for (int m = 0; m < 36; m++) S[m] = (m % 7 == 0) ? W.diag[w][m / 7] : 0.0;
    }
#pragma unroll
    for (int c = 0; c < 4; c++) eq[4 * e + c] = p7[c];
#pragma unroll
    for (int c = 0; c < 3; c++) et[3 * e + c] = p7[4 + c];
  }
}

// K17b: item i < K is keyframe i, item K + l is landmark l.  A landmark recomputes its reference keyframe's Tc with the same
// function, so it never reads what another thread of this launch writes.
__global__ void __launch_bounds__(PGO_THREADS) pgo_writeback_kernel(int K, int L, const double* __restrict__ pose, const double* __restrict__ T_ws,
                                                                    const double* __restrict__ vel, const double* __restrict__ lm,
                                                                    const int32_t* __restrict__ lm_ref, const uint8_t* __restrict__ has_obs,
                                                                    double* __restrict__ T_out, double* __restrict__ pose_out,
                                                                    double* __restrict__ vel_out, double* __restrict__ lm_out,
                                                                    uint8_t* __restrict__ erase) {
  using cvb_pose::add;
  using cvb_pose::mul;
  using cvb_pose::sub;
  const int64_t n = (int64_t)K + L;
  for (int64_t i = (int64_t)blockIdx.x * PGO_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * PGO_THREADS) {
    double p7[7], Tc[16], Tu[16];
    if (i < K) {
#pragma unroll
      for (int c = 0; c < 7; c++) p7[c] = pose[7 * i + c];
      cvb_pose::pose7_to_transform(p7, Tc);
      double2* dst = reinterpret_cast<double2*>(T_out + 16 * i);
#pragma unroll
      for (int j = 0; j < 8; j++) dst[j] = make_double2(Tc[2 * j], Tc[2 * j + 1]);
#pragma unroll
      for (int c = 0; c < 7; c++) pose_out[7 * i + c] = p7[c];
      if (vel) {   // R_corr R_uncorr^T v (optimization_be.cpp:1046-1047)
        load16(T_ws + 16 * i, Tu);
        const double v[3] = {vel[3 * i], vel[3 * i + 1], vel[3 * i + 2]};
#pragma unroll
        for (int r = 0; r < 3; r++) {
          double s = 0;
#pragma unroll
          for (int c = 0; c < 3; c++) {
            double m = 0;
#pragma unroll
            for (int x = 0; x < 3; x++) m = add(m, mul(Tc[4 * r + x], Tu[4 * c + x]));
            s = add(s, mul(m, v[c]));
          }
          vel_out[3 * i + r] = s;
        }
      }
      continue;
    }
    const int64_t l = i - K;
    const int ref = lm_ref[l];
    const double pw[3] = {lm[3 * l], lm[3 * l + 1], lm[3 * l + 2]};
    if (ref < 0) {   // -1: no reference keyframe (erased when observed), -2: reference not among the keyframes (erased)
#pragma unroll
      for (int c = 0; c < 3; c++) lm_out[3 * l + c] = pw[c];
      erase[l] = (ref == -2 || has_obs[l]) ? 1 : 0;
      continue;
    }
    load16(T_ws + 16 * (int64_t)ref, Tu);
#pragma unroll
    for (int c = 0; c < 7; c++) p7[c] = pose[7 * (int64_t)ref + c];
    cvb_pose::pose7_to_transform(p7, Tc);
    double ps[3];
#pragma unroll
    for (int r = 0; r < 3; r++) {
      double s = 0;
#pragma unroll
      for (int c = 0; c < 3; c++) s = add(s, mul(Tu[4 * c + r], sub(pw[c], Tu[4 * c + 3])));
      ps[r] = s;
    }
#pragma unroll
    for (int r = 0; r < 3; r++)
      lm_out[3 * l + r] = add(add(add(mul(Tc[4 * r], ps[0]), mul(Tc[4 * r + 1], ps[1])), mul(Tc[4 * r + 2], ps[2])), Tc[4 * r + 3]);
    erase[l] = 0;
  }
}

bool all_finite(const double* a, size_t n) {
  for (size_t i = 0; i < n; i++)
    if (!std::isfinite(a[i])) return false;
  return true;
}

}  // namespace

extern "C" int cvb_pgo(cvb_ctx* ctx, const cvb_pgo_problem* p, const cvb_pgo_options* o, cvb_pgo_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, p && o && r, "cvb_pgo: problem, options and result are required");
  r->bad_loop = -1;
  r->n_edge = 0;
  const int K = p->K, NL = p->n_loop, L = p->L;
  CVB_REQUIRE(ctx, K >= 1, "cvb_pgo: the problem has no keyframes (K %d)", K);
  CVB_REQUIRE(ctx, NL >= 0 && L >= 0, "cvb_pgo: negative size (n_loop %d, L %d)", NL, L);
  CVB_REQUIRE(ctx, p->T_ws && p->T_ws_vio && p->kf_pred && p->kf_succ && p->kf_id && p->pose_const,
              "cvb_pgo: T_ws, T_ws_vio, kf_pred, kf_succ, kf_id and pose_const are required");
  CVB_REQUIRE(ctx, NL == 0 || (p->loop_i && p->loop_j && p->loop_q && p->loop_t), "cvb_pgo: loop_i, loop_j, loop_q and loop_t are required");
  CVB_REQUIRE(ctx, L == 0 || (p->lm_pos && p->lm_ref && p->lm_has_obs), "cvb_pgo: lm_pos, lm_ref and lm_has_obs are required");
  CVB_REQUIRE(ctx, r->T_ws_out && (!p->velocity || r->velocity_out) && (L == 0 || (r->lm_out && r->lm_erase)),
              "cvb_pgo: T_ws_out, velocity_out (with velocities) and lm_out / lm_erase (with landmarks) are required");
  CVB_REQUIRE(ctx, o->iteration_limit >= 0, "cvb_pgo: iteration_limit %d < 0", o->iteration_limit);
  CVB_REQUIRE(ctx, all_finite(p->T_ws, 16 * (size_t)K) && all_finite(p->T_ws_vio, 16 * (size_t)K) &&
                       (!p->T_ws_init || all_finite(p->T_ws_init, 16 * (size_t)K)),
              "cvb_pgo: T_ws, T_ws_init and T_ws_vio must be finite");
  for (int k = 0; k < K; k++)
    CVB_REQUIRE(ctx, p->kf_pred[k] >= -2 && p->kf_pred[k] < K && p->kf_succ[k] >= -2 && p->kf_succ[k] < K,
                "cvb_pgo: keyframe %d: kf_pred %d / kf_succ %d outside [-2, K)", k, p->kf_pred[k], p->kf_succ[k]);
  for (int l = 0; l < L; l++)
    CVB_REQUIRE(ctx, p->lm_ref[l] >= -2 && p->lm_ref[l] < K, "cvb_pgo: landmark %d: lm_ref %d outside [-2, K)", l, p->lm_ref[l]);

  // ---- edge topology, in the order of the rule ----
  std::vector<int32_t> einfo;   // [n_edge][3] = i, j, kind
  std::vector<uint8_t> robust;
  for (int l = 0; l < NL; l++) {   // 1. loops (:910-943)
    if (p->loop_cov) {
      double S[36];
      if (!cvb_pose::sqrt_info_from_cov(p->loop_cov + 36 * (size_t)l, S)) {
        r->bad_loop = l;
        return cvb_fail(ctx, CVB_ERR_INVALID, "cvb_pgo: loop %d: covariance is not positive definite", l);
      }
    }
    const int a = p->loop_i[l], b = p->loop_j[l];
    CVB_REQUIRE(ctx, a >= 0 && a < K && b >= 0 && b < K && a != b, "cvb_pgo: loop %d: keyframes (%d, %d) invalid", l, a, b);
    einfo.insert(einfo.end(), {a, b, EDGE_LOOP});
    robust.push_back(o->use_robust_loss ? 1 : 0);
  }
  std::unordered_set<int64_t> inserted;   // ordered pairs of successor and neighbour edges (:907)
  inserted.reserve((size_t)K * 6);
  auto push = [&](int a, int b, int kind) {
    if (!inserted.insert((int64_t)a * K + b).second) return;
    einfo.insert(einfo.end(), {a, b, kind});
    robust.push_back(0);
  };
  for (int k = 0; k < K; k++) {   // 2. successors (:947-972)
    const int s = p->kf_succ[k];
    CVB_REQUIRE(ctx, s != -2, "cvb_pgo: keyframe %d: its successor is not among the keyframes", k);
    if (s >= 0) push(k, s, EDGE_S1);
  }
  if (o->use_nbr_kfs) {   // 3. neighbours (:976-1021)
    static const int kind_of_step[6] = {0, EDGE_S1, EDGE_S23, EDGE_S23, EDGE_S45, EDGE_S45};
    for (int k = 0; k < K; k++) {
      int t = k, n = 0;
      int conn[5];
      for (int j = 1; j < 6; ++j)
        if (p->kf_id[k] - j > 0) {
          t = p->kf_pred[t];
          CVB_REQUIRE(ctx, t >= 0, "cvb_pgo: keyframe %d: neighbour %d is %s", k, j,
                      t == -1 ? "absent (no predecessor)" : "not among the keyframes");
          conn[n++] = t;
        }
      for (int c = 0; c < n; c++) push(k, conn[c], kind_of_step[c + 1]);
    }
  }
  const int n_edge = (int)robust.size();
  r->n_edge = n_edge;
  std::vector<int32_t> ei(n_edge), ej(n_edge);
  for (int e = 0; e < n_edge; e++) {
    ei[e] = einfo[3 * (size_t)e];
    ej[e] = einfo[3 * (size_t)e + 1];
  }
  PgoWeights W;
  for (int d = 0; d < 6; d++) {   // :896-903
    W.diag[0][d] = (d < 3 ? o->wt_kf_r : o->wt_kf_t) * o->wt_kf_n1;
    W.diag[1][d] = W.diag[0][d] / o->wt_kf_n23;
    W.diag[2][d] = W.diag[0][d] / o->wt_kf_n45;
  }

  // ---- device block: inputs, then the outputs, the optional ones last ----
  cudaStream_t st = ctx->stream;
  cvb_block B(ctx, st);
  const double *d_T_ws, *d_T_init = nullptr, *d_T_vio, *d_lq = nullptr, *d_lt = nullptr, *d_lcov = nullptr, *d_vel = nullptr, *d_lm;
  const int32_t *d_einfo, *d_lm_ref;
  const uint8_t* d_has_obs;
  double *d_T_out, *d_lm_out, *d_vel_out, *d_pose_out;
  uint8_t* d_erase;
  B.in(d_T_ws, p->T_ws, 16 * (size_t)K);
  if (p->T_ws_init) B.in(d_T_init, p->T_ws_init, 16 * (size_t)K);
  B.in(d_T_vio, p->T_ws_vio, 16 * (size_t)K);
  B.in(d_einfo, einfo.data(), einfo.size());
  if (NL) {
    B.in(d_lq, p->loop_q, 4 * (size_t)NL);
    B.in(d_lt, p->loop_t, 3 * (size_t)NL);
    if (p->loop_cov) B.in(d_lcov, p->loop_cov, 36 * (size_t)NL);
  }
  if (p->velocity) B.in(d_vel, p->velocity, 3 * (size_t)K);
  B.in(d_lm, p->lm_pos, 3 * (size_t)L);
  B.in(d_lm_ref, p->lm_ref, L);
  B.in(d_has_obs, p->lm_has_obs, L);
  B.out(d_T_out, r->T_ws_out, 16 * (size_t)K);
  B.out(d_lm_out, r->lm_out, 3 * (size_t)L);
  B.out(d_erase, r->lm_erase, L);
  B.out(d_vel_out, p->velocity ? r->velocity_out : nullptr, 3 * (size_t)K);
  B.out(d_pose_out, r->ba.pose, 7 * (size_t)K);
  if (const int rc = B.place()) return rc;
  if (const int rc = B.upload()) return rc;
  if (!d_T_init) d_T_init = d_T_ws;

  // ---- the solve's problem: topology and constants on the host, start poses and measurements from K17a ----
  std::vector<int32_t> lm_obs_ptr(1, 0);
  const double extr[7] = {0, 0, 0, 1, 0, 0, 0}, intr[4] = {1, 1, 1, 1}, dist[4] = {0, 0, 0, 0};
  cvb_ba_problem bp{};
  bp.K = K; bp.L = 0; bp.n_obs = 0; bp.n_imu = 0; bp.n_edge = n_edge; bp.n_cam = 1;
  bp.pose_const = p->pose_const; bp.extr = extr; bp.intr = intr; bp.dist = dist; bp.lm_obs_ptr = lm_obs_ptr.data();
  bp.edge_i = ei.data(); bp.edge_j = ej.data(); bp.edge_robust = robust.data();
  cvb_ba_options bo{};
  bo.max_iterations = o->iteration_limit;
  bo.visual_only = 1;
  bo.cauchy_reproj = 0.0;
  bo.cauchy_edge = o->robust_loss_th;
  bo.rank = 0;
  bo.world = 1;
  cvb_ba_result br = r->ba;
  br.pose = nullptr; br.speedbias = nullptr; br.lm = nullptr; br.lm_owner = nullptr;
  const int64_t n_a = (int64_t)K + n_edge, n_b = (int64_t)K + L;
  const auto grid = [ctx](int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + PGO_THREADS - 1) / PGO_THREADS, (int64_t)ctx->sm_count * 8)); };
  const cvb_dev_edges_fill fill = [&](double* pose, double* pose0, double* eq, double* et, double* eS) {
    pgo_edges_kernel<<<grid(n_a), PGO_THREADS, 0, st>>>(W, K, n_edge, d_T_init, d_T_vio, d_einfo, d_lq, d_lt, d_lcov, pose, pose0, eq, et, eS);
    CVB_CHECK_LAUNCH(ctx);
    return (int)CVB_OK;
  };
  const auto finish = [&](const double* d_pose) {
    pgo_writeback_kernel<<<grid(n_b), PGO_THREADS, 0, st>>>(K, L, d_pose, d_T_ws, d_vel, d_lm, d_lm_ref, d_has_obs, d_T_out, d_pose_out,
                                                            d_vel_out, d_lm_out, d_erase);
    CVB_CHECK_LAUNCH(ctx);
    return (int)CVB_OK;
  };
  if (const int rc = cvb_ba_solve_dev_edges(ctx, &bp, &bo, &br, fill, finish)) return rc;
  br.pose = r->ba.pose; br.speedbias = r->ba.speedbias; br.lm = r->ba.lm; br.lm_owner = r->ba.lm_owner;
  r->ba = br;
  return B.download();
}
