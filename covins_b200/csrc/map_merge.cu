// map_merge.cu — K16 cvb_map_rigid_transform: the rigid transform of the merge constructor Map(map_target, map_tofuse, T)
// (include/covins_b200.h states the rule and its assumptions).
//
// One launch, a grid-stride over K + L items: item i < K is keyframe i (16 pose entries and, when given, 3 velocity
// entries), item K + l is landmark l (3 entries).  Every entry is written, an unselected one as it was read, so the
// download brings back the caller's own bits for it.  Products and sums are __dmul_rn / __dadd_rn: ptxas may not contract
// them into DFMA, so each entry is rounded exactly as the float64 restatement of oracle/merge.py rounds it.  The call moves
// 2 x (128 K + 24 K + 24 L) bytes through HBM and the same over PCIe: it is bound by the copies, not by arithmetic.
#include <algorithm>
#include <cmath>

#include "cvb_internal.cuh"

namespace {

constexpr int RT_THREADS = 256;

struct RigidT {
  double m[16];   // row-major T_wtarget_wtofuse
};

// (a0 b0 + a1 b1) + a2 b2, rounded step by step
__device__ __forceinline__ double rt_dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

__global__ void __launch_bounds__(RT_THREADS) rigid_transform_kernel(const __grid_constant__ RigidT T, int K, const double* __restrict__ ws_in,
                                                                     double* __restrict__ ws_out, const double* __restrict__ vel_in,
                                                                     double* __restrict__ vel_out, int L, const double* __restrict__ lm_in,
                                                                     double* __restrict__ lm_out, const uint8_t* __restrict__ kf_sel,
                                                                     const uint8_t* __restrict__ lm_sel) {
  const double* t = T.m;
  const int64_t n = (int64_t)K + L;
  for (int64_t i = (int64_t)blockIdx.x * RT_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * RT_THREADS) {
    if (i < K) {
      const bool sel = !kf_sel || kf_sel[i];
      const double2* src = reinterpret_cast<const double2*>(ws_in + 16 * i);
      double x[16];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const double2 v = src[j];
        x[2 * j] = v.x;
        x[2 * j + 1] = v.y;
      }
      double y[16];
#pragma unroll
      for (int r = 0; r < 4; r++)
#pragma unroll
        for (int c = 0; c < 4; c++)
          y[4 * r + c] = sel ? __dadd_rn(rt_dot3(t[4 * r], t[4 * r + 1], t[4 * r + 2], x[c], x[4 + c], x[8 + c]), __dmul_rn(t[4 * r + 3], x[12 + c]))
                             : x[4 * r + c];
      double2* dst = reinterpret_cast<double2*>(ws_out + 16 * i);
#pragma unroll
      for (int j = 0; j < 8; j++) dst[j] = make_double2(y[2 * j], y[2 * j + 1]);
      if (vel_in) {
        const double v0 = vel_in[3 * i], v1 = vel_in[3 * i + 1], v2 = vel_in[3 * i + 2];
#pragma unroll
        for (int r = 0; r < 3; r++) vel_out[3 * i + r] = sel ? rt_dot3(t[4 * r], t[4 * r + 1], t[4 * r + 2], v0, v1, v2) : vel_in[3 * i + r];
      }
    } else {
      const int64_t l = i - K;
      const bool sel = !lm_sel || lm_sel[l];
      const double p0 = lm_in[3 * l], p1 = lm_in[3 * l + 1], p2 = lm_in[3 * l + 2];
#pragma unroll
      for (int r = 0; r < 3; r++)
        lm_out[3 * l + r] = sel ? __dadd_rn(rt_dot3(t[4 * r], t[4 * r + 1], t[4 * r + 2], p0, p1, p2), t[4 * r + 3]) : lm_in[3 * l + r];
    }
  }
}

// The rigidity test of include/covins_b200.h, in the order oracle/merge.py's is_rigid restates it
bool is_rigid(const double* T) {
  for (int i = 0; i < 16; i++)
    if (!std::isfinite(T[i])) return false;
  if (T[12] != 0.0 || T[13] != 0.0 || T[14] != 0.0 || T[15] != 1.0) return false;
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {   // (R^T R)[a][b] = sum_m R[m][a] R[m][b]
      const double s = (T[a] * T[b] + T[4 + a] * T[4 + b]) + T[8 + a] * T[8 + b];
      if (!(std::fabs(s - (a == b ? 1.0 : 0.0)) <= 1e-9)) return false;
    }
  const double det = (T[0] * (T[5] * T[10] - T[6] * T[9]) - T[1] * (T[4] * T[10] - T[6] * T[8])) + T[2] * (T[4] * T[9] - T[5] * T[8]);
  return det > 0.0;
}

}  // namespace

extern "C" int cvb_map_rigid_transform(cvb_ctx* ctx, const double T[16], int K, double* T_ws, double* vel, int L, double* lm_pos,
                                       const uint8_t* kf_sel, const uint8_t* lm_sel) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, T, "cvb_map_rigid_transform: T is required");
  CVB_REQUIRE(ctx, K >= 0 && L >= 0, "cvb_map_rigid_transform: negative size (K %d, L %d)", K, L);
  CVB_REQUIRE(ctx, (T_ws || K == 0) && (lm_pos || L == 0), "cvb_map_rigid_transform: T_ws and lm_pos are required");
  CVB_REQUIRE(ctx, is_rigid(T),
              "cvb_map_rigid_transform: T is not rigid (finite entries, R^T R = I within 1e-9, det R > 0, last row [0 0 0 1])");
  if ((int64_t)K + L == 0) return CVB_OK;
  cudaStream_t st = ctx->stream;
  cvb_block B(ctx, st, false);   // direct: one copy per array each way
  const double *d_ws_in, *d_vel_in = nullptr, *d_lm_in;
  const uint8_t *d_kf_sel = nullptr, *d_lm_sel = nullptr;
  double *d_ws_out, *d_vel_out = nullptr, *d_lm_out;
  B.in(d_ws_in, T_ws, 16 * (size_t)K);
  if (vel) B.in(d_vel_in, vel, 3 * (size_t)K);
  B.in(d_lm_in, lm_pos, 3 * (size_t)L);
  if (kf_sel) B.in(d_kf_sel, kf_sel, K);
  if (lm_sel) B.in(d_lm_sel, lm_sel, L);
  B.out(d_ws_out, T_ws, 16 * (size_t)K);
  if (vel) B.out(d_vel_out, vel, 3 * (size_t)K);
  B.out(d_lm_out, lm_pos, 3 * (size_t)L);
  if (const int rc = B.place()) return rc;
  if (const int rc = B.upload()) return rc;
  RigidT t;
  memcpy(t.m, T, sizeof(t.m));
  const int64_t n = (int64_t)K + L;
  const int grid = (int)std::min<int64_t>((n + RT_THREADS - 1) / RT_THREADS, (int64_t)ctx->sm_count * 8);
  rigid_transform_kernel<<<grid, RT_THREADS, 0, st>>>(t, K, d_ws_in, d_ws_out, d_vel_in, d_vel_out, L, d_lm_in, d_lm_out, d_kf_sel, d_lm_sel);
  CVB_CHECK_LAUNCH(ctx);
  return B.download();
}
