// ba_engine.cu — global bundle adjustment / pose-graph optimisation on the GPU (K4-K9).
//
// Replaces, behind the flat problem format of include/covins_b200.h, what the reference hands to Ceres in
//   Optimization::GlobalBundleAdjustment   optimization_be.cpp:56-618   (ceres::Solve at :265 and :567)
//   Optimization::PoseGraphOptimization    optimization_be.cpp:833-1086 (ceres::Solve at :1031)
// i.e. cost-function evaluation (robopt_open), CauchyLoss + corrector, Jacobi scaling, the SPARSE_SCHUR linear
// solve and the DOGLEG trust-region loop (Ceres 1.x defaults; assumptions in SURVEY.md Appendix A.7).
//
// One outer iteration =
//   lin_obs / lin_imu / lin_edge   residuals + analytic Jacobians per factor, loss-corrected, Jacobi-scaled (K4-K6)
//   lm_reduce, lm_damp_inv, obs_Y  per-landmark 3x3 blocks, their inverses, Y = W Hll^-1
//   kf_visual, factor_gather       camera blocks of J^T J into the dense reduced system S, gradient
//   cam_diag, schur                damping + S -= sum_l Y W^T over precomputed (block → observation pair) lists (K7)
//   cvb_chol::factor / solve       dense FP64 tiled Cholesky on DMMA (K8), landmark back-substitution
//   dogleg algebra + J*step        Cauchy point, interpolation, model decrease
//   plus + residual-only pass      candidate state and its cost (K9)
// Every accumulation is a gather in a fixed order (no floating-point atomics): results are bit-reproducible.
//
// HBM layout: per observation an 160-B record {r[2], Jp[12], Jl[6]} and a 288-B record {W[18], Y[18]} (AoS so the
// per-keyframe and per-pair gathers read whole records), per landmark Hll/Hll^-1/b (15 doubles), S as the packed list
// of the 128x128 tiles of L's structure (cholesky.cuh: TilePlan::h_tile_of; lower triangle), state double-buffered for
// accept/reject.
//
// Multi-GPU (one process per GPU): landmark blocks are sharded, every rank builds its partial S; the tile columns of S
// are OWNED by ranks (IMU chain → one rank, pose columns cyclic).  With peer access (CUDA IPC over NVLink,
// cvb_ba_enable_p2p) the owners pull-and-sum the partial tiles of their columns out of the peers' memory (reduce-scatter
// without a staging buffer) and the factorisation is distributed by columns (cholesky.cu: DistView); without it the
// packed tiles are all-reduced through the injected collective and the factorisation is replicated.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <functional>
#include <numeric>
#include <string>
#include <vector>

#include <cub/cub.cuh>

#include <thread>

#include "ba_group.cuh"
#include "ba_math.cuh"
#include "cholesky.cuh"
#include "cvb_internal.cuh"


namespace {

using namespace bam;

struct ObsLin {
  double r[2], Jp[12], Jl[6];
};
struct __align__(16) ObsW {   // 16-byte aligned: gathered as nine 16-byte loads
  double W[18];
};

// Column of (keyframe kf, local parameter c) in the reduced camera system: c < 6 pose, c >= 6 speed-bias.  The
// speed-bias blocks are ordered FIRST (off_sb < off_pose): along the IMU chain they form a block-banded system whose
// elimination costs almost nothing in the tile-sparse Cholesky, leaving only the dense 6K pose part.
__device__ __forceinline__ int cam_col(const int* __restrict__ off_pose, const int* __restrict__ off_sb, int kf, int c) {
  return c < 6 ? off_pose[kf] + c : off_sb[kf] + (c - 6);
}

// View of the packed reduced camera system: element (r >= c) lives in tile (r/128, c/128) of L's structure.
struct SView {
  double* p;
  const int* __restrict__ tile_of;
  int nt;
};
__device__ __forceinline__ double* s_at(const SView& S, int r, int c) {
  const int t = S.tile_of[(size_t)(r >> 7) * S.nt + (c >> 7)];
  if (t < 0) __trap();   // an element outside L's structure (or above the diagonal): a bug, never silent
  return S.p + ((size_t)t << 14) + ((r & 127) << 7) + (c & 127);
}
static_assert(cvb_chol::T == 128, "s_at assumes 128-wide tiles");

constexpr int RED_BLOCKS = 512;   // fixed grid for reducing kernels → fixed summation order
constexpr int RED_SLOTS = 8;

// The engine's device arrays come from the stream-ordered allocator on the engine's stream: the pool (release threshold
// raised in cvb_ctx_create) keeps freed blocks, so building a second problem re-uses the first one's memory instead of
// paying cudaMalloc/cudaFree (which cost ~100 ms of a 180 ms set-up at C3, the 7.4 GB S buffer alone several ms each way).
struct Engine {
  cvb_ctx* ctx = nullptr;
  cudaStream_t st = nullptr;
  // sizes
  int K = 0, L_in = 0, n_obs = 0, n_imu = 0, n_edge = 0, per = 6, n_c = 0, n_c_pad = 0, n_vec = 0;
  int visual_only = 1;
  double a2_reproj = 1.0, a2_edge = 0.25, g = 9.81;
  int rank = 0, world = 1;
  // host-side maps
  std::vector<int> lm_of_compact;        // compact landmark → original index
  std::vector<int> obs_of_compact;       // compact observation → original index
  std::vector<uint8_t> h_const;
  // device state (double buffered)
  cvb_dev_arr<double> pose[2], sb[2], lm[2];
  cvb_dev_arr<double> pose0, sb0, lm0;   // the state the problem was created with (cvb_ba_restart returns to it)
  cvb_dev_arr<uint8_t> pose_const;
  cvb_dev_arr<int> off_pose, off_sb;
  // multi-GPU exchange of the reduced camera system: packed ids of the structurally non-zero (pre-fill) tiles — all of
  // them (all-reduce fallback, through xbuf) / those of the tile columns this rank owns (reduce-scatter by peer pull)
  cvb_dev_arr<int> xt_all, xt_own, col_owner;
  cvb_dev_arr<double> xbuf, flagd;
  int n_xt_all = 0, n_xt_own = 0;
  size_t n_tiles = 0;                           // tiles of L's structure = length of S in tiles
  // peer access: S, linv and the panel flags of every rank are mapped here (enable_p2p: through CUDA IPC, or handed over
  // by an in-process group, peer_ipc = false)
  bool p2p = false, peer_ipc = false;
  cvb_chol::DistView dv;
  cvb_dev_arr<int> epoch;                       // dv.d_epoch
  cvb_dev_arr<int*> peer_flag;                  // dv.d_peer_flag
  cvb_dev_arr<double*> peer_S;                  // dv.peer_S on the device (reduce_pull_kernel)
  std::vector<uint8_t> h_prefill;               // tile mask of S before fill (the distributed plan is rebuilt from it)
  std::vector<int> h_owner;                     // tile column → owning rank
  std::vector<int> h_off_pose, h_off_sb;
  cvb_chol::TilePlan plan;
  cvb_dev_arr<double> extr_kf, intr_kf, dist_kf, xi_kf;
  cvb_dev_arr<int> model_kf;   // cam model | dist model << 8, per keyframe
  cvb_dev_arr<int> obs_kf, obs_lm, lm_ptr, kf_ptr, kf_obs;
  cvb_dev_arr<double> obs_uv, obs_sigma;
  cvb_dev_arr<ObsLin> lin;
  cvb_dev_arr<ObsW> ow;
  cvb_dev_arr<double> Hll, HllInv, bl;
  // imu
  cvb_dev_arr<ImuPre> pre;
  cvb_dev_arr<int> imu_i, imu_j;
  cvb_dev_arr<double> Jimu, rimu;
  // edges
  cvb_dev_arr<int> edge_i, edge_j;
  cvb_dev_arr<double> edge_q, edge_t, edge_S, Jedge, redge;
  cvb_dev_arr<uint8_t> edge_robust;
  // gather structures
  cvb_dev_arr<int> fb_hi, fb_lo, fb_ptr, ft_type, ft_fac, ft_rhi, ft_rlo;   // factor blocks / terms
  int n_fb = 0;
  cvb_dev_arr<int> sb_hi, sb_lo, sb_ptr, sp_a, sp_b;                        // schur blocks / pairs
  cvb_dev_arr<int> kf_sb;                                                   // first schur block of each hi keyframe
  int n_sb = 0, row_stage = 0;                                              // row_stage: observations schur_row_kernel stages
  // vectors of size n_vec: [cam part n_c_pad | landmark part 3 L_in]
  cvb_dev_arr<double> scale, colsq, diag, gvec, grad, sgrad, gn, step, xsol, yb, gs, tmp;
  cvb_dev_arr<double> scale0;   // 0/1 activity mask of this rank's columns: engine_begin derives `scale` from it
  // S, the tile inverses and (world > 1) the panel flags; from cudaMalloc when world > 1, to be exported through CUDA IPC
  cvb_dev_arr<double> S, linv;
  cvb_dev_arr<int> pflag;
  // S's fill tiles (in L's structure, not in S's): zeroed on st_fill beside the block kernels, joined before the factor
  cvb_dev_arr<int> xt_fill;
  int n_xt_fill = 0;
  cudaStream_t st_fill = nullptr;
  cudaEvent_t ev_fill_fork = nullptr, ev_fill_done = nullptr;
  bool fill_pending = false;
  cvb_dev_arr<int> flag;
  cvb_dev_arr<double> partials, scalars, rankmax;
  double* h_scalars = nullptr;   // pinned
  int cur = 0;
  // trust-region state (Ceres DoglegStrategy / TrustRegionMinimizer)
  double radius = 1e4, mu = 1e-8, cost = 0.0, x_norm = 0.0, alpha = 0.0, dogleg_norm = 0.0;
  double gn2 = 0.0, gg = 0.0, g_gn = 0.0;   // |gn|^2, |grad|^2, grad.gn of the current Gauss-Newton solve
  bool reuse = false, have_lin = false, scaled = false;
  int invalid_run = 0, iterations = 0, termination = 0;
  std::vector<double> cost_hist;
  std::vector<int> step_status;
  std::function<int(void*, size_t)> allreduce;   // (device ptr, count of doubles) in-place sum over ranks
  // phase timing (CUDA events on the engine stream): 0 linearise, 1 block build + Schur, 2 Cholesky factor,
  // 3 triangular solves + back-substitution, 4 dogleg / J*step / plus / candidate cost
  cudaEvent_t ev[8] = {};
  cvb_chol::FactorStreams fs;            // lookahead / chain streams of the factorisation
  cudaGraphExec_t g_factor = nullptr, g_solve = nullptr;   // the ~700 launches of one factorisation / the solve, captured once
  int n_factor_calls = 0, n_solve_calls = 0;
  double phase_ms[5] = {0, 0, 0, 0, 0};
  double chol_flops = 0.0;
  ~Engine() {
    if (st_fill) { cudaStreamSynchronize(st_fill); cudaStreamDestroy(st_fill); }   // S may still be being cleared
    if (ev_fill_fork) cudaEventDestroy(ev_fill_fork);
    if (ev_fill_done) cudaEventDestroy(ev_fill_done);
    for (int g = 0; g < dv.world && p2p && peer_ipc; g++) {
      if (g == dv.rank) continue;
      if (dv.peer_S[g]) cudaIpcCloseMemHandle(dv.peer_S[g]);
      if (dv.peer_linv[g]) cudaIpcCloseMemHandle(dv.peer_linv[g]);
      if (dv.peer_flag[g]) cudaIpcCloseMemHandle(dv.peer_flag[g]);
    }
    if (h_scalars) cudaFreeHost(h_scalars);
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    fs.destroy();
    if (g_factor) cudaGraphExecDestroy(g_factor);
    if (g_solve) cudaGraphExecDestroy(g_solve);
  }
};

// ------------------------------------------------------------------------------------------------
// reductions: every reducing kernel writes RED_BLOCKS partials per slot; reduce_final sums them in a fixed tree
// ------------------------------------------------------------------------------------------------
template <int NV>
__device__ __forceinline__ void block_reduce_store(double (&v)[NV], double* partials, const int (&slots)[NV]) {
  __shared__ double sm[NV][256];
  const int tid = threadIdx.x;
#pragma unroll
  for (int i = 0; i < NV; i++) sm[i][tid] = v[i];
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) {
#pragma unroll
      for (int i = 0; i < NV; i++) sm[i][tid] += sm[i][tid + s];
    }
    __syncthreads();
  }
  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < NV; i++) partials[slots[i] * RED_BLOCKS + blockIdx.x] = sm[i][0];
  }
}

__global__ void __launch_bounds__(256) reduce_final(const double* __restrict__ partials, double* __restrict__ scalars,
                                                    int nslots, int add) {
  __shared__ double sm[256];
  for (int s = 0; s < nslots; s++) {
    double v = 0.0;
    for (int i = threadIdx.x; i < RED_BLOCKS; i += 256) v += partials[s * RED_BLOCKS + i];
    sm[threadIdx.x] = v;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
      if (threadIdx.x < k) sm[threadIdx.x] += sm[threadIdx.x + k];
      __syncthreads();
    }
    if (threadIdx.x == 0) scalars[s] = (add ? scalars[s] : 0.0) + sm[0];
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// K4: reprojection linearisation.  mode 0: residual + Jacobian records + cost; 1: cost only; 2: corrected norms
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 2) lin_obs_kernel(int n_obs, const int* __restrict__ obs_kf, const int* __restrict__ obs_lm,
                                                      const double* __restrict__ obs_uv, const double* __restrict__ obs_sigma,
                                                      const double* __restrict__ pose, const double* __restrict__ lm,
                                                      const double* __restrict__ extr_kf, const double* __restrict__ intr_kf,
                                                      const double* __restrict__ dist_kf, const int* __restrict__ model_kf,
                                                      const double* __restrict__ xi_kf, const double* __restrict__ scale,
                                                      const int* __restrict__ off_pose, int n_c_pad, double a2, int mode,
                                                      ObsLin* __restrict__ lin,
                                                      ObsW* __restrict__ ow, double* __restrict__ norms,
                                                      double* __restrict__ partials, int slot) {
  double csum[1] = {0.0};
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < n_obs; o += gridDim.x * blockDim.x) {
    const int k = obs_kf[o], l = obs_lm[o];
    double r[2], Jp[12], Jl[6];
    const int mk = model_kf[k];
    const CamModel cm{mk & 0xff, mk >> 8, xi_kf[k]};
    reproj(pose + 7 * k, extr_kf + 7 * k, intr_kf + 4 * k, dist_kf + 4 * k, cm, lm + 3 * l, obs_uv[2 * o], obs_uv[2 * o + 1],
           obs_sigma[o], r, Jp, Jl, mode == 0);
    const double s = r[0] * r[0] + r[1] * r[1];
    double sc, c;
    cauchy(s, a2, &sc, &c);
    csum[0] += c;
    if (mode == 2) norms[o] = sqrt(s) * sc;
    if (mode != 0) continue;
    ObsLin rec;
    rec.r[0] = r[0] * sc;
    rec.r[1] = r[1] * sc;
    const double* sp = scale + off_pose[k];
    const double* sl = scale + n_c_pad + 3 * (size_t)l;
#pragma unroll
    for (int c2 = 0; c2 < 6; c2++) {
      rec.Jp[c2] = Jp[c2] * sc * sp[c2];
      rec.Jp[6 + c2] = Jp[6 + c2] * sc * sp[c2];
    }
#pragma unroll
    for (int c2 = 0; c2 < 3; c2++) {
      rec.Jl[c2] = Jl[c2] * sc * sl[c2];
      rec.Jl[3 + c2] = Jl[3 + c2] * sc * sl[c2];
    }
    lin[o] = rec;
    ObsW* w = ow + o;   // W = Jp^T Jl (6x3)
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
      for (int b = 0; b < 3; b++) w->W[3 * a + b] = rec.Jp[a] * rec.Jl[b] + rec.Jp[6 + a] * rec.Jl[3 + b];
  }
  const int slots[1] = {slot};
  block_reduce_store<1>(csum, partials, slots);
}

// K4b: the loss-corrected residual norm of every observation (cvb_ba_reproj_norms) through bam::corrected_norm, the function
// cvb_landmark_outliers calls too, so that the two report the same norms bit for bit
__global__ void reproj_norms_kernel(int n_obs, const int* __restrict__ obs_kf, const int* __restrict__ obs_lm, const double* __restrict__ obs_uv,
                                    const double* __restrict__ obs_sigma, const double* __restrict__ pose, const double* __restrict__ lm,
                                    const double* __restrict__ extr_kf, const double* __restrict__ intr_kf, const double* __restrict__ dist_kf,
                                    const int* __restrict__ model_kf, const double* __restrict__ xi_kf, double a2, double* __restrict__ norms) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n_obs) return;
  const int k = obs_kf[o], mk = model_kf[k];
  const CamModel cm{mk & 0xff, mk >> 8, xi_kf[k]};
  bool projectable;
  norms[o] = corrected_norm(pose + 7 * k, extr_kf + 7 * k, intr_kf + 4 * k, dist_kf + 4 * k, cm, lm + 3 * obs_lm[o], obs_uv[2 * o],
                            obs_uv[2 * o + 1], obs_sigma[o], a2, &projectable);
}

// per landmark: Hll = sum Jl^T Jl (6 unique: 00 01 02 11 12 22), bl = sum Jl^T r, colsq of the 3 columns
__global__ void lm_reduce_kernel(int L, const int* __restrict__ lm_ptr, const ObsLin* __restrict__ lin,
                                 double* __restrict__ Hll, double* __restrict__ bl, double* __restrict__ colsq_l,
                                 double* __restrict__ g_l) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  double h[6] = {0, 0, 0, 0, 0, 0}, b[3] = {0, 0, 0};
  for (int o = lm_ptr[l]; o < lm_ptr[l + 1]; o++) {
    const double* J = lin[o].Jl;
    const double r0 = lin[o].r[0], r1 = lin[o].r[1];
    h[0] += J[0] * J[0] + J[3] * J[3];
    h[1] += J[0] * J[1] + J[3] * J[4];
    h[2] += J[0] * J[2] + J[3] * J[5];
    h[3] += J[1] * J[1] + J[4] * J[4];
    h[4] += J[1] * J[2] + J[4] * J[5];
    h[5] += J[2] * J[2] + J[5] * J[5];
    b[0] += J[0] * r0 + J[3] * r1;
    b[1] += J[1] * r0 + J[4] * r1;
    b[2] += J[2] * r0 + J[5] * r1;
  }
  for (int i = 0; i < 6; i++) Hll[6 * (size_t)l + i] = h[i];
  for (int i = 0; i < 3; i++) {
    bl[3 * (size_t)l + i] = b[i];
    g_l[3 * (size_t)l + i] = b[i];
  }
  colsq_l[3 * (size_t)l + 0] = h[0];
  colsq_l[3 * (size_t)l + 1] = h[3];
  colsq_l[3 * (size_t)l + 2] = h[5];
}

__device__ __forceinline__ double clamp_diag(double v) { return fmin(fmax(v, 1e-6), 1e32); }

// (Hll + mu * diag_l^2)^-1, symmetric 3x3
__global__ void lm_damp_inv_kernel(int L, const double* __restrict__ Hll, const double* __restrict__ colsq_l, double mu,
                                   double* __restrict__ HllInv) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  const double* h = Hll + 6 * (size_t)l;
  const double a = h[0] + mu * clamp_diag(colsq_l[3 * (size_t)l]), b = h[1], c = h[2];
  const double d = h[3] + mu * clamp_diag(colsq_l[3 * (size_t)l + 1]), e = h[4];
  const double f = h[5] + mu * clamp_diag(colsq_l[3 * (size_t)l + 2]);
  const double A = d * f - e * e, B = c * e - b * f, C = b * e - c * d;
  const double det = a * A + b * B + c * C;
  const double id = 1.0 / det;
  double* o = HllInv + 6 * (size_t)l;
  o[0] = A * id;
  o[1] = B * id;
  o[2] = C * id;
  o[3] = (a * f - c * c) * id;
  o[4] = (b * c - a * e) * id;
  o[5] = (a * d - b * b) * id;
}

// Y = W * Hll^-1 (6x3) of one observation, h the packed symmetric inverse
__device__ __forceinline__ void obs_y(const double* __restrict__ W, const double* __restrict__ h, double (&Y)[18]) {
  const double H[9] = {h[0], h[1], h[2], h[1], h[3], h[4], h[2], h[4], h[5]};
#pragma unroll
  for (int a = 0; a < 6; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) Y[3 * a + b] = W[3 * a] * H[b] + W[3 * a + 1] * H[3 + b] + W[3 * a + 2] * H[6 + b];
}

// per keyframe (one warp): Hpp = sum Jp^T Jp → lower part of the 6x6 diagonal block of S; g_c = sum Jp^T r
__global__ void __launch_bounds__(128) kf_visual_kernel(int K, const int* __restrict__ kf_ptr, const int* __restrict__ kf_obs,
                                                        const ObsLin* __restrict__ lin, const int* __restrict__ off_pose,
                                                        SView S, double* __restrict__ g_c) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (k >= K) return;
  double h[21], b[6];
#pragma unroll
  for (int i = 0; i < 21; i++) h[i] = 0.0;
#pragma unroll
  for (int i = 0; i < 6; i++) b[i] = 0.0;
  for (int e = kf_ptr[k] + lane; e < kf_ptr[k + 1]; e += 32) {
    const ObsLin& L = lin[kf_obs[e]];
    int idx = 0;
#pragma unroll
    for (int r = 0; r < 6; r++)
#pragma unroll
      for (int c = 0; c <= r; c++) h[idx++] += L.Jp[r] * L.Jp[c] + L.Jp[6 + r] * L.Jp[6 + c];
#pragma unroll
    for (int r = 0; r < 6; r++) b[r] += L.Jp[r] * L.r[0] + L.Jp[6 + r] * L.r[1];
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
    for (int i = 0; i < 21; i++) h[i] += __shfl_xor_sync(0xffffffffu, h[i], off);
#pragma unroll
    for (int i = 0; i < 6; i++) b[i] += __shfl_xor_sync(0xffffffffu, b[i], off);
  }
  if (lane == 0) {
    const int base = off_pose[k];
    int idx = 0;
    for (int r = 0; r < 6; r++)
      for (int c = 0; c <= r; c++) *s_at(S, base + r, base + c) = h[idx++];   // lower triangle only
    for (int r = 0; r < 6; r++) g_c[base + r] = b[r];
  }
}

// ------------------------------------------------------------------------------------------------
// K5: IMU preintegration (repropagate) and factor linearisation
// ------------------------------------------------------------------------------------------------
// One thread per factor.  VINS-Mono IntegrationBase::midPointIntegration restated [A]; covariance P and Jacobian
// J (15x15) live in local memory.  Output: ImuPre with sqrt_info = chol(P^-1)^T.
__global__ void imu_repropagate_kernel(int n_imu, const int* __restrict__ imu_j, const int* __restrict__ imu_ptr,
                                       const double* __restrict__ dt, const double* __restrict__ acc,
                                       const double* __restrict__ gyr, const double* __restrict__ acc0,
                                       const double* __restrict__ gyr0, const double* __restrict__ sb,
                                       const double* __restrict__ noise, ImuPre* __restrict__ pre, int* __restrict__ flag) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_imu) return;
  const int j = imu_j[f];
  const V3 ba{sb[9 * j + 3], sb[9 * j + 4], sb[9 * j + 5]}, bg{sb[9 * j + 6], sb[9 * j + 7], sb[9 * j + 8]};
  const double q_[6] = {noise[0] * noise[0], noise[1] * noise[1], noise[0] * noise[0], noise[1] * noise[1],
                        noise[2] * noise[2], noise[3] * noise[3]};
  double Jm[225], P[225], F[225], V[270], Tm[225];
  for (int i = 0; i < 225; i++) { Jm[i] = 0.0; P[i] = 0.0; }
  for (int i = 0; i < 15; i++) Jm[16 * i] = 1.0;
  V3 dp{0, 0, 0}, dv{0, 0, 0};
  Q4 dq{0, 0, 0, 1};
  V3 a0{acc0[3 * f], acc0[3 * f + 1], acc0[3 * f + 2]}, g0{gyr0[3 * f], gyr0[3 * f + 1], gyr0[3 * f + 2]};
  double Tsum = 0.0;
  for (int s = imu_ptr[f]; s < imu_ptr[f + 1]; s++) {
    const double h = dt[s];
    const V3 a1{acc[3 * s], acc[3 * s + 1], acc[3 * s + 2]}, g1{gyr[3 * s], gyr[3 * s + 1], gyr[3 * s + 2]};
    const M3 R0 = q2R(dq);
    const V3 ua0 = mul(R0, a0 - ba);
    const V3 ug = 0.5 * (g0 + g1) - bg;
    const Q4 q1 = qnormalized(qmul(dq, Q4{ug.x * h / 2, ug.y * h / 2, ug.z * h / 2, 1.0}));
    const M3 R1 = q2R(q1);
    const V3 ua1 = mul(R1, a1 - ba);
    const V3 ua = 0.5 * (ua0 + ua1);
    const V3 ndp = dp + h * dv + (0.5 * h * h) * ua;
    const V3 ndv = dv + h * ua;
    const M3 Rw = skew(ug), Ra0 = skew(a0 - ba), Ra1 = skew(a1 - ba);
    M3 ImRw = eye3();
    for (int i = 0; i < 9; i++) ImRw.m[i] -= Rw.m[i] * h;
    const M3 R0Ra0 = mul(R0, Ra0), R1Ra1 = mul(R1, Ra1), R1Ra1I = mul(R1Ra1, ImRw);
    for (int i = 0; i < 225; i++) F[i] = 0.0;
    for (int i = 0; i < 270; i++) V[i] = 0.0;
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) {
        const int ab = 3 * a + b;
        const double I = (a == b) ? 1.0 : 0.0;
        F[15 * a + b] = I;
        F[15 * a + 3 + b] = -0.25 * R0Ra0.m[ab] * h * h - 0.25 * R1Ra1I.m[ab] * h * h;
        F[15 * a + 6 + b] = I * h;
        F[15 * a + 9 + b] = -0.25 * (R0.m[ab] + R1.m[ab]) * h * h;
        F[15 * a + 12 + b] = -0.25 * R1Ra1.m[ab] * h * h * (-h);
        F[15 * (3 + a) + 3 + b] = ImRw.m[ab];
        F[15 * (3 + a) + 12 + b] = -I * h;
        F[15 * (6 + a) + 3 + b] = -0.5 * R0Ra0.m[ab] * h - 0.5 * R1Ra1I.m[ab] * h;
        F[15 * (6 + a) + 6 + b] = I;
        F[15 * (6 + a) + 9 + b] = -0.5 * (R0.m[ab] + R1.m[ab]) * h;
        F[15 * (6 + a) + 12 + b] = -0.5 * R1Ra1.m[ab] * h * (-h);
        F[15 * (9 + a) + 9 + b] = I;
        F[15 * (12 + a) + 12 + b] = I;
        V[18 * a + b] = 0.25 * R0.m[ab] * h * h;
        V[18 * a + 3 + b] = 0.25 * (-R1Ra1.m[ab] * h * h) * 0.5 * h;
        V[18 * a + 6 + b] = 0.25 * R1.m[ab] * h * h;
        V[18 * a + 9 + b] = V[18 * a + 3 + b];
        V[18 * (3 + a) + 3 + b] = 0.5 * I * h;
        V[18 * (3 + a) + 9 + b] = 0.5 * I * h;
        V[18 * (6 + a) + b] = 0.5 * R0.m[ab] * h;
        V[18 * (6 + a) + 3 + b] = 0.5 * (-R1Ra1.m[ab] * h) * 0.5 * h;
        V[18 * (6 + a) + 6 + b] = 0.5 * R1.m[ab] * h;
        V[18 * (6 + a) + 9 + b] = V[18 * (6 + a) + 3 + b];
        V[18 * (9 + a) + 12 + b] = I * h;
        V[18 * (12 + a) + 15 + b] = I * h;
      }
    // Jm <- F Jm
    for (int r = 0; r < 15; r++)
      for (int c = 0; c < 15; c++) {
        double s2 = 0;
        for (int m = 0; m < 15; m++) s2 += F[15 * r + m] * Jm[15 * m + c];
        Tm[15 * r + c] = s2;
      }
    for (int i = 0; i < 225; i++) Jm[i] = Tm[i];
    // P <- F P F^T + V Q V^T
    for (int r = 0; r < 15; r++)
      for (int c = 0; c < 15; c++) {
        double s2 = 0;
        for (int m = 0; m < 15; m++) s2 += F[15 * r + m] * P[15 * m + c];
        Tm[15 * r + c] = s2;
      }
    for (int r = 0; r < 15; r++)
      for (int c = 0; c < 15; c++) {
        double s2 = 0;
        for (int m = 0; m < 15; m++) s2 += Tm[15 * r + m] * F[15 * c + m];
        for (int m = 0; m < 18; m++) s2 += V[18 * r + m] * q_[m / 3] * V[18 * c + m];
        P[15 * r + c] = s2;
      }
    dp = ndp; dv = ndv; dq = q1; a0 = a1; g0 = g1; Tsum += h;
  }
  ImuPre& O = pre[f];
  O.T = Tsum;
  O.alpha[0] = dp.x; O.alpha[1] = dp.y; O.alpha[2] = dp.z;
  O.beta[0] = dv.x; O.beta[1] = dv.y; O.beta[2] = dv.z;
  O.gamma[0] = dq.x; O.gamma[1] = dq.y; O.gamma[2] = dq.z; O.gamma[3] = dq.w;
  O.ba[0] = ba.x; O.ba[1] = ba.y; O.ba[2] = ba.z;
  O.bg[0] = bg.x; O.bg[1] = bg.y; O.bg[2] = bg.z;
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {
      O.dp_dba[3 * a + b] = Jm[15 * a + 9 + b];
      O.dp_dbg[3 * a + b] = Jm[15 * a + 12 + b];
      O.dq_dbg[3 * a + b] = Jm[15 * (3 + a) + 12 + b];
      O.dv_dba[3 * a + b] = Jm[15 * (6 + a) + 9 + b];
      O.dv_dbg[3 * a + b] = Jm[15 * (6 + a) + 12 + b];
    }
  // sqrt_info = chol(P^-1)^T :  P = Lp Lp^T,  P^-1 = Lp^-T Lp^-1;  chol(P^-1) = M with M M^T = P^-1.
  // Take X = Lp^-1 (lower).  P^-1 = X^T X.  Its Cholesky factor (lower, positive diagonal) is computed directly.
  // 1. Pinv via Cholesky of P
  bool ok = true;
  for (int c = 0; c < 15; c++) {   // F <- chol(P) lower
    for (int r = c; r < 15; r++) {
      double s2 = P[15 * r + c];
      for (int m = 0; m < c; m++) s2 -= F[15 * r + m] * F[15 * c + m];
      if (r == c) {
        if (!(s2 > 0.0)) { ok = false; s2 = 1.0; }
        F[15 * c + c] = sqrt(s2);
      } else {
        F[15 * r + c] = s2 / F[15 * c + c];
      }
    }
    for (int r = 0; r < c; r++) F[15 * r + c] = 0.0;
  }
  for (int c = 0; c < 15; c++)      // Tm <- F^-1 (lower)
    for (int r = 0; r < 15; r++) {
      if (r < c) { Tm[15 * r + c] = 0.0; continue; }
      double s2 = (r == c) ? 1.0 : 0.0;
      for (int m = c; m < r; m++) s2 -= F[15 * r + m] * Tm[15 * m + c];
      Tm[15 * r + c] = s2 / F[15 * r + r];
    }
  for (int r = 0; r < 15; r++)      // P <- Pinv = Tm^T Tm
    for (int c = 0; c < 15; c++) {
      double s2 = 0;
      for (int m = (r > c ? r : c); m < 15; m++) s2 += Tm[15 * m + r] * Tm[15 * m + c];
      P[15 * r + c] = s2;
    }
  for (int c = 0; c < 15; c++)      // F <- chol(Pinv) lower
    for (int r = c; r < 15; r++) {
      double s2 = P[15 * r + c];
      for (int m = 0; m < c; m++) s2 -= F[15 * r + m] * F[15 * c + m];
      if (r == c) {
        if (!(s2 > 0.0)) { ok = false; s2 = 1.0; }
        F[15 * c + c] = sqrt(s2);
      } else {
        F[15 * r + c] = s2 / F[15 * c + c];
      }
    }
  for (int r = 0; r < 15; r++)
    for (int c = 0; c < 15; c++) O.sqrt_info[15 * r + c] = (c >= r) ? F[15 * c + r] : 0.0;   // L^T (upper)
  if (!ok) atomicOr(flag, 2);
}

// IMU factor: whitened residual (15) and whitened, Jacobi-scaled Jacobian (15x30); mode 1: cost only.
// One WARP per factor (ncu r02: the one-thread-per-factor version ran 439 us for 2 k factors at 255 registers with the
// 450-double Jacobian in local memory): lane c < 30 owns column c of the Jacobian — raw column (ba_math.cuh:
// imu_raw_column), whitening by the upper-triangular sqrt_info (120 MACs), coalesced store along c; lane 30 whitens the
// residual.  Every lane recomputes the few shared 3x3 products (~600 flops) instead of exchanging them.
__global__ void __launch_bounds__(256) lin_imu_kernel(int n_imu, const int* __restrict__ imu_i, const int* __restrict__ imu_j,
                               const ImuPre* __restrict__ pre, const double* __restrict__ pose, const double* __restrict__ sb,
                               const double* __restrict__ scale, const int* __restrict__ off_pose,
                               const int* __restrict__ off_sb, double g, int mode, double* __restrict__ Jout,
                               double* __restrict__ rout, double* __restrict__ partials, int slot) {
  double csum[1] = {0.0};
  const int lane = threadIdx.x & 31, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  for (int f = warp; f < n_imu; f += n_warps) {
    const int i = imu_i[f], j = imu_j[f];
    const ImuPre& P = pre[f];
    const double* W = P.sqrt_info;
    if (lane == 30 || mode != 0) {
      // the residual: lane 30 (and, for the cost-only pass, nobody else is needed)
      if (lane == 30) {
        double r[15];
        imu_raw_column(pose + 7 * i, sb + 9 * i, pose + 7 * j, sb + 9 * j, P, g, 0, nullptr, r);
        double s = 0;
        for (int a = 0; a < 15; a++) {
          double v = 0;
          for (int m = a; m < 15; m++) v += W[15 * a + m] * r[m];   // upper triangular
          if (mode == 0) rout[15 * (size_t)f + a] = v;
          s += v * v;
        }
        csum[0] += 0.5 * s;
      }
      if (mode != 0) continue;
    }
    if (lane < 30) {
      double col[15];
      imu_raw_column(pose + 7 * i, sb + 9 * i, pose + 7 * j, sb + 9 * j, P, g, lane, col, nullptr);
      const int kf = lane < 15 ? i : j;
      const double sc = scale[cam_col(off_pose, off_sb, kf, lane < 15 ? lane : lane - 15)];
      for (int a = 0; a < 15; a++) {
        double v = 0;
        for (int m = a; m < 15; m++) v += W[15 * a + m] * col[m];
        Jout[(size_t)f * 450 + 30 * a + lane] = v * sc;
      }
    }
  }
  const int slots[1] = {slot};
  block_reduce_store<1>(csum, partials, slots);
}

// K6: between factor
__global__ void __launch_bounds__(256) lin_edge_kernel(int n_edge, const int* __restrict__ ei, const int* __restrict__ ej, const double* __restrict__ eq,
                                const double* __restrict__ et, const double* __restrict__ eS, const uint8_t* __restrict__ robust,
                                const double* __restrict__ pose, const double* __restrict__ scale,
                                const int* __restrict__ off_pose, double a2, int mode,
                                double* __restrict__ Jout, double* __restrict__ rout, double* __restrict__ partials, int slot) {
  double csum[1] = {0.0};
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_edge; e += gridDim.x * blockDim.x) {
    const int i = ei[e], j = ej[e];
    double r[6], J[72];
    between(pose + 7 * i, pose + 7 * j, eq + 4 * e, et + 3 * e, eS + 36 * (size_t)e, r, J, mode == 0);
    double s = 0;
    for (int a = 0; a < 6; a++) s += r[a] * r[a];
    double sc, c;
    cauchy(s, robust[e] ? a2 : 0.0, &sc, &c);
    csum[0] += c;
    if (mode != 0) continue;
    for (int a = 0; a < 6; a++) rout[6 * (size_t)e + a] = r[a] * sc;
    for (int a = 0; a < 6; a++)
      for (int c2 = 0; c2 < 12; c2++) {
        const int kf = c2 < 6 ? i : j;
        Jout[(size_t)e * 72 + 12 * a + c2] = J[12 * a + c2] * sc * scale[off_pose[kf] + (c2 < 6 ? c2 : c2 - 6)];
      }
  }
  const int slots[1] = {slot};
  block_reduce_store<1>(csum, partials, slots);
}

// gather J^T J of IMU (type 0, 15 cols per role) and edge (type 1, 6 cols per role) factors into the lower triangle of
// S, and J^T r into g_c.  One CTA per destination (keyframe hi >= keyframe lo) block, thread (r, c) owns one entry and
// sums its terms in list order.  Because speed-bias columns precede pose columns, an entry whose mapped row index is
// above its column index is stored at the mirrored position; for hi == lo only r >= c is processed.
__global__ void __launch_bounds__(256) factor_gather_kernel(int n_fb, const int* __restrict__ fb_hi, const int* __restrict__ fb_lo,
                                                            const int* __restrict__ fb_ptr, const int* __restrict__ ft_type,
                                                            const int* __restrict__ ft_fac, const int* __restrict__ ft_rhi,
                                                            const int* __restrict__ ft_rlo, const double* __restrict__ Jimu,
                                                            const double* __restrict__ rimu, const double* __restrict__ Jedge,
                                                            const double* __restrict__ redge, const int* __restrict__ off_pose,
                                                            const int* __restrict__ off_sb, int per, SView S,
                                                            double* __restrict__ g_c) {
  const int b = blockIdx.x;
  if (b >= n_fb) return;
  const int hi = fb_hi[b], lo = fb_lo[b];
  const int r = threadIdx.x / 15, c = threadIdx.x % 15;
  if (r >= 15) return;
  if (hi == lo && c > r) return;
  double acc = 0.0, gacc = 0.0;
  bool touched = false;   // an entry no factor of this block reaches is not part of S's structure (edge-only blocks: 6x6)
  for (int t = fb_ptr[b]; t < fb_ptr[b + 1]; t++) {
    const int type = ft_type[t], f = ft_fac[t];
    const int d = type == 0 ? 15 : 6, rows = type == 0 ? 15 : 6, ncol = type == 0 ? 30 : 12;
    if (r >= d || c >= d) continue;
    touched = true;
    const double* J = (type == 0 ? Jimu + (size_t)f * 450 : Jedge + (size_t)f * 72);
    const double* res = (type == 0 ? rimu + (size_t)f * 15 : redge + (size_t)f * 6);
    const int ca = ft_rhi[t] * d + r, cb = ft_rlo[t] * d + c;
    double s = 0.0, gs = 0.0;
    for (int m = 0; m < rows; m++) {
      s += J[ncol * m + ca] * J[ncol * m + cb];
      if (hi == lo && c == 0) gs += J[ncol * m + ca] * res[m];
    }
    acc += s;
    gacc += gs;
  }
  if (touched && r < per && c < per) {
    int ri = cam_col(off_pose, off_sb, hi, r), ci = cam_col(off_pose, off_sb, lo, c);
    if (ri < ci) { const int t2 = ri; ri = ci; ci = t2; }
    *s_at(S, ri, ci) += acc;
  }
  if (touched && hi == lo && c == 0 && r < per) g_c[cam_col(off_pose, off_sb, hi, r)] += gacc;
}

// camera part, step 1: colsq = diag(J^T J) (before damping / Schur)
__global__ void cam_colsq_kernel(int n_c_pad, const double* __restrict__ scale, SView S, double* __restrict__ colsq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_c_pad) return;
  colsq[i] = scale[i] != 0.0 ? *s_at(S, i, i) : 0.0;
}
__global__ void cam_diag_kernel(int n_c_pad, const double* __restrict__ scale, const double* __restrict__ colsq,
                                double* __restrict__ diag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_c_pad) return;
  diag[i] = scale[i] != 0.0 ? sqrt(clamp_diag(colsq[i])) : 1.0;
}
// camera part, step 2 (after the Schur subtraction): damping, reduced gradient, inactive rows → identity.  With a column
// owner map (distributed factorisation) a rank finishes only the diagonal of ITS tile columns — the others' diagonal
// tiles still hold this rank's partial sums, which their owners may be reading over NVLink at this moment.
__global__ void cam_finish_kernel(int n_c_pad, const double* __restrict__ scale, SView S,
                                  const double* __restrict__ diag, const double* __restrict__ g_c,
                                  const double* __restrict__ yb, double* __restrict__ gs, double mu,
                                  const int* __restrict__ col_owner, int rank) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_c_pad) return;
  const bool mine = col_owner == nullptr || col_owner[i >> 7] == rank;
  if (scale[i] != 0.0) {
    const double dg = diag[i];
    if (mine) *s_at(S, i, i) += mu * dg * dg;
    gs[i] = g_c[i] - yb[i];
  } else {
    if (mine) *s_at(S, i, i) = 1.0;
    gs[i] = 0.0;
  }
}

// K7: the Schur complement one hi keyframe k at a time (one CTA): S(k, lo) -= sum over (a, b) pairs of Y_a W_b^T for
// every block of the row, and yb[k] = sum over k's observations of Y b_l.  All Y_a of a row belong to k's observations
// (sp_a holds a's position in kf_obs[k]), so Y = W Hll^-1 is formed once per observation into shared memory and never
// written to HBM; only W_b is gathered.  A row longer than `stage` observations recomputes Y of the rest where it is
// used (same expression).  Summation orders: yb[k] by warp 0, lane-strided over kf_obs[k] then the xor tree; each
// block as by one warp, lane L summing terms L, L+32, ... of the block's pair list, then the xor-16/8/4/2/1 tree.
// A lane without a term holds +0.0 (never -0.0: 0.0 + t is +0.0 for t = -0.0), which adds nothing, so a tree level whose
// partner lanes hold no term is skipped, and two blocks of at most 16 terms share a warp, one per half-warp (levels
// 8/4/2/1 stay inside a half): the entries are bitwise those of the full 32-lane tree.  The lane holding a block's sum
// parks its 36 entries in shared memory, and the warp's lanes then write one entry each.
constexpr int ROW_THREADS = 128;
constexpr int ROW_STAGE_MAX = 512;   // observations staged per row: 72 KB of shared memory, 3 CTAs per SM

__device__ __forceinline__ void row_y(int i, int stage, const double2* __restrict__ ys, const int* __restrict__ kf_obs_k,
                                      const int* __restrict__ obs_lm, const ObsW* __restrict__ ow,
                                      const double* __restrict__ HllInv, double (&y)[18]) {
  if (i < stage) {
#pragma unroll
    for (int j = 0; j < 9; j++) {
      const double2 v = ys[9 * i + j];
      y[2 * j] = v.x;
      y[2 * j + 1] = v.y;
    }
  } else {
    const int o = kf_obs_k[i];
    obs_y(ow[o].W, HllInv + 6 * (size_t)obs_lm[o], y);
  }
}

// acc += Y_a W_b^T over the pair terms p0, p0 + 32, ... < p1
__device__ __forceinline__ void row_block_terms(int p0, int p1, int stage, const double2* __restrict__ ys,
                                                const int* __restrict__ kf_obs_k, const int* __restrict__ obs_lm,
                                                const ObsW* __restrict__ ow, const double* __restrict__ HllInv,
                                                const int* __restrict__ sp_a, const int* __restrict__ sp_b, double (&acc)[36]) {
#pragma unroll
  for (int i = 0; i < 36; i++) acc[i] = 0.0;
  for (int p = p0; p < p1; p += 32) {
    double y[18], w[18];
    row_y(sp_a[p], stage, ys, kf_obs_k, obs_lm, ow, HllInv, y);
    const double2* W = reinterpret_cast<const double2*>(ow[sp_b[p]].W);
#pragma unroll
    for (int j = 0; j < 9; j++) {
      const double2 v = W[j];
      w[2 * j] = v.x;
      w[2 * j + 1] = v.y;
    }
#pragma unroll
    for (int r = 0; r < 6; r++)
#pragma unroll
      for (int c = 0; c < 6; c++) acc[6 * r + c] += y[3 * r] * w[3 * c] + y[3 * r + 1] * w[3 * c + 1] + y[3 * r + 2] * w[3 * c + 2];
  }
}

// the xor tree over the levels whose partner lanes can hold a term: n = the most terms of a block in the warp
__device__ __forceinline__ void row_block_tree(int n, double (&acc)[36]) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1)
    if (n > off)
#pragma unroll
      for (int i = 0; i < 36; i++) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
}

__global__ void __launch_bounds__(ROW_THREADS) schur_row_kernel(int stage, const int* __restrict__ kf_ptr,
                                                                const int* __restrict__ kf_obs, const int* __restrict__ obs_lm,
                                                                const double* __restrict__ HllInv, const double* __restrict__ bl,
                                                                const ObsW* __restrict__ ow, const int* __restrict__ kf_sb,
                                                                const int* __restrict__ sb_lo, const int* __restrict__ sb_ptr,
                                                                const int* __restrict__ sp_a, const int* __restrict__ sp_b,
                                                                const int* __restrict__ off_pose, SView S, double* __restrict__ yb) {
  extern __shared__ double2 ys[];   // [min(n, stage)][9]: Y of the row's observations
  const int k = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int* kf_obs_k = kf_obs + kf_ptr[k];
  const int n = kf_ptr[k + 1] - kf_ptr[k];
  for (int i = threadIdx.x; i < min(n, stage); i += ROW_THREADS) {
    const int o = kf_obs_k[i];
    double y[18];
    obs_y(ow[o].W, HllInv + 6 * (size_t)obs_lm[o], y);
#pragma unroll
    for (int j = 0; j < 9; j++) ys[9 * i + j] = make_double2(y[2 * j], y[2 * j + 1]);
  }
  __syncthreads();
  const int br = off_pose[k];
  if (warp == 0) {
    double v[6];
#pragma unroll
    for (int r = 0; r < 6; r++) v[r] = 0.0;
    for (int i = lane; i < n; i += 32) {
      double y[18];
      row_y(i, stage, ys, kf_obs_k, obs_lm, ow, HllInv, y);
      const double* bb = bl + 3 * (size_t)obs_lm[kf_obs_k[i]];
#pragma unroll
      for (int r = 0; r < 6; r++) v[r] += y[3 * r] * bb[0] + y[3 * r + 1] * bb[1] + y[3 * r + 2] * bb[2];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
      for (int r = 0; r < 6; r++) v[r] += __shfl_xor_sync(0xffffffffu, v[r], off);
    if (lane == 0)
      for (int r = 0; r < 6; r++) yb[br + r] = v[r];
  }
  // two blocks per warp visit: both in one pass (a half-warp each) when both have at most 16 terms, else one after the other
  __shared__ double red_s[ROW_THREADS / 32][72];
  double* red = red_s[warp];
  for (int b = kf_sb[k] + 2 * warp; b < kf_sb[k + 1]; b += 2 * (ROW_THREADS / 32)) {
    const int nb = min(2, kf_sb[k + 1] - b);
    const int n0 = sb_ptr[b + 1] - sb_ptr[b], n1 = nb == 2 ? sb_ptr[b + 2] - sb_ptr[b + 1] : 0;
    double acc[36];
    if (nb == 2 && n0 <= 16 && n1 <= 16) {
      const int h = lane >> 4;
      row_block_terms(sb_ptr[b + h] + (lane & 15), sb_ptr[b + h + 1], stage, ys, kf_obs_k, obs_lm, ow, HllInv, sp_a, sp_b, acc);
      row_block_tree(max(n0, n1), acc);
      if ((lane & 15) == 0)
#pragma unroll
        for (int i = 0; i < 36; i++) red[36 * h + i] = acc[i];
    } else {
      for (int j = 0; j < nb; j++) {
        row_block_terms(sb_ptr[b + j] + lane, sb_ptr[b + j + 1], stage, ys, kf_obs_k, obs_lm, ow, HllInv, sp_a, sp_b, acc);
        row_block_tree(j ? n1 : n0, acc);
        if (lane == 0)
#pragma unroll
          for (int i = 0; i < 36; i++) red[36 * j + i] = acc[i];
      }
    }
    __syncwarp();
    for (int e = lane; e < 36 * nb; e += 32) {
      const int j = e >= 36, r = (e - 36 * j) / 6, c = (e - 36 * j) % 6, lo = sb_lo[b + j];
      // the pose columns are laid out chain by chain, so a block of keyframes k > lo may belong above the diagonal:
      // store it transposed in the lower triangle then
      const int bc = off_pose[lo];
      if (k == lo && c > r) continue;   // diagonal block: lower triangle only (the packed layout has no upper tiles)
      if (br >= bc) *s_at(S, br + r, bc + c) -= red[e];
      else *s_at(S, bc + c, br + r) -= red[e];
    }
    __syncwarp();
  }
}

// Multi-GPU exchange without peer access: the structurally non-zero tiles of the (pre-fill) lower triangle of S are
// packed into one buffer and summed across ranks by the injected all-reduce.  pack: tiles → buffer; unpack: buffer → tiles.
__global__ void __launch_bounds__(256) pack_tiles_kernel(double* __restrict__ St, const int* __restrict__ tid, double* __restrict__ buf,
                                                         int unpack) {
  double2* t = reinterpret_cast<double2*>(St + ((size_t)tid[blockIdx.x] << 14));
  double2* b = reinterpret_cast<double2*>(buf + ((size_t)blockIdx.x << 14));
  for (int u = threadIdx.x; u < cvb_chol::T * cvb_chol::T / 2; u += blockDim.x) {
    if (unpack) t[u] = b[u];
    else b[u] = t[u];
  }
}

// zero the listed tiles of S (one CTA per tile)
__global__ void __launch_bounds__(256) zero_tiles_kernel(double* __restrict__ St, const int* __restrict__ tid) {
  double2* t = reinterpret_cast<double2*>(St + ((size_t)tid[blockIdx.x] << 14));
  for (int u = threadIdx.x; u < cvb_chol::T * cvb_chol::T / 2; u += blockDim.x) t[u] = make_double2(0.0, 0.0);
}

// Reduce-scatter by pull (peer access): the owner of a tile column adds the peers' partial tiles — read straight out of
// their packed arrays over NVLink (same packed offset on every rank) — to its own, in rank order.  One CTA per owned
// exchange tile; 16-byte loads, L1 bypassed (the peers' memory is written by other GPUs between launches).
__global__ void __launch_bounds__(256) reduce_pull_kernel(double* __restrict__ St, double* const* __restrict__ peer_S, int world, int rank,
                                                          const int* __restrict__ tid) {
  const size_t off = (size_t)tid[blockIdx.x] << 14;
  double2* mine = reinterpret_cast<double2*>(St + off);
  for (int u = threadIdx.x; u < cvb_chol::T * cvb_chol::T / 2; u += blockDim.x) {
    double2 acc = make_double2(0.0, 0.0);
    for (int g = 0; g < world; g++) {
      const double2 v = g == rank ? mine[u] : __ldcg(reinterpret_cast<const double2*>(peer_S[g] + off) + u);
      acc.x += v.x;
      acc.y += v.y;
    }
    mine[u] = acc;
  }
}
__global__ void flag_to_double_kernel(const int* __restrict__ flag, double* __restrict__ out) { out[0] = (double)(flag[0] & 1); }

// landmark back-substitution: x_l = Hll^-1 (b_l - sum W^T x_c)
__global__ void backsub_kernel(int L, const int* __restrict__ lm_ptr, const int* __restrict__ obs_kf,
                               const ObsW* __restrict__ ow, const double* __restrict__ HllInv, const double* __restrict__ bl,
                               const double* __restrict__ xc, const int* __restrict__ off_pose, double* __restrict__ xl) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L) return;
  double t[3] = {bl[3 * (size_t)l], bl[3 * (size_t)l + 1], bl[3 * (size_t)l + 2]};
  for (int o = lm_ptr[l]; o < lm_ptr[l + 1]; o++) {
    const double* W = ow[o].W;
    const double* x = xc + off_pose[obs_kf[o]];
#pragma unroll
    for (int a = 0; a < 6; a++) {
      t[0] -= W[3 * a] * x[a];
      t[1] -= W[3 * a + 1] * x[a];
      t[2] -= W[3 * a + 2] * x[a];
    }
  }
  const double* h = HllInv + 6 * (size_t)l;
  xl[3 * (size_t)l + 0] = h[0] * t[0] + h[1] * t[1] + h[2] * t[2];
  xl[3 * (size_t)l + 1] = h[1] * t[0] + h[3] * t[1] + h[4] * t[2];
  xl[3 * (size_t)l + 2] = h[2] * t[0] + h[4] * t[1] + h[5] * t[2];
}

// ------------------------------------------------------------------------------------------------
// J * v over all residual blocks: sums (Jv)^2 and (Jv).r
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) jv_obs_kernel(int n_obs, const int* __restrict__ obs_kf, const int* __restrict__ obs_lm,
                                                     const ObsLin* __restrict__ lin, const double* __restrict__ v,
                                                     const int* __restrict__ off_pose, int n_c_pad,
                                                     double* __restrict__ partials, int slot0) {
  double s[2] = {0.0, 0.0};
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < n_obs; o += gridDim.x * blockDim.x) {
    const ObsLin& L = lin[o];
    const double* vp = v + off_pose[obs_kf[o]];
    const double* vl = v + n_c_pad + 3 * (size_t)obs_lm[o];
    double j0 = 0, j1 = 0;
#pragma unroll
    for (int c = 0; c < 6; c++) { j0 += L.Jp[c] * vp[c]; j1 += L.Jp[6 + c] * vp[c]; }
#pragma unroll
    for (int c = 0; c < 3; c++) { j0 += L.Jl[c] * vl[c]; j1 += L.Jl[3 + c] * vl[c]; }
    s[0] += j0 * j0 + j1 * j1;
    s[1] += j0 * L.r[0] + j1 * L.r[1];
  }
  const int slots[2] = {slot0, slot0 + 1};
  block_reduce_store<2>(s, partials, slots);
}

__global__ void __launch_bounds__(256) jv_factor_kernel(int n_imu, const int* __restrict__ imu_i, const int* __restrict__ imu_j,
                                                        const double* __restrict__ Jimu, const double* __restrict__ rimu,
                                                        int n_edge, const int* __restrict__ ei, const int* __restrict__ ej,
                                                        const double* __restrict__ Jedge, const double* __restrict__ redge,
                                                        const double* __restrict__ v, const int* __restrict__ off_pose,
                                                        const int* __restrict__ off_sb, double* __restrict__ partials,
                                                        int slot0) {
  double s[2] = {0.0, 0.0};
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_imu + n_edge; t += gridDim.x * blockDim.x) {
    if (t < n_imu) {
      const double* J = Jimu + (size_t)t * 450;
      double vi[15], vj[15];
      for (int c = 0; c < 15; c++) {
        vi[c] = v[cam_col(off_pose, off_sb, imu_i[t], c)];
        vj[c] = v[cam_col(off_pose, off_sb, imu_j[t], c)];
      }
      for (int a = 0; a < 15; a++) {
        double jv = 0;
        for (int c = 0; c < 15; c++) jv += J[30 * a + c] * vi[c] + J[30 * a + 15 + c] * vj[c];
        s[0] += jv * jv;
        s[1] += jv * rimu[15 * (size_t)t + a];
      }
    } else {
      const int e = t - n_imu;
      const double* J = Jedge + (size_t)e * 72;
      const double* vi = v + off_pose[ei[e]];
      const double* vj = v + off_pose[ej[e]];
      for (int a = 0; a < 6; a++) {
        double jv = 0;
        for (int c = 0; c < 6; c++) jv += J[12 * a + c] * vi[c] + J[12 * a + 6 + c] * vj[c];
        s[0] += jv * jv;
        s[1] += jv * redge[6 * (size_t)e + a];
      }
    }
  }
  const int slots[2] = {slot0, slot0 + 1};
  block_reduce_store<2>(s, partials, slots);
}

// ------------------------------------------------------------------------------------------------
// vector algebra on [cam | landmark] vectors
// ------------------------------------------------------------------------------------------------
// landmark part of diag / grad / sgrad and the whole-vector versions of grad = g / diag, sgrad = grad / diag
__global__ void prep_vectors_kernel(int n_vec, int n_c_pad, const double* __restrict__ scale, const double* __restrict__ colsq,
                                    double* __restrict__ diag, const double* __restrict__ g, double* __restrict__ grad,
                                    double* __restrict__ sgrad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_vec) return;
  const bool active = scale[i] != 0.0;
  if (i >= n_c_pad) diag[i] = active ? sqrt(clamp_diag(colsq[i])) : 1.0;
  const double d = diag[i];
  const double gr = active ? g[i] / d : 0.0;
  grad[i] = gr;
  sgrad[i] = gr / d;
}

// gn = -x * diag ; sums |gn|^2, |grad|^2, grad.gn
__global__ void __launch_bounds__(256) gn_norms_kernel(int n_vec, const double* __restrict__ x, const double* __restrict__ diag,
                                                       const double* __restrict__ grad, const double* __restrict__ scale,
                                                       double* __restrict__ gn, int n_c_pad, double cam_w,
                                                       double* __restrict__ partials, int slot0) {
  double s[3] = {0, 0, 0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += gridDim.x * blockDim.x) {
    const double v = scale[i] != 0.0 ? -x[i] * diag[i] : 0.0;
    gn[i] = v;
    const double w = i < n_c_pad ? cam_w : 1.0;
    s[0] += w * v * v;
    s[1] += w * grad[i] * grad[i];
    s[2] += w * grad[i] * v;
  }
  const int slots[3] = {slot0, slot0 + 1, slot0 + 2};
  block_reduce_store<3>(s, partials, slots);
}

// step = (ca * grad + cb * gn) / diag ; also |ca grad + cb gn|^2
__global__ void __launch_bounds__(256) dogleg_combine_kernel(int n_vec, double ca, double cb, const double* __restrict__ grad,
                                                             const double* __restrict__ gn, const double* __restrict__ diag,
                                                             const double* __restrict__ scale, double* __restrict__ step,
                                                             int n_c_pad, double cam_w, double* __restrict__ partials,
                                                             int slot0) {
  double s[1] = {0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += gridDim.x * blockDim.x) {
    const double d = ca * grad[i] + cb * gn[i];
    s[0] += (i < n_c_pad ? cam_w : 1.0) * d * d;
    step[i] = scale[i] != 0.0 ? d / diag[i] : 0.0;
  }
  const int slots[1] = {slot0};
  block_reduce_store<1>(s, partials, slots);
}

// candidate = Plus(current, step * scale); sums |cand - cur|^2 (ambient) and |cand|^2 over non-constant blocks
__global__ void __launch_bounds__(256) plus_kernel(int K, int L, const int* __restrict__ off_pose, const int* __restrict__ off_sb,
                                                   int n_c_pad, int visual_only,
                                                   const uint8_t* __restrict__ pose_const, const double* __restrict__ step,
                                                   const double* __restrict__ scale, const double* __restrict__ pose,
                                                   const double* __restrict__ sb, const double* __restrict__ lm,
                                                   double* __restrict__ cpose, double* __restrict__ csb, double* __restrict__ clm,
                                                   double cam_w, double* __restrict__ partials, int slot0) {
  double s[2] = {0, 0};
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < K + L; t += gridDim.x * blockDim.x) {
    if (t < K) {
      const int k = t;
      double d[6], out[7];
      const bool cst = pose_const[k] != 0;
      for (int c = 0; c < 6; c++) d[c] = cst ? 0.0 : step[off_pose[k] + c] * scale[off_pose[k] + c];
      if (cst) {
        for (int c = 0; c < 7; c++) out[c] = pose[7 * k + c];
      } else {
        pose_plus(pose + 7 * k, d, out);
      }
      for (int c = 0; c < 7; c++) {
        cpose[7 * k + c] = out[c];
        const double df = out[c] - pose[7 * k + c];
        s[0] += cam_w * df * df;
        if (!cst) s[1] += cam_w * out[c] * out[c];
      }
      for (int c = 0; c < 9; c++) {
        double v = sb[9 * k + c];
        if (!visual_only) {
          const double dd = step[off_sb[k] + c] * scale[off_sb[k] + c];
          v += dd;
          s[0] += cam_w * dd * dd;
          s[1] += cam_w * v * v;
        }
        csb[9 * k + c] = v;
      }
    } else {
      const int l = t - K;
      const bool own = scale[n_c_pad + 3 * (size_t)l] != 0.0;   // landmarks of other ranks are not touched here
      for (int c = 0; c < 3; c++) {
        const double dd = step[n_c_pad + 3 * (size_t)l + c] * scale[n_c_pad + 3 * (size_t)l + c];
        const double v = lm[3 * (size_t)l + c] + dd;
        clm[3 * (size_t)l + c] = v;
        if (own) {
          s[0] += dd * dd;
          s[1] += v * v;
        }
      }
    }
  }
  const int slots[2] = {slot0, slot0 + 1};
  block_reduce_store<2>(s, partials, slots);
}

// Jacobi scaling from the unscaled column norms: 1 / (1 + sqrt(colsq)); 0 for inactive columns
__global__ void jacobi_scale_kernel(int n_vec, const double* __restrict__ colsq, double* __restrict__ scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_vec) return;
  if (scale[i] != 0.0) scale[i] = 1.0 / (1.0 + sqrt(colsq[i]));
}

__global__ void max_abs_grad_kernel(int n_vec, const double* __restrict__ g, const double* __restrict__ scale,
                                    double* __restrict__ partials, int slot) {
  __shared__ double sm[256];
  double m = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += gridDim.x * blockDim.x)
    if (scale[i] != 0.0) m = fmax(m, fabs(g[i] / scale[i]));
  sm[threadIdx.x] = m;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] = fmax(sm[threadIdx.x], sm[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) partials[slot * RED_BLOCKS + blockIdx.x] = sm[0];
}
// the rank's maximum goes to rankmax[rank] of a zeroed world-sized vector: a SUM all-reduce of that vector hands every
// rank all the local maxima (the injected collective is sum-only)
__global__ void max_final_kernel(const double* __restrict__ partials, double* __restrict__ scalars, int slot,
                                 double* __restrict__ rankmax, int rank, int world) {
  double m = 0.0;
  for (int i = 0; i < RED_BLOCKS; i++) m = fmax(m, partials[slot * RED_BLOCKS + i]);
  scalars[slot] = m;
  for (int r = 0; r < world; r++) rankmax[r] = (r == rank) ? m : 0.0;
}
__global__ void max_ranks_kernel(const double* __restrict__ rankmax, int world, double* __restrict__ scalars, int slot) {
  double m = 0.0;
  for (int r = 0; r < world; r++) m = fmax(m, rankmax[r]);
  scalars[slot] = m;
}

}  // namespace

// =================================================================================================
// Host side
// =================================================================================================
namespace {

#define ENG_CUDA(call)                                                                                       \
  do {                                                                                                       \
    cudaError_t e_ = (call);                                                                                 \
    if (e_ != cudaSuccess)                                                                                   \
      return cvb_fail(E.ctx, CVB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, \
                      __LINE__);                                                                             \
  } while (0)
#define ENG_LAUNCH() CVB_CHECK_LAUNCH(E.ctx)

template <typename T>
int upload(Engine& E, cvb_dev_arr<T>& d, const T* h, size_t n) {
  if (d.alloc(n, E.st)) return cvb_fail(E.ctx, CVB_ERR_CUDA, "cudaMalloc failed (%zu bytes)", n * sizeof(T));
  if (n) ENG_CUDA(cudaMemcpyAsync(d.p, h, n * sizeof(T), cudaMemcpyHostToDevice, E.st));
  return CVB_OK;
}
template <typename T>
int upload(Engine& E, cvb_dev_arr<T>& d, const std::vector<T>& h) {
  return upload(E, d, h.data(), h.size());
}
// for_ipc: see cvb_dev_arr
template <typename T>
int zalloc(Engine& E, cvb_dev_arr<T>& d, size_t n, bool for_ipc = false) {
  if (d.alloc(n, E.st, for_ipc)) return cvb_fail(E.ctx, CVB_ERR_CUDA, "cudaMalloc failed (%zu bytes)", n * sizeof(T));
  ENG_CUDA(cudaMemsetAsync(d.p, 0, (n ? n : 1) * sizeof(T), E.st));
  return CVB_OK;
}

inline int grid1(size_t n, int b = 256) { return (int)((n + b - 1) / b); }

int ar(Engine& E, double* p, size_t n) {
  if (E.allreduce && E.world > 1) {
    int rc = E.allreduce(p, n);
    if (rc) return cvb_fail(E.ctx, CVB_ERR_CUDA, "allreduce callback failed (%d)", rc);
  }
  return CVB_OK;
}

int read_scalars(Engine& E, int nslots) {
  reduce_final<<<1, 256, 0, E.st>>>(E.partials.p, E.scalars.p, nslots, 0);
  ENG_LAUNCH();
  if (int rc = ar(E, E.scalars.p, (size_t)nslots)) return rc;
  ENG_CUDA(cudaMemcpyAsync(E.h_scalars, E.scalars.p, nslots * sizeof(double), cudaMemcpyDeviceToHost, E.st));
  ENG_CUDA(cudaStreamSynchronize(E.st));
  return CVB_OK;
}

// ---- Schur (block → observation-pair) lists, built on the device -----------------------------------------------
// For every S block (hi keyframe, lo keyframe) the Schur kernel needs the list of observation pairs (a, b) of the
// landmarks seen by both, in landmark order (fixed summation order → bit-reproducible).  3.6 M pairs at C3: generated by
// one thread per landmark, ordered by two stable LSD radix sorts (cub) over the keyframe indices, run-length encoded.
// (The host version of the same — two counting-sort passes — cost 120 ms of the 180 ms problem set-up.)
__global__ void gen_pairs_kernel(int L_in, const int* __restrict__ lm_ptr, const long long* __restrict__ pair_ptr,
                                 const int* __restrict__ obs_kf, unsigned long long* __restrict__ keys,
                                 unsigned long long* __restrict__ vals) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L_in) return;
  long long o = pair_ptr[l];
  const int o0 = lm_ptr[l], o1 = lm_ptr[l + 1];
  for (int a = o0; a < o1; a++) {
    const unsigned long long hi = (unsigned long long)(unsigned)obs_kf[a] << 32;
    for (int b = o0; b <= a; b++, o++) {
      keys[o] = hi | (unsigned)obs_kf[b];
      vals[o] = ((unsigned long long)(unsigned)a << 32) | (unsigned)b;
    }
  }
}
__global__ void pair_heads_kernel(long long np, const unsigned long long* __restrict__ keys, int* __restrict__ head) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < np) head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}
// position of every observation in its keyframe's kf_obs list
__global__ void kf_pos_kernel(int n_obs, const int* __restrict__ kf_ptr, const int* __restrict__ kf_obs,
                              const int* __restrict__ obs_kf, int* __restrict__ pos) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_obs) return;
  const int o = kf_obs[e];
  pos[o] = e - kf_ptr[obs_kf[o]];
}
// sp_a: a's position in kf_obs[hi] (schur_row_kernel finds Y_a there); sp_b: the observation b
__global__ void pair_scatter_kernel(long long np, const unsigned long long* __restrict__ keys,
                                    const unsigned long long* __restrict__ vals, const int* __restrict__ head,
                                    const int* __restrict__ blk /*exclusive scan of head*/, const int* __restrict__ kf_pos,
                                    int* __restrict__ sb_hi, int* __restrict__ sb_lo, int* __restrict__ sb_ptr,
                                    int* __restrict__ sp_a, int* __restrict__ sp_b) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const unsigned long long v = vals[i];
  sp_a[i] = kf_pos[v >> 32];
  sp_b[i] = (int)(v & 0xffffffffu);
  if (head[i]) {
    const int bidx = blk[i];
    sb_hi[bidx] = (int)(keys[i] >> 32);
    sb_lo[bidx] = (int)(keys[i] & 0xffffffffu);
    sb_ptr[bidx] = (int)i;
  }
}
// kf_sb[k] = first block whose hi keyframe is >= k (blocks are sorted by hi), k = 0..K
__global__ void kf_sb_kernel(int K, int n_sb, const int* __restrict__ sb_hi, int* __restrict__ kf_sb) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > K) return;
  int lo = 0, hi = n_sb;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sb_hi[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  kf_sb[k] = lo;
}

int build_schur_lists(Engine& E, const std::vector<int>& h_lm_ptr, int K) {
  std::vector<long long> h_pair_ptr((size_t)E.L_in + 1, 0);
  for (int l = 0; l < E.L_in; l++) {
    const long long n = h_lm_ptr[l + 1] - h_lm_ptr[l];
    h_pair_ptr[l + 1] = h_pair_ptr[l] + n * (n + 1) / 2;
  }
  const long long np = h_pair_ptr[E.L_in];
  if (np >= (1LL << 31)) return cvb_fail(E.ctx, CVB_ERR_UNSUPPORTED, "more than 2^31 Schur observation pairs");
  int rc;
  if ((rc = zalloc(E, E.sp_a, (size_t)np)) || (rc = zalloc(E, E.sp_b, (size_t)np)) || (rc = zalloc(E, E.kf_sb, (size_t)K + 1)))
    return rc;
  E.n_sb = 0;
  if (np == 0) {
    if ((rc = zalloc(E, E.sb_hi, 0)) || (rc = zalloc(E, E.sb_lo, 0)) || (rc = zalloc(E, E.sb_ptr, 1))) return rc;
    return CVB_OK;
  }
  cvb_dev_arr<long long> d_pair_ptr;
  cvb_dev_arr<unsigned long long> k0, k1, v0, v1;
  cvb_dev_arr<int> head, blk, kf_pos;
  cvb_dev_arr<unsigned char> tmp;
  if ((rc = upload(E, d_pair_ptr, h_pair_ptr))) return rc;
  if (k0.alloc((size_t)np, E.st) || k1.alloc((size_t)np, E.st) || v0.alloc((size_t)np, E.st) || v1.alloc((size_t)np, E.st) ||
      head.alloc((size_t)np + 1, E.st) || blk.alloc((size_t)np + 1, E.st) || kf_pos.alloc((size_t)E.n_obs, E.st))
    return cvb_fail(E.ctx, CVB_ERR_CUDA, "cudaMalloc failed (Schur pair scratch, %lld pairs)", np);
  kf_pos_kernel<<<grid1((size_t)E.n_obs), 256, 0, E.st>>>(E.n_obs, E.kf_ptr.p, E.kf_obs.p, E.obs_kf.p, kf_pos.p);
  ENG_LAUNCH();
  gen_pairs_kernel<<<grid1((size_t)E.L_in), 256, 0, E.st>>>(E.L_in, E.lm_ptr.p, d_pair_ptr.p, E.obs_kf.p, k0.p, v0.p);
  ENG_LAUNCH();
  int bits = 1;
  while ((1 << bits) < K) bits++;
  size_t t1 = 0, t2 = 0, t3 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t1, k0.p, k1.p, v0.p, v1.p, (int)np, 0, bits, E.st);
  cub::DeviceRadixSort::SortPairs(nullptr, t2, k1.p, k0.p, v1.p, v0.p, (int)np, 32, 32 + bits, E.st);
  cub::DeviceScan::ExclusiveSum(nullptr, t3, head.p, blk.p, (int)np + 1, E.st);
  size_t tb = std::max(t1, std::max(t2, t3));
  if (tmp.alloc(tb ? tb : 1, E.st)) return cvb_fail(E.ctx, CVB_ERR_CUDA, "cudaMalloc failed (sort scratch)");
  ENG_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, k0.p, k1.p, v0.p, v1.p, (int)np, 0, bits, E.st));        // by lo keyframe
  ENG_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, tb, k1.p, k0.p, v1.p, v0.p, (int)np, 32, 32 + bits, E.st));  // by hi (stable)
  pair_heads_kernel<<<grid1((size_t)np), 256, 0, E.st>>>(np, k0.p, head.p);
  ENG_LAUNCH();
  ENG_CUDA(cudaMemsetAsync(head.p + np, 0, sizeof(int), E.st));
  ENG_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, tb, head.p, blk.p, (int)np + 1, E.st));
  int n_sb = 0;
  ENG_CUDA(cudaMemcpyAsync(&n_sb, blk.p + np, sizeof(int), cudaMemcpyDeviceToHost, E.st));
  ENG_CUDA(cudaStreamSynchronize(E.st));
  E.n_sb = n_sb;
  if ((rc = zalloc(E, E.sb_hi, (size_t)n_sb)) || (rc = zalloc(E, E.sb_lo, (size_t)n_sb)) || (rc = zalloc(E, E.sb_ptr, (size_t)n_sb + 1)))
    return rc;
  pair_scatter_kernel<<<grid1((size_t)np), 256, 0, E.st>>>(np, k0.p, v0.p, head.p, blk.p, kf_pos.p, E.sb_hi.p, E.sb_lo.p,
                                                          E.sb_ptr.p, E.sp_a.p, E.sp_b.p);
  ENG_LAUNCH();
  kf_sb_kernel<<<grid1((size_t)K + 1), 256, 0, E.st>>>(K, n_sb, E.sb_hi.p, E.kf_sb.p);
  ENG_LAUNCH();
  const int np_i = (int)np;
  ENG_CUDA(cudaMemcpyAsync(E.sb_ptr.p + n_sb, &np_i, sizeof(int), cudaMemcpyHostToDevice, E.st));
  ENG_CUDA(cudaStreamSynchronize(E.st));   // scratch arrays are freed on return
  return CVB_OK;
}

// the host-side checks of a problem (cvb_ba_create's refusals; the group drivers run them before starting any rank)
int check_problem(cvb_ctx* ctx, const cvb_ba_problem* p, int visual_only) {
  CVB_REQUIRE(ctx, p->K > 0, "problem has no keyframes");
  const int K = p->K;
  CVB_REQUIRE(ctx, p->n_imu >= 0 && p->n_edge >= 0 && p->L >= 0, "negative problem size");
  if (!visual_only)
    for (int f = 0; f < p->n_imu; f++)
      CVB_REQUIRE(ctx, p->imu_i[f] >= 0 && p->imu_i[f] < K && p->imu_j[f] >= 0 && p->imu_j[f] < K && p->imu_i[f] != p->imu_j[f],
                  "bad IMU factor indices");
  for (int e = 0; e < p->n_edge; e++)
    CVB_REQUIRE(ctx, p->edge_i[e] >= 0 && p->edge_i[e] < K && p->edge_j[e] >= 0 && p->edge_j[e] < K && p->edge_i[e] != p->edge_j[e],
                "bad edge indices");
  for (int l = 0; l < p->L; l++)
    for (int ob = p->lm_obs_ptr[l]; ob < p->lm_obs_ptr[l + 1]; ob++)
      CVB_REQUIRE(ctx, p->obs_kf[ob] >= 0 && p->obs_kf[ob] < K, "obs_kf out of range");
  return CVB_OK;
}

// The connected components of the keyframes 0..K-1 under links (pairs of keyframes) that have at least min_size
// keyframes: each in ascending keyframe order, the components in order of their first keyframe.
std::vector<std::vector<int>> kf_components(int K, const std::vector<std::pair<int, int>>& links, int min_size) {
  std::vector<int> parent(K);
  std::iota(parent.begin(), parent.end(), 0);
  const auto find = [&](int x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
  for (const auto& l : links) {
    const int a = find(l.first), b = find(l.second);
    if (a != b) parent[std::max(a, b)] = std::min(a, b);   // the root of a component is its first keyframe
  }
  std::vector<std::vector<int>> of_root(K), comps;
  for (int k = 0; k < K; k++) of_root[find(k)].push_back(k);
  for (auto& c : of_root)
    if ((int)c.size() >= min_size) comps.push_back(std::move(c));
  return comps;
}

// Column layout of the reduced camera system (see cam_col()): the first column of every keyframe's pose block (off_pose)
// and speed-bias block (off_sb), and the column group of every tile nd_layout() laid out; returns the number of columns.
// The factorisation's schedule, and so the bits of the result, depend on this layout.
int column_layout(const cvb_ba_problem* p, bool visual_only, bool pose_graph, std::vector<int>& off_pose, std::vector<int>& off_sb,
                  std::vector<int>& group_of_tile) {
  const int K = p->K, TT = cvb_chol::T;
  const auto pad = [TT](int c) { return ((c + TT - 1) / TT) * TT; };
  off_pose.resize(K); off_sb.assign(K, 0);
  group_of_tile.clear();
  std::vector<char> in_chain(K, 0);
  if (!visual_only) {
    // [speed-bias blocks (9 each) | pad to a tile | pose blocks (6 each)].  Every IMU chain (connected component of the
    // IMU factor graph, i.e. one agent's trajectory) starts on a tile boundary, so that the tile-level elimination of one
    // chain never touches another chain's tiles (a tile shared by two chains would carry the first chain's pose clique
    // along the whole second chain).
    std::vector<std::pair<int, int>> links;
    for (int f = 0; f < p->n_imu; f++) links.push_back({p->imu_i[f], p->imu_j[f]});
    const auto chains = kf_components(K, links, 2);
    for (const auto& c : chains)
      for (int k : c) in_chain[k] = 1;
    int cursor = cvb_chol::nd_layout(chains, 9, off_sb, group_of_tile) * TT;
    for (int k = 0; k < K; k++)                     // keyframes without an IMU factor: isolated speed-bias blocks
      if (!in_chain[k]) { off_sb[k] = cursor; cursor += 9; }
    // poses: chain by chain, each chain on its own tiles (so that the chains' eliminations touch disjoint tiles and
    // can run concurrently), then the keyframes without IMU factors
    for (const auto& c : chains) {
      cursor = pad(cursor);
      for (int k : c) { off_pose[k] = cursor; cursor += 6; }
    }
    cursor = pad(cursor);
    for (int k = 0; k < K; k++)
      if (!in_chain[k]) { off_pose[k] = cursor; cursor += 6; }
    return cursor;
  }
  if (pose_graph) {
    // Pose graph (PoseGraphOptimization: no landmarks, only between-factors): the keyframes of one agent form a banded chain
    // (successor + 5 predecessor edges, optimization_be.cpp:947-1021) and the few loop edges couple distant keyframes.  In
    // plain keyframe order the tile columns are one long dependent chain (94 columns x ~100 us at C3).  Nested dissection
    // by hand: the endpoints of long-range edges go to a per-chain BORDER segment at the end; what remains are independent
    // banded chains, each laid out on its own tiles → they are eliminated concurrently as column groups (like the IMU chains
    // of the visual-inertial problem), then the small border is factored.  A chain's columns only ever touch its own tiles
    // and its own border segment, so concurrent groups never update the same tile.
    std::vector<char> border(K, 0);
    std::vector<std::pair<int, int>> links;   // a chain = connected through short-range edges (border keyframes included)
    for (int e = 0; e < p->n_edge; e++) {
      if (std::abs(p->edge_i[e] - p->edge_j[e]) > 8) border[p->edge_i[e]] = border[p->edge_j[e]] = 1;
      else links.push_back({p->edge_i[e], p->edge_j[e]});
    }
    const auto chains = kf_components(K, links, 64);
    std::vector<std::vector<int>> members;    // interiors of the big chains: one column group each
    for (const auto& c : chains) {
      members.emplace_back();
      for (int k : c) {
        in_chain[k] = 1;
        if (!border[k]) members.back().push_back(k);
      }
      if (members.back().empty()) members.pop_back();
    }
    int cursor = cvb_chol::nd_layout(members, 6, off_pose, group_of_tile) * TT;
    for (int k = 0; k < K; k++)                   // small components: main sequence
      if (!in_chain[k]) { off_pose[k] = cursor; cursor += 6; }
    for (const auto& c : chains) {                // per-chain border segments
      cursor = pad(cursor);
      for (int k : c)
        if (border[k]) { off_pose[k] = cursor; cursor += 6; }
    }
    return cursor;
  }
  for (int k = 0; k < K; k++) off_pose[k] = 6 * k;
  return 6 * K;
}

// fill (cvb_ba_solve_dev_edges, single rank only): the start poses and edge measurements are written on the device by
// fill(pose[0], pose0, edge_q, edge_t, edge_S) instead of uploaded from p->pose / edge_q / edge_t / edge_sqrt_info
int engine_setup(Engine& E, const cvb_ba_problem* p, const cvb_ba_options* o, const cvb_dev_edges_fill* fill = nullptr) {
  cvb_ctx* ctx = E.ctx;
  const bool trace = getenv("COVINS_B200_SETUP_TRACE") != nullptr;   // development aid: host-side phase times to stderr
  auto t_prev = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!trace) return;
    const auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[setup] %-28s %8.2f ms\n", what, std::chrono::duration<double, std::milli>(now - t_prev).count());
    t_prev = now;
  };
  E.visual_only = o->visual_only ? 1 : 0;
  E.per = E.visual_only ? 6 : 15;
  E.K = p->K;
  E.a2_reproj = o->cauchy_reproj > 0 ? o->cauchy_reproj * o->cauchy_reproj : 0.0;
  E.a2_edge = o->cauchy_edge > 0 ? o->cauchy_edge * o->cauchy_edge : 0.0;
  E.rank = o->rank;
  E.world = o->world > 0 ? o->world : 1;
  CVB_REQUIRE(ctx, E.rank >= 0 && E.rank < E.world, "bad rank/world");
  int rc = check_problem(ctx, p, E.visual_only);
  if (rc) return rc;
  const int K = p->K;
  // ---- landmarks with >= 2 usable observations (opt.cpp:158-171, 438-453), observations of this rank's landmarks ----
  std::vector<int> lm_compact(p->L > 0 ? p->L : 0, -1);
  E.lm_of_compact.clear();
  E.obs_of_compact.clear();
  std::vector<int> h_obs_kf, h_obs_lm, h_lm_ptr(1, 0);
  std::vector<double> h_uv, h_sigma, h_lm;
  for (int l = 0; l < p->L; l++) {
    int cnt = 0;
    for (int ob = p->lm_obs_ptr[l]; ob < p->lm_obs_ptr[l + 1]; ob++)
      if (!(p->obs_skip && p->obs_skip[ob])) cnt++;
    if (cnt < 2) continue;
    lm_compact[l] = (int)E.lm_of_compact.size();
    E.lm_of_compact.push_back(l);
    h_lm.push_back(p->lm[3 * (size_t)l]); h_lm.push_back(p->lm[3 * (size_t)l + 1]); h_lm.push_back(p->lm[3 * (size_t)l + 2]);
    // landmark blocks are sharded across ranks: a rank linearises only its own landmarks' observations
    const bool mine = (lm_compact[l] % E.world) == E.rank;
    if (mine) {
      int prev = -1;
      for (int ob = p->lm_obs_ptr[l]; ob < p->lm_obs_ptr[l + 1]; ob++) {
        if (p->obs_skip && p->obs_skip[ob]) continue;
        const int kf = p->obs_kf[ob];
        CVB_REQUIRE(ctx, kf > prev, "observations of a landmark must be sorted by keyframe index and unique");
        prev = kf;
        h_obs_kf.push_back(kf);
        h_obs_lm.push_back(lm_compact[l]);
        h_uv.push_back((double)p->obs_uv[2 * (size_t)ob]); h_uv.push_back((double)p->obs_uv[2 * (size_t)ob + 1]);
        h_sigma.push_back(p->obs_sigma[ob]);
        E.obs_of_compact.push_back(ob);
      }
    }
    h_lm_ptr.push_back((int)h_obs_kf.size());
  }
  E.L_in = (int)E.lm_of_compact.size();
  E.n_obs = (int)h_obs_kf.size();
  E.n_c = K * E.per;
  std::vector<int> group_of_tile;   // column group of every tile cvb_chol::nd_layout() laid out (tiles 0, 1, ...)
  const int n_total = column_layout(p, E.visual_only, E.L_in == 0 && p->n_edge > 0, E.h_off_pose, E.h_off_sb, group_of_tile);
  const int TT = cvb_chol::T;
  E.n_c_pad = ((n_total + TT - 1) / TT) * TT;
  E.n_vec = E.n_c_pad + 3 * E.L_in;
  auto col_of = [&](int kf, int c) { return c < 6 ? E.h_off_pose[kf] + c : E.h_off_sb[kf] + (c - 6); };
  lap("landmarks / observations");
  // ---- tile-level structure of S (every rank needs the structure of the WHOLE problem: S is all-reduced) ----
  const int nt = E.n_c_pad / TT;
  std::vector<uint8_t> tmask((size_t)nt * nt, 0);
  auto mark = [&](int a0, int alen, int b0, int blen) {
    for (int ta = a0 / TT; ta <= (a0 + alen - 1) / TT; ta++)
      for (int tb = b0 / TT; tb <= (b0 + blen - 1) / TT; tb++) tmask[(size_t)std::max(ta, tb) * nt + std::min(ta, tb)] = 1;
  };
  {
    // a landmark couples the pose blocks of all its observers pairwise: mark the pairs of the DISTINCT tiles they touch
    // (a landmark's ~8 observers fall into a handful of tiles, so this is several times cheaper than walking the pairs)
    std::vector<int> ts;
    for (int l = 0; l < p->L; l++) {
      if (lm_compact[l] < 0) continue;
      ts.clear();
      for (int a = p->lm_obs_ptr[l]; a < p->lm_obs_ptr[l + 1]; a++) {
        if (p->obs_skip && p->obs_skip[a]) continue;
        const int o0 = E.h_off_pose[p->obs_kf[a]];
        for (int t = o0 / TT; t <= (o0 + 5) / TT; t++)
          if (std::find(ts.begin(), ts.end(), t) == ts.end()) ts.push_back(t);
      }
      for (size_t x = 0; x < ts.size(); x++)
        for (size_t y = 0; y <= x; y++) tmask[(size_t)std::max(ts[x], ts[y]) * nt + std::min(ts[x], ts[y])] = 1;
    }
  }
  if (!E.visual_only)
    for (int f = 0; f < p->n_imu; f++) {
      const int ij[2] = {p->imu_i[f], p->imu_j[f]};
      for (int a = 0; a < 2; a++)
        for (int b = 0; b < 2; b++) {
          mark(E.h_off_pose[ij[a]], 6, E.h_off_pose[ij[b]], 6);
          mark(E.h_off_pose[ij[a]], 6, E.h_off_sb[ij[b]], 9);
          mark(E.h_off_sb[ij[a]], 9, E.h_off_sb[ij[b]], 9);
        }
    }
  for (int e = 0; e < p->n_edge; e++) {
    mark(E.h_off_pose[p->edge_i[e]], 6, E.h_off_pose[p->edge_j[e]], 6);
    mark(E.h_off_pose[p->edge_i[e]], 6, E.h_off_pose[p->edge_i[e]], 6);
    mark(E.h_off_pose[p->edge_j[e]], 6, E.h_off_pose[p->edge_j[e]], 6);
  }
  // column groups (IMU chains) first: the owner map of a distributed factorisation follows them
  std::vector<int> col_group(nt, -1);
  std::copy(group_of_tile.begin(), group_of_tile.end(), col_group.begin());
  // ownership of the tile columns (world > 1): an IMU chain's speed-bias columns — a pure latency chain — stay on one
  // rank, the remaining (pose) columns go round the ranks in blocks of COVINS_B200_DIST_BLOCK columns (default 6: every
  // change of owner puts a flag + a 128 KB NVLink copy on the critical chain; tools/mgpu_block_sweep.py)
  std::vector<int> h_owner;
  if (E.world > 1) {
    int blk = 6;
    if (const char* e = getenv("COVINS_B200_DIST_BLOCK")) blk = std::max(1, atoi(e));
    h_owner.assign(nt, 0);
    int seq = 0;
    for (int k = 0; k < nt; k++) {
      if (col_group[k] >= 0) h_owner[k] = col_group[k] % E.world;
      else h_owner[k] = ((seq++) / blk) % E.world;
    }
  }
  std::vector<uint8_t> pre_fill(tmask);
  // the replicated plan (every rank applies every update); cvb_ba_enable_p2p swaps in the owner-filtered one — same tile
  // structure, same packed layout — once peer access is known to work on every rank
  E.plan.build(nt, tmask, col_group);
  E.h_prefill = pre_fill;
  E.h_owner = h_owner;
  E.n_tiles = (size_t)E.plan.n_tiles_L;
  std::vector<int> h_xt_all, h_xt_own;
  for (int j = 0; j < nt; j++)
    for (int i = j; i < nt; i++)
      if (pre_fill[(size_t)i * nt + j] || i == j) {
        const int id = E.plan.h_tile_of[(size_t)i * nt + j];
        h_xt_all.push_back(id);
        if (E.world > 1 && h_owner[j] == E.rank) h_xt_own.push_back(id);
      }
  E.n_xt_all = (int)h_xt_all.size();
  E.n_xt_own = (int)h_xt_own.size();
  std::vector<int> h_xt_fill;
  for (int j = 0; j < nt; j++)
    for (int i = j; i < nt; i++)
      if (!(pre_fill[(size_t)i * nt + j] || i == j) && E.plan.h_tile_of[(size_t)i * nt + j] >= 0)
        h_xt_fill.push_back(E.plan.h_tile_of[(size_t)i * nt + j]);
  E.n_xt_fill = (int)h_xt_fill.size();
  if ((size_t)E.n_xt_all + E.n_xt_fill != E.n_tiles)
    return cvb_fail(E.ctx, CVB_ERR_CUDA, "tile lists (%d + %d) do not cover S (%zu tiles)", E.n_xt_all, E.n_xt_fill, E.n_tiles);
  lap("tile structure + plan");
  // ---- by-keyframe CSR ----
  std::vector<int> h_kf_ptr(K + 1, 0), h_kf_obs(E.n_obs);
  for (int ob = 0; ob < E.n_obs; ob++) h_kf_ptr[h_obs_kf[ob] + 1]++;
  for (int k = 0; k < K; k++) h_kf_ptr[k + 1] += h_kf_ptr[k];
  {
    std::vector<int> fill(h_kf_ptr.begin(), h_kf_ptr.end() - 1);
    for (int ob = 0; ob < E.n_obs; ob++) h_kf_obs[fill[h_obs_kf[ob]]++] = ob;
  }
  E.row_stage = 0;
  for (int k = 0; k < K; k++) E.row_stage = std::max(E.row_stage, std::min(h_kf_ptr[k + 1] - h_kf_ptr[k], ROW_STAGE_MAX));
  {   // the attribute is shared by every engine on the device (ranks of a group among them): the largest stage any may use
    static cvb_once_per_device once;
    std::lock_guard<std::mutex> once_lk(once.mtx);
    if (once.first(E.ctx->device))
      ENG_CUDA(cudaFuncSetAttribute(schur_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ROW_STAGE_MAX * 18 * (int)sizeof(double)));
  }
  lap("by-keyframe CSR");
  // ---- Schur (block → pair) lists: built on the device after the observation arrays are uploaded (build_schur_lists) ----
  lap("Schur pair lists");
  // ---- factors of this rank (round-robin) and their gather lists ----
  std::vector<int> h_imu_i, h_imu_j, sel_imu;
  if (!E.visual_only)
    for (int f = 0; f < p->n_imu; f++) {
      if (f % E.world != E.rank) continue;
      CVB_REQUIRE(ctx, p->imu_ptr[f + 1] > p->imu_ptr[f], "IMU factor with 0 measurements (drop it: opt.cpp:382-385)");
      h_imu_i.push_back(p->imu_i[f]);
      h_imu_j.push_back(p->imu_j[f]);
      sel_imu.push_back(f);
    }
  E.n_imu = (int)h_imu_i.size();
  std::vector<int> h_edge_i, h_edge_j, sel_edge;
  for (int e = 0; e < p->n_edge; e++) {
    if (e % E.world != E.rank) continue;
    h_edge_i.push_back(p->edge_i[e]);
    h_edge_j.push_back(p->edge_j[e]);
    sel_edge.push_back(e);
  }
  E.n_edge = (int)h_edge_i.size();
  struct Term { uint64_t key; int type, fac, rhi, rlo; };
  std::vector<Term> terms;
  auto add_terms = [&](int type, int f, int i, int j) {
    terms.push_back({((uint64_t)i << 32) | (uint32_t)i, type, f, 0, 0});
    terms.push_back({((uint64_t)j << 32) | (uint32_t)j, type, f, 1, 1});
    if (i > j) terms.push_back({((uint64_t)i << 32) | (uint32_t)j, type, f, 0, 1});
    else terms.push_back({((uint64_t)j << 32) | (uint32_t)i, type, f, 1, 0});
  };
  for (int f = 0; f < E.n_imu; f++) add_terms(0, f, h_imu_i[f], h_imu_j[f]);
  for (int e = 0; e < E.n_edge; e++) add_terms(1, e, h_edge_i[e], h_edge_j[e]);
  std::stable_sort(terms.begin(), terms.end(), [](const Term& a, const Term& b) { return a.key < b.key; });
  std::vector<int> h_fb_hi, h_fb_lo, h_fb_ptr, h_ft_type, h_ft_fac, h_ft_rhi, h_ft_rlo;
  for (size_t i = 0; i < terms.size(); i++) {
    if (i == 0 || terms[i].key != terms[i - 1].key) {
      h_fb_hi.push_back((int)(terms[i].key >> 32));
      h_fb_lo.push_back((int)(terms[i].key & 0xffffffffu));
      h_fb_ptr.push_back((int)i);
    }
    h_ft_type.push_back(terms[i].type); h_ft_fac.push_back(terms[i].fac);
    h_ft_rhi.push_back(terms[i].rhi); h_ft_rlo.push_back(terms[i].rlo);
  }
  h_fb_ptr.push_back((int)terms.size());
  E.n_fb = (int)h_fb_hi.size();

  lap("factor lists");
  // ---- uploads ----
  E.h_const.assign(p->pose_const, p->pose_const + K);
  if (fill) {
    if (E.pose[0].alloc((size_t)7 * K, E.st) || E.pose0.alloc((size_t)7 * K, E.st)) return cvb_fail(ctx, CVB_ERR_CUDA, "cudaMalloc failed (poses)");
  } else if ((rc = upload(E, E.pose[0], p->pose, (size_t)7 * K))) {
    return rc;
  }
  if ((rc = zalloc(E, E.pose[1], (size_t)7 * K))) return rc;
  std::vector<double> h_sb((size_t)9 * K, 0.0);
  if (p->speedbias) std::memcpy(h_sb.data(), p->speedbias, sizeof(double) * 9 * K);
  if ((rc = upload(E, E.sb[0], h_sb))) return rc;
  if ((rc = zalloc(E, E.sb[1], (size_t)9 * K))) return rc;
  if ((rc = upload(E, E.lm[0], h_lm))) return rc;
  if ((rc = zalloc(E, E.lm[1], (size_t)3 * E.L_in))) return rc;
  if ((!fill && (rc = upload(E, E.pose0, p->pose, (size_t)7 * K))) || (rc = upload(E, E.sb0, h_sb)) || (rc = upload(E, E.lm0, h_lm))) return rc;
  if ((rc = upload(E, E.pose_const, p->pose_const, (size_t)K))) return rc;
  cvb_kf_cameras cams;
  if ((rc = cvb_stage_kf_cameras(ctx, p, cams))) return rc;
  if ((rc = upload(E, E.extr_kf, cams.extr)) || (rc = upload(E, E.intr_kf, cams.intr)) || (rc = upload(E, E.dist_kf, cams.dist)) ||
      (rc = upload(E, E.model_kf, cams.model)) || (rc = upload(E, E.xi_kf, cams.xi)))
    return rc;
  if ((rc = upload(E, E.obs_kf, h_obs_kf)) || (rc = upload(E, E.obs_lm, h_obs_lm)) || (rc = upload(E, E.lm_ptr, h_lm_ptr)) ||
      (rc = upload(E, E.kf_ptr, h_kf_ptr)) || (rc = upload(E, E.kf_obs, h_kf_obs)) || (rc = upload(E, E.obs_uv, h_uv)) ||
      (rc = upload(E, E.obs_sigma, h_sigma)))
    return rc;
  if ((rc = zalloc(E, E.lin, (size_t)E.n_obs)) || (rc = zalloc(E, E.ow, (size_t)E.n_obs))) return rc;
  if ((rc = zalloc(E, E.Hll, (size_t)6 * E.L_in)) || (rc = zalloc(E, E.HllInv, (size_t)6 * E.L_in)) ||
      (rc = zalloc(E, E.bl, (size_t)3 * E.L_in)))
    return rc;
  if ((rc = build_schur_lists(E, h_lm_ptr, K))) return rc;
  lap("Schur pair lists (device)");
  if ((rc = upload(E, E.fb_hi, h_fb_hi)) || (rc = upload(E, E.fb_lo, h_fb_lo)) || (rc = upload(E, E.fb_ptr, h_fb_ptr)) ||
      (rc = upload(E, E.ft_type, h_ft_type)) || (rc = upload(E, E.ft_fac, h_ft_fac)) || (rc = upload(E, E.ft_rhi, h_ft_rhi)) ||
      (rc = upload(E, E.ft_rlo, h_ft_rlo)))
    return rc;
  // edges
  if (fill) {
    CVB_REQUIRE(ctx, E.world == 1, "device-written edges need a single rank");
    std::vector<uint8_t> rb(E.n_edge);
    for (int e = 0; e < E.n_edge; e++) rb[e] = p->edge_robust ? p->edge_robust[e] : 0;
    if ((rc = upload(E, E.edge_i, h_edge_i)) || (rc = upload(E, E.edge_j, h_edge_j)) || (rc = upload(E, E.edge_robust, rb))) return rc;
    if (E.edge_q.alloc((size_t)4 * E.n_edge, E.st) || E.edge_t.alloc((size_t)3 * E.n_edge, E.st) || E.edge_S.alloc((size_t)36 * E.n_edge, E.st))
      return cvb_fail(ctx, CVB_ERR_CUDA, "cudaMalloc failed (edges)");
    if ((rc = (*fill)(E.pose[0].p, E.pose0.p, E.edge_q.p, E.edge_t.p, E.edge_S.p))) return rc;
    if ((rc = zalloc(E, E.Jedge, (size_t)72 * E.n_edge)) || (rc = zalloc(E, E.redge, (size_t)6 * E.n_edge))) return rc;
  } else {
    std::vector<double> q((size_t)4 * E.n_edge), t((size_t)3 * E.n_edge), S((size_t)36 * E.n_edge);
    std::vector<uint8_t> rb(E.n_edge);
    for (int e = 0; e < E.n_edge; e++) {
      const int s = sel_edge[e];
      std::memcpy(&q[4 * (size_t)e], p->edge_q + 4 * (size_t)s, 4 * sizeof(double));
      std::memcpy(&t[3 * (size_t)e], p->edge_t + 3 * (size_t)s, 3 * sizeof(double));
      std::memcpy(&S[36 * (size_t)e], p->edge_sqrt_info + 36 * (size_t)s, 36 * sizeof(double));
      rb[e] = p->edge_robust ? p->edge_robust[s] : 0;
    }
    if ((rc = upload(E, E.edge_i, h_edge_i)) || (rc = upload(E, E.edge_j, h_edge_j)) || (rc = upload(E, E.edge_q, q)) ||
        (rc = upload(E, E.edge_t, t)) || (rc = upload(E, E.edge_S, S)) || (rc = upload(E, E.edge_robust, rb)))
      return rc;
    if ((rc = zalloc(E, E.Jedge, (size_t)72 * E.n_edge)) || (rc = zalloc(E, E.redge, (size_t)6 * E.n_edge))) return rc;
  }
  if ((rc = zalloc(E, E.flag, 4))) return rc;
  // IMU: raw samples → device, repropagate at the current bias of KF j (opt.cpp:132-140, 387-396)
  if ((rc = upload(E, E.imu_i, h_imu_i)) || (rc = upload(E, E.imu_j, h_imu_j))) return rc;
  if ((rc = zalloc(E, E.pre, (size_t)E.n_imu)) || (rc = zalloc(E, E.Jimu, (size_t)450 * E.n_imu)) ||
      (rc = zalloc(E, E.rimu, (size_t)15 * E.n_imu)))
    return rc;
  if (E.n_imu > 0) {
    E.g = p->imu_noise[4];
    std::vector<int> ptr(1, 0);
    std::vector<double> dt, acc, gyr, a0, g0;
    for (int f = 0; f < E.n_imu; f++) {
      const int s = sel_imu[f];
      for (int m = p->imu_ptr[s]; m < p->imu_ptr[s + 1]; m++) {
        dt.push_back(p->imu_dt[m]);
        for (int c = 0; c < 3; c++) { acc.push_back(p->imu_acc[3 * (size_t)m + c]); gyr.push_back(p->imu_gyr[3 * (size_t)m + c]); }
      }
      for (int c = 0; c < 3; c++) { a0.push_back(p->imu_acc0[3 * (size_t)s + c]); g0.push_back(p->imu_gyr0[3 * (size_t)s + c]); }
      ptr.push_back((int)dt.size());
    }
    cvb_dev_arr<int> d_ptr; cvb_dev_arr<double> d_dt, d_acc, d_gyr, d_a0, d_g0, d_noise;
    if ((rc = upload(E, d_ptr, ptr)) || (rc = upload(E, d_dt, dt)) || (rc = upload(E, d_acc, acc)) || (rc = upload(E, d_gyr, gyr)) ||
        (rc = upload(E, d_a0, a0)) || (rc = upload(E, d_g0, g0)) || (rc = upload(E, d_noise, p->imu_noise, 5)))
      return rc;
    imu_repropagate_kernel<<<grid1(E.n_imu, 64), 64, 0, E.st>>>(E.n_imu, E.imu_j.p, d_ptr.p, d_dt.p, d_acc.p, d_gyr.p, d_a0.p,
                                                               d_g0.p, E.sb[0].p, d_noise.p, E.pre.p, E.flag.p);
    ENG_LAUNCH();
    int flag = 0;
    ENG_CUDA(cudaMemcpyAsync(&flag, E.flag.p, sizeof(int), cudaMemcpyDeviceToHost, E.st));
    ENG_CUDA(cudaStreamSynchronize(E.st));
    // bit 2: a preintegrated covariance P that is not positive definite (e.g. a zero noise sigma in imu_noise); its
    // sqrt_info would be meaningless, and the reference's chol(P^-1) fails on the same input
    if (flag & 2)
      return cvb_fail(ctx, CVB_ERR_NUMERIC, "IMU preintegration covariance is not positive definite (check imu_noise)");
  }
  lap("uploads");
  // ---- vectors, S ----
  std::vector<double> h_scale(E.n_vec, 0.0);
  for (int k = 0; k < K; k++) {
    if (!p->pose_const[k])
      for (int c = 0; c < 6; c++) h_scale[(size_t)col_of(k, c)] = 1.0;
    if (!E.visual_only)
      for (int c = 6; c < 15; c++) h_scale[(size_t)col_of(k, c)] = 1.0;
  }
  for (int c = 0; c < E.L_in; c++)   // landmark blocks are owned by rank (c % world); others stay inactive here
    if (c % E.world == E.rank)
      for (int a = 0; a < 3; a++) h_scale[(size_t)E.n_c_pad + 3 * (size_t)c + a] = 1.0;
  if ((rc = upload(E, E.scale0, h_scale)) || (rc = zalloc(E, E.scale, (size_t)E.n_vec))) return rc;
  if ((rc = upload(E, E.off_pose, E.h_off_pose)) || (rc = upload(E, E.off_sb, E.h_off_sb))) return rc;
  if ((rc = E.plan.upload(E.ctx, E.st))) return rc;
  if ((rc = upload(E, E.xt_all, h_xt_all)) || (rc = upload(E, E.xt_fill, h_xt_fill))) return rc;
  if (E.world > 1) {
    if ((rc = upload(E, E.xt_own, h_xt_own)) || (rc = upload(E, E.col_owner, h_owner))) return rc;
    if ((rc = zalloc(E, E.flagd, 2))) return rc;
  }
  cvb_dev_arr<double>* vecs[] = {&E.colsq, &E.diag, &E.gvec, &E.grad, &E.sgrad, &E.gn, &E.step, &E.xsol, &E.yb, &E.gs, &E.tmp};
  for (auto* v : vecs)
    if ((rc = zalloc(E, *v, (size_t)E.n_vec))) return rc;
  // S = the packed tiles of L's structure; cleared at the start of every linearisation (cam_blocks).  With several ranks
  // S, the tile inverses and the panel flags come from cudaMalloc so that they can be exported through CUDA IPC.
  const size_t s_doubles = E.n_tiles * cvb_chol::T * cvb_chol::T, linv_doubles = (size_t)E.n_c_pad * cvb_chol::T;
  const bool ipc = E.world > 1;
  if (E.S.alloc(s_doubles, E.st, ipc)) return cvb_fail(E.ctx, CVB_ERR_CUDA, "cudaMalloc failed (reduced camera system, %zu bytes)", s_doubles * 8);
  if ((rc = zalloc(E, E.linv, linv_doubles, ipc)) || (ipc && (rc = zalloc(E, E.pflag, 2 * (size_t)E.plan.nt, ipc)))) return rc;
  if ((rc = zalloc(E, E.partials, (size_t)RED_SLOTS * RED_BLOCKS)) || (rc = zalloc(E, E.scalars, RED_SLOTS)) ||
      (rc = zalloc(E, E.rankmax, (size_t)E.world)))
    return rc;
  ENG_CUDA(cudaMallocHost(&E.h_scalars, RED_SLOTS * sizeof(double)));
  for (auto& e : E.ev) ENG_CUDA(cudaEventCreate(&e));
  ENG_CUDA(cudaStreamCreateWithFlags(&E.st_fill, cudaStreamNonBlocking));
  ENG_CUDA(cudaEventCreateWithFlags(&E.ev_fill_fork, cudaEventDisableTiming));
  ENG_CUDA(cudaEventCreateWithFlags(&E.ev_fill_done, cudaEventDisableTiming));
  if ((rc = E.fs.create(E.ctx, E.plan.nt))) return rc;
  ENG_CUDA(cudaStreamSynchronize(E.st));
  lap("vectors, S, streams (sync)");
  return CVB_OK;
}

// cost (and optionally full linearisation) at state buffer `b`; mode 0 = linearise, 1 = cost only
int evaluate(Engine& E, int b, int mode, double* cost_out) {
  const int rg = RED_BLOCKS;
  lin_obs_kernel<<<rg, 256, 0, E.st>>>(E.n_obs, E.obs_kf.p, E.obs_lm.p, E.obs_uv.p, E.obs_sigma.p, E.pose[b].p, E.lm[b].p,
                                       E.extr_kf.p, E.intr_kf.p, E.dist_kf.p, E.model_kf.p, E.xi_kf.p, E.scale.p, E.off_pose.p, E.n_c_pad, E.a2_reproj, mode,
                                       E.lin.p, E.ow.p, nullptr, E.partials.p, 0);
  ENG_LAUNCH();
  lin_imu_kernel<<<rg, 256, 0, E.st>>>(E.n_imu, E.imu_i.p, E.imu_j.p, E.pre.p, E.pose[b].p, E.sb[b].p, E.scale.p, E.off_pose.p, E.off_sb.p, E.g,
                                       mode, E.Jimu.p, E.rimu.p, E.partials.p, 1);
  ENG_LAUNCH();
  lin_edge_kernel<<<rg, 256, 0, E.st>>>(E.n_edge, E.edge_i.p, E.edge_j.p, E.edge_q.p, E.edge_t.p, E.edge_S.p, E.edge_robust.p,
                                        E.pose[b].p, E.scale.p, E.off_pose.p, E.a2_edge, mode, E.Jedge.p, E.redge.p, E.partials.p, 2);
  ENG_LAUNCH();
  int rc = read_scalars(E, 3);
  if (rc) return rc;
  *cost_out = E.h_scalars[0] + E.h_scalars[1] + E.h_scalars[2];
  return CVB_OK;
}


inline void tick(Engine& E, int i) { cudaEventRecord(E.ev[i], E.st); }
inline void tock(Engine& E, int a, int b, int phase) {   // both events must have completed (call after a stream sync)
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, E.ev[a], E.ev[b]) == cudaSuccess) E.phase_ms[phase] += ms;
}

// ---- per-linearisation blocks -----------------------------------------------------------------------------------
int lm_blocks(Engine& E) {
  if (E.L_in > 0) {
    lm_reduce_kernel<<<grid1(E.L_in), 256, 0, E.st>>>(E.L_in, E.lm_ptr.p, E.lin.p, E.Hll.p, E.bl.p, E.colsq.p + E.n_c_pad,
                                                      E.gvec.p + E.n_c_pad);
    ENG_LAUNCH();
  }
  return CVB_OK;
}

// camera blocks of J^T J (before Schur / damping) into S, camera gradient into gvec
int cam_blocks(Engine& E) {
  const size_t ld = (size_t)E.n_c_pad;
  const SView Sv{E.S.p, E.plan.d_tile_of.p, E.plan.nt};
  // S's own tiles (the ones the block kernels below add into) are cleared first on the engine stream; the fill tiles,
  // which only the factorisation writes, on st_fill beside the block kernels (factor_rcs waits for them)
  if (E.n_xt_fill > 0) {
    ENG_CUDA(cudaEventRecord(E.ev_fill_fork, E.st));
    ENG_CUDA(cudaStreamWaitEvent(E.st_fill, E.ev_fill_fork, 0));
    zero_tiles_kernel<<<E.n_xt_fill, 256, 0, E.st_fill>>>(E.S.p, E.xt_fill.p);
    ENG_LAUNCH();
    ENG_CUDA(cudaEventRecord(E.ev_fill_done, E.st_fill));
    E.fill_pending = true;
  }
  if (E.n_xt_all > 0) {
    zero_tiles_kernel<<<E.n_xt_all, 256, 0, E.st>>>(E.S.p, E.xt_all.p);
    ENG_LAUNCH();
  }
  ENG_CUDA(cudaMemsetAsync(E.gvec.p, 0, ld * sizeof(double), E.st));
  kf_visual_kernel<<<grid1((size_t)E.K * 32, 128), 128, 0, E.st>>>(E.K, E.kf_ptr.p, E.kf_obs.p, E.lin.p, E.off_pose.p, Sv,
                                                                  E.gvec.p);
  ENG_LAUNCH();
  if (E.n_fb > 0) {
    factor_gather_kernel<<<E.n_fb, 256, 0, E.st>>>(E.n_fb, E.fb_hi.p, E.fb_lo.p, E.fb_ptr.p, E.ft_type.p, E.ft_fac.p,
                                                   E.ft_rhi.p, E.ft_rlo.p, E.Jimu.p, E.rimu.p, E.Jedge.p, E.redge.p, E.off_pose.p, E.off_sb.p, E.per, Sv,
                                                   E.gvec.p);
    ENG_LAUNCH();
  }
  return CVB_OK;
}

int cam_colsq(Engine& E) {
  cam_colsq_kernel<<<grid1(E.n_c_pad), 256, 0, E.st>>>(E.n_c_pad, E.scale.p, SView{E.S.p, E.plan.d_tile_of.p, E.plan.nt}, E.colsq.p);
  ENG_LAUNCH();
  return ar(E, E.colsq.p, (size_t)E.n_c_pad);
}

// damped Schur complement + Cholesky for the given mu; *ok = false if the factorisation broke down
int factor_rcs(Engine& E, double mu, bool* ok) {
  const size_t ld = (size_t)E.n_c_pad;
  const SView Sv{E.S.p, E.plan.d_tile_of.p, E.plan.nt};
  const bool dist = E.p2p && E.world > 1;
  tick(E, 0);
  if (E.L_in > 0) {
    lm_damp_inv_kernel<<<grid1(E.L_in), 256, 0, E.st>>>(E.L_in, E.Hll.p, E.colsq.p + E.n_c_pad, mu, E.HllInv.p);
    ENG_LAUNCH();
  }
  ENG_CUDA(cudaMemsetAsync(E.yb.p, 0, ld * sizeof(double), E.st));
  schur_row_kernel<<<E.K, ROW_THREADS, (size_t)E.row_stage * 18 * sizeof(double), E.st>>>(
      E.row_stage, E.kf_ptr.p, E.kf_obs.p, E.obs_lm.p, E.HllInv.p, E.bl.p, E.ow.p, E.kf_sb.p, E.sb_lo.p, E.sb_ptr.p, E.sp_a.p,
      E.sp_b.p, E.off_pose.p, Sv, E.yb.p);
  ENG_LAUNCH();
  // the one exchange of the data path: sum the rank-partial reduced normal equations over NVLink
  int rc = CVB_OK;
  if (E.allreduce && E.world > 1 && !dist) {
    if (!E.xbuf.p && (rc = zalloc(E, E.xbuf, (size_t)E.n_xt_all * cvb_chol::T * cvb_chol::T))) return rc;
    pack_tiles_kernel<<<E.n_xt_all, 256, 0, E.st>>>(E.S.p, E.xt_all.p, E.xbuf.p, 0);
    ENG_LAUNCH();
    if ((rc = ar(E, E.xbuf.p, (size_t)E.n_xt_all * cvb_chol::T * cvb_chol::T))) return rc;
    pack_tiles_kernel<<<E.n_xt_all, 256, 0, E.st>>>(E.S.p, E.xt_all.p, E.xbuf.p, 1);
    ENG_LAUNCH();
  }
  // this all-reduce is also the hand-shake of the peer pull below: when it completes here, every rank has finished
  // writing its partial S (stream order on each rank)
  if ((rc = ar(E, E.yb.p, ld))) return rc;
  if (dist && E.n_xt_own > 0) {
    reduce_pull_kernel<<<E.n_xt_own, 256, 0, E.st>>>(E.S.p, E.peer_S.p, E.world, E.rank, E.xt_own.p);
    ENG_LAUNCH();
  }
  cam_finish_kernel<<<grid1(E.n_c_pad), 256, 0, E.st>>>(E.n_c_pad, E.scale.p, Sv, E.diag.p, E.gvec.p, E.yb.p, E.gs.p, mu,
                                                        dist ? E.col_owner.p : nullptr, E.rank);
  ENG_LAUNCH();
  if (E.fill_pending) {
    ENG_CUDA(cudaStreamWaitEvent(E.st, E.ev_fill_done, 0));
    E.fill_pending = false;
  }
  tick(E, 1);
  // first call: plain launches (sets kernel attributes); second call: stream-capture into a graph; then replay
  if (E.g_factor) {
    ENG_CUDA(cudaGraphLaunch(E.g_factor, E.st));
    E.ctx->launches += 1 + (int64_t)E.plan.nt * 3;   // kernels inside the graph (distributed: pulls are copies, not kernels)
  } else if (E.n_factor_calls == 1) {
    cudaGraph_t g = nullptr;
    ENG_CUDA(cudaStreamBeginCapture(E.st, cudaStreamCaptureModeThreadLocal));
    rc = cvb_chol::factor(E.ctx, E.S.p, E.linv.p, E.flag.p, E.plan, E.st, E.fs, dist ? &E.dv : nullptr);
    cudaError_t ce = cudaStreamEndCapture(E.st, &g);
    if (rc) return rc;
    if (ce != cudaSuccess) return cvb_fail(E.ctx, CVB_ERR_CUDA, "graph capture of the factorisation failed: %s", cudaGetErrorString(ce));
    ENG_CUDA(cudaGraphInstantiate(&E.g_factor, g, 0));
    cudaGraphDestroy(g);
    ENG_CUDA(cudaGraphLaunch(E.g_factor, E.st));
  } else {
    rc = cvb_chol::factor(E.ctx, E.S.p, E.linv.p, E.flag.p, E.plan, E.st, E.fs, dist ? &E.dv : nullptr);
    if (rc) return rc;
  }
  E.n_factor_calls++;
  tick(E, 2);
  int flag = 0;
  if (dist) {   // a pivot failure on any owner fails the factorisation on every rank
    flag_to_double_kernel<<<1, 1, 0, E.st>>>(E.flag.p, E.flagd.p);
    ENG_LAUNCH();
    if ((rc = ar(E, E.flagd.p, 1))) return rc;
    double fd = 0.0;
    ENG_CUDA(cudaMemcpyAsync(&fd, E.flagd.p, sizeof(double), cudaMemcpyDeviceToHost, E.st));
    ENG_CUDA(cudaStreamSynchronize(E.st));
    flag = fd != 0.0 ? 1 : 0;
  } else {
    ENG_CUDA(cudaMemcpyAsync(&flag, E.flag.p, sizeof(int), cudaMemcpyDeviceToHost, E.st));
    ENG_CUDA(cudaStreamSynchronize(E.st));
  }
  tock(E, 0, 1, 1);
  tock(E, 1, 2, 2);
  E.chol_flops += E.plan.flops;
  *ok = (flag & 1) == 0;
  return CVB_OK;
}

enum { TERM_NO_CONVERGENCE = 0, TERM_GRADIENT = 1, TERM_PARAMETER = 2, TERM_FUNCTION = 3, TERM_FAILURE = 4 };
enum { STEP_ACCEPTED = 1, STEP_REJECTED = 2, STEP_INVALID = 3, STEP_CONVERGED = 4 };

// full linearisation at the current state (cost included)
int linearize(Engine& E, double* cost) {
  int rc = evaluate(E, E.cur, 0, cost);
  if (rc) return rc;
  return lm_blocks(E);
}

int engine_begin(Engine& E) {
  // iteration 0 of TrustRegionMinimizer: evaluate, fix the Jacobi scaling at x0, re-linearise in the scaled space.
  // The first evaluation must see the unscaled Jacobian, so `scale` starts from the activity mask every time: a restart
  // that kept the previous solve's scaling would take the column norms of an already scaled Jacobian.
  ENG_CUDA(cudaMemcpyAsync(E.scale.p, E.scale0.p, (size_t)E.n_vec * sizeof(double), cudaMemcpyDeviceToDevice, E.st));
  double c0;
  int rc = linearize(E, &c0);
  if (rc) return rc;
  if ((rc = cam_blocks(E)) || (rc = cam_colsq(E))) return rc;
  jacobi_scale_kernel<<<grid1(E.n_vec), 256, 0, E.st>>>(E.n_vec, E.colsq.p, E.scale.p);
  ENG_LAUNCH();
  if ((rc = linearize(E, &E.cost))) return rc;
  // |x| over the non-constant parameter blocks
  ENG_CUDA(cudaMemsetAsync(E.step.p, 0, (size_t)E.n_vec * sizeof(double), E.st));
  const int nxt = E.cur ^ 1;
  plus_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.K, E.L_in, E.off_pose.p, E.off_sb.p, E.n_c_pad, E.visual_only, E.pose_const.p, E.step.p, E.scale.p,
                                            E.pose[E.cur].p, E.sb[E.cur].p, E.lm[E.cur].p, E.pose[nxt].p, E.sb[nxt].p,
                                            E.lm[nxt].p, E.rank == 0 ? 1.0 : 0.0, E.partials.p, 0);
  ENG_LAUNCH();
  if ((rc = read_scalars(E, 2))) return rc;
  E.x_norm = std::sqrt(E.h_scalars[1]);
  E.cost_hist.assign(1, E.cost);
  E.step_status.clear();
  E.radius = 1e4; E.mu = 1e-8; E.reuse = false; E.invalid_run = 0; E.iterations = 0; E.termination = TERM_NO_CONVERGENCE;
  E.have_lin = true;
  return CVB_OK;
}

// DoglegStrategy::ComputeStep up to the Gauss-Newton solve; *solver_ok false → step invalid; *converged on gradient tol.
int prepare_step(Engine& E, bool* solver_ok, bool* grad_converged) {
  constexpr double MAX_MU = 1.0, MU_INC = 10.0;
  *solver_ok = true;
  *grad_converged = false;
  int rc;
  tick(E, 5);
  if ((rc = cam_blocks(E))) return rc;
  if ((rc = ar(E, E.gvec.p, (size_t)E.n_c_pad))) return rc;
  if ((rc = cam_colsq(E))) return rc;
  cam_diag_kernel<<<grid1(E.n_c_pad), 256, 0, E.st>>>(E.n_c_pad, E.scale.p, E.colsq.p, E.diag.p);
  ENG_LAUNCH();
  prep_vectors_kernel<<<grid1(E.n_vec), 256, 0, E.st>>>(E.n_vec, E.n_c_pad, E.scale.p, E.colsq.p, E.diag.p, E.gvec.p, E.grad.p,
                                                        E.sgrad.p);
  ENG_LAUNCH();
  // gradient tolerance (max-norm of the unscaled gradient)
  max_abs_grad_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.n_vec, E.gvec.p, E.scale.p, E.partials.p, 7);
  ENG_LAUNCH();
  max_final_kernel<<<1, 1, 0, E.st>>>(E.partials.p, E.scalars.p, 7, E.rankmax.p, E.rank, E.world);
  ENG_LAUNCH();
  if (E.world > 1) {
    if ((rc = ar(E, E.rankmax.p, (size_t)E.world))) return rc;
  }
  // Cauchy point: alpha = |grad|^2 / |J (grad / diag)|^2
  jv_obs_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.n_obs, E.obs_kf.p, E.obs_lm.p, E.lin.p, E.sgrad.p, E.off_pose.p, E.n_c_pad,
                                              E.partials.p, 3);
  ENG_LAUNCH();
  jv_factor_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.n_imu, E.imu_i.p, E.imu_j.p, E.Jimu.p, E.rimu.p, E.n_edge, E.edge_i.p,
                                                 E.edge_j.p, E.Jedge.p, E.redge.p, E.sgrad.p, E.off_pose.p, E.off_sb.p, E.partials.p, 5);
  ENG_LAUNCH();
  tick(E, 6);
  bool cam_fresh = true;
  bool solved = false;
  bool first_try = true;
  while (E.mu < MAX_MU) {
    if (!cam_fresh) {
      if ((rc = cam_blocks(E))) return rc;
      if ((rc = ar(E, E.gvec.p, (size_t)E.n_c_pad))) return rc;
    }
    bool ok = false;
    if ((rc = factor_rcs(E, E.mu, &ok))) return rc;
    if (first_try) tock(E, 5, 6, 1);
    first_try = false;
    cam_fresh = false;
    if (!ok) {
      E.mu *= MU_INC;
      continue;
    }
    tick(E, 3);
    if (E.g_solve) {
      ENG_CUDA(cudaGraphLaunch(E.g_solve, E.st));
      E.ctx->launches += 2;   // the two substitution kernels inside the graph
    } else if (E.n_solve_calls == 1) {
      cudaGraph_t g = nullptr;
      ENG_CUDA(cudaStreamBeginCapture(E.st, cudaStreamCaptureModeThreadLocal));
      rc = cvb_chol::solve(E.ctx, E.S.p, E.linv.p, E.gs.p, E.tmp.p, E.xsol.p, E.plan, E.st, E.fs);
      cudaError_t ce = cudaStreamEndCapture(E.st, &g);
      if (rc) return rc;
      if (ce != cudaSuccess) return cvb_fail(E.ctx, CVB_ERR_CUDA, "graph capture of the solve failed: %s", cudaGetErrorString(ce));
      ENG_CUDA(cudaGraphInstantiate(&E.g_solve, g, 0));
      cudaGraphDestroy(g);
      ENG_CUDA(cudaGraphLaunch(E.g_solve, E.st));
    } else {
      if ((rc = cvb_chol::solve(E.ctx, E.S.p, E.linv.p, E.gs.p, E.tmp.p, E.xsol.p, E.plan, E.st, E.fs))) return rc;
    }
    E.n_solve_calls++;
    if (E.L_in > 0) {
      backsub_kernel<<<grid1(E.L_in), 256, 0, E.st>>>(E.L_in, E.lm_ptr.p, E.obs_kf.p, E.ow.p, E.HllInv.p, E.bl.p, E.xsol.p, E.off_pose.p,
                                                      E.xsol.p + E.n_c_pad);
      ENG_LAUNCH();
    }
    gn_norms_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.n_vec, E.xsol.p, E.diag.p, E.grad.p, E.scale.p, E.gn.p, E.n_c_pad,
                                                  E.rank == 0 ? 1.0 : 0.0, E.partials.p, 0);
    ENG_LAUNCH();
    // slots: 0 |gn|^2, 1 |grad|^2, 2 grad.gn, 3 |J sgrad|^2 (obs), 5 (factors); slot 7 = max |g| (not summed over ranks)
    reduce_final<<<1, 256, 0, E.st>>>(E.partials.p, E.scalars.p, 7, 0);
    ENG_LAUNCH();
    if ((rc = ar(E, E.scalars.p, 7))) return rc;
    if (E.world > 1) {   // slot 7 (max-norm of the gradient) = max over the ranks' maxima
      max_ranks_kernel<<<1, 1, 0, E.st>>>(E.rankmax.p, E.world, E.scalars.p, 7);
      ENG_LAUNCH();
    }
    tick(E, 4);
    ENG_CUDA(cudaMemcpyAsync(E.h_scalars, E.scalars.p, RED_SLOTS * sizeof(double), cudaMemcpyDeviceToHost, E.st));
    ENG_CUDA(cudaStreamSynchronize(E.st));
    tock(E, 3, 4, 3);
    if (!std::isfinite(E.h_scalars[0])) {
      E.mu *= MU_INC;
      continue;
    }
    solved = true;
    break;
  }
  if (!solved) {
    *solver_ok = false;
    return CVB_OK;
  }
  E.gn2 = E.h_scalars[0]; E.gg = E.h_scalars[1]; E.g_gn = E.h_scalars[2];
  const double JgJg = E.h_scalars[3] + E.h_scalars[5];
  E.alpha = E.gg / JgJg;
  if (E.h_scalars[7] <= 1e-10) *grad_converged = true;
  return CVB_OK;
}

// one TrustRegionMinimizer iteration; returns CVB_OK and sets *done when the minimiser terminates
int engine_iterate(Engine& E, bool* done) {
  constexpr double MU_INC = 10.0, MIN_MU = 1e-8;
  *done = false;
  int rc;
  E.iterations++;
  bool solver_ok = true, gconv = false;
  if (!E.reuse) {
    E.reuse = true;
    if ((rc = prepare_step(E, &solver_ok, &gconv))) return rc;
    if (gconv && E.iterations == 1) {   // gradient tolerance reached at the start point
      E.termination = TERM_GRADIENT;
      E.iterations = 0;
      *done = true;
      return CVB_OK;
    }
  }
  double model_change = -1.0;
  if (solver_ok) {
    const double gn_norm = std::sqrt(E.gn2), g_norm = std::sqrt(E.gg), g_dot_gn = E.g_gn;
    double ca, cb;
    if (gn_norm <= E.radius) {
      ca = 0.0; cb = 1.0;
    } else if (g_norm * E.alpha >= E.radius) {
      ca = -(E.radius / g_norm); cb = 0.0;
    } else {
      const double b_dot_a = -E.alpha * g_dot_gn;
      const double a2 = (E.alpha * g_norm) * (E.alpha * g_norm);
      const double bma2 = a2 - 2.0 * b_dot_a + gn_norm * gn_norm;
      const double c = b_dot_a - a2;
      const double d = std::sqrt(c * c + bma2 * (E.radius * E.radius - a2));
      const double beta = (c <= 0) ? (d - c) / bma2 : (E.radius * E.radius - a2) / (d + c);
      ca = -E.alpha * (1.0 - beta); cb = beta;
    }
    tick(E, 5);
    dogleg_combine_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.n_vec, ca, cb, E.grad.p, E.gn.p, E.diag.p, E.scale.p, E.step.p,
                                                        E.n_c_pad, E.rank == 0 ? 1.0 : 0.0, E.partials.p, 0);
    ENG_LAUNCH();
    jv_obs_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.n_obs, E.obs_kf.p, E.obs_lm.p, E.lin.p, E.step.p, E.off_pose.p, E.n_c_pad,
                                                E.partials.p, 1);
    ENG_LAUNCH();
    jv_factor_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.n_imu, E.imu_i.p, E.imu_j.p, E.Jimu.p, E.rimu.p, E.n_edge, E.edge_i.p,
                                                   E.edge_j.p, E.Jedge.p, E.redge.p, E.step.p, E.off_pose.p, E.off_sb.p, E.partials.p, 3);
    ENG_LAUNCH();
    // candidate state + its cost in the same sync
    const int nxt = E.cur ^ 1;
    plus_kernel<<<RED_BLOCKS, 256, 0, E.st>>>(E.K, E.L_in, E.off_pose.p, E.off_sb.p, E.n_c_pad, E.visual_only, E.pose_const.p, E.step.p, E.scale.p,
                                              E.pose[E.cur].p, E.sb[E.cur].p, E.lm[E.cur].p, E.pose[nxt].p, E.sb[nxt].p,
                                              E.lm[nxt].p, E.rank == 0 ? 1.0 : 0.0, E.partials.p, 5);
    ENG_LAUNCH();
    tick(E, 6);
    if ((rc = read_scalars(E, 7))) return rc;
    tock(E, 5, 6, 4);
    const double dl2 = E.h_scalars[0];
    const double jv2 = E.h_scalars[1] + E.h_scalars[3], jvr = E.h_scalars[2] + E.h_scalars[4];
    const double step2 = E.h_scalars[5], cand_x2 = E.h_scalars[6];
    E.dogleg_norm = std::sqrt(dl2);
    model_change = -(jvr + 0.5 * jv2);
    if (model_change > 0.0) {
      E.invalid_run = 0;
      double ccost;
      tick(E, 5);
      if ((rc = evaluate(E, nxt, 1, &ccost))) return rc;
      tick(E, 6);
      cudaEventSynchronize(E.ev[6]);
      tock(E, 5, 6, 4);
      const double step_norm = std::sqrt(step2);
      if (step_norm <= 1e-8 * (E.x_norm + 1e-8)) {
        E.termination = TERM_PARAMETER; E.step_status.push_back(STEP_CONVERGED); *done = true;
        return CVB_OK;
      }
      if (std::fabs(E.cost - ccost) <= 1e-6 * E.cost) {
        E.termination = TERM_FUNCTION; E.step_status.push_back(STEP_CONVERGED); *done = true;
        return CVB_OK;
      }
      const double rho = (E.cost - ccost) / model_change;
      if (rho > 1e-3) {
        E.cur = nxt;
        E.cost = ccost;
        E.x_norm = std::sqrt(cand_x2);
        double c2;
        tick(E, 5);
        if ((rc = linearize(E, &c2))) return rc;
        tick(E, 6);
        cudaEventSynchronize(E.ev[6]);
        tock(E, 5, 6, 0);
        if (rho < 0.25) E.radius *= 0.5;
        if (rho > 0.75) E.radius = std::max(E.radius, 3.0 * E.dogleg_norm);
        E.mu = std::max(MIN_MU, 2.0 * E.mu / MU_INC);
        E.reuse = false;
        E.step_status.push_back(STEP_ACCEPTED);
      } else {
        E.radius *= 0.5;
        E.reuse = true;
        E.step_status.push_back(STEP_REJECTED);
      }
      E.cost_hist.push_back(E.cost);
      return CVB_OK;
    }
  }
  // invalid step (solver failure or non-positive model decrease)
  E.invalid_run++;
  E.step_status.push_back(STEP_INVALID);
  E.cost_hist.push_back(E.cost);
  if (E.invalid_run > 5) {
    E.termination = TERM_FAILURE;
    *done = true;
    return CVB_OK;
  }
  E.mu *= MU_INC;
  E.reuse = false;
  return CVB_OK;
}

int engine_corrected_norms(Engine& E, double* h_norms_full, int n_obs_full) {
  cvb_dev_arr<double> d;
  if (d.alloc((size_t)E.n_obs, E.st)) return cvb_fail(E.ctx, CVB_ERR_CUDA, "cudaMalloc failed");
  if (E.n_obs) {
    reproj_norms_kernel<<<(E.n_obs + 255) / 256, 256, 0, E.st>>>(E.n_obs, E.obs_kf.p, E.obs_lm.p, E.obs_uv.p, E.obs_sigma.p, E.pose[E.cur].p,
                                                                 E.lm[E.cur].p, E.extr_kf.p, E.intr_kf.p, E.dist_kf.p, E.model_kf.p, E.xi_kf.p,
                                                                 E.a2_reproj, d.p);
    ENG_LAUNCH();
  }
  std::vector<double> h(E.n_obs);
  ENG_CUDA(cudaMemcpyAsync(h.data(), d.p, sizeof(double) * E.n_obs, cudaMemcpyDeviceToHost, E.st));
  ENG_CUDA(cudaStreamSynchronize(E.st));
  for (int i = 0; i < n_obs_full; i++) h_norms_full[i] = -1.0;   // -1: observation not in this rank's problem
  for (int i = 0; i < E.n_obs; i++) h_norms_full[E.obs_of_compact[i]] = h[i];
  return CVB_OK;
}

int engine_download(Engine& E, const cvb_ba_problem* p, cvb_ba_result* r) {
  const int K = E.K;
  if (r->pose) ENG_CUDA(cudaMemcpyAsync(r->pose, E.pose[E.cur].p, sizeof(double) * 7 * K, cudaMemcpyDeviceToHost, E.st));
  if (r->speedbias) ENG_CUDA(cudaMemcpyAsync(r->speedbias, E.sb[E.cur].p, sizeof(double) * 9 * K, cudaMemcpyDeviceToHost, E.st));
  std::vector<double> h_lm((size_t)3 * E.L_in);
  if (E.L_in) ENG_CUDA(cudaMemcpyAsync(h_lm.data(), E.lm[E.cur].p, sizeof(double) * 3 * E.L_in, cudaMemcpyDeviceToHost, E.st));
  ENG_CUDA(cudaStreamSynchronize(E.st));
  if (r->lm) {
    std::memcpy(r->lm, p->lm, sizeof(double) * 3 * (size_t)p->L);
    for (int c = 0; c < E.L_in; c++)
      if (c % E.world == E.rank) std::memcpy(r->lm + 3 * (size_t)E.lm_of_compact[c], &h_lm[3 * (size_t)c], 3 * sizeof(double));
  }
  if (r->lm_owner) {
    for (int l = 0; l < p->L; l++) r->lm_owner[l] = -1;
    for (int c = 0; c < E.L_in; c++) r->lm_owner[E.lm_of_compact[c]] = c % E.world;
  }
  r->iterations = E.iterations;
  r->termination = E.termination;
  r->initial_cost = E.cost_hist.empty() ? 0.0 : E.cost_hist.front();
  r->final_cost = E.cost;
  r->n_cost_history = 0;
  if (r->cost_history && r->cost_history_cap > 0) {
    const int n = std::min<int>(r->cost_history_cap, (int)E.cost_hist.size());
    for (int i = 0; i < n; i++) r->cost_history[i] = E.cost_hist[i];
    r->n_cost_history = n;
  }
  if (r->step_status && r->cost_history_cap > 0) {
    const int n = std::min<int>(r->cost_history_cap, (int)E.step_status.size());
    for (int i = 0; i < n; i++) r->step_status[i] = (uint8_t)E.step_status[i];
  }
  return CVB_OK;
}

// Peer access for the multi-GPU path: every rank maps the packed S, tile inverses and panel flags of every other rank
// (map_peers: the source of the peers' pointers, which reports through *opened whether this rank mapped them all), the
// ranks agree through the installed collective that all of them did, and from then on the reduced camera system is
// reduce-scattered by peer pull and the factorisation is distributed by tile columns.  unmap undoes map_peers when some
// rank failed.
int enable_p2p(Engine& E, bool ipc, const std::function<int(cvb_chol::DistView&, bool*)>& map_peers,
               const std::function<void(cvb_chol::DistView&)>& unmap) {
  if (E.world <= 1) return CVB_OK;
  if (E.p2p) return CVB_OK;
  if (!E.allreduce) return cvb_fail(E.ctx, CVB_ERR_INVALID, "cvb_ba_enable_p2p: install the all-reduce first (cvb_ba_set_allreduce)");
  if (E.world > 16) return cvb_fail(E.ctx, CVB_ERR_UNSUPPORTED, "peer path supports up to 16 ranks");
  if (E.g_factor) return cvb_fail(E.ctx, CVB_ERR_INVALID, "cvb_ba_enable_p2p must precede the first iterations");
  cvb_chol::DistView dv;
  dv.rank = E.rank; dv.world = E.world;
  dv.peer_S[E.rank] = E.S.p; dv.peer_linv[E.rank] = E.linv.p; dv.peer_flag[E.rank] = E.pflag.p;
  bool opened = false;
  int rc;
  if ((rc = map_peers(dv, &opened))) return rc;
  // everybody must have mapped everybody: min over ranks via the sum of (1 - opened)
  {
    cvb_dev_arr<double> d_ok;
    std::vector<double> v(1, opened ? 0.0 : 1.0);
    if ((rc = upload(E, d_ok, v))) return rc;
    if ((rc = ar(E, d_ok.p, 1))) return rc;
    ENG_CUDA(cudaMemcpyAsync(v.data(), d_ok.p, sizeof(double), cudaMemcpyDeviceToHost, E.st));
    ENG_CUDA(cudaStreamSynchronize(E.st));
    if (v[0] != 0.0) {
      unmap(dv);
      return cvb_fail(E.ctx, CVB_ERR_UNSUPPORTED, "peer mapping is not available between all ranks (all-reduce fallback stays in use)");
    }
  }
  if ((rc = zalloc(E, E.epoch, 1)) || (rc = upload(E, E.peer_flag, dv.peer_flag, 16)) || (rc = upload(E, E.peer_S, dv.peer_S, 16)))
    return rc;
  dv.d_epoch = E.epoch.p;
  dv.d_peer_flag = E.peer_flag.p;
  ENG_CUDA(cudaStreamSynchronize(E.st));
  // distributed plan: same structure, pair lists restricted to the tile columns this rank owns
  E.plan.build(E.plan.nt, E.h_prefill, E.plan.h_col_group, &E.h_owner, E.rank);
  if ((rc = E.plan.upload(E.ctx, E.st))) return rc;
  E.dv = dv;
  E.p2p = true;
  E.peer_ipc = ipc;
  return CVB_OK;
}

// The peers' pointers through CUDA IPC (one process per GPU on one NVLink node): every rank exports its three buffers and
// gathers every rank's handles with the installed collective (each rank writes its bytes into its slot of a zeroed table,
// the SUM all-reduce is the all-gather), then opens them.
int enable_p2p_ipc(Engine& E) {
  const auto close = [&E](cvb_chol::DistView& dv) {
    for (int g = 0; g < E.world; g++) {
      if (g == E.rank) continue;
      if (dv.peer_S[g]) cudaIpcCloseMemHandle(dv.peer_S[g]);
      if (dv.peer_linv[g]) cudaIpcCloseMemHandle(dv.peer_linv[g]);
      if (dv.peer_flag[g]) cudaIpcCloseMemHandle(dv.peer_flag[g]);
    }
  };
  const auto map_peers = [&E](cvb_chol::DistView& dv, bool* opened) {
    constexpr int HB = (int)sizeof(cudaIpcMemHandle_t);   // 64
    const int per_rank = 3 * HB + 1;                     // three handles + an "ok" byte
    std::vector<double> table((size_t)E.world * per_rank, 0.0);
    cudaIpcMemHandle_t hs[3];
    bool ok = cudaIpcGetMemHandle(&hs[0], E.S.p) == cudaSuccess && cudaIpcGetMemHandle(&hs[1], E.linv.p) == cudaSuccess &&
              cudaIpcGetMemHandle(&hs[2], E.pflag.p) == cudaSuccess;
    cudaGetLastError();
    for (int q = 0; q < 3 && ok; q++)
      for (int b = 0; b < HB; b++) table[(size_t)E.rank * per_rank + q * HB + b] = (double)reinterpret_cast<unsigned char*>(&hs[q])[b];
    table[(size_t)E.rank * per_rank + 3 * HB] = ok ? 1.0 : 0.0;
    cvb_dev_arr<double> d_table;
    int rc;
    if ((rc = upload(E, d_table, table))) return rc;
    if ((rc = ar(E, d_table.p, table.size()))) return rc;
    ENG_CUDA(cudaMemcpyAsync(table.data(), d_table.p, table.size() * sizeof(double), cudaMemcpyDeviceToHost, E.st));
    ENG_CUDA(cudaStreamSynchronize(E.st));
    for (int g = 0; g < E.world; g++) ok = ok && table[(size_t)g * per_rank + 3 * HB] == 1.0;
    *opened = ok;
    for (int g = 0; g < E.world && ok; g++) {
      if (g == E.rank) continue;
      cudaIpcMemHandle_t ph[3];
      for (int q = 0; q < 3; q++)
        for (int b = 0; b < HB; b++) reinterpret_cast<unsigned char*>(&ph[q])[b] = (unsigned char)table[(size_t)g * per_rank + q * HB + b];
      void* ptr[3] = {nullptr, nullptr, nullptr};
      for (int q = 0; q < 3; q++)
        if (cudaIpcOpenMemHandle(&ptr[q], ph[q], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { *opened = false; cudaGetLastError(); }
      dv.peer_S[g] = (double*)ptr[0]; dv.peer_linv[g] = (double*)ptr[1]; dv.peer_flag[g] = (int*)ptr[2];
    }
    return (int)CVB_OK;
  };
  return enable_p2p(E, true, map_peers, close);
}

// The peers' pointers from an in-process group (cvb_group_create enabled peer access between the ranks' devices).
int enable_p2p_group(Engine& E, cvb_group* g, int rank) {
  const auto map_peers = [&E, g, rank](cvb_chol::DistView& dv, bool* opened) {
    const void* mine[3] = {E.S.p, E.linv.p, E.pflag.p};
    const void* all[3 * CVB_GROUP_MAX];
    int rc = cvb_grp::exchange(g, rank, mine, 3, all);
    if (rc) return cvb_fail(E.ctx, rc, "peer pointer exchange failed (group failed)");
    for (int q = 0; q < E.world; q++) {
      dv.peer_S[q] = (double*)all[3 * q]; dv.peer_linv[q] = (double*)all[3 * q + 1]; dv.peer_flag[q] = (int*)all[3 * q + 2];
    }
    *opened = true;
    return (int)CVB_OK;
  };
  return enable_p2p(E, false, map_peers, [](cvb_chol::DistView&) {});
}

}  // namespace

// =================================================================================================
// C-ABI
// =================================================================================================
struct cvb_ba {
  Engine E;
  const cvb_ba_problem* prob = nullptr;
  cvb_ba_problem prob_copy;
};

extern "C" {

int cvb_ba_create(cvb_ctx* ctx, const cvb_ba_problem* p, const cvb_ba_options* o, cvb_ba** out) {
  if (!ctx || !p || !o || !out) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  *out = nullptr;
  cvb_ba* h = new cvb_ba();
  h->E.ctx = ctx;
  h->E.st = ctx->stream;
  h->prob_copy = *p;
  int rc = engine_setup(h->E, p, o);
  if (!rc) rc = engine_begin(h->E);
  if (rc) {
    delete h;
    return rc;
  }
  *out = h;
  return CVB_OK;
}

int cvb_ba_set_allreduce(cvb_ba* h, cvb_allreduce_fn fn, void* user) {
  if (!h) return CVB_ERR_INVALID;
  cudaStream_t st = h->E.st;
  if (fn)
    h->E.allreduce = [fn, user, st](void* p, size_t n) { return fn(user, p, n, (void*)st); };
  else
    h->E.allreduce = nullptr;
  return CVB_OK;
}

int cvb_ba_enable_p2p(cvb_ba* h) {
  if (!h) return CVB_ERR_INVALID;
  CVB_GUARD(h->E.ctx);
  return enable_p2p_ipc(h->E);
}

// Back to the state the problem was created with (the preintegrations were propagated at those biases), then iteration 0
// again: a restarted solve repeats the original one bit for bit.
int cvb_ba_restart(cvb_ba* h) {
  if (!h) return CVB_ERR_INVALID;
  CVB_GUARD(h->E.ctx);
  Engine& E = h->E;
  E.cur = 0;
  ENG_CUDA(cudaMemcpyAsync(E.pose[0].p, E.pose0.p, sizeof(double) * 7 * E.K, cudaMemcpyDeviceToDevice, E.st));
  ENG_CUDA(cudaMemcpyAsync(E.sb[0].p, E.sb0.p, sizeof(double) * 9 * E.K, cudaMemcpyDeviceToDevice, E.st));
  if (E.L_in) ENG_CUDA(cudaMemcpyAsync(E.lm[0].p, E.lm0.p, sizeof(double) * 3 * E.L_in, cudaMemcpyDeviceToDevice, E.st));
  return engine_begin(E);
}

int cvb_ba_iterate(cvb_ba* h, int max_iterations, int* iterations_done) {
  if (!h) return CVB_ERR_INVALID;
  CVB_GUARD(h->E.ctx);
  Engine& E = h->E;
  int n = 0;
  bool done = E.termination != TERM_NO_CONVERGENCE;
  while (!done && n < max_iterations) {
    int rc = engine_iterate(E, &done);
    if (rc) return rc;
    n++;
  }
  if (iterations_done) *iterations_done = n;
  return CVB_OK;
}

int cvb_ba_result_get(cvb_ba* h, const cvb_ba_problem* p, cvb_ba_result* r) {
  if (!h || !p || !r) return CVB_ERR_INVALID;
  CVB_GUARD(h->E.ctx);
  return engine_download(h->E, p, r);
}

int cvb_ba_reproj_norms(cvb_ba* h, double* norms, int n_obs) {
  if (!h || !norms) return CVB_ERR_INVALID;
  CVB_GUARD(h->E.ctx);
  return engine_corrected_norms(h->E, norms, n_obs);
}

// diagnostic: copy an internal vector ([camera part n_c_pad | landmark part 3 L_in]) to the host.
// which: 0 scale, 1 colsq, 2 diag, 3 gradient g, 4 grad/diag, 5 gn, 6 step, 7 x (linear solve), 8 reduced rhs
int cvb_ba_debug_vector(cvb_ba* h, int which, double* out, int64_t cap, int64_t* n_cam, int64_t* n_total) {
  if (!h) return CVB_ERR_INVALID;
  CVB_GUARD(h->E.ctx);
  Engine& E = h->E;
  const cvb_dev_arr<double>* v[] = {&E.scale, &E.colsq, &E.diag, &E.gvec, &E.grad, &E.gn, &E.step, &E.xsol, &E.gs};
  if (which < 0 || which > 8) return CVB_ERR_INVALID;
  const int64_t nc = (int64_t)E.K * E.per, tot = nc + 3 * (int64_t)E.L_in;
  if (n_cam) *n_cam = nc;
  if (n_total) *n_total = tot;
  if (out && cap >= tot) {
    std::vector<double> hv((size_t)E.n_vec);
    if (cudaMemcpyAsync(hv.data(), v[which]->p, hv.size() * sizeof(double), cudaMemcpyDeviceToHost, E.st) != cudaSuccess)
      return CVB_ERR_CUDA;
    cudaStreamSynchronize(E.st);
    for (int k = 0; k < E.K; k++)       // canonical order: keyframe-major [pose 6 | speed-bias 9]
      for (int c = 0; c < E.per; c++) out[(size_t)k * E.per + c] = hv[c < 6 ? E.h_off_pose[k] + c : E.h_off_sb[k] + (c - 6)];
    for (int64_t i = 0; i < 3 * (int64_t)E.L_in; i++) out[nc + i] = hv[(size_t)E.n_c_pad + i];
  }
  return CVB_OK;
}

// accumulated device time per phase (ms): [0] linearise, [1] block build + Schur, [2] Cholesky factorisation,
// [3] triangular solves + back-substitution, [4] dogleg / J*step / plus / candidate cost; [5] = dense-equivalent
// factorisation flops (n^3/3 per factorisation).  reset != 0 clears the counters after reading.
int cvb_ba_timing(cvb_ba* h, double out[6], int reset) {
  if (!h || !out) return CVB_ERR_INVALID;
  for (int i = 0; i < 5; i++) out[i] = h->E.phase_ms[i];
  out[5] = h->E.chol_flops;
  if (reset) {
    for (int i = 0; i < 5; i++) h->E.phase_ms[i] = 0.0;
    h->E.chol_flops = 0.0;
  }
  return CVB_OK;
}

int cvb_ba_destroy(cvb_ba* h) {
  if (h) {
    CVB_GUARD(h->E.ctx);
    cudaStreamSynchronize(h->E.st);
    delete h;
  }
  return CVB_OK;
}

// Optimization::PoseGraphOptimization / one round of GlobalBundleAdjustment: build, iterate, read back.
int cvb_ba_solve(cvb_ctx* ctx, const cvb_ba_problem* p, const cvb_ba_options* o, cvb_ba_result* r) {
  cvb_ba* h = nullptr;
  int rc = cvb_ba_create(ctx, p, o, &h);
  if (rc) return rc;
  rc = cvb_ba_iterate(h, o->max_iterations, nullptr);
  if (!rc) rc = cvb_ba_result_get(h, p, r);
  cvb_ba_destroy(h);
  return rc;
}

}  // extern "C"

int cvb_ba_solve_dev_edges(cvb_ctx* ctx, const cvb_ba_problem* p, const cvb_ba_options* o, cvb_ba_result* r, const cvb_dev_edges_fill& fill,
                           const std::function<int(const double* d_pose)>& finish) {
  CVB_GUARD(ctx);
  cvb_ba* h = new cvb_ba();
  h->E.ctx = ctx;
  h->E.st = ctx->stream;
  h->prob_copy = *p;
  Engine& E = h->E;
  int rc = engine_setup(E, p, o, &fill);
  if (!rc) rc = engine_begin(E);
  bool done = false;
  for (int n = 0; !rc && !done && n < o->max_iterations; n++) rc = engine_iterate(E, &done);
  if (!rc) rc = finish(E.pose[E.cur].p);
  if (!rc) rc = engine_download(E, p, r);
  cudaStreamSynchronize(E.st);
  delete h;
  return rc;
}

namespace {

// The two rounds of Optimization::GlobalBundleAdjustment (optimization_be.cpp:56-618) on the flat problem, around two
// solvers: round1(p1, o, norms) runs round 1 (5 iterations, loop edges without loss) and writes the loss-corrected
// residual norm of every observation; round2(p2, o) is round 2 from the ORIGINAL state (the reference re-reads the map at
// :325,454-457; round 1 only removes observations) with Cauchy(1) on loops, after the outlier purge of :270-290.
template <class Round1, class Round2>
int gba_rounds(const cvb_ba_problem* p, const cvb_gba_options* g, uint8_t* obs_removed, Round1 round1, Round2 round2) {
  std::vector<uint8_t> skip(p->n_obs > 0 ? p->n_obs : 1, 0), rb0(p->n_edge > 0 ? p->n_edge : 1, 0), rb1(p->n_edge > 0 ? p->n_edge : 1, 1);
  if (p->obs_skip) std::memcpy(skip.data(), p->obs_skip, (size_t)p->n_obs);
  cvb_ba_options o{};
  o.visual_only = g->visual_only;
  o.cauchy_reproj = 1.0;   // ceres::CauchyLoss(1.0), optimization_be.cpp:68,302
  o.cauchy_edge = 1.0;
  o.world = 1;
  int rc;
  if (g->outlier_removal) {
    cvb_ba_problem p1 = *p;
    p1.edge_robust = rb0.data();   // round 1: loop edges without loss (optimization_be.cpp:253)
    o.max_iterations = 5;          // :261
    std::vector<double> norms(p->n_obs > 0 ? p->n_obs : 1);
    if ((rc = round1(&p1, &o, norms.data()))) return rc;
    for (int i = 0; i < p->n_obs; i++)
      if (norms[i] > g->th_outlier) skip[i] = 1;   // th_gba_outlier_global, :277-281
  }
  if (obs_removed)
    for (int i = 0; i < p->n_obs; i++) obs_removed[i] = skip[i] && !(p->obs_skip && p->obs_skip[i]);
  cvb_ba_problem p2 = *p;
  p2.obs_skip = skip.data();
  p2.edge_robust = rb1.data();     // round 2: loss_function on the loop edges (:555)
  o.max_iterations = g->iterations_limit;
  return round2(&p2, &o);
}

// One sharded solve over an in-process group: one host thread per rank runs create -> group all-reduce -> [peer path] ->
// restart -> iterate on its context; then (after every rank's stream is idle) each rank's handle goes to done(rank, h)
// and is destroyed.  The handles outlive the rank threads so that no rank frees buffers a peer may still read.
int group_solve(cvb_group* g, const cvb_ba_problem* p, const cvb_ba_options* o_in, int peer_path,
                const std::function<int(int, cvb_ba*)>& done) {
  const int n = g->n;
  std::vector<cvb_ba*> h(n, nullptr);
  int rc = cvb_grp::run(g, [&](int r) {
    cvb_ba_options o = *o_in;
    o.rank = r;
    o.world = n;
    int rr = cvb_ba_create(g->ctx[r], p, &o, &h[r]);
    if (!rr) rr = cvb_ba_set_allreduce(h[r], cvb_grp::allreduce, &g->bind[r]);
    if (!rr && peer_path && n > 1) {
      CVB_GUARD(h[r]->E.ctx);
      rr = enable_p2p_group(h[r]->E, g, r);
    }
    if (!rr) rr = cvb_ba_restart(h[r]);
    if (!rr) rr = cvb_ba_iterate(h[r], o.max_iterations, nullptr);
    return rr;
  });
  for (int r = 0; r < n; r++)
    if (h[r]) {
      CVB_GUARD(h[r]->E.ctx);
      cudaStreamSynchronize(h[r]->E.st);
    }
  for (int r = 0; r < n && !rc; r++) {
    rc = done(r, h[r]);
    if (rc && r) cvb_fail(g->ctx[0], rc, "rank %d: %s", r, g->ctx[r]->err.c_str());
  }
  for (int r = 0; r < n; r++) cvb_ba_destroy(h[r]);
  return rc;
}

// every rank's result of a group solve, merged: rank 0's trajectory (checked bitwise against every other rank's), each
// landmark from its owner
int group_solve_merged(cvb_group* g, const cvb_ba_problem* p, const cvb_ba_options* o, int peer_path, cvb_ba_result* r,
                       const std::function<int(int, cvb_ba*)>& extra = nullptr) {
  const int n = g->n, K = p->K, L = p->L;
  const int cap = std::max(o->max_iterations, 0) + 2;   // iteration 0 + one cost per iteration
  struct Out {
    std::vector<double> pose, sb, lm, hist;
    std::vector<int32_t> owner;
    std::vector<uint8_t> steps;
    cvb_ba_result res{};
  };
  std::vector<Out> out(n);
  int rc = group_solve(g, p, o, peer_path, [&](int q, cvb_ba* h) {
    Out& x = out[q];
    x.pose.resize(7 * (size_t)K); x.sb.resize(9 * (size_t)K); x.lm.resize(3 * (size_t)std::max(L, 1)); x.hist.resize(cap);
    x.owner.resize(std::max(L, 1)); x.steps.resize(cap);
    x.res.pose = x.pose.data(); x.res.speedbias = x.sb.data(); x.res.lm = x.lm.data(); x.res.lm_owner = x.owner.data();
    x.res.cost_history = x.hist.data(); x.res.step_status = x.steps.data(); x.res.cost_history_cap = cap;
    int rr = cvb_ba_result_get(h, p, &x.res);
    if (!rr && extra) rr = extra(q, h);
    return rr;
  });
  if (rc) return rc;
  const Out& a = out[0];
  for (int q = 1; q < n; q++) {
    const Out& b = out[q];
    const bool same = a.res.n_cost_history == b.res.n_cost_history && a.res.iterations == b.res.iterations &&
                      a.res.termination == b.res.termination && a.pose == b.pose && a.sb == b.sb &&
                      std::memcmp(a.hist.data(), b.hist.data(), sizeof(double) * a.res.n_cost_history) == 0 &&
                      std::memcmp(a.steps.data(), b.steps.data(), (size_t)std::max(a.res.n_cost_history - 1, 0)) == 0;
    if (!same) return cvb_fail(g->ctx[0], CVB_ERR_NUMERIC, "rank %d's poses, speed-biases or cost history differ from rank 0's", q);
  }
  if (r->pose) std::memcpy(r->pose, a.pose.data(), sizeof(double) * 7 * (size_t)K);
  if (r->speedbias) std::memcpy(r->speedbias, a.sb.data(), sizeof(double) * 9 * (size_t)K);
  for (int l = 0; l < L; l++) {
    const int w = a.owner[l];
    if (r->lm) std::memcpy(r->lm + 3 * (size_t)l, (w >= 0 ? out[w].lm.data() : a.lm.data()) + 3 * (size_t)l, 3 * sizeof(double));
    if (r->lm_owner) r->lm_owner[l] = w;
  }
  r->iterations = a.res.iterations;
  r->termination = a.res.termination;
  r->initial_cost = a.res.initial_cost;
  r->final_cost = a.res.final_cost;
  r->n_cost_history = 0;
  if (r->cost_history && r->cost_history_cap > 0) {
    r->n_cost_history = std::min(r->cost_history_cap, a.res.n_cost_history);
    std::memcpy(r->cost_history, a.hist.data(), sizeof(double) * r->n_cost_history);
  }
  if (r->step_status && r->cost_history_cap > 0)
    std::memcpy(r->step_status, a.steps.data(), (size_t)std::min(r->cost_history_cap, std::max(a.res.n_cost_history - 1, 0)));
  return CVB_OK;
}

int group_check(cvb_group* g, const cvb_ba_problem* p, int visual_only, const void* o, const cvb_ba_result* r, int peer_path) {
  if (!g) return CVB_ERR_INVALID;
  if (!p || !o || !r) return cvb_fail(g->ctx[0], CVB_ERR_INVALID, "NULL problem, options or result");
  // The peer path needs a device per rank.  With two ranks on one device it stalled past the 20 s panel-wait bound (C1) and
  // once ended away from the world = 1 solve without reporting a failure (DESIGN.md §6), so it is refused there.
  if (peer_path)
    for (int a = 0; a < g->n; a++)
      for (int b = 0; b < a; b++)
        if (g->ctx[a]->device == g->ctx[b]->device)
          return cvb_fail(g->ctx[0], CVB_ERR_UNSUPPORTED, "peer path needs a device per rank: ranks %d and %d share device %d", b, a,
                          g->ctx[a]->device);
  return check_problem(g->ctx[0], p, visual_only);
}

}  // namespace

extern "C" {

int cvb_gba(cvb_ctx* ctx, const cvb_ba_problem* p, const cvb_gba_options* g, cvb_ba_result* r, uint8_t* obs_removed) {
  if (!ctx || !p || !g || !r) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  const auto round1 = [ctx, p](const cvb_ba_problem* p1, const cvb_ba_options* o, double* norms) {
    cvb_ba* h = nullptr;
    int rc = cvb_ba_create(ctx, p1, o, &h);
    if (rc) return rc;
    rc = cvb_ba_iterate(h, o->max_iterations, nullptr);
    if (!rc) rc = cvb_ba_reproj_norms(h, norms, p->n_obs);
    cvb_ba_destroy(h);
    return rc;
  };
  const auto round2 = [ctx, r](const cvb_ba_problem* p2, const cvb_ba_options* o) { return cvb_ba_solve(ctx, p2, o, r); };
  return gba_rounds(p, g, obs_removed, round1, round2);
}

int cvb_ba_solve_group(cvb_group* g, const cvb_ba_problem* p, const cvb_ba_options* o, int peer_path, cvb_ba_result* r) {
  if (!g) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> call_lk(g->call_mtx);   // the engines outlive the rank threads (group_solve)
  int rc = group_check(g, p, o ? o->visual_only : 0, o, r, peer_path);
  if (rc) return rc;
  return group_solve_merged(g, p, o, peer_path, r);
}

int cvb_gba_group(cvb_group* g, const cvb_ba_problem* p, const cvb_gba_options* gba, int peer_path, cvb_ba_result* r,
                  uint8_t* obs_removed) {
  if (!g) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> call_lk(g->call_mtx);
  int rc = group_check(g, p, gba ? gba->visual_only : 0, gba, r, peer_path);
  if (rc) return rc;
  const auto round1 = [g, p, peer_path](const cvb_ba_problem* p1, const cvb_ba_options* o, double* norms) {
    // each observation's norm from the rank that owns its landmark (the others report -1 for it)
    std::vector<std::vector<double>> per(g->n, std::vector<double>(p->n_obs > 0 ? p->n_obs : 1));
    cvb_ba_result r1{};
    int rc = group_solve_merged(g, p1, o, peer_path, &r1,
                                [&](int q, cvb_ba* h) { return cvb_ba_reproj_norms(h, per[q].data(), p->n_obs); });
    if (rc) return rc;
    for (int i = 0; i < p->n_obs; i++) {
      norms[i] = -1.0;
      for (int q = 0; q < g->n; q++)
        if (per[q][i] != -1.0) norms[i] = per[q][i];
    }
    return (int)CVB_OK;
  };
  const auto round2 = [g, r, peer_path](const cvb_ba_problem* p2, const cvb_ba_options* o) {
    return group_solve_merged(g, p2, o, peer_path, r);
  };
  return gba_rounds(p, gba, obs_removed, round1, round2);
}

}  // extern "C"
