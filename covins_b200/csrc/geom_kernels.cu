// geom_kernels.cu — guided search (FeatureMatcher::SearchBySE3) and RANSAC hypothesis scoring on the GPU
// (SURVEY.md §8a M8 / V1; the steps right after the k-NN / DenseMatcher stage of the place-recognition path).
//
// Replaces, behind include/covins_b200.h,
//   FeatureMatcher::SearchBySE3                      src/covins_backend/feature_matcher_be.cpp:293-498
//     (KeyframeBase::GetFeaturesInArea keyframe_base.cpp:262-318, IsInImage :414-416, LandmarkBase::PredictScale
//      landmark_base.cpp:120-133, DescriptorDistanceHamming feature_matcher_be.cpp:49-64)
//   FrameAbsolutePoseSacProblem::getSelectedDistancesToModel   include/covins/matcher/opengv/sac_problems/FrameAbsolutePoseSacProblem.h:95-126
//   FrameRelativePoseSacProblem::getSelectedDistancesToModel   include/covins/matcher/opengv/sac_problems/frame-relative-pose-sac-problem.hpp:69-104
// Both are small, latency-/HBM-bound stages: the search is one CTA per candidate keyframe pair (both directions and the
// agreement test in one launch for the whole batch of candidates), the scoring one thread per (hypothesis,
// correspondence) with a warp-shuffle + shared-memory inlier count.  All arithmetic uses explicit round-to-nearest
// non-fused operations (__dmul_rn / __dadd_rn / …) so that indices and scores are reproducible bit for bit against a
// plain IEEE evaluation (oracle/geom_oracle.c, compiled with -ffp-contract=off).
#include <float.h>
#include <limits.h>

#include <vector>

#include "ba_math.cuh"
#include "cvb_internal.cuh"
#include "geom_common.cuh"
#include "ransac_common.cuh"

namespace {

constexpr int GRID_COLS = 64, GRID_ROWS = 48;   // FRAME_GRID_COLS / FRAME_GRID_ROWS, typedefs_base.hpp:59-60

struct DevKf {
  int n;
  const float* kp; const float* octave; const uint8_t* desc; const uint8_t* lm_valid; const double* lm_pos;
  const double* lm_maxdist; const uint8_t* lm_desc; const int* grid_ptr; const int* grid_idx;
  double grid_w_inv, grid_h_inv, K[9], Tcw[16], img[4];
};
struct DevPair {
  DevKf k2;
  double T12[16], T21[16];
  const uint8_t* already1; const uint8_t* already2;
  int* match1; int* match2; int* match12; int* n_found;
};

__device__ __forceinline__ void rt_apply(const double* T, const double* p, double* o) {
#pragma unroll
  for (int r = 0; r < 3; r++) o[r] = add(dot3(T[4 * r], T[4 * r + 1], T[4 * r + 2], p), T[4 * r + 3]);
}
__device__ __forceinline__ int ham256(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b) {
  const uint4 a0 = __ldg(reinterpret_cast<const uint4*>(a)), a1 = __ldg(reinterpret_cast<const uint4*>(a) + 1);
  const uint4 b0 = __ldg(reinterpret_cast<const uint4*>(b)), b1 = __ldg(reinterpret_cast<const uint4*>(b) + 1);
  return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) +
         __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}
__device__ __forceinline__ bool in_image(const double* img, double x, double y) { return x >= img[0] && x < img[1] && y >= img[2] && y < img[3]; }

// LandmarkBase::PredictScale: ceil(log(ratio) / log(scale_factor)) clamped to [0, num_octaves - 1], as libm evaluates it.  That
// level is monotone in ratio, so it is n = #{k : ratio > steps[k]} for the num_octaves - 1 ratios where it steps up (scale_table,
// on the host).  Repeated multiplication by scale_factor is not the same: at scale_factor 1.2, ratio = 1.2 * 1.2 rounded gives
// level 3 by the logarithms and 2 by the products.
__device__ __forceinline__ int predict_scale(double maxdist, double dist3d, const double* steps, int num_octaves) {
  const double ratio = __ddiv_rn(maxdist, (double)(float)dist3d);   // `const float& currentDist`
  int n = 0;
  while (n < num_octaves - 1 && ratio > steps[n]) n++;
  return n;
}

// best keypoint of `dst` for landmark i of `src` (float_best: direction 1→2 keeps the best distance as float — the same
// integers — and both directions take the FIRST strict minimum in the grid's candidate order)
__device__ int search_one(const DevKf& src, int i, const double* Tcw_src, const double* Tab, const double* Kdst, const DevKf& dst,
                          const double* img, double th, const double* steps, int num_octaves, int* best_dist) {
  double pw[3] = {src.lm_pos[3 * (size_t)i], src.lm_pos[3 * (size_t)i + 1], src.lm_pos[3 * (size_t)i + 2]};
  double pc_src[3], pc[3];
  rt_apply(Tcw_src, pw, pc_src);
  rt_apply(Tab, pc_src, pc);
  if (pc[2] < 0.0) return -1;
  const double p0 = dot3(Kdst[0], Kdst[1], Kdst[2], pc), p1 = dot3(Kdst[3], Kdst[4], Kdst[5], pc), p2 = dot3(Kdst[6], Kdst[7], Kdst[8], pc);
  const double u = __ddiv_rn(p0, p2), v = __ddiv_rn(p1, p2);
  if (!in_image(img, u, v)) return -1;
  const double dist3d = __dsqrt_rn(add(add(mul(pc[0], pc[0]), mul(pc[1], pc[1])), mul(pc[2], pc[2])));
  const int level = predict_scale(src.lm_maxdist[i], dist3d, steps, num_octaves);
  const double radius = mul(th, scalbn(1.0, level));
  const float tx = (float)u, ty = (float)v;
  int min_cx = (int)floor(mul(sub((double)tx, radius), dst.grid_w_inv)); if (min_cx < 0) min_cx = 0;
  if (min_cx >= GRID_COLS) return -1;
  int max_cx = (int)ceil(mul(add((double)tx, radius), dst.grid_w_inv)); if (max_cx > GRID_COLS - 1) max_cx = GRID_COLS - 1;
  if (max_cx < 0) return -1;
  int min_cy = (int)floor(mul(sub((double)ty, radius), dst.grid_h_inv)); if (min_cy < 0) min_cy = 0;
  if (min_cy >= GRID_ROWS) return -1;
  int max_cy = (int)ceil(mul(add((double)ty, radius), dst.grid_h_inv)); if (max_cy > GRID_ROWS - 1) max_cy = GRID_ROWS - 1;
  if (max_cy < 0) return -1;
  int bd = INT_MAX, best = -1;
  const uint8_t* dl = src.lm_desc + 32 * (size_t)i;
  for (int ix = min_cx; ix <= max_cx; ix++)
    for (int iy = min_cy; iy <= max_cy; iy++) {
      const int c = ix * GRID_ROWS + iy;
      for (int q = dst.grid_ptr[c]; q < dst.grid_ptr[c + 1]; q++) {
        const int idx = dst.grid_idx[q];
        const float dx = __fsub_rn(dst.kp[2 * (size_t)idx], tx), dy = __fsub_rn(dst.kp[2 * (size_t)idx + 1], ty);
        const float nrm = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
        if (!((double)nrm <= radius)) continue;
        const int lvl = (int)dst.octave[idx];
        if (lvl < level - 1 || lvl > level) continue;
        const int d = ham256(dl, dst.desc + 32 * (size_t)idx);
        if (d < bd) { bd = d; best = idx; }
      }
    }
  *best_dist = bd;
  return best;
}

__global__ void __launch_bounds__(256) search_se3_kernel(DevKf k1, const DevPair* __restrict__ pairs, double th, int th_low, const double* __restrict__ steps,
                                                         int num_octaves) {
  const DevPair& P = pairs[blockIdx.x];
  const DevKf& k2 = P.k2;
  const int n1 = k1.n, n2 = k2.n;
  __shared__ int found;
  if (threadIdx.x == 0) found = 0;
  for (int i = threadIdx.x; i < n1; i += blockDim.x) {   // KF1 → KF2 (:327-406)
    int m = -1;
    if (k1.lm_valid[i] && !P.already1[i]) {
      int bd;
      const int b = search_one(k1, i, k1.Tcw, P.T21, k2.K, k2, k2.img, th, steps, num_octaves, &bd);
      if (b >= 0 && bd <= th_low) m = b;              // bestDist <= desc_matching_th_low_ (:403)
    }
    P.match1[i] = m;
  }
  for (int i = threadIdx.x; i < n2; i += blockDim.x) {   // KF2 → KF1 (:409-482); IsInImage of pKF2 (:433)
    int m = -1;
    if (k2.lm_valid[i] && !P.already2[i]) {
      int bd;
      const int b = search_one(k2, i, k2.Tcw, P.T12, k1.K, k1, k2.img, th, steps, num_octaves, &bd);
      if (b >= 0 && bd < th_low) m = b;               // bestDist < desc_matching_th_low_ (:479)
    }
    P.match2[i] = m;
  }
  __syncthreads();   // this CTA wrote match1 / match2 itself: block-level visibility is enough
  int cnt = 0;
  for (int i = threadIdx.x; i < n1; i += blockDim.x) {   // agreement (:485-496): match2[i], not match2[idx2]
    const int idx2 = P.match1[i];
    int out = -1;
    if (idx2 >= 0 && i < n2 && P.match2[i] == i) { out = idx2; cnt++; }
    P.match12[i] = out;
  }
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&found, cnt);
  __syncthreads();
  if (threadIdx.x == 0) *P.n_found = found;
}

// ---- FeatureMatcher::SearchByProjection (feature_matcher_be.cpp:168-291) ---------------------------------------------
// Phase A (all threads of ONE CTA): every candidate landmark is projected with the keyframe's full camera model, gated
// (image bounds, distance invariance, viewing angle) and its keypoints in the search radius are listed — in the grid's
// candidate order, with their Hamming distances, octave gate applied (at most kProjCap per landmark).  Phase B (thread 0):
// the reference's sequential semantics — a keypoint taken by an earlier landmark is skipped, the first strict minimum wins,
// RemapLandmark bookkeeping — over those short lists.  The order dependence is inherent to the reference (vpMatched is
// updated while the loop runs); the expensive part (projection, radius search, distances) is what runs in parallel.
constexpr int kProjCap = 48;
struct ProjDev {
  int m;
  const uint8_t* valid; const double* pos; const double* normal; const double* min_dist; const double* max_dist;
  const double* max_distance; const uint8_t* desc; const int* feat_idx;
  double Tcw[16], intr[4], dist[4], xi;
  int cam, dm;
  int* cand_idx; int* cand_dist; int* cand_n;      // [m][kProjCap], [m]
  uint8_t* matched; uint8_t* has_lm; int* lm_cand; int* feat;   // working copies [n], [n], [n], [m]
  int* action; int* best_idx; int* n_matches; int* overflow;
};

__global__ void __launch_bounds__(256, 1) search_proj_kernel(DevKf kf, ProjDev P, double th, int th_low, const double* __restrict__ scale, int num_octaves) {
  double Ow[3];
#pragma unroll
  for (int r = 0; r < 3; r++) Ow[r] = -add(add(mul(P.Tcw[r], P.Tcw[3]), mul(P.Tcw[4 + r], P.Tcw[7])), mul(P.Tcw[8 + r], P.Tcw[11]));
  for (int i = threadIdx.x; i < P.m; i += blockDim.x) {
    int cnt = -1;   // -1 = gated out
    do {
      if (!P.valid[i]) break;
      const double pw[3] = {P.pos[3 * (size_t)i], P.pos[3 * (size_t)i + 1], P.pos[3 * (size_t)i + 2]};
      double pc[3];
      rt_apply(P.Tcw, pw, pc);
      if (pc[2] < 0.0) break;
      double u, v;
      if (!project3_rn(P.intr, P.dist, P.cam, P.dm, P.xi, pc, &u, &v)) break;
      if (!in_image(kf.img, u, v)) break;
      const double PO[3] = {sub(pw[0], Ow[0]), sub(pw[1], Ow[1]), sub(pw[2], Ow[2])};
      const double d3 = __dsqrt_rn(add(add(mul(PO[0], PO[0]), mul(PO[1], PO[1])), mul(PO[2], PO[2])));
      if (d3 < P.min_dist[i] || d3 > P.max_dist[i]) break;
      if (add(add(mul(PO[0], P.normal[3 * (size_t)i]), mul(PO[1], P.normal[3 * (size_t)i + 1])), mul(PO[2], P.normal[3 * (size_t)i + 2])) < mul(0.5, d3)) break;
      const int level = predict_scale(P.max_distance[i], d3, scale, num_octaves);
      const double radius = mul(th, scale[num_octaves - 1 + level]);   // th * pow(scale_factor, level)
      const float tx = (float)u, ty = (float)v;
      int min_cx = (int)floor(mul(sub((double)tx, radius), kf.grid_w_inv)); if (min_cx < 0) min_cx = 0;
      if (min_cx >= GRID_COLS) break;
      int max_cx = (int)ceil(mul(add((double)tx, radius), kf.grid_w_inv)); if (max_cx > GRID_COLS - 1) max_cx = GRID_COLS - 1;
      if (max_cx < 0) break;
      int min_cy = (int)floor(mul(sub((double)ty, radius), kf.grid_h_inv)); if (min_cy < 0) min_cy = 0;
      if (min_cy >= GRID_ROWS) break;
      int max_cy = (int)ceil(mul(add((double)ty, radius), kf.grid_h_inv)); if (max_cy > GRID_ROWS - 1) max_cy = GRID_ROWS - 1;
      if (max_cy < 0) break;
      cnt = 0;
      const uint8_t* dl = P.desc + 32 * (size_t)i;
      for (int ix = min_cx; ix <= max_cx; ix++)
        for (int iy = min_cy; iy <= max_cy; iy++) {
          const int c = ix * GRID_ROWS + iy;
          for (int q = kf.grid_ptr[c]; q < kf.grid_ptr[c + 1]; q++) {
            const int idx = kf.grid_idx[q];
            const float dx = __fsub_rn(kf.kp[2 * (size_t)idx], tx), dy = __fsub_rn(kf.kp[2 * (size_t)idx + 1], ty);
            if (!((double)__fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) <= radius)) continue;
            const int lvl = (int)kf.octave[idx];
            if (lvl < level - 1 || lvl > level) continue;
            if (cnt < kProjCap) { P.cand_idx[(size_t)i * kProjCap + cnt] = idx; P.cand_dist[(size_t)i * kProjCap + cnt] = ham256(dl, kf.desc + 32 * (size_t)idx); }
            cnt++;
          }
        }
      if (cnt > kProjCap) atomicExch(P.overflow, 1);
    } while (false);
    P.cand_n[i] = cnt;
    P.action[i] = 0; P.best_idx[i] = -1;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  int nm = 0;
  for (int i = 0; i < P.m; i++) {
    const int cn = P.cand_n[i] < kProjCap ? P.cand_n[i] : kProjCap;
    int bd = 256, best = -1;
    for (int q = 0; q < cn; q++) {
      const int idx = P.cand_idx[(size_t)i * kProjCap + q];
      if (P.matched[idx]) continue;                                     // if (vpMatched[idx]) continue (:239)
      const int d = P.cand_dist[(size_t)i * kProjCap + q];
      if (d < bd) { bd = d; best = idx; }
    }
    if (best < 0 || bd > th_low) continue;                             // bestDist <= desc_matching_th_low_ (:258)
    P.best_idx[i] = best;
    const int existing = P.feat[i];
    if (existing != -1) {                                               // already observed (:260-282)
      const uint8_t* dl = P.desc + 32 * (size_t)i;
      bool keep = ham256(dl, kf.desc + 32 * (size_t)existing) < bd;
      if (P.has_lm[best] && ham256(dl, kf.desc + 32 * (size_t)best) < bd) keep = true;
      if (keep) { P.action[i] = 3; continue; }
      const int displaced = P.lm_cand[best];                            // RemapLandmark (keyframe_be.cpp:484-495)
      const bool had = P.has_lm[best] != 0;
      P.has_lm[existing] = 0; P.lm_cand[existing] = -1;
      P.has_lm[best] = 1; P.lm_cand[best] = i; P.feat[i] = best;
      if (had && displaced >= 0) P.feat[displaced] = -1;                // lm_new->EraseObservation comes LAST (:494): existing == best un-observes lm itself
      P.action[i] = 2;
    } else {
      P.matched[best] = 1;                                              // vpMatched[bestIdx] = pMP (:285)
      P.action[i] = 1; nm++;
    }
  }
  *P.n_matches = nm;
}

// ---- V1 scoring: block = (chunk of 256 correspondences, hypothesis) ------------------------------------------------
__global__ void __launch_bounds__(256) score_abs_kernel(const double* __restrict__ model, const double* __restrict__ pts,
                                                        const double* __restrict__ f, const double* __restrict__ sigma, int n,
                                                        const double* __restrict__ cam, double threshold, double* __restrict__ scores,
                                                        uint8_t* __restrict__ inlier, int* __restrict__ n_inliers) {
  const int h = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const double* M = model + 12 * (size_t)h;
  int in = 0;
  if (i < n) {
    double Ri[9], ti[3];
    abs_inverse(M, Ri, ti);
    const double s = abs_score(Ri, ti, pts + 3 * (size_t)i, f + 3 * (size_t)i, sigma[i], cam);
    in = s < threshold;
    if (scores) scores[(size_t)h * n + i] = s;
    if (inlier) inlier[(size_t)h * n + i] = (uint8_t)in;
  }
  for (int o = 16; o > 0; o >>= 1) in += __shfl_xor_sync(0xffffffffu, in, o);
  if ((threadIdx.x & 31) == 0 && in) atomicAdd(n_inliers + h, in);   // integer: order-independent
}

__global__ void __launch_bounds__(256) score_rel_kernel(const double* __restrict__ model, const double* __restrict__ f1,
                                                        const double* __restrict__ f2, const double* __restrict__ s1,
                                                        const double* __restrict__ s2, int n, double threshold, double* __restrict__ scores,
                                                        uint8_t* __restrict__ inlier, int* __restrict__ n_inliers) {
  const int h = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const double* M = model + 12 * (size_t)h;
  int in = 0;
  if (i < n) {
    const double s = rel_score(M, f1, f2, s1, s2, i);
    in = s < threshold;
    if (scores) scores[(size_t)h * n + i] = s;
    if (inlier) inlier[(size_t)h * n + i] = (uint8_t)in;
  }
  for (int o = 16; o > 0; o >>= 1) in += __shfl_xor_sync(0xffffffffu, in, o);
  if ((threadIdx.x & 31) == 0 && in) atomicAdd(n_inliers + h, in);
}

// keyframe view v into d: its arrays bound as inputs of B, its scalars copied (with_desc = false: the caller binds the
// descriptor rows)
void bind_kf(cvb_block& B, DevKf& d, const cvb_kf_view* v, bool with_desc = true) {
  const size_t n = (size_t)v->n;
  B.in(d.kp, v->kp, n * 2); B.in(d.octave, v->octave, n);
  if (with_desc) B.in(d.desc, v->desc, n * 32);
  B.in(d.lm_valid, v->lm_valid, n); B.in(d.lm_pos, v->lm_pos, n * 3); B.in(d.lm_maxdist, v->lm_maxdist, n); B.in(d.lm_desc, v->lm_desc, n * 32);
  B.in(d.grid_ptr, v->grid_ptr, GRID_COLS * GRID_ROWS + 1); B.in(d.grid_idx, v->grid_idx, (size_t)v->grid_ptr[GRID_COLS * GRID_ROWS]);
  d.n = v->n;
  d.grid_w_inv = v->grid_w_inv; d.grid_h_inv = v->grid_h_inv;
  memcpy(d.K, v->K, sizeof(d.K)); memcpy(d.Tcw, v->Tcw, sizeof(d.Tcw)); memcpy(d.img, v->img, sizeof(d.img));
}
bool kf_ok(const cvb_kf_view* v) {
  if (!v || v->n < 0 || !v->grid_ptr) return false;
  if (v->n > 0 && (!v->kp || !v->octave || !v->desc || !v->lm_valid || !v->lm_pos || !v->lm_maxdist || !v->lm_desc)) return false;
  if (v->grid_ptr[0] != 0) return false;
  for (int c = 0; c < GRID_COLS * GRID_ROWS; c++)
    if (v->grid_ptr[c + 1] < v->grid_ptr[c]) return false;
  const int m = v->grid_ptr[GRID_COLS * GRID_ROWS];
  if (m > v->n || (m > 0 && !v->grid_idx)) return false;
  for (int q = 0; q < m; q++)
    if (v->grid_idx[q] < 0 || v->grid_idx[q] >= v->n) return false;
  return true;
}

// the host half of predict_scale and of SearchByProjection's radius th * pow(scale_factor, level), both by host libm as
// LandmarkBase::PredictScale and the search evaluate them: [0, num_octaves - 1) the largest ratio of each level k below the
// last (ratio > steps[k] <=> level > k; +inf if no finite ratio reaches level k + 1), then pow(scale_factor, l) for
// l = 0 .. num_octaves - 1.  Requires scale_factor > 1.
std::vector<double> scale_table(double sf, int num_octaves) {
  auto level = [&](double r) {
    const int n = (int)ceil(log(r) / log(sf));
    return n < 0 ? 0 : (n >= num_octaves ? num_octaves - 1 : n);
  };
  auto bits = [](double d) { uint64_t u; memcpy(&u, &d, 8); return u; };
  std::vector<double> t(2 * (size_t)num_octaves - 1);
  for (int k = 0; k + 1 < num_octaves; k++) {
    if (level(DBL_MAX) <= k) { t[k] = INFINITY; continue; }
    uint64_t lo = bits(1.0), hi = bits(DBL_MAX);   // level(lo) <= k < level(hi); positive doubles order like their bits
    while (hi - lo > 1) {
      const uint64_t mid = lo + (hi - lo) / 2;
      double r;
      memcpy(&r, &mid, 8);
      (level(r) <= k ? lo : hi) = mid;
    }
    memcpy(&t[k], &lo, 8);
  }
  for (int l = 0; l < num_octaves; l++) t[num_octaves - 1 + l] = pow(sf, (double)l);
  return t;
}

}  // namespace

extern "C" {

int cvb_search_by_se3_batch(cvb_ctx* ctx, const cvb_kf_view* kf1, const cvb_kf_view* kf2, int n_pairs, const double* T12,
                            const double* T21, const uint8_t* already1, const uint8_t* already2, const cvb_search_params* prm,
                            int32_t* match12, int32_t* n_found, int32_t* match1, int32_t* match2) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, kf1 && prm && n_pairs >= 0 && (n_pairs == 0 || (kf2 && T12 && T21 && already1 && match12 && n_found)), "search_by_se3: bad arguments");
  CVB_REQUIRE(ctx, kf_ok(kf1), "search_by_se3: malformed keyframe view (kf1)");
  CVB_REQUIRE(ctx, prm->num_octaves >= 1 && prm->scale_factor > 1.0 && prm->th > 0.0, "search_by_se3: bad parameters");
  if (n_pairs == 0) return CVB_OK;
  size_t n2_total = 0;
  for (int p = 0; p < n_pairs; p++) {
    CVB_REQUIRE(ctx, kf_ok(kf2 + p), "search_by_se3: malformed keyframe view (kf2[%d])", p);
    n2_total += (size_t)kf2[p].n;
  }
  CVB_REQUIRE(ctx, n2_total == 0 || already2, "search_by_se3: already2 is null");
  const size_t n1 = (size_t)kf1->n;
  cvb_block B(ctx, ctx->stream);
  DevKf d1{};
  bind_kf(B, d1, kf1);
  std::vector<DevPair> hp((size_t)n_pairs);   // the records the kernel reads, uploaded at d_pairs
  for (int p = 0; p < n_pairs; p++) bind_kf(B, hp[p].k2, kf2 + p);
  const uint8_t *d_a1, *d_a2;
  DevPair* d_pairs;
  int *d_m1, *d_m2, *d_m12, *d_nf;
  const std::vector<double> scale = scale_table(prm->scale_factor, prm->num_octaves);
  const double* d_scale;
  B.in(d_a1, already1, (size_t)n_pairs * n1); B.in(d_a2, already2, n2_total); B.in(d_pairs, nullptr, n_pairs); B.in(d_scale, scale.data(), scale.size());
  B.out(d_m1, match1, (size_t)n_pairs * n1); B.out(d_m2, match2, n2_total); B.out(d_m12, match12, (size_t)n_pairs * n1); B.out(d_nf, n_found, n_pairs);
  if (const int rc = B.place()) return rc;
  size_t a2 = 0;
  for (int p = 0; p < n_pairs; p++) {
    DevPair& P = hp[p];
    memcpy(P.T12, T12 + 16 * (size_t)p, sizeof(P.T12)); memcpy(P.T21, T21 + 16 * (size_t)p, sizeof(P.T21));
    P.already1 = d_a1 + (size_t)p * n1; P.already2 = d_a2 + a2;
    P.match1 = d_m1 + (size_t)p * n1; P.match2 = d_m2 + a2; P.match12 = d_m12 + (size_t)p * n1; P.n_found = d_nf + p;
    a2 += (size_t)kf2[p].n;
  }
  memcpy(B.host(d_pairs), hp.data(), hp.size() * sizeof(DevPair));
  if (const int rc = B.upload()) return rc;
  search_se3_kernel<<<n_pairs, 256, 0, ctx->stream>>>(d1, d_pairs, prm->th, prm->desc_th_low, d_scale, prm->num_octaves);
  CVB_CHECK_LAUNCH(ctx);
  return B.download();
}

static int score_common(cvb_ctx* ctx, bool relative, const double* model, int n_hyp, const double* a, const double* b, const double* s1,
                        const double* s2, int n, const double* cam_off, const double* cam_rot, double threshold, double* scores,
                        uint8_t* inlier, int32_t* n_inliers) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, n_hyp >= 0 && n >= 0 && n_inliers && (n_hyp == 0 || model), "score: bad arguments");
  CVB_REQUIRE(ctx, n == 0 || (a && b && s1 && (relative ? s2 != nullptr : (cam_off && cam_rot))), "score: null correspondence arrays");
  CVB_REQUIRE(ctx, n_hyp <= 65535, "score: at most 65535 hypotheses per call");
  for (int h = 0; h < n_hyp; h++) n_inliers[h] = 0;
  if (n_hyp == 0 || n == 0) return CVB_OK;
  const size_t hn = (size_t)n_hyp * n;
  double cam[12];   // one camera: offset (3) directly followed by the rotation (9, row-major)
  cvb_block B(ctx, ctx->stream);
  const double *d_model, *d_a, *d_b, *d_s1, *d_s2, *d_cam;
  int* d_cnt;
  double* d_sc = nullptr;
  uint8_t* d_in = nullptr;
  B.in(d_model, model, (size_t)n_hyp * 12); B.in(d_a, a, (size_t)n * 3); B.in(d_b, b, (size_t)n * 3); B.in(d_s1, s1, n);
  if (relative) {
    B.in(d_s2, s2, n);
  } else {
    memcpy(cam, cam_off, 24); memcpy(cam + 3, cam_rot, 72);
    B.in(d_cam, cam, 12);
  }
  B.out(d_cnt, n_inliers, n_hyp);
  if (scores) B.out(d_sc, scores, hn);
  if (inlier) B.out(d_in, inlier, hn);
  if (const int rc = B.place()) return rc;
  if (const int rc = B.upload()) return rc;
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, (size_t)n_hyp * 4, st));
  const dim3 grid((unsigned)((n + 255) / 256), (unsigned)n_hyp);
  if (relative) score_rel_kernel<<<grid, 256, 0, st>>>(d_model, d_a, d_b, d_s1, d_s2, n, threshold, d_sc, d_in, d_cnt);
  else score_abs_kernel<<<grid, 256, 0, st>>>(d_model, d_a, d_b, d_s1, n, d_cam, threshold, d_sc, d_in, d_cnt);
  CVB_CHECK_LAUNCH(ctx);
  return B.download();
}

int cvb_score_absolute_pose_batch(cvb_ctx* ctx, const double* model, int n_hyp, const double* pts, const double* f, const double* sigma,
                                  int n, const double* cam_off, const double* cam_rot, double threshold, double* scores, uint8_t* inlier,
                                  int32_t* n_inliers) {
  return score_common(ctx, false, model, n_hyp, pts, f, sigma, nullptr, n, cam_off, cam_rot, threshold, scores, inlier, n_inliers);
}

int cvb_score_relative_pose_batch(cvb_ctx* ctx, const double* model, int n_hyp, const double* f1, const double* f2, const double* sigma1,
                                  const double* sigma2, int n, double threshold, double* scores, uint8_t* inlier, int32_t* n_inliers) {
  return score_common(ctx, true, model, n_hyp, f1, f2, sigma1, sigma2, n, nullptr, nullptr, threshold, scores, inlier, n_inliers);
}

int cvb_search_by_projection(cvb_ctx* ctx, const cvb_kf_view* kf, const int32_t* kf_lm_cand, const double* Tcw, const double* intr,
                             const double* dist, int cam_model, int dist_model, double xi, const cvb_proj_landmarks* lms,
                             const uint8_t* matched, const cvb_search_params* prm, int32_t* action, int32_t* best_idx, int32_t* n_matches) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, kf && Tcw && intr && dist && lms && prm && n_matches && lms->m >= 0, "search_by_projection: bad arguments");
  CVB_REQUIRE(ctx, kf->n >= 0 && kf->grid_ptr && (kf->n == 0 || (kf->kp && kf->octave && kf->desc && kf->lm_valid && kf_lm_cand && matched)),
              "search_by_projection: malformed keyframe view");
  CVB_REQUIRE(ctx, kf->grid_ptr[0] == 0 && kf->grid_ptr[GRID_COLS * GRID_ROWS] <= kf->n, "search_by_projection: malformed grid");
  CVB_REQUIRE(ctx, prm->num_octaves >= 1 && prm->scale_factor > 1.0 && prm->th > 0.0, "search_by_projection: bad parameters");
  if (cam_model < 0 || cam_model > 1) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown projection type.");
  if (dist_model < 0 || dist_model > 2) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown distortion type.");
  const int n = kf->n, m = lms->m;
  *n_matches = 0;
  if (m == 0) return CVB_OK;
  CVB_REQUIRE(ctx, lms->valid && lms->pos && lms->normal && lms->min_dist && lms->max_dist && lms->max_distance && lms->desc && lms->feat_idx &&
              action && best_idx, "search_by_projection: null landmark arrays");
  for (int i = 0; i < m; i++) CVB_REQUIRE(ctx, lms->feat_idx[i] >= -1 && lms->feat_idx[i] < n, "search_by_projection: feat_idx out of range");
  for (int i = 0; i < n; i++) CVB_REQUIRE(ctx, kf_lm_cand[i] >= -1 && kf_lm_cand[i] < m, "search_by_projection: kf_lm_cand out of range");
  cvb_block B(ctx, ctx->stream);
  DevKf K{};
  ProjDev P{};
  B.in(K.kp, kf->kp, (size_t)n * 2); B.in(K.octave, kf->octave, n); B.in(K.desc, kf->desc, (size_t)n * 32);
  B.in(K.grid_ptr, kf->grid_ptr, GRID_COLS * GRID_ROWS + 1); B.in(K.grid_idx, kf->grid_idx, (size_t)kf->grid_ptr[GRID_COLS * GRID_ROWS]);
  B.in(P.has_lm, kf->lm_valid, n); B.in(P.lm_cand, kf_lm_cand, n); B.in(P.matched, matched, n);
  B.in(P.valid, lms->valid, m); B.in(P.pos, lms->pos, (size_t)m * 3); B.in(P.normal, lms->normal, (size_t)m * 3); B.in(P.min_dist, lms->min_dist, m);
  B.in(P.max_dist, lms->max_dist, m); B.in(P.max_distance, lms->max_distance, m); B.in(P.desc, lms->desc, (size_t)m * 32);
  B.in(P.feat_idx, lms->feat_idx, m); B.in(P.feat, lms->feat_idx, m);
  const std::vector<double> scale = scale_table(prm->scale_factor, prm->num_octaves);
  const double* d_scale;
  B.in(d_scale, scale.data(), scale.size());
  B.tmp(P.cand_idx, (size_t)m * kProjCap); B.tmp(P.cand_dist, (size_t)m * kProjCap); B.tmp(P.cand_n, m);
  B.out_host(P.action, m); B.out_host(P.best_idx, m); B.out_host(P.n_matches, 2);   // n_matches, then the overflow flag
  if (const int rc = B.place()) return rc;
  if (const int rc = B.upload()) return rc;
  K.n = n; K.grid_w_inv = kf->grid_w_inv; K.grid_h_inv = kf->grid_h_inv;
  memcpy(K.img, kf->img, sizeof(K.img));
  P.m = m;
  memcpy(P.Tcw, Tcw, sizeof(P.Tcw)); memcpy(P.intr, intr, 32); memcpy(P.dist, dist, 32);
  P.xi = xi; P.cam = cam_model; P.dm = dist_model;
  P.overflow = P.n_matches + 1;
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemsetAsync(P.n_matches, 0, 8, st));
  search_proj_kernel<<<1, 256, 0, st>>>(K, P, prm->th, prm->desc_th_low, d_scale, prm->num_octaves);
  CVB_CHECK_LAUNCH(ctx);
  if (const int rc = B.download()) return rc;
  const int* tail = B.host(P.n_matches);
  if (tail[1]) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "search_by_projection: more than %d keypoints in a search radius", kProjCap);
  memcpy(action, B.host(P.action), (size_t)m * 4); memcpy(best_idx, B.host(P.best_idx), (size_t)m * 4);
  *n_matches = tail[0];
  return CVB_OK;
}

}  // extern "C"

// ---- the COVINS verification chain of cvb_verify_landmark_candidates_seeded_batch on the device ----
// The DenseMatcher scan and assignment (cvb_landmark_match_batch_dev), lmv_gather_kernel (matches -> RANSAC problems),
// ransac_abs_kernel<SeededSamples<4>> (cvb_abs_ransac_seeded_dev), lmv_pose_kernel (gate, T12 / T21, already-masks),
// search_se3_kernel, lmv_residual_kernel (LandmarkVector -> residual pairs) and relpose_kernel (cvb_relpose_batch_dev), all on
// the arrays of one device block (cvb_block).  The per-candidate arrays are sized by the host-known bound n_cand x n_query; the RANSAC
// problems are packed to the front in candidate order.  The DevPair and relpose records hold pointers that depend only on
// sizes, so the host fills them; the device writes their T12 / T21 and n.
namespace {

struct LmvDev {
  int nq, min_matches, min_inliers;
  const int* seg;                                       // [C+1] the candidates' rows in the concatenated B
  const int* outA; const int* outB; const int* n_out;   // the matcher's matches, per segment ordered by B
  const double* q_bear; const double* q_sig;            // query [nq][3], [nq]
  const uint8_t* q_valid; const double* q_pos; const float* q_kp; const float* q_oct;
  double q_Tsc[16], TcwA[16];
  const double* TcwB;                                   // [C][16]
  int* row;                                             // [C][nq] the idxB matched to query keypoint i, or -1
  int* prob_ptr; double* pts; double* f; double* sg; int* srcA;   // the RANSAC problems, packed
  const int* best_sample; const double* best_model; const int* best_count; const uint8_t* mask;
  uint8_t* already1; uint8_t* stage; int* match12;      // [C][nq]
  double* T12; double* T21; double* pose_in;            // [C][16], [C][16], [C][7]
  double* pA; double* pB; float* kA; float* kB; double* sA; double* sB;   // residual pairs of candidate c from c * nq
  int* n_corr;
};

// rows 0..2 of A * B (4x4 row-major), each entry four products summed left to right; row 3 = 0 0 0 1
__device__ void mul44_rn(const double* A, const double* B, double* O) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++)
      O[4 * r + c] = add(add(add(mul(A[4 * r], B[c]), mul(A[4 * r + 1], B[4 + c])), mul(A[4 * r + 2], B[8 + c])), mul(A[4 * r + 3], B[12 + c]));
  O[12] = O[13] = O[14] = 0.0; O[15] = 1.0;
}
// [R^T | -R^T t] of rows 0..2 of T, the shim's inv_rigid order; row 3 = 0 0 0 1
__device__ void rigid_inv_rn(const double* T, double* I) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) I[4 * r + c] = T[4 * c + r];
  for (int r = 0; r < 3; r++) I[4 * r + 3] = -add(add(mul(T[r], T[3]), mul(T[4 + r], T[7])), mul(T[8 + r], T[11]));
  I[12] = I[13] = I[14] = 0.0; I[15] = 1.0;
}
// the shim's transform_to_pose7: [qx, qy, qz, qw, x, y, z] by Eigen's matrix-to-quaternion branches
__device__ void pose7_rn(const double* T, double* out) {
  double q[4];
  const double tr = add(add(T[0], T[5]), T[10]);
  if (tr > 0) {
    double t = __dsqrt_rn(add(tr, 1.0));
    q[3] = mul(0.5, t);
    t = __ddiv_rn(0.5, t);
    q[0] = mul(sub(T[9], T[6]), t); q[1] = mul(sub(T[2], T[8]), t); q[2] = mul(sub(T[4], T[1]), t);
  } else {
    int i = 0;
    if (T[5] > T[0]) i = 1;
    if (T[10] > T[5 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double t = __dsqrt_rn(add(sub(sub(T[5 * i], T[5 * j]), T[5 * k]), 1.0));
    q[i] = mul(0.5, t);
    t = __ddiv_rn(0.5, t);
    q[3] = mul(sub(T[4 * k + j], T[4 * j + k]), t);
    q[j] = mul(add(T[4 * j + i], T[4 * i + j]), t);
    q[k] = mul(add(T[4 * k + i], T[4 * i + k]), t);
  }
  for (int c = 0; c < 4; c++) out[c] = q[c];
  out[4] = T[3]; out[5] = T[7]; out[6] = T[11];
}

// one CTA per candidate: its matches scattered into the dense row idxA -> idxB, then (n_matches >= min_matches) compacted in
// ascending idxA into its RANSAC problem, at the offset of the used matches of the candidates before it
__global__ void __launch_bounds__(kGlueThreads) lmv_gather_kernel(LmvDev V, const DevPair* __restrict__ pairs) {
  const int c = blockIdx.x, nq = V.nq;
  __shared__ int off, use;
  if (threadIdx.x == 0) {
    int o = 0;
    for (int q = 0; q < c; q++) o += V.n_out[q] >= V.min_matches ? V.n_out[q] : 0;
    off = o;
    use = V.n_out[c] >= V.min_matches;
    if (c == 0) V.prob_ptr[0] = 0;
    V.prob_ptr[c + 1] = o + (use ? V.n_out[c] : 0);
  }
  int* row = V.row + (size_t)c * nq;
  for (int i = threadIdx.x; i < nq; i += kGlueThreads) row[i] = -1;
  __syncthreads();
  const int s0 = V.seg[c], m = V.n_out[c];
  for (int k = threadIdx.x; k < m; k += kGlueThreads) row[V.outA[s0 + k]] = V.outB[s0 + k];
  __syncthreads();
  if (!use) return;
  const double* lm = pairs[c].k2.lm_pos;
  const int o = off;
  scan_emit(nq, [&](int i) { return row[i] >= 0; }, [&](int i, int r) {
    const size_t j = (size_t)o + r, b = (size_t)row[i];
    for (int k = 0; k < 3; k++) { V.pts[3 * j + k] = lm[3 * b + k]; V.f[3 * j + k] = V.q_bear[3 * (size_t)i + k]; }
    V.sg[j] = V.q_sig[i]; V.srcA[j] = i;
  });
}

// one CTA per candidate: the gate, T12 / T21 (also into its DevPair) and the refinement's start pose, then the already-masks and
// stages 1 / 2.  A candidate that stops gets all-ones masks, so the search finds nothing for it.
__global__ void __launch_bounds__(kGlueThreads) lmv_pose_kernel(LmvDev V, DevPair* __restrict__ pairs) {
  const int c = blockIdx.x, nq = V.nq;
  DevPair& P = pairs[c];
  __shared__ int go;
  if (threadIdx.x == 0) {
    go = V.best_sample[c] >= 0 && V.best_count[c] >= V.min_inliers;
    double T12[16], T21[16], p7[7];
    for (int i = 0; i < 16; i++) T12[i] = T21[i] = 0.0;
    for (int i = 0; i < 7; i++) p7[i] = 0.0;
    if (go) {
      double M[16], A[16], B[16], Cw[16];
      for (int i = 0; i < 12; i++) M[i] = V.best_model[12 * (size_t)c + i];
      M[12] = M[13] = M[14] = 0.0; M[15] = 1.0;
      mul44_rn(M, V.q_Tsc, A);      // T_wc of the query camera
      rigid_inv_rn(A, B);           // T_c1_w
      rigid_inv_rn(P.k2.Tcw, Cw);   // T_w_c2
      mul44_rn(B, Cw, T12);
      rigid_inv_rn(T12, T21);
      pose7_rn(T12, p7);
    }
    for (int i = 0; i < 16; i++) { P.T12[i] = T12[i]; P.T21[i] = T21[i]; V.T12[16 * (size_t)c + i] = T12[i]; V.T21[16 * (size_t)c + i] = T21[i]; }
    for (int i = 0; i < 7; i++) V.pose_in[7 * (size_t)c + i] = p7[i];
  }
  __syncthreads();
  const bool g = go;
  const int n2 = P.k2.n;
  uint8_t* a1 = V.already1 + (size_t)c * nq;
  uint8_t* a2 = const_cast<uint8_t*>(P.already2);
  uint8_t* st = V.stage + (size_t)c * nq;
  const int* row = V.row + (size_t)c * nq;
  for (int i = threadIdx.x; i < nq; i += kGlueThreads) { a1[i] = !g; st[i] = row[i] >= 0; }
  for (int b = threadIdx.x; b < n2; b += kGlueThreads) a2[b] = !g;
  __syncthreads();
  if (!g) return;
  for (int j = V.prob_ptr[c] + threadIdx.x; j < V.prob_ptr[c + 1]; j += kGlueThreads)
    if (V.mask[j]) {
      const int i = V.srcA[j];
      a1[i] = 1; a2[row[i]] = 1; st[i] = 2;
    }
}

// one CTA per candidate: the LandmarkVector (RANSAC inliers, then the search's matches: stage 3) and, in ascending query
// keypoint, the residual pairs of its entries whose two landmarks are valid; n into the candidate's relpose record
__global__ void __launch_bounds__(kGlueThreads) lmv_residual_kernel(LmvDev V, const DevPair* __restrict__ pairs, cvb_relpose_dev* __restrict__ recs) {
  const int c = blockIdx.x, nq = V.nq;
  const DevPair& P = pairs[c];
  const size_t base = (size_t)c * nq;
  const int* row = V.row + base;
  const int* ms = P.match12;
  uint8_t* st = V.stage + base;
  int* m12 = V.match12 + base;
  for (int i = threadIdx.x; i < nq; i += kGlueThreads) {
    int b = -1;
    if (st[i] == 2) b = row[i];
    else if (ms[i] >= 0) { b = ms[i]; st[i] = 3; }
    m12[i] = b;
  }
  __syncthreads();
  const uint8_t* v2 = P.k2.lm_valid;
  const double* lm2 = P.k2.lm_pos;
  const float* kp2 = P.k2.kp;
  const float* oc2 = P.k2.octave;
  const double* TB = V.TcwB + 16 * (size_t)c;
  const int n = scan_emit(nq, [&](int i) { const int b = m12[i]; return b >= 0 && V.q_valid[i] && v2[b]; }, [&](int i, int r) {
    const size_t j = base + r, b = (size_t)m12[i];
    rt_apply(V.TcwA, V.q_pos + 3 * (size_t)i, V.pA + 3 * j);
    rt_apply(TB, lm2 + 3 * b, V.pB + 3 * j);
    V.kA[2 * j] = V.q_kp[2 * (size_t)i]; V.kA[2 * j + 1] = V.q_kp[2 * (size_t)i + 1];
    V.kB[2 * j] = kp2[2 * b]; V.kB[2 * j + 1] = kp2[2 * b + 1];
    V.sA[j] = mul((double)__fadd_rn(V.q_oct[i], 1.0f), 2.0);   // (keypoints_aors_[i][1] + 1) * 2.0: a float sum, then double
    V.sB[j] = mul((double)__fadd_rn(oc2[b], 1.0f), 2.0);
  });
  if (threadIdx.x == 0) { recs[c].n = n; V.n_corr[c] = n; }
}

// the shim's mul4 / inv_rigid (host, no fused multiply-add)
void host_mul4(const double* A, const double* B, double* O) {
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      double s = 0;
      for (int k = 0; k < 4; k++) s += A[4 * r + k] * B[4 * k + c];
      O[4 * r + c] = s;
    }
}
void host_inv_rigid(const double* T, double* I) {
  for (int i = 0; i < 16; i++) I[i] = i % 5 == 0 ? 1.0 : 0.0;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) I[4 * r + c] = T[4 * c + r];
  for (int r = 0; r < 3; r++) I[4 * r + 3] = -(I[4 * r] * T[3] + I[4 * r + 1] * T[7] + I[4 * r + 2] * T[11]);
}

cvb_relcam relcam(const cvb_landmark_kf* k) {
  cvb_relcam c{};
  for (int i = 0; i < 4; i++) { c.intr[i] = k->intr[i]; c.dist[i] = k->dist[i]; }
  c.cam = k->cam_model; c.dm = k->dist_model; c.xi = k->xi;
  return c;
}

int verify_landmark(cvb_ctx* ctx, const cvb_landmark_kf* q, const cvb_landmark_kf* cand, int C, const cvb_landmark_verify_params* prm,
                    const uint64_t* seed, cvb_landmark_verify_result* r) {
  const char* name = "verify_landmark_candidates_seeded";
  constexpr int kMaxIt = (INT32_MAX - kWave) / 11;   // the seeded RANSAC's limit: every sample number fits an int
  CVB_REQUIRE(ctx, q && prm && r && C >= 0, "%s: bad arguments", name);
  CVB_REQUIRE(ctx, prm->num_best >= 1 && prm->num_best <= 4, "%s: num_best must be in 1..4", name);
  CVB_REQUIRE(ctx, prm->thr > 0.f && prm->thr <= 257.f, "%s: distance threshold out of range", name);
  CVB_REQUIRE(ctx, prm->max_iterations >= 0 && prm->max_iterations <= kMaxIt, "%s: max_iterations outside [0, %d]", name, kMaxIt);
  CVB_REQUIRE(ctx, prm->search.num_octaves >= 1 && prm->search.scale_factor > 1.0 && prm->search.th > 0.0, "%s: bad search parameters", name);
  if (C == 0) return CVB_OK;
  CVB_REQUIRE(ctx, cand && seed, "%s: null candidates / seed", name);
  CVB_REQUIRE(ctx, r->n_matches && r->best_sample && r->best_model && r->best_count && r->iterations && r->consumed && r->T12 && r->T21 &&
                   r->n_found && r->n_corr && r->T12_out && r->n_inliers && r->solve_iterations, "%s: null result pointer", name);
  CVB_REQUIRE(ctx, kf_ok(&q->view), "%s: malformed keyframe view (query)", name);
  const int nq = q->view.n;
  CVB_REQUIRE(ctx, nq == 0 || (q->bearings && q->sigma_angle), "%s: null query bearings / sigma_angle", name);
  std::vector<int32_t> seg((size_t)C + 1, 0);
  for (int c = 0; c < C; c++) {
    CVB_REQUIRE(ctx, kf_ok(&cand[c].view), "%s: malformed keyframe view (cand[%d])", name, c);
    CVB_REQUIRE(ctx, (int64_t)seg[c] + cand[c].view.n <= INT32_MAX, "%s: candidate rows exceed the int32 range", name);
    seg[c + 1] = seg[c] + cand[c].view.n;
  }
  CVB_REQUIRE(ctx, (int64_t)C * nq <= INT32_MAX, "%s: n_cand x n_query exceeds the int32 range", name);
  for (int c = -1; c < C; c++) {   // OptimizeRelativePose's model checks (optimization_be.cpp:684-688, :705-707)
    const cvb_landmark_kf* k = c < 0 ? q : cand + c;
    if (k->cam_model < 0 || k->cam_model > 1) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown projection type.");
    if (k->dist_model < 0 || k->dist_model > 2) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown distortion type.");
  }
  const size_t NB = (size_t)seg[C], L = (size_t)C * nq;
  // the refinement's camera poses: TcwA = (T_ws1 T_sc1)^-1, TcwB = (T_ws2 T_sc1)^-1, as the shim forms them
  double TA[16], TcwA[16];
  host_mul4(q->T_ws, q->T_sc, TA);
  host_inv_rigid(TA, TcwA);
  std::vector<double> TcwB((size_t)C * 16);
  std::vector<double> cam((size_t)C * 12);
  for (int c = 0; c < C; c++) {
    double TB[16];
    host_mul4(cand[c].T_ws, q->T_sc, TB);
    host_inv_rigid(TB, &TcwB[16 * (size_t)c]);
    for (int k = 0; k < 3; k++) cam[12 * (size_t)c + k] = q->T_sc[4 * k + 3];   // one camera per problem: c, then Rc row-major
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) cam[12 * (size_t)c + 3 + 3 * a + b] = q->T_sc[4 * a + b];
  }
  std::vector<uint8_t> skipA(nq);
  for (int i = 0; i < nq; i++) skipA[i] = !q->view.lm_valid[i];
  // the device block; the DevPair records are completed here and by the device (T12 / T21), the relpose records by the device (n)
  cvb_block B(ctx, ctx->stream);
  DevKf d1{};
  bind_kf(B, d1, &q->view);
  std::vector<DevPair> hp((size_t)C);
  for (int c = 0; c < C; c++) bind_kf(B, hp[c].k2, &cand[c].view, false);   // descriptors: the DenseMatcher's rows d_B below
  LmvDev V{};
  const uint8_t *d_skA, *d_B, *d_skB;
  const uint64_t* d_seed;
  const double* d_cam;
  DevPair* d_pairs;
  cvb_relpose_dev* d_recs;
  int *d_oA, *d_oB, *d_mt1, *d_mt2, *d_ms, *d_nm, *d_bs, *d_bc, *d_it, *d_us, *d_nf;
  float* d_oD;
  double *d_bm, *d_ro;
  uint8_t *d_mask, *d_a2, *d_rem;
  B.in(V.q_bear, q->bearings, (size_t)nq * 3); B.in(V.q_sig, q->sigma_angle, nq);
  B.in(d_skA, skipA.data(), nq); B.in(d_B, nullptr, NB * 32); B.in(d_skB, nullptr, NB);
  B.in(V.seg, seg.data(), (size_t)C + 1); B.in(d_seed, seed, C); B.in(d_cam, cam.data(), cam.size()); B.in(V.TcwB, TcwB.data(), TcwB.size());
  B.in(d_pairs, nullptr, C); B.in(d_recs, nullptr, C);
  const std::vector<double> scale = scale_table(prm->search.scale_factor, prm->search.num_octaves);
  const double* d_scale;
  B.in(d_scale, scale.data(), scale.size());
  B.tmp(d_oA, NB); B.tmp(d_oB, NB); B.tmp(d_oD, NB); B.tmp(V.row, L); B.tmp(V.prob_ptr, (size_t)C + 1);
  B.tmp(V.pts, L * 3); B.tmp(V.f, L * 3); B.tmp(V.sg, L); B.tmp(V.srcA, L); B.tmp(d_mask, L);
  B.tmp(V.already1, L); B.tmp(d_a2, NB); B.tmp(d_mt1, L); B.tmp(d_mt2, NB); B.tmp(d_ms, L);
  B.tmp(V.pA, L * 3); B.tmp(V.pB, L * 3); B.tmp(V.kA, L * 2); B.tmp(V.kB, L * 2); B.tmp(V.sA, L); B.tmp(V.sB, L);
  B.tmp(V.pose_in, (size_t)C * 7);
  B.out(d_nm, r->n_matches, C); B.out(d_bs, r->best_sample, C); B.out(d_bm, r->best_model, (size_t)C * 12); B.out(d_bc, r->best_count, C);
  B.out(d_it, r->iterations, C); B.out(d_us, r->consumed, C); B.out(V.T12, r->T12, (size_t)C * 16); B.out(V.T21, r->T21, (size_t)C * 16);
  B.out(d_nf, r->n_found, C); B.out(V.n_corr, r->n_corr, C); B.out_host(d_ro, (size_t)C * CVB_RELPOSE_OUT);
  B.out(V.match12, r->match12, L); B.out(V.stage, r->stage, L); B.out_host(d_rem, L, r->removed != nullptr);   // the nullable outputs last
  if (const int rc = B.place()) return rc;
  uint8_t *hB = B.host(d_B), *hskB = B.host(d_skB);
  cvb_relpose_dev* hr = B.host(d_recs);
  for (int c = 0; c < C; c++) {
    const size_t n = (size_t)cand[c].view.n;
    if (n) memcpy(hB + 32 * (size_t)seg[c], cand[c].view.desc, n * 32);
    for (size_t b = 0; b < n; b++) hskB[seg[c] + b] = !cand[c].view.lm_valid[b];
    DevPair& P = hp[c];
    P.k2.desc = d_B + 32 * (size_t)seg[c];   // the search reads its rows of d_B
    P.already1 = V.already1 + (size_t)c * nq; P.already2 = d_a2 + seg[c];
    P.match1 = d_mt1 + (size_t)c * nq; P.match2 = d_mt2 + seg[c]; P.match12 = d_ms + (size_t)c * nq; P.n_found = d_nf + c;
    cvb_relpose_dev& R = hr[c];
    memset(&R, 0, sizeof(R));
    const size_t b = (size_t)c * nq;
    R.pA = V.pA + 3 * b; R.pB = V.pB + 3 * b; R.kpA = V.kA + 2 * b; R.kpB = V.kB + 2 * b; R.sA = V.sA + b; R.sB = V.sB + b;
    R.camA = relcam(q); R.camB = relcam(cand + c);
    R.pose_in = V.pose_in + 7 * (size_t)c; R.removed = d_rem + b; R.out = d_ro + CVB_RELPOSE_OUT * (size_t)c;
  }
  memcpy(B.host(d_pairs), hp.data(), hp.size() * sizeof(DevPair));
  if (const int rc = B.upload()) return rc;
  cudaStream_t st = ctx->stream;
  V.nq = nq; V.min_matches = prm->min_matches; V.min_inliers = prm->min_ransac_inliers;
  V.outA = d_oA; V.outB = d_oB; V.n_out = d_nm;
  V.q_valid = d1.lm_valid; V.q_pos = d1.lm_pos; V.q_kp = d1.kp; V.q_oct = d1.octave;
  memcpy(V.q_Tsc, q->T_sc, sizeof(V.q_Tsc)); memcpy(V.TcwA, TcwA, sizeof(V.TcwA));
  V.best_sample = d_bs; V.best_model = d_bm; V.best_count = d_bc; V.mask = d_mask;
  // 1. DenseMatcher
  if (NB > 0) {
    if (const int rc = cvb_landmark_match_batch_dev(ctx, d1.desc, d_skA, nq, d_B, d_skB, V.seg, seg.data(), C, prm->thr, prm->num_best, d_oA, d_oB,
                                                    d_oD, d_nm, nullptr))
      return rc;
  } else {
    CVB_CUDA(ctx, cudaMemsetAsync(d_nm, 0, (size_t)C * 4, st));
  }
  // 2. the RANSAC problems and their RANSACs
  lmv_gather_kernel<<<C, kGlueThreads, 0, st>>>(V, d_pairs);
  CVB_CHECK_LAUNCH(ctx);
  if (const int rc = cvb_abs_ransac_seeded_dev(ctx, C, V.prob_ptr, V.pts, V.f, V.sg, d_cam, d_seed, prm->threshold, prm->max_iterations,
                                               prm->probability, d_bs, d_bm, d_bc, d_it, d_us, d_mask))
    return rc;
  // 3. gate, T12 / T21, already-masks
  lmv_pose_kernel<<<C, kGlueThreads, 0, st>>>(V, d_pairs);
  CVB_CHECK_LAUNCH(ctx);
  // 4. SearchBySE3
  search_se3_kernel<<<C, 256, 0, st>>>(d1, d_pairs, prm->search.th, prm->search.desc_th_low, d_scale, prm->search.num_octaves);
  CVB_CHECK_LAUNCH(ctx);
  // 5. the residual pairs and the refinement
  lmv_residual_kernel<<<C, kGlueThreads, 0, st>>>(V, d_pairs, d_recs);
  CVB_CHECK_LAUNCH(ctx);
  if (const int rc = cvb_relpose_batch_dev(ctx, d_recs, C, prm->th_outlier_align)) return rc;
  if (const int rc = B.download()) return rc;
  const double* ro = B.host(d_ro);
  for (int c = 0; c < C; c++) {
    const double* o = ro + CVB_RELPOSE_OUT * (size_t)c;
    for (int k = 0; k < 7; k++) r->T12_out[7 * (size_t)c + k] = o[k];
    r->n_inliers[c] = (int32_t)o[7];
    r->solve_iterations[2 * (size_t)c] = (int32_t)o[8]; r->solve_iterations[2 * (size_t)c + 1] = (int32_t)o[9];
  }
  if (r->removed) {   // defined for r < n_corr; the rest of a candidate's row is 0
    memset(r->removed, 0, L);
    for (int c = 0; c < C; c++) memcpy(r->removed + (size_t)c * nq, B.host(d_rem) + (size_t)c * nq, (size_t)r->n_corr[c]);
  }
  return CVB_OK;
}

}  // namespace

extern "C" int cvb_verify_landmark_candidates_seeded_batch(cvb_ctx* ctx, const cvb_landmark_kf* query, const cvb_landmark_kf* cand, int n_cand,
                                                           const cvb_landmark_verify_params* prm, const uint64_t* seed,
                                                           cvb_landmark_verify_result* r) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return verify_landmark(ctx, query, cand, n_cand, prm, seed, r);
}
