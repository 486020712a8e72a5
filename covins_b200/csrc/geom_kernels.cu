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

// LandmarkBase::PredictScale: ceil(log(ratio) / log(scale_factor)) clamped to [0, num_octaves - 1] = the smallest n >= 0
// with scale_factor^n >= ratio (n capped): evaluated with exact repeated multiplication instead of two libm calls
__device__ __forceinline__ int predict_scale(double maxdist, double dist3d, double sf, int num_octaves) {
  const double ratio = __ddiv_rn(maxdist, (double)(float)dist3d);   // `const float& currentDist`
  int n = 0;
  double p = 1.0;
  while (p < ratio && n < num_octaves - 1) { p = mul(p, sf); n++; }
  return n;
}

// best keypoint of `dst` for landmark i of `src` (float_best: direction 1→2 keeps the best distance as float — the same
// integers — and both directions take the FIRST strict minimum in the grid's candidate order)
__device__ int search_one(const DevKf& src, int i, const double* Tcw_src, const double* Tab, const double* Kdst, const DevKf& dst,
                          const double* img, double th, double sf, int num_octaves, int* best_dist) {
  double pw[3] = {src.lm_pos[3 * (size_t)i], src.lm_pos[3 * (size_t)i + 1], src.lm_pos[3 * (size_t)i + 2]};
  double pc_src[3], pc[3];
  rt_apply(Tcw_src, pw, pc_src);
  rt_apply(Tab, pc_src, pc);
  if (pc[2] < 0.0) return -1;
  const double p0 = dot3(Kdst[0], Kdst[1], Kdst[2], pc), p1 = dot3(Kdst[3], Kdst[4], Kdst[5], pc), p2 = dot3(Kdst[6], Kdst[7], Kdst[8], pc);
  const double u = __ddiv_rn(p0, p2), v = __ddiv_rn(p1, p2);
  if (!in_image(img, u, v)) return -1;
  const double dist3d = __dsqrt_rn(add(add(mul(pc[0], pc[0]), mul(pc[1], pc[1])), mul(pc[2], pc[2])));
  const int level = predict_scale(src.lm_maxdist[i], dist3d, sf, num_octaves);
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

__global__ void __launch_bounds__(256) search_se3_kernel(DevKf k1, const DevPair* __restrict__ pairs, double th, int th_low, double sf,
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
      const int b = search_one(k1, i, k1.Tcw, P.T21, k2.K, k2, k2.img, th, sf, num_octaves, &bd);
      if (b >= 0 && bd <= th_low) m = b;              // bestDist <= desc_matching_th_low_ (:403)
    }
    P.match1[i] = m;
  }
  for (int i = threadIdx.x; i < n2; i += blockDim.x) {   // KF2 → KF1 (:409-482); IsInImage of pKF2 (:433)
    int m = -1;
    if (k2.lm_valid[i] && !P.already2[i]) {
      int bd;
      const int b = search_one(k2, i, k2.Tcw, P.T12, k1.K, k1, k2.img, th, sf, num_octaves, &bd);
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

__global__ void __launch_bounds__(256, 1) search_proj_kernel(DevKf kf, ProjDev P, double th, int th_low, double sf, int num_octaves) {
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
      const bam::CamModel cm{P.cam, P.dm, P.xi};
      double x, y, xd, yd;
      if (!bam::cam_normalise(cm, bam::V3{pc[0], pc[1], pc[2]}, &x, &y, nullptr, false)) break;
      bam::cam_distort(cm, P.dist, x, y, &xd, &yd, nullptr, false);
      const double u = P.intr[0] * xd + P.intr[2], v = P.intr[1] * yd + P.intr[3];
      if (!in_image(kf.img, u, v)) break;
      const double PO[3] = {sub(pw[0], Ow[0]), sub(pw[1], Ow[1]), sub(pw[2], Ow[2])};
      const double d3 = __dsqrt_rn(add(add(mul(PO[0], PO[0]), mul(PO[1], PO[1])), mul(PO[2], PO[2])));
      if (d3 < P.min_dist[i] || d3 > P.max_dist[i]) break;
      if (add(add(mul(PO[0], P.normal[3 * (size_t)i]), mul(PO[1], P.normal[3 * (size_t)i + 1])), mul(PO[2], P.normal[3 * (size_t)i + 2])) < mul(0.5, d3)) break;
      const int level = predict_scale(P.max_distance[i], d3, sf, num_octaves);
      double radius = th;
      for (int l = 0; l < level; l++) radius = mul(radius, sf);   // th * pow(scale_factor, level) for integer level
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

size_t stage_kf(Stager& S, const cvb_kf_view* v, size_t off[9]) {
  const size_t n = (size_t)v->n;
  off[0] = S.put(v->kp, n * 8); off[1] = S.put(v->octave, n * 4); off[2] = S.put(v->desc, n * 32); off[3] = S.put(v->lm_valid, n);
  off[4] = S.put(v->lm_pos, n * 24); off[5] = S.put(v->lm_maxdist, n * 8); off[6] = S.put(v->lm_desc, n * 32);
  off[7] = S.put(v->grid_ptr, (GRID_COLS * GRID_ROWS + 1) * 4);
  off[8] = S.put(v->grid_idx, (size_t)v->grid_ptr[GRID_COLS * GRID_ROWS] * 4);
  return off[8];
}
void fill_dev(DevKf& d, const cvb_kf_view* v, const unsigned char* base, const size_t off[9]) {
  d.n = v->n;
  d.kp = (const float*)(base + off[0]); d.octave = (const float*)(base + off[1]); d.desc = base + off[2]; d.lm_valid = base + off[3];
  d.lm_pos = (const double*)(base + off[4]); d.lm_maxdist = (const double*)(base + off[5]); d.lm_desc = base + off[6];
  d.grid_ptr = (const int*)(base + off[7]); d.grid_idx = (const int*)(base + off[8]);
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
  // ---- stage inputs ----
  Stager S;
  size_t off1[9];
  stage_kf(S, kf1, off1);
  std::vector<size_t> off2((size_t)n_pairs * 9);
  for (int p = 0; p < n_pairs; p++) stage_kf(S, kf2 + p, &off2[(size_t)p * 9]);
  const size_t o_a1 = S.put(already1, (size_t)n_pairs * n1), o_a2 = S.put(already2, n2_total);
  const size_t o_pairs = S.reserve((size_t)n_pairs * sizeof(DevPair));
  const size_t in_bytes = S.h.size();
  // outputs live behind the inputs in the same device block
  const size_t o_m1 = S.reserve((size_t)n_pairs * n1 * 4), o_m2 = S.reserve(n2_total * 4), o_m12 = S.reserve((size_t)n_pairs * n1 * 4),
               o_nf = S.reserve((size_t)n_pairs * 4);
  const size_t total = S.h.size();
  unsigned char* dbase = (unsigned char*)cvb_ws(ctx, WS_GS0, total);
  unsigned char* hpin = (unsigned char*)cvb_pinned(ctx, total);
  if (!dbase || !hpin) return CVB_ERR_CUDA;
  DevKf d1;
  fill_dev(d1, kf1, dbase, off1);
  DevPair* hp = reinterpret_cast<DevPair*>(S.h.data() + o_pairs);
  size_t a2 = 0;
  for (int p = 0; p < n_pairs; p++) {
    DevPair& P = hp[p];
    fill_dev(P.k2, kf2 + p, dbase, &off2[(size_t)p * 9]);
    memcpy(P.T12, T12 + 16 * (size_t)p, sizeof(P.T12)); memcpy(P.T21, T21 + 16 * (size_t)p, sizeof(P.T21));
    P.already1 = dbase + o_a1 + (size_t)p * n1; P.already2 = dbase + o_a2 + a2;
    P.match1 = (int*)(dbase + o_m1) + (size_t)p * n1; P.match2 = (int*)(dbase + o_m2) + a2;
    P.match12 = (int*)(dbase + o_m12) + (size_t)p * n1; P.n_found = (int*)(dbase + o_nf) + p;
    a2 += (size_t)kf2[p].n;
  }
  memcpy(hpin, S.h.data(), in_bytes);
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemcpyAsync(dbase, hpin, in_bytes, cudaMemcpyHostToDevice, st));
  search_se3_kernel<<<n_pairs, 256, 0, st>>>(d1, reinterpret_cast<const DevPair*>(dbase + o_pairs), prm->th, prm->desc_th_low,
                                             prm->scale_factor, prm->num_octaves);
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaMemcpyAsync(hpin + o_m1, dbase + o_m1, total - o_m1, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(match12, hpin + o_m12, (size_t)n_pairs * n1 * 4);
  memcpy(n_found, hpin + o_nf, (size_t)n_pairs * 4);
  if (match1) memcpy(match1, hpin + o_m1, (size_t)n_pairs * n1 * 4);
  if (match2) memcpy(match2, hpin + o_m2, n2_total * 4);
  return CVB_OK;
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
  Stager S;
  const size_t o_model = S.put(model, (size_t)n_hyp * 96), o_a = S.put(a, (size_t)n * 24), o_b = S.put(b, (size_t)n * 24),
               o_s1 = S.put(s1, (size_t)n * 8);
  size_t o_s2 = 0, o_cam = 0;
  if (relative) o_s2 = S.put(s2, (size_t)n * 8);
  else {   // one camera: offset (3) directly followed by the rotation (9, row-major)
    double cam[12];
    memcpy(cam, cam_off, 24); memcpy(cam + 3, cam_rot, 72);
    o_cam = S.put(cam, sizeof(cam));
  }
  const size_t in_bytes = S.h.size();
  const size_t o_cnt = S.reserve((size_t)n_hyp * 4), o_sc = scores ? S.reserve(hn * 8) : 0, o_in = inlier ? S.reserve(hn) : 0;
  const size_t total = S.h.size();
  unsigned char* d = (unsigned char*)cvb_ws(ctx, WS_GS1, total);
  unsigned char* hpin = (unsigned char*)cvb_pinned(ctx, total);
  if (!d || !hpin) return CVB_ERR_CUDA;
  memcpy(hpin, S.h.data(), in_bytes);
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemcpyAsync(d, hpin, in_bytes, cudaMemcpyHostToDevice, st));
  CVB_CUDA(ctx, cudaMemsetAsync(d + o_cnt, 0, (size_t)n_hyp * 4, st));
  const dim3 grid((unsigned)((n + 255) / 256), (unsigned)n_hyp);
  if (relative)
    score_rel_kernel<<<grid, 256, 0, st>>>((const double*)(d + o_model), (const double*)(d + o_a), (const double*)(d + o_b), (const double*)(d + o_s1),
                                           (const double*)(d + o_s2), n, threshold, scores ? (double*)(d + o_sc) : nullptr,
                                           inlier ? d + o_in : nullptr, (int*)(d + o_cnt));
  else
    score_abs_kernel<<<grid, 256, 0, st>>>((const double*)(d + o_model), (const double*)(d + o_a), (const double*)(d + o_b), (const double*)(d + o_s1), n,
                                           (const double*)(d + o_cam), threshold, scores ? (double*)(d + o_sc) : nullptr,
                                           inlier ? d + o_in : nullptr, (int*)(d + o_cnt));
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaMemcpyAsync(hpin + o_cnt, d + o_cnt, total - o_cnt, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(n_inliers, hpin + o_cnt, (size_t)n_hyp * 4);
  if (scores) memcpy(scores, hpin + o_sc, hn * 8);
  if (inlier) memcpy(inlier, hpin + o_in, hn);
  return CVB_OK;
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
  if (cam_model < 0 || cam_model > 1) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown projection type.");
  if (dist_model < 0 || dist_model > 2) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "Unknown distortion type.");
  const int n = kf->n, m = lms->m;
  *n_matches = 0;
  if (m == 0) return CVB_OK;
  CVB_REQUIRE(ctx, lms->valid && lms->pos && lms->normal && lms->min_dist && lms->max_dist && lms->max_distance && lms->desc && lms->feat_idx &&
              action && best_idx, "search_by_projection: null landmark arrays");
  for (int i = 0; i < m; i++) CVB_REQUIRE(ctx, lms->feat_idx[i] >= -1 && lms->feat_idx[i] < n, "search_by_projection: feat_idx out of range");
  for (int i = 0; i < n; i++) CVB_REQUIRE(ctx, kf_lm_cand[i] >= -1 && kf_lm_cand[i] < m, "search_by_projection: kf_lm_cand out of range");
  Stager S;
  const size_t ng = (size_t)kf->grid_ptr[GRID_COLS * GRID_ROWS];
  const size_t o_kp = S.put(kf->kp, (size_t)n * 8), o_oc = S.put(kf->octave, (size_t)n * 4), o_de = S.put(kf->desc, (size_t)n * 32),
               o_gp = S.put(kf->grid_ptr, (GRID_COLS * GRID_ROWS + 1) * 4), o_gi = S.put(kf->grid_idx, ng * 4);
  const size_t o_hl = S.put(kf->lm_valid, (size_t)n), o_lc = S.put(kf_lm_cand, (size_t)n * 4), o_ma = S.put(matched, (size_t)n);
  const size_t o_va = S.put(lms->valid, (size_t)m), o_po = S.put(lms->pos, (size_t)m * 24), o_no = S.put(lms->normal, (size_t)m * 24),
               o_mi = S.put(lms->min_dist, (size_t)m * 8), o_mx = S.put(lms->max_dist, (size_t)m * 8), o_md = S.put(lms->max_distance, (size_t)m * 8),
               o_ld = S.put(lms->desc, (size_t)m * 32), o_fi = S.put(lms->feat_idx, (size_t)m * 4), o_fe = S.put(lms->feat_idx, (size_t)m * 4);
  const size_t in_bytes = S.h.size();
  const size_t o_ci = S.reserve((size_t)m * kProjCap * 4), o_cd = S.reserve((size_t)m * kProjCap * 4), o_cn = S.reserve((size_t)m * 4);
  const size_t o_out = S.reserve(0), o_ac = S.reserve((size_t)m * 4), o_bi = S.reserve((size_t)m * 4), o_nm = S.reserve(8);
  const size_t total = S.h.size();
  unsigned char* d = (unsigned char*)cvb_ws(ctx, WS_GS4, total);
  unsigned char* hpin = (unsigned char*)cvb_pinned(ctx, total);
  if (!d || !hpin) return CVB_ERR_CUDA;
  DevKf K{};
  K.n = n; K.kp = (const float*)(d + o_kp); K.octave = (const float*)(d + o_oc); K.desc = d + o_de; K.grid_ptr = (const int*)(d + o_gp);
  K.grid_idx = (const int*)(d + o_gi); K.grid_w_inv = kf->grid_w_inv; K.grid_h_inv = kf->grid_h_inv;
  memcpy(K.img, kf->img, sizeof(K.img));
  ProjDev P{};
  P.m = m; P.valid = d + o_va; P.pos = (const double*)(d + o_po); P.normal = (const double*)(d + o_no); P.min_dist = (const double*)(d + o_mi);
  P.max_dist = (const double*)(d + o_mx); P.max_distance = (const double*)(d + o_md); P.desc = d + o_ld; P.feat_idx = (const int*)(d + o_fi);
  memcpy(P.Tcw, Tcw, sizeof(P.Tcw)); memcpy(P.intr, intr, 32); memcpy(P.dist, dist, 32);
  P.xi = xi; P.cam = cam_model; P.dm = dist_model;
  P.cand_idx = (int*)(d + o_ci); P.cand_dist = (int*)(d + o_cd); P.cand_n = (int*)(d + o_cn);
  P.matched = d + o_ma; P.has_lm = d + o_hl; P.lm_cand = (int*)(d + o_lc); P.feat = (int*)(d + o_fe);
  P.action = (int*)(d + o_ac); P.best_idx = (int*)(d + o_bi); P.n_matches = (int*)(d + o_nm); P.overflow = (int*)(d + o_nm) + 1;
  memcpy(hpin, S.h.data(), in_bytes);
  cudaStream_t st = ctx->stream;
  CVB_CUDA(ctx, cudaMemcpyAsync(d, hpin, in_bytes, cudaMemcpyHostToDevice, st));
  CVB_CUDA(ctx, cudaMemsetAsync(d + o_nm, 0, 8, st));
  search_proj_kernel<<<1, 256, 0, st>>>(K, P, prm->th, prm->desc_th_low, prm->scale_factor, prm->num_octaves);
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaMemcpyAsync(hpin + o_out, d + o_out, total - o_out, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  const int* tail = (const int*)(hpin + o_nm);
  if (tail[1]) return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "search_by_projection: more than %d keypoints in a search radius", kProjCap);
  memcpy(action, hpin + o_ac, (size_t)m * 4); memcpy(best_idx, hpin + o_bi, (size_t)m * 4);
  *n_matches = tail[0];
  return CVB_OK;
}

}  // extern "C"
