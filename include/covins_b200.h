/*
 * covins_b200.h — C-ABI of libcovins_b200.so: the H100-native (sm_90a) implementation of the COVINS
 * server hot path (place-recognition descriptor matching + PGO / global BA).
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference has no FFI layer — its seams are C++
 * symbols — so each entry point below names the reference call it replaces (paths relative to
 * covins_backend/ in VIS4ROB-lab/covins).  The C++ host shim that keeps the reference's own signatures
 * (Optimization::*, the ComputeSE3 matching blocks) and calls these functions is
 * covins_b200/csrc/host/covins_b200_shim.hpp; the binding a maintainer adds is shown in INTEGRATION.md.
 *
 * Conventions
 *   - plain pointers + sizes, no C++/torch types; every function returns a cvb_status (0 = OK);
 *     cvb_last_error(ctx) gives the message of the last failure on that ctx.
 *   - functions without suffix take HOST buffers and include all H2D/D2H copies (synchronous on
 *     return); `_dev` variants take DEVICE pointers and enqueue on `stream` (a cudaStream_t passed as
 *     void*; NULL = the ctx's own stream) without synchronising.
 *   - a ctx owns one device, one stream and a pinned staging buffer; each call takes its device memory as one block from
 *     the device's stream-ordered pool on the stream its work runs on.  Every entry point makes the ctx's device
 *     current for the calling thread and holds the ctx's lock for its duration: a ctx may be shared between host threads
 *     (calls are serialised per ctx); for concurrency use one ctx per host thread (the reference runs one
 *     place-recognition thread per agent, src/covins_backend/handler_be.cpp:52-56, and at most one optimisation per map).
 *   - no CPU fallback exists: without a CUDA device every compute call fails with CVB_ERR_CUDA.
 */
#ifndef COVINS_B200_H_
#define COVINS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CVB_API __attribute__((visibility("default")))

typedef enum cvb_status {
  CVB_OK = 0,
  CVB_ERR_INVALID = 1,     /* bad argument */
  CVB_ERR_CUDA = 2,        /* CUDA runtime error / no device */
  CVB_ERR_UNSUPPORTED = 3, /* valid request outside the implemented envelope */
  CVB_ERR_NUMERIC = 4      /* factorisation failed / non-finite state */
} cvb_status;

typedef struct cvb_ctx cvb_ctx;
typedef struct cvb_group cvb_group;   /* in-process rank group of the bundle adjustment (cvb_group_create) */

CVB_API int cvb_version(void);
CVB_API int cvb_ctx_create(int device, cvb_ctx** out);
CVB_API int cvb_ctx_destroy(cvb_ctx* ctx);
CVB_API const char* cvb_last_error(const cvb_ctx* ctx);
CVB_API int cvb_ctx_sync(cvb_ctx* ctx);
/* number of kernels this ctx has launched so far (bench.py's gpu_launches) */
CVB_API int64_t cvb_launch_count(const cvb_ctx* ctx);

/* ------------------------------------------------------------------------------------------------
 * Matching half (SURVEY.md §8a M1-M6)
 * ---------------------------------------------------------------------------------------------- */

/*
 * Replaces cv::BFMatcher(cv::NORM_HAMMING)::knnMatch(query, train, out, k)
 *   src/covins_backend/placerec_gen_be.cpp:82-100, src/covins_backend/RelNonCentralPosSolver.cpp:303-324.
 * The train set is the concatenation of n_seg candidate keyframes (seg_ptr[n_seg+1] row offsets,
 * seg_ptr[0] = 0); one independent knnMatch per (segment, query), exactly the per-candidate loop of
 * placerec_gen_be.cpp:72-125 — n_seg = 1 is the plain call.  Descriptors are 32-byte ORB rows
 * (desc_length 32, config/config_backend.yaml:28-29).
 * Output idx/dist are [n_seg][nq][k] (k in 1..4): trainIdx LOCAL to the segment, Hamming distance as
 * int32 (DMatch::distance is this value as float).  Order and ties as OpenCV: ascending distance,
 * equal distances by ascending trainIdx.  Slots beyond the segment length: idx -1, dist INT32_MAX.
 */
CVB_API int cvb_knn_hamming_batch(cvb_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t,
                                  const int32_t* seg_ptr, int n_seg, int k, int32_t* idx, int32_t* dist);
CVB_API int cvb_knn_hamming_batch_dev(cvb_ctx* ctx, const uint8_t* d_q, int nq, const uint8_t* d_t,
                                      const int32_t* d_seg_ptr, const int32_t* h_seg_ptr, int n_seg, int k,
                                      int32_t* d_idx, int32_t* d_dist, void* stream);

/*
 * knnMatch(k=2) fused with the distance + Lowe-ratio filter of placerec_gen_be.cpp:102-114
 * (== RelNonCentralPosSolver.cpp:326-337): keep m iff m.distance <= thr && m.distance < ratio*n.distance,
 * float arithmetic as in the reference (config_backend.hpp:119-120 reads both as float).
 * match_train [n_seg][nq]: accepted trainIdx (segment-local) or -1; match_dist [n_seg][nq]: its
 * distance (float) or FLT_MAX; n_matches [n_seg]: img_matches.size(), the number compared with
 * matches_thres at placerec_gen_be.cpp:116-124.  The reference's Matches vector is the accepted rows
 * in query order.
 */
CVB_API int cvb_match_hamming_batch(cvb_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t,
                                    const int32_t* seg_ptr, int n_seg, float thr, float ratio,
                                    int32_t* match_train, float* match_dist, int32_t* n_matches);
CVB_API int cvb_match_hamming_batch_dev(cvb_ctx* ctx, const uint8_t* d_q, int nq, const uint8_t* d_t,
                                        const int32_t* d_seg_ptr, const int32_t* h_seg_ptr, int n_seg,
                                        float thr, float ratio, int32_t* d_match_train, float* d_match_dist,
                                        int32_t* d_n_matches, void* stream);

/*
 * Resident descriptor database: the ORB or SIFT descriptors of the merged map's keyframes stay in HBM.
 * Replaces, for the place-recognition loop of placerec_gen_be.cpp:60-135 (one knnMatch + filter per
 * candidate keyframe, :82-114), the per-call upload of the train descriptors: a keyframe's descriptor
 * matrix is immutable once the keyframe exists (keyframe_be.cpp:106-137), so it is appended once
 * (cvb_db_append, one segment per keyframe, in the caller's keyframe order) and a request moves only
 * the query keyframe up (nq*32 B) and the ACCEPTED matches down.
 *
 * cvb_db_match_hamming: same semantics as cvb_match_hamming_batch against every keyframe of the
 * database.  n_matches [n_kf] (may be NULL) = img_matches.size() per keyframe (:116-124); the accepted
 * matches are returned compacted, ordered by (keyframe, queryIdx) — per keyframe exactly the
 * reference's img_matches vector: m_kf / m_query / m_train (keyframe-local trainIdx) / m_dist.
 * *n_total = number of accepted matches over all keyframes; at most `cap` are written (call again with
 * a larger cap if *n_total > cap).
 *
 * cvb_db_create: desc_bytes 32 = ORB rows (cvb_db_append, cvb_db_match_hamming[_dev]); 128 = SIFT rows (cvb_db_append_sift,
 * cvb_db_match_l2[_dev]); any other value → CVB_ERR_UNSUPPORTED.  A call of the other row kind → CVB_ERR_INVALID with a
 * message.  cvb_db_reserve, cvb_db_remove, cvb_db_remove_batch and cvb_db_size serve both kinds.
 */
typedef struct cvb_db cvb_db;
CVB_API int cvb_db_create(cvb_ctx* ctx, int desc_bytes, cvb_db** out);
CVB_API int cvb_db_destroy(cvb_ctx* ctx, cvb_db* db);
CVB_API int cvb_db_reserve(cvb_ctx* ctx, cvb_db* db, int64_t rows);
CVB_API int cvb_db_append(cvb_ctx* ctx, cvb_db* db, const uint8_t* rows, const int32_t* rows_per_kf, int n_kf);
CVB_API int cvb_db_size(const cvb_db* db, int32_t* n_kf, int64_t* n_rows);
/* A keyframe leaves the map (Keyframe::SetInvalid / culling, keyframe_be.cpp:413-440; Map::EraseKeyframe): its segment is
 * cut out of the resident descriptor array; the database indices of the keyframes appended after it drop by one (the
 * order of the remaining keyframes is kept, like erasing from a vector).  It is cvb_db_remove_batch of one index. */
CVB_API int cvb_db_remove(cvb_ctx* ctx, cvb_db* db, int kf_index);
/*
 * A batch of keyframes leaves the map in one call (the keyframes Map::Clean culls, keyframe_be.cpp:413-440, or erases).
 * kf_index [n]: database indices as they are BEFORE the call, in any order.  The result is that of calling cvb_db_remove
 * for each index from the highest to the lowest: every later cvb_db_size, request (cvb_db_match_hamming / _l2 and their
 * _dev forms), append, remove and merge is bit-identical to what it would be after that loop.  A surviving keyframe's new
 * index is its old index minus the number of removed indices below it.  ORB and SIFT databases alike.
 *   n == 0 does nothing and launches nothing.
 *   Refusals, before any device work and with the database unchanged, each CVB_ERR_INVALID with a message naming the
 *   index: n < 0, kf_index == NULL with n > 0, an index out of range, an index given twice.
 *   Device work: only the suffix from the first removed keyframe moves.  Its kept keyframes' rows, and then their operand
 *   tiles, are gathered into a scratch block of the stream-ordered pool by one launch per array and copied back by one
 *   device-to-device copy per array (so a single removal moves exactly the bytes it always did, and the extra memory is at
 *   most the moved suffix of one array).  Nothing is launched for an array when no kept byte follows the first removed
 *   keyframe.  The host segment tables are rebuilt once; at most one host synchronisation, however many keyframes go.
 */
CVB_API int cvb_db_remove_batch(cvb_ctx* ctx, cvb_db* db, const int32_t* kf_index, int n);
CVB_API int cvb_db_match_hamming(cvb_ctx* ctx, cvb_db* db, const uint8_t* q, int nq, float thr, float ratio,
                                 int32_t* n_matches, int32_t* m_kf, int32_t* m_query, int32_t* m_train,
                                 float* m_dist, int cap, int32_t* n_total);
/* device variant of the same request (query already in HBM, dense device outputs as cvb_match_hamming_batch_dev:
 * d_match_train/d_match_dist [n_kf][nq], d_n_matches [n_kf]; no copies, asynchronous on `stream`).  The database's
 * keyframes are matched from their resident tensor-core operand tiles (written once by cvb_db_append). */
CVB_API int cvb_db_match_hamming_dev(cvb_ctx* ctx, cvb_db* db, const uint8_t* d_q, int nq, float thr, float ratio,
                                     int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches, void* stream);
/*
 * The SIFT form of the database (desc_bytes == 128), for the SIFT branch of the same loop (placerec_gen_be.cpp:86-87,99-114).
 * cvb_db_append_sift: rows = the new keyframes' descriptors_add_ (CV_32F, rows x 128 each, concatenated).  The values are
 * checked and quantised to u8 on the host while staged, the rule of cvb_verify_noncentral_relative_pose_sift_seeded_batch: a
 * value that is not an integer in [0,255] (NaN and +-inf included) → CVB_ERR_UNSUPPORTED before any device work, the database
 * unchanged.  The rows are kept as exact u8 (as cvb_knn_l2_u8_batch_dev takes them) next to their tensor-core operand tiles
 * (128-row tiles of the u8 rows and their |t|^2, written once here).
 * cvb_db_match_l2: per keyframe the semantics of cvb_match_l2_batch with the caller's thresholds (SIFT config:
 * img_match_thres about 500, ratio 0.8): exact brute-force 2-NN, dist = sqrtf(d2) in fp32, OpenCV's tie rule on the float
 * distance (L2Metric::less: the lower trainIdx wins among equal floats), accepted iff d0 <= thr && d0 < ratio*d1.  q = the
 * query keyframe's CV_32F rows [nq][128], checked like the appended rows (before any device work).  The outputs are exactly
 * those of cvb_db_match_hamming: n_matches per keyframe, matches compacted by (keyframe, queryIdx), at most `cap`, *n_total.
 * cvb_db_match_l2_dev: the device request, d_q = u8 [nq][128] in HBM (16-byte aligned), dense device outputs as
 * cvb_db_match_hamming_dev.
 */
CVB_API int cvb_db_append_sift(cvb_ctx* ctx, cvb_db* db, const float* rows, const int32_t* rows_per_kf, int n_kf);
CVB_API int cvb_db_match_l2(cvb_ctx* ctx, cvb_db* db, const float* q, int nq, float thr, float ratio,
                            int32_t* n_matches, int32_t* m_kf, int32_t* m_query, int32_t* m_train,
                            float* m_dist, int cap, int32_t* n_total);
CVB_API int cvb_db_match_l2_dev(cvb_ctx* ctx, cvb_db* db, const uint8_t* d_q, int nq, float thr, float ratio,
                                int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches, void* stream);
/*
 * Two agents' maps are merged (MapManager::PerformMerge, map_be.cpp:192-244): the fused map's keyframes join the target's
 * database without leaving HBM.  src's keyframes are appended after dst's, in src's order; src is left unchanged.  Every
 * later request (cvb_db_match_hamming / _l2 and their _dev forms), cvb_db_size, cvb_db_remove and append on dst is
 * bit-identical to that of a database that received dst's keyframes and then src's from the host.  A tile image depends
 * only on the rows of its keyframe (the key's column is the row within the tile), so src's rows and operand tiles are
 * copied device to device on ctx's stream and the segment tables rebased: no descriptor byte crosses PCIe and nothing is
 * launched.  dst grows through the same reservation as an append.
 * Refusals, before any device work and with dst unchanged: dst == src or databases of different row kinds ->
 * CVB_ERR_INVALID; a database created on another ctx (so possibly another device) -> CVB_ERR_UNSUPPORTED; more than 2^31
 * rows together -> CVB_ERR_INVALID.
 */
CVB_API int cvb_db_merge(cvb_ctx* ctx, cvb_db* dst, const cvb_db* src);

/*
 * Replaces the SIFT branch, cv::FlannBasedMatcher()::knnMatch(query, train, out, 2)
 *   (placerec_gen_be.cpp:86-87,99; RelNonCentralPosSolver.cpp:310-311,323), with the EXACT brute-force
 *   result cv::BFMatcher(NORM_L2) gives (FLANN is approximate and randomised; SURVEY.md §8a M2).
 * q/t are CV_32F rows of `dim` floats (dim == 128, SIFT; other lengths → CVB_ERR_UNSUPPORTED).  Descriptors must be
 * integer-valued in [0,255] (what cv::xfeatures2d::SIFT emits) — then every fp32 partial sum of the
 * reference is exact and the result is bit-identical to OpenCV; other inputs → CVB_ERR_UNSUPPORTED.
 * dist = sqrtf(sum (a-b)^2) as float.
 */
CVB_API int cvb_knn_l2_batch(cvb_ctx* ctx, const float* q, int nq, const float* t, const int32_t* seg_ptr,
                             int n_seg, int dim, int k, int32_t* idx, float* dist);
/* device variant on the HBM-resident layout: descriptors quantised to u8 [rows][dim] (exact) */
CVB_API int cvb_knn_l2_u8_batch_dev(cvb_ctx* ctx, const uint8_t* d_q, int nq, const uint8_t* d_t,
                                    const int32_t* d_seg_ptr, const int32_t* h_seg_ptr, int n_seg, int dim,
                                    int k, int32_t* d_idx, float* d_dist, void* stream);
CVB_API int cvb_match_l2_batch(cvb_ctx* ctx, const float* q, int nq, const float* t, const int32_t* seg_ptr,
                               int n_seg, int dim, float thr, float ratio, int32_t* match_train,
                               float* match_dist, int32_t* n_matches);
/*
 * Map-wide k-NN with the database sharded by keyframe block over G GPUs (SURVEY §8e "KNN (map-wide)"): every rank
 * runs cvb_knn_hamming_batch_dev / cvb_knn_l2_u8_batch_dev on its shard, the per-shard lists are all-gathered
 * (idx_all / dist_all: [n_shards][n][k], n = n_seg*nq rows; shard-local trainIdx) and this call merges them by
 * (distance, global trainIdx = local + row_offset[shard]) — exactly the list one BFMatcher::knnMatch over the
 * concatenated database returns (ties → lower trainIdx first).  dist_is_float: 0 = int32 Hamming, 1 = float L2.
 * Missing neighbours: idx -1, distance INT_MAX / FLT_MAX.  1 <= k <= 8.
 */
CVB_API int cvb_knn_merge_shards_dev(cvb_ctx* ctx, const int32_t* d_idx_all, const void* d_dist_all, int dist_is_float,
                                     const int32_t* d_row_offset, int n_shards, int64_t n, int k, int32_t* d_idx_out,
                                     void* d_dist_out, void* stream);

/*
 * Landmark::ComputeDescriptor (src/covins_backend/landmark_be.cpp:49-92), batched over landmarks (SURVEY §8a M7;
 * called for every landmark of a new keyframe, communicator_be.cpp:190-198, and after map maintenance).
 * cand: the 32-byte descriptor rows of the valid observing keyframes of every landmark (kf->descriptors_.row(feat_idx),
 * :57-64), concatenated in the landmark's observation order; lm_ptr[n_lm+1] row offsets.  Per landmark the row with the
 * least median Hamming distance to all rows (zero diagonal included; median = sorted[(int)(0.5 (n-1))]; first row
 * wins ties, :80-90): best_idx[l] = landmark-local row or -1 if the landmark has no candidate, out_desc[l] = its 32
 * bytes (left as passed in when -1: the reference returns early and keeps the old descriptor, :53-55,65-67).
 */
CVB_API int cvb_landmark_descriptor_batch(cvb_ctx* ctx, const uint8_t* cand, const int32_t* lm_ptr, int n_lm,
                                          int32_t* best_idx, uint8_t* out_desc);
CVB_API int cvb_landmark_descriptor_batch_dev(cvb_ctx* ctx, const uint8_t* d_cand, const int32_t* d_lm_ptr, int n_lm,
                                              int32_t* d_best_idx, uint8_t* d_out_desc, void* stream);

/* f32 [rows][dim] (device) → u8 [rows][dim] (device); *d_bad (int32, device) is set to 1 if any value is
 * not an integer in [0,255]. */
CVB_API int cvb_quantize_u8_dev(cvb_ctx* ctx, const float* d_src, int64_t n, uint8_t* d_dst, int32_t* d_bad,
                                void* stream);

/*
 * Replaces estd2::DenseMatcher(8).match<LandmarkMatchingAlgorithm>(algo) with
 * LandmarkMatchingAlgorithm(50.0), src/covins_backend/placerec_be.cpp:85-90:
 *   top-numBest scan   include/covins/dense_matcher/implementation/DenseMatcher.hpp:152-220
 *   mutual assignment  src/dense_matcher/DenseMatcher.cpp:62-104
 *   final sweep        include/covins/dense_matcher/implementation/DenseMatcher.hpp:93-121
 *   distance           include/covins/matcher/LandmarkMatchingAlgorithm.h:103-114 (256-bit Hamming,
 *                      src/covins_backend/feature_matcher_be.cpp:49-64; FLT_MAX if >= thr)
 * in the canonical A-sequential order (the reference with numMatcherThreads = 1; with 8 threads its
 * tie outcome depends on thread arrival order).  A = query KF descriptors [nA][32], skipA[nA] = 1 where
 * the keypoint has no valid landmark (LandmarkMatchingAlgorithm.cpp:76-84); B = concatenated candidate
 * KFs with seg_ptr as above.  num_best in 1..4 (reference: 4), thr 50.0.
 * Output per segment s, in the slice [seg_ptr[s], seg_ptr[s]+n_out[s]): matches ordered by B index,
 * outA = idxA, outB = idxB (segment-local), outD = distance — the Matches vector of placerec_be.cpp:91.
 */
CVB_API int cvb_landmark_match_batch(cvb_ctx* ctx, const uint8_t* A, const uint8_t* skipA, int nA,
                                     const uint8_t* B, const uint8_t* skipB, const int32_t* seg_ptr,
                                     int n_seg, float thr, int num_best, int32_t* outA, int32_t* outB,
                                     float* outD, int32_t* n_out);
CVB_API int cvb_landmark_match_batch_dev(cvb_ctx* ctx, const uint8_t* d_A, const uint8_t* d_skipA, int nA,
                                         const uint8_t* d_B, const uint8_t* d_skipB, const int32_t* d_seg_ptr,
                                         const int32_t* h_seg_ptr, int n_seg, float thr, int num_best,
                                         int32_t* d_outA, int32_t* d_outB, float* d_outD, int32_t* d_n_out,
                                         void* stream);

/* ------------------------------------------------------------------------------------------------
 * Guided search and geometric-verification scoring (SURVEY.md §8a M8 / V1, §8f-3)
 * ---------------------------------------------------------------------------------------------- */

/* What FeatureMatcher::SearchBySE3 reads of one keyframe (src/covins_backend/feature_matcher_be.cpp:293-498), flattened
 * by the host shim; all pointers HOST memory, arrays indexed by keypoint. */
typedef struct cvb_kf_view {
  int32_t n;                 /* keypoints_distorted_.size() == GetLandmarks().size() */
  const float* kp;           /* [n][2] keypoints_distorted_ (float, typedefs_base.hpp:130) */
  const float* octave;       /* [n]    keypoints_aors_[i][1]; the reference truncates it to int (:379,:456) */
  const uint8_t* desc;       /* [n][32] descriptors_ rows (GetDescriptorCV, keyframe_base.cpp:258-260) */
  const uint8_t* lm_valid;   /* [n]    1 = GetLandmarks()[i] != nullptr && !IsInvalid() (:335-341,:411-419) */
  const double* lm_pos;      /* [n][3] GetWorldPos() */
  const double* lm_maxdist;  /* [n]    max_distance_ (LandmarkBase::PredictScale, landmark_base.cpp:120-133) */
  const uint8_t* lm_desc;    /* [n][32] Landmark::GetDescriptor() */
  const int32_t* grid_ptr;   /* [64*48+1] CSR of keypoint_grid_[ix][iy], cell = ix*48 + iy (FRAME_GRID_COLS x ROWS,
                                typedefs_base.hpp:59-60), members in insertion (= ascending keypoint) order
                                (KeyframeBase::AssignFeaturesToGrid, keyframe_base.cpp:122-143) */
  const int32_t* grid_idx;   /* [grid_ptr[3072]] */
  double grid_w_inv, grid_h_inv;   /* grid_width_inv_, grid_height_inv_ */
  double K[9];               /* calibration_.K, row-major */
  double Tcw[16];            /* GetPoseTcw(), row-major 4x4 */
  double img[4];             /* img_dim_x_min_, img_dim_x_max_, img_dim_y_min_, img_dim_y_max_ (IsInImage, keyframe_base.cpp:414-416) */
} cvb_kf_view;

typedef struct cvb_search_params {
  double th;                 /* search radius factor (matcher.search_radius_SE3 = 9.5) */
  int32_t desc_th_low;       /* matcher.desc_matching_th_low = 50 */
  int32_t num_octaves;       /* feat.num_octaves */
  double scale_factor;       /* feat.scale_factor (> 1; PredictScale); SearchBySE3's radius uses pow(2.0, level) (:366,:443),
                                SearchByProjection's pow(scale_factor, level) */
} cvb_search_params;

/*
 * Replaces FeatureMatcher::SearchBySE3(pKF1, pKF2, matches12, T12, th) for a batch of candidate keyframes pKF2[p]
 * (the loop of placerec_be.cpp:113-160 calls it once per surviving candidate).  T12 / T21 [n_pairs][16] row-major: T21 is
 * T12.inverse() as the caller's Eigen computes it (:300).  already1 [n_pairs][kf1->n] / already2 (concatenated,
 * kf2[p].n each): the alreadyMatched1/2 masks of :312-324.  Reference behaviour reproduced on purpose:
 *   - direction 2→1 tests pKF2->IsInImage for a projection into KF1 (:433);
 *   - the agreement test reads match2[i], not match2[idx2] (:489) (i >= n2 counts as no match — the reference indexes
 *     out of bounds there);
 *   - direction 1→2 accepts bestDist <= th_low (float), direction 2→1 bestDist < th_low (int) (:403,:479);
 *   - keypoints whose grid cell index falls outside the 64x48 grid (x*grid_w_inv rounds to 64) are not in the grid
 *     (the reference writes out of bounds there).
 * Outputs: match12 [n_pairs][kf1->n] = index of the KF2 keypoint whose landmark becomes matches12[i], or -1;
 * n_found [n_pairs] = the return value; match1 [n_pairs][n1] / match2 (concatenated like already2) = the two
 * directional results (nullable, for tests).
 */
CVB_API int cvb_search_by_se3_batch(cvb_ctx* ctx, const cvb_kf_view* kf1, const cvb_kf_view* kf2, int n_pairs,
                                    const double* T12, const double* T21, const uint8_t* already1, const uint8_t* already2,
                                    const cvb_search_params* prm, int32_t* match12, int32_t* n_found, int32_t* match1,
                                    int32_t* match2);

/*
 * Replaces FeatureMatcher::SearchByProjection(pKF, Tcw, vpPoints, vpMatched, th) (feature_matcher_be.cpp:168-291; called at
 * placerec_be.cpp:194 with the loop map points).  kf: kp / octave / desc / grid / img of pKF, lm_valid[idx] = pKF->GetLandmark(idx)
 * != nullptr (the other cvb_kf_view fields are not read); kf_lm_cand [n]: index into the candidate list of the landmark that
 * sits at keypoint idx, -1 if none or not in the list (RemapLandmark bookkeeping, keyframe_be.cpp:484-495); Tcw row-major;
 * intr/dist + cam_model/dist_model/xi: the camera_->project3 model (as in cvb_ba_problem); matched [n] = vpMatched[idx] != nullptr
 * on entry.  Per candidate landmark i: action 0 = nothing, 1 = vpMatched[best_idx[i]] = pMP (counted in *n_matches),
 * 2 = RemapLandmark(pMP, feat_idx[i], best_idx[i]), 3 = already observed and not replaced.  The reference's sequential
 * semantics (earlier landmarks take keypoints first) are reproduced exactly.
 */
typedef struct cvb_proj_landmarks {
  int32_t m;
  const uint8_t* valid;        /* [m] !IsInvalid() && not in spAlreadyFound (:177-187) */
  const double* pos;           /* [m][3] GetWorldPos() */
  const double* normal;        /* [m][3] GetNormal() */
  const double* min_dist;      /* [m] GetMinDistanceInvariance() */
  const double* max_dist;      /* [m] GetMaxDistanceInvariance() */
  const double* max_distance;  /* [m] max_distance_ (PredictScale) */
  const uint8_t* desc;         /* [m][32] GetDescriptor() */
  const int32_t* feat_idx;     /* [m] GetFeatureIndex(pKF) or -1 */
} cvb_proj_landmarks;
CVB_API int cvb_search_by_projection(cvb_ctx* ctx, const cvb_kf_view* kf, const int32_t* kf_lm_cand, const double* Tcw, const double* intr,
                                     const double* dist, int cam_model, int dist_model, double xi, const cvb_proj_landmarks* lms,
                                     const uint8_t* matched, const cvb_search_params* prm, int32_t* action, int32_t* best_idx,
                                     int32_t* n_matches);

/*
 * RANSAC hypothesis scoring, batched over hypotheses (the inner loop of opengv's Ransac::computeModel —
 * countWithinDistance / selectWithinDistance over all correspondences — for every hypothesis in one launch; sampling and the
 * minimal solvers stay with the caller, SURVEY §8a V1: "given the same sampled minimal sets, identical scores / inlier masks").
 *
 * Absolute pose (Se3Solver::projectiveAlignment, Se3Solver.cpp:59-110, GP3P; score of
 * include/covins/matcher/opengv/sac_problems/FrameAbsolutePoseSacProblem.h:95-126):
 *   model [n_hyp][12] = 3x4 [R|t] row-major (body in world); per correspondence i: world point pts[i], bearing f[i],
 *   camera offset/rotation (one camera: cam_off[3], cam_rot[9] row-major), sigma[i] = getSigmaAngle(i);
 *   score = |normalize(Rc^T (R^T (p - t) - c)) - f|^2 / sigma;  inlier iff score < threshold (opengv Ransac).
 * Relative pose (RelNonCentralPosSolver::computePose, RelNonCentralPosSolver.cpp:343-377;
 * frame-relative-pose-sac-problem.hpp:69-104 with opengv::triangulation::triangulate2):
 *   model [n_hyp][12] = [R12|t12]; bearings f1[i], f2[i], sigma1[i], sigma2[i];
 *   score = 0.5 |normalize(X) - f1|^2 / sigma1 + 0.5 |normalize(R12^T (X - t12)) - f2|^2 / sigma2, X = triangulate2.
 * Outputs: scores [n_hyp][n] (nullable), inlier [n_hyp][n] u8 (nullable), n_inliers [n_hyp].
 */
CVB_API int cvb_score_absolute_pose_batch(cvb_ctx* ctx, const double* model, int n_hyp, const double* pts, const double* f,
                                          const double* sigma, int n, const double* cam_off, const double* cam_rot,
                                          double threshold, double* scores, uint8_t* inlier, int32_t* n_inliers);
CVB_API int cvb_score_relative_pose_batch(cvb_ctx* ctx, const double* model, int n_hyp, const double* f1, const double* f2,
                                          const double* sigma1, const double* sigma2, int n, double threshold,
                                          double* scores, uint8_t* inlier, int32_t* n_inliers);

/*
 * The whole absolute-pose RANSAC of Se3Solver::projectiveAlignment (GP3P, Se3Solver.cpp:59-110) for a batch of problems
 * (candidate keyframes) in one launch, from the caller's samples: minimal solve, hypothesis choice, scoring, the sequential
 * model selection of opengv's Ransac::computeModel and the inlier mask of the selected model.  Samples stay an input
 * (opengv's random number generator cannot be reproduced, SURVEY §8c).
 *   Hypothesis of a sample: P3P (Lambda Twist) on its first three correspondences; the solutions with positive depth for all
 *   three points, as body-in-world models [R|t] (the scoring's convention); the one whose predicted direction of the fourth
 *   point has the smallest 1 - cos angle to its bearing (strict <: the first of equal values wins).  A sample is invalid (no
 *   hypothesis) if no solution survives, a value is non-finite, an index repeats within the sample or the problem has fewer
 *   than 4 correspondences.  With one camera per problem the three rays share a centre, so GP3P's solution set is P3P's.
 *   ASSUMPTION (opengv is not in the tree): sample size 4 and the fourth-point choice follow opengv's AbsolutePoseSacProblem.
 *   Score: exactly cvb_score_absolute_pose_batch's per-correspondence score (the same device function), inlier iff
 *   score < threshold.
 *   Selection: samples are consumed in order; an invalid sample does not consume an iteration (ASSUMPTION: opengv's
 *   skipped_count, at most 10 * max_iterations skips); valid hypotheses go through covins_b200.placerec.ransac_select with
 *   sample_size 4 — the result equals ransac_select over the inlier counts of the valid samples in order, mapped back to
 *   sample indices.  w^4 is computed as plain products and log on the device: the adaptive bound can differ from a host
 *   evaluation (pow / glibc log) by an ulp, which only matters when it lands within an ulp of an integer.
 * Inputs: correspondences concatenated over problems (prob_ptr[n_prob+1], prob_ptr[0] = 0): world point pts[i], unit bearing
 * f[i], sigma[i] as in cvb_score_absolute_pose_batch; one camera per problem, cam_off [n_prob][3], cam_rot [n_prob][9]
 * (row-major, in the body frame); samples [n_prob][n_samples][4], indices local to their problem (checked against the
 * problem's size; the samples of a problem with fewer than 4 correspondences are not read).
 * Outputs per problem: best_sample (-1 = none), best_model [12] (zeros if none), best_count, iterations (valid samples
 * scored by the selection), consumed (samples read by the selection).  inlier_mask [N] (nullable): the selected model's
 * inlier flags, 0 where there is none.  sample_model [n_prob][n_samples][12] / sample_valid / sample_count (nullable
 * together, for tests): every sample's hypothesis (zeros if invalid) and inlier count — when requested, every sample is
 * solved and scored, not only the consumed ones.
 * Errors: CVB_ERR_INVALID for negative sizes, null required pointers or an out-of-range index, before any launch;
 * n_prob = 0 succeeds.
 */
typedef struct cvb_abs_ransac_problems {
  int32_t n_prob;
  const int32_t* prob_ptr;   /* [n_prob+1] */
  const double* pts;         /* [N][3] world points */
  const double* f;           /* [N][3] unit bearings, camera frame */
  const double* sigma;       /* [N] getSigmaAngle(i) */
  const double* cam_off;     /* [n_prob][3] camera offset c in the body frame */
  const double* cam_rot;     /* [n_prob][9] camera rotation Rc in the body frame, row-major */
  const int32_t* samples;    /* [n_prob][n_samples][4] */
  int32_t n_samples;
} cvb_abs_ransac_problems;
typedef struct cvb_abs_ransac_result {
  int32_t* best_sample;      /* [n_prob] */
  double* best_model;        /* [n_prob][12] 3x4 [R|t] row-major, body in world */
  int32_t* best_count;       /* [n_prob] */
  int32_t* iterations;       /* [n_prob] */
  int32_t* consumed;         /* [n_prob] */
  uint8_t* inlier_mask;      /* [N] nullable */
  double* sample_model;      /* [n_prob][n_samples][12] nullable */
  uint8_t* sample_valid;     /* [n_prob][n_samples]     nullable */
  int32_t* sample_count;     /* [n_prob][n_samples]     nullable */
} cvb_abs_ransac_result;
CVB_API int cvb_ransac_absolute_pose_batch(cvb_ctx* ctx, const cvb_abs_ransac_problems* p, double threshold, int max_iterations,
                                           double probability, cvb_abs_ransac_result* r);

/*
 * The non-central relative-pose RANSAC of RelNonCentralPosSolver::computeNonCentralRelPose (17-point,
 * RelNonCentralPosSolver.cpp:146-173: the COVINS_G verification of a candidate, each side a rig of a keyframe and its
 * neighbours) for a batch of problems in one launch, from the caller's samples: 17-point solve, scoring per camera pair,
 * the sequential model selection of opengv's Ransac::computeModel and the inlier mask of the selected model.  Samples stay
 * an input, as in cvb_ransac_absolute_pose_batch.
 *   Rigs: a point x_c in camera frame j of a rig maps to Rc_j x_c + c_j in the rig frame.  At most CVB_REL_MAX_CAMS cameras
 *   per rig.  A caller with one rig for both views (opengv's own adapter) passes it twice.
 *   Model: [R|t] row-major 3x4 with X1 = R X2 + t (rig frames; cvb_score_relative_pose_batch's [R12|t12] convention).
 *   Hypothesis of a sample (17 problem-local indices):
 *     1. Plücker lines d = Rc f, m = c x d per side; row i of A (17x18), in sample order, is
 *        [vec(d1 d2^T), vec(d1 m2^T + m1 d2^T)] (vec = row-major), from the generalised epipolar constraint
 *        d1^T E d2 + d1^T R m2 + m1^T R d2 = 0, E = [t]x R.
 *     2. Null vector x of A: Householder QR of A^T (18x17), x = Q e18.  The sample is invalid if
 *        min_k |r_kk| < 1e-10 max_k |r_kk| (rank below 17: a rig whose cameras share one centre, repeated points).
 *     3. R' = x[9:18] (row-major); if det R' < 0 it is negated, if det R' = 0 the sample is invalid.  R is the orthonormal
 *        polar factor of R', from R' scaled to |R'|_F = sqrt(3) by 12 Newton steps X <- (X + X^-T) / 2.
 *     4. t: least squares over the sample's 17 rows with R fixed, (R d2 x d1) . t = -(d1^T R m2 + m1^T R d2), by the 3x3
 *        normal equations summed in sample order.
 *     ASSUMPTION (opengv is not in the tree): opengv's seventeenpt may recover t from E instead; on noise-free data both give
 *     the same model.
 *     The sample is also invalid if the problem has fewer than 17 correspondences, an index repeats within the sample, a
 *     bearing of the sample or a camera of either rig is not finite, or the model is not finite.
 *   Score of correspondence i: with the camera-pair model R_p = Rc1^T R Rc2, t_p = Rc1^T (R c2 + t - c1) of its cameras
 *   (cam1[i], cam2[i]), exactly cvb_score_relative_pose_batch's per-correspondence score (the same device function), inlier
 *   iff score < threshold.  ASSUMPTION: the 17-point RANSAC scores with the same FrameRelativePoseSacProblem score as the
 *   5-point one, applied per camera pair.
 *   Selection: as cvb_ransac_absolute_pose_batch with sample size 17 (invalid samples do not consume an iteration, at most
 *   10 * max_iterations are skipped; ransac_select's rule).  w^17 is a left-to-right product chain and log runs on the device:
 *   the adaptive bound can differ from a host evaluation (pow / glibc log) by an ulp, which only matters when it lands within
 *   an ulp of an integer.
 * Inputs: correspondences concatenated over problems (prob_ptr[n_prob+1], prob_ptr[0] = 0): unit bearings f1[i], f2[i], each
 * in its own camera's frame, sigma1[i], sigma2[i] as in cvb_score_relative_pose_batch, camera indices cam1[i], cam2[i] local to
 * the problem's rigs.  Rig 1 of problem p is cameras cam_ptr1[p] .. cam_ptr1[p+1]-1 of cam_off1 [.][3] / cam_rot1 [.][9]
 * (row-major), rig 2 likewise.  samples [n_prob][n_samples][17], indices local to their problem (the samples of a problem with
 * fewer than 17 correspondences are not read).
 * Outputs: as cvb_ransac_absolute_pose_batch (best_model = [R|t] above).
 * Errors: CVB_ERR_INVALID before any launch for negative sizes, null required pointers, a decreasing prob_ptr / cam_ptr1 /
 * cam_ptr2, an out-of-range sample index, a camera index outside its rig, a rig of more than CVB_REL_MAX_CAMS cameras, or
 * per-sample outputs not requested together; n_prob = 0 succeeds.
 */
#define CVB_REL_MAX_CAMS 8
typedef struct cvb_rel_ransac_problems {
  int32_t n_prob;
  const int32_t* prob_ptr;   /* [n_prob+1] */
  const double* f1;          /* [N][3] unit bearings, frame of camera cam1[i] of rig 1 */
  const double* f2;          /* [N][3] unit bearings, frame of camera cam2[i] of rig 2 */
  const double* sigma1;      /* [N] */
  const double* sigma2;      /* [N] */
  const int32_t* cam1;       /* [N] camera of rig 1, local to the problem */
  const int32_t* cam2;       /* [N] camera of rig 2, local to the problem */
  const int32_t* cam_ptr1;   /* [n_prob+1] cameras of rig 1 per problem */
  const double* cam_off1;    /* [cam_ptr1[n_prob]][3] camera centre c in the rig frame */
  const double* cam_rot1;    /* [cam_ptr1[n_prob]][9] camera rotation Rc in the rig frame, row-major */
  const int32_t* cam_ptr2;   /* [n_prob+1] */
  const double* cam_off2;    /* [cam_ptr2[n_prob]][3] */
  const double* cam_rot2;    /* [cam_ptr2[n_prob]][9] */
  const int32_t* samples;    /* [n_prob][n_samples][17] */
  int32_t n_samples;
} cvb_rel_ransac_problems;
typedef struct cvb_rel_ransac_result {
  int32_t* best_sample;      /* [n_prob] */
  double* best_model;        /* [n_prob][12] 3x4 [R|t] row-major, X1 = R X2 + t */
  int32_t* best_count;       /* [n_prob] */
  int32_t* iterations;       /* [n_prob] */
  int32_t* consumed;         /* [n_prob] */
  uint8_t* inlier_mask;      /* [N] nullable */
  double* sample_model;      /* [n_prob][n_samples][12] nullable */
  uint8_t* sample_valid;     /* [n_prob][n_samples]     nullable */
  int32_t* sample_count;     /* [n_prob][n_samples]     nullable */
} cvb_rel_ransac_result;
CVB_API int cvb_ransac_noncentral_relative_pose_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, double threshold, int max_iterations,
                                                      double probability, cvb_rel_ransac_result* r);

/*
 * The central relative-pose RANSAC of RelNonCentralPosSolver::computePose (5-point, RelNonCentralPosSolver.cpp:343-377: opengv's
 * Stewénius solver inside FrameRelativePoseSacProblem, run after each of the six pairwise matchings of
 * computeNonCentralRelPose) for a batch of problems in one launch, from the caller's samples: 5-point solve, scoring, the
 * sequential model selection of opengv's Ransac::computeModel and the inlier mask of the selected model.  Samples stay an input.
 *   Model: [R|t] row-major 3x4 with X1 = R X2 + t, |t| = 1 (cvb_score_relative_pose_batch's [R12|t12] convention).
 *   Hypothesis of a sample (5 problem-local indices), with only + - * / and sqrt, fixed iteration counts and fixed summation
 *   order (bit-identical to a -ffp-contract=off C restatement):
 *     1. q_i = vec(f1_i f2_i^T) (row-major, q_i . vec(E) = f1^T E f2).  Householder QR of Q^T (9x5); null-space basis
 *        X, Y, Z, W = H_0..H_4 e_5..e_8.  The sample is invalid if min_k |r_kk| < 1e-10 max_k |r_kk|.
 *     2. E = xX + yY + zZ + W; the nine entries of 2 E E^T E - tr(E E^T) E and det E give a 10x20 coefficient matrix in
 *        Nistér's monomial order (Nistér 2004, §3).
 *     3. Gauss-Jordan elimination of its left 10x10 block with partial pivoting (largest |value|, first row on ties); the
 *        sample is invalid if a pivot is below 1e-10 times the largest |entry| of the matrix.  B(z) has rows <e> - z<f>,
 *        <g> - z<h>, <i> - z<j>; n(z) = det B(z) has degree 10.  Real roots of n inside the Cauchy bound (invalid if it is not
 *        finite): the real roots of n', n'', ... bracket those of n, so the roots of n^(9), n^(8), ..., n are found in turn,
 *        one per sign change between consecutive roots of the previous derivative, by 64 bisection steps and 4 Newton steps
 *        kept inside the bracket.  Per root, in ascending z: (x, y, 1) ~ the largest cross product of two rows of B(z) (the
 *        first on ties), then at most 6 Gauss-Newton steps on the ten cubics in (x, y, z) (the first step that does not
 *        lower their squared residual is undone and ends the polish), then E.
 *     4. E scaled to tr(E E^T) / 2 = 1.  b = the largest of E's three column cross products (the first on ties), normalised:
 *        the unit left null vector.  R_+- = cof(E) -+ [b]x E (cof(E)_ij = (-1)^(i+j) M_ij, not transposed): both are rotations
 *        whatever the sign of E.  Candidates in this order: (R_+, b), (R_+, -b), (R_-, b), (R_-, -b).
 *     5. quality = sum over the sample's 5 correspondences, in sample order, of (1 - f1 . X/|X|) + (1 - f2 . r2/|r2|), X and
 *        r2 = R^T (X - t) from the score's triangulation.  The strictly lowest finite quality over roots x candidates wins.
 *     The sample is also invalid if no real root or no finite candidate exists, the problem has fewer than 5 correspondences,
 *     an index repeats within the sample, a bearing of the sample is not finite, or the model is not finite.
 *     ASSUMPTIONS (opengv is not in the tree): Stewénius' eigen-decomposition is replaced by Nistér's polynomial, and only its
 *     real roots are kept, where opengv takes the real parts of all ten complex solutions; |t| = 1, where opengv scales t by
 *     E's largest singular value (the score does not depend on |t|); the quality test of
 *     CentralRelativePoseSacProblem::computeModelCoefficients runs on the sample's points only.  Every solution satisfies the
 *     five epipolar constraints, so on noise-free data several can tie near zero quality and rounding decides between them:
 *     the chosen hypothesis of one sample need not be the true pose.
 *   Score of correspondence i: exactly cvb_score_relative_pose_batch's per-correspondence score (the same device function),
 *   inlier iff score < threshold.
 *   Selection: as cvb_ransac_noncentral_relative_pose_batch with sample size 5.
 * Inputs: correspondences concatenated over problems (prob_ptr[n_prob+1], prob_ptr[0] = 0): unit bearings f1[i], f2[i],
 * sigma1[i], sigma2[i] as in cvb_score_relative_pose_batch; samples [n_prob][n_samples][5], indices local to their problem (the
 * samples of a problem with fewer than 5 correspondences are not read).
 * Outputs: cvb_rel_ransac_result, as cvb_ransac_noncentral_relative_pose_batch.
 * Errors: CVB_ERR_INVALID before any launch for negative sizes, null required pointers, a decreasing prob_ptr, an out-of-range
 * sample index, or per-sample outputs not requested together; n_prob = 0 succeeds.
 */
typedef struct cvb_central_rel_ransac_problems {
  int32_t n_prob;
  const int32_t* prob_ptr;   /* [n_prob+1], prob_ptr[0] = 0 */
  const double* f1;          /* [N][3] unit bearings, camera 1 */
  const double* f2;          /* [N][3] unit bearings, camera 2 */
  const double* sigma1;      /* [N] */
  const double* sigma2;      /* [N] */
  const int32_t* samples;    /* [n_prob][n_samples][5], problem-local indices */
  int32_t n_samples;
} cvb_central_rel_ransac_problems;
CVB_API int cvb_ransac_central_relative_pose_batch(cvb_ctx* ctx, const cvb_central_rel_ransac_problems* p, double threshold,
                                                   int max_iterations, double probability, cvb_rel_ransac_result* r);

/*
 * The sampling-based 6x6 covariance of the non-central relative pose (RelNonCentralPosSolver::computeNonCentralRelPose,
 * RelNonCentralPosSolver.cpp:199,236,276-279: up to 300 17-point re-solves on subsets of the selected model's inliers, the
 * matrix that becomes LoopConstraint::cov_mat) for a batch of problems (candidates), from the caller's samples.  Sampling
 * stays with the caller: the samples are normally drawn from the inlier mask of cvb_ransac_noncentral_relative_pose_batch,
 * but their indices need not be inliers.
 *   Inputs per problem: the correspondences and rigs of cvb_rel_ransac_problems (sigma1 / sigma2 are not read and may be
 *   null), samples [n_prob][n_samples][17], and a reference model ref_model [n_prob][12] = [R_ref|t_ref] (X1 = R X2 + t,
 *   normally the problem's best_model).
 *   Per sample: the 17-point hypothesis [R_s|t_s] of cvb_ransac_noncentral_relative_pose_batch, with exactly its rules for
 *   an invalid sample (an invalid sample is skipped and not counted).  Its deviation from the reference is
 *     delta = [dtheta; dt], dtheta = 2 vec(q), q = (x, y, z, w) the quaternion of R_ref^T R_s by Eigen's matrix-to-quaternion
 *     branches (trace > 0, else the largest diagonal entry), negated if w < 0; dt = t_s - t_ref.
 *   Per problem: cov = (1 / n_valid) sum delta delta^T over the valid samples, summed in sample order; cov = 0 when
 *   n_valid = 0.  A problem whose reference model is all zeros (a RANSAC without a model) is skipped: n_valid = 0, and its
 *   samples are not read.
 *   Only + - * / and sqrt as non-fused operations and fixed summation orders: the results are bit-identical to a
 *   -ffp-contract=off C restatement, and cov is exactly symmetric.
 *   ASSUMPTIONS (robopt and opengv are not in the tree):
 *     - rotation first, right-side deviation, 2 vec(q) rather than Log: cov is in the coordinates of the residual it whitens,
 *       the pose-graph between factor e = [2 vec(q_m^-1 q_hat); t_hat - t_m].  (robopt's quaternion::Minus may be a left-side
 *       Log instead.)
 *     - the second moment about the reference, divided by n_valid: the mean is not subtracted and the divisor is not n - 1.
 *     - minimal 17-point re-solves, not a non-minimal solver.
 * Outputs: cov [n_prob][36] row-major, n_valid [n_prob]; on request (both or neither) every sample's delta
 * [n_prob][n_samples][6] (0 for an invalid sample) and valid flag.
 * Errors: CVB_ERR_INVALID before any launch for the errors of cvb_ransac_noncentral_relative_pose_batch (negative sizes, null
 * required pointers, a decreasing prob_ptr / cam_ptr1 / cam_ptr2, an out-of-range sample index of a problem that is read, a
 * camera index outside its rig, a rig of more than CVB_REL_MAX_CAMS cameras, per-sample outputs not requested together), and
 * for a non-zero reference model that is not finite or whose R is not a rotation (max |R^T R - I| > 1e-6); n_prob = 0
 * succeeds.
 */
typedef struct cvb_rel_cov_result {
  double* cov;               /* [n_prob][36] row-major, dtheta then dt */
  int32_t* n_valid;          /* [n_prob] */
  double* sample_delta;      /* [n_prob][n_samples][6] nullable */
  uint8_t* sample_valid;     /* [n_prob][n_samples]    nullable together */
} cvb_rel_cov_result;
CVB_API int cvb_noncentral_relative_pose_covariance_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, const double* ref_model,
                                                          cvb_rel_cov_result* r);

/*
 * Seeded samples: the four calls above with the samples drawn on the device from one 64-bit seed per problem, so the call
 * sites need no sampler of their own (opengv draws inside Ransac::computeModel, and computeNonCentralRelPose draws its
 * covariance subsets itself, RelNonCentralPosSolver.cpp:199,236).
 *   Sampler (this project's own definition; oracle/sampler_oracle.c restates it):
 *     Generator: Philox4x64-10 (Salmon et al., SC'11), the bit generator of numpy.random.Philox, with key (seed_p, stream):
 *     seed_p the problem's seed, stream 0 for RANSAC samples and 1 for covariance samples (one seed per candidate serves
 *     both).  Sample s of a problem uses counters (s, b, 0, 0), b = 0, 1, ...; each block gives four 64-bit words, each
 *     word two 32-bit values, low half first: the stream u_0, u_1, ...  (One block serves sample sizes 4 and 5, three serve 17.)
 *     Ordered k-subset of [0, m): a partial Fisher-Yates shuffle of the identity permutation; for i = 0 .. k-1,
 *     j = i + (uint32)(((uint64)u_i * (m - i)) >> 32), swap perm[i] and perm[j], sample[i] = perm[i].  A sample never repeats
 *     an index.  A problem's samples depend only on (seed_p, stream, m, k, s): it gives the same results alone or anywhere
 *     in a batch, and sample s is drawn without drawing samples 0 .. s-1.
 *     ASSUMPTION (opengv's std::mt19937 is seeded from the clock, so no reference run can be replayed): only the
 *     distribution is kept.  Like opengv's shuffle, the subsets are uniform up to a bias of at most m / 2^32.
 *   RANSAC (m = n, indices local to the problem): the selection of the sample-supplied call, never limited by a sample
 *   count: samples are drawn until opengv's bound ends it (max_iterations valid samples, the adaptive bound, or
 *   10 * max_iterations skipped).  A problem with fewer than k correspondences (4, 17, 5) draws nothing: iterations =
 *   consumed = 0, best_sample = -1 (opengv's getSamples returns an empty selection and computeModel stops).  p->samples must
 *   be NULL; p->n_samples only sizes the optional per-sample outputs (sample_model / sample_valid / sample_count, which
 *   cover samples 0 .. n_samples-1 whether or not the selection reads them) and drawn.
 *   Covariance (m = the problem's number of inliers in inlier_mask [N]; index j of a subset means the j-th inlier in
 *   ascending correspondence order): p->n_samples subsets per problem (the reference's 300).  A problem with fewer than 17
 *   inliers, or with an all-zero ref_model, draws nothing and gets n_valid = 0.
 *   drawn (nullable): [n_prob][n_samples][k] the drawn samples as problem-local correspondence indices, -1 in the rows that
 *   were not drawn.
 * Errors: those of the sample-supplied twin except the sample-index check, and CVB_ERR_INVALID before any launch for a
 * non-null p->samples, a null seed with n_prob > 0, (covariance) a null inlier_mask, or (RANSAC) max_iterations above
 * (INT32_MAX - 64) / 11, so that every sample number the selection can reach (at most 11 * max_iterations) fits an int32.
 */
CVB_API int cvb_ransac_absolute_pose_seeded_batch(cvb_ctx* ctx, const cvb_abs_ransac_problems* p, const uint64_t* seed, double threshold,
                                                  int max_iterations, double probability, cvb_abs_ransac_result* r, int32_t* drawn);
CVB_API int cvb_ransac_noncentral_relative_pose_seeded_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, const uint64_t* seed,
                                                             double threshold, int max_iterations, double probability,
                                                             cvb_rel_ransac_result* r, int32_t* drawn);
CVB_API int cvb_ransac_central_relative_pose_seeded_batch(cvb_ctx* ctx, const cvb_central_rel_ransac_problems* p, const uint64_t* seed,
                                                          double threshold, int max_iterations, double probability,
                                                          cvb_rel_ransac_result* r, int32_t* drawn);
CVB_API int cvb_noncentral_relative_pose_covariance_seeded_batch(cvb_ctx* ctx, const cvb_rel_ransac_problems* p, const double* ref_model,
                                                                 const uint8_t* inlier_mask, const uint64_t* seed, cvb_rel_cov_result* r,
                                                                 int32_t* drawn);

/*
 * The COVINS_G verification of place-recognition candidates (RelNonCentralPosSolver::computeNonCentralRelPose: pairwise ORB
 * matching, a 5-point RANSAC per pairing, one 17-point RANSAC per candidate on their inliers, the sampling-based covariance)
 * for all candidates of one query keyframe in one call: one upload, every stage on the ctx's stream, one download.
 *   Semantics: exactly the composition of the calls above on the same inputs and seeds:
 *     1. Matches of pairing (kf1, kf2, cam1, cam2): cvb_match_hamming_batch(query = the rows of kf1, train = the rows of kf2,
 *        img_match_thres, ratio_thres); the accepted rows are kept in query order.  n_matches is its count.
 *     2. 5-point problem of the pairing, one correspondence per match: f1 = bearings[row of kf1], f2 = bearings[row of kf2],
 *        sigma1 / sigma2 likewise; solved by cvb_ransac_central_relative_pose_seeded_batch (threshold5, max_iterations5,
 *        probability) with seed5[pairing].
 *     3. 17-point problem of a candidate: its pairings in order, of each the matches in the 5-point model's inlier mask in
 *        match order, with camera indices (cam1, cam2) of the pairing; solved by cvb_ransac_noncentral_relative_pose_seeded_batch
 *        (threshold17, max_iterations17, probability) with seed[candidate] and the candidate's rigs.
 *        ASSUMPTION (the reference source is not in the tree): the inlier sets of the 5-point RANSACs feed the 17-point one
 *        in this order; the caller chooses the pairings (the reference uses six).
 *     4. Covariance: cvb_noncentral_relative_pose_covariance_seeded_batch with n_cov_samples samples (the reference's 300),
 *        ref_model = the 17-point best_model, its inlier mask and seed[candidate].
 *   So a pairing with fewer than 5 matches selects nothing and contributes no correspondence, a candidate with fewer than 17
 *   merged correspondences gets best_sample = -1 and n_valid = 0, and a keyframe with fewer than 2 rows has no accepted match.
 * Inputs:
 *   Keyframe table (every keyframe any rig uses, once): kf_ptr [n_kf+1] row offsets (kf_ptr[0] = 0) into desc [R][32] (ORB
 *   rows), bearings [R][3] (unit, in the keyframe's camera frame) and sigma [R] (the score's per-keypoint sigma).
 *   Candidates: rigs cam_ptr1 / cam_off1 / cam_rot1 and cam_ptr2 / ... as in cvb_rel_ransac_problems (rig 1 is normally the
 *   query keyframe's rig, the same for every candidate); pair_ptr [n_cand+1] the candidate's pairings, pairs [n_pairings][4] =
 *   (kf1, kf2, cam1, cam2): kf1 / kf2 index the keyframe table, cam1 / cam2 are those keyframes' cameras in the candidate's
 *   rigs.  seed5 [n_pairings], seed [n_cand] (stream 0 for the 17-point RANSAC, stream 1 for the covariance).
 * Outputs (cvb_verify_result): per pairing n_matches and the 5-point best_sample / best_model / best_count / iterations /
 * consumed; per candidate the 17-point best_sample / best_model / best_count / iterations / consumed, cov [36] and n_valid;
 * n_total, the number of matches over all pairings; and, when corr is not null and n_total <= corr_cap, the correspondence list
 * corr [n_total][5] = (pairing, row1, row2, inlier5, inlier17) in pairing then match order (row1 / row2 local to kf1 / kf2;
 * inlier17 is the 17-point inlier flag of a correspondence that entered the 17-point problem, else 0).  With n_total >
 * corr_cap only n_total is written.
 * Errors: CVB_ERR_INVALID before any launch for negative sizes, null required pointers, a decreasing kf_ptr / pair_ptr /
 * cam_ptr1 / cam_ptr2, a keyframe or camera index out of range, a rig of more than CVB_REL_MAX_CAMS cameras, a null seed5 /
 * seed, a negative n_cov_samples or corr_cap, or max_iterations5 / max_iterations17 outside [0, (INT32_MAX - 64) / 11];
 * n_cand = 0 succeeds.
 */
typedef struct cvb_verify_keyframes {
  int32_t n_kf;
  const int32_t* kf_ptr;     /* [n_kf+1] */
  const uint8_t* desc;       /* [R][32] */
  const double* bearings;    /* [R][3] */
  const double* sigma;       /* [R] */
} cvb_verify_keyframes;
typedef struct cvb_verify_candidates {
  int32_t n_cand;
  const int32_t* cam_ptr1;   /* [n_cand+1] */
  const double* cam_off1;    /* [cam_ptr1[n_cand]][3] */
  const double* cam_rot1;    /* [cam_ptr1[n_cand]][9] row-major */
  const int32_t* cam_ptr2;   /* [n_cand+1] */
  const double* cam_off2;    /* [cam_ptr2[n_cand]][3] */
  const double* cam_rot2;    /* [cam_ptr2[n_cand]][9] */
  const int32_t* pair_ptr;   /* [n_cand+1] */
  const int32_t* pairs;      /* [pair_ptr[n_cand]][4] kf1, kf2, cam1, cam2 */
} cvb_verify_candidates;
typedef struct cvb_verify_params {
  float img_match_thres, ratio_thres;
  double threshold5;
  int32_t max_iterations5;
  double threshold17;
  int32_t max_iterations17;
  double probability;
  int32_t n_cov_samples;
} cvb_verify_params;
typedef struct cvb_verify_result {
  int32_t* n_matches;        /* [n_pairings] */
  int32_t* best_sample5;     /* [n_pairings] */
  double* best_model5;       /* [n_pairings][12] */
  int32_t* best_count5;      /* [n_pairings] */
  int32_t* iterations5;      /* [n_pairings] */
  int32_t* consumed5;        /* [n_pairings] */
  int32_t* best_sample;      /* [n_cand] */
  double* best_model;        /* [n_cand][12] */
  int32_t* best_count;       /* [n_cand] */
  int32_t* iterations;       /* [n_cand] */
  int32_t* consumed;         /* [n_cand] */
  double* cov;               /* [n_cand][36] */
  int32_t* n_valid;          /* [n_cand] */
  int32_t* corr;             /* [corr_cap][5] nullable */
  int32_t corr_cap;
  int32_t n_total;           /* written */
} cvb_verify_result;
CVB_API int cvb_verify_noncentral_relative_pose_seeded_batch(cvb_ctx* ctx, const cvb_verify_keyframes* kf, const cvb_verify_candidates* cand,
                                                             const cvb_verify_params* prm, const uint64_t* seed5, const uint64_t* seed,
                                                             cvb_verify_result* r);

/*
 * The same verification with SIFT descriptors (the SIFT branch of computeNonCentralRelPose, RelNonCentralPosSolver.cpp:310-311):
 * the keyframe table holds desc [R][128] CV_32F rows, as the reference holds descriptors_add_.
 *   Semantics: exactly the composition of cvb_verify_noncentral_relative_pose_seeded_batch above on the same inputs and seeds,
 *   except step 1: the matches of pairing (kf1, kf2, cam1, cam2) are cvb_match_l2_batch(query = the rows of kf1, train = the
 *   rows of kf2 as one segment, dim = 128, img_match_thres, ratio_thres); the accepted rows are kept in query order.  Steps 2-4,
 *   the outputs and the correspondence list are those of the ORB call.
 *   Deviation from the reference: the matches are the exact brute-force L2 2-NN, where the reference calls FLANN (approximate and
 *   randomised), as cvb_match_l2_batch documents.
 * Errors: every CVB_ERR_INVALID case of cvb_verify_noncentral_relative_pose_seeded_batch; CVB_ERR_UNSUPPORTED for a descriptor
 * value that is not an integer in [0, 255] (rintf(v) == v && 0 <= v <= 255, as cv::xfeatures2d::SIFT writes them; NaN and
 * +-inf fail it).  Both before any launch: the descriptors are checked and quantised to u8 on the host while they are staged,
 * so the call uploads R x 128 bytes of them.  n_cand = 0 succeeds.
 * Usage: the thresholds are the caller's; the reference's SIFT configuration uses img_match_thres about 500 and ratio_thres 0.8.
 */
typedef struct cvb_verify_keyframes_sift {
  int32_t n_kf;
  const int32_t* kf_ptr;     /* [n_kf+1] */
  const float* desc;         /* [R][128]  CV_32F rows as the reference holds descriptors_add_ */
  const double* bearings;    /* [R][3] */
  const double* sigma;       /* [R] */
} cvb_verify_keyframes_sift;
CVB_API int cvb_verify_noncentral_relative_pose_sift_seeded_batch(cvb_ctx* ctx, const cvb_verify_keyframes_sift* kf,
                                                                  const cvb_verify_candidates* cand, const cvb_verify_params* prm,
                                                                  const uint64_t* seed5, const uint64_t* seed, cvb_verify_result* r);

/*
 * The COVINS verification of place-recognition candidates (PlaceRecognition::ComputeSE3, placerec_be.cpp:63-220, up to the
 * acceptance test: DenseMatcher landmark matching, the nmatches < matches_thres discard, Se3Solver's GP3P RANSAC,
 * FeatureMatcher::SearchBySE3 and Optimization::OptimizeRelativePose) for all candidates of one query keyframe in one call: one
 * upload, every stage on the ctx's stream, one download.
 *   Semantics: exactly the composition of the calls above on the same inputs and seeds, n = query->view.n:
 *     1. Matches: cvb_landmark_match_batch(A = query desc, skipA = !query lm_valid, B = the candidates' desc concatenated (one
 *        segment each), skipB = !lm_valid, thr, num_best).  n_matches[c] = the candidate's match count.
 *     2. RANSAC problem of candidate c: none if n_matches[c] < min_matches (placerec_be.cpp:93-99: nothing is drawn,
 *        best_sample = -1); otherwise one correspondence per match in ascending idxA: pts = cand lm_pos[idxB] (world),
 *        f = query bearings[idxA], sigma = query sigma_angle[idxA], camera = the query's T_sc (c = its translation, Rc = its
 *        rotation).  Solved by cvb_ransac_absolute_pose_seeded_batch(threshold, max_iterations, probability) with seed[c].
 *        ASSUMPTIONS (Se3Solver is not in the tree): it walks the LandmarkVector in keypoint order, and it takes world points and
 *        the body-frame camera, as cvb_ransac_absolute_pose_batch does.  DenseMatcher gives each A at most one B, so the order
 *        is well defined.
 *     3. Gate: a candidate continues iff best_sample >= 0 && best_count >= min_ransac_inliers.  Then, M the model as a 4x4,
 *        T12 = rigid_inv(M * query T_sc) * rigid_inv(cand view.Tcw) (T_c1_w times T_w_c2) and T21 = rigid_inv(T12), with
 *        rigid_inv([R|t]) = [R^T | -R^T t]; every entry of a product is its four (rigid_inv: three) products summed left to
 *        right without fused multiply-add, so a float64 restatement in the same order gives the same bits.  (The reference
 *        computes T21 with Eigen's general inverse().)  A candidate that stops gets n_found = n_corr = n_inliers = 0, zero
 *        T12 / T21 / T12_out and no entry after the RANSAC stage.
 *     4. SearchBySE3: cvb_search_by_se3_batch(kf1 = query view, kf2 = candidate view, T12, T21, search) with already1[i] = 1
 *        iff query keypoint i holds a RANSAC inlier and already2[b] = 1 iff candidate keypoint b is the idxB of one (the flat
 *        form identifies a candidate landmark's GetFeatureIndex(kf2) with the keypoint b where it sits).  The LandmarkVector
 *        after this stage: the RANSAC inliers (i -> idxB) plus the search's match12 (disjoint: the search skips already1).
 *     5. Refinement: one residual pair per LandmarkVector entry (i -> b) in ascending i whose two landmarks are valid (query
 *        lm_valid[i], cand lm_valid[b]; the reference skips a null or invalid landmark), as the shim's OptimizeRelativePose builds
 *        it: pA_c = TcwA * query lm_pos[i], pB_c = TcwB * cand lm_pos[b], TcwA = rigid_inv(query T_ws * query T_sc), TcwB =
 *        rigid_inv(cand T_ws * query T_sc) (kf1's extrinsics for both, optimization_be.cpp:643; these two are formed on the
 *        host), kpA / kpB the two keypoints, sigma = (double)(octave + 1.0f) * 2.0, each keyframe's camera; T12 as [q, t] by
 *        the shim's transform_to_pose7 (Eigen's matrix-to-quaternion branches).  Then cvb_optimize_relative_pose
 *        (th_outlier_align) gives T12_out, n_inliers and removed.  The acceptance test (n_inliers against the reference's
 *        threshold, the first accepted candidate) stays with the caller.
 * Inputs: query and cand [n_cand] (cvb_landmark_kf: the cvb_kf_view of cvb_search_by_se3_batch plus bearings [n][3] (unit,
 * camera frame), sigma_angle [n], T_ws / T_sc (row-major 4x4 body in world, camera in body) and the camera model of
 * cvb_relpose_problem; only the query's bearings / sigma_angle / T_sc are read), seed [n_cand] (stream 0 of the seeded sampler).
 * Outputs per candidate (cvb_landmark_verify_result): n_matches; the RANSAC's best_sample / best_model [12] / best_count /
 * iterations / consumed; T12 / T21 [16] as used; n_found (the search's return value); n_corr (residual pairs); T12_out [7],
 * n_inliers and solve_iterations [2] (the two ceres::Solve iteration counts).  Nullable, each [n_cand][n]: match12 (the
 * LandmarkVector handed to the refinement: the candidate keypoint of query keypoint i, or -1), stage (u8: 0 none, 1 DenseMatcher
 * match that is not a RANSAC inlier of a candidate that continues, 2 RANSAC inlier, 3 added by SearchBySE3) and removed (u8,
 * indexed by the residual r < n_corr: the reference nulls matches1[r], optimization_be.cpp:815).
 * Errors: CVB_ERR_INVALID before any launch for null required pointers, a malformed view, num_best outside 1..4, thr outside
 * (0, 257], bad search parameters or max_iterations outside [0, (INT32_MAX - 64) / 11]; CVB_ERR_UNSUPPORTED ("Unknown
 * projection type." / "Unknown distortion type.") for a camera or distortion model of the query or a candidate that
 * cvb_optimize_relative_pose does not know; n_cand = 0 succeeds.
 */
typedef struct cvb_landmark_kf {
  cvb_kf_view view;
  const double* bearings;    /* [n][3] */
  const double* sigma_angle; /* [n] */
  double T_ws[16];           /* GetPoseTws(), row-major */
  double T_sc[16];           /* GetStateExtrinsics(), row-major */
  double intr[4], dist[4];
  int32_t cam_model, dist_model;
  double xi;
} cvb_landmark_kf;
typedef struct cvb_landmark_verify_params {
  float thr;                 /* DenseMatcher distance threshold (50) */
  int32_t num_best;          /* 1..4 (4) */
  int32_t min_matches;       /* matches_thres */
  double threshold;          /* RANSAC */
  int32_t max_iterations;
  double probability;
  int32_t min_ransac_inliers;
  cvb_search_params search;
  double th_outlier_align;
} cvb_landmark_verify_params;
typedef struct cvb_landmark_verify_result {
  int32_t* n_matches;        /* [n_cand] */
  int32_t* best_sample;      /* [n_cand] */
  double* best_model;        /* [n_cand][12] */
  int32_t* best_count;       /* [n_cand] */
  int32_t* iterations;       /* [n_cand] */
  int32_t* consumed;         /* [n_cand] */
  double* T12;               /* [n_cand][16] */
  double* T21;               /* [n_cand][16] */
  int32_t* n_found;          /* [n_cand] */
  int32_t* n_corr;           /* [n_cand] */
  double* T12_out;           /* [n_cand][7] */
  int32_t* n_inliers;        /* [n_cand] */
  int32_t* solve_iterations; /* [n_cand][2] */
  int32_t* match12;          /* [n_cand][n] nullable */
  uint8_t* stage;            /* [n_cand][n] nullable */
  uint8_t* removed;          /* [n_cand][n] nullable */
} cvb_landmark_verify_result;
CVB_API int cvb_verify_landmark_candidates_seeded_batch(cvb_ctx* ctx, const cvb_landmark_kf* query, const cvb_landmark_kf* cand, int n_cand,
                                                        const cvb_landmark_verify_params* prm, const uint64_t* seed,
                                                        cvb_landmark_verify_result* r);

/*
 * Optimization::OptimizeRelativePose(kf1, kf2, matches1, T12, th2) (optimization_be.cpp:620-831): the 6-dof refinement of
 * the relative pose T12 from the matched landmark pairs, both ceres::Solve calls (5 + 5 iterations, DOGLEG, CauchyLoss(1))
 * and the outlier purge between them, in one call.  The caller (shim) flattens, per residual pair r (the reference's
 * vIndex order, :656-780): pA_c = TcwA * P3DAw, pB_c = TcwB * P3DBw with TcwB built from kf1's extrinsics as the reference
 * does (:643), the two observations and sigmas.  Camera / distortion model as in cvb_ba_problem.
 * T12 / T12_out: [qx,qy,qz,qw, x,y,z] (the reference's ceresAB).  removed [n] (nullable): 1 = residual pair r purged (:812;
 * the reference nulls matches1[r] — indexed by the RESIDUAL index, :815 — the shim reproduces that).  *n_inliers = the return
 * value: numCorrespondences - numBad, or 0 (and T12_out = T12) when fewer than 12 remain (:821-823).
 * info (nullable, 19 doubles): iterations of the two solves, number of cost entries, cost history (tests).
 */
typedef struct cvb_relpose_problem {
  int32_t n;
  const double* pA_c;      /* [n][3] */
  const double* pB_c;      /* [n][3] */
  const float* kpA;        /* [n][2] kf1->keypoints_distorted_[i] */
  const float* kpB;        /* [n][2] kf2->keypoints_distorted_[iB] */
  const double* sigmaA;    /* [n] (octave + 1) * 2 */
  const double* sigmaB;
  double intrA[4], distA[4], intrB[4], distB[4];
  int32_t cam_model_A, dist_model_A, cam_model_B, dist_model_B;
  double xiA, xiB;
  double T12[7];
} cvb_relpose_problem;
CVB_API int cvb_optimize_relative_pose(cvb_ctx* ctx, const cvb_relpose_problem* p, double th_outlier_align, double* T12_out,
                                       uint8_t* removed, int32_t* n_inliers, double* info);

/* INT-pipe microbenchmark used for the Hamming roofline denominator (SURVEY.md §8d asks the builder to
 * measure the popc issue peak): runs `iters` dependent-free XOR+POPC+ADD rounds on every SM and
 * returns giga-(32-bit popc)/s in *gpopc_per_s. */
CVB_API int cvb_microbench_popc(cvb_ctx* ctx, int iters, double* gpopc_per_s);

/* Diagnostic: issue rate (lane-instructions per clock per SM) of 32-bit and packed 2x16-bit integer min/max. out2: double[2]. */
CVB_API int cvb_microbench_minmax(cvb_ctx* ctx, double* out2);
/* Diagnostic: latency of the diagonal-tile kernel of the tiled Cholesky (K8's serial chain), see cholesky.cu.
 * phase_cycles may be NULL, else int64[10]. */
CVB_API int cvb_microbench_potrf(cvb_ctx* ctx, int reps, double* us_per_tile, int64_t* phase_cycles);
/* Diagnostic: single-warp latencies (cycles per dependent DFMA, rsqrt, shuffle, ...), see microbench.cu. out8: double[8]. */
CVB_API int cvb_microbench_latency(cvb_ctx* ctx, double* out8);
/* Diagnostic: the group all-reduce of cvb_group_create alone.  in [n][count] (host): rank r's buffer; out [n][count] (host):
 * what each rank holds afterwards (the rank-order sum, on every rank).  One host thread per rank, as in the group drivers. */
CVB_API int cvb_group_allreduce_diag(cvb_group* g, const double* in, size_t count, double* out);

/* diagnostic: solve A x = b (host SPD matrix, row-major n x n) with the BA factorisation (tiled FP64 Cholesky on
 * DMMA); *factor_ms (nullable) receives the device time of the factorisation. */
CVB_API int cvb_dense_cholesky_solve(cvb_ctx* ctx, const double* A, int n, const double* b, double* x,
                                     double* factor_ms);

/* ------------------------------------------------------------------------------------------------
 * Optimisation half (SURVEY.md §8a O1-O2): flat problem format (SURVEY.md Appendix B)
 * ---------------------------------------------------------------------------------------------- */

/*
 * The pointer graph the reference walks (Map → Keyframe / Landmark / LoopConstraint containers,
 * optimization_be.cpp:75-254, 307-557, 846-1021) flattened to SoA arrays in the canonical orders of SURVEY §8c:
 * keyframes by (client id, kf id), landmarks by id, the observations of a landmark sorted by keyframe index.
 * All arrays are caller-owned host memory; the solver never keeps the pointers after a call returns.
 */
typedef struct cvb_ba_problem {
  int32_t K, L, n_obs, n_imu, n_edge, n_cam;
  const double* pose;         /* [K][7]  qx,qy,qz,qw,x,y,z = T_ws (keyframe_base.cpp:486-499) */
  const double* speedbias;    /* [K][9]  v_w, b_a, b_g (keyframe_base.cpp:512-521); may be NULL when visual_only */
  const uint8_t* pose_const;  /* [K]     1 = SetParameterBlockConstant (gauge KF, loaded / GBA-fixed KFs) */
  const int32_t* cam_of_kf;   /* [K]     calibration index, NULL = 0 */
  const double* extr;         /* [n_cam][7] T_sc (constant block, optimization_be.cpp:91-92) */
  const double* intr;         /* [n_cam][4] fx, fy, cx, cy (constant) */
  const double* dist;         /* [n_cam][4] distortion coefficients (constant); meaning per dist_model, default radtan k1, k2, p1, p2 */
  const double* lm;           /* [L][3]  world position */
  const int32_t* lm_obs_ptr;  /* [L+1]   CSR by landmark */
  const int32_t* obs_kf;      /* [n_obs] keyframe index */
  const float* obs_uv;        /* [n_obs][2] distorted keypoint (keypoints_distorted_, float) */
  const double* obs_sigma;    /* [n_obs] (octave + 1) * 2 (optimization_be.cpp:183-184) */
  const uint8_t* obs_skip;    /* [n_obs] nullable; 1 = observation not in the problem */
  /* IMU factor f links predecessor imu_i[f] → imu_j[f] with KF j's preintegration (optimization_be.cpp:119-143) */
  const int32_t* imu_i;
  const int32_t* imu_j;
  const int32_t* imu_ptr;     /* [n_imu+1] sample ranges */
  const double* imu_dt;       /* [samples] */
  const double* imu_acc;      /* [samples][3] */
  const double* imu_gyr;      /* [samples][3] */
  const double* imu_acc0;     /* [n_imu][3] first reading (keyframe_be.cpp:187) */
  const double* imu_gyr0;     /* [n_imu][3] */
  const double* imu_noise;    /* [5] sigma_a_c, sigma_g_c, sigma_aw_c, sigma_gw_c, g */
  /* 6-DoF between edges: loop constraints (GBA) or loop + successor + neighbour edges (PGO) */
  const int32_t* edge_i;
  const int32_t* edge_j;
  const double* edge_q;         /* [n_edge][4] measured q_12 (x,y,z,w) */
  const double* edge_t;         /* [n_edge][3] measured t_12 */
  const double* edge_sqrt_info; /* [n_edge][36] row-major, rotation rows first (optimization_be.cpp:896-897) */
  const uint8_t* edge_robust;   /* [n_edge] 1 = CauchyLoss(cauchy_edge) on this edge; NULL = none */
  /* camera / distortion model per calibration: the template arguments of GlobalEuclideanReprError<Camera, Distortion>
   * (optimization_be.cpp:186-231).  NULL = pinhole / radtan for every camera (what ORB-SLAM3 agents send). */
  const int32_t* cam_model;     /* [n_cam] 0 = aslam::PinholeCamera, 1 = aslam::UnifiedProjectionCamera */
  const int32_t* dist_model;    /* [n_cam] 0 = RadTan (k1,k2,p1,p2), 1 = Equidistant (k1..k4), 2 = Fisheye / FOV (w) — in `dist` */
  const double* cam_xi;         /* [n_cam] mirror parameter xi of the unified model (its intrinsics are [xi, fu, fv, cu, cv]) */
} cvb_ba_problem;

typedef struct cvb_ba_options {
  int32_t max_iterations;  /* solver_options.max_num_iterations */
  int32_t visual_only;     /* no speed-bias blocks, no IMU factors (optimization_be.cpp:90,117) */
  double cauchy_reproj;    /* CauchyLoss parameter on reprojection residuals (1.0); <= 0: none */
  double cauchy_edge;      /* CauchyLoss parameter on robust edges (GBA 1.0; PGO robust_loss_th 0.5) */
  int32_t rank, world;     /* landmark-block sharding across GPUs; world <= 1: single GPU */
} cvb_ba_options;

typedef struct cvb_ba_result {
  double* pose;            /* [K][7] out (nullable) */
  double* speedbias;       /* [K][9] out (nullable) */
  double* lm;              /* [L][3] out (nullable); landmarks not in the problem / owned by another rank keep the input */
  int32_t* lm_owner;       /* [L] out (nullable): rank that optimised the landmark, -1 = not in the problem */
  double* cost_history;    /* [cost_history_cap] out (nullable): cost after iteration 0,1,2,... */
  uint8_t* step_status;    /* [cost_history_cap] out (nullable): 1 accepted, 2 rejected, 3 invalid, 4 converged */
  int32_t cost_history_cap;
  int32_t n_cost_history;
  int32_t iterations;      /* successful + unsuccessful steps, as Ceres counts them */
  int32_t termination;     /* 0 NO_CONVERGENCE (iteration limit), 1 gradient, 2 parameter, 3 function tolerance, 4 failure */
  double initial_cost, final_cost;
} cvb_ba_result;

typedef struct cvb_gba_options {
  int32_t iterations_limit;  /* covins_params::opt::gba_iteration_limit (10) */
  int32_t visual_only;
  int32_t outlier_removal;   /* round 1 of optimization_be.cpp:62-291 */
  double th_outlier;         /* th_gba_outlier_global (0.92) */
} cvb_gba_options;

/* in-place sum over all ranks of `count` doubles at device pointer `ptr`, enqueued on `stream` */
typedef int (*cvb_allreduce_fn)(void* user, void* ptr, size_t count, void* stream);

typedef struct cvb_ba cvb_ba;

/* Replaces the ceres::Problem + ceres::Solve of one optimisation (SPARSE_SCHUR + DOGLEG, optimization_be.cpp:257-265,
 * 560-567, 1024-1031).  create = problem construction + iteration 0; iterate = that many trust-region iterations. */
CVB_API int cvb_ba_create(cvb_ctx* ctx, const cvb_ba_problem* p, const cvb_ba_options* o, cvb_ba** out);
/* Multi-GPU (o->world > 1; one process per GPU, the same problem on every rank, landmark blocks sharded by rank): the call
 * sequence is  cvb_ba_create → cvb_ba_set_allreduce → [cvb_ba_enable_p2p] → cvb_ba_restart → cvb_ba_iterate.
 * cvb_ba_create runs iteration 0 on the rank-local partial sums only; cvb_ba_restart repeats it with the collective
 * installed (and returns to the state the problem was created with), so it is REQUIRED before iterating when world > 1.
 * cvb_ba_enable_p2p (optional, all ranks on one NVLink node): maps every rank's reduced camera system through CUDA IPC;
 * the reduced normal equations are then reduce-scattered by peer pull onto tile-column owners and the factorisation is
 * distributed by tile columns (panels handed over through peer memory).  CVB_ERR_UNSUPPORTED → not available, the
 * all-reduce of the packed tiles + replicated factorisation stay in use. */
CVB_API int cvb_ba_set_allreduce(cvb_ba* h, cvb_allreduce_fn fn, void* user);
CVB_API int cvb_ba_enable_p2p(cvb_ba* h);
/* back to the state the problem was created with (bit-identical repeat of the solve), then iteration 0 */
CVB_API int cvb_ba_restart(cvb_ba* h);
CVB_API int cvb_ba_iterate(cvb_ba* h, int max_iterations, int* iterations_done);
CVB_API int cvb_ba_result_get(cvb_ba* h, const cvb_ba_problem* p, cvb_ba_result* r);
/* problem.Evaluate(residual_ids) of optimization_be.cpp:270-274: loss-corrected reprojection residual norm per
 * observation at the current state (-1 for observations that are not in the problem) */
CVB_API int cvb_ba_reproj_norms(cvb_ba* h, double* norms, int n_obs);
/* diagnostic: internal vector in canonical order [K x (pose 6 [+ speed-bias 9]) | landmarks 3 each]: 0 Jacobi scale, 1 column sq-norms, 2 dogleg
 * diagonal, 3 gradient, 4 gradient/diag, 5 Gauss-Newton step (scaled), 6 trust-region step, 7 linear-solve x, 8 reduced rhs */
CVB_API int cvb_ba_debug_vector(cvb_ba* h, int which, double* out, int64_t cap, int64_t* n_cam, int64_t* n_total);
/* accumulated device time (ms, CUDA events) per phase: [0] linearise, [1] block build + Schur, [2] Cholesky factor,
 * [3] triangular solves + back-substitution, [4] dogleg / J*step / Plus / candidate cost; [5] dense-equivalent
 * factorisation flops.  reset != 0 clears the counters. */
CVB_API int cvb_ba_timing(cvb_ba* h, double out[6], int reset);
CVB_API int cvb_ba_destroy(cvb_ba* h);
CVB_API int cvb_ba_solve(cvb_ctx* ctx, const cvb_ba_problem* p, const cvb_ba_options* o, cvb_ba_result* r);

/* Optimization::GlobalBundleAdjustment(map, iterations_limit, -, visual_only, outlier_removal, -)
 * (optimization_be.cpp:56-618) on the flat problem; obs_removed [n_obs] (nullable) marks the observations round 1
 * erases from the map (:285-287).  Edges are the map's loop constraints with sqrt_info diag(100 I3, 1e4 I3) (:238-240). */
CVB_API int cvb_gba(cvb_ctx* ctx, const cvb_ba_problem* p, const cvb_gba_options* g, cvb_ba_result* r,
                    uint8_t* obs_removed);

/*
 * Multi-GPU from one process: a rank group over contexts of this process (rank r = ctxs[r]), for a server whose bundle
 * adjustment runs on one of its own threads (no torchrun, no NCCL, no CUDA IPC).
 *   cvb_group_create: 1 <= n <= 16 (the peer path's limit), no NULL context, no context twice -> else CVB_ERR_INVALID before
 *   any device work.  Several contexts may be on one device (their ranks then share it).  For every pair of distinct devices
 *   peer access is enabled both ways (with access to the peer's stream-ordered pool; process-wide, it stays enabled after
 *   cvb_group_destroy); a pair without peer access (cudaDeviceCanAccessPeer) -> CVB_ERR_UNSUPPORTED naming the pair.
 *   Messages go to ctxs[0].
 *   Group all-reduce (what the drivers install through cvb_allreduce_fn): a host rendezvous of the n rank threads, after which
 *   each rank's stream waits on events the others recorded after producing their buffers; a kernel on each rank reads the n
 *   buffers (same device or peer access) and adds them in RANK ORDER 0..n-1 into rank-local scratch; a second rendezvous
 *   with events, so that no rank overwrites a buffer a peer still reads, then the copy back.  Every rank holds bit-identical
 *   sums, the same from run to run.  Buffers go in chunks of CVB_GROUP_ALLREDUCE_CHUNK doubles (bounded scratch: one chunk
 *   per rank).
 *   Failures: every rendezvous waits at most 20 s (the distributed factorisation's peer-flag bound).  A rank that fails marks
 *   the group failed; the other ranks then return an error from their next rendezvous instead of blocking.  The drivers
 *   join every rank thread and synchronise every rank's streams before they return: no host thread and no device work
 *   outlives a call.  The error is returned with "rank r: <message of the first failure>" on ctxs[0].
 *   Calls on one group are serialised (a second concurrent call waits); the group's contexts must not be used by other
 *   threads during a group call.
 * cvb_ba_solve_group / cvb_gba_group: cvb_ba_solve / cvb_gba sharded over the group (landmark blocks c % n, o->rank and
 * o->world are ignored); one host thread per rank runs create -> group all-reduce -> [peer path] -> restart -> iterate.
 *   peer_path != 0: the reduced camera system is reduce-scattered by peer pull and factorised by tile columns (as
 *   cvb_ba_enable_p2p, with the peers' buffers handed over inside the process); 0: all-reduce of the packed tiles and a
 *   replicated factorisation.  The peer path needs a device per rank: a group in which two ranks share a device refuses
 *   peer_path != 0 with CVB_ERR_UNSUPPORTED before any thread or launch.  The in-process peer path has not been verified
 *   against world 1 on several devices; the C++ shim and the Python wrappers leave it off by default.
 *   cvb_gba_group: cvb_gba's two rounds; each observation's round-1 norm comes from the rank that owns its landmark, and the
 *   outlier set is computed once, the same obs_skip for every rank in round 2.
 *   Result: poses, speed-biases, cost history, steps, iterations and termination of rank 0, each landmark from its owner,
 *   lm_owner filled in.  Every rank's poses, speed-biases and cost history must be bitwise equal -> else CVB_ERR_NUMERIC.
 *   A group of one is bitwise equal to cvb_ba_solve / cvb_gba; larger groups equal them up to summation order.
 *   A malformed problem is refused as cvb_ba_create refuses it, before any thread or launch.
 */
#define CVB_GROUP_ALLREDUCE_CHUNK (1 << 21)
CVB_API int cvb_group_create(cvb_ctx* const* ctxs, int n, cvb_group** out);
CVB_API int cvb_group_destroy(cvb_group* g);
CVB_API int cvb_ba_solve_group(cvb_group* g, const cvb_ba_problem* p, const cvb_ba_options* o, int peer_path, cvb_ba_result* r);
CVB_API int cvb_gba_group(cvb_group* g, const cvb_ba_problem* p, const cvb_gba_options* gba, int peer_path, cvb_ba_result* r,
                          uint8_t* obs_removed);

/*
 * The resident descriptor database (cvb_db_*) with its keyframes spread over the ranks of a group: every request scans each
 * rank's share of the map on that rank, concurrently.  The operations are those of cvb_db with the same argument meaning;
 * global keyframe indices, cvb_db_group_remove's index shift and every output (n_matches [n_kf], the matches compacted by
 * (global keyframe, queryIdx), cap truncation, *n_total) are bit-identical to those of ONE cvb_db that received the same
 * sequence of appends and removes.
 *   Placement: each appended keyframe goes to the rank that holds the fewest rows at that moment, the lowest rank winning a
 *   tie; the keyframes of one call are dealt one by one, in order.  Each rank keeps its keyframes in global order in an
 *   ordinary cvb_db on its context; the host keeps the global -> (rank, local index) table and updates it on remove.
 *   cvb_db_group_size: n_kf, n_rows as cvb_db_size; rows_per_rank [group size] (nullable) = the rows each rank holds.
 *   A request: a SIFT query is checked and quantised once into rank 0's pinned staging before any device work and copied to
 *   every rank; each rank holding keyframes runs the filtered 2-NN against them on its stream and compacts its accepted
 *   matches (at most cap); rank 0's stream waits on the ranks' events and a gather on rank 0 reads every rank's counts and
 *   compacted lists (same device, or over the peer access cvb_group_create enabled) into global keyframe order, so only
 *   the accepted matches cross between devices; one copy of counts, total and min(total, cap) matches to the host.  The
 *   calling thread enqueues everything; no host threads.
 *   Refusals (before any rank is touched, every rank unchanged): a call of the other row kind -> CVB_ERR_INVALID; a SIFT
 *   value that is not an integer in [0,255] -> CVB_ERR_UNSUPPORTED; a bad index, bad counts or bad arguments ->
 *   CVB_ERR_INVALID.  Messages go to the group's ctxs[0]; a CUDA failure is reported there as "rank r: <message>" and leaves
 *   the database undefined (destroy it).
 *   Concurrency: the calls of a database are serialised on the group (cvb_group_create's call lock), with each other and
 *   with the group's bundle-adjustment calls.  Give the database a group of its own (over the same devices if you like):
 *   on a group that also runs cvb_gba_group, a place-recognition request waits for the whole GBA.  Destroy the database
 *   before its group and the group's contexts.
 */
typedef struct cvb_db_group cvb_db_group;
CVB_API int cvb_db_group_create(cvb_group* g, int desc_bytes, cvb_db_group** out);   /* 32 ORB, 128 SIFT, else CVB_ERR_UNSUPPORTED */
CVB_API int cvb_db_group_destroy(cvb_db_group* db);
CVB_API int cvb_db_group_append(cvb_db_group* db, const uint8_t* rows, const int32_t* rows_per_kf, int n_kf);
CVB_API int cvb_db_group_append_sift(cvb_db_group* db, const float* rows, const int32_t* rows_per_kf, int n_kf);
CVB_API int cvb_db_group_remove(cvb_db_group* db, int kf_index);   /* cvb_db_group_remove_batch of one index */
/*
 * cvb_db_remove_batch for the group: same index meaning, result and refusals (before any rank is touched).  The removals
 * are dealt to the ranks that hold them through the global -> (rank, local index) table; each rank that loses keyframes
 * compacts its share as cvb_db_remove_batch does, on its own stream (the calling thread enqueues every rank's work, then
 * waits for each), and the table is rebuilt once.  Keyframes never move between ranks; rows_per_rank and the placement of
 * later appends follow from the new state.  A CUDA failure is reported as "rank r: <message>" on ctxs[0] and leaves the
 * database undefined.
 */
CVB_API int cvb_db_group_remove_batch(cvb_db_group* db, const int32_t* kf_index, int n);
CVB_API int cvb_db_group_size(const cvb_db_group* db, int32_t* n_kf, int64_t* n_rows, int64_t* rows_per_rank);
CVB_API int cvb_db_group_match_hamming(cvb_db_group* db, const uint8_t* q, int nq, float thr, float ratio, int32_t* n_matches,
                                       int32_t* m_kf, int32_t* m_query, int32_t* m_train, float* m_dist, int cap, int32_t* n_total);
CVB_API int cvb_db_group_match_l2(cvb_db_group* db, const float* q, int nq, float thr, float ratio, int32_t* n_matches,
                                  int32_t* m_kf, int32_t* m_query, int32_t* m_train, float* m_dist, int cap, int32_t* n_total);
/*
 * cvb_db_merge for two databases of the same group: each rank merges src's share into dst's share on its own device
 * (keyframes never move between devices), and the global -> (rank, local index) table takes src's entries after dst's.
 * The outputs are placement-independent, so the merged database is bit-identical to one cvb_db that received dst's
 * keyframes and then src's.  Later appends follow the fewest-rows rule from the merged state (each rank's rows are the
 * sum of both shares).  Refusals before any rank is touched: dst == src or different row kinds -> CVB_ERR_INVALID; another
 * group -> CVB_ERR_UNSUPPORTED; more than 2^31 rows together -> CVB_ERR_INVALID.  A CUDA failure is reported as
 * "rank r: <message>" on ctxs[0] and leaves dst undefined.
 */
CVB_API int cvb_db_group_merge(cvb_db_group* dst, const cvb_db_group* src);

/* ------------------------------------------------------------------------------------------------
 * Map maintenance (SURVEY.md §8f rank 4)
 * ---------------------------------------------------------------------------------------------- */

/*
 * Replaces Keyframe::UpdateCovisibilityConnections (keyframe_be.cpp:559-608) called for every keyframe of a map (after a
 * merge, a map load, or a GBA round that erased observations): the whole covisibility graph in one call, on the
 * landmark / observation CSR of cvb_ba_problem (lm_obs_ptr [L+1], obs_kf, obs_skip).  All pointers are host memory.
 * The reference's result depends on the order the keyframes were updated in and, for equal weights, on pointer order; this
 * call returns the canonical, order-independent graph:
 *   1. an observation takes part iff obs_skip is NULL or 0 for it, and its landmark iff lm_valid is NULL or 1 for it;
 *   2. w(i,j), i != j = the number of participating landmarks observed by both keyframes.  A keyframe appears at most
 *      once per landmark (a duplicate is CVB_ERR_INVALID);
 *   3. i and j are connected iff w(i,j) >= min_weight, or i has no neighbour reaching min_weight, w(i,j) > 0 and j is i's
 *      best neighbour (largest weight, lowest index among equals), or the same with i and j exchanged (the reference's
 *      "keep the single best one" with AddConnectedKeyframe on the other side);
 *   4. keyframe i's list, nbr_kf / nbr_w [nbr_ptr[i], nbr_ptr[i+1]), holds its connected keyframes by weight descending,
 *      then keyframe index ascending: GetConnectedKeyframes order, its first N entries GetBestCovisibilityKeyFrames(N).
 * min_weight >= 1 (the reference hard-codes 15).  nbr_ptr [K+1] and *n_total (= nbr_ptr[K]) are always written; nbr_kf and
 * nbr_w [cap] only when *n_total <= cap (call again with a larger cap otherwise); both may be NULL with cap == 0 to ask
 * for the size.  K == 0 or no observations: an empty graph.  Integer arithmetic only: the output is bit-identical from
 * run to run.  A pair or edge count beyond the 31-bit index range is CVB_ERR_UNSUPPORTED with the count in the message.
 */
CVB_API int cvb_covisibility(cvb_ctx* ctx, int K, int L, const int32_t* lm_obs_ptr, const int32_t* obs_kf,
                             const uint8_t* obs_skip /*nullable*/, const uint8_t* lm_valid /*nullable*/, int min_weight,
                             int32_t* nbr_ptr /*[K+1]*/, int32_t* nbr_kf, int32_t* nbr_w, int64_t cap, int64_t* n_total);

/*
 * Redundancy pruning of Map::Clean (map_be.cpp:745-811, behind the covins_prunemap service): which keyframes the
 * reference's sequential culling pass removes, in one call.  ASSUMPTION (parity unpinned beyond the source): the rule is
 * restated from the ORB-SLAM3 KeyFrameCulling lineage that pass follows (oracle/prune_oracle.c carries the same text).
 * Inputs: the landmark / observation CSR of cvb_ba_problem (lm_obs_ptr [L+1], obs_kf, nullable obs_skip / lm_valid with
 * rule 1 of cvb_covisibility), obs_octave [n_obs] (the keypoint's octave, obs_sigma / 2 - 1 of the GBA problem),
 * kf_pred [K] (the keyframe's predecessor in its agent's chain, -1 if none; kf_pred[k] < k, at most one successor per
 * keyframe), kf_time [K], kf_protect [K] (1 = never culled).  All pointers are host memory.
 * For a set C of keyframes culled so far:
 *   Λ(k)      k's participating landmarks, fixed for the whole pass (landmarks are not erased); n(k) = |Λ(k)|;
 *   red_C(k)  the number of l in Λ(k) observed by at least th_obs keyframes k' ∉ C, k' != k, with
 *             octave(k', l) <= octave(k, l) + 1;
 *   pred_C(k) k's nearest ancestor in its chain that is not in C; succ(k) its original successor.
 * The pass: for k = 0 .. K-1 in index order, C <- C ∪ {k} iff k is not protected, n(k) > 0,
 * (double)red_C(k) > th_red * (double)n(k), pred_C(k) and succ(k) both exist, and
 * kf_time[succ(k)] - kf_time[pred_C(k)] <= max_time_dist.  culled [K] (uint8) = 1 for the members of the final C.
 * Adding keyframes to C only lowers red_C and moves pred_C earlier, so the call evaluates it in parallel rounds whose commit
 * rule reproduces the sequential pass exactly; *n_rounds (nullable) receives their number.  Integer arithmetic except the
 * comparison against th_red and the time difference: the output is bit-identical from run to run.  CVB_ERR_INVALID, before
 * any launch: a duplicate observer, an octave outside [0, num_octaves), kf_pred[k] >= k or < -1, two successors of one
 * keyframe, th_red NaN or outside [0, 1], max_time_dist not > 0, th_obs < 1, num_octaves outside [1, 64], a decreasing
 * lm_obs_ptr.  K == 0: nothing is culled.
 */
CVB_API int cvb_redundant_keyframes(cvb_ctx* ctx, int K, int L, const int32_t* lm_obs_ptr, const int32_t* obs_kf,
                                    const int32_t* obs_octave, const uint8_t* obs_skip /*nullable*/,
                                    const uint8_t* lm_valid /*nullable*/, const int32_t* kf_pred, const double* kf_time,
                                    const uint8_t* kf_protect, double th_red, double max_time_dist, int th_obs,
                                    int num_octaves, uint8_t* culled /*[K]*/, int32_t* n_rounds /*nullable*/);

/*
 * Landmark outlier removal of Map::Clean (map_be.cpp:448-454, 698-743): which observations of a map are outliers and which
 * landmarks lose too many observers, in one call.  ASSUMPTION (parity unpinned beyond the source): the reference does not
 * record its rule; this call defines a canonical one from behaviour the library already pins (oracle/lm_outliers.py
 * carries the same text).  It reads only the map part of p: K, L, n_obs, n_cam, pose, cam_of_kf, extr, intr, dist,
 * cam_model, dist_model, cam_xi, lm, lm_obs_ptr, obs_kf, obs_uv, obs_sigma, obs_skip (no speed-biases, IMU data or edges).
 * All pointers are host memory.
 *   1. an observation takes part iff obs_skip is NULL or 0 for it, and its landmark iff lm_valid is NULL or non-zero for it
 *      (rule 1 of cvb_covisibility);
 *   2. norm of a participating observation = what cvb_ba_reproj_norms reports for it at the same state with
 *      cvb_ba_options.cauchy_reproj = cauchy, bit for bit: r = the reprojection residual of cvb_ba_problem, s = r.r,
 *      norm = sqrt(s) * sqrt(1 / (1 + s / cauchy^2)); cauchy <= 0 gives the plain |r|.  This is the test of
 *      optimization_be.cpp:270-290;
 *   3. obs_outlier [n_obs] = 2 if the point is not projectable in the keyframe's camera (behind the camera, or outside the
 *      unified model's field of view: the residual the bundle adjustment defines as zero, so its own purge never removes
 *      the observation; this clause follows the ORB-SLAM isDepthPositive lineage and is pure assumption), else 1 if
 *      norm > th_outlier (th_gba_outlier_global, 0.92), else 0; 0 for every observation that does not take part;
 *   4. lm_erase [L] = 1 iff the landmark takes part and fewer than min_obs of its participating observations have
 *      obs_outlier == 0 (min_obs 2: the bundle adjustment's own inclusion rule, optimization_be.cpp:158-171, 438-453).  A
 *      landmark that does not take part is never erased;
 *   5. norms [n_obs] (nullable) = the norm of each participating observation (0 for a non-projectable one), -1 for the
 *      others, as cvb_ba_reproj_norms reports an observation outside its problem.
 * *n_obs_outlier = the number of non-zero obs_outlier, *n_lm_erased = the number of erased landmarks.  Integer decisions on
 * fixed-order FP64 arithmetic, no floating-point atomics: the output is bit-identical from run to run.
 * CVB_ERR_INVALID, before any launch: a NULL required pointer, a negative size, lm_obs_ptr[0] != 0, a decreasing
 * lm_obs_ptr or lm_obs_ptr[L] != n_obs, obs_kf outside [0, K), cam_of_kf outside [0, n_cam), an obs_sigma that is not
 * positive and finite, th_outlier NaN or not > 0, cauchy not finite, min_obs < 1.  An unknown camera or distortion model:
 * CVB_ERR_UNSUPPORTED with cvb_ba_create's messages.  K == 0, L == 0 or n_obs == 0: nothing to judge, nothing flagged
 * (norms -1).
 */
CVB_API int cvb_landmark_outliers(cvb_ctx* ctx, const cvb_ba_problem* p, const uint8_t* lm_valid /*nullable*/,
                                  double th_outlier, double cauchy, int min_obs,
                                  uint8_t* obs_outlier /*[n_obs]*/, uint8_t* lm_erase /*[L]*/, double* norms /*nullable*/,
                                  int64_t* n_obs_outlier, int32_t* n_lm_erased);

/*
 * The rigid transform of the merge constructor Map(map_target, map_tofuse, T) (map_be.cpp:334-381, the loop at :365-380),
 * reached from MapManager::PerformMerge (map_be.cpp:192-244): the fused map's keyframes and landmarks moved into the
 * target map's world frame in one call.  T = T_wtarget_wtofuse, row-major 4x4 [R t; 0 0 0 1].  All pointers are host memory.
 *   keyframe k (selected iff kf_sel is NULL or kf_sel[k] != 0): T_ws[k] <- T * T_ws[k] (all 16 entries, row-major [K][16]),
 *     vel[k] <- R * vel[k] (vel [K][3], nullable: then no velocity is touched);
 *   landmark l (selected iff lm_sel is NULL or lm_sel[l] != 0): lm_pos[l] <- R * lm_pos[l] + t;
 *   unselected entries are left bit for bit as they were.
 * Every output entry is its products summed left to right without fused multiply-add: (T[r][0] X[0][c] + T[r][1] X[1][c])
 * + T[r][2] X[2][c] + T[r][3] X[3][c] for a pose, ((R[r][0] v0 + R[r][1] v1) + R[r][2] v2) (+ t[r]) for a velocity and a
 * position, so a float64 restatement in the same order (oracle/merge.py) gives the same bits.  Poses stay 4x4 matrices
 * as the containers hold them: a quaternion round trip would add rounding the reference does not have.
 * ASSUMPTIONS (the merge constructor is not in this tree; the rule is restated from SURVEY.md's citations, and
 * oracle/merge.py carries the same text): the fused map's T_ws and velocity are transformed and its IMU biases are not;
 * T_ws_vio_ is left unchanged (the pose graph reads it only as relative transforms between keyframes of one agent,
 * opt.cpp:947-1021, which a common left factor does not change); landmark positions are transformed.  Loop constraints,
 * ids and the union of the two maps are host container work (covins_b200::MergeMaps).
 * One launch whatever the map's size, a grid-stride over K + L, with one upload and one download per array.
 * CVB_ERR_INVALID, before any launch: T not rigid (an entry not finite, |R^T R - I| > 1e-9 in any entry, det R <= 0, or a
 * last row other than [0 0 0 1]), a negative size, a NULL T, or a NULL T_ws / lm_pos with K / L > 0.  K + L == 0: nothing
 * to do, no launch.
 */
CVB_API int cvb_map_rigid_transform(cvb_ctx* ctx, const double T[16], int K, double* T_ws /*[K][16] in/out*/,
                                    double* vel /*[K][3] in/out, nullable*/, int L, double* lm_pos /*[L][3] in/out*/,
                                    const uint8_t* kf_sel /*[K], nullable*/, const uint8_t* lm_sel /*[L], nullable*/);

/*
 * Optimization::PoseGraphOptimization (optimization_be.cpp:833-1086) on a flattened map in one call: the edges of the
 * keyframe chain, the solve and the write-back of velocities and landmarks.  All arrays are host memory, keyframes in the
 * canonical order (the valid keyframes of the map, id-sorted), poses row-major 4x4 as in cvb_map_rigid_transform.
 * Keyframe indices: kf_pred / kf_succ / lm_ref hold an index in [0, K), -1 for none, -2 for a keyframe that exists but is not
 * among the K (an invalid one).
 * EDGES, in this order (the shim's rule before this call, :886-1021):
 *   1. loop l = 0..n_loop-1 between loop_i[l] and loop_j[l], measurement (loop_q[l], loop_t[l]), sqrt_info chol(cov^-1)^T of
 *      loop_cov[l] (COVINS_G, :922-923) or S1 when loop_cov is NULL (COVINS), Cauchy(robust_loss_th) iff use_robust_loss;
 *   2. per keyframe k in order with kf_succ[k] >= 0: (k, kf_succ[k]) with S1 (:947-972);
 *   3. when use_nbr_kfs, per keyframe k in order: the walk through kf_pred j = 1..5 steps while int(kf_id[k]) - j > 0, the
 *      j-th keyframe reached with S1, S23, S23, S45, S45 (:976-1021).
 *   An ordered pair already inserted by 2. or 3. is skipped; loops are not in that set.  Steps 2. and 3. measure
 *   transform_to_pose7(rel_transform(T_ws_vio[i], T_ws_vio[j])).  S1 = diag(wt_kf_r x3, wt_kf_t x3) * wt_kf_n1, S23 = S1 /
 *   wt_kf_n23, S45 = S1 / wt_kf_n45 (:896-903).  Only loops are robust.
 * SOLVE: start poses transform_to_pose7(T_ws_init, or T_ws when NULL) (:854-868), pose_const as given, the bundle
 *   adjustment engine with visual_only, no reprojection loss, cauchy_edge = robust_loss_th, iteration_limit iterations.
 * WRITE-BACK, with Tu = T_ws[k] (the pose before the call) and Tc = pose7_to_transform(solved pose) (:1033-1083):
 *   T_ws_out[k] = Tc (what the shim passes to SetPoseTws);
 *   velocity_out[k][r] = sum_c (sum_x Tc(r,x) Tu(c,x)) velocity[k][c], each sum from 0 in that loop order (:1046-1047);
 *   landmark l with lm_ref[l] = k >= 0: ps = Tu^T (p - t_u) (sums from 0), lm_out[l][r] = ((Tc(r,0) ps0 + Tc(r,1) ps1) +
 *   Tc(r,2) ps2) + Tc(r,3), lm_erase[l] = 0; lm_ref -1: lm_erase = lm_has_obs[l]; lm_ref -2: lm_erase = 1; a landmark without
 *   a reference keyframe keeps its input bits in lm_out.
 *   Products and sums are rounded one by one in the order stated (include/covins_b200_pose.h), so oracle/pgo.py gives the
 *   same bits.
 * Device work: one launch for the start poses and the edge measurements (straight into the solver's arrays; the edge
 * topology is built on the host), the solve, one launch for the write-back over K + L items, one download of all outputs.
 * CVB_ERR_INVALID, before any launch: a NULL required pointer, K < 1, a negative n_loop / L, an index outside its range, a
 * loop with loop_i == loop_j, a successor that is not among the K (-2), a neighbour walk that needs a predecessor that is
 * absent (-1) or not among the K (-2), a non-finite entry in T_ws / T_ws_init / T_ws_vio, iteration_limit < 0.  A loop
 * covariance that is not positive definite sets r->bad_loop to that loop (else -1) and is refused the same way, naming it.
 */
typedef struct cvb_pgo_problem {
  int32_t K;
  const double* T_ws;       /* [K][16] the pose before the call (the write-back's "uncorrected" pose) */
  const double* T_ws_init;  /* [K][16] nullable: the start values of the solve (corrected_poses); NULL = T_ws */
  const double* T_ws_vio;   /* [K][16] */
  const int32_t* kf_pred;   /* [K] */
  const int32_t* kf_succ;   /* [K] */
  const int32_t* kf_id;     /* [K] id_.first */
  const uint8_t* pose_const;/* [K] */
  const double* velocity;   /* [K][3] nullable: then velocity_out is not written */
  int32_t n_loop;
  const int32_t* loop_i;    /* [n_loop] */
  const int32_t* loop_j;
  const double* loop_q;     /* [n_loop][4] x,y,z,w of T_s1_s2 */
  const double* loop_t;     /* [n_loop][3] */
  const double* loop_cov;   /* [n_loop][36] nullable: NULL = COVINS weights */
  int32_t L;
  const double* lm_pos;     /* [L][3] */
  const int32_t* lm_ref;    /* [L] reference keyframe */
  const uint8_t* lm_has_obs;/* [L] */
} cvb_pgo_problem;

typedef struct cvb_pgo_options {
  double wt_kf_r, wt_kf_t, wt_kf_n1, wt_kf_n23, wt_kf_n45;   /* 10, 1, 10, 2, 3 */
  int32_t use_nbr_kfs;       /* 1 */
  int32_t use_robust_loss;   /* 1 */
  double robust_loss_th;     /* 0.5 */
  int32_t iteration_limit;   /* pgo_iteration_limit 10 */
} cvb_pgo_options;

typedef struct cvb_pgo_result {
  double* T_ws_out;         /* [K][16] out */
  double* velocity_out;     /* [K][3] out; required when problem velocity is given */
  double* lm_out;           /* [L][3] out */
  uint8_t* lm_erase;        /* [L] out */
  cvb_ba_result ba;         /* the solve: ba.pose [K][7] (nullable), cost history, step status, iterations, termination;
                               speedbias, lm and lm_owner are not written */
  int32_t n_edge;           /* out: edges in the problem */
  int32_t bad_loop;         /* out: the loop whose covariance is not positive definite, -1 for none */
} cvb_pgo_result;

CVB_API int cvb_pgo(cvb_ctx* ctx, const cvb_pgo_problem* p, const cvb_pgo_options* o, cvb_pgo_result* r);

#ifdef __cplusplus
}
#endif
#endif /* COVINS_B200_H_ */
