// covins_b200_shim.hpp — host-side C++ shim that keeps the reference's own call surface and routes it to the
// C-ABI of libcovins_b200.so (include/covins_b200.h).  Header-only, C++17, no third-party headers.
//
// The reference has no plugin/FFI layer; its seams are C++ symbols (SURVEY.md §8b):
//   Optimization::GlobalBundleAdjustment(MapPtr, int, double, bool, bool, bool)   optimization_be.hpp:38-40
//   Optimization::PoseGraphOptimization(MapPtr, PoseMap)                          optimization_be.hpp:46-47
//   the per-candidate matching block of PlaceRecognitionG::ComputeSE3             placerec_gen_be.cpp:72-125
//   the per-candidate matching block of PlaceRecognition::ComputeSE3              placerec_be.cpp:75-113
// Each function below has the same name, argument meaning and write-back behaviour; the body is
//   flatten containers (canonical orders, SURVEY.md §8c) → one C-ABI call → scatter through the reference's setters
// in the same order the reference calls them.
//
// The functions are templates over the container types, and touch them ONLY through member names the reference
// classes already have (KeyframeBase/Keyframe: keyframe_base.hpp:159-237, keyframe_be.hpp:86-112; LandmarkBase/
// Landmark: landmark_base.hpp:87-119, landmark_be.hpp:60-77; MapBase/Map: map_base.hpp:97-112; LoopConstraint:
// typedefs_base.hpp:264-277).  Inside the covins_backend tree they instantiate with the real classes (INTEGRATION.md
// shows the two-line change in optimization_be.cpp / placerec_gen_be.cpp); in this repository they are instantiated
// with the mock containers of tests/cpp/mock_containers.hpp.  Three things the real classes reach through
// third-party types are funnelled through one adapter, covins_b200::Adapter<Keyframe>, which the integrator
// specialises (camera intrinsics / distortion from aslam::Camera, raw IMU samples from robopt PreintegrationBase).
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <set>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../../include/covins_b200.h"
#include "../../../include/covins_b200_pose.h"

namespace covins_b200 {

// ---------------------------------------------------------------------------------------------------------------
// RAII context; one per host thread (the reference runs one place-recognition thread per agent).
// ---------------------------------------------------------------------------------------------------------------
class Context {
 public:
  explicit Context(int device = 0) {
    if (cvb_ctx_create(device, &ctx_) != CVB_OK)
      throw std::runtime_error("covins_b200: no usable CUDA device (there is no CPU fallback)");
  }
  ~Context() { cvb_ctx_destroy(ctx_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  cvb_ctx* get() const { return ctx_; }
  // error convention of the reference: print + exit(-1) (optimization_be.cpp:113-114); soft failures return
  void check(int rc, const char* what) const {
    if (rc == CVB_OK) return;
    std::fprintf(stderr, "\033[1;31m!!!!! FATAL !!!!!\033[0m covins_b200 %s: status %d: %s\n", what, rc, cvb_last_error(ctx_));
    std::exit(-1);
  }

 private:
  cvb_ctx* ctx_ = nullptr;
};

// ---------------------------------------------------------------------------------------------------------------
// Several GPUs from one process: one Context per rank and the cvb_group over them (cvb_group_create).  Ranks may share a
// device.  The server builds one at start-up over its GPUs and hands it to the GlobalBundleAdjustment overload below.
// ---------------------------------------------------------------------------------------------------------------
class ContextGroup {
 public:
  explicit ContextGroup(const std::vector<int>& devices) {
    std::vector<cvb_ctx*> raw;
    for (int d : devices) {
      ctxs_.push_back(std::make_unique<Context>(d));
      raw.push_back(ctxs_.back()->get());
    }
    if (raw.empty()) throw std::runtime_error("covins_b200: a context group needs at least one device");
    const int rc = cvb_group_create(raw.data(), (int)raw.size(), &g_);
    if (rc != CVB_OK)
      throw std::runtime_error(std::string("covins_b200: cvb_group_create failed: ") + cvb_last_error(raw[0]));
  }
  ~ContextGroup() { cvb_group_destroy(g_); }
  ContextGroup(const ContextGroup&) = delete;
  ContextGroup& operator=(const ContextGroup&) = delete;
  cvb_group* get() const { return g_; }
  int size() const { return (int)ctxs_.size(); }
  Context& rank(int r) { return *ctxs_[r]; }   // rank 0's context carries the group calls' error messages
  void check(int rc, const char* what) const { ctxs_[0]->check(rc, what); }

 private:
  std::vector<std::unique_ptr<Context>> ctxs_;
  cvb_group* g_ = nullptr;
};

// ---------------------------------------------------------------------------------------------------------------
// Adapter: the only place that touches third-party types of the real containers.  Default = mock containers.
// ---------------------------------------------------------------------------------------------------------------
template <class KF>
struct Adapter {
  // camera: pinhole intrinsics [fx,fy,cx,cy] + radtan [k1,k2,p1,p2]   (aslam::PinholeCamera::getParameters(),
  // getDistortion().getParameters(); optimization_be.cpp:95-103).  Returns false for unsupported models.
  static bool camera(const KF& kf, double intr[4], double dist[4]) { return kf.GetCameraParams(intr, dist); }
  // camera / distortion type of the keyframe's aslam camera — the template arguments the reference picks for
  // GlobalEuclideanReprError at optimization_be.cpp:186-231: cam 0 = kPinhole, 1 = kUnifiedProjection (xi = its first
  // intrinsic); dist 0 = kRadTan, 1 = kEquidistant, 2 = kFisheye.  The default serves containers without the notion
  // (ORB-SLAM3 agents only send pinhole + radtan, orb_slam3/src/KeyFrame.cc:64-65); specialise for the real Keyframe:
  //   cam = kf.camera_->getType() == aslam::Camera::Type::kUnifiedProjection, dist from getDistortion().getType().
  static void camera_model(const KF& kf, int* cam, int* dist, double* xi) { (void)kf; *cam = 0; *dist = 0; *xi = 0.0; }
  // the unit bearing vector [n][3] (camera frame) and sigma angle [n] of every keypoint, what Se3Solver::projectiveAlignment reads of
  // the query keyframe (FrameAbsolutePoseSacProblem's getSigmaAngle); specialise for the real Keyframe
  static void bearings(const KF& kf, double* f, double* sigma_angle) { kf.GetBearings(f, sigma_angle); }
  // raw IMU samples of the KF's preintegration (robopt PreintegrationBase::getReadingsByIndex / getTimeDiffByIndex,
  // keyframe_base.cpp:145-173) and its first reading + noise (keyframe_be.cpp:187-203)
  static size_t imu_count(const KF& kf) { return kf.ImuDt().size(); }
  static void imu_samples(const KF& kf, std::vector<double>& dt, std::vector<double>& acc, std::vector<double>& gyr,
                          double acc0[3], double gyr0[3], double noise[5]) {
    kf.GetImu(dt, acc, gyr, acc0, gyr0, noise);
  }
};

namespace detail {

// The pose conversions on the containers' 4x4 transforms (operator()(r,c)), through the one implementation the kernels use
// too (include/covins_b200_pose.h): transform_to_pose7 is Eigen::Quaterniond(R) as keyframe_base.cpp:490-499 uses it,
// pose7_to_transform is Utils::Ceres2Transform (utils_base.cpp:28-43).
template <class T4>
inline void to_rowmajor(const T4& T, double* m) {
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) m[4 * r + c] = T(r, c);
}
template <class T4>
inline T4 from_rowmajor(const double* m) {
  T4 T = T4::Identity();
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) T(r, c) = m[4 * r + c];
  return T;
}
template <class T4>
inline void transform_to_pose7(const T4& T, double* out) {
  double m[16];
  to_rowmajor(T, m);
  cvb_pose::transform_to_pose7(m, out);
}
template <class T4>
inline T4 pose7_to_transform(const double* p) {
  double m[16];
  cvb_pose::pose7_to_transform(p, m);
  return from_rowmajor<T4>(m);
}
// Flattened problem with owning storage + the cvb_ba_problem view
struct Flat {
  std::vector<double> pose, sb, extr, intr, dist, lm, obs_sigma, imu_dt, imu_acc, imu_gyr, imu_acc0, imu_gyr0, edge_q, edge_t,
      edge_S, cam_xi;
  std::vector<int32_t> cam_model, dist_model;
  std::vector<float> obs_uv;
  std::vector<uint8_t> pose_const, edge_robust;
  std::vector<int32_t> cam_of_kf, lm_obs_ptr, obs_kf, imu_i, imu_j, imu_ptr, edge_i, edge_j;
  double imu_noise[5] = {0, 0, 0, 0, 9.81};
  cvb_ba_problem view() const {
    cvb_ba_problem p{};
    p.K = (int32_t)pose_const.size();
    p.L = (int32_t)(lm.size() / 3);
    p.n_obs = (int32_t)obs_kf.size();
    p.n_imu = (int32_t)imu_i.size();
    p.n_edge = (int32_t)edge_i.size();
    p.n_cam = (int32_t)(extr.size() / 7);
    p.pose = pose.data(); p.speedbias = sb.data(); p.pose_const = pose_const.data(); p.cam_of_kf = cam_of_kf.data();
    p.extr = extr.data(); p.intr = intr.data(); p.dist = dist.data(); p.lm = lm.data(); p.lm_obs_ptr = lm_obs_ptr.data();
    p.obs_kf = obs_kf.data(); p.obs_uv = obs_uv.data(); p.obs_sigma = obs_sigma.data(); p.obs_skip = nullptr;
    p.imu_i = imu_i.data(); p.imu_j = imu_j.data(); p.imu_ptr = imu_ptr.data(); p.imu_dt = imu_dt.data();
    p.imu_acc = imu_acc.data(); p.imu_gyr = imu_gyr.data(); p.imu_acc0 = imu_acc0.data(); p.imu_gyr0 = imu_gyr0.data();
    p.imu_noise = imu_noise;
    p.edge_i = edge_i.data(); p.edge_j = edge_j.data(); p.edge_q = edge_q.data(); p.edge_t = edge_t.data();
    p.edge_sqrt_info = edge_S.data(); p.edge_robust = edge_robust.data();
    if (cam_model.size() == (size_t)p.n_cam) { p.cam_model = cam_model.data(); p.dist_model = dist_model.data(); p.cam_xi = cam_xi.data(); }
    return p;
  }
};

// The canonical flattening of a map's containers (SURVEY.md §8c), shared by every function that hands the map's structure
// to the library: the valid keyframes in the map's id-sorted order with their index ...
template <class KeyframePtr, class KF>
inline void canonical_keyframes(const std::vector<KeyframePtr>& keyframes, std::map<const KF*, int>& kf_index, std::vector<KeyframePtr>& kfs) {
  for (auto& kf : keyframes) {
    if (kf->IsInvalid()) continue;
    kf_index[kf.get()] = (int)kfs.size();
    kfs.push_back(kf);
  }
}
// ... and the valid landmarks in id order with the CSR of their observations by valid keyframes, each landmark's sorted by
// keyframe index (the reference iterates a pointer-ordered std::map, typedefs_base.hpp:187).  on_obs(keyframe index,
// feature id, landmark index) is called once per observation in CSR order.
template <class LandmarkPtr, class KF, class OnObs>
inline void flatten_observations(const std::vector<LandmarkPtr>& landmarks, const std::map<const KF*, int>& kf_index, std::vector<LandmarkPtr>& lms,
                                 std::vector<int32_t>& lm_obs_ptr, std::vector<int32_t>& obs_kf, OnObs on_obs) {
  lm_obs_ptr.push_back(0);
  for (auto& lm : landmarks) {
    if (lm->IsInvalid()) continue;
    const auto observations = lm->GetObservations();
    std::vector<std::pair<int, int>> ob;   // (kf index, feature id)
    for (const auto& mit : observations) {
      auto kfx = mit.first;
      if (!kfx || kfx->IsInvalid()) continue;
      ob.emplace_back(kf_index.at(kfx.get()), (int)mit.second);
    }
    std::sort(ob.begin(), ob.end());
    for (auto& o : ob) {
      obs_kf.push_back(o.first);
      on_obs(o.first, o.second, (int)lms.size());
    }
    lm_obs_ptr.push_back((int32_t)obs_kf.size());
    lms.push_back(lm);
  }
}

// The camera and observation part of a map's flat problem, shared by GlobalBundleAdjustment and RemoveLandmarkOutliers: every
// keyframe of kfs (canonical order) with its state (UpdateCeresFromState, keyframe_base.cpp:486-521), its own calibration
// (cam_of_kf[k] = k) and camera model, pose_const cleared; then the valid landmarks (flatten_observations) with their
// positions and each observation's keypoint and sigma.  obs_ref[i] names observation i's keyframe, landmark and feature for
// the write-back.
template <class KeyframePtr>
struct ObsRef {
  KeyframePtr kf;
  int lm;
  int feat;
};
template <class KeyframePtr, class KF, class LandmarkPtr>
inline void flatten_cameras_and_observations(const std::vector<KeyframePtr>& kfs, const std::map<const KF*, int>& kf_index,
                                             const std::vector<LandmarkPtr>& landmarks, Flat& F, std::vector<LandmarkPtr>& lms,
                                             std::vector<ObsRef<KeyframePtr>>& obs_ref) {
  const int K = (int)kfs.size();
  F.pose.resize(7 * (size_t)K); F.sb.resize(9 * (size_t)K); F.extr.resize(7 * (size_t)K); F.intr.resize(4 * (size_t)K);
  F.dist.resize(4 * (size_t)K); F.pose_const.assign(K, 0); F.cam_of_kf.resize(K);
  F.cam_model.assign(K, 0); F.dist_model.assign(K, 0); F.cam_xi.assign(K, 0.0);
  for (int k = 0; k < K; k++) {
    auto& kf = kfs[k];
    kf->UpdateCeresFromState(&F.pose[7 * (size_t)k], &F.sb[9 * (size_t)k], &F.extr[7 * (size_t)k]);
    F.cam_of_kf[k] = k;
    if (!Adapter<KF>::camera(*kf, &F.intr[4 * (size_t)k], &F.dist[4 * (size_t)k])) {
      std::printf("FATAL: Unknown projection type.\n");                                            // optimization_be.cpp:112-114
      std::exit(-1);
    }
    Adapter<KF>::camera_model(*kf, &F.cam_model[k], &F.dist_model[k], &F.cam_xi[k]);                // :186-231
  }
  flatten_observations(landmarks, kf_index, lms, F.lm_obs_ptr, F.obs_kf, [&](int k, int feat, int l) {
    auto& kfx = kfs[k];
    const auto& kp = kfx->keypoints_distorted_[feat];
    F.obs_uv.push_back((float)kp[0]); F.obs_uv.push_back((float)kp[1]);
    F.obs_sigma.push_back((kfx->keypoints_aors_[feat][1] + 1) * 2.0);                              // :183-184, 477-478
    obs_ref.push_back({kfx, l, feat});
  });
  for (auto& lm : lms) {
    const auto pos = lm->GetWorldPos();
    F.lm.push_back(pos[0]); F.lm.push_back(pos[1]); F.lm.push_back(pos[2]);
  }
}

}  // namespace detail

// parameters the reference reads from covins_params (config/config_backend.yaml; SURVEY.md §5)
struct OptParams {
  double th_outlier_align = 1.3;            // opt.th_outlier_align (config_backend.yaml)
  bool gba_fix_poses_loaded_maps = false;       // opt.gba_fix_poses_loaded_maps (optimization_be.cpp:338)
  bool gba_use_map_loop_constraints = true;     // :539
  double th_gba_outlier_global = 0.92;          // :277
  bool pgo_fix_kfs_after_gba = true;            // :875
  bool pgo_fix_poses_loaded_maps = true;        // :878
  int pgo_iteration_limit = 10;                 // :1029
  bool use_nbr_kfs = true;                      // :976
  bool use_robust_loss = true;                  // :934
  double robust_loss_th = 0.5;                  // :840
  double wt_kf_r = 10.0, wt_kf_t = 1.0, wt_kf_n1 = 10.0, wt_kf_n23 = 2.0, wt_kf_n45 = 3.0;   // :896-903
  bool placerec_type_covins = false;            // placerec.type == "COVINS" (:929)
  float img_match_thres = 40.0f, ratio_thres = 0.8f;    // features (placerec_gen_be.cpp:107-108)
  int matches_thres = 25, matches_thres_merge = 25;     // placerec (placerec_gen_be.cpp:118-121)
};

namespace detail {
// Optimization::GlobalBundleAdjustment's flatten and write-back around one solver call:
// solve(problem, gba options, result, obs_removed) -> cvb_status (cvb_gba on one context, cvb_gba_group on a group).
template <class MapPtr, class Solve>
void global_bundle_adjustment(MapPtr map, int interations_limit, bool visual_only, bool outlier_removal, const OptParams& P,
                              Solve solve) {
  using KeyframePtr = typename std::decay<decltype(map->GetKeyframesVec()[0])>::type;
  using KF = typename KeyframePtr::element_type;
  using Transform = typename std::decay<decltype(map->GetKeyframesVec()[0]->GetPoseTws())>::type;
  std::printf("+++ GBA: Start +++\n");
  auto keyframes = map->GetKeyframesVec();   // id-sorted std::map order (map_base.cpp:63-69)
  auto landmarks = map->GetLandmarksVec();
  std::printf("--> KFs: %zu\n--> LMs: %zu\n", keyframes.size(), landmarks.size());

  detail::Flat F;
  std::map<const KF*, int> kf_index;
  std::vector<KeyframePtr> kfs;               // valid keyframes, canonical order
  detail::canonical_keyframes(keyframes, kf_index, kfs);
  const int K = (int)kfs.size();
  // keyframe states, cameras, landmarks + observations (detail::flatten_cameras_and_observations: the canonical landmark
  // order and observation CSR)
  using LandmarkPtr = typename std::decay<decltype(landmarks[0])>::type;
  std::vector<LandmarkPtr> lms;
  std::vector<detail::ObsRef<KeyframePtr>> obs_ref;
  detail::flatten_cameras_and_observations(kfs, kf_index, landmarks, F, lms, obs_ref);
  F.imu_ptr.push_back(0);
  for (int k = 0; k < K; k++) {
    auto& kf = kfs[k];
    if (kf->id_.first == 0 && kf->id_.second == map->id_map_) F.pose_const[k] = 1;                 // :88-89, 329-331
    if (kf->is_loaded_ && P.gba_fix_poses_loaded_maps) F.pose_const[k] = 1;                        // :338-341
    if (!visual_only) {                                                                             // :117-144, 367-421
      auto pred = kf->GetPredecessor();
      if (!pred || pred->IsInvalid()) {
        if (kf->id_.first != 0) {
          std::printf("FATAL: KF %zu|%zu: no predecessor\n", (size_t)kf->id_.first, (size_t)kf->id_.second);
          std::exit(-1);
        }
        continue;
      }
      if (Adapter<KF>::imu_count(*kf) == 0) {
        std::printf("KF %zu|%zu 0 IMU measurements - skip IMU factor\n", (size_t)kf->id_.first, (size_t)kf->id_.second);   // :382-385
        continue;
      }
      std::vector<double> dt, acc, gyr;
      double a0[3], g0[3];
      Adapter<KF>::imu_samples(*kf, dt, acc, gyr, a0, g0, F.imu_noise);
      F.imu_i.push_back(kf_index.at(pred.get()));
      F.imu_j.push_back(k);
      F.imu_dt.insert(F.imu_dt.end(), dt.begin(), dt.end());
      F.imu_acc.insert(F.imu_acc.end(), acc.begin(), acc.end());
      F.imu_gyr.insert(F.imu_gyr.end(), gyr.begin(), gyr.end());
      F.imu_acc0.insert(F.imu_acc0.end(), a0, a0 + 3);
      F.imu_gyr0.insert(F.imu_gyr0.end(), g0, g0 + 3);
      F.imu_ptr.push_back((int32_t)F.imu_dt.size());
    }
  }
  // loop edges (:236-254, 532-557): sqrt_info = diag(100 I3, 1e4 I3)
  if (P.gba_use_map_loop_constraints) {
    for (const auto& lc : map->GetLoopConstraints()) {
      auto i1 = kf_index.find(lc.kf1.get()), i2 = kf_index.find(lc.kf2.get());
      if (i1 == kf_index.end() || i2 == kf_index.end()) {
        std::printf("WARN: Loop KF missing -- skip loop\n");                                        // :546-549
        continue;
      }
      double p7[7];
      detail::transform_to_pose7(lc.T_s1_s2, p7);
      F.edge_i.push_back(i1->second); F.edge_j.push_back(i2->second);
      F.edge_q.insert(F.edge_q.end(), p7, p7 + 4);
      F.edge_t.insert(F.edge_t.end(), p7 + 4, p7 + 7);
      for (int r = 0; r < 6; r++)
        for (int c = 0; c < 6; c++) F.edge_S.push_back(r == c ? (r < 3 ? 100.0 : 1e4) : 0.0);
      F.edge_robust.push_back(1);
    }
  }
  const cvb_ba_problem prob = F.view();
  std::vector<double> o_pose(7 * (size_t)K), o_sb(9 * (size_t)K), o_lm(F.lm.size());
  std::vector<int32_t> owner(lms.size() ? lms.size() : 1);
  std::vector<uint8_t> removed(F.obs_kf.size() ? F.obs_kf.size() : 1, 0);
  cvb_ba_result res{};
  res.pose = o_pose.data(); res.speedbias = o_sb.data(); res.lm = o_lm.data(); res.lm_owner = owner.data();
  cvb_gba_options g{interations_limit, visual_only ? 1 : 0, outlier_removal ? 1 : 0, P.th_gba_outlier_global};
  solve(&prob, &g, &res, removed.data());

  // round-1 outlier purge, written into the map exactly like optimization_be.cpp:282-288
  size_t num_bad = 0;
  for (size_t i = 0; i < obs_ref.size(); i++)
    if (removed[i]) {
      obs_ref[i].kf->EraseLandmark(obs_ref[i].feat);
      lms[obs_ref[i].lm]->EraseObservation(obs_ref[i].kf);
      ++num_bad;
    }
  if (outlier_removal) std::printf("--> GBA removed %zu of %zu observations\n", num_bad, 2 * obs_ref.size());
  // Recover optimized data — keyframes (:572-595)
  for (int k = 0; k < K; k++) {
    auto& kf = kfs[k];
    kf->SetPoseTws(detail::pose7_to_transform<Transform>(&o_pose[7 * (size_t)k]));
    kf->SetPoseOptimized();
    if (!visual_only) {
      const double* s = &o_sb[9 * (size_t)k];
      kf->SetStateBias({s[3], s[4], s[5]}, {s[6], s[7], s[8]});
      kf->SetStateVelocity({s[0], s[1], s[2]});
      kf->SetVelBiasOptimized();
    }
    kf->is_gba_optimized_ = true;
  }
  // landmarks (:598-609): only those that were in the problem
  for (size_t l = 0; l < lms.size(); l++) {
    if (owner[l] < 0) continue;
    lms[l]->SetWorldPos({o_lm[3 * l], o_lm[3 * l + 1], o_lm[3 * l + 2]});
    lms[l]->SetOptimized();
    lms[l]->is_gba_optimized_ = true;
  }
  std::printf("--> Clean Map\n");
  map->Clean();                                                                                     // :614
  std::printf("--> done.\n+++ GBA: End +++\n");
}
}  // namespace detail

// ---------------------------------------------------------------------------------------------------------------
// Optimization::GlobalBundleAdjustment — same signature meaning as optimization_be.hpp:38-40.
// ---------------------------------------------------------------------------------------------------------------
template <class MapPtr>
void GlobalBundleAdjustment(Context& ctx, MapPtr map, int interations_limit, double /*time_limit*/, bool visual_only = false,
                            bool outlier_removal = true, bool /*estimate_bias*/ = false, const OptParams& P = OptParams()) {
  detail::global_bundle_adjustment(map, interations_limit, visual_only, outlier_removal, P,
                                   [&ctx](const cvb_ba_problem* p, const cvb_gba_options* g, cvb_ba_result* r, uint8_t* removed) {
                                     ctx.check(cvb_gba(ctx.get(), p, g, r, removed), "cvb_gba");
                                   });
}

// The same, with the merged map's landmarks sharded over the ranks of a ContextGroup (cvb_gba_group).  peer_path: reduce-scatter
// by peer pull and the column-distributed factorisation (a device per rank; not yet verified on several devices, so off by
// default), else the all-reduce of the packed reduced system.
template <class MapPtr>
void GlobalBundleAdjustment(ContextGroup& group, MapPtr map, int interations_limit, double /*time_limit*/, bool visual_only = false,
                            bool outlier_removal = true, bool /*estimate_bias*/ = false, const OptParams& P = OptParams(),
                            bool peer_path = false) {
  detail::global_bundle_adjustment(map, interations_limit, visual_only, outlier_removal, P,
                                   [&group, peer_path](const cvb_ba_problem* p, const cvb_gba_options* g, cvb_ba_result* r, uint8_t* removed) {
                                     group.check(cvb_gba_group(group.get(), p, g, peer_path ? 1 : 0, r, removed), "cvb_gba_group");
                                   });
}

// ---------------------------------------------------------------------------------------------------------------
// Keyframe::UpdateCovisibilityConnections (keyframe_be.cpp:559-608) for every keyframe of the map in one call — what the
// reference repeats keyframe by keyframe after a merge, a map load or a GBA round that erased observations.  Every valid
// keyframe receives its connected keyframes, ordered by weight (GetConnectedKeyframes order), through one setter,
// kf->SetCovisibility(keyframes, weights) (INTEGRATION.md shows it).  The graph is the canonical one cvb_covisibility
// defines; min_weight 15 is the value the reference hard-codes.
// ---------------------------------------------------------------------------------------------------------------
template <class MapPtr>
void UpdateCovisibilityConnections(Context& ctx, MapPtr map, int min_weight = 15) {
  using KeyframePtr = typename std::decay<decltype(map->GetKeyframesVec()[0])>::type;
  using KF = typename KeyframePtr::element_type;
  auto landmarks = map->GetLandmarksVec();
  using LandmarkPtr = typename std::decay<decltype(landmarks[0])>::type;
  std::map<const KF*, int> kf_index;
  std::vector<KeyframePtr> kfs;
  detail::canonical_keyframes(map->GetKeyframesVec(), kf_index, kfs);
  std::vector<LandmarkPtr> lms;
  std::vector<int32_t> lm_obs_ptr, obs_kf;
  detail::flatten_observations(landmarks, kf_index, lms, lm_obs_ptr, obs_kf, [](int, int, int) {});
  const int K = (int)kfs.size(), L = (int)lms.size();
  std::vector<int32_t> nbr_ptr((size_t)K + 1), nbr_kf, nbr_w;
  int64_t n_total = 0, cap = 0;
  do {   // the first call sizes the lists, the second fills them
    cap = n_total;
    nbr_kf.resize((size_t)cap + 1); nbr_w.resize((size_t)cap + 1);
    ctx.check(cvb_covisibility(ctx.get(), K, L, lm_obs_ptr.data(), obs_kf.data(), nullptr, nullptr, min_weight, nbr_ptr.data(), nbr_kf.data(),
                               nbr_w.data(), cap, &n_total), "cvb_covisibility");
  } while (n_total > cap);
  for (int k = 0; k < K; k++) {
    std::vector<KeyframePtr> connected;
    for (int t = nbr_ptr[k]; t < nbr_ptr[k + 1]; t++) connected.push_back(kfs[nbr_kf[t]]);
    kfs[k]->SetCovisibility(connected, std::vector<int>(nbr_w.begin() + nbr_ptr[k], nbr_w.begin() + nbr_ptr[k + 1]));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The redundancy pruning of Map::Clean (map_be.cpp:745-811, the covins_prunemap service): the keyframes the sequential
// culling pass removes, found in one cvb_redundant_keyframes call (the rule is in include/covins_b200.h).  Never culled:
// the first keyframe of every agent and every keyframe a loop constraint names.  The culled keyframes are handed to the
// reference's own kf->SetInvalid() in ascending canonical order (keyframe_be.cpp:413-440: the IMU samples go to the
// successor), then the covisibility graph of what remains is rebuilt.  Landmark erasure stays with the caller's
// map->Clean(), as after GlobalBundleAdjustment; th_red, max_time_dist and th_obs are the caller's values.
// ---------------------------------------------------------------------------------------------------------------
template <class MapPtr>
void PruneRedundantKeyframes(Context& ctx, MapPtr map, double th_red, double max_time_dist, int th_obs = 3) {
  using KeyframePtr = typename std::decay<decltype(map->GetKeyframesVec()[0])>::type;
  using KF = typename KeyframePtr::element_type;
  auto landmarks = map->GetLandmarksVec();
  using LandmarkPtr = typename std::decay<decltype(landmarks[0])>::type;
  std::map<const KF*, int> kf_index;
  std::vector<KeyframePtr> kfs;
  detail::canonical_keyframes(map->GetKeyframesVec(), kf_index, kfs);
  std::vector<LandmarkPtr> lms;
  std::vector<int32_t> lm_obs_ptr, obs_kf, obs_octave;
  detail::flatten_observations(landmarks, kf_index, lms, lm_obs_ptr, obs_kf,
                               [&](int k, int feat, int) { obs_octave.push_back((int32_t)kfs[k]->keypoints_aors_[feat][1]); });
  const int K = (int)kfs.size(), L = (int)lms.size();
  std::vector<int32_t> kf_pred((size_t)K, -1);
  std::vector<double> kf_time((size_t)K);
  std::vector<uint8_t> kf_protect((size_t)K, 0), culled((size_t)K + 1, 0);
  for (int k = 0; k < K; k++) {
    auto pred = kfs[k]->GetPredecessor();
    if (pred) {
      auto it = kf_index.find(pred.get());
      if (it != kf_index.end()) kf_pred[k] = it->second;
    }
    kf_time[k] = (double)kfs[k]->timestamp_;
    if (kfs[k]->id_.first == 0) kf_protect[k] = 1;   // an agent's first keyframe
  }
  for (const auto& lc : map->GetLoopConstraints())
    for (const auto& kf : {lc.kf1, lc.kf2}) {
      auto it = kf_index.find(kf.get());
      if (it != kf_index.end()) kf_protect[it->second] = 1;
    }
  // octaves above the largest one present change no count: the map's own range is the histogram's
  const int num_octaves = obs_octave.empty() ? 1 : 1 + *std::max_element(obs_octave.begin(), obs_octave.end());
  ctx.check(cvb_redundant_keyframes(ctx.get(), K, L, lm_obs_ptr.data(), obs_kf.data(), obs_octave.data(), nullptr, nullptr, kf_pred.data(),
                                    kf_time.data(), kf_protect.data(), th_red, max_time_dist, th_obs, num_octaves, culled.data(), nullptr),
            "cvb_redundant_keyframes");
  for (int k = 0; k < K; k++)
    if (culled[k]) kfs[k]->SetInvalid();
  UpdateCovisibilityConnections(ctx, map);
}

// ---------------------------------------------------------------------------------------------------------------
// The landmark outlier removal of Map::Clean (map_be.cpp:448-454, 698-743), found in one cvb_landmark_outliers call (the
// rule is in include/covins_b200.h) on the flat map the GBA builds (detail::flatten_cameras_and_observations).  Write-back in
// canonical order: each outlier observation through the calls of the GBA's round-1 purge (kf->EraseLandmark(feat),
// lm->EraseObservation(kf), optimization_be.cpp:282-288), then each erased landmark through map->EraseLandmark(lm), then
// the covisibility graph of what remains is rebuilt.  Map::Clean calls it in place of its own landmark pass
// (INTEGRATION.md §3.7), so the map->Clean() that ends GlobalBundleAdjustment picks it up.
// ---------------------------------------------------------------------------------------------------------------
template <class MapPtr>
void RemoveLandmarkOutliers(Context& ctx, MapPtr map, double th_outlier = 0.92, double cauchy = 1.0, int min_obs = 2) {
  using KeyframePtr = typename std::decay<decltype(map->GetKeyframesVec()[0])>::type;
  using KF = typename KeyframePtr::element_type;
  auto landmarks = map->GetLandmarksVec();
  using LandmarkPtr = typename std::decay<decltype(landmarks[0])>::type;
  std::map<const KF*, int> kf_index;
  std::vector<KeyframePtr> kfs;
  detail::canonical_keyframes(map->GetKeyframesVec(), kf_index, kfs);
  detail::Flat F;
  std::vector<LandmarkPtr> lms;
  std::vector<detail::ObsRef<KeyframePtr>> obs_ref;
  detail::flatten_cameras_and_observations(kfs, kf_index, landmarks, F, lms, obs_ref);
  const cvb_ba_problem prob = F.view();
  std::vector<uint8_t> outlier(obs_ref.size() + 1, 0), erase(lms.size() + 1, 0);
  int64_t n_outlier = 0;
  int32_t n_erased = 0;
  ctx.check(cvb_landmark_outliers(ctx.get(), &prob, nullptr, th_outlier, cauchy, min_obs, outlier.data(), erase.data(), nullptr, &n_outlier,
                                  &n_erased),
            "cvb_landmark_outliers");
  for (size_t i = 0; i < obs_ref.size(); i++)
    if (outlier[i]) {
      obs_ref[i].kf->EraseLandmark(obs_ref[i].feat);
      lms[obs_ref[i].lm]->EraseObservation(obs_ref[i].kf);
    }
  for (size_t l = 0; l < lms.size(); l++)
    if (erase[l]) map->EraseLandmark(lms[l]);
  std::printf("--> Landmark outliers: removed %lld of %zu observations, erased %d of %zu landmarks\n", (long long)n_outlier, obs_ref.size(),
              n_erased, lms.size());
  UpdateCovisibilityConnections(ctx, map);
}

// ---------------------------------------------------------------------------------------------------------------
// Optimization::PoseGraphOptimization — optimization_be.hpp:46-47.  PoseMap = std::map<idpair, Transform>.
// The chain is flattened in canonical keyframe order and handed to one cvb_pgo call (the edge rule, the solve and the
// write-back are stated in include/covins_b200.h).  Write-back: keyframes in canonical order (SetPoseTws, SetStateVelocity,
// SetPoseOptimized, :1033-1051), then the valid landmarks in map order: SetWorldPos + SetOptimized when re-anchored through
// their reference keyframe, map->EraseLandmark when cvb_pgo flags them (:1054-1083).
// ---------------------------------------------------------------------------------------------------------------
template <class MapPtr, class PoseMap>
void PoseGraphOptimization(Context& ctx, MapPtr map, PoseMap corrected_poses, const OptParams& P = OptParams()) {
  using KeyframePtr = typename std::decay<decltype(map->GetKeyframesVec()[0])>::type;
  using KF = typename KeyframePtr::element_type;
  using Transform = typename std::decay<decltype(map->GetKeyframesVec()[0]->GetPoseTws())>::type;
  auto landmarks = map->GetLandmarksVec();
  using LandmarkPtr = typename std::decay<decltype(landmarks[0])>::type;
  std::map<const KF*, int> kf_index;
  std::vector<KeyframePtr> kfs;
  detail::canonical_keyframes(map->GetKeyframesVec(), kf_index, kfs);
  const int K = (int)kfs.size();
  const auto index_of = [&](const KeyframePtr& kf) -> int32_t {   // -1 none, -2 not among the valid keyframes
    if (!kf) return -1;
    auto it = kf_index.find(kf.get());
    return it == kf_index.end() ? -2 : it->second;
  };
  std::vector<double> T_ws(16 * (size_t)K), T_init(16 * (size_t)K), T_vio(16 * (size_t)K), vel(3 * (size_t)K);
  std::vector<int32_t> pred(K), succ(K), kid(K);
  std::vector<uint8_t> pose_const(K, 0);
  for (int k = 0; k < K; k++) {
    auto& kf = kfs[k];
    detail::to_rowmajor(kf->GetPoseTws(), &T_ws[16 * (size_t)k]);
    auto mit = corrected_poses.find(kf->id_);                                                        // :854-868
    if (mit != corrected_poses.end()) detail::to_rowmajor(mit->second, &T_init[16 * (size_t)k]);
    else std::copy(&T_ws[16 * (size_t)k], &T_ws[16 * (size_t)k] + 16, &T_init[16 * (size_t)k]);
    detail::to_rowmajor(kf->GetPoseTws_vio(), &T_vio[16 * (size_t)k]);
    pred[k] = index_of(kf->GetPredecessor());
    succ[k] = index_of(kf->GetSuccessor());
    kid[k] = (int32_t)int(kf->id_.first);
    if (kf->id_.first == 0 && kf->id_.second == map->id_map_) pose_const[k] = 1;                    // :870-871
    if (kf->is_gba_optimized_ && P.pgo_fix_kfs_after_gba) pose_const[k] = 1;                        // :875-877
    else if (kf->is_loaded_ && P.pgo_fix_poses_loaded_maps) pose_const[k] = 1;                      // :878-881
    const auto v = kf->GetStateVelocity();
    for (int c = 0; c < 3; c++) vel[3 * (size_t)k + c] = v[c];
  }
  std::vector<int32_t> loop_i, loop_j;
  std::vector<double> loop_q, loop_t, loop_cov;
  for (const auto& lc : map->GetLoopConstraints()) {                                                 // :910-943
    double p7[7];
    detail::transform_to_pose7(lc.T_s1_s2, p7);
    loop_i.push_back(index_of(lc.kf1));
    loop_j.push_back(index_of(lc.kf2));
    loop_q.insert(loop_q.end(), p7, p7 + 4);
    loop_t.insert(loop_t.end(), p7 + 4, p7 + 7);
    for (int r = 0; r < 6; r++)
      for (int c = 0; c < 6; c++) loop_cov.push_back(lc.cov_mat(r, c));
  }
  std::vector<LandmarkPtr> lms;
  std::vector<double> lm_pos;
  std::vector<int32_t> lm_ref;
  std::vector<uint8_t> lm_has_obs;
  for (auto& lm : landmarks) {
    if (lm->IsInvalid()) continue;
    const auto pw = lm->GetWorldPos();
    lm_pos.insert(lm_pos.end(), {pw[0], pw[1], pw[2]});
    lm_ref.push_back(index_of(lm->GetReferenceKeyframe()));
    lm_has_obs.push_back(lm->GetObservations().empty() ? 0 : 1);
    lms.push_back(lm);
  }
  const int L = (int)lms.size();
  cvb_pgo_problem pp{};
  pp.K = K; pp.T_ws = T_ws.data(); pp.T_ws_init = T_init.data(); pp.T_ws_vio = T_vio.data();
  pp.kf_pred = pred.data(); pp.kf_succ = succ.data(); pp.kf_id = kid.data(); pp.pose_const = pose_const.data(); pp.velocity = vel.data();
  pp.n_loop = (int32_t)loop_i.size(); pp.loop_i = loop_i.data(); pp.loop_j = loop_j.data(); pp.loop_q = loop_q.data(); pp.loop_t = loop_t.data();
  pp.loop_cov = P.placerec_type_covins ? nullptr : loop_cov.data();                                 // :929
  pp.L = L; pp.lm_pos = lm_pos.data(); pp.lm_ref = lm_ref.data(); pp.lm_has_obs = lm_has_obs.data();
  cvb_pgo_options po{P.wt_kf_r, P.wt_kf_t, P.wt_kf_n1, P.wt_kf_n23, P.wt_kf_n45, P.use_nbr_kfs ? 1 : 0, P.use_robust_loss ? 1 : 0,
                     P.robust_loss_th, P.pgo_iteration_limit};
  std::vector<double> T_out(16 * (size_t)K), vel_out(3 * (size_t)K), lm_out(3 * (size_t)L);
  std::vector<uint8_t> lm_erase(L);
  cvb_pgo_result res{};
  res.T_ws_out = T_out.data(); res.velocity_out = vel_out.data(); res.lm_out = lm_out.data(); res.lm_erase = lm_erase.data();
  const int rc = cvb_pgo(ctx.get(), &pp, &po, &res);
  if (res.bad_loop >= 0) {
    std::printf("FATAL: loop covariance is not positive definite\n");
    std::exit(-1);
  }
  ctx.check(rc, "cvb_pgo");
  for (int k = 0; k < K; k++) {                                                                      // :1033-1051
    auto& kf = kfs[k];
    kf->SetPoseTws(detail::from_rowmajor<Transform>(&T_out[16 * (size_t)k]));
    kf->SetStateVelocity({vel_out[3 * (size_t)k], vel_out[3 * (size_t)k + 1], vel_out[3 * (size_t)k + 2]});
    kf->SetPoseOptimized();
  }
  for (int l = 0; l < L; l++) {                                                                      // :1054-1083
    if (lm_erase[l]) {
      map->EraseLandmark(lms[l]);
    } else if (lm_ref[l] >= 0) {
      lms[l]->SetWorldPos({lm_out[3 * (size_t)l], lm_out[3 * (size_t)l + 1], lm_out[3 * (size_t)l + 2]});
      lms[l]->SetOptimized();
    }
  }
  std::printf("--> PGO END \n");
}

// ---------------------------------------------------------------------------------------------------------------
// Optimization::OptimizeRelativePose — optimization_be.hpp:42-44.  Same signature meaning: matches1[i] (indexed by kf1's
// keypoints) holds the landmark of kf2 matched to kf1's landmark i; T12 is refined in place; rejected entries of matches1
// are nulled; returns the inlier count, 0 when fewer than 12 remain.  Reference quirks kept on purpose:
//   * TcwB is built with kf1's extrinsics (:643);
//   * the purge nulls matches1[r] with r the RESIDUAL index, not vIndex[r] (:815).
// ---------------------------------------------------------------------------------------------------------------
template <class KFPtr, class LandmarkVector, class Transform4>
inline int OptimizeRelativePose(Context& ctx, const KFPtr& kf1, const KFPtr& kf2, LandmarkVector& matches1, Transform4& T12,
                                double /*th2, unused by the reference*/, const OptParams& P) {
  using KF = typename std::decay<decltype(*kf1)>::type;
  cvb_relpose_problem prob{};
  detail::transform_to_pose7(T12, prob.T12);                                                          // :629-638
  // TcwA = (T_ws1 * T_sc1)^-1, TcwB = (T_ws2 * T_sc1)^-1  (kf1's extrinsics for both, :642-643)
  auto mul4 = [](const Transform4& A, const Transform4& B) {
    Transform4 C = Transform4::Identity();
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) { double s = 0; for (int k = 0; k < 4; k++) s += A(r, k) * B(k, c); C(r, c) = s; }
    return C;
  };
  auto inv_rigid = [](const Transform4& T) {
    Transform4 I = Transform4::Identity();
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) I(r, c) = T(c, r);
    for (int r = 0; r < 3; r++) I(r, 3) = -(I(r, 0) * T(0, 3) + I(r, 1) * T(1, 3) + I(r, 2) * T(2, 3));
    return I;
  };
  const Transform4 TcwA = inv_rigid(mul4(kf1->GetPoseTws(), kf1->GetStateExtrinsics()));
  const Transform4 TcwB = inv_rigid(mul4(kf2->GetPoseTws(), kf1->GetStateExtrinsics()));
  const auto lmsA = kf1->GetLandmarks();
  std::vector<double> pA, pB, sA, sB;
  std::vector<float> kA, kB;
  const int N = (int)matches1.size();
  for (int i = 0; i < N; i++) {                                                                        // :656-780
    if (!matches1[i]) continue;
    auto pMPA = lmsA[i];
    auto pMPB = matches1[i];
    const int iB = pMPB->GetFeatureIndex(kf2);
    if (!pMPA || pMPA->IsInvalid() || pMPB->IsInvalid() || iB < 0) continue;
    const auto wa = pMPA->GetWorldPos(), wb = pMPB->GetWorldPos();
    for (int r = 0; r < 3; r++) {
      pA.push_back(TcwA(r, 0) * wa[0] + TcwA(r, 1) * wa[1] + TcwA(r, 2) * wa[2] + TcwA(r, 3));
      pB.push_back(TcwB(r, 0) * wb[0] + TcwB(r, 1) * wb[1] + TcwB(r, 2) * wb[2] + TcwB(r, 3));
    }
    kA.push_back(kf1->keypoints_distorted_[i][0]); kA.push_back(kf1->keypoints_distorted_[i][1]);
    kB.push_back(kf2->keypoints_distorted_[iB][0]); kB.push_back(kf2->keypoints_distorted_[iB][1]);
    sA.push_back((kf1->keypoints_aors_[i][1] + 1) * 2.0); sB.push_back((kf2->keypoints_aors_[iB][1] + 1) * 2.0);
  }
  prob.n = (int32_t)sA.size();
  prob.pA_c = pA.data(); prob.pB_c = pB.data(); prob.kpA = kA.data(); prob.kpB = kB.data(); prob.sigmaA = sA.data(); prob.sigmaB = sB.data();
  if (!Adapter<KF>::camera(*kf1, prob.intrA, prob.distA) || !Adapter<KF>::camera(*kf2, prob.intrB, prob.distB)) {
    std::printf("FATAL: Unknown projection type.\n");                                                // :705-707
    std::exit(-1);
  }
  Adapter<KF>::camera_model(*kf1, &prob.cam_model_A, &prob.dist_model_A, &prob.xiA);
  Adapter<KF>::camera_model(*kf2, &prob.cam_model_B, &prob.dist_model_B, &prob.xiB);
  double out[7];
  std::vector<uint8_t> removed(prob.n > 0 ? prob.n : 1, 0);
  int32_t n_inl = 0;
  ctx.check(cvb_optimize_relative_pose(ctx.get(), &prob, P.th_outlier_align, out, removed.data(), &n_inl, nullptr), "cvb_optimize_relative_pose");
  for (int r = 0; r < prob.n; r++)
    if (removed[r]) matches1[r] = nullptr;                                                            // matches1[i] with i = residual index (:815)
  if (n_inl == 0) return 0;                                                                            // :821-823, T12 untouched
  T12 = detail::pose7_to_transform<Transform4>(out);                                                  // :829
  return n_inl;
}

// ---------------------------------------------------------------------------------------------------------------
// Matching blocks
// ---------------------------------------------------------------------------------------------------------------
struct Match {   // covins::Match (include/covins/matcher/MatchingAlgorithm.h:56-70)
  size_t idxA, idxB;
  float distance;
};
using Matches = std::vector<Match>;

// The ORB branch of the candidate loop of PlaceRecognitionG::ComputeSE3 (placerec_gen_be.cpp:72-125) for ALL
// candidates at once: knnMatch(query, cand, 2) + distance/ratio filter.  descriptors are row-major [n][32] uint8
// (cv::Mat descriptors_add_ rows).  Returns img_matches per candidate; discarded[i] is set as at :118-124.
inline std::vector<Matches> MatchCandidatesORB(Context& ctx, const uint8_t* query, int n_query,
                                               const std::vector<const uint8_t*>& cand_desc, const std::vector<int>& cand_rows,
                                               const std::vector<bool>& same_client, const OptParams& P,
                                               std::vector<bool>* discarded) {
  const int n_seg = (int)cand_desc.size();
  std::vector<int32_t> seg(n_seg + 1, 0);
  for (int s = 0; s < n_seg; s++) seg[s + 1] = seg[s] + cand_rows[s];
  std::vector<uint8_t> train((size_t)seg[n_seg] * 32);
  for (int s = 0; s < n_seg; s++) std::copy(cand_desc[s], cand_desc[s] + (size_t)cand_rows[s] * 32, train.begin() + (size_t)seg[s] * 32);
  std::vector<int32_t> mt((size_t)n_seg * n_query), nm(n_seg);
  std::vector<float> md((size_t)n_seg * n_query);
  ctx.check(cvb_match_hamming_batch(ctx.get(), query, n_query, train.data(), seg.data(), n_seg, P.img_match_thres, P.ratio_thres,
                                    mt.data(), md.data(), nm.data()),
            "cvb_match_hamming_batch");
  std::vector<Matches> out(n_seg);
  if (discarded) discarded->assign(n_seg, false);
  for (int s = 0; s < n_seg; s++) {
    for (int q = 0; q < n_query; q++) {
      const int32_t t = mt[(size_t)s * n_query + q];
      if (t >= 0) out[s].push_back(Match{(size_t)q, (size_t)t, md[(size_t)s * n_query + q]});
    }
    const int nmatches = (int)out[s].size();
    if (discarded) {
      if (same_client[s] && nmatches < P.matches_thres) (*discarded)[s] = true;        // placerec_gen_be.cpp:118-120
      else if (nmatches < P.matches_thres_merge) (*discarded)[s] = true;               // :121-123
    }
  }
  return out;
}

// The DenseMatcher block of PlaceRecognition::ComputeSE3 (placerec_be.cpp:85-91) for all candidates at once.
inline std::vector<Matches> LandmarkMatchCandidates(Context& ctx, const uint8_t* query, const uint8_t* skip_query, int n_query,
                                                    const std::vector<const uint8_t*>& cand_desc,
                                                    const std::vector<const uint8_t*>& cand_skip, const std::vector<int>& cand_rows,
                                                    float distance_threshold = 50.0f, int num_best = 4) {
  const int n_seg = (int)cand_desc.size();
  std::vector<int32_t> seg(n_seg + 1, 0);
  for (int s = 0; s < n_seg; s++) seg[s + 1] = seg[s] + cand_rows[s];
  const size_t rows = (size_t)seg[n_seg];
  std::vector<uint8_t> B(rows * 32), skipB(rows);
  for (int s = 0; s < n_seg; s++) {
    std::copy(cand_desc[s], cand_desc[s] + (size_t)cand_rows[s] * 32, B.begin() + (size_t)seg[s] * 32);
    std::copy(cand_skip[s], cand_skip[s] + cand_rows[s], skipB.begin() + seg[s]);
  }
  std::vector<int32_t> oA(rows ? rows : 1), oB(rows ? rows : 1), n(n_seg);
  std::vector<float> oD(rows ? rows : 1);
  ctx.check(cvb_landmark_match_batch(ctx.get(), query, skip_query, n_query, B.data(), skipB.data(), seg.data(), n_seg,
                                     distance_threshold, num_best, oA.data(), oB.data(), oD.data(), n.data()),
            "cvb_landmark_match_batch");
  std::vector<Matches> out(n_seg);
  for (int s = 0; s < n_seg; s++)
    for (int m = 0; m < n[s]; m++) out[s].push_back(Match{(size_t)oA[seg[s] + m], (size_t)oB[seg[s] + m], oD[seg[s] + m]});
  return out;
}

// The SIFT branch of the same candidate loop (placerec_gen_be.cpp:86-87,99: FlannBasedMatcher::knnMatch on CV_32F 128-d
// rows; here the exact brute-force 2-NN, SURVEY §8a M2) + the same filter with the SIFT thresholds (img_match_thres /
// ratio_thres of the yaml).  descriptors row-major [n][128] float, integer-valued 0..255 as cv::xfeatures2d::SIFT emits.
inline std::vector<Matches> MatchCandidatesSIFT(Context& ctx, const float* query, int n_query, const std::vector<const float*>& cand_desc,
                                                const std::vector<int>& cand_rows, const std::vector<bool>& same_client,
                                                const OptParams& P, std::vector<bool>* discarded) {
  const int n_seg = (int)cand_desc.size();
  std::vector<int32_t> seg(n_seg + 1, 0);
  for (int s = 0; s < n_seg; s++) seg[s + 1] = seg[s] + cand_rows[s];
  std::vector<float> train((size_t)seg[n_seg] * 128);
  for (int s = 0; s < n_seg; s++) std::copy(cand_desc[s], cand_desc[s] + (size_t)cand_rows[s] * 128, train.begin() + (size_t)seg[s] * 128);
  std::vector<int32_t> mt((size_t)n_seg * n_query), nm(n_seg);
  std::vector<float> md((size_t)n_seg * n_query);
  ctx.check(cvb_match_l2_batch(ctx.get(), query, n_query, train.data(), seg.data(), n_seg, 128, P.img_match_thres, P.ratio_thres, mt.data(),
                               md.data(), nm.data()),
            "cvb_match_l2_batch");
  std::vector<Matches> out(n_seg);
  if (discarded) discarded->assign(n_seg, false);
  for (int s = 0; s < n_seg; s++) {
    for (int q = 0; q < n_query; q++) {
      const int32_t t = mt[(size_t)s * n_query + q];
      if (t >= 0) out[s].push_back(Match{(size_t)q, (size_t)t, md[(size_t)s * n_query + q]});
    }
    const int nmatches = (int)out[s].size();
    if (discarded) {
      if (same_client[s] && nmatches < P.matches_thres) (*discarded)[s] = true;
      else if (nmatches < P.matches_thres_merge) (*discarded)[s] = true;
    }
  }
  return out;
}

// estd2::DenseMatcher-shaped adaptor (include/covins/dense_matcher/DenseMatcher.hpp:49-76): the same constructor
// arguments and the same templated match(algorithm) call, consuming the reference's MatchingAlgorithm policy interface
// (include/covins/matcher/MatchingAlgorithm.h:83-152: doSetup / sizeA / sizeB / skipA / skipB / distanceThreshold /
// reserveMatches / setBestMatch).  The one thing a GPU cannot take through that interface is the virtual distance(a, b)
// call per pair, so the algorithm additionally exposes its descriptor rows:
//     const unsigned char* descriptorA(size_t i) const;   // kfPtrA_->GetDescriptor(i)  (keyframe_base.cpp:254-256)
//     const unsigned char* descriptorB(size_t i) const;
// (two one-line accessors on LandmarkMatchingAlgorithm, shown in INTEGRATION.md); distance() itself — 256-bit Hamming,
// FLT_MAX at or above the threshold, LandmarkMatchingAlgorithm.h:103-114 — is what the kernel evaluates.
// Results arrive through setBestMatch in ascending B order, exactly as DenseMatcher::matchBody emits them
// (implementation/DenseMatcher.hpp:93-121); ties resolve as with numMatcherThreads = 1.
class DenseMatcher {
 public:
  DenseMatcher(Context& ctx, unsigned char /*numMatcherThreads*/ = 8, unsigned char numBest = 4, bool useDistanceRatioThreshold = false)
      : ctx_(ctx), num_best_(numBest), use_ratio_(useDistanceRatioThreshold) {}
  template <class MATCHING_ALGORITHM_T>
  void match(MATCHING_ALGORITHM_T& algo) {
    if (use_ratio_) { std::printf("FATAL: DenseMatcher ratio mode is not used by COVINS (placerec_be.cpp:87) and not implemented\n"); std::exit(-1); }
    algo.doSetup();
    const int nA = (int)algo.sizeA(), nB = (int)algo.sizeB();
    std::vector<uint8_t> A((size_t)nA * 32), B((size_t)nB * 32), sA(nA), sB(nB);
    for (int i = 0; i < nA; i++) { sA[i] = algo.skipA(i) ? 1 : 0; std::copy(algo.descriptorA(i), algo.descriptorA(i) + 32, A.begin() + (size_t)i * 32); }
    for (int i = 0; i < nB; i++) { sB[i] = algo.skipB(i) ? 1 : 0; std::copy(algo.descriptorB(i), algo.descriptorB(i) + 32, B.begin() + (size_t)i * 32); }
    const int32_t seg[2] = {0, nB};
    std::vector<int32_t> oA(nB > 0 ? nB : 1), oB(nB > 0 ? nB : 1);
    std::vector<float> oD(nB > 0 ? nB : 1);
    int32_t n = 0;
    ctx_.check(cvb_landmark_match_batch(ctx_.get(), A.data(), sA.data(), nA, B.data(), sB.data(), seg, 1, algo.distanceThreshold(), num_best_,
                                        oA.data(), oB.data(), oD.data(), &n),
               "cvb_landmark_match_batch");
    algo.reserveMatches((size_t)n);
    for (int m = 0; m < n; m++) algo.setBestMatch((size_t)oA[m], (size_t)oB[m], (double)oD[m]);
  }

 private:
  Context& ctx_;
  int num_best_;
  bool use_ratio_;
};

// What FeatureMatcher::SearchBySE3 reads of a keyframe, with owning storage (cvb_kf_view points into it).
struct KfViewStorage {
  std::vector<float> kp, octave;
  std::vector<uint8_t> desc, lm_valid, lm_desc;
  std::vector<double> lm_pos, lm_maxdist;
  std::vector<int32_t> grid_ptr, grid_idx;
  cvb_kf_view v{};
  // KeyframeBase::AssignFeaturesToGrid (keyframe_base.cpp:122-143) on the flat arrays
  void assign_grid(double img_w, double img_h) {
    const int n = (int)(kp.size() / 2);
    v.grid_w_inv = 64.0 / img_w; v.grid_h_inv = 48.0 / img_h;
    std::vector<int> cell(n, -1);
    grid_ptr.assign(64 * 48 + 1, 0);
    for (int i = 0; i < n; i++) {
      const long px = std::lround((double)kp[2 * (size_t)i] * v.grid_w_inv), py = std::lround((double)kp[2 * (size_t)i + 1] * v.grid_h_inv);
      if (px >= 0 && px < 64 && py >= 0 && py < 48) { cell[i] = (int)(px * 48 + py); grid_ptr[cell[i] + 1]++; }   // out-of-grid cells: UB in the reference
    }
    for (int c = 0; c < 64 * 48; c++) grid_ptr[c + 1] += grid_ptr[c];
    grid_idx.assign(grid_ptr.back(), 0);
    std::vector<int32_t> fill(grid_ptr.begin(), grid_ptr.end() - 1);
    for (int i = 0; i < n; i++) if (cell[i] >= 0) grid_idx[fill[cell[i]]++] = i;
  }
  const cvb_kf_view* view() {
    v.n = (int32_t)(kp.size() / 2);
    v.kp = kp.data(); v.octave = octave.data(); v.desc = desc.data(); v.lm_valid = lm_valid.data(); v.lm_pos = lm_pos.data();
    v.lm_maxdist = lm_maxdist.data(); v.lm_desc = lm_desc.data(); v.grid_ptr = grid_ptr.data(); v.grid_idx = grid_idx.data();
    return &v;
  }
};

namespace detail {
// the flat view of a keyframe that SearchBySE3 reads (KfViewStorage)
template <class KFPtr>
inline void flatten_kf_view(const KFPtr& kf, KfViewStorage& S) {
  const size_t n = kf->keypoints_distorted_.size();
  S.kp.resize(2 * n); S.octave.resize(n); S.desc.resize(32 * n); S.lm_valid.assign(n, 0); S.lm_pos.assign(3 * n, 0.0);
  S.lm_maxdist.assign(n, 1.0); S.lm_desc.assign(32 * n, 0);
  const auto lms = kf->GetLandmarks();
  for (size_t i = 0; i < n; i++) {
    S.kp[2 * i] = kf->keypoints_distorted_[i][0]; S.kp[2 * i + 1] = kf->keypoints_distorted_[i][1];
    S.octave[i] = kf->keypoints_aors_[i][1];
    std::copy(kf->GetDescriptor(i), kf->GetDescriptor(i) + 32, S.desc.begin() + 32 * i);
    if (lms[i] && !lms[i]->IsInvalid()) {
      S.lm_valid[i] = 1;
      const auto p = lms[i]->GetWorldPos();
      for (int c = 0; c < 3; c++) S.lm_pos[3 * i + c] = p[c];
      S.lm_maxdist[i] = lms[i]->GetMaxDistance();
      std::copy(lms[i]->GetDescriptorPtr(), lms[i]->GetDescriptorPtr() + 32, S.lm_desc.begin() + 32 * i);
    }
  }
  const auto Tcw = kf->GetPoseTcw();
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) S.v.Tcw[4 * r + c] = Tcw(r, c);
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) S.v.K[3 * r + c] = kf->calibration_K(r, c);
  S.v.img[0] = kf->img_dim_x_min_; S.v.img[1] = kf->img_dim_x_max_; S.v.img[2] = kf->img_dim_y_min_; S.v.img[3] = kf->img_dim_y_max_;
  S.assign_grid(kf->image_width(), kf->image_height());
}
}  // namespace detail

// FeatureMatcher::SearchBySE3(pKF1, pKF2, matches12, T12, th) (feature_matcher_be.cpp:293-498) for a batch of candidates:
// matches12[p] is updated in place exactly as the reference does (:485-496: matches12[i] = mapPoints2[idx2]); returns the
// number of matches found per candidate.  KF is touched through the member names the reference class has
// (keypoints_distorted_, keypoints_aors_, GetDescriptor(i), GetLandmarks(), calibration via Adapter<KF>::K, GetPoseTcw(),
// img_dim_*_); Landmark through IsInvalid / GetWorldPos / GetMaxDistance / GetDescriptorPtr / GetFeatureIndex.  GetMaxDistance() is
// the ONE getter a maintainer adds to LandmarkBase: PredictScale (landmark_base.cpp:120-133) divides the raw max_distance_
// (protected, landmark_base.hpp:107), and GetMaxDistanceInvariance() returns 1.2 x that (landmark_base.cpp:68-71).
template <class KFPtr, class LandmarkVector, class Transform4>
inline std::vector<int> SearchBySE3(Context& ctx, const KFPtr& kf1, const std::vector<KFPtr>& kf2, std::vector<LandmarkVector>& matches12,
                                    const std::vector<Transform4>& T12, const std::vector<Transform4>& T21, double th,
                                    int desc_matching_th_low, int num_octaves, double scale_factor) {
  const auto flatten = [](const KFPtr& kf, KfViewStorage& S) { detail::flatten_kf_view(kf, S); };
  const int n_pairs = (int)kf2.size();
  KfViewStorage S1;
  flatten(kf1, S1);
  std::vector<KfViewStorage> S2(n_pairs);
  std::vector<cvb_kf_view> v2(n_pairs);
  const size_t n1 = kf1->keypoints_distorted_.size();
  std::vector<uint8_t> a1((size_t)n_pairs * n1, 0), a2;
  std::vector<double> t12((size_t)n_pairs * 16), t21((size_t)n_pairs * 16);
  for (int p = 0; p < n_pairs; p++) {
    flatten(kf2[p], S2[p]);
    v2[p] = *S2[p].view();
    const size_t n2 = kf2[p]->keypoints_distorted_.size(), base = a2.size();
    a2.resize(base + n2, 0);
    for (size_t i = 0; i < n1; i++)                                                                // :312-324
      if (matches12[p][i]) {
        a1[(size_t)p * n1 + i] = 1;
        const int idx2 = matches12[p][i]->GetFeatureIndex(kf2[p]);
        if (idx2 >= 0 && idx2 < (int)n2) a2[base + idx2] = 1;
      }
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) { t12[(size_t)p * 16 + 4 * r + c] = T12[p](r, c); t21[(size_t)p * 16 + 4 * r + c] = T21[p](r, c); }
  }
  cvb_search_params prm{th, desc_matching_th_low, num_octaves, scale_factor};
  std::vector<int32_t> m12((size_t)n_pairs * n1 + 1), nf(n_pairs + 1);
  ctx.check(cvb_search_by_se3_batch(ctx.get(), S1.view(), v2.data(), n_pairs, t12.data(), t21.data(), a1.data(), a2.data(), &prm, m12.data(),
                                    nf.data(), nullptr, nullptr),
            "cvb_search_by_se3_batch");
  std::vector<int> found(n_pairs);
  for (int p = 0; p < n_pairs; p++) {
    const auto lms2 = kf2[p]->GetLandmarks();
    for (size_t i = 0; i < n1; i++)
      if (m12[(size_t)p * n1 + i] >= 0) matches12[p][i] = lms2[m12[(size_t)p * n1 + i]];            // :491
    found[p] = nf[p];
  }
  return found;
}

// The parameters of the COVINS verification (placerec_be.cpp:85-151 and the settings it reads).
struct LandmarkVerifyParams {
  float distance_threshold = 50.0f;   // LandmarkMatchingAlgorithm(50.0)
  int num_best = 4;                   // DenseMatcher numBest
  int matches_thres = 25;             // the nmatches discard (:93-99)
  double ransac_threshold = 0.0;      // Se3Solver's RANSAC threshold
  int ransac_max_iterations = 0;
  double ransac_probability = 0.99;
  int min_ransac_inliers = 0;         // the gate after the RANSAC
  double search_radius_SE3 = 9.5;     // SearchBySE3
  int desc_matching_th_low = 50;
  int num_octaves = 1;
  double scale_factor = 2.0;
  double th_outlier_align = 1.3;      // OptimizeRelativePose
};
template <class Transform4>
struct LandmarkVerifyOutcome {
  int n_matches = 0, best_sample = -1, best_count = 0, n_found = 0, n_corr = 0, n_inliers = 0;
  double T12_pose[7] = {0, 0, 0, 0, 0, 0, 0};   // [qx,qy,qz,qw, x,y,z] after OptimizeRelativePose (the start pose when n_inliers == 0)
  Transform4 T12;                                // refined when n_inliers > 0, else as handed to the refinement (zero if the candidate stopped)
};

// The candidate loop of PlaceRecognition::ComputeSE3 (placerec_be.cpp:85-151: DenseMatcher, the nmatches discard,
// Se3Solver::projectiveAlignment, SearchBySE3, OptimizeRelativePose) for every candidate of kf_query in one call
// (cvb_verify_landmark_candidates_seeded_batch).  vvpMapPointMatches[c] is written as the reference holds it after
// OptimizeRelativePose: kf_query's keypoint i -> the candidate's landmark (GetLandmarks()[b]) of the LandmarkVector handed to the
// refinement, with the reference's purge quirk applied (matches1[r] = nullptr for every purged RESIDUAL index r,
// optimization_be.cpp:815); all null for a candidate that stops before SearchBySE3.  The acceptance test stays with the caller.
// Members used beyond SearchBySE3's: KF::GetPoseTws / GetStateExtrinsics and, through Adapter<KF>, the camera, its model and the
// query's bearing vectors and sigma angles (Adapter<KF>::bearings).
template <class KFPtr, class LandmarkVector, class Transform4>
inline std::vector<LandmarkVerifyOutcome<Transform4>> VerifyLandmarkCandidates(Context& ctx, const KFPtr& kf_query, const std::vector<KFPtr>& candidates,
                                                                               std::vector<LandmarkVector>& vvpMapPointMatches,
                                                                               const LandmarkVerifyParams& P, const std::vector<uint64_t>& seeds) {
  using KF = typename std::decay<decltype(*kf_query)>::type;
  const int C = (int)candidates.size();
  if ((int)seeds.size() != C) {
    std::printf("FATAL: VerifyLandmarkCandidates: %d seeds for %d candidates\n", (int)seeds.size(), C);
    std::exit(-1);
  }
  const auto fill = [](const KFPtr& kf, KfViewStorage& S, cvb_landmark_kf& k) {
    detail::flatten_kf_view(kf, S);
    k.view = *S.view();
    const auto Tws = kf->GetPoseTws(), Tsc = kf->GetStateExtrinsics();
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) { k.T_ws[4 * r + c] = Tws(r, c); k.T_sc[4 * r + c] = Tsc(r, c); }
    if (!Adapter<KF>::camera(*kf, k.intr, k.dist)) {
      std::printf("FATAL: Unknown projection type.\n");                                              // optimization_be.cpp:705-707
      std::exit(-1);
    }
    Adapter<KF>::camera_model(*kf, &k.cam_model, &k.dist_model, &k.xi);
  };
  KfViewStorage Sq;
  cvb_landmark_kf q{};
  fill(kf_query, Sq, q);
  const int nq = q.view.n;
  std::vector<double> bear(3 * (size_t)nq), sig((size_t)nq);
  Adapter<KF>::bearings(*kf_query, bear.data(), sig.data());
  q.bearings = bear.data(); q.sigma_angle = sig.data();
  std::vector<KfViewStorage> S(C);
  std::vector<cvb_landmark_kf> cand(C > 0 ? C : 1);
  for (int c = 0; c < C; c++) fill(candidates[c], S[c], cand[c]);
  cvb_landmark_verify_params prm{P.distance_threshold, P.num_best, P.matches_thres, P.ransac_threshold, P.ransac_max_iterations,
                                 P.ransac_probability, P.min_ransac_inliers,
                                 {P.search_radius_SE3, P.desc_matching_th_low, P.num_octaves, P.scale_factor}, P.th_outlier_align};
  const size_t Cn = C > 0 ? (size_t)C : 1, L = (size_t)C * nq + 1;
  std::vector<int32_t> n_matches(Cn), best_sample(Cn), best_count(Cn), iterations(Cn), consumed(Cn), n_found(Cn), n_corr(Cn), n_inliers(Cn),
      solve_it(2 * Cn), match12(L);
  std::vector<double> best_model(12 * Cn), T12(16 * Cn), T21(16 * Cn), T12_out(7 * Cn);
  std::vector<uint8_t> stage(L), removed(L);
  cvb_landmark_verify_result res{n_matches.data(), best_sample.data(), best_model.data(), best_count.data(), iterations.data(), consumed.data(),
                                 T12.data(), T21.data(), n_found.data(), n_corr.data(), T12_out.data(), n_inliers.data(), solve_it.data(),
                                 match12.data(), stage.data(), removed.data()};
  ctx.check(cvb_verify_landmark_candidates_seeded_batch(ctx.get(), &q, cand.data(), C, &prm, seeds.data(), &res),
            "cvb_verify_landmark_candidates_seeded_batch");
  vvpMapPointMatches.assign(C, LandmarkVector(nq));
  std::vector<LandmarkVerifyOutcome<Transform4>> out(C);
  for (int c = 0; c < C; c++) {
    const auto lms2 = candidates[c]->GetLandmarks();
    LandmarkVector& v = vvpMapPointMatches[c];
    for (int i = 0; i < nq; i++) {
      const int32_t b = match12[(size_t)c * nq + i];
      if (b >= 0) v[i] = lms2[b];
    }
    for (int r = 0; r < n_corr[c]; r++)
      if (removed[(size_t)c * nq + r]) v[r] = nullptr;                                               // matches1[r], r = residual index (:815)
    auto& o = out[c];
    o.n_matches = n_matches[c]; o.best_sample = best_sample[c]; o.best_count = best_count[c]; o.n_found = n_found[c];
    o.n_corr = n_corr[c]; o.n_inliers = n_inliers[c];
    for (int k = 0; k < 7; k++) o.T12_pose[k] = T12_out[7 * (size_t)c + k];
    if (o.n_inliers > 0) {
      o.T12 = detail::pose7_to_transform<Transform4>(o.T12_pose);                                  // :829
    } else {
      o.T12 = Transform4::Identity();
      for (int r = 0; r < 4; r++) for (int k = 0; k < 4; k++) o.T12(r, k) = T12[16 * (size_t)c + 4 * r + k];
    }
  }
  return out;
}

// FeatureMatcher::SearchByProjection(pKF, Tcw, vpPoints, vpMatched, th) (feature_matcher_be.cpp:168-291): loop landmarks projected
// into a keyframe.  The kernel returns, in list order, the decision the reference's sequential loop takes for every landmark
// (cvb_search_by_projection); this wrapper flattens the containers and replays the decisions on them: a new match goes into
// vpMatched, a better keypoint for an already observed landmark becomes pKF->RemapLandmark(pMP, existing, best).  Returns nmatches.
// Members used beyond SearchBySE3's: KF::GetLandmark(i), KF::RemapLandmark; Landmark::GetNormal / GetMinDistanceInvariance /
// GetMaxDistanceInvariance / GetMaxDistance.  Camera: Adapter<KF>::camera (+ camera_model for the non-pinhole/radtan types).
template <class KFPtr, class LandmarkVector, class Transform4>
inline int SearchByProjection(Context& ctx, const KFPtr& pKF, const Transform4& Tcw, const LandmarkVector& vpPoints, LandmarkVector& vpMatched,
                              double th, int desc_matching_th_low, int num_octaves, double scale_factor) {
  using KF = typename std::remove_reference<decltype(*pKF)>::type;
  using LmPtr = typename std::remove_reference<decltype(vpPoints[0])>::type;
  const size_t n = pKF->keypoints_distorted_.size(), m = vpPoints.size();
  KfViewStorage S;
  S.kp.resize(2 * n); S.octave.resize(n); S.desc.resize(32 * n); S.lm_valid.assign(n, 0); S.lm_pos.assign(3 * n, 0.0);
  S.lm_maxdist.assign(n, 1.0); S.lm_desc.assign(32 * n, 0);
  std::map<const void*, int> index_of;                     // landmark object → first position in vpPoints
  for (size_t i = 0; i < m; i++)
    if (vpPoints[i]) index_of.emplace((const void*)&*vpPoints[i], (int)i);
  std::vector<int32_t> kf_lm_cand(n ? n : 1, -1);
  std::vector<uint8_t> matched(n ? n : 1, 0);
  std::set<const void*> already;                          // spAlreadyFound (:175-177)
  for (size_t i = 0; i < n; i++) {
    S.kp[2 * i] = pKF->keypoints_distorted_[i][0]; S.kp[2 * i + 1] = pKF->keypoints_distorted_[i][1];
    S.octave[i] = pKF->keypoints_aors_[i][1];
    std::copy(pKF->GetDescriptor(i), pKF->GetDescriptor(i) + 32, S.desc.begin() + 32 * i);
    const auto lm = pKF->GetLandmark(i);
    if (lm) {                                             // pKF->GetLandmark(bestIdx) != nullptr (:268); invalid ones count too
      S.lm_valid[i] = 1;
      const auto it = index_of.find((const void*)&*lm);
      if (it != index_of.end()) kf_lm_cand[i] = it->second;
    }
    if (i < vpMatched.size() && vpMatched[i]) { matched[i] = 1; already.insert((const void*)&*vpMatched[i]); }
  }
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) S.v.Tcw[4 * r + c] = Tcw(r, c);
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) S.v.K[3 * r + c] = pKF->calibration_K(r, c);
  S.v.img[0] = pKF->img_dim_x_min_; S.v.img[1] = pKF->img_dim_x_max_; S.v.img[2] = pKF->img_dim_y_min_; S.v.img[3] = pKF->img_dim_y_max_;
  S.assign_grid(pKF->image_width(), pKF->image_height());
  std::vector<uint8_t> valid(m ? m : 1, 0), desc(32 * (m ? m : 1), 0);
  std::vector<double> pos(3 * (m ? m : 1), 0.0), normal(3 * (m ? m : 1), 0.0), dmin(m ? m : 1, 0.0), dmax(m ? m : 1, 0.0), dist0(m ? m : 1, 1.0);
  std::vector<int32_t> feat(m ? m : 1, -1);
  for (size_t i = 0; i < m; i++) {
    const LmPtr& lm = vpPoints[i];
    if (!lm || lm->IsInvalid() || already.count((const void*)&*lm)) continue;                        // :184-187
    valid[i] = 1;
    const auto p = lm->GetWorldPos(), nn = lm->GetNormal();
    for (int c = 0; c < 3; c++) { pos[3 * i + c] = p[c]; normal[3 * i + c] = nn[c]; }
    dmin[i] = lm->GetMinDistanceInvariance(); dmax[i] = lm->GetMaxDistanceInvariance(); dist0[i] = lm->GetMaxDistance();
    std::copy(lm->GetDescriptorPtr(), lm->GetDescriptorPtr() + 32, desc.begin() + 32 * i);
    feat[i] = lm->GetFeatureIndex(pKF);
  }
  double intr[4], dist[4], xi = 0.0, tcw[16];
  int cam_model = 0, dist_model = 0;
  Adapter<KF>::camera(*pKF, intr, dist);
  Adapter<KF>::camera_model(*pKF, &cam_model, &dist_model, &xi);
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) tcw[4 * r + c] = Tcw(r, c);
  cvb_proj_landmarks L{(int32_t)m, valid.data(), pos.data(), normal.data(), dmin.data(), dmax.data(), dist0.data(), desc.data(), feat.data()};
  cvb_search_params prm{th, desc_matching_th_low, num_octaves, scale_factor};
  std::vector<int32_t> action(m ? m : 1, 0), best(m ? m : 1, -1);
  int32_t nmatches = 0;
  ctx.check(cvb_search_by_projection(ctx.get(), S.view(), kf_lm_cand.data(), tcw, intr, dist, cam_model, dist_model, xi, &L, matched.data(), &prm,
                                     action.data(), best.data(), &nmatches),
            "cvb_search_by_projection");
  if (vpMatched.size() < n) vpMatched.resize(n);
  for (size_t i = 0; i < m; i++) {                                                                    // the decisions, in list order
    if (action[i] == 1) vpMatched[best[i]] = vpPoints[i];                                              // :285
    else if (action[i] == 2) pKF->RemapLandmark(vpPoints[i], (size_t)vpPoints[i]->GetFeatureIndex(pKF), (size_t)best[i]);   // :281
  }
  return nmatches;
}

// RANSAC hypothesis scoring (the countWithinDistance / selectWithinDistance inner loops of opengv::sac::Ransac for
// Se3Solver::projectiveAlignment, Se3Solver.cpp:59-110, and RelNonCentralPosSolver::computePose, :343-377) — all
// hypotheses of one RANSAC run in one launch; sampling and the minimal solvers (GP3P / 5-pt / 17-pt) stay with opengv.
// models: n_hyp x 12 (3x4 row-major).  Returns the inlier count per hypothesis; inlier (optional) n_hyp x n flags.
inline std::vector<int> ScoreAbsolutePoseHypotheses(Context& ctx, const std::vector<double>& models, const std::vector<double>& points,
                                                    const std::vector<double>& bearings, const std::vector<double>& sigma_angles,
                                                    const double cam_offset[3], const double cam_rotation[9], double threshold,
                                                    std::vector<uint8_t>* inlier = nullptr) {
  const int n_hyp = (int)(models.size() / 12), n = (int)sigma_angles.size();
  std::vector<int32_t> cnt(n_hyp > 0 ? n_hyp : 1);
  if (inlier) inlier->assign((size_t)n_hyp * n, 0);
  ctx.check(cvb_score_absolute_pose_batch(ctx.get(), models.data(), n_hyp, points.data(), bearings.data(), sigma_angles.data(), n, cam_offset,
                                          cam_rotation, threshold, nullptr, inlier ? inlier->data() : nullptr, cnt.data()),
            "cvb_score_absolute_pose_batch");
  return std::vector<int>(cnt.begin(), cnt.begin() + n_hyp);
}
inline std::vector<int> ScoreRelativePoseHypotheses(Context& ctx, const std::vector<double>& models, const std::vector<double>& bearings1,
                                                    const std::vector<double>& bearings2, const std::vector<double>& sigma1,
                                                    const std::vector<double>& sigma2, double threshold, std::vector<uint8_t>* inlier = nullptr) {
  const int n_hyp = (int)(models.size() / 12), n = (int)sigma1.size();
  std::vector<int32_t> cnt(n_hyp > 0 ? n_hyp : 1);
  if (inlier) inlier->assign((size_t)n_hyp * n, 0);
  ctx.check(cvb_score_relative_pose_batch(ctx.get(), models.data(), n_hyp, bearings1.data(), bearings2.data(), sigma1.data(), sigma2.data(), n,
                                          threshold, nullptr, inlier ? inlier->data() : nullptr, cnt.data()),
            "cvb_score_relative_pose_batch");
  return std::vector<int>(cnt.begin(), cnt.begin() + n_hyp);
}

// The whole GP3P RANSAC of Se3Solver::projectiveAlignment (Se3Solver.cpp:59-110) for a batch of candidate keyframes in one
// call (cvb_ransac_absolute_pose_batch): P3P hypothesis per sample, scoring and opengv's sequential model selection on the GPU.
// Per problem: its correspondences (as ScoreAbsolutePoseHypotheses), its camera in the body frame and its samples (4 local
// indices each; every problem of a call has the same number of samples, e.g. max_iterations plus headroom for skipped ones).
struct AbsolutePoseRansacProblem {
  std::vector<double> points, bearings, sigma_angles;   // 3n, 3n, n
  double cam_offset[3] = {0, 0, 0};
  double cam_rotation[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};   // row-major
  std::vector<int32_t> samples;                          // 4 * n_samples
};
struct AbsolutePoseRansacResult {
  int best_sample = -1;             // -1: no model
  std::array<double, 12> model{};   // 3x4 [R|t] row-major, body in world
  int n_inliers = 0, iterations = 0, samples_used = 0;
  std::vector<uint8_t> inliers;     // n flags of the selected model
};
namespace detail {
// one RANSAC call fn on the flattened problems P (ptr: their correspondence ranges) → the per-problem results (Out:
// AbsolutePoseRansacResult or NonCentralRelativePoseRansacResult)
// call(&R) runs the RANSAC call into the result struct R
template <class Out, class Result, class Call>
std::vector<Out> ransac_results(const std::vector<int32_t>& ptr, const Call& call) {
  const int n_prob = (int)ptr.size() - 1;
  const size_t m = n_prob > 0 ? n_prob : 1;
  std::vector<int32_t> best(m), cnt(m), iters(m), used(m);
  std::vector<double> models(12 * m);
  std::vector<uint8_t> mask(ptr[n_prob] > 0 ? ptr[n_prob] : 1);
  Result R{best.data(), models.data(), cnt.data(), iters.data(), used.data(), mask.data(), nullptr, nullptr, nullptr};
  call(&R);
  std::vector<Out> out(n_prob);
  for (int i = 0; i < n_prob; i++) {
    out[i].best_sample = best[i]; out[i].n_inliers = cnt[i]; out[i].iterations = iters[i]; out[i].samples_used = used[i];
    std::copy(models.begin() + 12 * i, models.begin() + 12 * (i + 1), out[i].model.begin());
    out[i].inliers.assign(mask.begin() + ptr[i], mask.begin() + ptr[i + 1]);
  }
  return out;
}
template <class Out, class Problems, class Result>
std::vector<Out> ransac(Context& ctx, int (*fn)(cvb_ctx*, const Problems*, double, int, double, Result*), const char* what, const Problems& P,
                        const std::vector<int32_t>& ptr, double threshold, int max_iterations, double probability) {
  return ransac_results<Out, Result>(ptr, [&](Result* R) { ctx.check(fn(ctx.get(), &P, threshold, max_iterations, probability, R), what); });
}
// the seeded form: P.samples = NULL, one seed per problem
template <class Out, class Problems, class Result>
std::vector<Out> ransac_seeded(Context& ctx, int (*fn)(cvb_ctx*, const Problems*, const uint64_t*, double, int, double, Result*, int32_t*),
                               const char* what, const Problems& P, const std::vector<int32_t>& ptr, const std::vector<uint64_t>& seeds,
                               double threshold, int max_iterations, double probability) {
  if (seeds.size() != ptr.size() - 1) throw std::invalid_argument(std::string("covins_b200: ") + what + ": one seed per problem");
  return ransac_results<Out, Result>(
      ptr, [&](Result* R) { ctx.check(fn(ctx.get(), &P, seeds.data(), threshold, max_iterations, probability, R, nullptr), what); });
}
// every problem's samples left empty, as the seeded calls require
template <class Problem>
void require_no_samples(const std::vector<Problem>& problems, const char* what) {
  for (const Problem& p : problems)
    if (!p.samples.empty()) throw std::invalid_argument(std::string("covins_b200::") + what + ": the seeded form draws the samples; leave them empty");
}
// a batch of absolute-pose problems flattened into the arrays of cvb_abs_ransac_problems
struct FlatAbsProblems {
  std::vector<int32_t> ptr, samples;
  std::vector<double> pts, f, sigma, cam_off, cam_rot;
  int32_t n_samples = 0;
  cvb_abs_ransac_problems view() const {
    return cvb_abs_ransac_problems{(int32_t)ptr.size() - 1, ptr.data(), pts.data(), f.data(), sigma.data(), cam_off.data(), cam_rot.data(),
                                   samples.empty() ? nullptr : samples.data(), n_samples};
  }
};
inline FlatAbsProblems flatten_abs_problems(const std::vector<AbsolutePoseRansacProblem>& problems) {
  const int n_prob = (int)problems.size();
  FlatAbsProblems F;
  const size_t n_samples = n_prob ? problems[0].samples.size() / 4 : 0;
  F.n_samples = (int32_t)n_samples;
  F.ptr.assign(n_prob + 1, 0);
  for (int i = 0; i < n_prob; i++) {
    const AbsolutePoseRansacProblem& p = problems[i];
    if (p.samples.size() != 4 * n_samples || p.points.size() != 3 * p.sigma_angles.size() || p.bearings.size() != 3 * p.sigma_angles.size())
      throw std::invalid_argument("covins_b200::RansacAbsolutePose: inconsistent problem sizes");
    F.ptr[i + 1] = F.ptr[i] + (int32_t)p.sigma_angles.size();
    F.pts.insert(F.pts.end(), p.points.begin(), p.points.end());
    F.f.insert(F.f.end(), p.bearings.begin(), p.bearings.end());
    F.sigma.insert(F.sigma.end(), p.sigma_angles.begin(), p.sigma_angles.end());
    F.cam_off.insert(F.cam_off.end(), p.cam_offset, p.cam_offset + 3);
    F.cam_rot.insert(F.cam_rot.end(), p.cam_rotation, p.cam_rotation + 9);
    F.samples.insert(F.samples.end(), p.samples.begin(), p.samples.end());
  }
  return F;
}
}  // namespace detail
inline std::vector<AbsolutePoseRansacResult> RansacAbsolutePose(Context& ctx, const std::vector<AbsolutePoseRansacProblem>& problems, double threshold,
                                                                 int max_iterations, double probability = 0.99) {
  const detail::FlatAbsProblems F = detail::flatten_abs_problems(problems);
  return detail::ransac<AbsolutePoseRansacResult>(ctx, cvb_ransac_absolute_pose_batch, "cvb_ransac_absolute_pose_batch", F.view(), F.ptr, threshold,
                                                  max_iterations, probability);
}
// The same RANSAC with the samples drawn on the GPU (cvb_ransac_absolute_pose_seeded_batch): one seed per problem (e.g. from
// std::random_device, or fixed for reproducible runs), every problem's samples left empty.  The selection draws until opengv's
// bound ends it; a problem with fewer than 4 correspondences draws nothing (best_sample = -1, iterations = samples_used = 0).
inline std::vector<AbsolutePoseRansacResult> RansacAbsolutePose(Context& ctx, const std::vector<AbsolutePoseRansacProblem>& problems,
                                                                 const std::vector<uint64_t>& seeds, double threshold, int max_iterations,
                                                                 double probability = 0.99) {
  detail::require_no_samples(problems, "RansacAbsolutePose");
  const detail::FlatAbsProblems F = detail::flatten_abs_problems(problems);
  return detail::ransac_seeded<AbsolutePoseRansacResult>(ctx, cvb_ransac_absolute_pose_seeded_batch, "cvb_ransac_absolute_pose_seeded_batch", F.view(),
                                                         F.ptr, seeds, threshold, max_iterations, probability);
}

// The 17-point non-central relative-pose RANSAC of RelNonCentralPosSolver::computeNonCentralRelPose (RelNonCentralPosSolver.cpp:
// 146-173) for a batch of candidates in one call (cvb_ransac_noncentral_relative_pose_batch): 17-point hypothesis per sample,
// scoring per camera pair and opengv's sequential model selection on the GPU.  Per problem: its correspondences (bearings in
// their cameras' frames, sigmas, the camera of each side), its two rigs (at most CVB_REL_MAX_CAMS cameras each, in the rig
// frame) and its samples (17 local indices each; every problem of a call has the same number of samples).
struct NonCentralRelativePoseRansacProblem {
  std::vector<double> bearings1, bearings2, sigma1, sigma2;   // 3n, 3n, n, n
  std::vector<int32_t> cam1, cam2;                            // n camera indices into rig 1 / rig 2
  std::vector<double> rig1_offsets, rig1_rotations;           // 3 / 9 (row-major) per camera of rig 1
  std::vector<double> rig2_offsets, rig2_rotations;
  std::vector<int32_t> samples;                               // 17 * n_samples
};
struct NonCentralRelativePoseRansacResult {
  int best_sample = -1;             // -1: no model
  std::array<double, 12> model{};   // 3x4 [R|t] row-major, X1 = R X2 + t (rig frames)
  int n_inliers = 0, iterations = 0, samples_used = 0;
  std::vector<uint8_t> inliers;     // n flags of the selected model
};
namespace detail {
// a batch of non-central problems flattened into the arrays of cvb_rel_ransac_problems
struct FlatRelProblems {
  std::vector<int32_t> ptr, cp1, cp2, cam1, cam2, samples;
  std::vector<double> f1, f2, s1, s2, co1, cr1, co2, cr2;
  int32_t n_samples = 0;
  cvb_rel_ransac_problems view() const {
    return cvb_rel_ransac_problems{(int32_t)ptr.size() - 1, ptr.data(), f1.data(), f2.data(), s1.data(), s2.data(), cam1.data(), cam2.data(),
                                   cp1.data(), co1.data(), cr1.data(), cp2.data(), co2.data(), cr2.data(), samples.empty() ? nullptr : samples.data(),
                                   n_samples};
  }
};
inline FlatRelProblems flatten_rel_problems(const std::vector<NonCentralRelativePoseRansacProblem>& problems, const char* what) {
  const int n_prob = (int)problems.size();
  FlatRelProblems F;
  const size_t n_samples = n_prob ? problems[0].samples.size() / 17 : 0;
  F.n_samples = (int32_t)n_samples;
  F.ptr.assign(n_prob + 1, 0); F.cp1.assign(n_prob + 1, 0); F.cp2.assign(n_prob + 1, 0);
  for (int i = 0; i < n_prob; i++) {
    const NonCentralRelativePoseRansacProblem& p = problems[i];
    const size_t n = p.sigma1.size();
    if (p.samples.size() != 17 * n_samples || p.bearings1.size() != 3 * n || p.bearings2.size() != 3 * n || p.sigma2.size() != n ||
        p.cam1.size() != n || p.cam2.size() != n || p.rig1_rotations.size() != 3 * p.rig1_offsets.size() ||
        p.rig2_rotations.size() != 3 * p.rig2_offsets.size() || p.rig1_offsets.size() % 3 || p.rig2_offsets.size() % 3)
      throw std::invalid_argument(std::string("covins_b200::") + what + ": inconsistent problem sizes");
    F.ptr[i + 1] = F.ptr[i] + (int32_t)n;
    F.cp1[i + 1] = F.cp1[i] + (int32_t)(p.rig1_offsets.size() / 3);
    F.cp2[i + 1] = F.cp2[i] + (int32_t)(p.rig2_offsets.size() / 3);
    F.f1.insert(F.f1.end(), p.bearings1.begin(), p.bearings1.end()); F.f2.insert(F.f2.end(), p.bearings2.begin(), p.bearings2.end());
    F.s1.insert(F.s1.end(), p.sigma1.begin(), p.sigma1.end()); F.s2.insert(F.s2.end(), p.sigma2.begin(), p.sigma2.end());
    F.cam1.insert(F.cam1.end(), p.cam1.begin(), p.cam1.end()); F.cam2.insert(F.cam2.end(), p.cam2.begin(), p.cam2.end());
    F.co1.insert(F.co1.end(), p.rig1_offsets.begin(), p.rig1_offsets.end()); F.cr1.insert(F.cr1.end(), p.rig1_rotations.begin(), p.rig1_rotations.end());
    F.co2.insert(F.co2.end(), p.rig2_offsets.begin(), p.rig2_offsets.end()); F.cr2.insert(F.cr2.end(), p.rig2_rotations.begin(), p.rig2_rotations.end());
    F.samples.insert(F.samples.end(), p.samples.begin(), p.samples.end());
  }
  return F;
}
}  // namespace detail

inline std::vector<NonCentralRelativePoseRansacResult> RansacNonCentralRelativePose(Context& ctx,
                                                                                   const std::vector<NonCentralRelativePoseRansacProblem>& problems,
                                                                                   double threshold, int max_iterations, double probability = 0.99) {
  const detail::FlatRelProblems F = detail::flatten_rel_problems(problems, "RansacNonCentralRelativePose");
  return detail::ransac<NonCentralRelativePoseRansacResult>(ctx, cvb_ransac_noncentral_relative_pose_batch, "cvb_ransac_noncentral_relative_pose_batch",
                                                            F.view(), F.ptr, threshold, max_iterations, probability);
}
// The same RANSAC with the samples drawn on the GPU (cvb_ransac_noncentral_relative_pose_seeded_batch): one seed per problem,
// every problem's samples left empty (as RansacAbsolutePose's seeded form).
inline std::vector<NonCentralRelativePoseRansacResult> RansacNonCentralRelativePose(Context& ctx,
                                                                                   const std::vector<NonCentralRelativePoseRansacProblem>& problems,
                                                                                   const std::vector<uint64_t>& seeds, double threshold,
                                                                                   int max_iterations, double probability = 0.99) {
  detail::require_no_samples(problems, "RansacNonCentralRelativePose");
  const detail::FlatRelProblems F = detail::flatten_rel_problems(problems, "RansacNonCentralRelativePose");
  return detail::ransac_seeded<NonCentralRelativePoseRansacResult>(ctx, cvb_ransac_noncentral_relative_pose_seeded_batch,
                                                                   "cvb_ransac_noncentral_relative_pose_seeded_batch", F.view(), F.ptr, seeds, threshold,
                                                                   max_iterations, probability);
}

// RelNonCentralPosSolver::computeNonCentralRelPose's whole verification of a query keyframe's candidates in one call
// (cvb_verify_noncentral_relative_pose_seeded_batch): per pairing the ORB matching and a seeded 5-point RANSAC, per candidate a
// seeded 17-point RANSAC on the pairings' 5-point inliers and the seeded covariance, with one upload and one download.
// keyframes: flat views of every keyframe the rigs use (n rows of descriptors_add_ [32], bearings_add_ [3] and sigma each);
// a pairing names two of them and their cameras in the candidate's rigs.  One seed per pairing (seeds5) and per candidate.
struct VerifyKeyframeView {
  const uint8_t* desc; const double* bearings; const double* sigma; int n;
};
struct VerifyPairing { int kf1, kf2, cam1, cam2; };
struct VerifyCandidate {
  std::vector<double> rig1_offsets, rig1_rotations, rig2_offsets, rig2_rotations;   // 3 / 9 (row-major) per camera
  std::vector<VerifyPairing> pairings;
};
struct VerifyParams {
  float img_match_thres = 0.f, ratio_thres = 0.f;
  double threshold5 = 0.0; int max_iterations5 = 0;
  double threshold17 = 0.0; int max_iterations17 = 0;
  double probability = 0.99; int n_cov_samples = 300;
};
struct VerifyPairingResult {
  int n_matches = 0, best_sample = -1, n_inliers = 0, iterations = 0, samples_used = 0;
  std::array<double, 12> model{};   // 5-point [R|t], |t| = 1
};
struct VerifyCandidateResult {
  int best_sample = -1, n_inliers = 0, iterations = 0, samples_used = 0, n_valid = 0;
  std::array<double, 12> model{};   // 17-point [R|t], X1 = R X2 + t (rig frames)
  std::array<double, 36> cov{};
};
struct VerifyCorrespondence { int pairing, row1, row2, inlier5, inlier17; };
struct VerifyResult {
  std::vector<VerifyPairingResult> pairings;            // all candidates' pairings in order
  std::vector<VerifyCandidateResult> candidates;
  std::vector<VerifyCorrespondence> correspondences;    // every match, pairing then match order
};

// The same with SIFT descriptors (cvb_verify_noncentral_relative_pose_sift_seeded_batch): n rows of descriptors_add_ [128] as
// CV_32F, integer-valued in [0, 255] as cv::xfeatures2d::SIFT writes them; each pairing is matched by exact L2 2-NN + the filter.
struct VerifyKeyframeViewSIFT {
  const float* desc; const double* bearings; const double* sigma; int n;
};

namespace detail {
// the keyframe table of VerifyNonCentralRelativePose: the views' rows concatenated, kDim descriptor elements per row
template <size_t kDim, class View, class T>
void flatten_verify_keyframes(const std::vector<View>& keyframes, std::vector<int32_t>& kf_ptr, std::vector<T>& desc, std::vector<double>& bear,
                              std::vector<double>& sig) {
  kf_ptr.assign(keyframes.size() + 1, 0);
  for (size_t k = 0; k < keyframes.size(); k++) {
    const View& v = keyframes[k];
    kf_ptr[k + 1] = kf_ptr[k] + v.n;
    desc.insert(desc.end(), v.desc, v.desc + kDim * (size_t)v.n);
    bear.insert(bear.end(), v.bearings, v.bearings + 3 * (size_t)v.n);
    sig.insert(sig.end(), v.sigma, v.sigma + v.n);
  }
}

// the candidates, rigs, parameters and results of VerifyNonCentralRelativePose around one C call: call(D, prm, R) runs it on
// them (kf_ptr: the keyframe table's row offsets, which size the correspondence list)
template <class Call>
VerifyResult verify_noncentral(const std::vector<int32_t>& kf_ptr, const std::vector<VerifyCandidate>& candidates, const VerifyParams& params,
                               const std::vector<uint64_t>& seeds5, const std::vector<uint64_t>& seeds, const Call& call) {
  const int n_kf = (int)kf_ptr.size() - 1, C = (int)candidates.size();
  std::vector<int32_t> cp1(C + 1, 0), cp2(C + 1, 0), pair_ptr(C + 1, 0), pairs;
  std::vector<double> co1, cr1, co2, cr2;
  size_t bound = 0;
  for (int c = 0; c < C; c++) {
    const VerifyCandidate& cd = candidates[c];
    if (cd.rig1_rotations.size() != 3 * cd.rig1_offsets.size() || cd.rig2_rotations.size() != 3 * cd.rig2_offsets.size() ||
        cd.rig1_offsets.size() % 3 || cd.rig2_offsets.size() % 3)
      throw std::invalid_argument("covins_b200::VerifyNonCentralRelativePose: inconsistent rig sizes");
    cp1[c + 1] = cp1[c] + (int32_t)(cd.rig1_offsets.size() / 3); cp2[c + 1] = cp2[c] + (int32_t)(cd.rig2_offsets.size() / 3);
    co1.insert(co1.end(), cd.rig1_offsets.begin(), cd.rig1_offsets.end()); cr1.insert(cr1.end(), cd.rig1_rotations.begin(), cd.rig1_rotations.end());
    co2.insert(co2.end(), cd.rig2_offsets.begin(), cd.rig2_offsets.end()); cr2.insert(cr2.end(), cd.rig2_rotations.begin(), cd.rig2_rotations.end());
    pair_ptr[c + 1] = pair_ptr[c] + (int32_t)cd.pairings.size();
    for (const VerifyPairing& q : cd.pairings) {
      pairs.insert(pairs.end(), {q.kf1, q.kf2, q.cam1, q.cam2});
      if (q.kf1 >= 0 && q.kf1 < n_kf) bound += (size_t)(kf_ptr[q.kf1 + 1] - kf_ptr[q.kf1]);
    }
  }
  const int P = pair_ptr[C];
  if (seeds5.size() != (size_t)P || seeds.size() != (size_t)C)
    throw std::invalid_argument("covins_b200::VerifyNonCentralRelativePose: one seed per pairing and per candidate");
  std::vector<int32_t> nm(P), bs5(P), bc5(P), it5(P), us5(P), bs(C), bc(C), it(C), us(C), nv(C), corr(5 * bound);
  std::vector<double> bm5(12 * (size_t)P), bm(12 * (size_t)C), cov(36 * (size_t)C);
  const cvb_verify_candidates D{C, cp1.data(), co1.data(), cr1.data(), cp2.data(), co2.data(), cr2.data(), pair_ptr.data(), pairs.data()};
  const cvb_verify_params prm{params.img_match_thres, params.ratio_thres, params.threshold5, params.max_iterations5, params.threshold17,
                              params.max_iterations17, params.probability, params.n_cov_samples};
  cvb_verify_result R{nm.data(), bs5.data(), bm5.data(), bc5.data(), it5.data(), us5.data(), bs.data(), bm.data(), bc.data(), it.data(), us.data(),
                      cov.data(), nv.data(), corr.data(), (int32_t)bound, 0};
  call(D, prm, R);
  VerifyResult out;
  out.pairings.resize(P); out.candidates.resize(C);
  for (int q = 0; q < P; q++) {
    VerifyPairingResult& o = out.pairings[q];
    o.n_matches = nm[q]; o.best_sample = bs5[q]; o.n_inliers = bc5[q]; o.iterations = it5[q]; o.samples_used = us5[q];
    std::copy(bm5.begin() + 12 * (size_t)q, bm5.begin() + 12 * (size_t)(q + 1), o.model.begin());
  }
  for (int c = 0; c < C; c++) {
    VerifyCandidateResult& o = out.candidates[c];
    o.best_sample = bs[c]; o.n_inliers = bc[c]; o.iterations = it[c]; o.samples_used = us[c]; o.n_valid = nv[c];
    std::copy(bm.begin() + 12 * (size_t)c, bm.begin() + 12 * (size_t)(c + 1), o.model.begin());
    std::copy(cov.begin() + 36 * (size_t)c, cov.begin() + 36 * (size_t)(c + 1), o.cov.begin());
  }
  for (int j = 0; j < R.n_total; j++)
    out.correspondences.push_back({corr[5 * j], corr[5 * j + 1], corr[5 * j + 2], corr[5 * j + 3], corr[5 * j + 4]});
  return out;
}
}  // namespace detail

inline VerifyResult VerifyNonCentralRelativePose(Context& ctx, const std::vector<VerifyKeyframeView>& keyframes,
                                                 const std::vector<VerifyCandidate>& candidates, const VerifyParams& params,
                                                 const std::vector<uint64_t>& seeds5, const std::vector<uint64_t>& seeds) {
  std::vector<int32_t> kf_ptr;
  std::vector<uint8_t> desc;
  std::vector<double> bear, sig;
  detail::flatten_verify_keyframes<32>(keyframes, kf_ptr, desc, bear, sig);
  return detail::verify_noncentral(kf_ptr, candidates, params, seeds5, seeds,
                                   [&](const cvb_verify_candidates& D, const cvb_verify_params& prm, cvb_verify_result& R) {
                                     const cvb_verify_keyframes K{(int32_t)keyframes.size(), kf_ptr.data(), desc.data(), bear.data(), sig.data()};
                                     ctx.check(cvb_verify_noncentral_relative_pose_seeded_batch(ctx.get(), &K, &D, &prm, seeds5.data(), seeds.data(), &R),
                                               "cvb_verify_noncentral_relative_pose_seeded_batch");
                                   });
}

inline VerifyResult VerifyNonCentralRelativePose(Context& ctx, const std::vector<VerifyKeyframeViewSIFT>& keyframes,
                                                 const std::vector<VerifyCandidate>& candidates, const VerifyParams& params,
                                                 const std::vector<uint64_t>& seeds5, const std::vector<uint64_t>& seeds) {
  std::vector<int32_t> kf_ptr;
  std::vector<float> desc;
  std::vector<double> bear, sig;
  detail::flatten_verify_keyframes<128>(keyframes, kf_ptr, desc, bear, sig);
  return detail::verify_noncentral(kf_ptr, candidates, params, seeds5, seeds,
                                   [&](const cvb_verify_candidates& D, const cvb_verify_params& prm, cvb_verify_result& R) {
                                     const cvb_verify_keyframes_sift K{(int32_t)keyframes.size(), kf_ptr.data(), desc.data(), bear.data(), sig.data()};
                                     ctx.check(cvb_verify_noncentral_relative_pose_sift_seeded_batch(ctx.get(), &K, &D, &prm, seeds5.data(), seeds.data(),
                                                                                                     &R),
                                               "cvb_verify_noncentral_relative_pose_sift_seeded_batch");
                                   });
}

// The sampling-based 6x6 covariance of RelNonCentralPosSolver::computeNonCentralRelPose (RelNonCentralPosSolver.cpp:199,236,
// 276-279) for a batch of candidates in one call (cvb_noncentral_relative_pose_covariance_batch), in place of the loop of up to
// 300 host 17-point solves per candidate.  problems[i] are the candidate's correspondences and rigs, with samples = the
// covariance samples (17 local indices each, normally drawn from ransac_results[i].inliers); the reference model is
// ransac_results[i].model (all zeros when the RANSAC found none: the problem is skipped, n_valid = 0).  Per sample a 17-point
// re-solve and its deviation [2 vec(q); t_s - t_ref], q the quaternion of R_ref^T R_s; cov = the mean of delta delta^T over the
// valid samples (0 when none is).  cov (row-major, rotation then translation) is what LoopConstraint::cov_mat takes;
// PoseGraphOptimization whitens the loop edge with it and needs it positive definite.
struct RelativePoseCovariance {
  std::array<double, 36> cov{};
  int n_valid = 0;
};
inline std::vector<RelativePoseCovariance> NonCentralRelativePoseCovariance(Context& ctx, const std::vector<NonCentralRelativePoseRansacProblem>& problems,
                                                                            const std::vector<NonCentralRelativePoseRansacResult>& ransac_results) {
  const int n_prob = (int)problems.size();
  if (ransac_results.size() != problems.size())
    throw std::invalid_argument("covins_b200::NonCentralRelativePoseCovariance: one RANSAC result per problem");
  const detail::FlatRelProblems F = detail::flatten_rel_problems(problems, "NonCentralRelativePoseCovariance");
  const size_t m = n_prob > 0 ? n_prob : 1;
  std::vector<double> ref(12 * m), cov(36 * m);
  std::vector<int32_t> nv(m);
  for (int i = 0; i < n_prob; i++) std::copy(ransac_results[i].model.begin(), ransac_results[i].model.end(), ref.begin() + 12 * i);
  const cvb_rel_ransac_problems P = F.view();
  cvb_rel_cov_result R{cov.data(), nv.data(), nullptr, nullptr};
  ctx.check(cvb_noncentral_relative_pose_covariance_batch(ctx.get(), &P, ref.data(), &R), "cvb_noncentral_relative_pose_covariance_batch");
  std::vector<RelativePoseCovariance> out(n_prob);
  for (int i = 0; i < n_prob; i++) {
    std::copy(cov.begin() + 36 * i, cov.begin() + 36 * (i + 1), out[i].cov.begin());
    out[i].n_valid = nv[i];
  }
  return out;
}
// The same covariance with the samples drawn on the GPU (cvb_noncentral_relative_pose_covariance_seeded_batch): n_samples
// subsets of 17 (the reference's 300) of ransac_results[i].inliers per candidate, drawn from seeds[i] (the seed of the
// candidate's RANSAC may be reused: the two draw from separate streams); every problem's samples left empty.  A candidate with
// fewer than 17 inliers, or without a model, gets n_valid = 0.
inline std::vector<RelativePoseCovariance> NonCentralRelativePoseCovariance(Context& ctx, const std::vector<NonCentralRelativePoseRansacProblem>& problems,
                                                                            const std::vector<NonCentralRelativePoseRansacResult>& ransac_results,
                                                                            int n_samples, const std::vector<uint64_t>& seeds) {
  const int n_prob = (int)problems.size();
  if (ransac_results.size() != problems.size() || seeds.size() != problems.size())
    throw std::invalid_argument("covins_b200::NonCentralRelativePoseCovariance: one RANSAC result and one seed per problem");
  detail::require_no_samples(problems, "NonCentralRelativePoseCovariance");
  detail::FlatRelProblems F = detail::flatten_rel_problems(problems, "NonCentralRelativePoseCovariance");
  F.n_samples = n_samples;
  const size_t m = n_prob > 0 ? n_prob : 1;
  std::vector<double> ref(12 * m), cov(36 * m);
  std::vector<int32_t> nv(m);
  std::vector<uint8_t> mask;
  for (int i = 0; i < n_prob; i++) {
    if (ransac_results[i].inliers.size() != problems[i].sigma1.size())
      throw std::invalid_argument("covins_b200::NonCentralRelativePoseCovariance: one inlier flag per correspondence");
    std::copy(ransac_results[i].model.begin(), ransac_results[i].model.end(), ref.begin() + 12 * i);
    mask.insert(mask.end(), ransac_results[i].inliers.begin(), ransac_results[i].inliers.end());
  }
  if (mask.empty()) mask.push_back(0);
  const cvb_rel_ransac_problems P = F.view();
  cvb_rel_cov_result R{cov.data(), nv.data(), nullptr, nullptr};
  ctx.check(cvb_noncentral_relative_pose_covariance_seeded_batch(ctx.get(), &P, ref.data(), mask.data(), seeds.data(), &R, nullptr),
            "cvb_noncentral_relative_pose_covariance_seeded_batch");
  std::vector<RelativePoseCovariance> out(n_prob);
  for (int i = 0; i < n_prob; i++) {
    std::copy(cov.begin() + 36 * i, cov.begin() + 36 * (i + 1), out[i].cov.begin());
    out[i].n_valid = nv[i];
  }
  return out;
}

// The 5-point central relative-pose RANSAC of RelNonCentralPosSolver::computePose (RelNonCentralPosSolver.cpp:343-377) for a
// batch of pairings in one call (cvb_ransac_central_relative_pose_batch): 5-point hypothesis per sample, scoring and opengv's
// sequential model selection on the GPU.  Per problem: its correspondences (unit bearings, sigmas) and its samples (5 local
// indices each; every problem of a call has the same number of samples).  The six pairings of a place-recognition candidate
// are six problems of one call.  Result as RansacNonCentralRelativePose (model [R|t], X1 = R X2 + t, |t| = 1).
struct CentralRelativePoseRansacProblem {
  std::vector<double> bearings1, bearings2, sigma1, sigma2;   // 3n, 3n, n, n
  std::vector<int32_t> samples;                               // 5 * n_samples
};
inline std::vector<NonCentralRelativePoseRansacResult> RansacCentralRelativePose(Context& ctx, const std::vector<CentralRelativePoseRansacProblem>& problems,
                                                                                double threshold, int max_iterations, double probability = 0.99) {
  const int n_prob = (int)problems.size();
  const size_t n_samples = n_prob ? problems[0].samples.size() / 5 : 0;
  std::vector<int32_t> ptr(n_prob + 1, 0), samples;
  std::vector<double> f1, f2, s1, s2;
  for (int i = 0; i < n_prob; i++) {
    const CentralRelativePoseRansacProblem& p = problems[i];
    const size_t n = p.sigma1.size();
    if (p.samples.size() != 5 * n_samples || p.bearings1.size() != 3 * n || p.bearings2.size() != 3 * n || p.sigma2.size() != n)
      throw std::invalid_argument("covins_b200::RansacCentralRelativePose: inconsistent problem sizes");
    ptr[i + 1] = ptr[i] + (int32_t)n;
    f1.insert(f1.end(), p.bearings1.begin(), p.bearings1.end()); f2.insert(f2.end(), p.bearings2.begin(), p.bearings2.end());
    s1.insert(s1.end(), p.sigma1.begin(), p.sigma1.end()); s2.insert(s2.end(), p.sigma2.begin(), p.sigma2.end());
    samples.insert(samples.end(), p.samples.begin(), p.samples.end());
  }
  const cvb_central_rel_ransac_problems P{n_prob, ptr.data(), f1.data(), f2.data(), s1.data(), s2.data(), samples.data(), (int32_t)n_samples};
  return detail::ransac<NonCentralRelativePoseRansacResult>(ctx, cvb_ransac_central_relative_pose_batch, "cvb_ransac_central_relative_pose_batch", P,
                                                            ptr, threshold, max_iterations, probability);
}
// The same RANSAC with the samples drawn on the GPU (cvb_ransac_central_relative_pose_seeded_batch): one seed per problem,
// every problem's samples left empty (as RansacAbsolutePose's seeded form).
inline std::vector<NonCentralRelativePoseRansacResult> RansacCentralRelativePose(Context& ctx, const std::vector<CentralRelativePoseRansacProblem>& problems,
                                                                                const std::vector<uint64_t>& seeds, double threshold, int max_iterations,
                                                                                double probability = 0.99) {
  detail::require_no_samples(problems, "RansacCentralRelativePose");
  const int n_prob = (int)problems.size();
  std::vector<int32_t> ptr(n_prob + 1, 0);
  std::vector<double> f1, f2, s1, s2;
  for (int i = 0; i < n_prob; i++) {
    const CentralRelativePoseRansacProblem& p = problems[i];
    const size_t n = p.sigma1.size();
    if (p.bearings1.size() != 3 * n || p.bearings2.size() != 3 * n || p.sigma2.size() != n)
      throw std::invalid_argument("covins_b200::RansacCentralRelativePose: inconsistent problem sizes");
    ptr[i + 1] = ptr[i] + (int32_t)n;
    f1.insert(f1.end(), p.bearings1.begin(), p.bearings1.end()); f2.insert(f2.end(), p.bearings2.begin(), p.bearings2.end());
    s1.insert(s1.end(), p.sigma1.begin(), p.sigma1.end()); s2.insert(s2.end(), p.sigma2.begin(), p.sigma2.end());
  }
  const cvb_central_rel_ransac_problems P{n_prob, ptr.data(), f1.data(), f2.data(), s1.data(), s2.data(), nullptr, 0};
  return detail::ransac_seeded<NonCentralRelativePoseRansacResult>(ctx, cvb_ransac_central_relative_pose_seeded_batch,
                                                                   "cvb_ransac_central_relative_pose_seeded_batch", P, ptr, seeds, threshold, max_iterations,
                                                                   probability);
}

// Resident-map descriptor database (cvb_db_*): the ORB descriptors of the map's keyframes live in HBM; the candidate
// loop of PlaceRecognitionG::ComputeSE3 (placerec_gen_be.cpp:60-135) becomes one call per query keyframe.  The database
// index of a keyframe is its insertion order; keep it next to the keyframe (e.g. std::map<idpair, int>).
// A database constructed with the SiftDescriptors tag holds SIFT rows instead (feat.type SIFT, placerec_gen_be.cpp:86-87):
// AddKeyframe / MatchAll then take CV_32F rows x 128, matched with the exact L2 2-NN of MatchCandidatesSIFT.
// A database constructed over a ContextGroup spreads its keyframes over the group's GPUs (cvb_db_group_*): the same indices
// and the same MatchAll results, each request scanning every GPU's share of the map on that GPU.  Give it a group of its
// own (over the same devices if you like): its requests wait for any GlobalBundleAdjustment running on the same group.
struct SiftDescriptors {};
class DescriptorDatabase {
 public:
  explicit DescriptorDatabase(Context& ctx) : ctx_(&ctx) { ctx_->check(cvb_db_create(ctx_->get(), 32, &db_), "cvb_db_create"); }
  DescriptorDatabase(Context& ctx, SiftDescriptors) : ctx_(&ctx) { ctx_->check(cvb_db_create(ctx_->get(), 128, &db_), "cvb_db_create"); }
  explicit DescriptorDatabase(ContextGroup& group) : ctx_(&group.rank(0)) {
    ctx_->check(cvb_db_group_create(group.get(), 32, &gdb_), "cvb_db_group_create");
  }
  DescriptorDatabase(ContextGroup& group, SiftDescriptors) : ctx_(&group.rank(0)) {
    ctx_->check(cvb_db_group_create(group.get(), 128, &gdb_), "cvb_db_group_create");
  }
  ~DescriptorDatabase() {
    if (db_) cvb_db_destroy(ctx_->get(), db_);
    if (gdb_) cvb_db_group_destroy(gdb_);
  }
  DescriptorDatabase(const DescriptorDatabase&) = delete;
  DescriptorDatabase& operator=(const DescriptorDatabase&) = delete;
  // descriptors: kf->descriptors_add_ (CV_8U, continuous, rows x 32; keyframe_be.cpp:103,137) → returns the database index
  int AddKeyframe(const uint8_t* descriptors, int rows) {
    const int32_t r = rows;
    if (gdb_) ctx_->check(cvb_db_group_append(gdb_, descriptors, &r, 1), "cvb_db_group_append");
    else ctx_->check(cvb_db_append(ctx_->get(), db_, descriptors, &r, 1), "cvb_db_append");
    return n_kf_++;
  }
  // SIFT database: kf->descriptors_add_ as CV_32F, continuous, rows x 128, integer-valued in [0,255]
  int AddKeyframe(const float* descriptors, int rows) {
    const int32_t r = rows;
    if (gdb_) ctx_->check(cvb_db_group_append_sift(gdb_, descriptors, &r, 1), "cvb_db_group_append_sift");
    else ctx_->check(cvb_db_append_sift(ctx_->get(), db_, descriptors, &r, 1), "cvb_db_append_sift");
    return n_kf_++;
  }
  int size() const { return n_kf_; }
  // the keyframe leaves the map (culling, keyframe_be.cpp:413-440 / Map::EraseKeyframe): later indices drop by one
  void RemoveKeyframe(int db_index) {
    if (gdb_) ctx_->check(cvb_db_group_remove(gdb_, db_index), "cvb_db_group_remove");
    else ctx_->check(cvb_db_remove(ctx_->get(), db_, db_index), "cvb_db_remove");
    n_kf_--;
  }
  // a batch of keyframes leaves the map in one call (cvb_db_remove_batch / cvb_db_group_remove_batch), e.g. the keyframes
  // PruneRedundantKeyframes culled: db_indices as before the call, in any order; equal to RemoveKeyframe of each from the
  // highest to the lowest.  A survivor's index drops by the number of removed indices below it.
  void RemoveKeyframes(const std::vector<int>& db_indices) {
    const std::vector<int32_t> idx(db_indices.begin(), db_indices.end());
    const int n = (int)idx.size();
    if (gdb_) ctx_->check(cvb_db_group_remove_batch(gdb_, idx.data(), n), "cvb_db_group_remove_batch");
    else ctx_->check(cvb_db_remove_batch(ctx_->get(), db_, idx.data(), n), "cvb_db_remove_batch");
    n_kf_ -= n;
  }
  // two agents' maps are merged (MergeMaps): other's keyframes follow this database's, in other's order, copied in HBM
  // (cvb_db_merge / cvb_db_group_merge); other is left unchanged.  Both of one kind, on one Context or one ContextGroup.
  void Merge(const DescriptorDatabase& other) {
    if (gdb_) ctx_->check(other.gdb_ ? cvb_db_group_merge(gdb_, other.gdb_) : CVB_ERR_INVALID, "cvb_db_group_merge");
    else ctx_->check(other.db_ ? cvb_db_merge(ctx_->get(), db_, other.db_) : CVB_ERR_INVALID, "cvb_db_merge");
    n_kf_ += other.n_kf_;
  }
  // knnMatch(k=2) + distance/ratio filter of the query keyframe against EVERY keyframe of the database:
  // result[db index] == the reference's img_matches for that candidate (accepted queries ascending, :102-114)
  std::vector<Matches> MatchAll(const uint8_t* query, int n_query, const OptParams& P) {
    const float thr = P.img_match_thres, ratio = P.ratio_thres;
    return match_all(gdb_ ? "cvb_db_group_match_hamming" : "cvb_db_match_hamming", [&](auto... out) {
      return gdb_ ? cvb_db_group_match_hamming(gdb_, query, n_query, thr, ratio, out...)
                  : cvb_db_match_hamming(ctx_->get(), db_, query, n_query, thr, ratio, out...);
    });
  }
  // the same for a SIFT database: query = the query keyframe's CV_32F rows x 128
  std::vector<Matches> MatchAll(const float* query, int n_query, const OptParams& P) {
    const float thr = P.img_match_thres, ratio = P.ratio_thres;
    return match_all(gdb_ ? "cvb_db_group_match_l2" : "cvb_db_match_l2", [&](auto... out) {
      return gdb_ ? cvb_db_group_match_l2(gdb_, query, n_query, thr, ratio, out...)
                  : cvb_db_match_l2(ctx_->get(), db_, query, n_query, thr, ratio, out...);
    });
  }

 private:
  // fn(n_matches, m_kf, m_query, m_train, m_dist, cap, n_total): the request with the query bound
  template <class Fn>
  std::vector<Matches> match_all(const char* name, Fn fn) {
    std::vector<int32_t> nm(n_kf_ > 0 ? n_kf_ : 1);
    if (cap_ == 0) cap_ = 4096;
    for (;;) {
      m_kf_.resize(cap_); m_q_.resize(cap_); m_t_.resize(cap_); m_d_.resize(cap_);
      int32_t total = 0;
      ctx_->check(fn(nm.data(), m_kf_.data(), m_q_.data(), m_t_.data(), m_d_.data(), cap_, &total), name);
      if (total <= cap_) {
        std::vector<Matches> out(n_kf_);
        for (int i = 0; i < total; i++) out[m_kf_[i]].push_back(Match{(size_t)m_q_[i], (size_t)m_t_[i], m_d_[i]});
        return out;
      }
      cap_ = total + total / 4 + 16;
    }
  }

  Context* ctx_;                  // the single database's context, or the group's rank 0 (its messages)
  cvb_db* db_ = nullptr;
  cvb_db_group* gdb_ = nullptr;
  int n_kf_ = 0, cap_ = 0;
  std::vector<int32_t> m_kf_, m_q_, m_t_;
  std::vector<float> m_d_;
};

// Landmark::ComputeDescriptor (landmark_be.cpp:49-92) for a batch of landmarks: cand[l] = the descriptor rows
// (kf->descriptors_.row(feat_idx), 32 bytes each) of the landmark's valid observers in observation order.
// Returns per landmark the index of the chosen observer (-1: no observer, descriptor unchanged) and writes the chosen
// descriptor to out_desc[l] (32 bytes each; pass the current descriptors in, as the reference keeps them on early return).
inline std::vector<int> ComputeLandmarkDescriptors(Context& ctx, const std::vector<std::vector<const uint8_t*>>& cand,
                                                   uint8_t* out_desc) {
  const int n_lm = (int)cand.size();
  std::vector<int32_t> ptr(n_lm + 1, 0);
  for (int l = 0; l < n_lm; l++) ptr[l + 1] = ptr[l] + (int32_t)cand[l].size();
  std::vector<uint8_t> rows((size_t)ptr[n_lm] * 32 + 32);
  for (int l = 0; l < n_lm; l++)
    for (size_t j = 0; j < cand[l].size(); j++) std::copy(cand[l][j], cand[l][j] + 32, rows.begin() + ((size_t)ptr[l] + j) * 32);
  std::vector<int32_t> best(n_lm > 0 ? n_lm : 1);
  ctx.check(cvb_landmark_descriptor_batch(ctx.get(), rows.data(), ptr.data(), n_lm, best.data(), out_desc), "cvb_landmark_descriptor_batch");
  return std::vector<int>(best.begin(), best.begin() + n_lm);
}

// ---------------------------------------------------------------------------------------------------------------
// The merge constructor Map(map_target, map_tofuse, T_wtarget_wtofuse) (map_be.cpp:334-381), reached from
// MapManager::PerformMerge (map_be.cpp:192-244): the fused map's valid keyframes (T_ws, velocity) and valid landmarks
// (position) moved into the target's world frame by one cvb_map_rigid_transform call (the rule and its assumptions are in
// include/covins_b200.h), written back keyframes first (SetPoseTws, SetStateVelocity), then landmarks (SetWorldPos), as the
// constructor's loop does.  Then the union, on map_target, which becomes the merged map: every keyframe, landmark and loop
// constraint of map_tofuse through map_target->AddKeyframe / AddLandmark / AddLoopConstraint (ids are kept: two agents'
// ids do not collide).  With both databases given, db_tofuse's keyframes join db_target in HBM (their database indices
// shift by db_target's size before the call; db_tofuse is left unchanged).  Last, the merged map's covisibility graph.
// map_target's own keyframes and landmarks are not touched before the union.
// ---------------------------------------------------------------------------------------------------------------
template <class MapPtr, class Transform4>
void MergeMaps(Context& ctx, MapPtr map_target, MapPtr map_tofuse, const Transform4& T_wtarget_wtofuse, DescriptorDatabase* db_target = nullptr,
               DescriptorDatabase* db_tofuse = nullptr) {
  using KeyframePtr = typename std::decay<decltype(map_tofuse->GetKeyframesVec()[0])>::type;
  using KF = typename KeyframePtr::element_type;
  const auto keyframes = map_tofuse->GetKeyframesVec();
  const auto landmarks = map_tofuse->GetLandmarksVec();
  using LandmarkPtr = typename std::decay<decltype(landmarks[0])>::type;
  std::map<const KF*, int> kf_index;
  std::vector<KeyframePtr> kfs;
  detail::canonical_keyframes(keyframes, kf_index, kfs);
  std::vector<LandmarkPtr> lms;
  for (auto& lm : landmarks)
    if (!lm->IsInvalid()) lms.push_back(lm);
  const int K = (int)kfs.size(), L = (int)lms.size();
  double T[16];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) T[4 * r + c] = T_wtarget_wtofuse(r, c);
  std::vector<double> ws(16 * (size_t)K + 1), vel(3 * (size_t)K + 1), pos(3 * (size_t)L + 1);
  for (int k = 0; k < K; k++) {
    const auto Tws = kfs[k]->GetPoseTws();
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) ws[16 * (size_t)k + 4 * r + c] = Tws(r, c);
    const auto v = kfs[k]->GetStateVelocity();
    for (int i = 0; i < 3; i++) vel[3 * (size_t)k + i] = v[i];
  }
  for (int l = 0; l < L; l++) {
    const auto p = lms[l]->GetWorldPos();
    for (int i = 0; i < 3; i++) pos[3 * (size_t)l + i] = p[i];
  }
  ctx.check(cvb_map_rigid_transform(ctx.get(), T, K, ws.data(), vel.data(), L, pos.data(), nullptr, nullptr), "cvb_map_rigid_transform");
  for (int k = 0; k < K; k++) {
    auto Tws = kfs[k]->GetPoseTws();
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) Tws(r, c) = ws[16 * (size_t)k + 4 * r + c];
    kfs[k]->SetPoseTws(Tws);
    kfs[k]->SetStateVelocity({vel[3 * (size_t)k], vel[3 * (size_t)k + 1], vel[3 * (size_t)k + 2]});
  }
  for (int l = 0; l < L; l++) lms[l]->SetWorldPos({pos[3 * (size_t)l], pos[3 * (size_t)l + 1], pos[3 * (size_t)l + 2]});
  for (auto& kf : keyframes) map_target->AddKeyframe(kf);
  for (auto& lm : landmarks) map_target->AddLandmark(lm);
  for (const auto& lc : map_tofuse->GetLoopConstraints()) map_target->AddLoopConstraint(lc);
  if (db_target && db_tofuse) db_target->Merge(*db_tofuse);
  UpdateCovisibilityConnections(ctx, map_target);
}

}  // namespace covins_b200
