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
  // raw IMU samples of the KF's preintegration (robopt PreintegrationBase::getReadingsByIndex / getTimeDiffByIndex,
  // keyframe_base.cpp:145-173) and its first reading + noise (keyframe_be.cpp:187-203)
  static size_t imu_count(const KF& kf) { return kf.ImuDt().size(); }
  static void imu_samples(const KF& kf, std::vector<double>& dt, std::vector<double>& acc, std::vector<double>& gyr,
                          double acc0[3], double gyr0[3], double noise[5]) {
    kf.GetImu(dt, acc, gyr, acc0, gyr0, noise);
  }
};

namespace detail {

// rotation matrix (via operator()(r,c) of a 4x4 transform) → quaternion (x,y,z,w), the convention of
// Eigen::Quaterniond(R) used at keyframe_base.cpp:490-499 (w >= 0 branch of Eigen's algorithm)
template <class T4>
inline void transform_to_pose7(const T4& T, double* out) {
  const double m00 = T(0, 0), m11 = T(1, 1), m22 = T(2, 2);
  double q[4];  // x y z w
  const double tr = m00 + m11 + m22;
  if (tr > 0) {
    double t = std::sqrt(tr + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (T(2, 1) - T(1, 2)) * t;
    q[1] = (T(0, 2) - T(2, 0)) * t;
    q[2] = (T(1, 0) - T(0, 1)) * t;
  } else {
    int i = 0;
    if (m11 > m00) i = 1;
    if (m22 > T(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double t = std::sqrt(T(i, i) - T(j, j) - T(k, k) + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (T(k, j) - T(j, k)) * t;
    q[j] = (T(j, i) + T(i, j)) * t;
    q[k] = (T(k, i) + T(i, k)) * t;
  }
  out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3];
  out[4] = T(0, 3); out[5] = T(1, 3); out[6] = T(2, 3);
}

// Utils::Ceres2Transform (covins_comm/src/covins_base/utils_base.cpp:28-43): normalised quaternion → 4x4
template <class T4>
inline T4 pose7_to_transform(const double* p) {
  double x = p[0], y = p[1], z = p[2], w = p[3];
  const double n = 1.0 / std::sqrt(x * x + y * y + z * z + w * w);
  x *= n; y *= n; z *= n; w *= n;
  T4 T = T4::Identity();
  T(0, 0) = 1 - 2 * (y * y + z * z); T(0, 1) = 2 * (x * y - z * w); T(0, 2) = 2 * (x * z + y * w);
  T(1, 0) = 2 * (x * y + z * w); T(1, 1) = 1 - 2 * (x * x + z * z); T(1, 2) = 2 * (y * z - x * w);
  T(2, 0) = 2 * (x * z - y * w); T(2, 1) = 2 * (y * z + x * w); T(2, 2) = 1 - 2 * (x * x + y * y);
  T(0, 3) = p[4]; T(1, 3) = p[5]; T(2, 3) = p[6];
  return T;
}

template <class T4>
inline T4 rel_transform(const T4& Ta, const T4& Tb) {  // Ta^-1 * Tb for rigid transforms
  T4 R = T4::Identity();
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      double s = 0;
      for (int m = 0; m < 3; m++) s += Ta(m, r) * Tb(m, c);
      R(r, c) = s;
    }
  for (int r = 0; r < 3; r++) {
    double s = 0;
    for (int m = 0; m < 3; m++) s += Ta(m, r) * (Tb(m, 3) - Ta(m, 3));
    R(r, 3) = s;
  }
  return R;
}

// lower Cholesky of a symmetric 6x6, transposed: LLT(cov^-1).matrixL().transpose() (optimization_be.cpp:922-923)
inline bool sqrt_info_from_cov(const double* cov /*36 row-major*/, double* out /*36*/) {
  // invert via Cholesky of cov, then Cholesky of the inverse
  double L[36] = {0}, X[36] = {0}, P[36];
  for (int c = 0; c < 6; c++)
    for (int r = c; r < 6; r++) {
      double s = cov[6 * r + c];
      for (int m = 0; m < c; m++) s -= L[6 * r + m] * L[6 * c + m];
      if (r == c) {
        if (!(s > 0)) return false;
        L[6 * c + c] = std::sqrt(s);
      } else {
        L[6 * r + c] = s / L[6 * c + c];
      }
    }
  for (int c = 0; c < 6; c++)
    for (int r = c; r < 6; r++) {
      double s = (r == c) ? 1.0 : 0.0;
      for (int m = c; m < r; m++) s -= L[6 * r + m] * X[6 * m + c];
      X[6 * r + c] = s / L[6 * r + r];
    }
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) {
      double s = 0;
      for (int m = std::max(r, c); m < 6; m++) s += X[6 * m + r] * X[6 * m + c];
      P[6 * r + c] = s;
    }
  double M[36] = {0};
  for (int c = 0; c < 6; c++)
    for (int r = c; r < 6; r++) {
      double s = P[6 * r + c];
      for (int m = 0; m < c; m++) s -= M[6 * r + m] * M[6 * c + m];
      if (r == c) {
        if (!(s > 0)) return false;
        M[6 * c + c] = std::sqrt(s);
      } else {
        M[6 * r + c] = s / M[6 * c + c];
      }
    }
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) out[6 * r + c] = M[6 * c + r];
  return true;
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

// ---------------------------------------------------------------------------------------------------------------
// Optimization::GlobalBundleAdjustment — same signature meaning as optimization_be.hpp:38-40.
// ---------------------------------------------------------------------------------------------------------------
template <class MapPtr>
void GlobalBundleAdjustment(Context& ctx, MapPtr map, int interations_limit, double /*time_limit*/, bool visual_only = false,
                            bool outlier_removal = true, bool /*estimate_bias*/ = false, const OptParams& P = OptParams()) {
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
  for (auto& kf : keyframes) {
    if (kf->IsInvalid()) continue;
    kf_index[kf.get()] = (int)kfs.size();
    kfs.push_back(kf);
  }
  const int K = (int)kfs.size();
  F.pose.resize(7 * (size_t)K); F.sb.resize(9 * (size_t)K); F.extr.resize(7 * (size_t)K); F.intr.resize(4 * (size_t)K);
  F.dist.resize(4 * (size_t)K); F.pose_const.assign(K, 0); F.cam_of_kf.resize(K);
  F.imu_ptr.push_back(0);
  for (int k = 0; k < K; k++) {
    auto& kf = kfs[k];
    // UpdateCeresFromState (keyframe_base.cpp:486-521) restated on the flat arrays
    kf->UpdateCeresFromState(&F.pose[7 * (size_t)k], &F.sb[9 * (size_t)k], &F.extr[7 * (size_t)k]);
    F.cam_of_kf[k] = k;
    if (kf->id_.first == 0 && kf->id_.second == map->id_map_) F.pose_const[k] = 1;                 // :88-89, 329-331
    if (kf->is_loaded_ && P.gba_fix_poses_loaded_maps) F.pose_const[k] = 1;                        // :338-341
    if (!Adapter<KF>::camera(*kf, &F.intr[4 * (size_t)k], &F.dist[4 * (size_t)k])) {
      std::printf("FATAL: Unknown projection type.\n");                                            // :112-114
      std::exit(-1);
    }
    {
      int cm = 0, dm = 0; double xi = 0.0;
      Adapter<KF>::camera_model(*kf, &cm, &dm, &xi);                                               // :186-231
      F.cam_model.resize(F.pose_const.size(), 0); F.dist_model.resize(F.pose_const.size(), 0); F.cam_xi.resize(F.pose_const.size(), 0.0);
      F.cam_model[k] = cm; F.dist_model[k] = dm; F.cam_xi[k] = xi;
    }
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
  // landmarks + observations (canonical: observations sorted by keyframe index; the reference iterates a
  // pointer-ordered std::map, typedefs_base.hpp:187)
  struct ObsRef { KeyframePtr kf; int lm; int feat; };
  std::vector<ObsRef> obs_ref;
  using LandmarkPtr = typename std::decay<decltype(landmarks[0])>::type;
  std::vector<LandmarkPtr> lms;
  F.lm_obs_ptr.push_back(0);
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
    const auto pos = lm->GetWorldPos();
    F.lm.push_back(pos[0]); F.lm.push_back(pos[1]); F.lm.push_back(pos[2]);
    for (auto& o : ob) {
      auto& kfx = kfs[o.first];
      const auto& kp = kfx->keypoints_distorted_[o.second];
      F.obs_kf.push_back(o.first);
      F.obs_uv.push_back((float)kp[0]); F.obs_uv.push_back((float)kp[1]);
      F.obs_sigma.push_back((kfx->keypoints_aors_[o.second][1] + 1) * 2.0);                         // :183-184, 477-478
      obs_ref.push_back({kfx, (int)lms.size(), o.second});
    }
    F.lm_obs_ptr.push_back((int32_t)F.obs_kf.size());
    lms.push_back(lm);
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
  ctx.check(cvb_gba(ctx.get(), &prob, &g, &res, removed.data()), "cvb_gba");

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

// ---------------------------------------------------------------------------------------------------------------
// Optimization::PoseGraphOptimization — optimization_be.hpp:46-47.  PoseMap = std::map<idpair, Transform>.
// ---------------------------------------------------------------------------------------------------------------
template <class MapPtr, class PoseMap>
void PoseGraphOptimization(Context& ctx, MapPtr map, PoseMap corrected_poses, const OptParams& P = OptParams()) {
  using KeyframePtr = typename std::decay<decltype(map->GetKeyframesVec()[0])>::type;
  using KF = typename KeyframePtr::element_type;
  using Transform = typename std::decay<decltype(map->GetKeyframesVec()[0]->GetPoseTws())>::type;
  auto keyframes = map->GetKeyframesVec();
  auto landmarks = map->GetLandmarksVec();
  detail::Flat F;
  std::map<const KF*, int> kf_index;
  std::vector<KeyframePtr> kfs;
  for (auto& kf : keyframes) {
    if (kf->IsInvalid()) continue;
    kf_index[kf.get()] = (int)kfs.size();
    kfs.push_back(kf);
  }
  const int K = (int)kfs.size();
  F.pose.resize(7 * (size_t)K); F.sb.assign(9 * (size_t)K, 0.0); F.extr.resize(7 * (size_t)K);
  F.intr.assign(4 * (size_t)K, 1.0); F.dist.assign(4 * (size_t)K, 0.0); F.pose_const.assign(K, 0); F.cam_of_kf.resize(K);
  F.lm_obs_ptr.push_back(0); F.imu_ptr.push_back(0);
  for (int k = 0; k < K; k++) {
    auto& kf = kfs[k];
    double tmp_pose[7];
    kf->UpdateCeresFromState(tmp_pose, &F.sb[9 * (size_t)k], &F.extr[7 * (size_t)k]);
    auto mit = corrected_poses.find(kf->id_);                                                        // :854-868
    const Transform T_ws_init = (mit != corrected_poses.end()) ? mit->second : kf->GetPoseTws();
    detail::transform_to_pose7(T_ws_init, &F.pose[7 * (size_t)k]);
    F.cam_of_kf[k] = k;
    if (kf->id_.first == 0 && kf->id_.second == map->id_map_) F.pose_const[k] = 1;                  // :870-871
    if (kf->is_gba_optimized_ && P.pgo_fix_kfs_after_gba) F.pose_const[k] = 1;                      // :875-877
    else if (kf->is_loaded_ && P.pgo_fix_poses_loaded_maps) F.pose_const[k] = 1;                    // :878-881
  }
  double S1[36] = {0}, S23[36] = {0}, S45[36] = {0};
  for (int d = 0; d < 6; d++) {
    S1[7 * d] = (d < 3 ? P.wt_kf_r : P.wt_kf_t) * P.wt_kf_n1;                                        // :896-898
    S23[7 * d] = S1[7 * d] / P.wt_kf_n23;
    S45[7 * d] = S1[7 * d] / P.wt_kf_n45;
  }
  auto push_edge = [&](int i, int j, const Transform& T12, const double* S, bool robust) {
    double p7[7];
    detail::transform_to_pose7(T12, p7);
    F.edge_i.push_back(i); F.edge_j.push_back(j);
    F.edge_q.insert(F.edge_q.end(), p7, p7 + 4);
    F.edge_t.insert(F.edge_t.end(), p7 + 4, p7 + 7);
    F.edge_S.insert(F.edge_S.end(), S, S + 36);
    F.edge_robust.push_back(robust ? 1 : 0);
  };
  for (const auto& lc : map->GetLoopConstraints()) {                                                 // :910-943
    double Sl[36];
    if (P.placerec_type_covins) {
      std::copy(S1, S1 + 36, Sl);
    } else {
      double cov[36];
      for (int r = 0; r < 6; r++)
        for (int c = 0; c < 6; c++) cov[6 * r + c] = lc.cov_mat(r, c);
      if (!detail::sqrt_info_from_cov(cov, Sl)) {
        std::printf("FATAL: loop covariance is not positive definite\n");
        std::exit(-1);
      }
    }
    push_edge(kf_index.at(lc.kf1.get()), kf_index.at(lc.kf2.get()), lc.T_s1_s2, Sl, P.use_robust_loss);
  }
  std::set<std::pair<const KF*, const KF*>> inserted_edges;                                          // :907
  for (int k = 0; k < K; k++) {                                                                      // successor edges :947-972
    auto& kf = kfs[k];
    auto succ = kf->GetSuccessor();
    if (!succ) continue;
    auto key = std::make_pair((const KF*)kf.get(), (const KF*)succ.get());
    if (inserted_edges.count(key)) {
      std::printf("WARN: KF edge already added\n");
      continue;
    }
    inserted_edges.insert(key);
    push_edge(k, kf_index.at(succ.get()), detail::rel_transform(kf->GetPoseTws_vio(), succ->GetPoseTws_vio()), S1, false);
  }
  if (P.use_nbr_kfs) {                                                                               // :976-1021
    for (int k = 0; k < K; k++) {
      auto& kf = kfs[k];
      std::vector<KeyframePtr> connections;
      KeyframePtr temp_kf = kf;
      for (int j = 1; j < 6; ++j)
        if (int(kf->id_.first) - j > 0) {
          temp_kf = temp_kf->GetPredecessor();
          connections.push_back(temp_kf);
        }
      size_t n = 0;
      for (auto& kfc : connections) {
        n++;
        const double* S = (n <= 1) ? S1 : (n <= 3 ? S23 : S45);
        auto key = std::make_pair((const KF*)kf.get(), (const KF*)kfc.get());
        if (inserted_edges.count(key)) continue;
        inserted_edges.insert(key);
        push_edge(k, kf_index.at(kfc.get()), detail::rel_transform(kf->GetPoseTws_vio(), kfc->GetPoseTws_vio()), S, false);
      }
    }
  }
  const cvb_ba_problem prob = F.view();
  cvb_ba_options o{};
  o.max_iterations = P.pgo_iteration_limit;
  o.visual_only = 1;
  o.cauchy_reproj = 0.0;
  o.cauchy_edge = P.robust_loss_th;
  o.world = 1;
  std::vector<double> o_pose(7 * (size_t)K);
  cvb_ba_result res{};
  res.pose = o_pose.data();
  ctx.check(cvb_ba_solve(ctx.get(), &prob, &o, &res), "cvb_ba_solve(PGO)");

  // Recover the optimized data (:1033-1051)
  std::map<typename std::decay<decltype(kfs[0]->id_)>::type, Transform> non_corrected_poses;
  for (int k = 0; k < K; k++) {
    auto& kf = kfs[k];
    const Transform T_ws_uncorrected = kf->GetPoseTws();
    non_corrected_poses[kf->id_] = T_ws_uncorrected;
    const Transform T_ws_corrected = detail::pose7_to_transform<Transform>(&o_pose[7 * (size_t)k]);
    const auto vel = kf->GetStateVelocity();
    kf->SetPoseTws(T_ws_corrected);
    double v[3];   // R_corr * R_uncorr^T * v  (:1046-1047)
    for (int r = 0; r < 3; r++) {
      double s = 0;
      for (int c = 0; c < 3; c++) {
        double m = 0;
        for (int x = 0; x < 3; x++) m += T_ws_corrected(r, x) * T_ws_uncorrected(c, x);
        s += m * vel[c];
      }
      v[r] = s;
    }
    kf->SetStateVelocity({v[0], v[1], v[2]});
    kf->SetPoseOptimized();
  }
  // Landmarks re-anchored through their reference keyframe (:1054-1083)
  for (auto& lm : landmarks) {
    if (lm->IsInvalid()) continue;
    auto kf_ref = lm->GetReferenceKeyframe();
    if (!kf_ref) {
      if (!lm->GetObservations().empty()) map->EraseLandmark(lm);
      continue;
    }
    auto mit = non_corrected_poses.find(kf_ref->id_);
    if (mit == non_corrected_poses.end()) {
      map->EraseLandmark(lm);
      continue;
    }
    const Transform& Tu = mit->second;
    const auto pw = lm->GetWorldPos();
    double ps[3], pc[3];
    for (int r = 0; r < 3; r++) {
      double s = 0;
      for (int c = 0; c < 3; c++) s += Tu(c, r) * (pw[c] - Tu(c, 3));
      ps[r] = s;
    }
    const Transform Tc = kf_ref->GetPoseTws();
    for (int r = 0; r < 3; r++) pc[r] = Tc(r, 0) * ps[0] + Tc(r, 1) * ps[1] + Tc(r, 2) * ps[2] + Tc(r, 3);
    lm->SetWorldPos({pc[0], pc[1], pc[2]});
    lm->SetOptimized();
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
  auto flatten = [](const KFPtr& kf, KfViewStorage& S) {
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
  };
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
inline std::vector<AbsolutePoseRansacResult> RansacAbsolutePose(Context& ctx, const std::vector<AbsolutePoseRansacProblem>& problems, double threshold,
                                                                 int max_iterations, double probability = 0.99) {
  const int n_prob = (int)problems.size();
  const size_t n_samples = n_prob ? problems[0].samples.size() / 4 : 0;
  std::vector<int32_t> ptr(n_prob + 1, 0), samples;
  std::vector<double> pts, f, sigma, cam_off, cam_rot;
  for (int i = 0; i < n_prob; i++) {
    const AbsolutePoseRansacProblem& p = problems[i];
    if (p.samples.size() != 4 * n_samples || p.points.size() != 3 * p.sigma_angles.size() || p.bearings.size() != 3 * p.sigma_angles.size())
      throw std::invalid_argument("covins_b200::RansacAbsolutePose: inconsistent problem sizes");
    ptr[i + 1] = ptr[i] + (int32_t)p.sigma_angles.size();
    pts.insert(pts.end(), p.points.begin(), p.points.end());
    f.insert(f.end(), p.bearings.begin(), p.bearings.end());
    sigma.insert(sigma.end(), p.sigma_angles.begin(), p.sigma_angles.end());
    cam_off.insert(cam_off.end(), p.cam_offset, p.cam_offset + 3);
    cam_rot.insert(cam_rot.end(), p.cam_rotation, p.cam_rotation + 9);
    samples.insert(samples.end(), p.samples.begin(), p.samples.end());
  }
  const size_t m = n_prob > 0 ? n_prob : 1;
  std::vector<int32_t> best(m), cnt(m), iters(m), used(m);
  std::vector<double> models(12 * m);
  std::vector<uint8_t> mask(ptr[n_prob] > 0 ? ptr[n_prob] : 1);
  cvb_abs_ransac_problems P{n_prob, ptr.data(), pts.data(), f.data(), sigma.data(), cam_off.data(), cam_rot.data(), samples.data(), (int32_t)n_samples};
  cvb_abs_ransac_result R{best.data(), models.data(), cnt.data(), iters.data(), used.data(), mask.data(), nullptr, nullptr, nullptr};
  ctx.check(cvb_ransac_absolute_pose_batch(ctx.get(), &P, threshold, max_iterations, probability, &R), "cvb_ransac_absolute_pose_batch");
  std::vector<AbsolutePoseRansacResult> out(n_prob);
  for (int i = 0; i < n_prob; i++) {
    out[i].best_sample = best[i]; out[i].n_inliers = cnt[i]; out[i].iterations = iters[i]; out[i].samples_used = used[i];
    std::copy(models.begin() + 12 * i, models.begin() + 12 * (i + 1), out[i].model.begin());
    out[i].inliers.assign(mask.begin() + ptr[i], mask.begin() + ptr[i + 1]);
  }
  return out;
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
inline std::vector<NonCentralRelativePoseRansacResult> RansacNonCentralRelativePose(Context& ctx,
                                                                                   const std::vector<NonCentralRelativePoseRansacProblem>& problems,
                                                                                   double threshold, int max_iterations, double probability = 0.99) {
  const int n_prob = (int)problems.size();
  const size_t n_samples = n_prob ? problems[0].samples.size() / 17 : 0;
  std::vector<int32_t> ptr(n_prob + 1, 0), cp1(n_prob + 1, 0), cp2(n_prob + 1, 0), cam1, cam2, samples;
  std::vector<double> f1, f2, s1, s2, co1, cr1, co2, cr2;
  for (int i = 0; i < n_prob; i++) {
    const NonCentralRelativePoseRansacProblem& p = problems[i];
    const size_t n = p.sigma1.size();
    if (p.samples.size() != 17 * n_samples || p.bearings1.size() != 3 * n || p.bearings2.size() != 3 * n || p.sigma2.size() != n ||
        p.cam1.size() != n || p.cam2.size() != n || p.rig1_rotations.size() != 3 * p.rig1_offsets.size() ||
        p.rig2_rotations.size() != 3 * p.rig2_offsets.size() || p.rig1_offsets.size() % 3 || p.rig2_offsets.size() % 3)
      throw std::invalid_argument("covins_b200::RansacNonCentralRelativePose: inconsistent problem sizes");
    ptr[i + 1] = ptr[i] + (int32_t)n;
    cp1[i + 1] = cp1[i] + (int32_t)(p.rig1_offsets.size() / 3);
    cp2[i + 1] = cp2[i] + (int32_t)(p.rig2_offsets.size() / 3);
    f1.insert(f1.end(), p.bearings1.begin(), p.bearings1.end()); f2.insert(f2.end(), p.bearings2.begin(), p.bearings2.end());
    s1.insert(s1.end(), p.sigma1.begin(), p.sigma1.end()); s2.insert(s2.end(), p.sigma2.begin(), p.sigma2.end());
    cam1.insert(cam1.end(), p.cam1.begin(), p.cam1.end()); cam2.insert(cam2.end(), p.cam2.begin(), p.cam2.end());
    co1.insert(co1.end(), p.rig1_offsets.begin(), p.rig1_offsets.end()); cr1.insert(cr1.end(), p.rig1_rotations.begin(), p.rig1_rotations.end());
    co2.insert(co2.end(), p.rig2_offsets.begin(), p.rig2_offsets.end()); cr2.insert(cr2.end(), p.rig2_rotations.begin(), p.rig2_rotations.end());
    samples.insert(samples.end(), p.samples.begin(), p.samples.end());
  }
  const size_t m = n_prob > 0 ? n_prob : 1;
  std::vector<int32_t> best(m), cnt(m), iters(m), used(m);
  std::vector<double> models(12 * m);
  std::vector<uint8_t> mask(ptr[n_prob] > 0 ? ptr[n_prob] : 1);
  cvb_rel_ransac_problems P{n_prob,     ptr.data(), f1.data(), f2.data(), s1.data(),  s2.data(),  cam1.data(),    cam2.data(),
                            cp1.data(), co1.data(), cr1.data(), cp2.data(), co2.data(), cr2.data(), samples.data(), (int32_t)n_samples};
  cvb_rel_ransac_result R{best.data(), models.data(), cnt.data(), iters.data(), used.data(), mask.data(), nullptr, nullptr, nullptr};
  ctx.check(cvb_ransac_noncentral_relative_pose_batch(ctx.get(), &P, threshold, max_iterations, probability, &R),
            "cvb_ransac_noncentral_relative_pose_batch");
  std::vector<NonCentralRelativePoseRansacResult> out(n_prob);
  for (int i = 0; i < n_prob; i++) {
    out[i].best_sample = best[i]; out[i].n_inliers = cnt[i]; out[i].iterations = iters[i]; out[i].samples_used = used[i];
    std::copy(models.begin() + 12 * i, models.begin() + 12 * (i + 1), out[i].model.begin());
    out[i].inliers.assign(mask.begin() + ptr[i], mask.begin() + ptr[i + 1]);
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
  const size_t m = n_prob > 0 ? n_prob : 1;
  std::vector<int32_t> best(m), cnt(m), iters(m), used(m);
  std::vector<double> models(12 * m);
  std::vector<uint8_t> mask(ptr[n_prob] > 0 ? ptr[n_prob] : 1);
  cvb_central_rel_ransac_problems P{n_prob, ptr.data(), f1.data(), f2.data(), s1.data(), s2.data(), samples.data(), (int32_t)n_samples};
  cvb_rel_ransac_result R{best.data(), models.data(), cnt.data(), iters.data(), used.data(), mask.data(), nullptr, nullptr, nullptr};
  ctx.check(cvb_ransac_central_relative_pose_batch(ctx.get(), &P, threshold, max_iterations, probability, &R), "cvb_ransac_central_relative_pose_batch");
  std::vector<NonCentralRelativePoseRansacResult> out(n_prob);
  for (int i = 0; i < n_prob; i++) {
    out[i].best_sample = best[i]; out[i].n_inliers = cnt[i]; out[i].iterations = iters[i]; out[i].samples_used = used[i];
    std::copy(models.begin() + 12 * i, models.begin() + 12 * (i + 1), out[i].model.begin());
    out[i].inliers.assign(mask.begin() + ptr[i], mask.begin() + ptr[i + 1]);
  }
  return out;
}

// Resident-map descriptor database (cvb_db_*): the ORB descriptors of the map's keyframes live in HBM; the candidate
// loop of PlaceRecognitionG::ComputeSE3 (placerec_gen_be.cpp:60-135) becomes one call per query keyframe.  The database
// index of a keyframe is its insertion order; keep it next to the keyframe (e.g. std::map<idpair, int>).
class DescriptorDatabase {
 public:
  explicit DescriptorDatabase(Context& ctx) : ctx_(ctx) { ctx_.check(cvb_db_create(ctx_.get(), 32, &db_), "cvb_db_create"); }
  ~DescriptorDatabase() { if (db_) cvb_db_destroy(ctx_.get(), db_); }
  DescriptorDatabase(const DescriptorDatabase&) = delete;
  DescriptorDatabase& operator=(const DescriptorDatabase&) = delete;
  // descriptors: kf->descriptors_add_ (CV_8U, continuous, rows x 32; keyframe_be.cpp:103,137) → returns the database index
  int AddKeyframe(const uint8_t* descriptors, int rows) {
    const int32_t r = rows;
    ctx_.check(cvb_db_append(ctx_.get(), db_, descriptors, &r, 1), "cvb_db_append");
    return n_kf_++;
  }
  int size() const { return n_kf_; }
  // the keyframe leaves the map (culling, keyframe_be.cpp:413-440 / Map::EraseKeyframe): later indices drop by one
  void RemoveKeyframe(int db_index) {
    ctx_.check(cvb_db_remove(ctx_.get(), db_, db_index), "cvb_db_remove");
    n_kf_--;
  }
  // knnMatch(k=2) + distance/ratio filter of the query keyframe against EVERY keyframe of the database:
  // result[db index] == the reference's img_matches for that candidate (accepted queries ascending, :102-114)
  std::vector<Matches> MatchAll(const uint8_t* query, int n_query, const OptParams& P) {
    std::vector<int32_t> nm(n_kf_ > 0 ? n_kf_ : 1);
    if (cap_ == 0) cap_ = 4096;
    for (;;) {
      m_kf_.resize(cap_); m_q_.resize(cap_); m_t_.resize(cap_); m_d_.resize(cap_);
      int32_t total = 0;
      ctx_.check(cvb_db_match_hamming(ctx_.get(), db_, query, n_query, P.img_match_thres, P.ratio_thres, nm.data(), m_kf_.data(),
                                      m_q_.data(), m_t_.data(), m_d_.data(), cap_, &total),
                 "cvb_db_match_hamming");
      if (total <= cap_) {
        std::vector<Matches> out(n_kf_);
        for (int i = 0; i < total; i++) out[m_kf_[i]].push_back(Match{(size_t)m_q_[i], (size_t)m_t_[i], m_d_[i]});
        return out;
      }
      cap_ = total + total / 4 + 16;
    }
  }

 private:
  Context& ctx_;
  cvb_db* db_ = nullptr;
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

}  // namespace covins_b200
