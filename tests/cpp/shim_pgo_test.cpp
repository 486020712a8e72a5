// covins_b200::PoseGraphOptimization (one cvb_pgo call) against the composition it replaced, on two identical mock maps
// built from a flat problem dumped by tests/test_pose_graph.py.  Every container write is compared bit for bit: keyframe
// poses, velocities and SetPoseOptimized counts, landmark positions, SetOptimized counts and erasures.
//   shim_pgo_test <dir>   exit 0: identical, 1: a difference (printed), 2: nothing dumped
// Optional dumps: pose_vio (T_ws_vio differs from T_ws), pose_init (corrected_poses for the keyframes with init_mask 1),
// loop_cov (COVINS_G; without it COVINS weights), lm_ref_mode (per landmark: 0 first observer, 1 none with observations,
// 2 none without observations, 3 an invalid keyframe outside the chain).
#include <cstdio>
#include <cstring>
#include <fstream>
#include <string>

#include "../../covins_b200/csrc/host/covins_b200_shim.hpp"
#include "mock_containers.hpp"

using namespace mock;

template <class T>
static std::vector<T> rd(const std::string& dir, const char* name) {
  std::ifstream f(dir + "/" + name + ".bin", std::ios::binary | std::ios::ate);
  if (!f) return {};
  const size_t n = (size_t)f.tellg() / sizeof(T);
  std::vector<T> v(n);
  f.seekg(0);
  f.read(reinterpret_cast<char*>(v.data()), n * sizeof(T));
  return v;
}
static Transform pose7_to_T(const double* p) { return covins_b200::detail::pose7_to_transform<Transform>(p); }

void Keyframe::UpdateCeresFromState(double* pose, double* vb, double* extr) const {
  covins_b200::detail::transform_to_pose7(T_w_s_, pose);
  covins_b200::detail::transform_to_pose7(T_s_c_, extr);
  for (int k = 0; k < 3; k++) { vb[k] = velocity_[k]; vb[3 + k] = bias_accel_[k]; vb[6 + k] = bias_gyro_[k]; }
}

// ---------------------------------------------------------------------------------------------------------------
// REFERENCE COPY, kept for this comparison only: covins_b200::PoseGraphOptimization as it was before cvb_pgo (host edge
// construction, cvb_ba_solve, host write-back).  The conversions it called are the shim's detail:: functions of that
// time, copied here as they were, so that the comparison also checks include/covins_b200_pose.h against them.
// ---------------------------------------------------------------------------------------------------------------
namespace reference {
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

}  // namespace detail
template <class MapPtr, class PoseMap>
void PoseGraphOptimization(covins_b200::Context& ctx, MapPtr map, PoseMap corrected_poses, const covins_b200::OptParams& P) {
  using covins_b200::detail::Flat;
  using KF = Keyframe;
  auto keyframes = map->GetKeyframesVec();
  auto landmarks = map->GetLandmarksVec();
  Flat F;
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
    auto mit = corrected_poses.find(kf->id_);
    const Transform T_ws_init = (mit != corrected_poses.end()) ? mit->second : kf->GetPoseTws();
    detail::transform_to_pose7(T_ws_init, &F.pose[7 * (size_t)k]);
    F.cam_of_kf[k] = k;
    if (kf->id_.first == 0 && kf->id_.second == map->id_map_) F.pose_const[k] = 1;
    if (kf->is_gba_optimized_ && P.pgo_fix_kfs_after_gba) F.pose_const[k] = 1;
    else if (kf->is_loaded_ && P.pgo_fix_poses_loaded_maps) F.pose_const[k] = 1;
  }
  double S1[36] = {0}, S23[36] = {0}, S45[36] = {0};
  for (int d = 0; d < 6; d++) {
    S1[7 * d] = (d < 3 ? P.wt_kf_r : P.wt_kf_t) * P.wt_kf_n1;
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
  for (const auto& lc : map->GetLoopConstraints()) {
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
  std::set<std::pair<const KF*, const KF*>> inserted_edges;
  for (int k = 0; k < K; k++) {
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
  if (P.use_nbr_kfs) {
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
  std::map<idpair, Transform> non_corrected_poses;
  for (int k = 0; k < K; k++) {
    auto& kf = kfs[k];
    const Transform T_ws_uncorrected = kf->GetPoseTws();
    non_corrected_poses[kf->id_] = T_ws_uncorrected;
    const Transform T_ws_corrected = detail::pose7_to_transform<Transform>(&o_pose[7 * (size_t)k]);
    const auto vel = kf->GetStateVelocity();
    kf->SetPoseTws(T_ws_corrected);
    double v[3];
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
}  // namespace reference

struct Built {
  std::shared_ptr<Map> map;
  std::vector<KeyframePtr> kfs;
  std::vector<LandmarkPtr> lms;
  std::map<idpair, Transform> corrected;
};

static Built build(const std::string& dir) {
  auto pose = rd<double>(dir, "pose"); auto vio = rd<double>(dir, "pose_vio"); auto init = rd<double>(dir, "pose_init");
  auto init_mask = rd<uint8_t>(dir, "init_mask"); auto sb = rd<double>(dir, "speedbias"); auto lm = rd<double>(dir, "lm");
  auto ptr = rd<int32_t>(dir, "lm_obs_ptr"); auto okf = rd<int32_t>(dir, "obs_kf"); auto agent = rd<int32_t>(dir, "agent_of");
  auto kfid = rd<int32_t>(dir, "kf_id"); auto li = rd<int32_t>(dir, "loop_i"); auto lj = rd<int32_t>(dir, "loop_j");
  auto lq = rd<double>(dir, "loop_q"); auto lt = rd<double>(dir, "loop_t"); auto lcov = rd<double>(dir, "loop_cov");
  auto ref_mode = rd<int32_t>(dir, "lm_ref_mode");
  const int K = (int)pose.size() / 7, L = (int)lm.size() / 3;
  Built B;
  B.map = std::make_shared<Map>();
  B.kfs.resize(K);
  for (int k = 0; k < K; k++) {
    auto kf = std::make_shared<Keyframe>();
    kf->id_ = {(size_t)kfid[k], (size_t)agent[k]};
    kf->T_w_s_ = pose7_to_T(&pose[7 * k]);
    kf->T_w_s_vio_ = vio.empty() ? kf->T_w_s_ : pose7_to_T(&vio[7 * k]);
    if (!sb.empty())
      for (int c = 0; c < 3; c++) kf->velocity_[c] = sb[9 * k + c];
    if (k > 0 && agent[k - 1] == agent[k]) { kf->pred = B.kfs[k - 1]; B.kfs[k - 1]->succ = kf; }
    if (!init.empty() && init_mask[k]) B.corrected[kf->id_] = pose7_to_T(&init[7 * k]);
    B.kfs[k] = kf;
    B.map->keyframes_[kf->id_] = kf;
  }
  auto ghost = std::make_shared<Keyframe>();   // a culled keyframe: in the map, invalid, outside every chain
  ghost->id_ = {100000, 0};
  ghost->invalid = true;
  B.map->keyframes_[ghost->id_] = ghost;
  B.lms.resize(L);
  for (int l = 0; l < L; l++) {
    auto p = std::make_shared<Landmark>();
    p->id_ = {(size_t)l, 0};
    p->pos_w_ = {lm[3 * l], lm[3 * l + 1], lm[3 * l + 2]};
    const int mode = ref_mode.empty() ? 0 : ref_mode[l];
    if (mode != 2)
      for (int o = ptr[l]; o < ptr[l + 1]; o++) {
        p->observations_[B.kfs[okf[o]]] = (size_t)o;
        if (!p->ref_kf && mode == 0) p->ref_kf = B.kfs[okf[o]];
      }
    if (mode == 3) p->ref_kf = ghost;
    B.lms[l] = p;
    B.map->landmarks_[p->id_] = p;
  }
  for (size_t e = 0; e < li.size(); e++) {
    LoopConstraint lc;
    lc.kf1 = B.kfs[li[e]]; lc.kf2 = B.kfs[lj[e]];
    double p7[7] = {lq[4 * e], lq[4 * e + 1], lq[4 * e + 2], lq[4 * e + 3], lt[3 * e], lt[3 * e + 1], lt[3 * e + 2]};
    lc.T_s1_s2 = pose7_to_T(p7);
    for (int i = 0; i < 36; i++) lc.cov_mat.m[i] = lcov.empty() ? ((i % 7 == 0) ? 1.0 : 0.0) : lcov[36 * e + i];
    B.map->loops_.push_back(lc);
  }
  return B;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string dir = argv[1];
  if (rd<double>(dir, "pose").empty()) return 2;
  const bool covins = rd<double>(dir, "loop_cov").empty();
  covins_b200::Context ctx(0);
  covins_b200::OptParams P;
  P.placerec_type_covins = covins;
  Built A = build(dir), B = build(dir);
  reference::PoseGraphOptimization(ctx, A.map, A.corrected, P);
  covins_b200::PoseGraphOptimization(ctx, B.map, B.corrected, P);
  int bad = 0, moved = 0, erased = 0;
  for (size_t k = 0; k < A.kfs.size(); k++) {
    const Keyframe &a = *A.kfs[k], &b = *B.kfs[k];
    if (std::memcmp(a.T_w_s_.m, b.T_w_s_.m, sizeof(a.T_w_s_.m)) || std::memcmp(a.velocity_.data(), b.velocity_.data(), 24) ||
        a.n_pose_optimized != b.n_pose_optimized) {
      std::printf("keyframe %zu differs\n", k);
      bad++;
    }
    if (std::memcmp(a.T_w_s_.m, a.T_w_s_vio_.m, sizeof(a.T_w_s_.m))) moved++;
  }
  for (size_t l = 0; l < A.lms.size(); l++) {
    const bool ina = A.map->landmarks_.count(A.lms[l]->id_), inb = B.map->landmarks_.count(B.lms[l]->id_);
    erased += !ina;
    if (ina != inb || std::memcmp(A.lms[l]->pos_w_.data(), B.lms[l]->pos_w_.data(), 24) || A.lms[l]->n_optimized != B.lms[l]->n_optimized) {
      std::printf("landmark %zu differs\n", l);
      bad++;
    }
  }
  std::printf("shim_pgo_test: K=%zu L=%zu loops=%zu covins=%d moved=%d erased=%d differing=%d\n", A.kfs.size(), A.lms.size(),
              A.map->loops_.size(), (int)covins, moved, erased, bad);
  return bad ? 1 : 0;
}
