// GlobalBundleAdjustment through the C++ shim on mock containers, on one Context or on a ContextGroup of several contexts,
// from a flat problem dumped by tests/test_ba_group.py; dumps the states written back into the containers.
//   shim_group_test <dir> single|group <ranks> <peer_path>       (group: every rank on device 0)
#include <cstdio>
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
template <class T>
static void wr(const std::string& dir, const std::string& name, const std::vector<T>& v) {
  std::ofstream f(dir + "/" + name + ".bin", std::ios::binary);
  f.write(reinterpret_cast<const char*>(v.data()), v.size() * sizeof(T));
}
static Transform pose7_to_T(const double* p) { return covins_b200::detail::pose7_to_transform<Transform>(p); }

void Keyframe::UpdateCeresFromState(double* pose, double* vb, double* extr) const {
  covins_b200::detail::transform_to_pose7(T_w_s_, pose);
  covins_b200::detail::transform_to_pose7(T_s_c_, extr);
  for (int k = 0; k < 3; k++) { vb[k] = velocity_[k]; vb[3 + k] = bias_accel_[k]; vb[6 + k] = bias_gyro_[k]; }
}

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  const std::string dir = argv[1], mode = argv[2];
  const int ranks = std::atoi(argv[3]);
  const bool peer = std::atoi(argv[4]) != 0;
  auto pose = rd<double>(dir, "pose"); auto sb = rd<double>(dir, "speedbias"); auto extr = rd<double>(dir, "extr");
  auto intr = rd<double>(dir, "intr"); auto dist = rd<double>(dir, "dist"); auto lm = rd<double>(dir, "lm");
  auto ptr = rd<int32_t>(dir, "lm_obs_ptr"); auto okf = rd<int32_t>(dir, "obs_kf"); auto uv = rd<float>(dir, "obs_uv");
  auto sig = rd<double>(dir, "obs_sigma"); auto agent = rd<int32_t>(dir, "agent_of"); auto kfid = rd<int32_t>(dir, "kf_id");
  auto imu_j = rd<int32_t>(dir, "imu_j"); auto imu_ptr = rd<int32_t>(dir, "imu_ptr"); auto imu_dt = rd<double>(dir, "imu_dt");
  auto imu_acc = rd<double>(dir, "imu_acc"); auto imu_gyr = rd<double>(dir, "imu_gyr"); auto a0 = rd<double>(dir, "imu_acc0");
  auto g0 = rd<double>(dir, "imu_gyr0"); auto noise = rd<double>(dir, "imu_noise");
  auto li = rd<int32_t>(dir, "loop_i"); auto lj = rd<int32_t>(dir, "loop_j"); auto lq = rd<double>(dir, "loop_q"); auto lt = rd<double>(dir, "loop_t");
  const int K = (int)pose.size() / 7, L = (int)lm.size() / 3;
  auto map = std::make_shared<Map>();
  map->id_map_ = 0;
  std::vector<KeyframePtr> kfs(K);
  for (int k = 0; k < K; k++) {
    auto kf = std::make_shared<Keyframe>();
    kf->id_ = {(size_t)kfid[k], (size_t)agent[k]};
    kf->T_w_s_ = pose7_to_T(&pose[7 * k]);
    kf->T_w_s_vio_ = kf->T_w_s_;
    kf->T_s_c_ = pose7_to_T(&extr[0]);
    for (int c = 0; c < 3; c++) { kf->velocity_[c] = sb[9 * k + c]; kf->bias_accel_[c] = sb[9 * k + 3 + c]; kf->bias_gyro_[c] = sb[9 * k + 6 + c]; }
    for (int c = 0; c < 4; c++) { kf->intr[c] = intr[c]; kf->dist[c] = dist[c]; }
    if (k > 0 && agent[k - 1] == agent[k]) { kf->pred = kfs[k - 1]; kfs[k - 1]->succ = kf; }
    kfs[k] = kf;
    map->keyframes_[kf->id_] = kf;
  }
  for (size_t f = 0; f < imu_j.size(); f++) {
    auto& kf = kfs[imu_j[f]];
    kf->imu_dt.assign(imu_dt.begin() + imu_ptr[f], imu_dt.begin() + imu_ptr[f + 1]);
    kf->imu_acc.assign(imu_acc.begin() + 3 * imu_ptr[f], imu_acc.begin() + 3 * imu_ptr[f + 1]);
    kf->imu_gyr.assign(imu_gyr.begin() + 3 * imu_ptr[f], imu_gyr.begin() + 3 * imu_ptr[f + 1]);
    for (int c = 0; c < 3; c++) { kf->imu_acc0[c] = a0[3 * f + c]; kf->imu_gyr0[c] = g0[3 * f + c]; }
    for (int c = 0; c < 5; c++) kf->imu_noise[c] = noise[c];
  }
  std::vector<LandmarkPtr> lms(L);
  for (int l = 0; l < L; l++) {
    auto p = std::make_shared<Landmark>();
    p->id_ = {(size_t)l, 0};
    p->pos_w_ = {lm[3 * l], lm[3 * l + 1], lm[3 * l + 2]};
    for (int o = ptr[l]; o < ptr[l + 1]; o++) {
      auto& kf = kfs[okf[o]];
      const size_t feat = kf->keypoints_distorted_.size();
      kf->keypoints_distorted_.push_back({uv[2 * o], uv[2 * o + 1]});
      kf->keypoints_aors_.push_back({0.f, (float)(sig[o] / 2.0 - 1.0), 0.f, 0.f});
      kf->landmarks_.push_back(p);
      p->observations_[kf] = feat;
      if (!p->ref_kf) p->ref_kf = kf;
    }
    lms[l] = p;
    map->landmarks_[p->id_] = p;
  }
  for (size_t e = 0; e < li.size(); e++) {
    LoopConstraint lc;
    lc.kf1 = kfs[li[e]]; lc.kf2 = kfs[lj[e]];
    double p7[7] = {lq[4 * e], lq[4 * e + 1], lq[4 * e + 2], lq[4 * e + 3], lt[3 * e], lt[3 * e + 1], lt[3 * e + 2]};
    lc.T_s1_s2 = pose7_to_T(p7);
    for (int i = 0; i < 36; i++) lc.cov_mat.m[i] = (i % 7 == 0) ? 1.0 : 0.0;
    map->loops_.push_back(lc);
  }
  covins_b200::OptParams P;
  if (mode == "single") {
    covins_b200::Context ctx(0);
    covins_b200::GlobalBundleAdjustment(ctx, map, 4, -1.0, false, true, false, P);
  } else if (mode == "group") {
    covins_b200::ContextGroup group(std::vector<int>(ranks, 0));
    covins_b200::GlobalBundleAdjustment(group, map, 4, -1.0, false, true, false, P, peer);
  } else {
    return 2;
  }
  std::vector<double> o_pose(7 * (size_t)K), o_sb(9 * (size_t)K), o_lm(3 * (size_t)L);
  std::vector<int32_t> n_obs_left(L);
  for (int k = 0; k < K; k++) {
    covins_b200::detail::transform_to_pose7(kfs[k]->T_w_s_, &o_pose[7 * (size_t)k]);
    for (int c = 0; c < 3; c++) { o_sb[9 * k + c] = kfs[k]->velocity_[c]; o_sb[9 * k + 3 + c] = kfs[k]->bias_accel_[c]; o_sb[9 * k + 6 + c] = kfs[k]->bias_gyro_[c]; }
  }
  for (int l = 0; l < L; l++) {
    for (int c = 0; c < 3; c++) o_lm[3 * l + c] = lms[l]->pos_w_[c];
    n_obs_left[l] = (int32_t)lms[l]->observations_.size();
  }
  const std::string tag = mode == "single" ? "single" : "group";
  wr(dir, tag + "_pose", o_pose); wr(dir, tag + "_sb", o_sb); wr(dir, tag + "_lm", o_lm); wr(dir, tag + "_nobs", n_obs_left);
  std::printf("shim_group_test %s: K=%d L=%d ranks=%d\n", mode.c_str(), K, L, mode == "single" ? 1 : ranks);
  return 0;
}
