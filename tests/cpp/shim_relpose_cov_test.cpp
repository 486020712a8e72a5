// covins_b200::RansacNonCentralRelativePose, then covins_b200::NonCentralRelativePoseCovariance (covins_b200_shim.hpp) on a
// batch dumped by tests/test_relpose_covariance.py; writes what the wrappers return so that the test can compare it with the
// Python path.  Then every covariance with a model goes into a mock LoopConstraint (cov_mat, T_s1_s2 from the model) of a
// small keyframe chain and through covins_b200::PoseGraphOptimization in COVINS_G mode (the loop edge whitened by cov_mat,
// which exits if cov_mat is not positive definite); writes the optimised poses.
//   shim_relpose_cov_test <dir>
#include <fstream>
#include <string>
#include <vector>

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
static void wr(const std::string& dir, const char* name, const std::vector<T>& v) {
  std::ofstream f(dir + "/" + name + ".bin", std::ios::binary);
  f.write(reinterpret_cast<const char*>(v.data()), v.size() * sizeof(T));
}
template <class T>
static std::vector<T> slice(const std::vector<T>& v, size_t a, size_t b) {
  return std::vector<T>(v.begin() + a, v.begin() + b);
}

void Keyframe::UpdateCeresFromState(double* pose, double* vb, double* extr) const {
  covins_b200::detail::transform_to_pose7(T_w_s_, pose);
  covins_b200::detail::transform_to_pose7(T_s_c_, extr);
  for (int k = 0; k < 3; k++) { vb[k] = velocity_[k]; vb[3 + k] = bias_accel_[k]; vb[6 + k] = bias_gyro_[k]; }
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string dir = argv[1];
  const auto ptr = rd<int32_t>(dir, "prob_ptr"), samples = rd<int32_t>(dir, "samples"), cov_samples = rd<int32_t>(dir, "cov_samples"),
             cam1 = rd<int32_t>(dir, "cam1"), cam2 = rd<int32_t>(dir, "cam2"), cp1 = rd<int32_t>(dir, "cam_ptr1"), cp2 = rd<int32_t>(dir, "cam_ptr2");
  const auto f1 = rd<double>(dir, "f1"), f2 = rd<double>(dir, "f2"), s1 = rd<double>(dir, "sigma1"), s2 = rd<double>(dir, "sigma2"),
             co1 = rd<double>(dir, "cam_off1"), cr1 = rd<double>(dir, "cam_rot1"), co2 = rd<double>(dir, "cam_off2"), cr2 = rd<double>(dir, "cam_rot2"),
             prm = rd<double>(dir, "params");   // threshold, max_iterations, probability
  if (ptr.empty() || prm.size() != 3) return 2;
  const size_t n_prob = ptr.size() - 1, per = samples.size() / (n_prob ? n_prob : 1), per_cov = cov_samples.size() / (n_prob ? n_prob : 1);
  std::vector<covins_b200::NonCentralRelativePoseRansacProblem> problems(n_prob);
  for (size_t i = 0; i < n_prob; i++) {
    auto& p = problems[i];
    const size_t a = ptr[i], b = ptr[i + 1];
    p.bearings1 = slice(f1, 3 * a, 3 * b); p.bearings2 = slice(f2, 3 * a, 3 * b);
    p.sigma1 = slice(s1, a, b); p.sigma2 = slice(s2, a, b);
    p.cam1 = slice(cam1, a, b); p.cam2 = slice(cam2, a, b);
    p.rig1_offsets = slice(co1, 3 * cp1[i], 3 * cp1[i + 1]); p.rig1_rotations = slice(cr1, 9 * cp1[i], 9 * cp1[i + 1]);
    p.rig2_offsets = slice(co2, 3 * cp2[i], 3 * cp2[i + 1]); p.rig2_rotations = slice(cr2, 9 * cp2[i], 9 * cp2[i + 1]);
    p.samples = slice(samples, per * i, per * (i + 1));
  }
  covins_b200::Context ctx(0);
  const auto ransac = covins_b200::RansacNonCentralRelativePose(ctx, problems, prm[0], (int)prm[1], prm[2]);
  for (size_t i = 0; i < n_prob; i++) problems[i].samples = slice(cov_samples, per_cov * i, per_cov * (i + 1));
  const auto cov = covins_b200::NonCentralRelativePoseCovariance(ctx, problems, ransac);
  std::vector<double> models, covs;
  std::vector<int32_t> n_valid;
  for (size_t i = 0; i < n_prob; i++) {
    models.insert(models.end(), ransac[i].model.begin(), ransac[i].model.end());
    covs.insert(covs.end(), cov[i].cov.begin(), cov[i].cov.end());
    n_valid.push_back(cov[i].n_valid);
  }
  wr(dir, "out_models", models);
  wr(dir, "out_cov", covs);
  wr(dir, "out_n_valid", n_valid);

  // the loop edges of a 12-keyframe chain (one agent, keyframe 0 fixed): edge i between keyframes i and 11 - i, its relative
  // pose the problem's model, its information from the problem's covariance
  constexpr int K = 12;
  auto map = std::make_shared<Map>();
  std::vector<KeyframePtr> kfs(K);
  for (int k = 0; k < K; k++) {
    auto kf = std::make_shared<Keyframe>();
    kf->id_ = {(size_t)k, 0};
    kf->T_w_s_(0, 3) = 0.5 * k; kf->T_w_s_(1, 3) = 0.1 * k * k;
    kf->T_w_s_vio_ = kf->T_w_s_;
    if (k > 0) { kf->pred = kfs[k - 1]; kfs[k - 1]->succ = kf; }
    kfs[k] = kf;
    map->keyframes_[kf->id_] = kf;
  }
  int n_loops = 0;
  for (size_t i = 0; i < n_prob && n_loops < K / 2; i++) {
    if (cov[i].n_valid == 0) continue;
    LoopConstraint lc;
    lc.kf1 = kfs[n_loops]; lc.kf2 = kfs[K - 1 - n_loops];
    lc.T_s1_s2 = Transform::Identity();
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 4; c++) lc.T_s1_s2(r, c) = ransac[i].model[4 * r + c];
    for (int j = 0; j < 36; j++) lc.cov_mat.m[j] = cov[i].cov[j];
    map->loops_.push_back(lc);
    n_loops++;
  }
  covins_b200::OptParams P;   // placerec_type_covins = false: COVINS_G, loop edges whitened by cov_mat
  std::map<idpair, Transform> corrected;
  covins_b200::PoseGraphOptimization(ctx, map, corrected, P);
  std::vector<double> poses(7 * K + 1);
  for (int k = 0; k < K; k++) covins_b200::detail::transform_to_pose7(kfs[k]->T_w_s_, &poses[7 * k]);
  poses[7 * K] = n_loops;
  wr(dir, "out_pgo", poses);
  return 0;
}
