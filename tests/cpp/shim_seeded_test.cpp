// The seeded forms of the C++ wrapper (covins_b200_shim.hpp) on a batch dumped by tests/test_ransac_seeded.py: the problems
// with their samples left empty and one seed per problem (seeds.bin); writes what the wrappers return so that the test can
// compare it with the Python path.
//   shim_seeded_test abs|rel|rel5 <dir>   RansacAbsolutePose / RansacNonCentralRelativePose / RansacCentralRelativePose
//                                          → seeded_ints (best_sample, n_inliers, iterations, samples_used), seeded_models,
//                                          seeded_mask
//   shim_seeded_test cov <dir>             RansacNonCentralRelativePose, then NonCentralRelativePoseCovariance with 300 samples
//                                          → seeded_models, seeded_cov, seeded_n_valid
// params.bin: threshold, max_iterations, probability.
#include <fstream>
#include <string>
#include <vector>

#include "../../covins_b200/csrc/host/covins_b200_shim.hpp"

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

template <class Result>
static void write_ransac(const std::string& dir, const std::vector<Result>& res) {
  std::vector<int32_t> ints;
  std::vector<double> models;
  std::vector<uint8_t> mask;
  for (const auto& r : res) {
    ints.insert(ints.end(), {r.best_sample, r.n_inliers, r.iterations, r.samples_used});
    models.insert(models.end(), r.model.begin(), r.model.end());
    mask.insert(mask.end(), r.inliers.begin(), r.inliers.end());
  }
  wr(dir, "seeded_ints", ints);
  wr(dir, "seeded_models", models);
  wr(dir, "seeded_mask", mask);
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const std::string mode = argv[1], dir = argv[2];
  const auto ptr = rd<int32_t>(dir, "prob_ptr");
  const auto seeds = rd<uint64_t>(dir, "seeds");
  const auto prm = rd<double>(dir, "params");
  if (ptr.empty() || prm.size() != 3 || seeds.size() != ptr.size() - 1) return 2;
  const size_t n_prob = ptr.size() - 1;
  covins_b200::Context ctx(0);
  if (mode == "abs") {
    const auto pts = rd<double>(dir, "pts"), f = rd<double>(dir, "bearings"), sigma = rd<double>(dir, "sigma"), cam_off = rd<double>(dir, "cam_off"),
               cam_rot = rd<double>(dir, "cam_rot");
    std::vector<covins_b200::AbsolutePoseRansacProblem> problems(n_prob);
    for (size_t i = 0; i < n_prob; i++) {
      auto& p = problems[i];
      p.points = slice(pts, 3 * ptr[i], 3 * ptr[i + 1]); p.bearings = slice(f, 3 * ptr[i], 3 * ptr[i + 1]);
      p.sigma_angles = slice(sigma, ptr[i], ptr[i + 1]);
      for (int k = 0; k < 3; k++) p.cam_offset[k] = cam_off[3 * i + k];
      for (int k = 0; k < 9; k++) p.cam_rotation[k] = cam_rot[9 * i + k];
    }
    write_ransac(dir, covins_b200::RansacAbsolutePose(ctx, problems, seeds, prm[0], (int)prm[1], prm[2]));
    return 0;
  }
  const auto f1 = rd<double>(dir, "f1"), f2 = rd<double>(dir, "f2"), s1 = rd<double>(dir, "sigma1"), s2 = rd<double>(dir, "sigma2");
  if (mode == "rel5") {
    std::vector<covins_b200::CentralRelativePoseRansacProblem> problems(n_prob);
    for (size_t i = 0; i < n_prob; i++) {
      auto& p = problems[i];
      const size_t a = ptr[i], b = ptr[i + 1];
      p.bearings1 = slice(f1, 3 * a, 3 * b); p.bearings2 = slice(f2, 3 * a, 3 * b);
      p.sigma1 = slice(s1, a, b); p.sigma2 = slice(s2, a, b);
    }
    write_ransac(dir, covins_b200::RansacCentralRelativePose(ctx, problems, seeds, prm[0], (int)prm[1], prm[2]));
    return 0;
  }
  const auto cam1 = rd<int32_t>(dir, "cam1"), cam2 = rd<int32_t>(dir, "cam2"), cp1 = rd<int32_t>(dir, "cam_ptr1"), cp2 = rd<int32_t>(dir, "cam_ptr2");
  const auto co1 = rd<double>(dir, "cam_off1"), cr1 = rd<double>(dir, "cam_rot1"), co2 = rd<double>(dir, "cam_off2"), cr2 = rd<double>(dir, "cam_rot2");
  std::vector<covins_b200::NonCentralRelativePoseRansacProblem> problems(n_prob);
  for (size_t i = 0; i < n_prob; i++) {
    auto& p = problems[i];
    const size_t a = ptr[i], b = ptr[i + 1];
    p.bearings1 = slice(f1, 3 * a, 3 * b); p.bearings2 = slice(f2, 3 * a, 3 * b);
    p.sigma1 = slice(s1, a, b); p.sigma2 = slice(s2, a, b);
    p.cam1 = slice(cam1, a, b); p.cam2 = slice(cam2, a, b);
    p.rig1_offsets = slice(co1, 3 * cp1[i], 3 * cp1[i + 1]); p.rig1_rotations = slice(cr1, 9 * cp1[i], 9 * cp1[i + 1]);
    p.rig2_offsets = slice(co2, 3 * cp2[i], 3 * cp2[i + 1]); p.rig2_rotations = slice(cr2, 9 * cp2[i], 9 * cp2[i + 1]);
  }
  const auto ransac = covins_b200::RansacNonCentralRelativePose(ctx, problems, seeds, prm[0], (int)prm[1], prm[2]);
  if (mode == "rel") {
    write_ransac(dir, ransac);
    return 0;
  }
  if (mode != "cov") return 2;
  const auto cov = covins_b200::NonCentralRelativePoseCovariance(ctx, problems, ransac, 300, seeds);
  std::vector<double> models, covs;
  std::vector<int32_t> n_valid;
  for (size_t i = 0; i < n_prob; i++) {
    models.insert(models.end(), ransac[i].model.begin(), ransac[i].model.end());
    covs.insert(covs.end(), cov[i].cov.begin(), cov[i].cov.end());
    n_valid.push_back(cov[i].n_valid);
  }
  wr(dir, "seeded_models", models);
  wr(dir, "seeded_cov", covs);
  wr(dir, "seeded_n_valid", n_valid);
  return 0;
}
