// covins_b200::RansacNonCentralRelativePose (covins_b200_shim.hpp) on a batch dumped by tests/test_ransac_relative.py; writes
// what the wrapper returns so that the test can compare it with the Python path.
//   shim_ransac_rel_test <dir>
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

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string dir = argv[1];
  const auto ptr = rd<int32_t>(dir, "prob_ptr"), samples = rd<int32_t>(dir, "samples"), cam1 = rd<int32_t>(dir, "cam1"), cam2 = rd<int32_t>(dir, "cam2"),
             cp1 = rd<int32_t>(dir, "cam_ptr1"), cp2 = rd<int32_t>(dir, "cam_ptr2");
  const auto f1 = rd<double>(dir, "f1"), f2 = rd<double>(dir, "f2"), s1 = rd<double>(dir, "sigma1"), s2 = rd<double>(dir, "sigma2"),
             co1 = rd<double>(dir, "cam_off1"), cr1 = rd<double>(dir, "cam_rot1"), co2 = rd<double>(dir, "cam_off2"), cr2 = rd<double>(dir, "cam_rot2"),
             prm = rd<double>(dir, "params");   // threshold, max_iterations, probability
  if (ptr.empty() || prm.size() != 3) return 2;
  const size_t n_prob = ptr.size() - 1, per = samples.size() / (n_prob ? n_prob : 1);
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
  const auto res = covins_b200::RansacNonCentralRelativePose(ctx, problems, prm[0], (int)prm[1], prm[2]);
  std::vector<int32_t> ints;
  std::vector<double> models;
  std::vector<uint8_t> mask;
  for (const auto& r : res) {
    ints.insert(ints.end(), {r.best_sample, r.n_inliers, r.iterations, r.samples_used});
    models.insert(models.end(), r.model.begin(), r.model.end());
    mask.insert(mask.end(), r.inliers.begin(), r.inliers.end());
  }
  wr(dir, "out_ints", ints);
  wr(dir, "out_models", models);
  wr(dir, "out_mask", mask);
  return 0;
}
