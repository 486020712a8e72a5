// covins_b200::RansacCentralRelativePose (covins_b200_shim.hpp) on a batch dumped by tests/test_ransac_central.py; writes what
// the wrapper returns so that the test can compare it with the Python path.
//   shim_ransac_rel5_test <dir>
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
  const auto ptr = rd<int32_t>(dir, "prob_ptr"), samples = rd<int32_t>(dir, "samples");
  const auto f1 = rd<double>(dir, "f1"), f2 = rd<double>(dir, "f2"), s1 = rd<double>(dir, "sigma1"), s2 = rd<double>(dir, "sigma2"),
             prm = rd<double>(dir, "params");   // threshold, max_iterations, probability
  if (ptr.empty() || prm.size() != 3) return 2;
  const size_t n_prob = ptr.size() - 1, per = samples.size() / (n_prob ? n_prob : 1);
  std::vector<covins_b200::CentralRelativePoseRansacProblem> problems(n_prob);
  for (size_t i = 0; i < n_prob; i++) {
    auto& p = problems[i];
    const size_t a = ptr[i], b = ptr[i + 1];
    p.bearings1 = slice(f1, 3 * a, 3 * b); p.bearings2 = slice(f2, 3 * a, 3 * b);
    p.sigma1 = slice(s1, a, b); p.sigma2 = slice(s2, a, b);
    p.samples = slice(samples, per * i, per * (i + 1));
  }
  covins_b200::Context ctx(0);
  const auto res = covins_b200::RansacCentralRelativePose(ctx, problems, prm[0], (int)prm[1], prm[2]);
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
