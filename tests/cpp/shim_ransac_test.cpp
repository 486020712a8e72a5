// covins_b200::RansacAbsolutePose (covins_b200_shim.hpp) on a batch dumped by tests/test_ransac_absolute.py; writes what the
// wrapper returns so that the test can compare it with the Python path.
//   shim_ransac_test <dir>
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

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string dir = argv[1];
  const auto ptr = rd<int32_t>(dir, "prob_ptr"), samples = rd<int32_t>(dir, "samples");
  const auto pts = rd<double>(dir, "pts"), f = rd<double>(dir, "bearings"), sigma = rd<double>(dir, "sigma"), cam_off = rd<double>(dir, "cam_off"),
             cam_rot = rd<double>(dir, "cam_rot"), prm = rd<double>(dir, "params");   // threshold, max_iterations, probability
  if (ptr.empty() || prm.size() != 3) return 2;
  const size_t n_prob = ptr.size() - 1, per = samples.size() / (n_prob ? n_prob : 1);
  std::vector<covins_b200::AbsolutePoseRansacProblem> problems(n_prob);
  for (size_t i = 0; i < n_prob; i++) {
    auto& p = problems[i];
    p.points.assign(pts.begin() + 3 * ptr[i], pts.begin() + 3 * ptr[i + 1]);
    p.bearings.assign(f.begin() + 3 * ptr[i], f.begin() + 3 * ptr[i + 1]);
    p.sigma_angles.assign(sigma.begin() + ptr[i], sigma.begin() + ptr[i + 1]);
    for (int k = 0; k < 3; k++) p.cam_offset[k] = cam_off[3 * i + k];
    for (int k = 0; k < 9; k++) p.cam_rotation[k] = cam_rot[9 * i + k];
    p.samples.assign(samples.begin() + per * i, samples.begin() + per * (i + 1));
  }
  covins_b200::Context ctx(0);
  const auto res = covins_b200::RansacAbsolutePose(ctx, problems, prm[0], (int)prm[1], prm[2]);
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
