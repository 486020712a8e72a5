// VerifyNonCentralRelativePose of the C++ wrapper (covins_b200_shim.hpp), SIFT overload, on a scene dumped by
// tests/test_verify_relative_sift.py; writes what the wrapper returns so that the test can compare it with the Python path.
//   shim_verify_sift_test <dir>   → verify_ints (per pairing: n_matches, best_sample, n_inliers, iterations, samples_used; then
//                                   per candidate: best_sample, n_inliers, iterations, samples_used, n_valid), verify_models
//                                   (5-point, then 17-point), verify_cov, verify_corr
// desc.bin: float32 [R][128]; params.bin: img_match_thres, ratio_thres, threshold5, max_iterations5, threshold17, max_iterations17,
// probability, n_cov_samples.
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
  if (argc != 2) return 1;
  const std::string dir = argv[1];
  const auto kf_ptr = rd<int32_t>(dir, "kf_ptr"), cp1 = rd<int32_t>(dir, "cam_ptr1"), cp2 = rd<int32_t>(dir, "cam_ptr2");
  const auto pair_ptr = rd<int32_t>(dir, "pair_ptr"), pairs = rd<int32_t>(dir, "pairs");
  const auto desc = rd<float>(dir, "desc");
  const auto bear = rd<double>(dir, "bearings"), sig = rd<double>(dir, "sigma"), prm = rd<double>(dir, "params");
  const auto co1 = rd<double>(dir, "cam_off1"), cr1 = rd<double>(dir, "cam_rot1"), co2 = rd<double>(dir, "cam_off2"), cr2 = rd<double>(dir, "cam_rot2");
  const auto seeds5 = rd<uint64_t>(dir, "seeds5"), seeds = rd<uint64_t>(dir, "seeds");
  if (kf_ptr.empty() || pair_ptr.empty() || prm.size() != 8) return 2;   // nothing dumped: refused before any GPU work
  std::vector<covins_b200::VerifyKeyframeViewSIFT> kfs;
  for (size_t k = 0; k + 1 < kf_ptr.size(); k++)
    kfs.push_back({desc.data() + 128 * (size_t)kf_ptr[k], bear.data() + 3 * (size_t)kf_ptr[k], sig.data() + kf_ptr[k], kf_ptr[k + 1] - kf_ptr[k]});
  std::vector<covins_b200::VerifyCandidate> cands(pair_ptr.size() - 1);
  for (size_t c = 0; c < cands.size(); c++) {
    cands[c].rig1_offsets.assign(co1.begin() + 3 * cp1[c], co1.begin() + 3 * cp1[c + 1]);
    cands[c].rig1_rotations.assign(cr1.begin() + 9 * cp1[c], cr1.begin() + 9 * cp1[c + 1]);
    cands[c].rig2_offsets.assign(co2.begin() + 3 * cp2[c], co2.begin() + 3 * cp2[c + 1]);
    cands[c].rig2_rotations.assign(cr2.begin() + 9 * cp2[c], cr2.begin() + 9 * cp2[c + 1]);
    for (int q = pair_ptr[c]; q < pair_ptr[c + 1]; q++) cands[c].pairings.push_back({pairs[4 * q], pairs[4 * q + 1], pairs[4 * q + 2], pairs[4 * q + 3]});
  }
  covins_b200::VerifyParams P;
  P.img_match_thres = (float)prm[0]; P.ratio_thres = (float)prm[1]; P.threshold5 = prm[2]; P.max_iterations5 = (int)prm[3];
  P.threshold17 = prm[4]; P.max_iterations17 = (int)prm[5]; P.probability = prm[6]; P.n_cov_samples = (int)prm[7];
  covins_b200::Context ctx(0);
  const covins_b200::VerifyResult res = covins_b200::VerifyNonCentralRelativePose(ctx, kfs, cands, P, seeds5, seeds);
  std::vector<int32_t> ints, corr;
  std::vector<double> models, cov;
  for (const auto& q : res.pairings) {
    ints.insert(ints.end(), {q.n_matches, q.best_sample, q.n_inliers, q.iterations, q.samples_used});
    models.insert(models.end(), q.model.begin(), q.model.end());
  }
  for (const auto& c : res.candidates) {
    ints.insert(ints.end(), {c.best_sample, c.n_inliers, c.iterations, c.samples_used, c.n_valid});
    models.insert(models.end(), c.model.begin(), c.model.end());
    cov.insert(cov.end(), c.cov.begin(), c.cov.end());
  }
  for (const auto& e : res.correspondences) corr.insert(corr.end(), {e.pairing, e.row1, e.row2, e.inlier5, e.inlier17});
  wr(dir, "verify_ints", ints); wr(dir, "verify_models", models); wr(dir, "verify_cov", cov); wr(dir, "verify_corr", corr);
  return 0;
}
