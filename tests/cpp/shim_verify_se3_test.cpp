// VerifyLandmarkCandidates of the C++ wrapper (covins_b200_shim.hpp) on mock containers built from a scene dumped by
// tests/test_verify_landmark.py; writes what the wrapper returns so that the test can compare it with the Python path.
//   shim_verify_se3_test <dir>   → lmv_ints [C][6] (n_matches, best_sample, best_count, n_found, n_corr, n_inliers), lmv_pose [C][7],
//                                  lmv_T12 [C][16], lmv_lv [C][n_query] (the written-back LandmarkVector: the candidate keypoint
//                                  its landmark sits at, or -1)
// Keyframe k (0 = the query, 1.. the candidates): kf<k>_{kp,octave,desc,lm_valid,lm_pos,lm_maxdist,lm_desc,Tcw,Tws,Tsc,K,cam}.bin,
// the query also kf0_{bearings,sigma}.bin; seeds.bin; params.bin (12 doubles, LandmarkVerifyParams in declaration order).
// Exit 2 without a complete scene: refused before any GPU work.
#include <fstream>
#include <string>
#include <vector>

#include "../../covins_b200/csrc/host/covins_b200_shim.hpp"
#include "mock_containers.hpp"

// a keyframe with the bearing vectors and sigma angles the absolute-pose RANSAC reads
struct VKeyframe : mock::Keyframe {
  std::vector<double> bear, sig;
  void GetBearings(double* f, double* s) const {
    std::copy(bear.begin(), bear.end(), f);
    std::copy(sig.begin(), sig.end(), s);
  }
};
using VKeyframePtr = std::shared_ptr<VKeyframe>;
using LandmarkVector = std::vector<mock::LandmarkPtr>;

template <class T>
static std::vector<T> rd(const std::string& dir, const std::string& name) {
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

static bool load(const std::string& dir, int k, VKeyframePtr& kf) {
  const std::string p = "kf" + std::to_string(k) + "_";
  const auto kp = rd<float>(dir, p + "kp"), oct = rd<float>(dir, p + "octave");
  const auto md = rd<double>(dir, p + "lm_maxdist");
  const auto desc = rd<uint8_t>(dir, p + "desc"), lv = rd<uint8_t>(dir, p + "lm_valid"), ld = rd<uint8_t>(dir, p + "lm_desc");
  const auto pos = rd<double>(dir, p + "lm_pos"), Tcw = rd<double>(dir, p + "Tcw"), Tws = rd<double>(dir, p + "Tws"), Tsc = rd<double>(dir, p + "Tsc");
  const auto K = rd<double>(dir, p + "K"), cam = rd<double>(dir, p + "cam");
  const size_t n = oct.size();
  if (Tcw.size() != 16 || Tws.size() != 16 || Tsc.size() != 16 || K.size() != 9 || cam.size() != 8 || kp.size() != 2 * n || desc.size() != 32 * n ||
      lv.size() != n || ld.size() != 32 * n || pos.size() != 3 * n || md.size() != n)
    return false;
  kf = std::make_shared<VKeyframe>();
  kf->id_ = {0, (size_t)k};
  for (int i = 0; i < 16; i++) { kf->T_c_w_.m[i] = Tcw[i]; kf->T_w_s_.m[i] = Tws[i]; kf->T_s_c_.m[i] = Tsc[i]; }
  for (int i = 0; i < 9; i++) kf->K_[i] = K[i];
  for (int i = 0; i < 4; i++) { kf->intr[i] = cam[i]; kf->dist[i] = cam[4 + i]; }
  kf->keypoints_distorted_.resize(n); kf->keypoints_aors_.resize(n); kf->descriptors_.resize(n); kf->landmarks_.assign(n, nullptr);
  for (size_t i = 0; i < n; i++) {
    kf->keypoints_distorted_[i] = {kp[2 * i], kp[2 * i + 1]};
    kf->keypoints_aors_[i] = {0.f, oct[i], 0.f, 0.f};
    std::copy(desc.begin() + 32 * i, desc.begin() + 32 * (i + 1), kf->descriptors_[i].begin());
    if (!lv[i]) continue;
    auto lm = std::make_shared<mock::Landmark>();
    lm->id_ = {(size_t)k, i};
    lm->pos_w_ = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
    lm->max_distance_ = md[i];
    std::copy(ld.begin() + 32 * i, ld.begin() + 32 * (i + 1), lm->descriptor_.begin());
    lm->AddObservation(kf, i);
    kf->landmarks_[i] = lm;
  }
  return true;
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  const std::string dir = argv[1];
  const auto seeds = rd<uint64_t>(dir, "seeds");
  const auto prm = rd<double>(dir, "params");
  if (prm.size() != 12) return 2;
  VKeyframePtr query;
  if (!load(dir, 0, query)) return 2;
  query->bear = rd<double>(dir, "kf0_bearings"); query->sig = rd<double>(dir, "kf0_sigma");
  const size_t nq = query->keypoints_distorted_.size();
  if (query->bear.size() != 3 * nq || query->sig.size() != nq) return 2;
  std::vector<VKeyframePtr> cands(seeds.size());
  for (size_t c = 0; c < seeds.size(); c++)
    if (!load(dir, (int)c + 1, cands[c])) return 2;
  covins_b200::LandmarkVerifyParams P;
  P.distance_threshold = (float)prm[0]; P.num_best = (int)prm[1]; P.matches_thres = (int)prm[2]; P.ransac_threshold = prm[3];
  P.ransac_max_iterations = (int)prm[4]; P.ransac_probability = prm[5]; P.min_ransac_inliers = (int)prm[6]; P.search_radius_SE3 = prm[7];
  P.desc_matching_th_low = (int)prm[8]; P.num_octaves = (int)prm[9]; P.scale_factor = prm[10]; P.th_outlier_align = prm[11];
  covins_b200::Context ctx(0);
  std::vector<LandmarkVector> vv;
  const auto res = covins_b200::VerifyLandmarkCandidates<VKeyframePtr, LandmarkVector, mock::Transform>(ctx, query, cands, vv, P, seeds);
  std::vector<int32_t> ints, lv;
  std::vector<double> pose, T12;
  for (size_t c = 0; c < cands.size(); c++) {
    const auto& o = res[c];
    ints.insert(ints.end(), {o.n_matches, o.best_sample, o.best_count, o.n_found, o.n_corr, o.n_inliers});
    pose.insert(pose.end(), o.T12_pose, o.T12_pose + 7);
    T12.insert(T12.end(), o.T12.m, o.T12.m + 16);
    for (size_t i = 0; i < nq; i++) lv.push_back(vv[c][i] ? vv[c][i]->GetFeatureIndex(cands[c]) : -1);
  }
  wr(dir, "lmv_ints", ints); wr(dir, "lmv_pose", pose); wr(dir, "lmv_T12", T12); wr(dir, "lmv_lv", lv);
  return 0;
}
