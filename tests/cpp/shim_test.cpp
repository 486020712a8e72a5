// Exercises the C++ host shim (covins_b200_shim.hpp) on mock containers built from a flat problem dumped by
// tests/test_gpu_shim.py, then dumps the states the shim wrote back into the containers.
//   shim_test <dir> gba|gba_visual|pgo|match
#include <cmath>
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
template <class T>
static void wr(const std::string& dir, const char* name, const std::vector<T>& v) {
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
  if (argc < 3) return 2;
  const std::string dir = argv[1], mode = argv[2];
  covins_b200::Context ctx(0);
  if (mode == "match") {
    auto q = rd<uint8_t>(dir, "q"); auto t = rd<uint8_t>(dir, "t"); auto seg = rd<int32_t>(dir, "seg");
    const int n_seg = (int)seg.size() - 1, nq = (int)q.size() / 32;
    std::vector<const uint8_t*> desc; std::vector<int> rows; std::vector<bool> same;
    for (int s = 0; s < n_seg; s++) { desc.push_back(t.data() + (size_t)seg[s] * 32); rows.push_back(seg[s + 1] - seg[s]); same.push_back(s % 2 == 0); }
    covins_b200::OptParams P;
    std::vector<bool> disc;
    auto all = covins_b200::MatchCandidatesORB(ctx, q.data(), nq, desc, rows, same, P, &disc);
    std::vector<int32_t> out;
    for (int s = 0; s < n_seg; s++) {
      out.push_back((int32_t)all[s].size()); out.push_back(disc[s] ? 1 : 0);
      for (auto& m : all[s]) { out.push_back((int32_t)m.idxA); out.push_back((int32_t)m.idxB); out.push_back((int32_t)m.distance); }
    }
    wr(dir, "match_out", out);
    // resident-map database: append the candidates one by one, match the same query against all of them
    covins_b200::DescriptorDatabase db(ctx);
    for (int s = 0; s < n_seg; s++)
      if (db.AddKeyframe(desc[s], rows[s]) != s) return 3;
    auto all_db = db.MatchAll(q.data(), nq, P);
    std::vector<int32_t> out_db;
    for (int s = 0; s < n_seg; s++) {
      out_db.push_back((int32_t)all_db[s].size());
      for (auto& m : all_db[s]) { out_db.push_back((int32_t)m.idxA); out_db.push_back((int32_t)m.idxB); out_db.push_back((int32_t)m.distance); }
    }
    wr(dir, "match_db_out", out_db);
    // Landmark::ComputeDescriptor batched: every candidate segment plays the observers of one landmark (first 9 rows)
    std::vector<std::vector<const uint8_t*>> cand(n_seg);
    for (int s = 0; s < n_seg; s++)
      for (int j = 0; j < std::min(rows[s], 9); j++) cand[s].push_back(desc[s] + (size_t)j * 32);
    std::vector<uint8_t> od((size_t)n_seg * 32, 0xAB);
    auto best = covins_b200::ComputeLandmarkDescriptors(ctx, cand, od.data());
    std::vector<int32_t> out_lm(best.begin(), best.end());
    for (auto b : od) out_lm.push_back((int32_t)b);
    wr(dir, "lmdesc_out", out_lm);
    return 0;
  }
  if (mode == "relpose") {
    // Optimization::OptimizeRelativePose through the reference-shaped wrapper: two mock keyframes whose landmarks are the
    // dumped camera-frame points (identity poses / extrinsics: TcwA = TcwB = I, so pA_c = the world positions)
    auto pA = rd<double>(dir, "pA_c"); auto pB = rd<double>(dir, "pB_c"); auto kA = rd<float>(dir, "kpA"); auto kB = rd<float>(dir, "kpB");
    auto sA = rd<double>(dir, "sigmaA"); auto sB = rd<double>(dir, "sigmaB"); auto t12 = rd<double>(dir, "T12"); auto intr = rd<double>(dir, "intr"); auto dist = rd<double>(dir, "dist");
    const size_t n = sA.size();
    auto k1 = std::make_shared<Keyframe>(), k2 = std::make_shared<Keyframe>();
    for (int c = 0; c < 4; c++) { k1->intr[c] = k2->intr[c] = intr[c]; k1->dist[c] = k2->dist[c] = dist[c]; }
    std::vector<LandmarkPtr> matches1(n + 3);   // three trailing keypoints without a match
    for (size_t i = 0; i < n + 3; i++) {
      k1->keypoints_distorted_.push_back({i < n ? kA[2 * i] : 0.f, i < n ? kA[2 * i + 1] : 0.f});
      k1->keypoints_aors_.push_back({0.f, i < n ? (float)(sA[i] / 2.0 - 1.0) : 0.f, 0.f, 0.f});
      auto la = std::make_shared<Landmark>();
      if (i < n) la->pos_w_ = {pA[3 * i], pA[3 * i + 1], pA[3 * i + 2]};
      k1->landmarks_.push_back(la);
      if (i >= n) continue;
      k2->keypoints_distorted_.push_back({kB[2 * i], kB[2 * i + 1]});
      k2->keypoints_aors_.push_back({0.f, (float)(sB[i] / 2.0 - 1.0), 0.f, 0.f});
      auto lb = std::make_shared<Landmark>();
      lb->pos_w_ = {pB[3 * i], pB[3 * i + 1], pB[3 * i + 2]};
      lb->observations_[k2] = i;
      k2->landmarks_.push_back(lb);
      matches1[i] = lb;
    }
    Transform T12 = pose7_to_T(t12.data());
    covins_b200::OptParams P;
    P.th_outlier_align = rd<double>(dir, "th")[0];
    const int ninl = covins_b200::OptimizeRelativePose(ctx, k1, k2, matches1, T12, 4.0, P);
    std::vector<double> out(8 + n + 3);
    covins_b200::detail::transform_to_pose7(T12, out.data());
    out[7] = ninl;
    for (size_t i = 0; i < n + 3; i++) out[8 + i] = matches1[i] ? 1.0 : 0.0;
    wr(dir, "relpose_out", out);
    return 0;
  }
  if (mode == "search") {
    // FeatureMatcher::SearchBySE3 through the reference-shaped wrapper on two mock keyframes built from dumped arrays,
    // and the DenseMatcher-shaped adaptor on a MatchingAlgorithm-style policy object
    auto mk = [&](const char* pre) {
      auto kf = std::make_shared<Keyframe>();
      auto kp = rd<float>(dir, (std::string(pre) + "_kp").c_str()); auto oc = rd<float>(dir, (std::string(pre) + "_octave").c_str());
      auto de = rd<uint8_t>(dir, (std::string(pre) + "_desc").c_str()); auto lv = rd<uint8_t>(dir, (std::string(pre) + "_lm_valid").c_str());
      auto lp = rd<double>(dir, (std::string(pre) + "_lm_pos").c_str()); auto lm = rd<double>(dir, (std::string(pre) + "_lm_maxdist").c_str());
      auto ld = rd<uint8_t>(dir, (std::string(pre) + "_lm_desc").c_str()); auto K = rd<double>(dir, (std::string(pre) + "_K").c_str());
      auto T = rd<double>(dir, (std::string(pre) + "_Tcw").c_str());
      const size_t n = oc.size();
      for (size_t i = 0; i < n; i++) {
        kf->keypoints_distorted_.push_back({kp[2 * i], kp[2 * i + 1]});
        kf->keypoints_aors_.push_back({0.f, oc[i], 0.f, 0.f});
        std::array<unsigned char, 32> d; std::copy(de.begin() + 32 * i, de.begin() + 32 * i + 32, d.begin());
        kf->descriptors_.push_back(d);
        LandmarkPtr p;
        if (lv[i]) {
          p = std::make_shared<Landmark>();
          p->pos_w_ = {lp[3 * i], lp[3 * i + 1], lp[3 * i + 2]}; p->max_distance_ = lm[i];
          std::copy(ld.begin() + 32 * i, ld.begin() + 32 * i + 32, p->descriptor_.begin());
        }
        kf->landmarks_.push_back(p);
      }
      for (int i = 0; i < 9; i++) kf->K_[i] = K[i];
      for (int i = 0; i < 16; i++) kf->T_c_w_.m[i] = T[i];
      return kf;
    };
    auto k1 = mk("k1"), k2 = mk("k2");
    for (size_t i = 0; i < k2->landmarks_.size(); i++) if (k2->landmarks_[i]) k2->landmarks_[i]->observations_[k2] = i;
    auto t12 = rd<double>(dir, "T12"), t21 = rd<double>(dir, "T21");
    Transform T12, T21; for (int i = 0; i < 16; i++) { T12.m[i] = t12[i]; T21.m[i] = t21[i]; }
    std::vector<std::vector<LandmarkPtr>> m12(1, std::vector<LandmarkPtr>(k1->landmarks_.size()));
    auto found = covins_b200::SearchBySE3(ctx, k1, std::vector<KeyframePtr>{k2}, m12, std::vector<Transform>{T12}, std::vector<Transform>{T21}, 9.5, 50, 1, 2.0);
    std::vector<int32_t> out; out.push_back(found[0]);
    for (size_t i = 0; i < m12[0].size(); i++) out.push_back(m12[0][i] ? m12[0][i]->GetFeatureIndex(k2) : -1);
    wr(dir, "search_out", out);
    // DenseMatcher-shaped adaptor with a policy object that has the MatchingAlgorithm interface + the two descriptor accessors
    struct Algo {
      KeyframePtr a, b; std::vector<int32_t> res;
      void doSetup() {}
      size_t sizeA() const { return a->descriptors_.size(); }
      size_t sizeB() const { return b->descriptors_.size(); }
      bool skipA(size_t i) const { return !a->landmarks_[i] || a->landmarks_[i]->IsInvalid(); }   // LandmarkMatchingAlgorithm.cpp:76-84
      bool skipB(size_t i) const { return !b->landmarks_[i] || b->landmarks_[i]->IsInvalid(); }
      float distanceThreshold() const { return 50.0f; }
      const unsigned char* descriptorA(size_t i) const { return a->GetDescriptor(i); }
      const unsigned char* descriptorB(size_t i) const { return b->GetDescriptor(i); }
      void reserveMatches(size_t) {}
      void setBestMatch(size_t ia, size_t ib, double d) { res.push_back((int32_t)ia); res.push_back((int32_t)ib); res.push_back((int32_t)d); }
    } algo{k1, k2, {}};
    covins_b200::DenseMatcher dm(ctx, 8);
    dm.match<Algo>(algo);
    wr(dir, "dense_out", algo.res);
    return 0;
  }
  // ---- build the mock map from the flat arrays ----
  auto pose = rd<double>(dir, "pose"); auto sb = rd<double>(dir, "speedbias"); auto extr = rd<double>(dir, "extr");
  auto intr = rd<double>(dir, "intr"); auto dist = rd<double>(dir, "dist"); auto lm = rd<double>(dir, "lm");
  auto ptr = rd<int32_t>(dir, "lm_obs_ptr"); auto okf = rd<int32_t>(dir, "obs_kf"); auto uv = rd<float>(dir, "obs_uv");
  auto sig = rd<double>(dir, "obs_sigma"); auto agent = rd<int32_t>(dir, "agent_of"); auto kfid = rd<int32_t>(dir, "kf_id");
  auto imu_j = rd<int32_t>(dir, "imu_j"); auto imu_ptr = rd<int32_t>(dir, "imu_ptr"); auto imu_dt = rd<double>(dir, "imu_dt");
  auto imu_acc = rd<double>(dir, "imu_acc"); auto imu_gyr = rd<double>(dir, "imu_gyr"); auto a0 = rd<double>(dir, "imu_acc0");
  auto g0 = rd<double>(dir, "imu_gyr0"); auto noise = rd<double>(dir, "imu_noise");
  auto li = rd<int32_t>(dir, "loop_i"); auto lj = rd<int32_t>(dir, "loop_j"); auto lq = rd<double>(dir, "loop_q"); auto lt = rd<double>(dir, "loop_t");
  auto cam_of_kf = rd<int32_t>(dir, "cam_of_kf");   // one calibration per keyframe's camera (all camera 0 when absent)
  const int K = (int)pose.size() / 7, L = (int)lm.size() / 3;
  auto map = std::make_shared<Map>();
  map->id_map_ = 0;
  std::vector<KeyframePtr> kfs(K);
  for (int k = 0; k < K; k++) {
    const int cam = cam_of_kf.empty() ? 0 : cam_of_kf[k];
    auto kf = std::make_shared<Keyframe>();
    kf->id_ = {(size_t)kfid[k], (size_t)agent[k]};
    kf->T_w_s_ = pose7_to_T(&pose[7 * k]);
    kf->T_w_s_vio_ = kf->T_w_s_;
    kf->T_s_c_ = pose7_to_T(&extr[7 * cam]);
    for (int c = 0; c < 3; c++) { kf->velocity_[c] = sb[9 * k + c]; kf->bias_accel_[c] = sb[9 * k + 3 + c]; kf->bias_gyro_[c] = sb[9 * k + 6 + c]; }
    for (int c = 0; c < 4; c++) { kf->intr[c] = intr[4 * cam + c]; kf->dist[c] = dist[4 * cam + c]; }
    if (k > 0 && agent[k - 1] == agent[k]) { kf->pred = kfs[k - 1]; kfs[k - 1]->succ = kf; }
    kfs[k] = kf;
  }
  // canonical keyframe order of the flat problem is (agent, kf id); the map orders by idpair (kf id, client id), so the
  // shim's canonical index differs from the flat one — results are compared per id.
  for (auto& kf : kfs) map->keyframes_[kf->id_] = kf;
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
      kf->keypoints_aors_.push_back({0.f, (float)(sig[o] / 2.0 - 1.0), 0.f, 0.f});   // sigma = (octave+1)*2
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
  if (mode == "gba") covins_b200::GlobalBundleAdjustment(ctx, map, 4, -1.0, false, true, false, P);
  else if (mode == "gba_visual") covins_b200::GlobalBundleAdjustment(ctx, map, 4, -1.0, true, true, false, P);
  else if (mode == "pgo") {
    P.placerec_type_covins = true;
    std::map<idpair, Transform> corrected;
    covins_b200::PoseGraphOptimization(ctx, map, corrected, P);
  } else return 2;
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
  wr(dir, "out_pose", o_pose); wr(dir, "out_sb", o_sb); wr(dir, "out_lm", o_lm); wr(dir, "out_nobs", n_obs_left);
  std::printf("shim_test %s: K=%d L=%d clean=%d\n", mode.c_str(), K, L, map->n_clean);
  return 0;
}
