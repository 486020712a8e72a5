// covins_b200::RemoveLandmarkOutliers on mock containers (tests/test_landmark_outliers.py).
//   shim_outlier_test <dir> <th_outlier> <cauchy> <min_obs>
// reads <dir>/pose.bin (double [K][7] T_ws), cam.bin (double [18]: extr T_sc [7], intr [4], dist [4], unused [3]; one camera
// for every keyframe), lm.bin (double [L][3]), ptr.bin (int32 [L+1]), kf.bin (int32 [n_obs]: the observers by keyframe
// number, ascending within a landmark), uv.bin (float [n_obs][2]) and oct.bin (float [n_obs]: the keypoint octaves).
// Keyframe k has id (k, 0) and landmark l id (l, 0), so both canonical orders are the numbering.  Observation o of
// landmark l is feature o of its keyframe.  Builds the map, makes the call, and writes out_log.bin (int32 [n][3]: every
// erasing call in call order, see mock_outlier::CallLog) and what every keyframe's SetCovisibility received afterwards:
// out_cnt.bin (int32 [K], list lengths), out_kf.bin (the connected keyframes' numbers, list after list) and out_w.bin.
// Exit code 2: an input is missing (refused before any GPU work).
#include <cstdint>
#include <fstream>
#include <string>
#include <vector>

#include "../../covins_b200/csrc/host/covins_b200_shim.hpp"
#include "mock_outlier_containers.hpp"

using namespace mock_outlier;

template <class T>
static bool rd(const std::string& dir, const char* name, std::vector<T>& v) {
  std::ifstream f(dir + "/" + name + ".bin", std::ios::binary | std::ios::ate);
  if (!f) return false;
  v.resize((size_t)f.tellg() / sizeof(T));
  f.seekg(0);
  f.read(reinterpret_cast<char*>(v.data()), v.size() * sizeof(T));
  return true;
}
template <class T>
static void wr(const std::string& dir, const char* name, const std::vector<T>& v) {
  std::ofstream f(dir + "/" + name + ".bin", std::ios::binary);
  f.write(reinterpret_cast<const char*>(v.data()), v.size() * sizeof(T));
}

int main(int argc, char** argv) {
  if (argc != 5) return 2;
  const std::string dir = argv[1];
  std::vector<double> pose, cam, lm;
  std::vector<int32_t> ptr, kf;
  std::vector<float> uv, oct;
  if (!rd(dir, "pose", pose) || !rd(dir, "cam", cam) || !rd(dir, "lm", lm) || !rd(dir, "ptr", ptr) || !rd(dir, "kf", kf) || !rd(dir, "uv", uv) ||
      !rd(dir, "oct", oct) || ptr.empty() || cam.size() != 18 || pose.size() % 7 || lm.size() != 3 * (ptr.size() - 1) ||
      uv.size() != 2 * kf.size() || oct.size() != kf.size())
    return 2;
  CallLog log;
  auto map = std::make_shared<Map>();
  map->log = &log;
  std::vector<KeyframePtr> kfs;
  for (size_t k = 0; k < pose.size() / 7; k++) {
    auto p = std::make_shared<Keyframe>();
    p->id_ = {k, 0};
    p->number = (int)k;
    p->log = &log;
    for (int i = 0; i < 7; i++) { p->pose[i] = pose[7 * k + i]; p->extr[i] = cam[i]; }
    for (int i = 0; i < 4; i++) { p->intr[i] = cam[7 + i]; p->dist[i] = cam[11 + i]; }
    map->keyframes_[p->id_] = p;
    kfs.push_back(p);
  }
  for (size_t l = 0; l + 1 < ptr.size(); l++) {
    auto p = std::make_shared<Landmark>();
    p->id_ = {l, 0};
    p->number = (int)l;
    p->log = &log;
    p->pos_w_ = {lm[3 * l], lm[3 * l + 1], lm[3 * l + 2]};
    for (int o = ptr[l]; o < ptr[l + 1]; o++) {
      auto& k = kfs[kf[o]];
      k->keypoints_distorted_.push_back({uv[2 * (size_t)o], uv[2 * (size_t)o + 1]});
      k->keypoints_aors_.push_back({0.f, oct[o], 0.f, 0.f});
      k->has_landmark.push_back(true);
      p->AddObservation(k, k->keypoints_distorted_.size() - 1);
    }
    map->landmarks_[p->id_] = p;
  }
  covins_b200::Context ctx(0);
  covins_b200::RemoveLandmarkOutliers(ctx, map, std::atof(argv[2]), std::atof(argv[3]), std::atoi(argv[4]));
  std::vector<int32_t> out_log, cnt, out_kf, out_w;
  for (auto& c : log) out_log.insert(out_log.end(), c.begin(), c.end());
  for (auto& p : kfs) {
    if (p->connected_kfs_.size() != p->connected_n_.size()) return 5;
    cnt.push_back((int32_t)p->connected_kfs_.size());
    for (auto& c : p->connected_kfs_) out_kf.push_back((int32_t)c->number);
    out_w.insert(out_w.end(), p->connected_n_.begin(), p->connected_n_.end());
  }
  wr(dir, "out_log", out_log); wr(dir, "out_cnt", cnt); wr(dir, "out_kf", out_kf); wr(dir, "out_w", out_w);
  return 0;
}
