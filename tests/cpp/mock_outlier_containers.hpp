// Stand-ins for the reference containers with exactly the members covins_b200::RemoveLandmarkOutliers touches: those of
// mock_covis_containers.hpp (it ends with UpdateCovisibilityConnections) plus what the GBA's flatten reads of a keyframe
// (UpdateCeresFromState, GetCameraParams, keypoints_distorted_, keypoints_aors_) and of a landmark (GetWorldPos), and the
// three erasing calls: Keyframe::EraseLandmark, Landmark::EraseObservation and Map::EraseLandmark.  Each erasing call
// appends (call, a, b) to one shared log, so a test sees the order of every call.
#pragma once
#include <array>
#include <cstddef>
#include <cstdint>
#include <map>
#include <memory>
#include <utility>
#include <vector>

namespace mock_outlier {

using idpair = std::pair<size_t, size_t>;
struct Keyframe;
struct Landmark;
using KeyframePtr = std::shared_ptr<Keyframe>;
using LandmarkPtr = std::shared_ptr<Landmark>;

// (0, keyframe number, feature): Keyframe::EraseLandmark; (1, landmark number, keyframe number): Landmark::EraseObservation;
// (2, landmark number, 0): Map::EraseLandmark
using CallLog = std::vector<std::array<int32_t, 3>>;

struct Keyframe {
  idpair id_;
  int number = 0;   // the test's keyframe number
  bool invalid = false;
  double pose[7], extr[7], intr[4], dist[4];   // T_ws and T_sc as qx,qy,qz,qw,x,y,z
  std::vector<std::array<float, 2>> keypoints_distorted_;
  std::vector<std::array<float, 4>> keypoints_aors_;   // angle, octave, response, size
  std::vector<bool> has_landmark;
  std::vector<KeyframePtr> connected_kfs_;
  std::vector<int> connected_n_;
  CallLog* log = nullptr;
  bool IsInvalid() const { return invalid; }
  void UpdateCeresFromState(double* p, double* vb, double* e) const {
    for (int i = 0; i < 7; i++) { p[i] = pose[i]; e[i] = extr[i]; }
    for (int i = 0; i < 9; i++) vb[i] = 0.0;
  }
  bool GetCameraParams(double i[4], double d[4]) const {
    for (int k = 0; k < 4; k++) { i[k] = intr[k]; d[k] = dist[k]; }
    return true;
  }
  void EraseLandmark(size_t feat) {
    has_landmark[feat] = false;
    log->push_back({0, number, (int32_t)feat});
  }
  void SetCovisibility(std::vector<KeyframePtr> kfs, std::vector<int> weights) { connected_kfs_ = std::move(kfs); connected_n_ = std::move(weights); }
};

struct Landmark {
  idpair id_;
  int number = 0;
  bool invalid = false;
  std::array<double, 3> pos_w_{0, 0, 0};
  std::map<KeyframePtr, size_t> observations_;   // pointer-ordered like the reference (typedefs_base.hpp:187)
  CallLog* log = nullptr;
  bool IsInvalid() const { return invalid; }
  void AddObservation(const KeyframePtr& kf, size_t idx) { observations_[kf] = idx; }
  std::map<KeyframePtr, size_t> GetObservations() const { return observations_; }
  std::array<double, 3> GetWorldPos() const { return pos_w_; }
  void EraseObservation(const KeyframePtr& kf) {
    observations_.erase(kf);
    log->push_back({1, number, kf->number});
  }
};

struct Map {
  std::map<idpair, KeyframePtr> keyframes_;
  std::map<idpair, LandmarkPtr> landmarks_;
  CallLog* log = nullptr;
  std::vector<KeyframePtr> GetKeyframesVec() const {
    std::vector<KeyframePtr> v;
    for (auto& p : keyframes_) v.push_back(p.second);
    return v;
  }
  std::vector<LandmarkPtr> GetLandmarksVec() const {
    std::vector<LandmarkPtr> v;
    for (auto& p : landmarks_) v.push_back(p.second);
    return v;
  }
  void EraseLandmark(const LandmarkPtr& lm) {
    landmarks_.erase(lm->id_);
    log->push_back({2, lm->number, 0});
  }
};

}  // namespace mock_outlier
