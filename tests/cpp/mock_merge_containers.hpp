// Stand-ins for the reference containers with exactly the members covins_b200::MergeMaps touches: those of
// mock_covis_containers.hpp (it ends with UpdateCovisibilityConnections) plus Keyframe::GetPoseTws / SetPoseTws /
// GetStateVelocity / SetStateVelocity, Landmark::GetWorldPos / SetWorldPos and Map::AddKeyframe / AddLandmark /
// GetLoopConstraints / AddLoopConstraint.  Each setter appends (call, number) to one shared log, so a test sees the order
// of the write-back.
#pragma once
#include <array>
#include <cstddef>
#include <cstdint>
#include <map>
#include <memory>
#include <utility>
#include <vector>

namespace mock_merge {

struct Transform {   // Eigen::Matrix4d stand-in
  double m[16];
  double& operator()(int r, int c) { return m[4 * r + c]; }
  double operator()(int r, int c) const { return m[4 * r + c]; }
};
using Vector3 = std::array<double, 3>;
using idpair = std::pair<size_t, size_t>;
struct Keyframe;
struct Landmark;
using KeyframePtr = std::shared_ptr<Keyframe>;
using LandmarkPtr = std::shared_ptr<Landmark>;

// (0, keyframe number): SetPoseTws; (1, keyframe number): SetStateVelocity; (2, landmark number): SetWorldPos
using CallLog = std::vector<std::array<int32_t, 2>>;

struct Keyframe {
  idpair id_;
  int number = 0;
  bool invalid = false;
  Transform T_w_s_{};
  Vector3 velocity_{0, 0, 0};
  std::vector<KeyframePtr> connected_kfs_;
  std::vector<int> connected_n_;
  CallLog* log = nullptr;
  bool IsInvalid() const { return invalid; }
  Transform GetPoseTws() const { return T_w_s_; }
  void SetPoseTws(const Transform& T) { T_w_s_ = T; log->push_back({0, number}); }
  Vector3 GetStateVelocity() const { return velocity_; }
  void SetStateVelocity(const Vector3& v) { velocity_ = v; log->push_back({1, number}); }
  void SetCovisibility(std::vector<KeyframePtr> kfs, std::vector<int> weights) { connected_kfs_ = std::move(kfs); connected_n_ = std::move(weights); }
};

struct Landmark {
  idpair id_;
  int number = 0;
  bool invalid = false;
  Vector3 pos_w_{0, 0, 0};
  std::map<KeyframePtr, size_t> observations_;   // pointer-ordered like the reference (typedefs_base.hpp:187)
  CallLog* log = nullptr;
  bool IsInvalid() const { return invalid; }
  void AddObservation(const KeyframePtr& kf, size_t idx) { observations_[kf] = idx; }
  std::map<KeyframePtr, size_t> GetObservations() const { return observations_; }
  Vector3 GetWorldPos() const { return pos_w_; }
  void SetWorldPos(const Vector3& p) { pos_w_ = p; log->push_back({2, number}); }
};

struct LoopConstraint {   // typedefs_base.hpp:264-277, the two keyframes only
  KeyframePtr kf1, kf2;
};

struct Map {
  std::map<idpair, KeyframePtr> keyframes_;
  std::map<idpair, LandmarkPtr> landmarks_;
  std::vector<LoopConstraint> loop_constraints_;
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
  void AddKeyframe(const KeyframePtr& kf) { keyframes_[kf->id_] = kf; }
  void AddLandmark(const LandmarkPtr& lm) { landmarks_[lm->id_] = lm; }
  std::vector<LoopConstraint> GetLoopConstraints() const { return loop_constraints_; }
  void AddLoopConstraint(const LoopConstraint& lc) { loop_constraints_.push_back(lc); }
};

}  // namespace mock_merge
