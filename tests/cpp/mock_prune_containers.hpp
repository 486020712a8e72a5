// Stand-ins for the reference containers with exactly the members covins_b200::PruneRedundantKeyframes touches: those of
// mock_covis_containers.hpp (it ends with UpdateCovisibilityConnections) plus Keyframe::timestamp_, keypoints_aors_,
// GetPredecessor and SetInvalid, and Map::GetLoopConstraints.  SetInvalid does what the reference's does to the chain
// (keyframe_be.cpp:413-440: the successor takes over the predecessor) and records the order of the calls.
#pragma once
#include <array>
#include <cstddef>
#include <map>
#include <memory>
#include <utility>
#include <vector>

namespace mock_prune {

using idpair = std::pair<size_t, size_t>;
struct Keyframe;
struct Landmark;
using KeyframePtr = std::shared_ptr<Keyframe>;
using LandmarkPtr = std::shared_ptr<Landmark>;

struct Keyframe {
  idpair id_;   // (keyframe id, agent id)
  int number = 0;   // the test's keyframe number
  double timestamp_ = 0.0;
  bool invalid = false;
  std::vector<std::array<float, 4>> keypoints_aors_;   // angle, octave, response, size
  KeyframePtr pred, succ;
  std::vector<KeyframePtr> connected_kfs_;
  std::vector<int> connected_n_;
  std::vector<int>* invalidated = nullptr;   // the order of SetInvalid calls
  bool IsInvalid() const { return invalid; }
  KeyframePtr GetPredecessor() const { return pred; }
  void SetInvalid() {
    invalid = true;
    if (succ) succ->pred = pred;
    if (pred) pred->succ = succ;
    invalidated->push_back(number);
  }
  void SetCovisibility(std::vector<KeyframePtr> kfs, std::vector<int> weights) { connected_kfs_ = std::move(kfs); connected_n_ = std::move(weights); }
};

struct Landmark {
  idpair id_;
  bool invalid = false;
  std::map<KeyframePtr, size_t> observations_;   // pointer-ordered like the reference (typedefs_base.hpp:187)
  bool IsInvalid() const { return invalid; }
  void AddObservation(const KeyframePtr& kf, size_t idx) { observations_[kf] = idx; }
  std::map<KeyframePtr, size_t> GetObservations() const { return observations_; }
};

struct LoopConstraint {
  KeyframePtr kf1, kf2;
};

struct Map {
  std::map<idpair, KeyframePtr> keyframes_;
  std::map<idpair, LandmarkPtr> landmarks_;
  std::vector<LoopConstraint> loops_;
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
  std::vector<LoopConstraint> GetLoopConstraints() const { return loops_; }
};

}  // namespace mock_prune
