// Stand-ins for the reference containers with exactly the members covins_b200::UpdateCovisibilityConnections touches
// (Map::GetKeyframesVec / GetLandmarksVec, Keyframe / Landmark::IsInvalid, Landmark::GetObservations) and the one member it
// needs added to the reference's Keyframe: SetCovisibility, which fills connected_kfs_ / connected_n_ (keyframe_be.hpp; the
// setter a maintainer adds is shown in INTEGRATION.md §3.5).  Field names follow mock_containers.hpp.
#pragma once
#include <cstddef>
#include <map>
#include <memory>
#include <utility>
#include <vector>

namespace mock_covis {

using idpair = std::pair<size_t, size_t>;
struct Keyframe;
struct Landmark;
using KeyframePtr = std::shared_ptr<Keyframe>;
using LandmarkPtr = std::shared_ptr<Landmark>;

struct Keyframe {
  idpair id_;
  bool invalid = false;
  std::vector<KeyframePtr> connected_kfs_;   // ordered by weight: GetConnectedKeyframes order
  std::vector<int> connected_n_;
  bool IsInvalid() const { return invalid; }
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

struct Map {
  std::map<idpair, KeyframePtr> keyframes_;
  std::map<idpair, LandmarkPtr> landmarks_;
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
};

}  // namespace mock_covis
