// covins_b200::PruneRedundantKeyframes on mock containers (tests/test_prune.py).
//   shim_prune_test <dir> <th_red> <max_time_dist> <th_obs>
// reads <dir>/ptr.bin (int32 [L+1]), kf.bin (int32 [n_obs]: the observers by keyframe number), oct.bin (int32 [n_obs]: the
// octaves), agent.bin / kfid.bin (int32 [K]: each keyframe's agent and its id within the agent; keyframe (a, i) follows
// (a, i-1) in its chain), time.bin (double [K]) and loops.bin (int32 pairs of keyframe numbers a loop constraint joins).
// Builds the map, makes the call, and writes out_invalidated.bin (the keyframe numbers SetInvalid was called on, in call
// order) and what every keyframe's SetCovisibility received afterwards: out_cnt.bin (int32 [K], list lengths),
// out_kf.bin (the connected keyframes' numbers, list after list) and out_w.bin (their weights).
// Exit code 2: an input is missing (refused before any GPU work).
#include <cstdint>
#include <fstream>
#include <string>
#include <vector>

#include "../../covins_b200/csrc/host/covins_b200_shim.hpp"
#include "mock_prune_containers.hpp"

using namespace mock_prune;

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
  std::vector<int32_t> ptr, kf, oct, agent, kfid, loops;
  std::vector<double> time;
  if (!rd(dir, "ptr", ptr) || !rd(dir, "kf", kf) || !rd(dir, "oct", oct) || !rd(dir, "agent", agent) || !rd(dir, "kfid", kfid) ||
      !rd(dir, "time", time) || !rd(dir, "loops", loops) || ptr.empty() || oct.size() != kf.size() || kfid.size() != agent.size() ||
      time.size() != agent.size())
    return 2;
  auto map = std::make_shared<Map>();
  std::vector<KeyframePtr> kfs;
  std::vector<int> invalidated;
  std::map<std::pair<int, int>, KeyframePtr> by_id;
  for (size_t k = 0; k < agent.size(); k++) {
    auto p = std::make_shared<Keyframe>();
    p->id_ = {(size_t)kfid[k], (size_t)agent[k]};
    p->number = (int)k;
    p->timestamp_ = time[k];
    p->invalidated = &invalidated;
    map->keyframes_[p->id_] = p;
    kfs.push_back(p);
    by_id[{agent[k], kfid[k]}] = p;
  }
  for (auto& p : kfs) {
    auto it = by_id.find({(int)p->id_.second, (int)p->id_.first - 1});
    if (it != by_id.end()) {
      p->pred = it->second;
      it->second->succ = p;
    }
  }
  for (size_t l = 0; l + 1 < ptr.size(); l++) {
    auto p = std::make_shared<Landmark>();
    p->id_ = {l, 0};
    for (int o = ptr[l]; o < ptr[l + 1]; o++) {
      auto& k = kfs[kf[o]];
      k->keypoints_aors_.push_back({0.f, (float)oct[o], 0.f, 0.f});
      p->AddObservation(k, k->keypoints_aors_.size() - 1);
    }
    map->landmarks_[p->id_] = p;
  }
  for (size_t i = 0; i + 1 < loops.size(); i += 2) map->loops_.push_back({kfs[loops[i]], kfs[loops[i + 1]]});
  covins_b200::Context ctx(0);
  covins_b200::PruneRedundantKeyframes(ctx, map, std::atof(argv[2]), std::atof(argv[3]), std::atoi(argv[4]));
  std::vector<int32_t> cnt, out_kf, out_w, inv(invalidated.begin(), invalidated.end());
  for (auto& p : kfs) {
    if (p->connected_kfs_.size() != p->connected_n_.size()) return 5;
    cnt.push_back((int32_t)p->connected_kfs_.size());
    for (auto& c : p->connected_kfs_) out_kf.push_back((int32_t)c->number);
    out_w.insert(out_w.end(), p->connected_n_.begin(), p->connected_n_.end());
  }
  wr(dir, "out_invalidated", inv); wr(dir, "out_cnt", cnt); wr(dir, "out_kf", out_kf); wr(dir, "out_w", out_w);
  return 0;
}
