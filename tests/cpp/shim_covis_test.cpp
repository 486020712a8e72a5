// covins_b200::UpdateCovisibilityConnections on mock containers (tests/test_covisibility.py).
//   shim_covis_test <dir> <min_weight>
// reads <dir>/ptr.bin (int32 [L+1]) and kf.bin (int32 [n_obs]): the landmarks' observers by keyframe number, and
// kf_invalid.bin (uint8 [K]) / lm_invalid.bin (uint8 [L]): the keyframes and landmarks whose IsInvalid() is true.  Builds
// the map, makes the call, and writes what every keyframe's SetCovisibility received: out_cnt.bin (int32 [K], list
// lengths), out_kf.bin (the connected keyframes' numbers, list after list) and out_w.bin (their weights).
// Exit code 2: an input is missing (refused before any GPU work).
#include <cstdint>
#include <fstream>
#include <string>
#include <vector>

#include "../../covins_b200/csrc/host/covins_b200_shim.hpp"
#include "mock_covis_containers.hpp"

using namespace mock_covis;

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
  if (argc != 3) return 2;
  const std::string dir = argv[1];
  std::vector<int32_t> ptr, kf;
  std::vector<uint8_t> kf_invalid, lm_invalid;
  if (!rd(dir, "ptr", ptr) || !rd(dir, "kf", kf) || !rd(dir, "kf_invalid", kf_invalid) || !rd(dir, "lm_invalid", lm_invalid) ||
      ptr.size() != lm_invalid.size() + 1)
    return 2;
  auto map = std::make_shared<Map>();
  std::vector<KeyframePtr> kfs;
  for (size_t k = 0; k < kf_invalid.size(); k++) {
    auto p = std::make_shared<Keyframe>();
    p->id_ = {k, 0};
    p->invalid = kf_invalid[k] != 0;
    map->keyframes_[p->id_] = p;
    kfs.push_back(p);
  }
  for (size_t l = 0; l < lm_invalid.size(); l++) {
    auto p = std::make_shared<Landmark>();
    p->id_ = {l, 0};
    p->invalid = lm_invalid[l] != 0;
    for (int o = ptr[l]; o < ptr[l + 1]; o++) p->AddObservation(kfs[kf[o]], (size_t)o);
    map->landmarks_[p->id_] = p;
  }
  covins_b200::Context ctx(0);
  covins_b200::UpdateCovisibilityConnections(ctx, map, std::atoi(argv[2]));
  std::vector<int32_t> cnt, out_kf, out_w;
  for (auto& p : kfs) {
    if (p->connected_kfs_.size() != p->connected_n_.size()) return 5;
    cnt.push_back((int32_t)p->connected_kfs_.size());
    for (auto& c : p->connected_kfs_) out_kf.push_back((int32_t)c->id_.first);
    out_w.insert(out_w.end(), p->connected_n_.begin(), p->connected_n_.end());
  }
  wr(dir, "out_cnt", cnt); wr(dir, "out_kf", out_kf); wr(dir, "out_w", out_w);
  return 0;
}
