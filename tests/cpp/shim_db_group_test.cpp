// covins_b200::DescriptorDatabase over a ContextGroup (covins_b200_shim.hpp) against the single-context one, ORB and SIFT, on
// mock keyframes dumped by tests/test_shim_db_group.py.
//   shim_db_group_test <dir> <group size>
//     orb_q.bin u8 [nq][32], orb_t.bin u8 [rows][32], sift_q.bin float32 [nq][128], sift_t.bin float32 [rows][128],
//     seg.bin int32 [n_kf + 1] (both maps' keyframe boundaries), thr.bin float32 [4] (ORB thr, ratio, SIFT thr, ratio)
//   → exit 0 iff MatchAll on the group database equals MatchAll on the single one (indices and distance bits), after the
//     appends and after RemoveKeyframe(1); counts.bin int32 [4]: the accepted matches of the four ORB / SIFT requests
#include <cstring>
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

static bool same(const std::vector<covins_b200::Matches>& a, const std::vector<covins_b200::Matches>& b, int32_t* count) {
  if (a.size() != b.size()) return false;
  *count = 0;
  for (size_t k = 0; k < a.size(); k++) {
    if (a[k].size() != b[k].size()) return false;
    for (size_t i = 0; i < a[k].size(); i++)
      if (a[k][i].idxA != b[k][i].idxA || a[k][i].idxB != b[k][i].idxB || std::memcmp(&a[k][i].distance, &b[k][i].distance, 4))
        return false;
    *count += (int32_t)a[k].size();
  }
  return true;
}

template <class T>
static bool run(covins_b200::DescriptorDatabase& one, covins_b200::DescriptorDatabase& grp, const std::vector<T>& q,
                const std::vector<T>& t, const std::vector<int32_t>& seg, int dim, const covins_b200::OptParams& P, int32_t* counts) {
  const int n_kf = (int)seg.size() - 1, nq = (int)(q.size() / dim);
  for (int s = 0; s < n_kf; s++) {
    const T* rows = t.data() + (size_t)seg[s] * dim;
    if (one.AddKeyframe(rows, seg[s + 1] - seg[s]) != s || grp.AddKeyframe(rows, seg[s + 1] - seg[s]) != s) return false;
  }
  if (!same(one.MatchAll(q.data(), nq, P), grp.MatchAll(q.data(), nq, P), &counts[0])) return false;
  one.RemoveKeyframe(1);
  grp.RemoveKeyframe(1);
  return same(one.MatchAll(q.data(), nq, P), grp.MatchAll(q.data(), nq, P), &counts[1]);
}

int main(int argc, char** argv) {
  if (argc != 3) return 1;
  const std::string dir = argv[1];
  const int n = std::atoi(argv[2]);
  const auto oq = rd<uint8_t>(dir, "orb_q"), ot = rd<uint8_t>(dir, "orb_t");
  const auto sq = rd<float>(dir, "sift_q"), st = rd<float>(dir, "sift_t"), thr = rd<float>(dir, "thr");
  const auto seg = rd<int32_t>(dir, "seg");
  if (seg.size() < 3 || thr.size() != 4 || n < 1) return 2;   // nothing dumped: stop before any GPU work
  covins_b200::Context ctx(0);
  covins_b200::ContextGroup group(std::vector<int>(n, 0));
  int32_t counts[4] = {};
  covins_b200::OptParams P;
  P.img_match_thres = thr[0];
  P.ratio_thres = thr[1];
  {
    covins_b200::DescriptorDatabase one(ctx), grp(group);
    if (!run(one, grp, oq, ot, seg, 32, P, counts)) return 3;
  }
  P.img_match_thres = thr[2];
  P.ratio_thres = thr[3];
  {
    covins_b200::DescriptorDatabase one(ctx, covins_b200::SiftDescriptors{}), grp(group, covins_b200::SiftDescriptors{});
    if (!run(one, grp, sq, st, seg, 128, P, counts + 2)) return 4;
  }
  std::ofstream f(dir + "/counts.bin", std::ios::binary);
  f.write(reinterpret_cast<const char*>(counts), sizeof(counts));
  return 0;
}
