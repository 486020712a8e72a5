// covins_b200::DescriptorDatabase::RemoveKeyframes (covins_b200_shim.hpp) against a loop of RemoveKeyframe from the highest
// index down, on a single-context database and on one over a ContextGroup, ORB and SIFT, on mock keyframes dumped by
// tests/test_shim_db_remove.py.
//   shim_db_remove_test <dir> <group size>
//     orb_q.bin u8 [nq][32], orb_t.bin u8 [rows][32], sift_q.bin float32 [nq][128], sift_t.bin float32 [rows][128],
//     seg.bin int32 [n_kf + 1] (the keyframe boundaries), rm.bin int32 [n_rm] (the indices to remove, any order),
//     thr.bin float32 [4] (ORB thr, ratio, SIFT thr, ratio)
//   → exit 0 iff, for every database form and row kind, size() and MatchAll (indices and distance bits) agree between the
//     batch and the loop after the removal, and again after one more RemoveKeyframe(0) and an AddKeyframe on both;
//     counts.bin int32 [4]: the accepted matches after the removal: single ORB, single SIFT, group ORB, group SIFT
#include <algorithm>
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
static bool run(covins_b200::DescriptorDatabase& batch, covins_b200::DescriptorDatabase& loop, const std::vector<T>& q,
                const std::vector<T>& t, const std::vector<int32_t>& seg, const std::vector<int32_t>& rm, int dim,
                const covins_b200::OptParams& P, int32_t* count) {
  const int n_kf = (int)seg.size() - 1, nq = (int)(q.size() / dim);
  for (int s = 0; s < n_kf; s++) {
    const T* rows = t.data() + (size_t)seg[s] * dim;
    if (batch.AddKeyframe(rows, seg[s + 1] - seg[s]) != s || loop.AddKeyframe(rows, seg[s + 1] - seg[s]) != s) return false;
  }
  batch.RemoveKeyframes(std::vector<int>(rm.begin(), rm.end()));
  std::vector<int> down(rm.begin(), rm.end());
  std::sort(down.rbegin(), down.rend());
  for (const int i : down) loop.RemoveKeyframe(i);
  if (batch.size() != n_kf - (int)rm.size() || loop.size() != batch.size()) return false;
  if (!same(batch.MatchAll(q.data(), nq, P), loop.MatchAll(q.data(), nq, P), count)) return false;
  batch.RemoveKeyframes({});   // nothing leaves
  batch.RemoveKeyframe(0);
  loop.RemoveKeyframe(0);
  const int last = batch.AddKeyframe(t.data(), seg[1]);
  if (loop.AddKeyframe(t.data(), seg[1]) != last || last != batch.size() - 1) return false;
  int32_t again = 0;
  return same(batch.MatchAll(q.data(), nq, P), loop.MatchAll(q.data(), nq, P), &again);
}

int main(int argc, char** argv) {
  if (argc != 3) return 1;
  const std::string dir = argv[1];
  const int n = std::atoi(argv[2]);
  const auto oq = rd<uint8_t>(dir, "orb_q"), ot = rd<uint8_t>(dir, "orb_t");
  const auto sq = rd<float>(dir, "sift_q"), st = rd<float>(dir, "sift_t"), thr = rd<float>(dir, "thr");
  const auto seg = rd<int32_t>(dir, "seg"), rm = rd<int32_t>(dir, "rm");
  if (seg.size() < 3 || rm.empty() || thr.size() != 4 || n < 1) return 2;   // nothing dumped: stop before any GPU work
  covins_b200::Context ctx(0);
  covins_b200::ContextGroup group(std::vector<int>(n, 0));
  int32_t counts[4] = {};
  covins_b200::OptParams orb, sift;
  orb.img_match_thres = thr[0];
  orb.ratio_thres = thr[1];
  sift.img_match_thres = thr[2];
  sift.ratio_thres = thr[3];
  {
    covins_b200::DescriptorDatabase batch(ctx), loop(ctx);
    if (!run(batch, loop, oq, ot, seg, rm, 32, orb, &counts[0])) return 3;
  }
  {
    covins_b200::DescriptorDatabase batch(ctx, covins_b200::SiftDescriptors{}), loop(ctx, covins_b200::SiftDescriptors{});
    if (!run(batch, loop, sq, st, seg, rm, 128, sift, &counts[1])) return 4;
  }
  {
    covins_b200::DescriptorDatabase batch(group), loop(group);
    if (!run(batch, loop, oq, ot, seg, rm, 32, orb, &counts[2])) return 5;
  }
  {
    covins_b200::DescriptorDatabase batch(group, covins_b200::SiftDescriptors{}), loop(group, covins_b200::SiftDescriptors{});
    if (!run(batch, loop, sq, st, seg, rm, 128, sift, &counts[3])) return 6;
  }
  std::ofstream f(dir + "/counts.bin", std::ios::binary);
  f.write(reinterpret_cast<const char*>(counts), sizeof(counts));
  return 0;
}
