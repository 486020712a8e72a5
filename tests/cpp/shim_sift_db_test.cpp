// The SIFT form of covins_b200::DescriptorDatabase (covins_b200_shim.hpp) on mock keyframes dumped by tests/test_shim_sift_db.py,
// next to MatchCandidatesSIFT on the same candidates.
//   shim_sift_db_test <dir>   q.bin float32 [nq][128], t.bin float32 [rows][128], seg.bin int32 [n_kf + 1], thr.bin float32 [2]
//                             → sift_all.bin (MatchCandidatesSIFT), sift_db.bin (DescriptorDatabase::MatchAll), sift_db_rm.bin
//                             (MatchAll after RemoveKeyframe(1)); each per keyframe: n, then n x (queryIdx, trainIdx, distance bits)
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
static void wr(const std::string& dir, const char* name, const std::vector<covins_b200::Matches>& all) {
  std::vector<int32_t> v;
  for (const auto& ms : all) {
    v.push_back((int32_t)ms.size());
    for (const auto& m : ms) {
      int32_t bits;
      std::memcpy(&bits, &m.distance, 4);
      v.insert(v.end(), {(int32_t)m.idxA, (int32_t)m.idxB, bits});
    }
  }
  std::ofstream f(dir + "/" + name + ".bin", std::ios::binary);
  f.write(reinterpret_cast<const char*>(v.data()), v.size() * sizeof(int32_t));
}

int main(int argc, char** argv) {
  if (argc != 2) return 1;
  const std::string dir = argv[1];
  const auto q = rd<float>(dir, "q"), t = rd<float>(dir, "t"), thr = rd<float>(dir, "thr");
  const auto seg = rd<int32_t>(dir, "seg");
  if (seg.size() < 3 || thr.size() != 2) return 2;   // nothing dumped: stop before any GPU work
  const int n_kf = (int)seg.size() - 1, nq = (int)(q.size() / 128);
  std::vector<const float*> desc;
  std::vector<int> rows;
  std::vector<bool> same(n_kf, false);
  for (int s = 0; s < n_kf; s++) { desc.push_back(t.data() + (size_t)seg[s] * 128); rows.push_back(seg[s + 1] - seg[s]); }
  covins_b200::OptParams P;
  P.img_match_thres = thr[0];
  P.ratio_thres = thr[1];
  covins_b200::Context ctx(0);
  wr(dir, "sift_all", covins_b200::MatchCandidatesSIFT(ctx, q.data(), nq, desc, rows, same, P, nullptr));
  covins_b200::DescriptorDatabase db(ctx, covins_b200::SiftDescriptors{});
  for (int s = 0; s < n_kf; s++)
    if (db.AddKeyframe(desc[s], rows[s]) != s) return 3;
  wr(dir, "sift_db", db.MatchAll(q.data(), nq, P));
  db.RemoveKeyframe(1);
  wr(dir, "sift_db_rm", db.MatchAll(q.data(), nq, P));
  return 0;
}
