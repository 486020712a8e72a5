// covins_b200::MergeMaps on mock containers (tests/test_map_merge.py).
//   shim_merge_test <dir>
// reads <dir>/T.bin (double [16], T_wtarget_wtofuse row-major), pose.bin (double [K][16] T_ws row-major), vel.bin (double
// [K][3]), kf_agent.bin (int32 [K]: 0 = the target map, 1 = the fused map), kf_inv.bin (uint8 [K]), lm.bin (double [L][3]),
// lm_agent.bin (int32 [L]), lm_inv.bin (uint8 [L]), ptr.bin (int32 [L+1]) and kf.bin (int32 [n_obs]: each landmark's
// observers by keyframe number), desc.bin (uint8 [rows][32], every keyframe's ORB rows in keyframe order), rpk.bin (int32
// [K], rows per keyframe) and q.bin (uint8 [nq][32], a query keyframe).  Keyframe k has id (k, agent) and landmark l id
// (l, agent), so both canonical orders of the merged map are the numbering.  Each map gets one loop constraint (its first
// and last keyframe).  The target's keyframes go to one ORB database, the fused map's to another; MergeMaps joins them.
// Writes out_pose.bin / out_vel.bin / out_lm.bin (every keyframe's and landmark's state afterwards, by number), out_log.bin
// (int32 [n][2], every setter call in call order, see mock_merge::CallLog), out_cnt.bin / out_kf.bin / out_w.bin (what every
// keyframe's SetCovisibility received, by number; empty for one that received nothing) and out_sizes.bin (int32: the
// merged map's keyframes, landmarks and loop constraints, then both databases' sizes).
// Exit code 2: an input is missing (refused before any GPU work); 6: the merged database's MatchAll differs from that of a
// database that received the same keyframes from the host.
#include <cstdint>
#include <fstream>
#include <string>
#include <vector>

#include "../../covins_b200/csrc/host/covins_b200_shim.hpp"
#include "mock_merge_containers.hpp"

using namespace mock_merge;

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
  if (argc != 2) return 2;
  const std::string dir = argv[1];
  std::vector<double> T, pose, vel, lm;
  std::vector<int32_t> kf_agent, lm_agent, ptr, kf, rpk;
  std::vector<uint8_t> kf_inv, lm_inv, desc, q;
  if (!rd(dir, "T", T) || !rd(dir, "pose", pose) || !rd(dir, "vel", vel) || !rd(dir, "kf_agent", kf_agent) || !rd(dir, "kf_inv", kf_inv) ||
      !rd(dir, "lm", lm) || !rd(dir, "lm_agent", lm_agent) || !rd(dir, "lm_inv", lm_inv) || !rd(dir, "ptr", ptr) || !rd(dir, "kf", kf) ||
      !rd(dir, "desc", desc) || !rd(dir, "rpk", rpk) || !rd(dir, "q", q))
    return 2;
  const size_t K = kf_agent.size(), L = lm_agent.size();
  if (T.size() != 16 || pose.size() != 16 * K || vel.size() != 3 * K || kf_inv.size() != K || lm.size() != 3 * L || lm_inv.size() != L ||
      ptr.size() != L + 1 || rpk.size() != K)
    return 2;
  CallLog log;
  auto maps = std::vector<std::shared_ptr<Map>>{std::make_shared<Map>(), std::make_shared<Map>()};
  std::vector<KeyframePtr> kfs;
  for (size_t k = 0; k < K; k++) {
    auto p = std::make_shared<Keyframe>();
    p->id_ = {k, (size_t)kf_agent[k]};
    p->number = (int)k;
    p->invalid = kf_inv[k] != 0;
    p->log = &log;
    for (int i = 0; i < 16; i++) p->T_w_s_.m[i] = pose[16 * k + i];
    for (int i = 0; i < 3; i++) p->velocity_[i] = vel[3 * k + i];
    maps[kf_agent[k]]->keyframes_[p->id_] = p;
    kfs.push_back(p);
  }
  for (auto& m : maps) {
    const auto v = m->GetKeyframesVec();
    if (!v.empty()) m->loop_constraints_.push_back({v.front(), v.back()});
  }
  for (size_t l = 0; l < L; l++) {
    auto p = std::make_shared<Landmark>();
    p->id_ = {l, (size_t)lm_agent[l]};
    p->number = (int)l;
    p->invalid = lm_inv[l] != 0;
    p->log = &log;
    p->pos_w_ = {lm[3 * l], lm[3 * l + 1], lm[3 * l + 2]};
    for (int o = ptr[l]; o < ptr[l + 1]; o++) p->AddObservation(kfs[kf[o]], (size_t)o);
    maps[lm_agent[l]]->landmarks_[p->id_] = p;
  }
  covins_b200::Context ctx(0);
  covins_b200::DescriptorDatabase db_target(ctx), db_tofuse(ctx), db_ref(ctx);
  std::vector<size_t> first(K + 1, 0);
  for (size_t k = 0; k < K; k++) first[k + 1] = first[k] + (size_t)rpk[k];
  for (int a = 0; a < 2; a++)
    for (size_t k = 0; k < K; k++)
      if (kf_agent[k] == a) {
        (a == 0 ? db_target : db_tofuse).AddKeyframe(desc.data() + 32 * first[k], rpk[k]);
        db_ref.AddKeyframe(desc.data() + 32 * first[k], rpk[k]);
      }
  Transform Tm;
  for (int i = 0; i < 16; i++) Tm.m[i] = T[i];
  covins_b200::MergeMaps(ctx, maps[0], maps[1], Tm, &db_target, &db_tofuse);

  covins_b200::OptParams P;
  const auto got = db_target.MatchAll(q.data(), (int)(q.size() / 32), P), ref = db_ref.MatchAll(q.data(), (int)(q.size() / 32), P);
  if (got.size() != ref.size()) return 6;
  for (size_t s = 0; s < got.size(); s++) {
    if (got[s].size() != ref[s].size()) return 6;
    for (size_t i = 0; i < got[s].size(); i++)
      if (got[s][i].idxA != ref[s][i].idxA || got[s][i].idxB != ref[s][i].idxB || got[s][i].distance != ref[s][i].distance) return 6;
  }

  std::vector<double> out_pose, out_vel, out_lm;
  std::vector<int32_t> out_log, cnt, out_kf, out_w;
  for (auto& p : kfs) {
    out_pose.insert(out_pose.end(), p->T_w_s_.m, p->T_w_s_.m + 16);
    out_vel.insert(out_vel.end(), p->velocity_.begin(), p->velocity_.end());
    if (p->connected_kfs_.size() != p->connected_n_.size()) return 5;
    cnt.push_back((int32_t)p->connected_kfs_.size());
    for (auto& c : p->connected_kfs_) out_kf.push_back((int32_t)c->number);
    out_w.insert(out_w.end(), p->connected_n_.begin(), p->connected_n_.end());
  }
  std::vector<LandmarkPtr> lms(L);
  for (auto& m : maps)
    for (auto& p : m->landmarks_) lms[p.second->number] = p.second;
  for (auto& p : lms) out_lm.insert(out_lm.end(), p->pos_w_.begin(), p->pos_w_.end());
  for (auto& c : log) out_log.insert(out_log.end(), c.begin(), c.end());
  const std::vector<int32_t> sizes{(int32_t)maps[0]->keyframes_.size(), (int32_t)maps[0]->landmarks_.size(), (int32_t)maps[0]->loop_constraints_.size(),
                                   db_target.size(), db_tofuse.size()};
  wr(dir, "out_pose", out_pose); wr(dir, "out_vel", out_vel); wr(dir, "out_lm", out_lm); wr(dir, "out_log", out_log);
  wr(dir, "out_cnt", cnt); wr(dir, "out_kf", out_kf); wr(dir, "out_w", out_w); wr(dir, "out_sizes", sizes);
  return 0;
}
