// ba_group.cuh — the in-process rank group of cvb_group_create (ba_group.cu), as the BA engine's group drivers use it.
// Not part of the public boundary.
#pragma once
#include <condition_variable>
#include <functional>
#include <mutex>
#include <string>

#include "cvb_internal.cuh"

constexpr int CVB_GROUP_MAX = 16;   // the peer path's limit (cvb_chol::DistView)

struct cvb_group;
namespace cvb_grp {
struct Binding {      // the `user` argument of the group all-reduce for one rank
  cvb_group* g;
  int rank;
};
}  // namespace cvb_grp

struct cvb_group {
  int n = 0;
  cvb_ctx* ctx[CVB_GROUP_MAX] = {};
  cvb_grp::Binding bind[CVB_GROUP_MAX];
  double* scratch[CVB_GROUP_MAX] = {};        // rank-local sum of one chunk (cudaMalloc on the rank's device)
  cudaEvent_t ev[CVB_GROUP_MAX][2] = {};      // per rank, by rendezvous parity
  // one rendezvous: what each rank publishes before it arrives, double-buffered by rendezvous parity (a rank may publish
  // for rendezvous k+1 while a slower peer still reads what was published for k)
  struct Slot {
    const void* p[3];
    size_t count;
  } slot[2][CVB_GROUP_MAX];
  long step[CVB_GROUP_MAX] = {};              // rendezvous count of each rank in the current call
  std::recursive_mutex call_mtx;   // one group call at a time: held by the drivers for the whole call and by cvb_grp::run
  // host barrier
  std::mutex mtx;
  std::condition_variable cv;
  int arrived = 0;
  long gen = 0;
  bool failed = false;
  int fail_rank = -1, fail_code = CVB_OK;
  std::string fail_msg;
};

namespace cvb_grp {
// cvb_allreduce_fn of the group: in-place sum of `count` doubles over the ranks, in rank order, on `stream`; user = Binding*
int allreduce(void* user, void* ptr, size_t count, void* stream);
// rendezvous of all ranks that gathers k pointers per rank: all[q * k + i] = mine[i] of rank q
int exchange(cvb_group* g, int rank, const void* const* mine, int k, const void** all);
// marks the group failed (the first failure's rank, code and message are kept) and wakes every waiting rank
void fail(cvb_group* g, int rank, int code, const std::string& msg);
// runs fn(rank) on one host thread per rank and joins them; a non-zero return marks the group failed.  Returns the first
// failure's code, with "rank r: <message>" on rank 0's context, or CVB_OK.
int run(cvb_group* g, const std::function<int(int)>& fn);
}  // namespace cvb_grp
