// ba_group.cu — in-process rank group: several contexts (GPUs, or ranks sharing one GPU) of one process driven as the ranks
// of one sharded bundle adjustment, with a peer-memory all-reduce in place of a cross-process collective.
//
// All-reduce of one call, per rank r (host thread r, its stream st_r):
//   rendezvous 1   r publishes its buffer, records an event after the work that produced it and waits (host) for all ranks;
//                  st_r then waits on every peer's event
//   per chunk      group_sum_kernel reads the chunk of every rank's buffer (same device, or over peer access) and adds them
//                  in rank order 0..n-1 into r's scratch; rendezvous 2 (event + host barrier + stream waits) guarantees that
//                  no peer still reads r's chunk when st_r copies the scratch back over it
// The host never waits on the device: the rendezvous only order the ranks' streams.  Every rank computes the same
// additions in the same order, so all ranks hold bit-identical sums, the same from run to run.
#include <algorithm>
#include <chrono>
#include <thread>
#include <vector>

#include "ba_group.cuh"

namespace {

constexpr int kRendezvousSeconds = 20;   // the bound of the distributed factorisation's peer-flag wait (cholesky.cu)

struct SumPtrs {
  const double* p[CVB_GROUP_MAX];
};

// out[i] = ((b0[i] + b1[i]) + b2[i]) + ... : plain adds in rank order (no FMA can contract them).  __grid_constant__: the
// pointer table is indexed in place in the parameter bank, not copied to a local-memory stack frame
__global__ void __launch_bounds__(256) group_sum_kernel(const __grid_constant__ SumPtrs b, int n, size_t len, double* __restrict__ out) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) {
    double s = b.p[0][i];
    for (int q = 1; q < n; q++) s += b.p[q][i];
    out[i] = s;
  }
}

void fail_locked(cvb_group* g, int rank, int code, const std::string& msg) {
  if (!g->failed) {
    g->failed = true;
    g->fail_rank = rank;
    g->fail_code = code;
    g->fail_msg = msg;
  }
  g->cv.notify_all();
}

// host barrier of the n rank threads, bounded: a rank that does not arrive within kRendezvousSeconds fails the group
int arrive(cvb_group* g, int rank) {
  std::unique_lock<std::mutex> lk(g->mtx);
  if (g->failed) return CVB_ERR_CUDA;
  const long my = g->gen;
  if (++g->arrived == g->n) {
    g->arrived = 0;
    g->gen++;
    g->cv.notify_all();
    return CVB_OK;
  }
  g->cv.wait_for(lk, std::chrono::seconds(kRendezvousSeconds), [&] { return g->gen != my || g->failed; });
  if (g->gen != my) return CVB_OK;
  fail_locked(g, rank, CVB_ERR_CUDA, "group rendezvous timed out after 20 s (a rank did not arrive)");
  return CVB_ERR_CUDA;
}

// publish `mine`, record this rank's event of the rendezvous on st (nullptr: host-only), arrive; then st waits on every
// peer's event.  *par = the slot parity the peers' publications are in.
int rendezvous(cvb_group* g, int r, cudaStream_t st, const cvb_group::Slot& mine, int* par) {
  const int p = (int)(g->step[r]++ & 1);
  g->slot[p][r] = mine;
  if (st) {
    const cudaError_t e = cudaEventRecord(g->ev[r][p], st);
    if (e != cudaSuccess) {
      cvb_grp::fail(g, r, CVB_ERR_CUDA, std::string("cudaEventRecord failed: ") + cudaGetErrorString(e));
      return CVB_ERR_CUDA;
    }
  }
  int rc = arrive(g, r);
  if (rc) return rc;
  if (st)
    for (int q = 0; q < g->n; q++) {
      if (q == r) continue;
      const cudaError_t e = cudaStreamWaitEvent(st, g->ev[q][p], 0);
      if (e != cudaSuccess) {
        cvb_grp::fail(g, r, CVB_ERR_CUDA, std::string("cudaStreamWaitEvent failed: ") + cudaGetErrorString(e));
        return CVB_ERR_CUDA;
      }
    }
  *par = p;
  return CVB_OK;
}

}  // namespace

namespace cvb_grp {

void fail(cvb_group* g, int rank, int code, const std::string& msg) {
  std::lock_guard<std::mutex> lk(g->mtx);
  fail_locked(g, rank, code, msg);
}

int allreduce(void* user, void* ptr, size_t count, void* stream) {
  const Binding* b = (const Binding*)user;
  cvb_group* g = b->g;
  const int r = b->rank, n = g->n;
  cudaStream_t st = (cudaStream_t)stream;
  int par = 0;
  int rc = rendezvous(g, r, st, cvb_group::Slot{{ptr, nullptr, nullptr}, count}, &par);
  if (rc) return rc;
  SumPtrs src{};
  for (int q = 0; q < n; q++) {
    if (g->slot[par][q].count != count) {
      fail(g, r, CVB_ERR_INVALID, "group all-reduce: the ranks passed different element counts");
      return CVB_ERR_INVALID;
    }
    src.p[q] = (const double*)g->slot[par][q].p[0];
  }
  const int blocks_max = 4 * g->ctx[r]->sm_count;
  for (size_t off = 0; off < count; off += CVB_GROUP_ALLREDUCE_CHUNK) {
    const size_t len = std::min<size_t>(CVB_GROUP_ALLREDUCE_CHUNK, count - off);
    SumPtrs c = src;
    for (int q = 0; q < n; q++) c.p[q] += off;
    const int blocks = (int)std::min<size_t>((len + 255) / 256, (size_t)blocks_max);
    group_sum_kernel<<<blocks, 256, 0, st>>>(c, n, len, g->scratch[r]);
    g->ctx[r]->launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      fail(g, r, CVB_ERR_CUDA, std::string("group_sum_kernel launch failed: ") + cudaGetErrorString(e));
      return CVB_ERR_CUDA;
    }
    if ((rc = rendezvous(g, r, st, cvb_group::Slot{{nullptr, nullptr, nullptr}, 0}, &par))) return rc;
    e = cudaMemcpyAsync((double*)ptr + off, g->scratch[r], len * sizeof(double), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) {
      fail(g, r, CVB_ERR_CUDA, std::string("all-reduce copy-back failed: ") + cudaGetErrorString(e));
      return CVB_ERR_CUDA;
    }
  }
  return CVB_OK;
}

int exchange(cvb_group* g, int rank, const void* const* mine, int k, const void** all) {
  cvb_group::Slot s{{nullptr, nullptr, nullptr}, 0};
  for (int i = 0; i < k && i < 3; i++) s.p[i] = mine[i];
  int par = 0;
  const int rc = rendezvous(g, rank, nullptr, s, &par);
  if (rc) return rc;
  for (int q = 0; q < g->n; q++)
    for (int i = 0; i < k && i < 3; i++) all[q * k + i] = g->slot[par][q].p[i];
  return CVB_OK;
}

int run(cvb_group* g, const std::function<int(int)>& fn) {
  std::lock_guard<std::recursive_mutex> call_lk(g->call_mtx);   // concurrent calls on one group would mix their rendezvous
  {
    std::lock_guard<std::mutex> lk(g->mtx);
    g->arrived = 0;
    g->failed = false;
    g->fail_rank = -1;
    g->fail_code = CVB_OK;
    g->fail_msg.clear();
  }
  for (int r = 0; r < g->n; r++) g->step[r] = 0;
  std::vector<std::thread> th;
  th.reserve(g->n);
  for (int r = 0; r < g->n; r++) {
    try {
      th.emplace_back([g, r, &fn] {
        int rc;
        try {
          rc = fn(r);
        } catch (const std::exception& e) {
          rc = cvb_fail(g->ctx[r], CVB_ERR_CUDA, "exception: %s", e.what());
        }
        if (rc) fail(g, r, rc, g->ctx[r]->err);
      });
    } catch (const std::exception& e) {   // no thread for rank r: the started ranks meet a failed group
      fail(g, r, CVB_ERR_CUDA, std::string("cannot start the rank thread: ") + e.what());
      break;
    }
  }
  for (auto& t : th) t.join();
  if (g->failed) return cvb_fail(g->ctx[0], g->fail_code, "rank %d: %s", g->fail_rank, g->fail_msg.c_str());
  return CVB_OK;
}

}  // namespace cvb_grp

extern "C" {

int cvb_group_create(cvb_ctx* const* ctxs, int n, cvb_group** out) {
  if (!out) return CVB_ERR_INVALID;
  *out = nullptr;
  cvb_ctx* c0 = ctxs && n >= 1 ? ctxs[0] : nullptr;
  if (!ctxs || n < 1 || n > CVB_GROUP_MAX) return cvb_fail(c0, CVB_ERR_INVALID, "cvb_group_create: n = %d outside 1..%d", n, CVB_GROUP_MAX);
  for (int i = 0; i < n; i++) {
    if (!ctxs[i]) return cvb_fail(c0, CVB_ERR_INVALID, "cvb_group_create: context of rank %d is NULL", i);
    for (int j = 0; j < i; j++)
      if (ctxs[j] == ctxs[i]) return cvb_fail(c0, CVB_ERR_INVALID, "cvb_group_create: ranks %d and %d are the same context", j, i);
  }
  for (int i = 0; i < n; i++)
    for (int j = 0; j < n; j++) {
      const int a = ctxs[i]->device, b = ctxs[j]->device;
      if (a == b) continue;
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, a, b) != cudaSuccess || !can)
        return cvb_fail(c0, CVB_ERR_UNSUPPORTED, "cvb_group_create: device %d (rank %d) cannot access device %d (rank %d) as a peer",
                        a, i, b, j);
    }
  int prev = 0;
  cudaGetDevice(&prev);
  cvb_group* g = new cvb_group();
  g->n = n;
  int rc = CVB_OK;
  // peer access both ways for every pair of distinct devices, and to the peers' stream-ordered pools (the engine's vectors
  // and scalars live there); both are process-wide and stay enabled after the group is destroyed
  for (int i = 0; i < n && !rc; i++)
    for (int j = 0; j < n && !rc; j++) {
      const int a = ctxs[i]->device, b = ctxs[j]->device;
      if (a == b) continue;
      cudaSetDevice(a);
      cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
      cudaMemPool_t pool;
      if (e == cudaSuccess) e = cudaDeviceGetDefaultMemPool(&pool, b);
      if (e == cudaSuccess) {
        cudaMemAccessDesc d{};
        d.location.type = cudaMemLocationTypeDevice;
        d.location.id = a;
        d.flags = cudaMemAccessFlagsProtReadWrite;
        e = cudaMemPoolSetAccess(pool, &d, 1);
      }
      if (e != cudaSuccess) rc = cvb_fail(c0, CVB_ERR_CUDA, "cvb_group_create: peer access %d -> %d: %s", a, b, cudaGetErrorString(e));
    }
  for (int r = 0; r < n && !rc; r++) {
    g->ctx[r] = ctxs[r];
    g->bind[r] = cvb_grp::Binding{g, r};
    cudaSetDevice(ctxs[r]->device);
    cudaError_t e = cudaMalloc(&g->scratch[r], sizeof(double) * CVB_GROUP_ALLREDUCE_CHUNK);
    for (int k = 0; k < 2 && e == cudaSuccess; k++) e = cudaEventCreateWithFlags(&g->ev[r][k], cudaEventDisableTiming);
    if (e != cudaSuccess) rc = cvb_fail(c0, CVB_ERR_CUDA, "cvb_group_create: rank %d: %s", r, cudaGetErrorString(e));
  }
  cudaSetDevice(prev);
  if (rc) {
    cvb_group_destroy(g);
    return rc;
  }
  *out = g;
  return CVB_OK;
}

int cvb_group_destroy(cvb_group* g) {
  if (!g) return CVB_OK;
  int prev = 0;
  cudaGetDevice(&prev);
  for (int r = 0; r < g->n; r++) {
    if (!g->ctx[r]) continue;
    cudaSetDevice(g->ctx[r]->device);
    if (g->scratch[r]) cudaFree(g->scratch[r]);
    for (auto& e : g->ev[r])
      if (e) cudaEventDestroy(e);
  }
  cudaSetDevice(prev);
  delete g;
  return CVB_OK;
}

int cvb_group_allreduce_diag(cvb_group* g, const double* in, size_t count, double* out) {
  if (!g || (count > 0 && (!in || !out))) return CVB_ERR_INVALID;
  return cvb_grp::run(g, [&](int r) {
    cvb_ctx* ctx = g->ctx[r];
    CVB_GUARD(ctx);
    cudaStream_t st = ctx->stream;
    double* d = nullptr;
    CVB_CUDA(ctx, cudaMallocAsync(&d, sizeof(double) * std::max<size_t>(count, 1), st));
    int rc = CVB_OK;
    if (count && cudaMemcpyAsync(d, in + r * count, sizeof(double) * count, cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = cvb_fail(ctx, CVB_ERR_CUDA, "upload failed");
    if (!rc && (rc = cvb_grp::allreduce(&g->bind[r], d, count, st))) cvb_fail(ctx, rc, "group all-reduce failed");
    if (!rc && count && cudaMemcpyAsync(out + r * count, d, sizeof(double) * count, cudaMemcpyDeviceToHost, st) != cudaSuccess)
      rc = cvb_fail(ctx, CVB_ERR_CUDA, "download failed");
    cudaFreeAsync(d, st);
    if (cudaStreamSynchronize(st) != cudaSuccess && !rc) rc = cvb_fail(ctx, CVB_ERR_CUDA, "stream synchronisation failed");
    return rc;
  });
}

}  // extern "C"
