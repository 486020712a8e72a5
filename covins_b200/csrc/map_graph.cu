// map_graph.cu — cvb_covisibility: the covisibility graph of a whole map in one call (include/covins_b200.h, "Map
// maintenance"; Keyframe::UpdateCovisibilityConnections, keyframe_be.cpp:559-608, for every keyframe).
//
// The graph is the sparse integer product A·Aᵀ of the 0/1 keyframe x landmark matrix, thresholded and ordered per row:
//   host    one pass over the observations validates them and keeps the participating ones of every landmark that still has
//           two observers, with the exclusive 64-bit scan of its pairs n(n-1)/2 (the pass has to read every observation
//           for the duplicate check anyway);
//   K1      mg_expand_pairs_kernel: one key (i << bits | j), i < j, per shared pair.  The work is cut by PAIR, 2048 per
//           CTA, wherever that falls inside a landmark: a landmark seen by 2 000 keyframes (2 M pairs) spreads over
//           1 000 CTAs, thirty short tracks share one;
//   cub     radix sort over the 2·bits significant bits, run-length encode → (i, j, w).  With more pairs than the budget
//           the pair range is processed in chunks and the partial (key, count) lists merged by sort + reduce-by-key;
//           integer sums, so the result does not depend on the chunking;
//   K2      mg_row_stats_kernel: per keyframe the number of neighbours reaching min_weight and the fallback argmax
//           (max weight, min index) — integer atomicAdd / atomicMax, whose results do not depend on their order;
//   K3      mg_connect_kernel: rule 3 per edge, the degree of both ends, and one sort key (row, ~weight, col) per direction;
//   cub     exclusive scan of the degrees → nbr_ptr; radix sort of the directed keys (unconnected ones sort last);
//   K4      mg_decode_kernel: sorted keys → nbr_kf / nbr_w.
// Integer arithmetic throughout: the output is bit-identical from run to run.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>

#include <cuda/std/functional>

#include <algorithm>

#include "cvb_internal.cuh"

namespace {

constexpr int MG_THREADS = 256;
constexpr int MG_TILE = 2048;                        // pairs per CTA of the expansion
constexpr int64_t MG_PAIR_BUDGET = int64_t(1) << 26;  // pairs expanded at a time: 2 x 512 MB of keys
constexpr int64_t MG_INDEX_MAX = 0x7fffffff;          // cub item counts and nbr_ptr are 32-bit

// The t-th unordered pair (a, b) of n items, by integer division only: the pairs at circular distance d = 1..h, h = (n-1)/2,
// are n each — (a, a+d mod n) — and for even n the distance n/2 adds the n/2 pairs (a, a+n/2).
__device__ __forceinline__ void mg_pair_of(int64_t t, int n, int& a, int& b) {
  const int h = (n - 1) >> 1;
  const int64_t full = (int64_t)n * h;
  if (t < full) {
    if (full <= 0x7fffffff) {
      a = (int)((uint32_t)t / (uint32_t)h);
      b = a + (int)((uint32_t)t % (uint32_t)h) + 1;
    } else {
      a = (int)(t / h);
      b = a + (int)(t % h) + 1;
    }
    if (b >= n) b -= n;
  } else {
    a = (int)(t - full);
    b = a + (n >> 1);
  }
}

// pairs [p0, p0 + count) of the compact CSR (every landmark has >= 2 observers, so >= 1 pair): keys[p - p0]
__global__ void __launch_bounds__(MG_THREADS) mg_expand_pairs_kernel(const int32_t* __restrict__ lm_ptr, const int32_t* __restrict__ kf,
                                                                     const int64_t* __restrict__ pair_off, int n_lm, int64_t p0, int64_t count,
                                                                     int bits_k, uint64_t* __restrict__ keys) {
  __shared__ int64_t s_off[MG_TILE + 1];
  __shared__ int s_l0;
  const int64_t tile0 = p0 + (int64_t)blockIdx.x * MG_TILE;
  const int tile_n = (int)min((int64_t)MG_TILE, p0 + count - tile0);
  if (threadIdx.x == 0) {   // the landmark that holds the tile's first pair: the largest l with pair_off[l] <= tile0
    int lo = 0, hi = n_lm;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (pair_off[mid] <= tile0) lo = mid; else hi = mid;
    }
    s_l0 = lo;
  }
  __syncthreads();
  const int l0 = s_l0;
  const int nl = min(n_lm - l0, tile_n);   // a landmark holds at least one pair: the tile ends within nl landmarks
  for (int i = threadIdx.x; i <= nl; i += MG_THREADS) s_off[i] = pair_off[l0 + i];
  __syncthreads();
  for (int i = threadIdx.x; i < tile_n; i += MG_THREADS) {
    const int64_t p = tile0 + i;
    int lo = 0, hi = nl;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (s_off[mid] <= p) lo = mid; else hi = mid;
    }
    const int base = lm_ptr[l0 + lo];
    int a, b;
    mg_pair_of(p - s_off[lo], lm_ptr[l0 + lo + 1] - base, a, b);
    const uint32_t ka = (uint32_t)kf[base + a], kb = (uint32_t)kf[base + b];
    keys[p - p0] = ((uint64_t)min(ka, kb) << bits_k) | max(ka, kb);
  }
}

__device__ __forceinline__ uint64_t mg_rank(int w, uint32_t col) { return ((uint64_t)(uint32_t)w << 32) | (uint32_t)~col; }

__global__ void __launch_bounds__(MG_THREADS) mg_row_stats_kernel(const uint64_t* __restrict__ edge, const int32_t* __restrict__ weight, int n_edge,
                                                                  int bits_k, int min_weight, int32_t* strong, unsigned long long* best) {
  const int e = blockIdx.x * MG_THREADS + threadIdx.x;
  if (e >= n_edge) return;
  const uint32_t i = (uint32_t)(edge[e] >> bits_k), j = (uint32_t)(edge[e] & ((1ull << bits_k) - 1));
  const int w = weight[e];
  if (w >= min_weight) {
    atomicAdd(&strong[i], 1);
    atomicAdd(&strong[j], 1);
  } else {   // a fallback target is below min_weight by definition
    atomicMax(&best[i], (unsigned long long)mg_rank(w, j));
    atomicMax(&best[j], (unsigned long long)mg_rank(w, i));
  }
}

__global__ void __launch_bounds__(MG_THREADS) mg_connect_kernel(const uint64_t* __restrict__ edge, const int32_t* __restrict__ weight, int n_edge,
                                                                int bits_k, int bits_w, int min_weight, const int32_t* __restrict__ strong,
                                                                const unsigned long long* __restrict__ best, int32_t* deg, uint64_t* __restrict__ row_key) {
  const int e = blockIdx.x * MG_THREADS + threadIdx.x;
  if (e >= n_edge) return;
  const uint32_t i = (uint32_t)(edge[e] >> bits_k), j = (uint32_t)(edge[e] & ((1ull << bits_k) - 1));
  const int w = weight[e];
  const bool connected = w >= min_weight || (strong[i] == 0 && best[i] == mg_rank(w, j)) || (strong[j] == 0 && best[j] == mg_rank(w, i));
  const uint64_t unconnected = 1ull << (2 * bits_k + bits_w);            // above every real key: sorts last
  const uint64_t wkey = (((1ull << bits_w) - 1) - (uint64_t)w) << bits_k;   // descending weight
  row_key[2 * (size_t)e] = connected ? ((uint64_t)i << (bits_k + bits_w)) | wkey | j : unconnected;
  row_key[2 * (size_t)e + 1] = connected ? ((uint64_t)j << (bits_k + bits_w)) | wkey | i : unconnected;
  if (connected) {
    atomicAdd(&deg[i], 1);
    atomicAdd(&deg[j], 1);
  }
}

__global__ void __launch_bounds__(MG_THREADS) mg_decode_kernel(const uint64_t* __restrict__ row_key, int n, int bits_k, int bits_w,
                                                               int32_t* __restrict__ nbr_kf, int32_t* __restrict__ nbr_w) {
  const int t = blockIdx.x * MG_THREADS + threadIdx.x;
  if (t >= n) return;
  const uint64_t wmask = (1ull << bits_w) - 1;
  nbr_kf[t] = (int32_t)(row_key[t] & ((1ull << bits_k) - 1));
  nbr_w[t] = (int32_t)(wmask - ((row_key[t] >> bits_k) & wmask));
}

int mg_bits(int64_t v) {   // bits that hold 0..v
  int b = 1;
  while ((v >> b) != 0) b++;
  return b;
}

// carves one workspace slot into 256-byte aligned arrays: first pass sizes, second pass hands out pointers
struct mg_carver {
  char* base = nullptr;
  size_t off = 0;
  template <class T>
  T* take(size_t n) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += (n * sizeof(T) + 255) & ~size_t(255);
    return p;
  }
};

#define MG_CUB(ctx, call)                                                                                                         \
  do {                                                                                                                            \
    cudaError_t e_ = (call);                                                                                                      \
    if (e_ != cudaSuccess) return cvb_fail((ctx), CVB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    (ctx)->launches++;                                                                                                            \
  } while (0)

}  // namespace

int cvb_covisibility_budgeted(cvb_ctx* ctx, int K, int L, const int32_t* lm_obs_ptr, const int32_t* obs_kf, const uint8_t* obs_skip,
                              const uint8_t* lm_valid, int min_weight, int32_t* nbr_ptr, int32_t* nbr_kf, int32_t* nbr_w, int64_t cap,
                              int64_t* n_total, int64_t pair_budget) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, K >= 0 && L >= 0, "cvb_covisibility: negative size (K %d, L %d)", K, L);
  CVB_REQUIRE(ctx, nbr_ptr && n_total, "cvb_covisibility: nbr_ptr and n_total are required");
  CVB_REQUIRE(ctx, cap >= 0 && ((nbr_kf && nbr_w) || cap == 0), "cvb_covisibility: nbr_kf / nbr_w may be null only with cap == 0 (cap %lld)", (long long)cap);
  CVB_REQUIRE(ctx, min_weight >= 1, "cvb_covisibility: min_weight %d < 1", min_weight);
  CVB_REQUIRE(ctx, lm_obs_ptr || L == 0, "cvb_covisibility: lm_obs_ptr is null");
  CVB_REQUIRE(ctx, pair_budget >= 1, "cvb_covisibility: pair budget %lld < 1", (long long)pair_budget);
  CVB_REQUIRE(ctx, L == 0 || lm_obs_ptr[0] == 0, "cvb_covisibility: lm_obs_ptr[0] = %d, not 0", L ? lm_obs_ptr[0] : 0);
  for (int l = 0; l < L; l++)
    CVB_REQUIRE(ctx, lm_obs_ptr[l + 1] >= lm_obs_ptr[l], "cvb_covisibility: lm_obs_ptr decreases at landmark %d", l);
  CVB_REQUIRE(ctx, obs_kf || L == 0 || lm_obs_ptr[L] == 0, "cvb_covisibility: obs_kf is null");

  // participating observations of the landmarks that keep two observers, and the exclusive scan of their pair counts
  std::vector<int32_t> c_ptr(1, 0), c_kf, seen_in((size_t)K, -1), kf_obs((size_t)K, 0);
  std::vector<int64_t> c_poff(1, 0);
  int64_t n_pairs = 0;
  for (int l = 0; l < L; l++) {
    const size_t start = c_kf.size();
    const bool lm_in = !lm_valid || lm_valid[l];
    for (int o = lm_obs_ptr[l]; o < lm_obs_ptr[l + 1]; o++) {
      const int k = obs_kf[o];
      CVB_REQUIRE(ctx, k >= 0 && k < K, "cvb_covisibility: obs_kf[%d] = %d outside [0, %d)", o, k, K);
      CVB_REQUIRE(ctx, seen_in[k] != l, "cvb_covisibility: keyframe %d observes landmark %d twice", k, l);
      seen_in[k] = l;
      if (lm_in && !(obs_skip && obs_skip[o])) c_kf.push_back(k);
    }
    const int64_t n = (int64_t)(c_kf.size() - start);
    if (n < 2) {
      c_kf.resize(start);
      continue;
    }
    for (size_t t = start; t < c_kf.size(); t++) kf_obs[c_kf[t]]++;
    if (__builtin_add_overflow(n_pairs, n * (n - 1) / 2, &n_pairs))
      return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "cvb_covisibility: more than %lld shared-landmark pairs", (long long)INT64_MAX);
    c_ptr.push_back((int32_t)c_kf.size());
    c_poff.push_back(n_pairs);
  }
  *n_total = 0;
  std::fill(nbr_ptr, nbr_ptr + (size_t)K + 1, 0);
  if (n_pairs == 0) return CVB_OK;

  const int n_lm = (int)c_ptr.size() - 1;
  const int bits_k = mg_bits(K - 1), bits_w = mg_bits(*std::max_element(kf_obs.begin(), kf_obs.end()));   // w(i,j) <= observations of i
  if (2 * bits_k + bits_w > 63)
    return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "cvb_covisibility: %d keyframes with up to %d observations each need a %d-bit ordering key (63 available)",
                    K, *std::max_element(kf_obs.begin(), kf_obs.end()), 2 * bits_k + bits_w);
  const int64_t chunk = std::min(std::min(pair_budget, MG_PAIR_BUDGET), n_pairs);
  const int64_t n_chunks = (n_pairs + chunk - 1) / chunk;
  const int64_t edge_bound = std::min(n_pairs, (int64_t)K * (K - 1) / 2);
  const int64_t acc_cap = edge_bound + (n_chunks > 1 ? chunk : 0);
  if (2 * acc_cap > MG_INDEX_MAX)
    return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "cvb_covisibility: %lld shared-landmark pairs over %d keyframes may give %lld directed edges, beyond the 31-bit index range",
                    (long long)n_pairs, K, (long long)(2 * acc_cap));

  cudaStream_t st = ctx->stream;
  const int key_bits = 2 * bits_k;
  // ---- phase 1: (i, j, w) for every pair of keyframes that share a landmark ----
  size_t temp_bytes = 0, tb = 0;
  CVB_CUDA(ctx, cub::DeviceRadixSort::SortKeys(nullptr, tb, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)chunk, 0, key_bits, st));
  temp_bytes = std::max(temp_bytes, tb);
  CVB_CUDA(ctx, cub::DeviceRunLengthEncode::Encode(nullptr, tb, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int32_t*)nullptr, (int32_t*)nullptr, (int)chunk, st));
  temp_bytes = std::max(temp_bytes, tb);
  if (n_chunks > 1) {
    CVB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, tb, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr,
                                                  (int)acc_cap, 0, key_bits, st));
    temp_bytes = std::max(temp_bytes, tb);
    CVB_CUDA(ctx, cub::DeviceReduce::ReduceByKey(nullptr, tb, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr,
                                                 (int32_t*)nullptr, ::cuda::std::plus<int32_t>(), (int)acc_cap, st));
    temp_bytes = std::max(temp_bytes, tb);
  }
  mg_carver c1;
  int32_t *d_ptr = nullptr, *d_kf = nullptr, *d_num = nullptr, *acc_w = nullptr, *acc_w2 = nullptr;
  int64_t* d_poff = nullptr;
  uint64_t *keys_a = nullptr, *keys_b = nullptr, *acc_k = nullptr, *acc_k2 = nullptr;
  void* d_temp = nullptr;
  for (int pass = 0; pass < 2; pass++) {
    c1.off = 0;
    d_ptr = c1.take<int32_t>((size_t)n_lm + 1);
    d_kf = c1.take<int32_t>(c_kf.size());
    d_poff = c1.take<int64_t>((size_t)n_lm + 1);
    keys_a = c1.take<uint64_t>((size_t)chunk);
    keys_b = c1.take<uint64_t>((size_t)chunk);
    acc_k = c1.take<uint64_t>((size_t)acc_cap);
    acc_w = c1.take<int32_t>((size_t)acc_cap);
    if (n_chunks > 1) {
      acc_k2 = c1.take<uint64_t>((size_t)acc_cap);
      acc_w2 = c1.take<int32_t>((size_t)acc_cap);
    }
    d_num = c1.take<int32_t>(1);
    d_temp = c1.take<char>(temp_bytes);
    if (pass == 0 && !(c1.base = (char*)cvb_ws(ctx, WS_MG_EDGES, c1.off))) return CVB_ERR_CUDA;
  }
  CVB_CUDA(ctx, cudaMemcpyAsync(d_ptr, c_ptr.data(), c_ptr.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CVB_CUDA(ctx, cudaMemcpyAsync(d_kf, c_kf.data(), c_kf.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CVB_CUDA(ctx, cudaMemcpyAsync(d_poff, c_poff.data(), c_poff.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  int64_t n_edge = 0;
  for (int64_t c = 0; c < n_chunks; c++) {
    const int64_t p0 = c * chunk, cnt = std::min(chunk, n_pairs - p0);
    mg_expand_pairs_kernel<<<(unsigned)((cnt + MG_TILE - 1) / MG_TILE), MG_THREADS, 0, st>>>(d_ptr, d_kf, d_poff, n_lm, p0, cnt, bits_k, keys_a);
    CVB_CHECK_LAUNCH(ctx);
    tb = temp_bytes;
    MG_CUB(ctx, cub::DeviceRadixSort::SortKeys(d_temp, tb, (const uint64_t*)keys_a, keys_b, (int)cnt, 0, key_bits, st));
    tb = temp_bytes;
    MG_CUB(ctx, cub::DeviceRunLengthEncode::Encode(d_temp, tb, (const uint64_t*)keys_b, acc_k + n_edge, acc_w + n_edge, d_num, (int)cnt, st));
    int32_t h_num = 0;
    CVB_CUDA(ctx, cudaMemcpyAsync(&h_num, d_num, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaStreamSynchronize(st));
    n_edge += h_num;
    if (c == 0) continue;
    // merge the chunk's counts into the map's: equal keys become adjacent, their counts add
    tb = temp_bytes;
    MG_CUB(ctx, cub::DeviceRadixSort::SortPairs(d_temp, tb, (const uint64_t*)acc_k, acc_k2, (const int32_t*)acc_w, acc_w2, (int)n_edge, 0, key_bits, st));
    tb = temp_bytes;
    MG_CUB(ctx, cub::DeviceReduce::ReduceByKey(d_temp, tb, (const uint64_t*)acc_k2, acc_k, (const int32_t*)acc_w2, acc_w, d_num, ::cuda::std::plus<int32_t>(), (int)n_edge, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(&h_num, d_num, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaStreamSynchronize(st));
    n_edge = h_num;
  }

  // ---- phase 2: rule 3 per edge, the rows' sizes, and the rows ordered by (weight descending, index ascending) ----
  const int n_dir = (int)(2 * n_edge);
  const int row_bits = 2 * bits_k + bits_w + 1;
  size_t temp2 = 0;
  CVB_CUDA(ctx, cub::DeviceRadixSort::SortKeys(nullptr, tb, (const uint64_t*)nullptr, (uint64_t*)nullptr, n_dir, 0, row_bits, st));
  temp2 = std::max(temp2, tb);
  CVB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb, (const int32_t*)nullptr, (int32_t*)nullptr, K + 1, st));
  temp2 = std::max(temp2, tb);
  mg_carver c2;
  int32_t *strong = nullptr, *deg = nullptr, *d_nbr_ptr = nullptr, *d_nbr_kf = nullptr, *d_nbr_w = nullptr;
  unsigned long long* best = nullptr;
  uint64_t *row_a = nullptr, *row_b = nullptr;
  size_t zero_bytes = 0;
  for (int pass = 0; pass < 2; pass++) {
    c2.off = 0;
    strong = c2.take<int32_t>((size_t)K);
    deg = c2.take<int32_t>((size_t)K + 1);   // [K] stays 0: the scan of K + 1 items puts the total at nbr_ptr[K]
    best = c2.take<unsigned long long>((size_t)K);
    zero_bytes = c2.off;
    d_nbr_ptr = c2.take<int32_t>((size_t)K + 1);
    row_a = c2.take<uint64_t>((size_t)n_dir);
    row_b = c2.take<uint64_t>((size_t)n_dir);
    d_nbr_kf = c2.take<int32_t>((size_t)n_dir);
    d_nbr_w = c2.take<int32_t>((size_t)n_dir);
    d_temp = c2.take<char>(temp2);
    if (pass == 0 && !(c2.base = (char*)cvb_ws(ctx, WS_MG_ROWS, c2.off))) return CVB_ERR_CUDA;
  }
  CVB_CUDA(ctx, cudaMemsetAsync(strong, 0, zero_bytes, st));
  const unsigned edge_grid = (unsigned)((n_edge + MG_THREADS - 1) / MG_THREADS);
  mg_row_stats_kernel<<<edge_grid, MG_THREADS, 0, st>>>(acc_k, acc_w, (int)n_edge, bits_k, min_weight, strong, best);
  CVB_CHECK_LAUNCH(ctx);
  mg_connect_kernel<<<edge_grid, MG_THREADS, 0, st>>>(acc_k, acc_w, (int)n_edge, bits_k, bits_w, min_weight, strong, best, deg, row_a);
  CVB_CHECK_LAUNCH(ctx);
  tb = temp2;
  MG_CUB(ctx, cub::DeviceScan::ExclusiveSum(d_temp, tb, (const int32_t*)deg, d_nbr_ptr, K + 1, st));
  CVB_CUDA(ctx, cudaMemcpyAsync(nbr_ptr, d_nbr_ptr, ((size_t)K + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  *n_total = nbr_ptr[K];
  if (*n_total > cap || *n_total == 0) return CVB_OK;
  tb = temp2;
  MG_CUB(ctx, cub::DeviceRadixSort::SortKeys(d_temp, tb, (const uint64_t*)row_a, row_b, n_dir, 0, row_bits, st));
  mg_decode_kernel<<<(unsigned)((*n_total + MG_THREADS - 1) / MG_THREADS), MG_THREADS, 0, st>>>(row_b, (int)*n_total, bits_k, bits_w, d_nbr_kf, d_nbr_w);
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaMemcpyAsync(nbr_kf, d_nbr_kf, (size_t)*n_total * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaMemcpyAsync(nbr_w, d_nbr_w, (size_t)*n_total * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  return CVB_OK;
}

extern "C" int cvb_covisibility(cvb_ctx* ctx, int K, int L, const int32_t* lm_obs_ptr, const int32_t* obs_kf, const uint8_t* obs_skip,
                                const uint8_t* lm_valid, int min_weight, int32_t* nbr_ptr, int32_t* nbr_kf, int32_t* nbr_w, int64_t cap,
                                int64_t* n_total) {
  return cvb_covisibility_budgeted(ctx, K, L, lm_obs_ptr, obs_kf, obs_skip, lm_valid, min_weight, nbr_ptr, nbr_kf, nbr_w, cap, n_total,
                                   MG_PAIR_BUDGET);
}
