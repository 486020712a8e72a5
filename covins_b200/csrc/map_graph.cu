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
  cvb_block B1(ctx, st, false);   // direct: the observation lists are large
  const int32_t *d_ptr, *d_kf;
  const int64_t* d_poff;
  int32_t *d_num, *acc_w, *acc_w2 = nullptr;
  uint64_t *keys_a, *keys_b, *acc_k, *acc_k2 = nullptr;
  char* d_temp;
  B1.in(d_ptr, c_ptr.data(), c_ptr.size()); B1.in(d_kf, c_kf.data(), c_kf.size()); B1.in(d_poff, c_poff.data(), c_poff.size());
  B1.tmp(keys_a, chunk); B1.tmp(keys_b, chunk); B1.tmp(acc_k, acc_cap); B1.tmp(acc_w, acc_cap);
  if (n_chunks > 1) { B1.tmp(acc_k2, acc_cap); B1.tmp(acc_w2, acc_cap); }
  B1.tmp(d_num, 1); B1.tmp(d_temp, temp_bytes);
  if (const int rc = B1.place()) return rc;
  if (const int rc = B1.upload()) return rc;
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
  cvb_block B2(ctx, st);
  int32_t *strong, *deg, *d_nbr_ptr, *d_nbr_kf, *d_nbr_w;
  unsigned long long* best;
  uint64_t *row_a, *row_b;
  B2.tmp(strong, K);
  B2.tmp(deg, (size_t)K + 1);   // [K] stays 0: the scan of K + 1 items puts the total at nbr_ptr[K]
  B2.tmp(best, K);
  B2.tmp(d_nbr_ptr, (size_t)K + 1); B2.tmp(row_a, n_dir); B2.tmp(row_b, n_dir); B2.tmp(d_nbr_kf, n_dir); B2.tmp(d_nbr_w, n_dir);
  B2.tmp(d_temp, temp2);
  if (const int rc = B2.place()) return rc;
  // strong, deg and best are adjacent: one memset zeroes the three
  CVB_CUDA(ctx, cudaMemsetAsync(strong, 0, (size_t)((char*)d_nbr_ptr - (char*)strong), st));
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

// ======================================================================================================================
// K14 cvb_redundant_keyframes: the sequential culling pass of Map::Clean's redundancy pruning (include/covins_b200.h), as
// parallel rounds that commit exactly the keyframes the sequential pass culls.
//   state   hist[l * num_octaves + o] = keyframes not culled that observe l (participating) at octave o; pred_c[k] = pred_C(k);
//           the undecided keyframes in a list.  A keyframe is undecided until it is kept or culled; the host keeps at once
//           every keyframe that fails whatever C is (protected, n(k) = 0, no predecessor, no successor);
//   round   pr_eval_kernel    one warp per undecided k evaluates the rule under the committed C.  A failure is final (adding
//                             keyframes to C only lowers red_C and moves pred_C earlier): k is kept.  The keyframes that pass
//                             form T; each writes itself into lowt[l] of its landmarks (64-bit atomicMin of (round, k), so
//                             the slot needs no reset between rounds);
//           pr_commit_kernel  k in T is culled iff no lower member of T shares a participating landmark with it and its
//                             pred_C is not in T; a culled k's observations leave hist (integer atomics);
//           pr_relink_kernel  pred_C[succ(k)] = pred_C[k] for the culled k, and the keyframes still undecided form the next
//                             list.
//   Why this is exact: a culled k's test depends only on culls below it; of those, the committed ones are exact by
//   induction, and the members of T below k that are still undecided touch neither red_C(k) (no shared landmark) nor
//   pred_C(k) (not its pred_C; any other ancestor is behind it), whether they are culled later or not.  A cull above k
//   committed before k is decided shares no landmark with k either.  Two keyframes adjacent in a chain never commit in the
//   same round (the lower is the higher's pred_C), so the re-links do not chain, and the lowest member of T always commits:
//   the loop ends after at most as many rounds as there are undecided keyframes.
// Integer arithmetic except the th_red and time comparisons (one rounded product, one rounded difference, each the same on
// the host): the output is bit-identical from run to run.
// ======================================================================================================================
namespace {

constexpr int PR_THREADS = 256;
constexpr int PR_WARPS = PR_THREADS / 32;
constexpr uint32_t PR_ROUND_TOP = 0xfffffffeu;   // lowt key (PR_ROUND_TOP - round) << 32 | k: a later round sorts lower

__device__ __forceinline__ unsigned long long pr_key(int round, int k) {
  return ((unsigned long long)(PR_ROUND_TOP - (uint32_t)round) << 32) | (uint32_t)k;
}

__global__ void __launch_bounds__(PR_THREADS) pr_hist_kernel(const int32_t* __restrict__ kf_h, int n, int32_t* hist) {
  const int t = blockIdx.x * PR_THREADS + threadIdx.x;
  if (t < n) atomicAdd(&hist[kf_h[t]], 1);
}

// kf_h[kf_ptr[k] .. kf_ptr[k+1]) = l * num_octaves + octave of k's participating observations
__global__ void __launch_bounds__(PR_THREADS) pr_eval_kernel(const int32_t* __restrict__ und, int n_und, const int32_t* __restrict__ kf_ptr,
                                                             const int32_t* __restrict__ kf_h, const int32_t* __restrict__ hist, int num_octaves,
                                                             int th_obs, double th_red, double max_time_dist, const int32_t* __restrict__ succ,
                                                             const int32_t* __restrict__ pred_c, const double* __restrict__ kf_time, int round,
                                                             int32_t* mark, uint8_t* state, unsigned long long* lowt) {
  const int w = blockIdx.x * PR_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= n_und) return;
  const int k = und[w], b = kf_ptr[k], e = kf_ptr[k + 1];
  int red = 0;
  for (int t = b + lane; t < e; t += 32) {
    const int h = kf_h[t];
    const int o = h % num_octaves, base = h - o;
    const int top = min(o + 1, num_octaves - 1);
    int others = -1;   // k itself is not culled and observes l at o <= o + 1
    for (int q = 0; q <= top; q++) others += hist[base + q];
    red += others >= th_obs;
  }
  for (int s = 16; s; s >>= 1) red += __shfl_xor_sync(0xffffffffu, red, s);
  const bool pass = (double)red > __dmul_rn(th_red, (double)(e - b)) && __dsub_rn(kf_time[succ[k]], kf_time[pred_c[k]]) <= max_time_dist;
  if (!pass) {
    if (lane == 0) state[k] = 1;
    return;
  }
  if (lane == 0) mark[k] = round;
  const unsigned long long key = pr_key(round, k);
  for (int t = b + lane; t < e; t += 32) atomicMin(&lowt[kf_h[t] / num_octaves], key);
}

__global__ void __launch_bounds__(PR_THREADS) pr_commit_kernel(const int32_t* __restrict__ und, int n_und, const int32_t* __restrict__ kf_ptr,
                                                               const int32_t* __restrict__ kf_h, int num_octaves, const int32_t* __restrict__ pred_c,
                                                               const int32_t* __restrict__ mark, const unsigned long long* __restrict__ lowt, int round,
                                                               int32_t* hist, uint8_t* state) {
  const int w = blockIdx.x * PR_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= n_und) return;
  const int k = und[w];
  if (mark[k] != round) return;
  const int b = kf_ptr[k], e = kf_ptr[k + 1];
  const unsigned long long key = pr_key(round, k);
  bool blocked = false;
  if (lane == 0) {
    const int p = pred_c[k];
    blocked = mark[p] == round;
  }
  for (int t = b + lane; t < e && !blocked; t += 32) blocked = lowt[kf_h[t] / num_octaves] < key;   // a lower member of T observes l
  if (__any_sync(0xffffffffu, blocked)) return;
  if (lane == 0) state[k] = 2;
  for (int t = b + lane; t < e; t += 32) atomicSub(&hist[kf_h[t]], 1);
}

__global__ void __launch_bounds__(PR_THREADS) pr_relink_kernel(const int32_t* __restrict__ und, int n_und, const int32_t* __restrict__ succ,
                                                               const uint8_t* __restrict__ state, int32_t* pred_c, int32_t* und_next, int32_t* n_next) {
  const int i = blockIdx.x * PR_THREADS + threadIdx.x;
  if (i >= n_und) return;
  const int k = und[i];
  if (state[k] == 2) pred_c[succ[k]] = pred_c[k];
  else if (state[k] == 0) und_next[atomicAdd(n_next, 1)] = k;
}

}  // namespace

extern "C" int cvb_redundant_keyframes(cvb_ctx* ctx, int K, int L, const int32_t* lm_obs_ptr, const int32_t* obs_kf, const int32_t* obs_octave,
                                       const uint8_t* obs_skip, const uint8_t* lm_valid, const int32_t* kf_pred, const double* kf_time,
                                       const uint8_t* kf_protect, double th_red, double max_time_dist, int th_obs, int num_octaves, uint8_t* culled,
                                       int32_t* n_rounds) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, K >= 0 && L >= 0, "cvb_redundant_keyframes: negative size (K %d, L %d)", K, L);
  CVB_REQUIRE(ctx, th_red >= 0.0 && th_red <= 1.0, "cvb_redundant_keyframes: th_red %g is not in [0, 1]", th_red);
  CVB_REQUIRE(ctx, max_time_dist > 0.0, "cvb_redundant_keyframes: max_time_dist %g is not > 0", max_time_dist);
  CVB_REQUIRE(ctx, th_obs >= 1, "cvb_redundant_keyframes: th_obs %d < 1", th_obs);
  CVB_REQUIRE(ctx, num_octaves >= 1 && num_octaves <= 64, "cvb_redundant_keyframes: num_octaves %d is not in [1, 64]", num_octaves);
  CVB_REQUIRE(ctx, lm_obs_ptr || L == 0, "cvb_redundant_keyframes: lm_obs_ptr is null");
  CVB_REQUIRE(ctx, K == 0 || (kf_pred && kf_time && kf_protect && culled), "cvb_redundant_keyframes: kf_pred, kf_time, kf_protect and culled are required");
  CVB_REQUIRE(ctx, L == 0 || lm_obs_ptr[0] == 0, "cvb_redundant_keyframes: lm_obs_ptr[0] = %d, not 0", L ? lm_obs_ptr[0] : 0);
  for (int l = 0; l < L; l++)
    CVB_REQUIRE(ctx, lm_obs_ptr[l + 1] >= lm_obs_ptr[l], "cvb_redundant_keyframes: lm_obs_ptr decreases at landmark %d", l);
  const int n_obs = L ? lm_obs_ptr[L] : 0;
  CVB_REQUIRE(ctx, (obs_kf && obs_octave) || n_obs == 0, "cvb_redundant_keyframes: obs_kf and obs_octave are required");
  if ((int64_t)L * num_octaves > MG_INDEX_MAX)
    return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "cvb_redundant_keyframes: %d landmarks x %d octaves exceed the 31-bit index range", L, num_octaves);

  // the chains: successors, at most one per keyframe
  std::vector<int32_t> succ((size_t)K, -1);
  for (int k = 0; k < K; k++) {
    const int p = kf_pred[k];
    CVB_REQUIRE(ctx, p >= -1 && p < k, "cvb_redundant_keyframes: kf_pred[%d] = %d is not in [-1, %d)", k, p, k);
    if (p < 0) continue;
    CVB_REQUIRE(ctx, succ[p] < 0, "cvb_redundant_keyframes: keyframe %d has two successors (%d and %d)", p, succ[p], k);
    succ[p] = k;
  }
  // one pass over the observations: validation and the participating ones per keyframe (counting sort by keyframe)
  std::vector<int32_t> seen_in((size_t)K, -1), kf_ptr((size_t)K + 1, 0);
  for (int l = 0; l < L; l++) {
    const bool lm_in = !lm_valid || lm_valid[l];
    for (int o = lm_obs_ptr[l]; o < lm_obs_ptr[l + 1]; o++) {
      const int k = obs_kf[o];
      CVB_REQUIRE(ctx, k >= 0 && k < K, "cvb_redundant_keyframes: obs_kf[%d] = %d outside [0, %d)", o, k, K);
      CVB_REQUIRE(ctx, seen_in[k] != l, "cvb_redundant_keyframes: keyframe %d observes landmark %d twice", k, l);
      CVB_REQUIRE(ctx, obs_octave[o] >= 0 && obs_octave[o] < num_octaves, "cvb_redundant_keyframes: obs_octave[%d] = %d outside [0, %d)", o,
                  obs_octave[o], num_octaves);
      seen_in[k] = l;
      if (lm_in && !(obs_skip && obs_skip[o])) kf_ptr[k + 1]++;
    }
  }
  if (n_rounds) *n_rounds = 0;
  if (K == 0) return CVB_OK;
  for (int k = 0; k < K; k++) kf_ptr[k + 1] += kf_ptr[k];
  // every keyframe that fails whatever C is stays: protected, n(k) = 0, no predecessor, no successor
  std::vector<uint8_t> state((size_t)K, 1);
  std::vector<int32_t> und;
  for (int k = 0; k < K; k++)
    if (!kf_protect[k] && kf_ptr[k + 1] > kf_ptr[k] && kf_pred[k] >= 0 && succ[k] >= 0) {
      state[k] = 0;
      und.push_back(k);
    }
  std::fill(culled, culled + K, 0);
  const int n0 = (int)und.size();
  if (n0 == 0) return CVB_OK;
  const int n_part = kf_ptr[K];
  std::vector<int32_t> kf_h((size_t)n_part), fill(kf_ptr.begin(), kf_ptr.end() - 1);
  for (int l = 0; l < L; l++) {
    if (lm_valid && !lm_valid[l]) continue;
    for (int o = lm_obs_ptr[l]; o < lm_obs_ptr[l + 1]; o++)
      if (!(obs_skip && obs_skip[o])) kf_h[fill[obs_kf[o]]++] = l * num_octaves + obs_octave[o];
  }

  cudaStream_t st = ctx->stream;
  const size_t n_bins = (size_t)L * num_octaves;
  cvb_block B(ctx, st, false);   // direct: the observation lists are large
  const int32_t *d_kf_ptr, *d_kf_h, *d_succ;
  const double* d_time;
  int32_t *hist, *pred_c, *mark, *und_a, *und_b, *d_cnt;
  uint8_t* d_state;
  unsigned long long* lowt;
  B.in(d_kf_ptr, kf_ptr.data(), kf_ptr.size()); B.in(d_kf_h, kf_h.data(), kf_h.size()); B.in(pred_c, kf_pred, K); B.in(d_succ, succ.data(), K);
  B.in(d_time, kf_time, K); B.in(d_state, state.data(), K); B.in(und_a, und.data(), n0);
  B.tmp(und_b, n0); B.tmp(hist, n_bins);
  B.tmp(d_cnt, (size_t)n0 + 1);   // round r counts its survivors in d_cnt[r]: no reset between rounds
  B.tmp(mark, K); B.tmp(lowt, L);
  if (const int rc = B.place()) return rc;
  if (const int rc = B.upload()) return rc;
  // hist and d_cnt are adjacent: one memset zeroes both; mark = -1 and lowt = all ones match no round
  CVB_CUDA(ctx, cudaMemsetAsync(hist, 0, (size_t)((char*)mark - (char*)hist), st));
  CVB_CUDA(ctx, cudaMemsetAsync(mark, 0xff, (size_t)((char*)(lowt + L) - (char*)mark), st));
  pr_hist_kernel<<<(unsigned)((n_part + PR_THREADS - 1) / PR_THREADS), PR_THREADS, 0, st>>>(d_kf_h, n_part, hist);
  CVB_CHECK_LAUNCH(ctx);
  int n_und = n0, round = 0;
  while (n_und > 0) {
    const unsigned warp_grid = (unsigned)((n_und + PR_WARPS - 1) / PR_WARPS);
    pr_eval_kernel<<<warp_grid, PR_THREADS, 0, st>>>(und_a, n_und, d_kf_ptr, d_kf_h, hist, num_octaves, th_obs, th_red, max_time_dist, d_succ,
                                                     pred_c, d_time, round, mark, d_state, lowt);
    CVB_CHECK_LAUNCH(ctx);
    pr_commit_kernel<<<warp_grid, PR_THREADS, 0, st>>>(und_a, n_und, d_kf_ptr, d_kf_h, num_octaves, pred_c, mark, lowt, round, hist, d_state);
    CVB_CHECK_LAUNCH(ctx);
    pr_relink_kernel<<<(unsigned)((n_und + PR_THREADS - 1) / PR_THREADS), PR_THREADS, 0, st>>>(und_a, n_und, d_succ, d_state, pred_c, und_b,
                                                                                               d_cnt + round);
    CVB_CHECK_LAUNCH(ctx);
    int32_t next = 0;
    CVB_CUDA(ctx, cudaMemcpyAsync(&next, d_cnt + round, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaStreamSynchronize(st));
    if (next >= n_und)   // the lowest member of T always commits: a round that decides nothing is a device fault
      return cvb_fail(ctx, CVB_ERR_CUDA, "cvb_redundant_keyframes: round %d decided no keyframe (%d undecided)", round, n_und);
    n_und = next;
    std::swap(und_a, und_b);
    round++;
  }
  CVB_CUDA(ctx, cudaMemcpyAsync(state.data(), d_state, (size_t)K, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  for (int k = 0; k < K; k++) culled[k] = state[k] == 2;
  if (n_rounds) *n_rounds = round;
  return CVB_OK;
}
