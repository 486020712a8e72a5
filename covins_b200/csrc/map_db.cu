// map_db.cu — the merged map's ORB or SIFT descriptors resident in HBM, queried per place-recognition request.
//
// Reference flow (covins_backend/src/covins_backend/placerec_gen_be.cpp:60-135): for every candidate keyframe the
// query keyframe's descriptor matrix is matched (knnMatch k=2 → distance + ratio filter) and only the accepted
// matches (img_matches, :102-114) and their count (:116-124) are consumed.  The descriptors of the map's keyframes
// never change after a keyframe is added (keyframe_be.cpp:106-137 fills them once from the message), so they are
// uploaded once (cvb_db_append / cvb_db_append_sift) and stay in HBM; a query moves nq*32 B (ORB) or nq*128 B (SIFT, u8)
// up and the accepted matches down.  Both row kinds share the code below; they differ in the row size, the tensor-core
// tile image (cvb_tc::tile_bytes / expand_tiles by metric) and the host staging of SIFT rows (checked and quantised to u8).
//
// cvb_db_group (end of file): the same database with its keyframes dealt over the ranks of a cvb_group, one ordinary cvb_db
// per rank.  A request runs the per-rank 2-NN and compaction above on every rank's stream; a gather on rank 0 then reads
// the ranks' counts and compacted lists (same device or peer access) and writes them in global keyframe order, so the
// outputs are bit-identical to one cvb_db holding every keyframe.
#include <string.h>

#include <algorithm>
#include <memory>

#include "ba_group.cuh"
#include "cvb_internal.cuh"
#include "tc_match.cuh"

struct cvb_buf {
  void* p = nullptr;
  size_t cap = 0;
};

struct cvb_db {
  const cvb_ctx* owner = nullptr;   // the ctx of cvb_db_create: the device the rows live on
  int desc_bytes = 32;   // 32: ORB rows (Hamming); 128: SIFT rows as exact u8 (L2)
  uint8_t* d_rows = nullptr;
  size_t cap_rows = 0;
  std::vector<int32_t> seg_ptr{0};
  int32_t* d_seg = nullptr;
  size_t cap_seg = 0;
  bool seg_dirty = true;
  // the tensor-core matcher's operand tiles of every keyframe (tc_match.cu, "pre-expanded operand tiles"): written once
  // at append time, 128-row tiles, seg_tile[s] = first tile of keyframe s
  uint8_t* d_xt = nullptr;
  size_t cap_tiles = 0;
  std::vector<int32_t> seg_tile{0};
  int32_t* d_seg_tile = nullptr;
  // per-query scratch (grow-only)
  cvb_buf q, mt, md, nm, off, out_seg, out_q, out_t, out_d;
  int metric() const { return desc_bytes == 32 ? 0 : 1; }   // cvb_tc metric of the rows
};

namespace {

int grow(cvb_ctx* ctx, cvb_buf& b, size_t bytes) {
  if (b.p && b.cap >= bytes) return CVB_OK;
  if (b.p) {
    CVB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    CVB_CUDA(ctx, cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
  }
  const size_t want = std::max<size_t>(256, bytes + bytes / 4);
  CVB_CUDA(ctx, cudaMalloc(&b.p, want));
  b.cap = want;
  return CVB_OK;
}

// device copies of the segment tables
int refresh_seg(cvb_ctx* ctx, cvb_db* db) {
  if (!db->seg_dirty) return CVB_OK;
  cudaStream_t st = ctx->stream;
  if (db->cap_seg < db->seg_ptr.size()) {
    CVB_CUDA(ctx, cudaStreamSynchronize(st));
    if (db->d_seg) CVB_CUDA(ctx, cudaFree(db->d_seg));
    if (db->d_seg_tile) CVB_CUDA(ctx, cudaFree(db->d_seg_tile));
    db->d_seg = db->d_seg_tile = nullptr;
    db->cap_seg = db->seg_ptr.size() * 3 / 2 + 16;
    CVB_CUDA(ctx, cudaMalloc(&db->d_seg, db->cap_seg * sizeof(int32_t)));
    CVB_CUDA(ctx, cudaMalloc(&db->d_seg_tile, db->cap_seg * sizeof(int32_t)));
  }
  CVB_CUDA(ctx, cudaMemcpyAsync(db->d_seg, db->seg_ptr.data(), db->seg_ptr.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CVB_CUDA(ctx, cudaMemcpyAsync(db->d_seg_tile, db->seg_tile.data(), db->seg_tile.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  db->seg_dirty = false;
  return CVB_OK;
}

int reserve_tiles(cvb_ctx* ctx, cvb_db* db, size_t tiles, size_t used_tiles) {
  if (tiles <= db->cap_tiles) return CVB_OK;
  const size_t want = std::max(tiles, db->cap_tiles * 3 / 2), tb = cvb_tc::tile_bytes(db->metric());
  uint8_t* p = nullptr;
  CVB_CUDA(ctx, cudaMalloc(&p, want * tb));
  const size_t used = used_tiles * tb;
  if (used) CVB_CUDA(ctx, cudaMemcpyAsync(p, db->d_xt, used, cudaMemcpyDeviceToDevice, ctx->stream));
  CVB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (db->d_xt) CVB_CUDA(ctx, cudaFree(db->d_xt));
  db->d_xt = p;
  db->cap_tiles = want;
  return CVB_OK;
}

// exclusive scan of the per-segment match counts; off[n_seg] = total.  One CTA, chunks of 1024 with a carry.
__global__ void __launch_bounds__(1024) db_offsets_kernel(const int32_t* __restrict__ cnt, int n_seg,
                                                           int32_t* __restrict__ off) {
  __shared__ int32_t warp_sum[32];
  __shared__ int32_t carry_s;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < n_seg; base += 1024) {
    const int i = base + threadIdx.x;
    const int32_t v = i < n_seg ? cnt[i] : 0;
    int32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int32_t y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int32_t w = warp_sum[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += y;
      }
      warp_sum[lane] = w;
    }
    __syncthreads();
    const int32_t carry = carry_s;
    const int32_t incl = x + (warp ? warp_sum[warp - 1] : 0) + carry;
    if (i < n_seg) off[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) off[n_seg] = carry_s;
}

// One warp per segment: accepted rows in query order (== the order of the reference's img_matches vector).
__global__ void __launch_bounds__(256) db_compact_kernel(const int32_t* __restrict__ mt, const float* __restrict__ md,
                                                          int nq, int n_seg, const int32_t* __restrict__ off, int cap,
                                                          int32_t* __restrict__ o_seg, int32_t* __restrict__ o_q,
                                                          int32_t* __restrict__ o_t, float* __restrict__ o_d) {
  const int seg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (seg >= n_seg) return;
  const int lane = threadIdx.x & 31;
  int pos = off[seg];
  const int32_t* row_t = mt + (size_t)seg * nq;
  const float* row_d = md + (size_t)seg * nq;
  for (int q0 = 0; q0 < nq; q0 += 32) {
    const int q = q0 + lane;
    const int32_t t = q < nq ? row_t[q] : -1;
    const unsigned m = __ballot_sync(0xffffffffu, t >= 0);
    if (t >= 0) {
      const int p = pos + __popc(m & ((1u << lane) - 1u));
      if (p < cap) {
        o_seg[p] = seg;
        o_q[p] = q;
        o_t[p] = t;
        o_d[p] = row_d[q];
      }
    }
    pos += __popc(m);
  }
}

// K18: the gather of a batch removal.  dst[v] = src[run_src[r] + (v - run_dst[r])] for every 16-byte vector v < n_vec of
// the destination, r the kept run with run_dst[r] <= v < run_dst[r + 1] (offsets in vectors, run_dst strictly increasing,
// run_dst[n_runs] = n_vec).  A CTA copies kGatherVecs * 256 consecutive vectors: its first thread finds the runs of its
// first and last vector by binary search over the whole table, and every thread then searches only between those two
// (one run for most CTAs).  Each thread issues its loads before its stores.
constexpr int kGatherThreads = 256, kGatherVecs = 8;

__device__ __forceinline__ int run_of(const int64_t* __restrict__ run_dst, int lo, int hi, int64_t v) {
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (run_dst[mid] <= v) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kGatherThreads) db_remove_gather_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst,
                                                                          const int64_t* __restrict__ run_dst,
                                                                          const int64_t* __restrict__ run_src, int n_runs, int64_t n_vec) {
  __shared__ int lo_s, hi_s;
  const int64_t v0 = (int64_t)blockIdx.x * (kGatherThreads * kGatherVecs);
  const int64_t v_end = v0 + kGatherThreads * kGatherVecs, v_last = (v_end < n_vec ? v_end : n_vec) - 1;
  if (threadIdx.x == 0) {
    lo_s = run_of(run_dst, 0, n_runs - 1, v0);
    hi_s = run_of(run_dst, lo_s, n_runs - 1, v_last);
  }
  __syncthreads();
  const int lo = lo_s, hi = hi_s;
  uint4 x[kGatherVecs];
#pragma unroll
  for (int j = 0; j < kGatherVecs; j++) {
    const int64_t v = v0 + j * kGatherThreads + threadIdx.x;
    if (v <= v_last) {
      const int r = run_of(run_dst, lo, hi, v);
      x[j] = src[run_src[r] + (v - run_dst[r])];
    }
  }
#pragma unroll
  for (int j = 0; j < kGatherVecs; j++) {
    const int64_t v = v0 + j * kGatherThreads + threadIdx.x;
    if (v <= v_last) dst[v] = x[j];
  }
}

// The refusals of a batch removal from n_kf keyframes: gone[k] = 1 for every listed index k
int check_removals(cvb_ctx* ctx, const int32_t* kf_index, int n, int n_kf, const char* fn, std::vector<char>& gone) {
  CVB_REQUIRE(ctx, n >= 0, "%s: negative count n = %d", fn, n);
  CVB_REQUIRE(ctx, n == 0 || kf_index, "%s: null index list with n = %d", fn, n);
  gone.assign((size_t)n_kf, 0);
  for (int i = 0; i < n; i++) {
    const int k = kf_index[i];
    CVB_REQUIRE(ctx, k >= 0 && k < n_kf, "%s: keyframe index %d out of range (database holds %d)", fn, k, n_kf);
    CVB_REQUIRE(ctx, !gone[k], "%s: keyframe index %d given twice", fn, k);
    gone[k] = 1;
  }
  return CVB_OK;
}

// The kept keyframes of [first, n_seg) of one array, keyframe s spanning units [off[s], off[s + 1]) of `unit` bytes, as runs
// of 16-byte vectors relative to off[first]: run_src [n_runs] and run_dst [n_runs + 1] (the last entry: the vectors kept).
// Kept keyframes that are adjacent in the source, removed empty ones between them included, form one run.
void kept_runs(const std::vector<int32_t>& off, const std::vector<char>& gone, int first, size_t unit, std::vector<int64_t>& run_dst,
               std::vector<int64_t>& run_src) {
  const int64_t base = off[first];
  int64_t total = 0, src_end = -1;
  for (size_t s = (size_t)first; s + 1 < off.size(); s++) {
    if (gone[s] || off[s + 1] == off[s]) continue;
    const int64_t a = (off[s] - base) * (int64_t)unit / 16, b = (off[s + 1] - base) * (int64_t)unit / 16;
    if (a != src_end) {
      run_src.push_back(a);
      run_dst.push_back(total);
    }
    total += b - a;
    src_end = b;
  }
  run_dst.push_back(total);
}

// K18 on one array: the kept vectors from `base` on gathered into a scratch block of the pool, then copied back to `base`
int gather_runs(cvb_ctx* ctx, uint8_t* base, const int64_t* d_run_dst, const int64_t* d_run_src, int n_runs, int64_t n_vec) {
  if (n_vec == 0) return CVB_OK;
  cudaStream_t st = ctx->stream;
  cvb_block B(ctx, st, false);
  uint4* tmp;
  B.tmp(tmp, (size_t)n_vec);
  if (const int rc = B.place()) return rc;
  const int64_t per_cta = kGatherThreads * kGatherVecs;
  db_remove_gather_kernel<<<(unsigned)((n_vec + per_cta - 1) / per_cta), kGatherThreads, 0, st>>>((const uint4*)base, tmp, d_run_dst,
                                                                                                  d_run_src, n_runs, n_vec);
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaMemcpyAsync(base, tmp, (size_t)n_vec * 16, cudaMemcpyDeviceToDevice, st));
  return CVB_OK;
}

// Removes the checked keyframes gone[] from db: the device work enqueued on ctx->stream, the host tables rebuilt.  Only the
// suffix from the first removed keyframe that holds rows moves (removing empty keyframes moves nothing).  `stage` receives
// the block of the uploaded run tables when there is device work: it reads pinned memory, so the caller keeps it until it
// has synchronised the stream.
int compact(cvb_ctx* ctx, cvb_db* db, const std::vector<char>& gone, std::unique_ptr<cvb_block>& stage) {
  const int n_seg = (int)db->seg_ptr.size() - 1;
  int first = 0, moved = n_seg;
  while (first < n_seg && !gone[first]) first++;
  for (int s = first; s < n_seg && moved == n_seg; s++)
    if (gone[s] && db->seg_ptr[s + 1] > db->seg_ptr[s]) moved = s;
  if (moved < n_seg) {
    const size_t tb = cvb_tc::tile_bytes(db->metric());
    std::vector<int64_t> rd, rs, td, ts;
    kept_runs(db->seg_ptr, gone, moved, (size_t)db->desc_bytes, rd, rs);
    kept_runs(db->seg_tile, gone, moved, tb, td, ts);
    if (rd.back()) {   // kept rows follow the first moved keyframe (and so kept tiles)
      stage.reset(new cvb_block(ctx, ctx->stream));
      int64_t *d_rd, *d_rs, *d_td, *d_ts;
      stage->in(d_rd, rd.data(), rd.size());
      stage->in(d_rs, rs.data(), rs.size());
      stage->in(d_td, td.data(), td.size());
      stage->in(d_ts, ts.data(), ts.size());
      int rc;
      if ((rc = stage->place()) || (rc = stage->upload())) return rc;
      if ((rc = gather_runs(ctx, db->d_rows + (size_t)db->seg_ptr[moved] * db->desc_bytes, d_rd, d_rs, (int)rs.size(), rd.back())))
        return rc;
      if ((rc = gather_runs(ctx, db->d_xt + (size_t)db->seg_tile[moved] * tb, d_td, d_ts, (int)ts.size(), td.back()))) return rc;
    }
  }
  std::vector<int32_t> p(db->seg_ptr.begin(), db->seg_ptr.begin() + first + 1), t(db->seg_tile.begin(), db->seg_tile.begin() + first + 1);
  for (int s = first; s < n_seg; s++)
    if (!gone[s]) {
      p.push_back(p.back() + (db->seg_ptr[s + 1] - db->seg_ptr[s]));
      t.push_back(t.back() + (db->seg_tile[s + 1] - db->seg_tile[s]));
    }
  db->seg_ptr.swap(p);
  db->seg_tile.swap(t);
  db->seg_dirty = true;
  return CVB_OK;
}

int remove_batch(cvb_ctx* ctx, cvb_db* db, const int32_t* kf_index, int n, const char* fn) {
  std::vector<char> gone;
  int rc = check_removals(ctx, kf_index, n, (int)db->seg_ptr.size() - 1, fn, gone);
  if (rc || n == 0) return rc;
  std::unique_ptr<cvb_block> stage;
  rc = compact(ctx, db, gone, stage);
  if (stage) {
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (!rc && e != cudaSuccess) rc = cvb_fail(ctx, CVB_ERR_CUDA, "%s: cudaStreamSynchronize failed: %s", fn, cudaGetErrorString(e));
  }
  return rc;
}

// calls of one row kind on a database of the other are refused
int require_kind(cvb_ctx* ctx, const cvb_db* db, bool sift, const char* fn) {
  if ((db->desc_bytes == 128) != sift)
    return cvb_fail(ctx, CVB_ERR_INVALID, "%s: the database holds %s descriptors", fn, db->desc_bytes == 128 ? "SIFT" : "ORB");
  return CVB_OK;
}

int check_rows_per_kf(cvb_ctx* ctx, const cvb_db* db, const void* rows, const int32_t* rows_per_kf, int n_kf, const char* fn,
                      int64_t* add) {
  CVB_REQUIRE(ctx, n_kf >= 0 && (n_kf == 0 || rows_per_kf), "%s: bad arguments", fn);
  *add = 0;
  for (int i = 0; i < n_kf; ++i) {
    CVB_REQUIRE(ctx, rows_per_kf[i] >= 0, "%s: negative row count", fn);
    *add += rows_per_kf[i];
  }
  CVB_REQUIRE(ctx, db->seg_ptr.back() + *add < (int64_t)1 << 31, "%s: more than 2^31 rows", fn);
  CVB_REQUIRE(ctx, *add == 0 || rows, "%s: null rows", fn);
  return CVB_OK;
}

// appends checked keyframes whose rows are already in the database's u8 layout (host memory)
int append_rows(cvb_ctx* ctx, cvb_db* db, const uint8_t* rows, const int32_t* rows_per_kf, int n_kf, int64_t add) {
  const int64_t have = db->seg_ptr.back();
  if ((size_t)(have + add) > db->cap_rows) {
    const int rc = cvb_db_reserve(ctx, db, std::max<int64_t>(have + add, (int64_t)(db->cap_rows * 3 / 2)));
    if (rc) return rc;
  }
  if (add) {
    CVB_CUDA(ctx, cudaMemcpyAsync(db->d_rows + (size_t)have * db->desc_bytes, rows, (size_t)add * db->desc_bytes,
                                  cudaMemcpyHostToDevice, ctx->stream));
    CVB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // `rows` may be freed by the caller on return
  }
  const int seg_old = (int)db->seg_ptr.size() - 1, tile_old = db->seg_tile.back();
  for (int i = 0; i < n_kf; ++i) {
    db->seg_ptr.push_back(db->seg_ptr.back() + rows_per_kf[i]);
    db->seg_tile.push_back(db->seg_tile.back() + (rows_per_kf[i] + 127) / 128);
  }
  db->seg_dirty = true;
  // the new keyframes' operand tiles (HBM-bound, once per keyframe; every later query reads them through the TMA engine)
  int rc = reserve_tiles(ctx, db, (size_t)db->seg_tile.back(), (size_t)tile_old);
  if (rc) return rc;
  if ((rc = refresh_seg(ctx, db))) return rc;
  rc = cvb_tc::expand_tiles(ctx, db->metric(), db->d_rows, db->d_seg, db->d_seg_tile, seg_old, seg_old + n_kf, tile_old,
                            db->seg_tile.back() - tile_old, db->d_xt, ctx->stream);
  if (rc) return rc;
  CVB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return CVB_OK;
}

// the filtered 2-NN of the device query d_q (database layout) against every keyframe, dense device outputs; the keyframes
// are matched from their resident operand tiles when the tensor-core kernel runs
int match_dev(cvb_ctx* ctx, cvb_db* db, const uint8_t* d_q, int nq, float thr, float ratio, int32_t* d_mt, float* d_md, int32_t* d_nm,
              void* stream) {
  const int n_seg = (int)db->seg_ptr.size() - 1;
  int rc = refresh_seg(ctx, db);
  if (rc) return rc;
  return cvb_match_dev(ctx, db->metric(), d_q, nq, db->d_rows, db->d_seg, db->seg_ptr.data(), n_seg, db->d_xt, db->d_seg_tile, thr,
                       ratio, d_mt, d_md, d_nm, cvb_stream(ctx, stream));
}

// host request: q = ORB rows (u8) or SIFT rows (CV_32F, checked and quantised into the pinned staging buffer before any device
// work); accepted matches compacted by (keyframe, queryIdx)
int match_host(cvb_ctx* ctx, cvb_db* db, const void* q, int nq, float thr, float ratio, int32_t* n_matches, int32_t* m_kf,
               int32_t* m_query, int32_t* m_train, float* m_dist, int cap, int32_t* n_total, const char* fn) {
  const int n_seg = (int)db->seg_ptr.size() - 1;
  CVB_REQUIRE(ctx, nq >= 0 && cap >= 0 && n_total && (nq == 0 || q), "%s: bad arguments", fn);
  CVB_REQUIRE(ctx, cap == 0 || (m_kf && m_query && m_train && m_dist), "%s: null outputs", fn);
  *n_total = 0;
  const size_t qb = (size_t)nq * db->desc_bytes;
  // pinned staging: [query | counts | offsets tail]
  const size_t pin_q = (qb + 255) & ~(size_t)255;
  uint8_t* pin = (uint8_t*)cvb_pinned(ctx, pin_q + (size_t)(n_seg + 1) * 4 + 64);
  if (!pin) return CVB_ERR_CUDA;
  if (db->desc_bytes == 32) memcpy(pin, q, qb);
  else if (!cvb_quantize_sift((const float*)q, qb, pin))
    return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "%s: SIFT descriptors must be integer-valued in [0,255] (cv::xfeatures2d::SIFT output)", fn);
  if (n_seg == 0) return CVB_OK;
  if (nq == 0) {
    if (n_matches) std::fill(n_matches, n_matches + n_seg, 0);
    return CVB_OK;
  }
  cudaStream_t st = ctx->stream;
  int rc;
  const size_t on = (size_t)n_seg * nq;
  if ((rc = grow(ctx, db->q, qb))) return rc;
  if ((rc = grow(ctx, db->mt, on * 4))) return rc;
  if ((rc = grow(ctx, db->md, on * 4))) return rc;
  if ((rc = grow(ctx, db->nm, (size_t)n_seg * 4))) return rc;
  if ((rc = grow(ctx, db->off, (size_t)(n_seg + 1) * 4))) return rc;
  if (cap) {
    if ((rc = grow(ctx, db->out_seg, (size_t)cap * 4))) return rc;
    if ((rc = grow(ctx, db->out_q, (size_t)cap * 4))) return rc;
    if ((rc = grow(ctx, db->out_t, (size_t)cap * 4))) return rc;
    if ((rc = grow(ctx, db->out_d, (size_t)cap * 4))) return rc;
  }
  CVB_CUDA(ctx, cudaMemcpyAsync(db->q.p, pin, qb, cudaMemcpyHostToDevice, st));
  rc = match_dev(ctx, db, (const uint8_t*)db->q.p, nq, thr, ratio, (int32_t*)db->mt.p, (float*)db->md.p, (int32_t*)db->nm.p, nullptr);
  if (rc) return rc;
  db_offsets_kernel<<<1, 1024, 0, st>>>((const int32_t*)db->nm.p, n_seg, (int32_t*)db->off.p);
  CVB_CHECK_LAUNCH(ctx);
  if (cap) {
    db_compact_kernel<<<(n_seg + 7) / 8, 256, 0, st>>>((const int32_t*)db->mt.p, (const float*)db->md.p, nq, n_seg,
                                                       (const int32_t*)db->off.p, cap, (int32_t*)db->out_seg.p,
                                                       (int32_t*)db->out_q.p, (int32_t*)db->out_t.p,
                                                       (float*)db->out_d.p);
    CVB_CHECK_LAUNCH(ctx);
  }
  int32_t* pin_cnt = (int32_t*)(pin + pin_q);
  int32_t* pin_tot = pin_cnt + n_seg;
  CVB_CUDA(ctx, cudaMemcpyAsync(pin_cnt, db->nm.p, (size_t)n_seg * 4, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaMemcpyAsync(pin_tot, (int32_t*)db->off.p + n_seg, 4, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  const int total = *pin_tot;
  *n_total = total;
  if (n_matches) memcpy(n_matches, pin_cnt, (size_t)n_seg * 4);
  const int n_out = std::min(total, cap);
  if (n_out) {
    CVB_CUDA(ctx, cudaMemcpyAsync(m_kf, db->out_seg.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(m_query, db->out_q.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(m_train, db->out_t.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaMemcpyAsync(m_dist, db->out_d.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(ctx, cudaStreamSynchronize(st));
  }
  return CVB_OK;
}

}  // namespace

extern "C" {

int cvb_db_create(cvb_ctx* ctx, int desc_bytes, cvb_db** out) {
  if (!ctx || !out) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  *out = nullptr;
  if (desc_bytes != 32 && desc_bytes != 128)
    return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "descriptor database: 32-byte ORB or 128-byte SIFT descriptors, got %d", desc_bytes);
  cvb_db* db = new cvb_db();
  db->owner = ctx;
  db->desc_bytes = desc_bytes;
  *out = db;
  return CVB_OK;
}

int cvb_db_destroy(cvb_ctx* ctx, cvb_db* db) {
  if (!db) return CVB_OK;
  if (ctx) cudaStreamSynchronize(ctx->stream);
  if (db->d_rows) cudaFree(db->d_rows);
  if (db->d_seg) cudaFree(db->d_seg);
  if (db->d_seg_tile) cudaFree(db->d_seg_tile);
  if (db->d_xt) cudaFree(db->d_xt);
  for (cvb_buf* b : {&db->q, &db->mt, &db->md, &db->nm, &db->off, &db->out_seg, &db->out_q, &db->out_t, &db->out_d})
    if (b->p) cudaFree(b->p);
  delete db;
  return CVB_OK;
}

int cvb_db_reserve(cvb_ctx* ctx, cvb_db* db, int64_t rows) {
  if (!ctx || !db || rows < 0) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  if ((size_t)rows <= db->cap_rows) return CVB_OK;
  uint8_t* p = nullptr;
  CVB_CUDA(ctx, cudaMalloc(&p, (size_t)rows * db->desc_bytes));
  const size_t used = (size_t)db->seg_ptr.back() * db->desc_bytes;
  if (used) CVB_CUDA(ctx, cudaMemcpyAsync(p, db->d_rows, used, cudaMemcpyDeviceToDevice, ctx->stream));
  CVB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (db->d_rows) CVB_CUDA(ctx, cudaFree(db->d_rows));
  db->d_rows = p;
  db->cap_rows = (size_t)rows;
  return CVB_OK;
}

int cvb_db_append(cvb_ctx* ctx, cvb_db* db, const uint8_t* rows, const int32_t* rows_per_kf, int n_kf) {
  if (!ctx || !db) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  int64_t add = 0;
  int rc;
  if ((rc = require_kind(ctx, db, false, "cvb_db_append")) || (rc = check_rows_per_kf(ctx, db, rows, rows_per_kf, n_kf, "cvb_db_append", &add)))
    return rc;
  return append_rows(ctx, db, rows, rows_per_kf, n_kf, add);
}

int cvb_db_append_sift(cvb_ctx* ctx, cvb_db* db, const float* rows, const int32_t* rows_per_kf, int n_kf) {
  if (!ctx || !db) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  int64_t add = 0;
  int rc;
  if ((rc = require_kind(ctx, db, true, "cvb_db_append_sift")) ||
      (rc = check_rows_per_kf(ctx, db, rows, rows_per_kf, n_kf, "cvb_db_append_sift", &add)))
    return rc;
  std::vector<uint8_t> u8((size_t)add * 128);   // checked and quantised while staged: a refusal leaves the database unchanged
  if (!cvb_quantize_sift(rows, u8.size(), u8.data()))
    return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "cvb_db_append_sift: SIFT descriptors must be integer-valued in [0,255] (cv::xfeatures2d::SIFT output)");
  return append_rows(ctx, db, u8.data(), rows_per_kf, n_kf, add);
}

int cvb_db_remove(cvb_ctx* ctx, cvb_db* db, int kf_index) {
  if (!ctx || !db) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  const int32_t k = kf_index;
  return remove_batch(ctx, db, &k, 1, "cvb_db_remove");
}

int cvb_db_remove_batch(cvb_ctx* ctx, cvb_db* db, const int32_t* kf_index, int n) {
  if (!ctx || !db) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  return remove_batch(ctx, db, kf_index, n, "cvb_db_remove_batch");
}

int cvb_db_size(const cvb_db* db, int32_t* n_kf, int64_t* n_rows) {
  if (!db) return CVB_ERR_INVALID;
  if (n_kf) *n_kf = (int32_t)db->seg_ptr.size() - 1;
  if (n_rows) *n_rows = db->seg_ptr.back();
  return CVB_OK;
}

int cvb_db_match_hamming_dev(cvb_ctx* ctx, cvb_db* db, const uint8_t* d_q, int nq, float thr, float ratio,
                             int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches, void* stream) {
  if (!ctx || !db) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  if (const int rc = require_kind(ctx, db, false, "cvb_db_match_hamming_dev")) return rc;
  const int n_seg = (int)db->seg_ptr.size() - 1;
  CVB_REQUIRE(ctx, nq >= 0 && (nq == 0 || d_q) && (n_seg == 0 || d_n_matches), "cvb_db_match_hamming_dev: bad arguments");
  if (n_seg == 0) return CVB_OK;
  return match_dev(ctx, db, d_q, nq, thr, ratio, d_match_train, d_match_dist, d_n_matches, stream);
}

int cvb_db_match_hamming(cvb_ctx* ctx, cvb_db* db, const uint8_t* q, int nq, float thr, float ratio,
                         int32_t* n_matches, int32_t* m_kf, int32_t* m_query, int32_t* m_train, float* m_dist,
                         int cap, int32_t* n_total) {
  if (!ctx || !db) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  if (const int rc = require_kind(ctx, db, false, "cvb_db_match_hamming")) return rc;
  return match_host(ctx, db, q, nq, thr, ratio, n_matches, m_kf, m_query, m_train, m_dist, cap, n_total, "cvb_db_match_hamming");
}

int cvb_db_match_l2_dev(cvb_ctx* ctx, cvb_db* db, const uint8_t* d_q, int nq, float thr, float ratio,
                        int32_t* d_match_train, float* d_match_dist, int32_t* d_n_matches, void* stream) {
  if (!ctx || !db) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  if (const int rc = require_kind(ctx, db, true, "cvb_db_match_l2_dev")) return rc;
  const int n_seg = (int)db->seg_ptr.size() - 1;
  CVB_REQUIRE(ctx, nq >= 0 && (nq == 0 || d_q) && (n_seg == 0 || d_n_matches), "cvb_db_match_l2_dev: bad arguments");
  if (n_seg == 0) return CVB_OK;
  return match_dev(ctx, db, d_q, nq, thr, ratio, d_match_train, d_match_dist, d_n_matches, stream);
}

int cvb_db_match_l2(cvb_ctx* ctx, cvb_db* db, const float* q, int nq, float thr, float ratio,
                    int32_t* n_matches, int32_t* m_kf, int32_t* m_query, int32_t* m_train, float* m_dist,
                    int cap, int32_t* n_total) {
  if (!ctx || !db) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  if (const int rc = require_kind(ctx, db, true, "cvb_db_match_l2")) return rc;
  return match_host(ctx, db, q, nq, thr, ratio, n_matches, m_kf, m_query, m_train, m_dist, cap, n_total, "cvb_db_match_l2");
}

// src's rows and operand tiles are copied behind dst's: an operand tile is a function of its keyframe's rows alone (the
// key's column is the row within the tile, expand_tiles_kernel), so the copies equal what appending the rows would expand
int cvb_db_merge(cvb_ctx* ctx, cvb_db* dst, const cvb_db* src) {
  if (!ctx || !dst || !src) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  CVB_REQUIRE(ctx, dst != src, "cvb_db_merge: dst and src are the same database");
  CVB_REQUIRE(ctx, dst->desc_bytes == src->desc_bytes, "cvb_db_merge: dst holds %s descriptors, src %s", dst->desc_bytes == 128 ? "SIFT" : "ORB",
              src->desc_bytes == 128 ? "SIFT" : "ORB");
  if (dst->owner != ctx || src->owner != ctx)
    return cvb_fail(ctx, CVB_ERR_UNSUPPORTED, "cvb_db_merge: the %s database was created on another context (device %d); merge databases of one "
                    "context", dst->owner != ctx ? "dst" : "src", (dst->owner != ctx ? dst->owner : src->owner)->device);
  const int64_t have = dst->seg_ptr.back(), add = src->seg_ptr.back();
  CVB_REQUIRE(ctx, have + add < (int64_t)1 << 31, "cvb_db_merge: more than 2^31 rows");
  if ((size_t)(have + add) > dst->cap_rows) {
    const int rc = cvb_db_reserve(ctx, dst, std::max<int64_t>(have + add, (int64_t)(dst->cap_rows * 3 / 2)));
    if (rc) return rc;
  }
  const int tile_old = dst->seg_tile.back(), tiles = src->seg_tile.back();
  if (const int rc = reserve_tiles(ctx, dst, (size_t)tile_old + tiles, (size_t)tile_old)) return rc;
  cudaStream_t st = ctx->stream;
  if (add)
    CVB_CUDA(ctx, cudaMemcpyAsync(dst->d_rows + (size_t)have * dst->desc_bytes, src->d_rows, (size_t)add * dst->desc_bytes,
                                  cudaMemcpyDeviceToDevice, st));
  const size_t tb = cvb_tc::tile_bytes(dst->metric());
  if (tiles) CVB_CUDA(ctx, cudaMemcpyAsync(dst->d_xt + (size_t)tile_old * tb, src->d_xt, (size_t)tiles * tb, cudaMemcpyDeviceToDevice, st));
  for (size_t i = 1; i < src->seg_ptr.size(); i++) {
    dst->seg_ptr.push_back((int32_t)have + src->seg_ptr[i]);
    dst->seg_tile.push_back(tile_old + src->seg_tile[i]);
  }
  dst->seg_dirty = true;
  CVB_CUDA(ctx, cudaStreamSynchronize(st));
  return CVB_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// The database over a rank group
// ---------------------------------------------------------------------------------------------------------------------
struct cvb_db_group {
  cvb_group* g = nullptr;
  int desc_bytes = 32;
  cvb_db* db[CVB_GROUP_MAX] = {};         // rank r's keyframes, in global order
  int64_t rows[CVB_GROUP_MAX] = {};
  std::vector<int2> loc;                  // global keyframe -> (rank, index in the rank's cvb_db)
  bool loc_dirty = true;
  cudaEvent_t done[CVB_GROUP_MAX] = {};   // rank r's part of a request is complete
  // rank 0: the device copy of `loc` and the gather's buffers
  cvb_buf d_loc, cnt, src, goff, o_kf, o_q, o_t, o_d;
};

namespace {

// per rank: the request's per-keyframe counts, their exclusive offsets (db_offsets_kernel) and the compacted lists
// (db_compact_kernel), in the rank's cvb_db scratch
struct DbGatherSrc {
  const int32_t* nm[CVB_GROUP_MAX];
  const int32_t* off[CVB_GROUP_MAX];
  const int32_t* q[CVB_GROUP_MAX];
  const int32_t* t[CVB_GROUP_MAX];
  const float* d[CVB_GROUP_MAX];
};

// The gather, part 1: every global keyframe's count and the start of its slice in its rank's list.  The counts are then
// scanned in global keyframe order by db_offsets_kernel.  __grid_constant__: the pointer table is indexed in place in the
// parameter bank (as group_sum_kernel's).
__global__ void __launch_bounds__(256) db_group_counts_kernel(const __grid_constant__ DbGatherSrc s, const int2* __restrict__ loc,
                                                               int n_kf, int32_t* __restrict__ cnt, int32_t* __restrict__ src) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_kf) return;
  const int2 rl = loc[i];
  cnt[i] = s.nm[rl.x][rl.y];
  src[i] = s.off[rl.x][rl.y];
}

// The gather, part 2: one warp per global keyframe copies its slice of its rank's list to its global position goff[kf],
// m_kf rewritten to the global index.  As db_compact_kernel, a match is written iff its global position p < cap.  The ranks
// compacted with the same cap, and nothing below cap is lost by that: a rank's earlier keyframes are a subset of the
// globally earlier ones, in the same order, so a match's position in its rank's list is never larger than its global
// position p (src[kf] + j <= goff[kf] + j < cap).
__global__ void __launch_bounds__(256) db_group_gather_kernel(const __grid_constant__ DbGatherSrc s, const int2* __restrict__ loc,
                                                               const int32_t* __restrict__ cnt, const int32_t* __restrict__ src,
                                                               const int32_t* __restrict__ goff, int n_kf, int cap,
                                                               int32_t* __restrict__ o_kf, int32_t* __restrict__ o_q,
                                                               int32_t* __restrict__ o_t, float* __restrict__ o_d) {
  const int kf = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (kf >= n_kf) return;
  const int r = loc[kf].x, n = cnt[kf], p0 = goff[kf], s0 = src[kf];
  for (int j = threadIdx.x & 31; j < n && p0 + j < cap; j += 32) {
    const int p = p0 + j, ps = s0 + j;
    o_kf[p] = kf;
    o_q[p] = s.q[r][ps];
    o_t[p] = s.t[r][ps];
    o_d[p] = s.d[r][ps];
  }
}

// a failure of rank r's work, reported on rank 0's context as the group drivers do
int rank_fail(cvb_db_group* db, int r, int rc) {
  const std::string m = db->g->ctx[r]->err;
  return cvb_fail(db->g->ctx[0], rc, "rank %d: %s", r, m.c_str());
}

// no rank's stream still works on the request (the error path; the normal path ends in rank 0's synchronise, after the
// gather that waited on every rank)
void settle(cvb_db_group* db) {
  for (int r = 0; r < db->g->n; r++) {
    CVB_GUARD(db->g->ctx[r]);
    cudaStreamSynchronize(db->g->ctx[r]->stream);
  }
}

// Each keyframe to the rank holding the fewest rows at that moment (the lowest rank on a tie), one by one; rank r's
// keyframes are appended to its cvb_db in their global order.  rows: u8, the database layout (host).
int group_append(cvb_db_group* db, const uint8_t* rows, const int32_t* rows_per_kf, int n_kf) {
  cvb_group* g = db->g;
  const int n = g->n;
  std::vector<int> dest((size_t)n_kf);
  int64_t load[CVB_GROUP_MAX];
  std::copy(db->rows, db->rows + n, load);
  for (int i = 0; i < n_kf; i++) {
    const int r = (int)(std::min_element(load, load + n) - load);
    dest[i] = r;
    load[r] += rows_per_kf[i];
  }
  std::vector<int64_t> first((size_t)n_kf + 1, 0);
  for (int i = 0; i < n_kf; i++) first[i + 1] = first[i] + rows_per_kf[i];
  int base[CVB_GROUP_MAX];
  for (int r = 0; r < n; r++) {
    base[r] = (int)db->db[r]->seg_ptr.size() - 1;
    std::vector<uint8_t> buf;
    std::vector<int32_t> cnt;
    for (int i = 0; i < n_kf; i++)
      if (dest[i] == r) {
        buf.insert(buf.end(), rows + first[i] * db->desc_bytes, rows + first[i + 1] * db->desc_bytes);
        cnt.push_back(rows_per_kf[i]);
      }
    if (cnt.empty()) continue;
    CVB_GUARD(g->ctx[r]);
    if (const int rc = append_rows(g->ctx[r], db->db[r], buf.data(), cnt.data(), (int)cnt.size(), (int64_t)buf.size() / db->desc_bytes))
      return rank_fail(db, r, rc);
    db->rows[r] = load[r];
  }
  for (int i = 0; i < n_kf; i++) db->loc.push_back(make_int2(dest[i], base[dest[i]]++));
  db->loc_dirty = true;
  return CVB_OK;
}

int group_append_checked(cvb_db_group* db, bool sift, const void* rows, const int32_t* rows_per_kf, int n_kf, const char* fn) {
  cvb_ctx* c0 = db->g->ctx[0];
  if (const int rc = require_kind(c0, db->db[0], sift, fn)) return rc;   // every rank's cvb_db holds the group's row kind
  CVB_REQUIRE(c0, n_kf >= 0 && (n_kf == 0 || rows_per_kf), "%s: bad arguments", fn);
  int64_t add = 0, have = 0;
  for (int i = 0; i < n_kf; ++i) {
    CVB_REQUIRE(c0, rows_per_kf[i] >= 0, "%s: negative row count", fn);
    add += rows_per_kf[i];
  }
  for (int r = 0; r < db->g->n; r++) have += db->rows[r];
  // the single database's limit, so that the group refuses what one cvb_db would refuse
  CVB_REQUIRE(c0, have + add < (int64_t)1 << 31, "%s: more than 2^31 rows", fn);
  CVB_REQUIRE(c0, add == 0 || rows, "%s: null rows", fn);
  if (!sift) return group_append(db, (const uint8_t*)rows, rows_per_kf, n_kf);
  std::vector<uint8_t> u8((size_t)add * 128);   // checked and quantised before any rank is touched
  if (!cvb_quantize_sift((const float*)rows, u8.size(), u8.data()))
    return cvb_fail(c0, CVB_ERR_UNSUPPORTED, "%s: SIFT descriptors must be integer-valued in [0,255] (cv::xfeatures2d::SIFT output)", fn);
  return group_append(db, u8.data(), rows_per_kf, n_kf);
}

// rank r's part of a request, enqueued on its stream: the query from the pinned staging, the filtered 2-NN against its
// keyframes, the scan of its counts and the compaction (at most cap), then its event
int rank_request(cvb_ctx* ctx, cvb_db* d, const uint8_t* pin, size_t qb, int nq, float thr, float ratio, int cap, cudaEvent_t done) {
  CVB_GUARD(ctx);
  const int n_seg = (int)d->seg_ptr.size() - 1;
  const size_t on = (size_t)n_seg * nq;
  cudaStream_t st = ctx->stream;
  int rc;
  if ((rc = grow(ctx, d->q, qb)) || (rc = grow(ctx, d->mt, on * 4)) || (rc = grow(ctx, d->md, on * 4)) ||
      (rc = grow(ctx, d->nm, (size_t)n_seg * 4)) || (rc = grow(ctx, d->off, (size_t)(n_seg + 1) * 4)))
    return rc;
  if (cap && ((rc = grow(ctx, d->out_seg, (size_t)cap * 4)) || (rc = grow(ctx, d->out_q, (size_t)cap * 4)) ||
              (rc = grow(ctx, d->out_t, (size_t)cap * 4)) || (rc = grow(ctx, d->out_d, (size_t)cap * 4))))
    return rc;
  CVB_CUDA(ctx, cudaMemcpyAsync(d->q.p, pin, qb, cudaMemcpyHostToDevice, st));
  if ((rc = match_dev(ctx, d, (const uint8_t*)d->q.p, nq, thr, ratio, (int32_t*)d->mt.p, (float*)d->md.p, (int32_t*)d->nm.p, nullptr)))
    return rc;
  db_offsets_kernel<<<1, 1024, 0, st>>>((const int32_t*)d->nm.p, n_seg, (int32_t*)d->off.p);
  CVB_CHECK_LAUNCH(ctx);
  if (cap) {
    db_compact_kernel<<<(n_seg + 7) / 8, 256, 0, st>>>((const int32_t*)d->mt.p, (const float*)d->md.p, nq, n_seg, (const int32_t*)d->off.p,
                                                       cap, (int32_t*)d->out_seg.p, (int32_t*)d->out_q.p, (int32_t*)d->out_t.p,
                                                       (float*)d->out_d.p);
    CVB_CHECK_LAUNCH(ctx);
  }
  CVB_CUDA(ctx, cudaEventRecord(done, st));
  return CVB_OK;
}

// everything after the checks: *fail_rank = the rank whose work failed
int group_request(cvb_db_group* db, const uint8_t* pin, size_t pin_q, int nq, float thr, float ratio, int32_t* n_matches,
                  int32_t* m_kf, int32_t* m_query, int32_t* m_train, float* m_dist, int cap, int32_t* n_total, int* fail_rank) {
  cvb_group* g = db->g;
  cvb_ctx* c0 = g->ctx[0];
  cudaStream_t st = c0->stream;
  const int n_kf = (int)db->loc.size();
  const size_t qb = (size_t)nq * db->desc_bytes;
  int rc;
  *fail_rank = 0;
  // rank 0's buffers first: the table upload synchronises rank 0's stream, before any rank's work is enqueued
  if ((rc = grow(c0, db->d_loc, (size_t)n_kf * sizeof(int2))) || (rc = grow(c0, db->cnt, (size_t)n_kf * 4)) ||
      (rc = grow(c0, db->src, (size_t)n_kf * 4)) || (rc = grow(c0, db->goff, (size_t)(n_kf + 1) * 4)))
    return rc;
  if (cap && ((rc = grow(c0, db->o_kf, (size_t)cap * 4)) || (rc = grow(c0, db->o_q, (size_t)cap * 4)) ||
              (rc = grow(c0, db->o_t, (size_t)cap * 4)) || (rc = grow(c0, db->o_d, (size_t)cap * 4))))
    return rc;
  if (db->loc_dirty) {
    CVB_CUDA(c0, cudaMemcpyAsync(db->d_loc.p, db->loc.data(), (size_t)n_kf * sizeof(int2), cudaMemcpyHostToDevice, st));
    CVB_CUDA(c0, cudaStreamSynchronize(st));
    db->loc_dirty = false;
  }
  DbGatherSrc s{};
  bool ran[CVB_GROUP_MAX] = {};
  for (int r = 0; r < g->n; r++) {
    cvb_db* d = db->db[r];
    if (d->seg_ptr.size() == 1) continue;   // a rank without keyframes has no part in the request
    if ((rc = rank_request(g->ctx[r], d, pin, qb, nq, thr, ratio, cap, db->done[r]))) {
      *fail_rank = r;
      return rc;
    }
    s.nm[r] = (const int32_t*)d->nm.p;
    s.off[r] = (const int32_t*)d->off.p;
    s.q[r] = (const int32_t*)d->out_q.p;
    s.t[r] = (const int32_t*)d->out_t.p;
    s.d[r] = (const float*)d->out_d.p;
    ran[r] = true;
  }
  for (int r = 1; r < g->n; r++)
    if (ran[r]) CVB_CUDA(c0, cudaStreamWaitEvent(st, db->done[r], 0));
  const int2* loc = (const int2*)db->d_loc.p;
  int32_t *cnt = (int32_t*)db->cnt.p, *src = (int32_t*)db->src.p, *goff = (int32_t*)db->goff.p;
  db_group_counts_kernel<<<(n_kf + 255) / 256, 256, 0, st>>>(s, loc, n_kf, cnt, src);
  CVB_CHECK_LAUNCH(c0);
  db_offsets_kernel<<<1, 1024, 0, st>>>(cnt, n_kf, goff);
  CVB_CHECK_LAUNCH(c0);
  if (cap) {
    db_group_gather_kernel<<<(n_kf + 7) / 8, 256, 0, st>>>(s, loc, cnt, src, goff, n_kf, cap, (int32_t*)db->o_kf.p,
                                                           (int32_t*)db->o_q.p, (int32_t*)db->o_t.p, (float*)db->o_d.p);
    CVB_CHECK_LAUNCH(c0);
  }
  int32_t* pin_cnt = (int32_t*)(pin + pin_q);
  int32_t* pin_tot = pin_cnt + n_kf;
  CVB_CUDA(c0, cudaMemcpyAsync(pin_cnt, cnt, (size_t)n_kf * 4, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(c0, cudaMemcpyAsync(pin_tot, goff + n_kf, 4, cudaMemcpyDeviceToHost, st));
  CVB_CUDA(c0, cudaStreamSynchronize(st));
  const int total = *pin_tot;
  *n_total = total;
  if (n_matches) memcpy(n_matches, pin_cnt, (size_t)n_kf * 4);
  const int n_out = std::min(total, cap);
  if (n_out) {
    CVB_CUDA(c0, cudaMemcpyAsync(m_kf, db->o_kf.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(c0, cudaMemcpyAsync(m_query, db->o_q.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(c0, cudaMemcpyAsync(m_train, db->o_t.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(c0, cudaMemcpyAsync(m_dist, db->o_d.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    CVB_CUDA(c0, cudaStreamSynchronize(st));
  }
  return CVB_OK;
}

int group_match(cvb_db_group* db, bool sift, const void* q, int nq, float thr, float ratio, int32_t* n_matches, int32_t* m_kf,
                int32_t* m_query, int32_t* m_train, float* m_dist, int cap, int32_t* n_total, const char* fn) {
  cvb_ctx* c0 = db->g->ctx[0];
  if (const int rc = require_kind(c0, db->db[0], sift, fn)) return rc;
  const int n_kf = (int)db->loc.size();
  CVB_REQUIRE(c0, nq >= 0 && cap >= 0 && n_total && (nq == 0 || q), "%s: bad arguments", fn);
  CVB_REQUIRE(c0, cap == 0 || (m_kf && m_query && m_train && m_dist), "%s: null outputs", fn);
  *n_total = 0;
  // pinned staging on rank 0's context: [query | counts | total]; every rank copies the query from it
  const size_t qb = (size_t)nq * db->desc_bytes, pin_q = (qb + 255) & ~(size_t)255;
  uint8_t* pin = (uint8_t*)cvb_pinned(c0, pin_q + (size_t)(n_kf + 1) * 4 + 64);
  if (!pin) return CVB_ERR_CUDA;
  if (!sift) memcpy(pin, q, qb);
  else if (!cvb_quantize_sift((const float*)q, qb, pin))
    return cvb_fail(c0, CVB_ERR_UNSUPPORTED, "%s: SIFT descriptors must be integer-valued in [0,255] (cv::xfeatures2d::SIFT output)", fn);
  if (n_kf == 0) return CVB_OK;
  if (nq == 0) {
    if (n_matches) std::fill(n_matches, n_matches + n_kf, 0);
    return CVB_OK;
  }
  int r = 0;
  const int rc = group_request(db, pin, pin_q, nq, thr, ratio, n_matches, m_kf, m_query, m_train, m_dist, cap, n_total, &r);
  if (!rc) return CVB_OK;
  settle(db);
  *n_total = 0;
  return rank_fail(db, r, rc);
}

// The removals dealt to the ranks holding them; every rank that loses keyframes compacts its share on its own stream (all
// enqueued first, then each stream waited for), and the global table is rebuilt once.  A rank keeps its keyframes in global
// order, so a survivor's new local index is its rank in that order.
int group_remove(cvb_db_group* db, const int32_t* kf_index, int n, const char* fn) {
  cvb_group* g = db->g;
  std::vector<char> gone;
  int rc = check_removals(g->ctx[0], kf_index, n, (int)db->loc.size(), fn, gone);
  if (rc || n == 0) return rc;
  std::vector<char> rgone[CVB_GROUP_MAX];
  bool loses[CVB_GROUP_MAX] = {};
  for (int r = 0; r < g->n; r++) rgone[r].assign(db->db[r]->seg_ptr.size() - 1, 0);
  for (size_t i = 0; i < gone.size(); i++)
    if (gone[i]) {
      rgone[db->loc[i].x][db->loc[i].y] = 1;
      loses[db->loc[i].x] = true;
    }
  std::unique_ptr<cvb_block> stage[CVB_GROUP_MAX];
  int fail = 0;
  for (int r = 0; r < g->n && !rc; r++) {
    if (!loses[r]) continue;
    CVB_GUARD(g->ctx[r]);
    cvb_db* d = db->db[r];
    const int64_t before = d->seg_ptr.back();
    if ((rc = compact(g->ctx[r], d, rgone[r], stage[r]))) fail = r;
    db->rows[r] -= before - d->seg_ptr.back();
  }
  for (int r = 0; r < g->n; r++) {
    if (!stage[r]) continue;
    CVB_GUARD(g->ctx[r]);
    const cudaError_t e = cudaStreamSynchronize(g->ctx[r]->stream);
    if (!rc && e != cudaSuccess) {
      rc = cvb_fail(g->ctx[r], CVB_ERR_CUDA, "%s: cudaStreamSynchronize failed: %s", fn, cudaGetErrorString(e));
      fail = r;
    }
    stage[r].reset();
  }
  if (rc) return rank_fail(db, fail, rc);
  int next[CVB_GROUP_MAX] = {};
  size_t w = 0;
  for (size_t i = 0; i < gone.size(); i++)
    if (!gone[i]) db->loc[w++] = make_int2(db->loc[i].x, next[db->loc[i].x]++);
  db->loc.resize(w);
  db->loc_dirty = true;
  return CVB_OK;
}

}  // namespace

extern "C" {

int cvb_db_group_create(cvb_group* g, int desc_bytes, cvb_db_group** out) {
  if (!g || !out) return CVB_ERR_INVALID;
  *out = nullptr;
  std::lock_guard<std::recursive_mutex> lk(g->call_mtx);
  cvb_ctx* c0 = g->ctx[0];
  if (desc_bytes != 32 && desc_bytes != 128)
    return cvb_fail(c0, CVB_ERR_UNSUPPORTED, "descriptor database: 32-byte ORB or 128-byte SIFT descriptors, got %d", desc_bytes);
  cvb_db_group* db = new cvb_db_group();
  db->g = g;
  db->desc_bytes = desc_bytes;
  int rc = CVB_OK;
  for (int r = 0; r < g->n && !rc; r++) {
    if ((rc = cvb_db_create(g->ctx[r], desc_bytes, &db->db[r]))) {
      rc = rank_fail(db, r, rc);
      break;
    }
    CVB_GUARD(g->ctx[r]);
    const cudaError_t e = cudaEventCreateWithFlags(&db->done[r], cudaEventDisableTiming);
    if (e != cudaSuccess) rc = cvb_fail(c0, CVB_ERR_CUDA, "cvb_db_group_create: rank %d: %s", r, cudaGetErrorString(e));
  }
  if (rc) {
    cvb_db_group_destroy(db);
    return rc;
  }
  *out = db;
  return CVB_OK;
}

int cvb_db_group_destroy(cvb_db_group* db) {
  if (!db) return CVB_OK;
  cvb_group* g = db->g;
  std::lock_guard<std::recursive_mutex> lk(g->call_mtx);
  for (int r = 0; r < g->n; r++) {
    CVB_GUARD(g->ctx[r]);
    if (db->db[r]) cvb_db_destroy(g->ctx[r], db->db[r]);
    if (db->done[r]) cudaEventDestroy(db->done[r]);
  }
  {
    CVB_GUARD(g->ctx[0]);
    for (cvb_buf* b : {&db->d_loc, &db->cnt, &db->src, &db->goff, &db->o_kf, &db->o_q, &db->o_t, &db->o_d})
      if (b->p) cudaFree(b->p);
  }
  delete db;
  return CVB_OK;
}

int cvb_db_group_append(cvb_db_group* db, const uint8_t* rows, const int32_t* rows_per_kf, int n_kf) {
  if (!db) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> lk(db->g->call_mtx);
  return group_append_checked(db, false, rows, rows_per_kf, n_kf, "cvb_db_group_append");
}

int cvb_db_group_append_sift(cvb_db_group* db, const float* rows, const int32_t* rows_per_kf, int n_kf) {
  if (!db) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> lk(db->g->call_mtx);
  return group_append_checked(db, true, rows, rows_per_kf, n_kf, "cvb_db_group_append_sift");
}

int cvb_db_group_remove(cvb_db_group* db, int kf_index) {
  if (!db) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> lk(db->g->call_mtx);
  const int32_t k = kf_index;
  return group_remove(db, &k, 1, "cvb_db_group_remove");
}

int cvb_db_group_remove_batch(cvb_db_group* db, const int32_t* kf_index, int n) {
  if (!db) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> lk(db->g->call_mtx);
  return group_remove(db, kf_index, n, "cvb_db_group_remove_batch");
}

int cvb_db_group_size(const cvb_db_group* db, int32_t* n_kf, int64_t* n_rows, int64_t* rows_per_rank) {
  if (!db) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> lk(db->g->call_mtx);
  int64_t all = 0;
  for (int r = 0; r < db->g->n; r++) {
    all += db->rows[r];
    if (rows_per_rank) rows_per_rank[r] = db->rows[r];
  }
  if (n_kf) *n_kf = (int32_t)db->loc.size();
  if (n_rows) *n_rows = all;
  return CVB_OK;
}

int cvb_db_group_match_hamming(cvb_db_group* db, const uint8_t* q, int nq, float thr, float ratio, int32_t* n_matches,
                               int32_t* m_kf, int32_t* m_query, int32_t* m_train, float* m_dist, int cap, int32_t* n_total) {
  if (!db) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> lk(db->g->call_mtx);
  CVB_GUARD(db->g->ctx[0]);
  return group_match(db, false, q, nq, thr, ratio, n_matches, m_kf, m_query, m_train, m_dist, cap, n_total, "cvb_db_group_match_hamming");
}

int cvb_db_group_match_l2(cvb_db_group* db, const float* q, int nq, float thr, float ratio, int32_t* n_matches, int32_t* m_kf,
                          int32_t* m_query, int32_t* m_train, float* m_dist, int cap, int32_t* n_total) {
  if (!db) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> lk(db->g->call_mtx);
  CVB_GUARD(db->g->ctx[0]);
  return group_match(db, true, q, nq, thr, ratio, n_matches, m_kf, m_query, m_train, m_dist, cap, n_total, "cvb_db_group_match_l2");
}

// Rank r's share of src follows its share of dst, so every rank still holds its keyframes in global order
int cvb_db_group_merge(cvb_db_group* dst, const cvb_db_group* src) {
  if (!dst || !src) return CVB_ERR_INVALID;
  std::lock_guard<std::recursive_mutex> lk(dst->g->call_mtx);
  cvb_group* g = dst->g;
  cvb_ctx* c0 = g->ctx[0];
  CVB_REQUIRE(c0, dst != src, "cvb_db_group_merge: dst and src are the same database");
  CVB_REQUIRE(c0, dst->desc_bytes == src->desc_bytes, "cvb_db_group_merge: dst holds %s descriptors, src %s",
              dst->desc_bytes == 128 ? "SIFT" : "ORB", src->desc_bytes == 128 ? "SIFT" : "ORB");
  if (src->g != g) return cvb_fail(c0, CVB_ERR_UNSUPPORTED, "cvb_db_group_merge: src is on another group; merge databases of one group");
  int64_t all = 0;
  for (int r = 0; r < g->n; r++) all += dst->rows[r] + src->rows[r];
  CVB_REQUIRE(c0, all < (int64_t)1 << 31, "cvb_db_group_merge: more than 2^31 rows");
  int base[CVB_GROUP_MAX];
  for (int r = 0; r < g->n; r++) {
    base[r] = (int)dst->db[r]->seg_ptr.size() - 1;
    if (src->db[r]->seg_ptr.size() == 1) continue;
    if (const int rc = cvb_db_merge(g->ctx[r], dst->db[r], src->db[r])) return rank_fail(dst, r, rc);
    dst->rows[r] += src->rows[r];
  }
  for (const int2 rl : src->loc) dst->loc.push_back(make_int2(rl.x, base[rl.x] + rl.y));
  dst->loc_dirty = true;
  return CVB_OK;
}

}  // extern "C"
