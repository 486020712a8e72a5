// Standalone timing of the Cholesky's bulk trailing update (tools/tile_update_bench.py builds and runs this).
// cholesky.cu is compiled into this translation unit, as tests/cpp/chol_harness.cu does; CHOLESKY_CU names the source, so
// two builds of the kernel can be timed side by side.
//   usage: tile_update_bench <reps>
// A dense pose part of NT = 94 tile columns (the lower triangle, 4465 tiles, 585 MB) is filled with a fixed pattern.  Each
// pass is one tile_update_kernel launch over the targets (i, j), nt > i >= j >= m0, with the 4 panels m0 - 4 .. m0 - 1,
// in the order TilePlan::build lists a bulk pass (column j ascending, then row i):
//   first  m0 = 4:  the first bulk pass, 4095 targets;
//   mid    m0 = 47: a pass half way through, 1128 targets.
// Every pass is timed with CUDA events around the launch alone, L2-warm (back-to-back launches) and cold (a 256 MB buffer
// written between launches), and so is a register-only DMMA probe with the same grid, warps and DMMA count per warp.
// One JSON line per measurement: median and best of <reps> launches.  Also printed: a hash of the tile array after one
// launch of each pass from the fixed pattern, to compare builds bit for bit.
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <vector>

#ifndef CHOLESKY_CU
#define CHOLESKY_CU "../covins_b200/csrc/cholesky.cu"
#endif
#include CHOLESKY_CU

int cvb_fail(cvb_ctx*, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vfprintf(stderr, fmt, ap);
  va_end(ap);
  fputc('\n', stderr);
  return code;
}

using namespace cvb_chol;

#define CK(call)                                                                                      \
  do {                                                                                                \
    cudaError_t e_ = (call);                                                                          \
    if (e_ != cudaSuccess) {                                                                          \
      fprintf(stderr, "%s failed: %s (%s:%d)\n", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      exit(3);                                                                                        \
    }                                                                                                 \
  } while (0)

constexpr int NT = 94;

// small values of both signs (|x| < 2^-6), so repeated launches stay finite
__global__ void fill_kernel(double* S, size_t n) {
  for (size_t u = blockIdx.x * (size_t)blockDim.x + threadIdx.x; u < n; u += (size_t)gridDim.x * blockDim.x) {
    uint64_t h = (u + 1) * 0x9E3779B97F4A7C15ull;
    h ^= h >> 29;
    h *= 0xBF58476D1CE4E5B9ull;
    h ^= h >> 32;
    S[u] = ((double)(h >> 11) * 0x1p-53 - 0.5) * 0x1p-5;
  }
}

// Register-only DMMA: each warp runs the 16 independent m16n8k16 accumulations of a 64x32 warp tile for `chunks` K chunks,
// as tile_update's consumer warps do, with fragments that never touch memory.
__global__ void __launch_bounds__(256, 1) dmma_probe_kernel(int chunks, double seed, double* out) {
  double acc[4][4][4], a[4][8], b[4][4];
  const double v = seed * (threadIdx.x + 1);
#pragma unroll
  for (int x = 0; x < 4; x++) {
#pragma unroll
    for (int e = 0; e < 8; e++) a[x][e] = v + e;
#pragma unroll
    for (int e = 0; e < 4; e++) b[x][e] = v - e;
#pragma unroll
    for (int y = 0; y < 4; y++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[x][y][e] = 0.0;
  }
#pragma unroll 1
  for (int c = 0; c < chunks; c++)
#pragma unroll
    for (int x = 0; x < 4; x++)
#pragma unroll
      for (int y = 0; y < 4; y++) dmma16816(acc[x][y], a[x], b[y]);
  double s = 0.0;
#pragma unroll
  for (int x = 0; x < 4; x++)
#pragma unroll
    for (int y = 0; y < 4; y++)
#pragma unroll
      for (int e = 0; e < 4; e++) s += acc[x][y][e];
  if (s == 1.0) out[0] = s;   // never true: keeps the DMMAs live
}

static uint64_t fnv(const std::vector<double>& v) {
  uint64_t h = 1469598103934665603ull;
  const uint64_t* p = reinterpret_cast<const uint64_t*>(v.data());
  for (size_t u = 0; u < v.size(); u++) h = (h ^ p[u]) * 1099511628211ull;
  return h;
}

int main(int argc, char** argv) {
  const int reps = argc > 1 ? atoi(argv[1]) : 20;
  if (reps < 1) return 2;
  CK(cudaSetDevice(0));
  cudaStream_t st;
  CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  CK(cudaFuncSetAttribute(tile_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTileSmem));
  std::vector<int> tile_of(NT * NT, -1);
  int n_tiles = 0;
  for (int i = 0; i < NT; i++)
    for (int j = 0; j <= i; j++) tile_of[i * NT + j] = n_tiles++;
  const size_t nS = (size_t)n_tiles * TT;
  double *dS = nullptr, *dout = nullptr;
  char* dflush = nullptr;
  const size_t flush_bytes = (size_t)256 << 20;
  int* d_tile_of = nullptr;
  CK(cudaMalloc(&dS, nS * 8));
  CK(cudaMalloc(&dout, 8));
  CK(cudaMalloc(&dflush, flush_bytes));
  CK(cudaMalloc(&d_tile_of, tile_of.size() * 4));
  CK(cudaMemcpy(d_tile_of, tile_of.data(), tile_of.size() * 4, cudaMemcpyHostToDevice));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  std::vector<double> hS(nS);

  struct Pass {
    const char* name;
    int m0;
  };
  for (const Pass ps : {Pass{"first", 4}, Pass{"mid", 47}}) {
    std::vector<int> pi, pj, pm;
    for (int j = ps.m0; j < NT; j++)
      for (int i = j; i < NT; i++) {
        pi.push_back(i);
        pj.push_back(j);
        pm.push_back(0xF);
      }
    const int np = (int)pi.size(), k0 = ps.m0 - 4;
    int *d_pi, *d_pj, *d_pm;
    CK(cudaMalloc(&d_pi, np * 4));
    CK(cudaMalloc(&d_pj, np * 4));
    CK(cudaMalloc(&d_pm, np * 4));
    CK(cudaMemcpy(d_pi, pi.data(), np * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_pj, pj.data(), np * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_pm, pm.data(), np * 4, cudaMemcpyHostToDevice));
    // flops counted as full tiles (the idle quadrant of the diagonal targets included); bytes: 4 panels x 2 operand tiles
    // read and C read + written, per target
    const double flop = (double)np * 4 * 2.0 * T * T * T, bytes = (double)np * (8 + 2) * TT * 8;

    fill_kernel<<<1056, 256, 0, st>>>(dS, nS);
    tile_update_kernel<<<np, TILE_THREADS, kTileSmem, st>>>(dS, d_tile_of, NT, k0, d_pi, d_pj, d_pm);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(hS.data(), dS, nS * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    printf("{\"pass\": \"%s\", \"targets\": %d, \"hash\": \"%016llx\"}\n", ps.name, np, (unsigned long long)fnv(hS));

    for (int kind = 0; kind < 3; kind++) {   // 0 warm, 1 cold (flushed), 2 register-only probe
      std::vector<float> ms;
      for (int r = -2; r < reps; r++) {   // two untimed launches first
        if (kind == 1) CK(cudaMemsetAsync(dflush, r & 0xFF, flush_bytes, st));
        CK(cudaEventRecord(e0, st));
        if (kind < 2)
          tile_update_kernel<<<np, TILE_THREADS, kTileSmem, st>>>(dS, d_tile_of, NT, k0, d_pi, d_pj, d_pm);
        else
          dmma_probe_kernel<<<np, 256, 0, st>>>(4 * T / KC, 1e-3, dout);
        CK(cudaGetLastError());
        CK(cudaEventRecord(e1, st));
        CK(cudaEventSynchronize(e1));
        float t = 0.f;
        CK(cudaEventElapsedTime(&t, e0, e1));
        if (r >= 0) ms.push_back(t);
      }
      std::sort(ms.begin(), ms.end());
      const double med = ms[ms.size() / 2], best = ms[0];
      printf("{\"pass\": \"%s\", \"kernel\": \"%s\", \"targets\": %d, \"gflop\": %.2f, \"gbytes\": %.2f, \"ms_median\": %.4f, "
             "\"ms_best\": %.4f, \"tflops_median\": %.2f, \"tbytes_per_s_median\": %.2f}\n",
             ps.name, kind == 0 ? "tile_update_warm" : kind == 1 ? "tile_update_cold" : "dmma_probe", np, flop * 1e-9,
             bytes * 1e-9, med, best, flop / med * 1e-9, kind == 2 ? 0.0 : bytes / med * 1e-9);
    }
    CK(cudaFree(d_pi));
    CK(cudaFree(d_pj));
    CK(cudaFree(d_pm));
  }
  CK(cudaDeviceSynchronize());
  return 0;
}
