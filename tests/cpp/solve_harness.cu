// GPU harness for tests/test_cholesky_solve.py: factors a host matrix with the tiled Cholesky (covins_b200/csrc/cholesky.cu,
// compiled into this translation unit) once, then runs the triangular solves (solve_grid, the launch helper behind
// solve()) with several grid sizes and repeatedly with one FactorStreams.
//   usage: solve_harness in.bin out.bin
// Both files are a sequence of arrays, each an int64 byte count followed by the raw values (int32 or float64, row-major).
//   in:  {nt, n, reps, plan (0 blocked, 1 col_group)}, mask[nt*nt], col_group[nt], A[n*n], b[n], grids[]
//   out: flag, then x[nt*T] per grid size (in the order given; 0 = as many CTAs as fit on the device), then x[nt*T] of
//        each of `reps` further solves with grid 0
// The scratch and solution buffers are filled with NaN (all bytes 0xFF) before every solve, as a reused workspace would
// hold stale values.  Every CUDA error is reported on stderr and makes the exit code non-zero.
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../covins_b200/csrc/cholesky.cu"

// the library's error helper (defined in ctx.cu, which is not part of this harness)
int cvb_fail(cvb_ctx*, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vfprintf(stderr, fmt, ap);
  va_end(ap);
  fputc('\n', stderr);
  return code;
}

using namespace cvb_chol;

#define CK(call)                                                                                         \
  do {                                                                                                   \
    cudaError_t e_ = (call);                                                                             \
    if (e_ != cudaSuccess) {                                                                             \
      fprintf(stderr, "%s failed: %s (%s:%d)\n", #call, cudaGetErrorString(e_), __FILE__, __LINE__);    \
      exit(3);                                                                                           \
    }                                                                                                    \
  } while (0)

template <class V>
static std::vector<V> get(FILE* f) {
  int64_t nb = 0;
  if (fread(&nb, 8, 1, f) != 1 || nb < 0 || nb % (int64_t)sizeof(V)) {
    fprintf(stderr, "malformed input\n");
    exit(2);
  }
  std::vector<V> v((size_t)nb / sizeof(V));
  if (nb && fread(v.data(), 1, (size_t)nb, f) != (size_t)nb) {
    fprintf(stderr, "short input\n");
    exit(2);
  }
  return v;
}
static void put(FILE* f, const void* p, size_t bytes) {
  const int64_t nb = (int64_t)bytes;
  fwrite(&nb, 8, 1, f);
  if (bytes) fwrite(p, 1, bytes, f);
}

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]);
    return 2;
  }
  FILE* fin = fopen(argv[1], "rb");
  if (!fin) return 2;
  const auto hdr = get<int32_t>(fin);
  const auto m32 = get<int32_t>(fin), group = get<int32_t>(fin);
  const auto A = get<double>(fin), b = get<double>(fin);
  const auto grids = get<int32_t>(fin);
  fclose(fin);
  const int nt = hdr[0], n = hdr[1], reps = hdr[2], np = nt * T;
  if ((int)m32.size() != nt * nt || (int)group.size() != nt || A.size() != (size_t)n * n || (int)b.size() != n || n > np) {
    fprintf(stderr, "inconsistent input\n");
    return 2;
  }
  cvb_ctx ctx;
  ctx.device = 0;
  CK(cudaSetDevice(0));
  CK(cudaStreamCreateWithFlags(&ctx.stream, cudaStreamNonBlocking));
  cudaStream_t st = ctx.stream;
  CK(cudaFuncSetAttribute(trsm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrsmSmem));
  CK(cudaFuncSetAttribute(syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSyrkSmem));
  CK(cudaFuncSetAttribute(tile_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTileSmem));
  CK(cudaFuncSetAttribute(potrf_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPotrfSmem));
  CK(cudaFuncSetAttribute(chain_gemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kChainSmem));
  CK(cudaFuncSetAttribute(chain_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kChainSmem));
  TilePlan plan;
  if (hdr[3] == 0) plan.build(nt, std::vector<uint8_t>(m32.begin(), m32.end()));
  else plan.build(nt, std::vector<uint8_t>(m32.begin(), m32.end()), std::vector<int>(group.begin(), group.end()));
  if (plan.upload(&ctx, st)) return 3;
  FactorStreams fs;
  if (fs.create(&ctx, nt)) return 3;
  const size_t nL = (size_t)plan.n_tiles_L * TT;
  std::vector<double> hs(nL, 0.0), hb(np, 0.0), x(np);
  for (int i = 0; i < n; i++)
    for (int j = 0; j <= i; j++)
      if (A[(size_t)i * n + j] != 0.0) {
        const int t = plan.h_tile_of[(size_t)(i / T) * nt + (j / T)];
        if (t < 0) {
          fprintf(stderr, "A(%d,%d) lies outside the tile mask\n", i, j);
          return 2;
        }
        hs[(size_t)t * TT + (size_t)(i % T) * T + (j % T)] = A[(size_t)i * n + j];
      }
  for (int i = n; i < np; i++) hs[plan.tile_index(i / T, i / T) * TT + (size_t)(i % T) * T + (i % T)] = 1.0;
  for (int i = 0; i < n; i++) hb[i] = b[i];
  double *dS = nullptr, *dl = nullptr, *dv = nullptr;
  int* dflag = nullptr;
  CK(cudaMalloc(&dS, nL * 8));
  CK(cudaMalloc(&dl, (size_t)nt * TT * 8));
  CK(cudaMalloc(&dv, (size_t)np * 3 * 8));
  CK(cudaMalloc(&dflag, 4));
  CK(cudaMemcpyAsync(dS, hs.data(), nL * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(dv, hb.data(), (size_t)np * 8, cudaMemcpyHostToDevice, st));
  if (factor(&ctx, dS, dl, dflag, plan, st, fs, nullptr)) return 3;
  int flag = 0;
  CK(cudaMemcpyAsync(&flag, dflag, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::vector<std::vector<char>> out;
  out.emplace_back((const char*)&flag, (const char*)&flag + 4);
  auto run = [&](int grid) {
    CK(cudaMemsetAsync(dv + np, 0xFF, (size_t)np * 2 * 8, st));
    if (solve_grid(&ctx, dS, dl, dv, dv + np, dv + 2 * np, plan, st, fs, grid)) exit(3);
    CK(cudaMemcpyAsync(x.data(), dv + 2 * (size_t)np, (size_t)np * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    out.emplace_back((const char*)x.data(), (const char*)(x.data() + np));
  };
  for (int g : grids) run(g);
  for (int r = 0; r < reps; r++) run(0);
  CK(cudaDeviceSynchronize());
  fs.destroy();
  plan.release();
  FILE* f = fopen(argv[2], "wb");
  if (!f) return 2;
  for (const auto& v : out) put(f, v.data(), v.size());
  fclose(f);
  return 0;
}
