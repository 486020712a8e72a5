// GPU harness for tests/test_cholesky_kernels.py: runs the tiled Cholesky's kernels (covins_b200/csrc/cholesky.cu, compiled
// into this translation unit) one launch at a time on host-supplied tiles, or the whole factor + solve on a host matrix.
//   usage: chol_harness <mode> in.bin out.bin
// Both files are a sequence of arrays, each an int64 byte count followed by the raw values (int32 or float64, row-major).
//   update   in: {nt, k0, kernel (0 tile_update_kernel, 1 syrk_kernel)}, tile_of[nt*nt], pi[], pj[], pmask[], S[]
//            out: S after one launch over the pair list
//   trsm     in: {m}, panel[m*T*T], linv[T*T]       out: panel after trsm_kernel
//   chain0   in: C[T*T], Q[T*T]                       out: C = C Q^T (chain_gemm_kernel<0>, P = C in place, as in factor())
//   chain1   in: C[T*T], P[T*T]                       out: C -= P P^T on j <= i (chain_gemm_kernel<1>, Q = P)
//   potrf    in: tiles[nb*T*T]                        out: tiles (L in place), inverses[nb*T*T], flags[nb]
//   factor   in: {nt, n, plan (0 blocked, 1 col_group, 2 one-rank owner map), R}, mask[nt*nt], col_group[nt],
//                A[R*n*n], b[R*n]
//            out per run: packed L, tile_of[nt*nt], inverses[nt*T*T], x[nt*T], flag — as cvb_dense_cholesky_solve
//            packs, factors and solves (zero tiles skipped, padding rows with a unit diagonal)
// Output buffers (tile inverses, x) are filled with NaN (all bytes 0xFF) before the launch, as a reused workspace would
// hold stale values: every element the tests read, the zeros above the diagonal of an inverse included, must be written.
// Every CUDA error is reported on stderr and makes the exit code non-zero.
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <limits>
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
#define CK_LAUNCH() CK(cudaGetLastError())

struct In {
  FILE* f;
  template <class V>
  std::vector<V> get() {
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
};
static void put(FILE* f, const void* p, size_t bytes) {
  const int64_t nb = (int64_t)bytes;
  fwrite(&nb, 8, 1, f);
  if (bytes) fwrite(p, 1, bytes, f);
}

template <class V>
static V* to_dev(const std::vector<V>& h) {
  V* d = nullptr;
  CK(cudaMalloc(&d, (h.size() ? h.size() : 1) * sizeof(V)));
  if (h.size()) CK(cudaMemcpy(d, h.data(), h.size() * sizeof(V), cudaMemcpyHostToDevice));
  return d;
}
template <class V>
static void to_host(std::vector<V>& h, const V* d) {
  if (h.size()) CK(cudaMemcpy(h.data(), d, h.size() * sizeof(V), cudaMemcpyDeviceToHost));
}

int main(int argc, char** argv) {
  if (argc != 4) {
    fprintf(stderr, "usage: %s update|trsm|chain0|chain1|potrf|factor in.bin out.bin\n", argv[0]);
    return 2;
  }
  const char* mode = argv[1];
  In in{fopen(argv[2], "rb")};
  if (!in.f) return 2;
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
  std::vector<std::vector<char>> out;   // arrays written to out.bin, in order
  auto emit = [&](const void* p, size_t bytes) { out.emplace_back((const char*)p, (const char*)p + bytes); };

  if (!strcmp(mode, "update")) {
    const auto hdr = in.get<int32_t>();
    const auto tile_of = in.get<int32_t>(), pi = in.get<int32_t>(), pj = in.get<int32_t>(), pm = in.get<int32_t>();
    auto S = in.get<double>();
    const int nt = hdr[0], k0 = hdr[1], np = (int)pi.size();
    int *d_tile_of = to_dev(tile_of), *d_pi = to_dev(pi), *d_pj = to_dev(pj), *d_pm = to_dev(pm);
    double* d_S = to_dev(S);
    if (hdr[2] == 0)
      tile_update_kernel<<<np, TILE_THREADS, kTileSmem, st>>>(d_S, d_tile_of, nt, k0, d_pi, d_pj, d_pm);
    else
      syrk_kernel<<<4 * np, SYRK_THREADS, kSyrkSmem, st>>>(d_S, d_tile_of, nt, k0, d_pi, d_pj, d_pm);
    CK_LAUNCH();
    CK(cudaStreamSynchronize(st));
    to_host(S, d_S);
    emit(S.data(), S.size() * 8);
  } else if (!strcmp(mode, "trsm")) {
    const int m = in.get<int32_t>()[0];
    auto panel = in.get<double>();
    const auto linv = in.get<double>();
    double *d_p = to_dev(panel), *d_l = to_dev(linv);
    trsm_kernel<<<2 * m, TRSM_THREADS, kTrsmSmem, st>>>(d_p, d_l);
    CK_LAUNCH();
    CK(cudaStreamSynchronize(st));
    to_host(panel, d_p);
    emit(panel.data(), panel.size() * 8);
  } else if (!strcmp(mode, "chain0") || !strcmp(mode, "chain1")) {
    auto C = in.get<double>();
    const auto Q = in.get<double>();
    double *d_c = to_dev(C), *d_q = to_dev(Q);
    if (mode[5] == '0')
      chain_gemm_kernel<0><<<T / CHAIN_ROWS, T, kChainSmem, st>>>(d_c, d_c, d_q);
    else
      chain_gemm_kernel<1><<<T / CHAIN_ROWS, T, kChainSmem, st>>>(d_c, d_q, d_q);
    CK_LAUNCH();
    CK(cudaStreamSynchronize(st));
    to_host(C, d_c);
    emit(C.data(), C.size() * 8);
  } else if (!strcmp(mode, "potrf")) {
    auto tiles = in.get<double>();
    const int nb = (int)(tiles.size() / TT);
    std::vector<double> inv(tiles.size(), std::numeric_limits<double>::quiet_NaN());
    std::vector<int32_t> flags(nb, 0);
    double *d_a = to_dev(tiles), *d_inv = to_dev(inv);
    int* d_flag = to_dev(flags);
    for (int t = 0; t < nb; t++) {   // each tile is its own 128 x 128 matrix (ld = T, k = 0)
      potrf_inv_kernel<<<1, POTRF_THREADS, kPotrfSmem, st>>>(d_a + (size_t)t * TT, (size_t)T, 0, d_inv + (size_t)t * TT,
                                                             d_flag + t, nullptr, 0);
      CK_LAUNCH();
    }
    CK(cudaStreamSynchronize(st));
    to_host(tiles, d_a);
    to_host(inv, d_inv);
    to_host(flags, d_flag);
    emit(tiles.data(), tiles.size() * 8);
    emit(inv.data(), inv.size() * 8);
    emit(flags.data(), flags.size() * 4);
  } else if (!strcmp(mode, "factor")) {
    const auto hdr = in.get<int32_t>();
    const auto m32 = in.get<int32_t>(), group = in.get<int32_t>();
    const auto A = in.get<double>(), b = in.get<double>();
    const int nt = hdr[0], n = hdr[1], opt = hdr[2], R = hdr[3], np = nt * T;
    if ((int)m32.size() != nt * nt || (size_t)A.size() != (size_t)R * n * n || (int)b.size() != R * n || n > np) {
      fprintf(stderr, "inconsistent factor input\n");
      return 2;
    }
    TilePlan plan;
    const std::vector<int> owner(nt, 0);
    if (opt == 0) plan.build(nt, std::vector<uint8_t>(m32.begin(), m32.end()));
    else if (opt == 1) plan.build(nt, std::vector<uint8_t>(m32.begin(), m32.end()), std::vector<int>(group.begin(), group.end()));
    else plan.build(nt, std::vector<uint8_t>(m32.begin(), m32.end()), {}, &owner, 0);
    if (plan.upload(&ctx, st)) return 3;
    FactorStreams fs;
    if (fs.create(&ctx, nt)) return 3;
    const size_t nL = (size_t)plan.n_tiles_L * TT;
    double *dS = nullptr, *dl = nullptr, *dv = nullptr;
    int* dflag = nullptr;
    CK(cudaMalloc(&dS, nL * 8));
    CK(cudaMalloc(&dl, (size_t)nt * TT * 8));
    CK(cudaMalloc(&dv, (size_t)np * 3 * 8));
    CK(cudaMalloc(&dflag, 16));
    std::vector<double> hs(nL), hb(np), linv((size_t)nt * TT), x(np);
    for (int r = 0; r < R; r++) {
      const double* Ar = A.data() + (size_t)r * n * n;
      std::fill(hs.begin(), hs.end(), 0.0);
      std::fill(hb.begin(), hb.end(), 0.0);
      for (int i = 0; i < n; i++)
        for (int j = 0; j <= i; j++)
          if (Ar[(size_t)i * n + j] != 0.0) {
            const int t = plan.h_tile_of[(size_t)(i / T) * nt + (j / T)];
            if (t < 0) {
              fprintf(stderr, "A(%d,%d) lies outside the tile mask\n", i, j);
              return 2;
            }
            hs[(size_t)t * TT + (size_t)(i % T) * T + (j % T)] = Ar[(size_t)i * n + j];
          }
      for (int i = n; i < np; i++) hs[plan.tile_index(i / T, i / T) * TT + (size_t)(i % T) * T + (i % T)] = 1.0;
      for (int i = 0; i < n; i++) hb[i] = b[(size_t)r * n + i];
      CK(cudaMemcpyAsync(dS, hs.data(), nL * 8, cudaMemcpyHostToDevice, st));
      CK(cudaMemcpyAsync(dv, hb.data(), (size_t)np * 8, cudaMemcpyHostToDevice, st));
      CK(cudaMemsetAsync(dl, 0xFF, (size_t)nt * TT * 8, st));
      CK(cudaMemsetAsync(dv + np, 0xFF, (size_t)np * 2 * 8, st));
      if (factor(&ctx, dS, dl, dflag, plan, st, fs, nullptr)) return 3;
      if (solve(&ctx, dS, dl, dv, dv + np, dv + 2 * np, plan, st, fs)) return 3;
      int flag = 0;
      CK(cudaMemcpyAsync(&flag, dflag, 4, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(hs.data(), dS, nL * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(linv.data(), dl, linv.size() * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(x.data(), dv + 2 * (size_t)np, (size_t)np * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      emit(hs.data(), hs.size() * 8);
      emit(plan.h_tile_of.data(), plan.h_tile_of.size() * 4);
      emit(linv.data(), linv.size() * 8);
      emit(x.data(), x.size() * 8);
      emit(&flag, 4);
    }
    CK(cudaDeviceSynchronize());
    fs.destroy();
    plan.release();
  } else {
    fprintf(stderr, "unknown mode %s\n", mode);
    return 2;
  }
  fclose(in.f);
  CK(cudaDeviceSynchronize());
  FILE* f = fopen(argv[3], "wb");
  if (!f) return 2;
  for (const auto& v : out) put(f, v.data(), v.size());
  fclose(f);
  return 0;
}
