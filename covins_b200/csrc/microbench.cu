// microbench.cu — INT-pipe (XOR+POPC+IADD) issue-rate microbenchmark.  SURVEY.md §8d: the Hamming k-NN
// kernel is bound by the POPC pipe, whose peak is not in MEASURED_PEAKS.json, so it is measured here and
// used as the second roofline denominator next to HBM bandwidth.
#include "cvb_internal.cuh"

namespace {
__global__ void __launch_bounds__(256) popc_kernel(int iters, uint32_t seed, uint32_t* out) {
  uint32_t x[8], acc[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    x[i] = seed * (threadIdx.x + 1) + i * 0x9E3779B9u;
    acc[i] = 0;
  }
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      acc[i] += __popc(x[i] ^ (uint32_t)it);
      x[i] += acc[i];  // keeps the chain alive without adding POPC work
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) s += acc[i];
  if (s == 0xFFFFFFFFu) out[0] = s;  // never true in practice; defeats dead-code elimination
}
}  // namespace

extern "C" int cvb_microbench_popc(cvb_ctx* ctx, int iters, double* gpopc_per_s) {
  if (!ctx || !gpopc_per_s || iters <= 0) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  cvb_block B(ctx, ctx->stream);
  uint32_t* d;
  B.tmp(d, 1);
  if (const int rc = B.place()) return rc;
  const int blocks = ctx->sm_count * 8;
  cudaEvent_t e0, e1;
  CVB_CUDA(ctx, cudaEventCreate(&e0));
  CVB_CUDA(ctx, cudaEventCreate(&e1));
  popc_kernel<<<blocks, 256, 0, ctx->stream>>>(iters / 4 + 1, 12345u, d);  // warm-up
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaEventRecord(e0, ctx->stream));
  popc_kernel<<<blocks, 256, 0, ctx->stream>>>(iters, 12345u, d);
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaEventRecord(e1, ctx->stream));
  CVB_CUDA(ctx, cudaEventSynchronize(e1));
  float ms = 0.f;
  CVB_CUDA(ctx, cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *gpopc_per_s = (double)blocks * 256.0 * (double)iters * 8.0 / (ms * 1e-3) / 1e9;
  return CVB_OK;
}

// ------------------------------------------------------------------------------------------------
// Single-warp latency probes for the serial part of the diagonal-tile factorisation (cholesky.cu): cycles per
// dependent operation, measured with clock64 over a chain of N operations.
//   out[0] dependent DFMA      out[1] 8 independent DFMA chains (cycles per DFMA)   out[2] dependent rsqrt(double)
//   out[3] dependent SHFL.IDX of a double   out[4] dependent STS.64+LDS.64 round trip (with __syncwarp)
//   out[5] dependent DMUL      out[6] dependent FFMA (fp32, for scale)     out[7] SM clock estimate (MHz)
// ------------------------------------------------------------------------------------------------
namespace {
__global__ void latency_kernel(double* out, double seed, int n) {
  __shared__ double sh[32];
  const int lane = threadIdx.x;
  long long t0, t1;
  double x = seed + lane * 1e-3, y = 1.0 - 1e-9;
  t0 = clock64();
  for (int i = 0; i < n; i++) x = fma(x, y, 1e-9);
  t1 = clock64();
  double r0 = (double)(t1 - t0) / n;
  double c[8];
#pragma unroll
  for (int k = 0; k < 8; k++) c[k] = seed + k;
  t0 = clock64();
  for (int i = 0; i < n; i++) {
#pragma unroll
    for (int k = 0; k < 8; k++) c[k] = fma(c[k], y, 1e-9);
  }
  t1 = clock64();
  double r1 = (double)(t1 - t0) / (8.0 * n);
#pragma unroll
  for (int k = 0; k < 8; k++) x += c[k];
  double z = 1.0 + x * 1e-30;
  t0 = clock64();
  for (int i = 0; i < n; i++) z = rsqrt(z) + 0.5;
  t1 = clock64();
  double r2 = (double)(t1 - t0) / n;
  double s = z;
  t0 = clock64();
  for (int i = 0; i < n; i++) s = __shfl_sync(0xffffffffu, s, (lane + 1) & 31);
  t1 = clock64();
  double r3 = (double)(t1 - t0) / n;
  double w = s;
  t0 = clock64();
  for (int i = 0; i < n; i++) {
    sh[lane] = w;
    __syncwarp();
    w = sh[(lane + 1) & 31];
    __syncwarp();
  }
  t1 = clock64();
  double r4 = (double)(t1 - t0) / n;
  double m = w + 1.0;
  t0 = clock64();
  for (int i = 0; i < n; i++) m = m * y;
  t1 = clock64();
  double r5 = (double)(t1 - t0) / n;
  float f = (float)m, g = 0.999999f;
  t0 = clock64();
  for (int i = 0; i < n; i++) f = fmaf(f, g, 1e-9f);
  t1 = clock64();
  double r6 = (double)(t1 - t0) / n;
  if (lane == 0) {
    out[0] = r0; out[1] = r1; out[2] = r2; out[3] = r3; out[4] = r4; out[5] = r5; out[6] = r6;
    out[8] = x + z + s + w + m + f;   // keep everything live
  }
}
}  // namespace

extern "C" int cvb_microbench_latency(cvb_ctx* ctx, double* out8) {
  if (!ctx || !out8) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  double h[9];
  cvb_block B(ctx, ctx->stream);
  double* d;
  B.out(d, h, 9);
  if (const int rc = B.place()) return rc;
  cudaEvent_t e0, e1;
  CVB_CUDA(ctx, cudaEventCreate(&e0));
  CVB_CUDA(ctx, cudaEventCreate(&e1));
  const int n = 4096;
  latency_kernel<<<1, 32, 0, ctx->stream>>>(d, 1.0, n);   // warm-up
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaEventRecord(e0, ctx->stream));
  latency_kernel<<<1, 32, 0, ctx->stream>>>(d, 1.0, n);
  CVB_CHECK_LAUNCH(ctx);
  CVB_CUDA(ctx, cudaEventRecord(e1, ctx->stream));
  if (const int rc = B.download()) return rc;
  float ms = 0.f;
  CVB_CUDA(ctx, cudaEventElapsedTime(&ms, e0, e1));
  for (int i = 0; i < 7; i++) out8[i] = h[i];
  const double cycles = n * (h[0] + 8 * h[1] + h[2] + h[3] + h[4] + h[5] + h[6]);
  out8[7] = cycles / (ms * 1e-3) / 1e6;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return CVB_OK;
}

// ------------------------------------------------------------------------------------------------
// Issue rate of the integer min/max forms the matching epilogue can use (per SM per clock, all SMs busy):
//   out[0] 32-bit signed min/max (VIMNMX.S32)   out[1] packed 2 x u16 min/max (VIMNMX.U16x2), counted per instruction
// ------------------------------------------------------------------------------------------------
namespace {
template <int MODE>
__global__ void __launch_bounds__(256) minmax_kernel(unsigned* out, unsigned seed, int iters) {
  unsigned w[8], x = seed * (threadIdx.x + 1) + blockIdx.x;
#pragma unroll
  for (int c = 0; c < 8; c++) w[c] = 0xffffffffu - c * seed;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int c = 0; c < 8; c++) {
      if (MODE == 0) {
        const int lo = min((int)w[c], (int)x);
        x = (unsigned)max((int)w[c], (int)x);
        w[c] = (unsigned)lo;
      } else {
        const unsigned lo = __vminu2(w[c], x);
        x = __vmaxu2(w[c], x);
        w[c] = lo;
      }
    }
    x = x * 1664525u + 1013904223u;
  }
  unsigned r = x;
#pragma unroll
  for (int c = 0; c < 8; c++) r ^= w[c];
  if (r == 0x12345678u) out[0] = r;
}
}  // namespace

extern "C" int cvb_microbench_minmax(cvb_ctx* ctx, double* out2) {
  if (!ctx || !out2) return CVB_ERR_INVALID;
  CVB_GUARD(ctx);
  cvb_block B(ctx, ctx->stream);
  unsigned* d;
  B.tmp(d, 1);
  if (const int rc = B.place()) return rc;
  cudaEvent_t e0, e1;
  CVB_CUDA(ctx, cudaEventCreate(&e0));
  CVB_CUDA(ctx, cudaEventCreate(&e1));
  const int iters = 4096, blocks = ctx->sm_count * 8;
  int clk_khz = 0;
  cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, ctx->device);
  for (int mode = 0; mode < 2; mode++) {
    for (int rep = 0; rep < 2; rep++) {
      CVB_CUDA(ctx, cudaEventRecord(e0, ctx->stream));
      if (mode == 0) minmax_kernel<0><<<blocks, 256, 0, ctx->stream>>>(d, 12345u, iters);
      else minmax_kernel<1><<<blocks, 256, 0, ctx->stream>>>(d, 12345u, iters);
      CVB_CHECK_LAUNCH(ctx);
      CVB_CUDA(ctx, cudaEventRecord(e1, ctx->stream));
      CVB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    float ms = 0.f;
    CVB_CUDA(ctx, cudaEventElapsedTime(&ms, e0, e1));
    const double lane_ops = (double)blocks * 256 * iters * 16;   // 2 instructions x 8 chains per iteration
    out2[mode] = lane_ops / (ms * 1e-3) / ((double)clk_khz * 1e3) / ctx->sm_count;   // lane-instructions / clk / SM
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return CVB_OK;
}
