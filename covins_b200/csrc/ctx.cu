// ctx.cu — context lifetime, error reporting.
#include <stdarg.h>

#include "cvb_internal.cuh"

int cvb_fail(cvb_ctx* ctx, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf;
  return code;
}

extern "C" {

int cvb_version(void) { return 100; }

int cvb_ctx_create(int device, cvb_ctx** out) {
  if (!out) return CVB_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0 || device < 0 || device >= n) return CVB_ERR_CUDA;  // no CPU fallback
  if (cudaSetDevice(device) != cudaSuccess) return CVB_ERR_CUDA;
  cvb_ctx* c = new cvb_ctx();
  c->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
    delete c;
    return CVB_ERR_CUDA;
  }
  c->sm_count = prop.multiProcessorCount;
  int prio_lo = 0, prio_hi = 0;   // the ctx stream carries the critical path (diagonal tiles, panels): greatest priority
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if (cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_hi) != cudaSuccess) {
    delete c;
    return CVB_ERR_CUDA;
  }
  {   // keep memory freed by the stream-ordered allocator in the pool (problem set-up re-uses it)
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      unsigned long long thr = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
  }
  *out = c;
  return CVB_OK;
}

int cvb_ctx_destroy(cvb_ctx* ctx) {
  if (!ctx) return CVB_OK;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->h_pin) cudaFreeHost(ctx->h_pin);
  cudaStreamDestroy(ctx->stream);
  delete ctx;
  return CVB_OK;
}

const char* cvb_last_error(const cvb_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }

int cvb_ctx_sync(cvb_ctx* ctx) {
  if (!ctx) return CVB_ERR_INVALID;
  CVB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return CVB_OK;
}

int64_t cvb_launch_count(const cvb_ctx* ctx) { return ctx ? ctx->launches : 0; }

}  // extern "C"
