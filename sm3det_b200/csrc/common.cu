#include "common.cuh"
#include <cstdlib>
#include <cstdarg>
#include <cstdio>
#include <mutex>

namespace sm3 {

static thread_local char g_last_error[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

const char* last_error() { return g_last_error; }

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: %s", what, cudaGetErrorString(e));
    return SM3_ERR_CUDA;
  }
  return SM3_OK;
}

int num_sms() {
  static int cached[64];
  static std::once_flag once[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  std::call_once(once[dev], [dev]() {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 132;
  });
  return cached[dev];
}

// Persistent GEMM kernels occupy a whole SM each (all of its registers / shared memory), so a collective launched on
// another stream (NCCL's gradient all-reduce under DDP) cannot co-reside and is serialised behind them.  SM3_RESERVE_SMS=n
// keeps n SMs out of the persistent grids so that NCCL's CTAs run concurrently with the backward GEMMs.
int persistent_grid_sms() {
  static const int reserve = []() { const char* e = getenv("SM3_RESERVE_SMS"); const int v = e ? atoi(e) : 0; return v < 0 ? 0 : v; }();
  const int n = num_sms() - reserve;
  return n < 1 ? 1 : n;
}

}  // namespace sm3
