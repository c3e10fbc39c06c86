// Error reporting and device queries of libpipegcn_b200.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace pg {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      n = 132;
    }
  }
  return n;
}
}  // namespace pg

extern "C" int pg_abi_version(void) { return PG_ABI_VERSION; }
extern "C" const char* pg_last_error(void) { return pg::g_err; }

extern "C" int pg_device_info(int device, int* sm_arch, int* sm_count, int64_t* l2_bytes) {
  cudaDeviceProp p;
  PG_CHECK_CUDA(cudaGetDeviceProperties(&p, device));
  if (sm_arch) *sm_arch = p.major * 10 + p.minor;
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (l2_bytes) *l2_bytes = p.l2CacheSize;
  return PG_OK;
}
