// Error reporting and library identification for libkakveda_b200.
#include "kv_internal.h"

#include <cuda_runtime_api.h>

#include <cstring>

namespace {
thread_local char g_err[512] = "";
}

int kv_fail(int code, const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void kv_clear_error() { g_err[0] = 0; }

extern "C" {

const char *kv_last_error(void) { return g_err; }

const char *kv_version(void) { return "kakveda_b200 0.1 (sm_90a)"; }

int kv_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

}  // extern "C"
