// Error reporting, library identification and the host helpers the index handles share (device selection, tensor
// maps) for libkakveda_b200.
#include "kv_cuda.cuh"
#include "sm90.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <thread>

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

int host_threads() {
  int t = (int)std::thread::hardware_concurrency();
  if (const char *e = getenv("KAKVEDA_B200_THREADS")) t = atoi(e);
  return std::max(1, std::min(t, 64));
}

int open_device(int device, const char *fn, int *sm_count) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return kv_fail(KV_ERR_CUDA, "%s: no CUDA device visible (this library has no CPU path)", fn);
  }
  if (device < 0 || device >= n) return kv_fail(KV_ERR_INVALID, "%s: device %d out of range", fn, device);
  KV_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  KV_CUDA(cudaGetDeviceProperties(&prop, device));
  *sm_count = prop.multiProcessorCount;
  return KV_OK;
}

int make_map_2d(CUtensorMap *map, CUtensorMapDataType dtype, const void *base, int64_t rows, int64_t cols, int box_rows) {
  typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                      const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static const PFN_encodeTiled fn = [] {  // looked up once per process (thread-safe static initialisation)
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess) p = nullptr;
    return (PFN_encodeTiled)p;
  }();
  if (!fn) return kv_fail(KV_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, dtype, 2, const_cast<void *>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return kv_fail(KV_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return KV_OK;
}

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
