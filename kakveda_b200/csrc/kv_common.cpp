// Error reporting, library identification and the host helpers the index handles share (device selection, tensor
// maps) for libkakveda_b200.
#include "kv_cuda.cuh"
#include "sm90.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <new>
#include <thread>
#include <type_traits>
#include <vector>

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

namespace {
// score and row of a record in the order range_order sorts by
inline float pair_score(const RangePair &p) { return p.score; }
inline int64_t pair_row(const RangePair &p) { return p.row; }
inline float pair_score(const JaccardPair &p) { return (float)p.inter / (float)p.uni; }
inline int64_t pair_row(const JaccardPair &p) { return p.row; }
}  // namespace

template <class Rec>
int range_order(const Rec *rec, int64_t n, int64_t n_q, int64_t row_base, int64_t *indptr, int64_t *rows, float *scores,
                int32_t *inter, int32_t *uni, const char *fn) {
  std::vector<Rec> by_q;
  try {
    by_q.resize((size_t)n);
  } catch (const std::bad_alloc &) {
    return kv_fail(KV_ERR_NOMEM, "%s: out of host memory", fn);
  }
  for (int64_t q = 0; q <= n_q; q++) indptr[q] = 0;
  for (int64_t i = 0; i < n; i++) indptr[rec[i].q + 1]++;
  for (int64_t q = 0; q < n_q; q++) indptr[q + 1] += indptr[q];
  std::vector<int64_t> next(indptr, indptr + n_q);
  for (int64_t i = 0; i < n; i++) by_q[(size_t)next[(size_t)rec[i].q]++] = rec[i];
  // thread t orders queries [n_q t / T, n_q (t + 1) / T)
  const int T = (int)std::max<int64_t>(1, std::min<int64_t>(n >= 65536 ? host_threads() : 1, n_q));
  auto body = [&](int t) {
    for (int64_t q = n_q * t / T; q < n_q * (t + 1) / T; q++) {
      Rec *lo = by_q.data() + indptr[q], *hi = by_q.data() + indptr[q + 1];
      std::sort(lo, hi, [](const Rec &x, const Rec &y) {
        const float sx = pair_score(x), sy = pair_score(y);
        return sx != sy ? sx > sy : pair_row(x) < pair_row(y);
      });
      for (Rec *p = lo; p < hi; p++) {
        const size_t i = (size_t)(p - by_q.data());
        rows[i] = row_base + pair_row(*p);
        scores[i] = pair_score(*p);
        if constexpr (std::is_same_v<Rec, JaccardPair>) {
          inter[i] = p->inter;
          uni[i] = p->uni;
        }
      }
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < T; t++) th.emplace_back(body, t);
  body(0);
  for (auto &x : th) x.join();
  return KV_OK;
}

template int range_order<RangePair>(const RangePair *, int64_t, int64_t, int64_t, int64_t *, int64_t *, float *, int32_t *,
                                    int32_t *, const char *);
template int range_order<JaccardPair>(const JaccardPair *, int64_t, int64_t, int64_t, int64_t *, int64_t *, float *,
                                      int32_t *, int32_t *, const char *);

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
