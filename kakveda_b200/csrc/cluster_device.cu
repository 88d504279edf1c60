// Connected components of a CSR graph on the device (kv_cluster_csr_device): the contract of kv_cluster_csr
// (cluster.cpp) for inputs that already live in HBM, such as what kv_range_fetch_device returns for a self-join.
//
// A lock-free union-find over the labels array itself: every edge hooks the larger of its two roots under the smaller
// with a compare-and-swap, and finds shorten the paths they walk.  A parent is never larger than its child, so each
// root is the smallest vertex of its tree and the final labels (smallest row of the component) do not depend on the
// order the atomics take.  One thread per edge, its source found by binary search in indptr, so one long adjacency list
// spreads over many threads like many short ones.  Validation passes (indptr, then rows) run before any hooking.
#include "kv_cuda.cuh"

namespace {

constexpr int CC_THREADS = 256;

inline unsigned cc_grid(int64_t n) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + CC_THREADS - 1) / CC_THREADS, 1 << 16));
}

// flag |= 1 unless 0 <= indptr[0] <= indptr[1] <= ... <= indptr[n]
__global__ void cc_check_indptr_kernel(const int64_t *indptr, int64_t n, unsigned long long *flag) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (indptr[i + 1] < indptr[i] || (i == 0 && indptr[0] < 0)) atomicOr(flag, 1ull);
}

// flag |= 2 if a row of rows[lo, hi) is >= n
__global__ void cc_check_rows_kernel(const int64_t *rows, int64_t lo, int64_t hi, int64_t n, unsigned long long *flag) {
  for (int64_t j = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < hi; j += (int64_t)gridDim.x * blockDim.x)
    if (rows[j] >= n) atomicOr(flag, 2ull);
}

__global__ void cc_init_kernel(int64_t *parent, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) parent[i] = i;
}

// Root of x; every vertex passed on the way is pointed at its grandparent (still an ancestor, never below the root).
// Loads bypass L1: other SMs hook roots while this runs.
__device__ __forceinline__ int64_t cc_find(int64_t *parent, int64_t x) {
  int64_t p = __ldcg(parent + x);
  while (p != x) {
    const int64_t gp = __ldcg(parent + p);
    if (gp != p) parent[x] = gp;
    x = p;
    p = gp;
  }
  return x;
}

__global__ void cc_hook_kernel(const int64_t *indptr, const int64_t *rows, int64_t n, int64_t *parent) {
  const int64_t base = indptr[0], m = indptr[n] - base;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = base + e, r = rows[j];
    if (r < 0) continue;
    int64_t lo = 0, hi = n;  // the source: the last i with indptr[i] <= j
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(indptr + mid) <= j) lo = mid;
      else hi = mid;
    }
    int64_t a = cc_find(parent, lo), b = cc_find(parent, r);
    while (a != b) {
      if (a > b) { const int64_t t = a; a = b; b = t; }
      // b is (or was) a root larger than a: hook it under a, or follow it to the root it has meanwhile been hooked to
      const unsigned long long old = atomicCAS((unsigned long long *)(parent + b), (unsigned long long)b, (unsigned long long)a);
      if (old == (unsigned long long)b) break;
      b = cc_find(parent, (int64_t)old);
    }
  }
}

// labels[i] = root of i (labels is the parent array); *count += roots
__global__ void cc_finish_kernel(int64_t *parent, int64_t n, unsigned long long *count) {
  unsigned c = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t x = i, p;
    while ((p = __ldcg(parent + x)) != x) x = p;
    parent[i] = x;
    c += x == i;
  }
  c = __reduce_add_sync(0xFFFFFFFFu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}

}  // namespace

extern "C" int kv_cluster_csr_device(int device, int64_t n, const void *d_indptr, const void *d_rows, void *d_labels,
                                     int64_t *n_clusters) {
  const char *fn = "kv_cluster_csr_device";
  if (n < 0) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  int sm_count = 0;
  int rc = open_device(device, fn, &sm_count);
  if (rc != KV_OK) return rc;
  if (n == 0) {
    if (n_clusters) *n_clusters = 0;
    return KV_OK;
  }
  if ((rc = check_device_ptr(d_indptr, device, 8, "indptr", fn)) != KV_OK) return rc;
  if ((rc = check_device_ptr(d_labels, device, 8, "labels", fn)) != KV_OK) return rc;
  const int64_t *indptr = (const int64_t *)d_indptr, *rows = (const int64_t *)d_rows;
  int64_t *labels = (int64_t *)d_labels;
  CudaStream s;
  KV_CUDA(s.create());
  DevBuf<unsigned long long> flag;  // [0] validation flags, [1] root count
  KV_CUDA(flag.ensure(2));
  KV_CUDA(cudaMemsetAsync(flag.p, 0, 2 * sizeof(unsigned long long), s));
  cc_check_indptr_kernel<<<cc_grid(n), CC_THREADS, 0, s>>>(indptr, n, flag.p);
  KV_CUDA(cudaGetLastError());
  unsigned long long bad = 0;
  int64_t ends[2] = {0, 0};
  KV_CUDA(cudaMemcpyAsync(&bad, flag.p, sizeof(bad), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaMemcpyAsync(&ends[0], indptr, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaMemcpyAsync(&ends[1], indptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  if (bad) return kv_fail(KV_ERR_INVALID, "%s: indptr not monotone (or indptr[0] < 0)", fn);
  if (ends[1] > ends[0]) {
    if ((rc = check_device_ptr(d_rows, device, 8, "rows", fn)) != KV_OK) return rc;
    cc_check_rows_kernel<<<cc_grid(ends[1] - ends[0]), CC_THREADS, 0, s>>>(rows, ends[0], ends[1], n, flag.p);
    KV_CUDA(cudaGetLastError());
    KV_CUDA(cudaMemcpyAsync(&bad, flag.p, sizeof(bad), cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaStreamSynchronize(s));
    if (bad) return kv_fail(KV_ERR_INVALID, "%s: a neighbour row outside 0..%lld", fn, (long long)n);
  }
  cc_init_kernel<<<cc_grid(n), CC_THREADS, 0, s>>>(labels, n);
  if (ends[1] > ends[0]) cc_hook_kernel<<<cc_grid(ends[1] - ends[0]), CC_THREADS, 0, s>>>(indptr, rows, n, labels);
  cc_finish_kernel<<<cc_grid(n), CC_THREADS, 0, s>>>(labels, n, flag.p + 1);
  KV_CUDA(cudaGetLastError());
  unsigned long long count = 0;
  KV_CUDA(cudaMemcpyAsync(&count, flag.p + 1, sizeof(count), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  if (n_clusters) *n_clusters = (int64_t)count;
  return KV_OK;
}
