// W-way merge of ordered threshold-search results (kv_merge_range_device_on): the CSR results of W row shards --
// indptr by query, each query's pairs by (score desc, row asc), as kv_range_fetch_device writes them -- become the
// one CSR a single index over all the rows returns.  Every run is ordered already, so one pass places every record:
//
//   rm_count_kernel    per query, the sum of its segment lengths over the runs (checking every run's indptr);
//   exclusive_scan_u32 of those sums (the ro_scan_* kernels of range_order.cu) gives the output indptr;
//   rm_place_kernel    one thread per input record: its query by binary search in its run's indptr, and its output
//                      slot = indptr_out[q] + its index in its own segment + its lower bound in the segment of q in
//                      every other run.  The shards hold disjoint rows, so (score, row) is a total order of the union
//                      and the slots are a permutation.
//
// Invalid input is found on the way, without a pass of its own: a decreasing indptr, indptr[0] != 0 or
// indptr[n_q] != the run's announced count (count kernel); a segment out of (score desc, row asc) order -- each record
// compares itself with its predecessor -- and a (score, row) key present in two runs -- a lower bound that lands on an
// equal key (place kernel).  The place kernel reads the count kernel's flags and writes nothing when the indptrs are
// bad, so no bound search ever leaves its segment.  Work: one read and one write of every record plus (W-1) binary
// searches of at most log2(segment) probes.
#include "kv_cuda.cuh"

namespace {

constexpr int RM_THREADS = 256;
constexpr int RM_MAX_RUNS = 64;

enum : unsigned { RM_BAD_INDPTR = 1u, RM_BAD_ORDER = 2u, RM_DUPLICATE = 4u, RM_BAD_SCORE = 8u };

// The runs, passed by value: run w's indptr at indptr + w * indptr_stride, its record arrays at base + w * rec_stride
// bytes; start[w] = records of runs before w (start[n_runs] = all records).
struct Runs {
  const int64_t *indptr;
  const char *rows, *scores, *inter, *uni;
  int64_t indptr_stride, rec_stride, n_q;
  int n_runs;
  int64_t pairs[RM_MAX_RUNS];
  int64_t start[RM_MAX_RUNS + 1];
};

__device__ __forceinline__ const int64_t *run_indptr(const Runs &R, int w) { return R.indptr + w * R.indptr_stride; }
__device__ __forceinline__ const int64_t *run_rows(const Runs &R, int w) {
  return reinterpret_cast<const int64_t *>(R.rows + w * R.rec_stride);
}
__device__ __forceinline__ const float *run_scores(const Runs &R, int w) {
  return reinterpret_cast<const float *>(R.scores + w * R.rec_stride);
}

// (s, r) strictly before (s2, r2) in the (score desc, row asc) order
__device__ __forceinline__ bool before(float s, int64_t r, float s2, int64_t r2) { return s > s2 || (s == s2 && r < r2); }

// counts[q] = pairs of query q over all runs (q < n_q), counts[n_q] = 0; flags |= RM_BAD_INDPTR on a bad indptr
__global__ void __launch_bounds__(RM_THREADS) rm_count_kernel(Runs R, unsigned *counts, unsigned *flags) {
  bool bad = false;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q <= R.n_q; q += (int64_t)gridDim.x * blockDim.x) {
    unsigned long long c = 0;
    for (int w = 0; w < R.n_runs; w++) {
      const int64_t *ip = run_indptr(R, w);
      if (q == R.n_q) {
        bad |= ip[0] != 0 || ip[R.n_q] != R.pairs[w];
        continue;
      }
      const int64_t a = ip[q], b = ip[q + 1];
      bad |= b < a;
      c += (unsigned long long)(b - a);
    }
    counts[q] = q == R.n_q ? 0u : (unsigned)c;
    bad |= c > 0xFFFFFFFFull;
  }
  if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) atomicOr(flags, RM_BAD_INDPTR);
}

// Records of segment [a, b) of run v strictly before (s, r); *dup when the first record not before it equals it.
__device__ __forceinline__ int64_t lower_bound(const float *sc, const int64_t *rw, int64_t a, int64_t b, float s, int64_t r,
                                               bool *dup) {
  int64_t lo = a, hi = b;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (before(__ldg(sc + mid), __ldg(rw + mid), s, r)) lo = mid + 1;
    else hi = mid;
  }
  if (lo < b && __ldg(sc + lo) == s && __ldg(rw + lo) == r) *dup = true;
  return lo - a;
}

// One thread per input record (grid-stride over all runs' records), and indptr_out[q] = scan[q] for q <= n_q.
template <bool JAC>
__global__ void __launch_bounds__(RM_THREADS) rm_place_kernel(Runs R, const unsigned *scan, unsigned *flags, int64_t *indptr_out,
                                                              int64_t *rows_out, float *scores_out, int32_t *inter_out,
                                                              int32_t *uni_out) {
  if (*flags & RM_BAD_INDPTR) return;
  const int64_t total = R.start[R.n_runs], stride = (int64_t)gridDim.x * blockDim.x;
  unsigned bad = 0;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g <= R.n_q; g += stride) indptr_out[g] = (int64_t)scan[g];
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += stride) {
    int w = 0;  // the run of record g: the last w with start[w] <= g
    for (int lo = 0, hi = R.n_runs; hi - lo > 1;) {
      const int mid = (lo + hi) >> 1;
      if (R.start[mid] <= g) lo = mid;
      else hi = mid;
      w = lo;
    }
    const int64_t i = g - R.start[w];
    const int64_t *ip = run_indptr(R, w);
    int64_t q = 0;  // its query: the last q with ip[q] <= i (ip[n_q] = pairs[w] > i)
    for (int64_t lo = 0, hi = R.n_q; hi - lo > 1;) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(ip + mid) <= i) lo = mid;
      else hi = mid;
      q = lo;
    }
    const int64_t a = __ldg(ip + q);
    const float s = __ldg(run_scores(R, w) + i);
    const int64_t r = __ldg(run_rows(R, w) + i);
    if (!(s == s)) bad |= RM_BAD_SCORE;
    if (i > a && !before(__ldg(run_scores(R, w) + i - 1), __ldg(run_rows(R, w) + i - 1), s, r)) bad |= RM_BAD_ORDER;
    int64_t pos = (int64_t)scan[q] + (i - a);
    bool dup = false;
    for (int v = 0; v < R.n_runs; v++) {
      if (v == w) continue;
      const int64_t *ipv = run_indptr(R, v);
      pos += lower_bound(run_scores(R, v), run_rows(R, v), __ldg(ipv + q), __ldg(ipv + q + 1), s, r, &dup);
    }
    if (dup) bad |= RM_DUPLICATE;
    if (pos < 0 || pos >= total) {  // only reachable through the order faults flagged above
      bad |= RM_BAD_ORDER;
      continue;
    }
    rows_out[pos] = r;
    scores_out[pos] = s;
    if constexpr (JAC) {
      inter_out[pos] = reinterpret_cast<const int32_t *>(R.inter + w * R.rec_stride)[i];
      uni_out[pos] = reinterpret_cast<const int32_t *>(R.uni + w * R.rec_stride)[i];
    }
  }
  bad = __reduce_or_sync(0xFFFFFFFFu, bad);
  if (bad && (threadIdx.x & 31) == 0) atomicOr(flags, bad);
}

inline unsigned rm_grid(int64_t n, int sm_count) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + RM_THREADS - 1) / RM_THREADS, 8LL * sm_count * (2048 / RM_THREADS)));
}

}  // namespace

extern "C" int kv_merge_range_device_on(int device, int n_runs, int64_t n_q, const void *d_indptr, int64_t indptr_stride,
                                        const void *d_rows, const void *d_scores, const void *d_inter, const void *d_uni,
                                        int64_t rec_stride_bytes, const int64_t *run_pairs, void *d_indptr_out,
                                        void *d_rows_out, void *d_scores_out, void *d_inter_out, void *d_uni_out, void *stream) {
  const char *fn = "kv_merge_range_device";
  const bool jac = d_inter || d_uni;
  if (n_runs < 1 || n_runs > RM_MAX_RUNS || n_q < 0 || !run_pairs || !d_indptr || !d_indptr_out ||
      (jac && (!d_inter || !d_uni)) || (!jac && (d_inter_out || d_uni_out)))
    return kv_fail(KV_ERR_INVALID, "%s: bad arguments (1 to %d runs; inter and uni both set or both NULL)", fn, RM_MAX_RUNS);
  if (n_runs > 1 && (indptr_stride < n_q + 1 || rec_stride_bytes < 0 || rec_stride_bytes % 8 != 0))
    return kv_fail(KV_ERR_INVALID, "%s: indptr stride below n_q + 1, or a record stride that is not a multiple of 8 bytes", fn);
  Runs R{};
  R.indptr = (const int64_t *)d_indptr;
  R.rows = (const char *)d_rows;
  R.scores = (const char *)d_scores;
  R.inter = (const char *)d_inter;
  R.uni = (const char *)d_uni;
  R.indptr_stride = indptr_stride;
  R.rec_stride = rec_stride_bytes;
  R.n_q = n_q;
  R.n_runs = n_runs;
  int64_t total = 0;
  for (int w = 0; w < n_runs; w++) {
    if (run_pairs[w] < 0) return kv_fail(KV_ERR_INVALID, "%s: run %d announces %lld pairs", fn, w, (long long)run_pairs[w]);
    if (n_runs > 1 && run_pairs[w] * 8 > rec_stride_bytes)
      return kv_fail(KV_ERR_INVALID, "%s: run %d: %lld pairs do not fit the record stride of %lld bytes", fn, w,
                     (long long)run_pairs[w], (long long)rec_stride_bytes);
    R.pairs[w] = run_pairs[w];
    R.start[w] = total;
    total += run_pairs[w];
  }
  R.start[n_runs] = total;
  // the per-query sums are scanned in 32 bits (exclusive_scan_u32)
  if (total >= (int64_t)0xFFFFFFFFll)
    return kv_fail(KV_ERR_NOMEM, "%s: %lld pairs: too many to merge in one call (split the query batch)", fn, (long long)total);
  int sm_count = 0;
  int rc = open_device(device, fn, &sm_count);
  if (rc != KV_OK) return rc;
  if ((rc = check_device_ptr(d_indptr, device, 8, "indptr", fn)) != KV_OK) return rc;
  if ((rc = check_device_ptr(d_indptr_out, device, 8, "indptr_out", fn)) != KV_OK) return rc;
  if (total > 0) {
    const struct { const void *p; size_t al; const char *what; } ptrs[] = {
        {d_rows, 8, "rows"}, {d_scores, 4, "scores"}, {d_rows_out, 8, "rows_out"}, {d_scores_out, 4, "scores_out"},
        {d_inter, 4, "inter"}, {d_uni, 4, "uni"}, {d_inter_out, 4, "inter_out"}, {d_uni_out, 4, "uni_out"}};
    for (int j = 0; j < (jac ? 8 : 4); j++)
      if ((rc = check_device_ptr(ptrs[j].p, device, ptrs[j].al, ptrs[j].what, fn)) != KV_OK) return rc;
  }
  cudaStream_t s = (cudaStream_t)stream;
  // scratch in the stream-ordered pool: the caller's stream keeps the order, and no device-wide sync is needed
  const int64_t n_counts = n_q + 1, n_part = (n_counts + 4095) / 4096;
  unsigned *scratch = nullptr;
  KV_CUDA(cudaMallocAsync((void **)&scratch, (size_t)(1 + n_counts + n_part) * sizeof(unsigned), s));
  unsigned *flags = scratch, *counts = scratch + 1;
  DevBuf<unsigned> part;  // exclusive_scan_u32's tile sums: borrows the end of the scratch (released below, never freed)
  part.p = scratch + 1 + n_counts;
  part.cap = n_part;
  auto run = [&]() -> int {
    KV_CUDA(cudaMemsetAsync(flags, 0, sizeof(unsigned), s));
    rm_count_kernel<<<rm_grid(n_counts, sm_count), RM_THREADS, 0, s>>>(R, counts, flags);
    KV_CUDA(cudaGetLastError());
    int rc2 = exclusive_scan_u32(counts, n_counts, part, s);
    if (rc2 != KV_OK) return rc2;
    const unsigned grid = rm_grid(std::max<int64_t>(total, n_counts), sm_count);
    if (jac)
      rm_place_kernel<true><<<grid, RM_THREADS, 0, s>>>(R, counts, flags, (int64_t *)d_indptr_out, (int64_t *)d_rows_out,
                                                        (float *)d_scores_out, (int32_t *)d_inter_out, (int32_t *)d_uni_out);
    else
      rm_place_kernel<false><<<grid, RM_THREADS, 0, s>>>(R, counts, flags, (int64_t *)d_indptr_out, (int64_t *)d_rows_out,
                                                         (float *)d_scores_out, nullptr, nullptr);
    KV_CUDA(cudaGetLastError());
    return KV_OK;
  };
  rc = run();
  part.p = nullptr;
  part.cap = 0;
  unsigned bad = 0;
  if (rc == KV_OK) {
    cudaError_t e = cudaMemcpyAsync(&bad, flags, sizeof(bad), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = kv_fail(KV_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(e));
  }
  cudaFreeAsync(scratch, s);
  if (rc != KV_OK) return rc;
  if (bad & RM_BAD_INDPTR)
    return kv_fail(KV_ERR_INVALID, "%s: a run's indptr decreases, does not start at 0, or does not end at its pair count", fn);
  if (bad & RM_BAD_SCORE) return kv_fail(KV_ERR_INVALID, "%s: a NaN score", fn);
  if (bad & RM_BAD_ORDER) return kv_fail(KV_ERR_INVALID, "%s: a query's segment is not ordered by (score desc, row asc)", fn);
  if (bad & RM_DUPLICATE) return kv_fail(KV_ERR_INVALID, "%s: one (score, row) pair in two runs (runs must hold disjoint rows)", fn);
  return KV_OK;
}
