// Device ordering of threshold-search results: the records a range scan (K1b-R, K2-R, K3-R) appended in emit order
// become the CSR the fetch functions return -- indptr by query, then each query's pairs by (score desc, row asc).
//
// An LSD radix sort of the records themselves (16 bytes each) on the composite key (query, score descending, row), one
// stable counting pass per 8-bit digit: row digits first, then score, then query.  A min/max reduction over the records
// first fixes each field's range, and only digits that vary are sorted (100k queries x 10M rows: about 9 passes).
// A pass is three steps: per-tile digit counts, an exclusive scan of the counts in digit-major order, and a stable
// scatter in which every tile ranks its records digit by digit with warp match masks.  indptr then comes from a binary
// search of each query in the sorted records.  Scores are positive (they reach a threshold in (0, 1]); the key maps
// float32 bits to an order-preserving unsigned value all the same.  The Jaccard score is __fdiv_rn(inter, uni), the
// bits the host's IEEE division of the two integer-valued floats gives.
//
// A host fetch of fewer than RANGE_HOST_ORDER_MAX pairs plus queries copies the records back and orders them on one
// host core instead (host_order): below that size the device ordering's fixed cost is larger than the sort (DESIGN §6).
#include "kv_cuda.cuh"

#include <cstring>
#include <new>
#include <type_traits>
#include <vector>

namespace {

constexpr int RO_THREADS = 256, RO_WARPS = RO_THREADS / 32, RO_ROUNDS = 16;
constexpr int64_t RO_TILE = (int64_t)RO_THREADS * RO_ROUNDS;  // records per tile of a pass, entries per tile of a scan
constexpr unsigned long long SIGN64 = 1ull << 63;

enum : int { F_ROW = 0, F_SCORE = 1, F_QUERY = 2 };

static_assert(sizeof(RangePair) == 16 && sizeof(JaccardPair) == 16, "records move as one 16-byte word");

template <class Rec>
__device__ __forceinline__ Rec ld_rec(const Rec *p) {
  const int4 v = *reinterpret_cast<const int4 *>(p);
  Rec r;
  memcpy(&r, &v, sizeof(r));
  return r;
}

template <class Rec>
__device__ __forceinline__ void st_rec(Rec *p, const Rec &r) {
  int4 v;
  memcpy(&v, &r, sizeof(v));
  *reinterpret_cast<int4 *>(p) = v;
}

__device__ __forceinline__ float rec_score(const RangePair &p) { return p.score; }
__device__ __forceinline__ float rec_score(const JaccardPair &p) { return __fdiv_rn((float)p.inter, (float)p.uni); }

// unsigned order of the result = float order of s (NaN excluded)
__device__ __forceinline__ unsigned score_key(float s) {
  const unsigned b = __float_as_uint(s);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// unsigned order of the result = signed order of the row
__device__ __forceinline__ unsigned long long row_key(const RangePair &p) { return (unsigned long long)p.row ^ SIGN64; }
__device__ __forceinline__ unsigned long long row_key(const JaccardPair &p) {
  return (unsigned long long)(long long)p.row ^ SIGN64;
}

// The digit of a pass: bits [shift, shift + 8) of the field's key relative to `base` (the field's minimum, or for the
// score its maximum, so that higher scores come first).
template <class Rec>
__device__ __forceinline__ unsigned rec_digit(const Rec &r, int field, int shift, unsigned long long base) {
  unsigned long long k;
  if (field == F_ROW) k = row_key(r) - base;
  else if (field == F_SCORE) k = base - score_key(rec_score(r));
  else k = (unsigned long long)(unsigned)r.q - base;
  return (unsigned)(k >> shift) & 255u;
}

// Exclusive scan of one value per thread over the block; *total (optional) receives the sum.
__device__ __forceinline__ unsigned block_exclusive_scan(unsigned v, unsigned *total) {
  __shared__ unsigned ws[RO_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xFFFFFFFFu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) ws[warp] = x;
  __syncthreads();
  if (warp == 0) {
    unsigned w = lane < RO_WARPS ? ws[lane] : 0;
    for (int o = 1; o < RO_WARPS; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xFFFFFFFFu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < RO_WARPS) ws[lane] = w;
  }
  __syncthreads();
  const unsigned pre = warp ? ws[warp - 1] : 0;
  if (total) *total = ws[RO_WARPS - 1];
  __syncthreads();  // ws is reused by the next call
  return pre + x - v;
}

// st[0..5] = min / max of the query, of score_key and of row_key over the n records
template <class Rec>
__global__ void __launch_bounds__(RO_THREADS) ro_minmax_kernel(const Rec *in, int64_t n, unsigned long long *st) {
  unsigned qlo = ~0u, qhi = 0, slo = ~0u, shi = 0;
  unsigned long long rlo = ~0ull, rhi = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const Rec r = ld_rec(in + i);
    const unsigned q = (unsigned)r.q, s = score_key(rec_score(r));
    const unsigned long long w = row_key(r);
    qlo = min(qlo, q); qhi = max(qhi, q);
    slo = min(slo, s); shi = max(shi, s);
    rlo = min(rlo, w); rhi = max(rhi, w);
  }
  qlo = __reduce_min_sync(0xFFFFFFFFu, qlo); qhi = __reduce_max_sync(0xFFFFFFFFu, qhi);
  slo = __reduce_min_sync(0xFFFFFFFFu, slo); shi = __reduce_max_sync(0xFFFFFFFFu, shi);
  for (int o = 16; o; o >>= 1) {
    rlo = min(rlo, __shfl_xor_sync(0xFFFFFFFFu, rlo, o));
    rhi = max(rhi, __shfl_xor_sync(0xFFFFFFFFu, rhi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMin(&st[0], (unsigned long long)qlo); atomicMax(&st[1], (unsigned long long)qhi);
    atomicMin(&st[2], (unsigned long long)slo); atomicMax(&st[3], (unsigned long long)shi);
    atomicMin(&st[4], rlo); atomicMax(&st[5], rhi);
  }
}

// counts[d * n_tiles + t] = records of tile t whose digit is d
template <class Rec>
__global__ void __launch_bounds__(RO_THREADS) ro_count_kernel(const Rec *in, int64_t n, int field, int shift,
                                                               unsigned long long base, unsigned *counts, int64_t n_tiles) {
  __shared__ unsigned h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t t0 = (int64_t)blockIdx.x * RO_TILE;
  const unsigned lane_lt = (1u << (threadIdx.x & 31)) - 1;
  for (int r = 0; r < RO_ROUNDS; r++) {
    const int64_t i = t0 + (int64_t)r * RO_THREADS + threadIdx.x;
    const unsigned d = i < n ? rec_digit(ld_rec(in + i), field, shift, base) : 256u;
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, d);  // one shared atomic per distinct digit of the warp
    if (d < 256u && (peers & lane_lt) == 0) atomicAdd(&h[d], (unsigned)__popc(peers));
  }
  __syncthreads();
  counts[(int64_t)threadIdx.x * n_tiles + blockIdx.x] = h[threadIdx.x];
}

// Exclusive scan of x[0, m) in place: tile sums (ro_scan_reduce_kernel), their scan in one block
// (ro_scan_partials_kernel), then every tile's scan from its carry (ro_scan_down_kernel).
__global__ void __launch_bounds__(RO_THREADS) ro_scan_reduce_kernel(const unsigned *x, int64_t m, unsigned *part) {
  const int64_t t0 = (int64_t)blockIdx.x * RO_TILE;
  unsigned s = 0;
  for (int r = 0; r < RO_ROUNDS; r++) {
    const int64_t i = t0 + (int64_t)r * RO_THREADS + threadIdx.x;
    if (i < m) s += x[i];
  }
  unsigned total;
  block_exclusive_scan(s, &total);
  if (threadIdx.x == 0) part[blockIdx.x] = total;
}

__global__ void __launch_bounds__(RO_THREADS) ro_scan_partials_kernel(unsigned *part, int64_t np) {
  unsigned carry = 0;
  for (int64_t b = 0; b < np; b += RO_THREADS) {
    const int64_t i = b + threadIdx.x;
    const unsigned v = i < np ? part[i] : 0;
    unsigned total;
    const unsigned e = block_exclusive_scan(v, &total);
    if (i < np) part[i] = carry + e;
    carry += total;
  }
}

__global__ void __launch_bounds__(RO_THREADS) ro_scan_down_kernel(unsigned *x, int64_t m, const unsigned *part) {
  const int64_t t0 = (int64_t)blockIdx.x * RO_TILE + (int64_t)threadIdx.x * RO_ROUNDS;
  unsigned v[RO_ROUNDS], s = 0;
#pragma unroll
  for (int k = 0; k < RO_ROUNDS; k++) {
    v[k] = t0 + k < m ? x[t0 + k] : 0;
    s += v[k];
  }
  unsigned e = block_exclusive_scan(s, nullptr) + part[blockIdx.x];
#pragma unroll
  for (int k = 0; k < RO_ROUNDS; k++) {
    if (t0 + k < m) x[t0 + k] = e;
    e += v[k];
  }
}

// Stable scatter of one pass.  A tile is RO_ROUNDS rounds of RO_THREADS consecutive records.  In a round, each warp
// ranks its 32 records among equal digits (match mask), writes per-digit counts, and thread d turns column d of those
// counts into the output bases of warps 0..7 for digit d, starting from the tile's running offset run[d].  The two
// count buffers alternate between rounds, so a round's clearing never races the previous round's scatter.
template <class Rec>
__global__ void __launch_bounds__(RO_THREADS) ro_scatter_kernel(const Rec *in, Rec *out, int64_t n, int field, int shift,
                                                                 unsigned long long base, const unsigned *offs,
                                                                 int64_t n_tiles) {
  __shared__ unsigned run[256];
  __shared__ unsigned wc[2][RO_WARPS][256];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  run[tid] = offs[(int64_t)tid * n_tiles + blockIdx.x];
  const int64_t t0 = (int64_t)blockIdx.x * RO_TILE;
  for (int r = 0; r < RO_ROUNDS; r++) {
    unsigned (*c)[256] = wc[r & 1];
#pragma unroll
    for (int w = 0; w < RO_WARPS; w++) c[w][tid] = 0;
    __syncthreads();
    const int64_t i = t0 + (int64_t)r * RO_THREADS + tid;
    const bool valid = i < n;
    Rec rec{};
    unsigned d = 256u;
    if (valid) {
      rec = ld_rec(in + i);
      d = rec_digit(rec, field, shift, base);
    }
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, d);
    const unsigned rank = __popc(peers & ((1u << lane) - 1));
    if (valid && rank == 0) c[warp][d] = __popc(peers);
    __syncthreads();
    unsigned s = run[tid];
#pragma unroll
    for (int w = 0; w < RO_WARPS; w++) {
      const unsigned x = c[w][tid];
      c[w][tid] = s;
      s += x;
    }
    run[tid] = s;
    __syncthreads();
    if (valid) st_rec(out + c[warp][d] + rank, rec);
  }
}

// rows / scores (/ inter / uni) of the ordered records
template <class Rec>
__global__ void __launch_bounds__(RO_THREADS) ro_emit_kernel(const Rec *in, int64_t n, int64_t row_base, int64_t *rows,
                                                              float *scores, int32_t *inter, int32_t *uni) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const Rec r = ld_rec(in + i);
    if constexpr (std::is_same_v<Rec, JaccardPair>) {
      rows[i] = row_base + r.row;
      inter[i] = r.inter;
      uni[i] = r.uni;
    } else {
      rows[i] = r.row;
    }
    scores[i] = rec_score(r);
  }
}

// indptr[q] = first record of query q or later (q = 0..n_q), by binary search of the ordered records
template <class Rec>
__global__ void __launch_bounds__(RO_THREADS) ro_indptr_kernel(const Rec *in, int64_t n, int64_t n_q, int64_t *indptr) {
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q <= n_q; q += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if ((int64_t)in[mid].q < q) lo = mid + 1;
      else hi = mid;
    }
    indptr[q] = lo;
  }
}

inline unsigned grid_for(int64_t n) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + RO_THREADS - 1) / RO_THREADS, 1 << 16)); }

inline int key_bits(unsigned long long range) { return range ? 64 - __builtin_clzll(range) : 0; }

}  // namespace

int check_device_ptr(const void *p, int device, size_t align, const char *what, const char *fn) {
  cudaPointerAttributes a;
  if (!p || cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return kv_fail(KV_ERR_INVALID, "%s: %s is not a device pointer", fn, what);
  }
  if (a.type != cudaMemoryTypeDevice || a.device != device)
    return kv_fail(KV_ERR_INVALID, "%s: %s is not device memory of device %d", fn, what, device);
  if ((uintptr_t)p % align != 0) return kv_fail(KV_ERR_INVALID, "%s: %s is not aligned to %zu bytes", fn, what, align);
  return KV_OK;
}

template <class Rec>
int range_order_device(Rec *rec, int64_t n, int64_t n_q, int64_t row_base, int64_t *indptr, int64_t *rows, float *scores,
                       int32_t *inter, int32_t *uni, RangeOrderScratch &sc, cudaStream_t s, const char *fn) {
  Rec *cur = rec;
  if (n > 1) {
    // offsets are 32-bit: 2^32 records would be 64 GB before any scratch
    if (n > (int64_t)0xFFFFFFFFll - RO_TILE)
      return kv_fail(KV_ERR_NOMEM, "%s: %lld pairs: too many to order on the device", fn, (long long)n);
    const int64_t n_tiles = (n + RO_TILE - 1) / RO_TILE, m = 256 * n_tiles, n_part = (m + RO_TILE - 1) / RO_TILE;
    if (sc.alt.ensure(n) != cudaSuccess || sc.counts.ensure(m) != cudaSuccess || sc.partials.ensure(n_part) != cudaSuccess ||
        sc.stats.ensure(6) != cudaSuccess) {
      cudaGetLastError();
      return kv_fail(KV_ERR_NOMEM, "%s: %lld pairs: the scratch of their device ordering does not fit in device memory "
                                   "(raise the threshold or split the query batch)", fn, (long long)n);
    }
    unsigned long long st[6] = {~0ull, 0, ~0ull, 0, ~0ull, 0};
    KV_CUDA(cudaMemcpyAsync(sc.stats.p, st, sizeof(st), cudaMemcpyHostToDevice, s));
    ro_minmax_kernel<Rec><<<grid_for(n), RO_THREADS, 0, s>>>(rec, n, sc.stats.p);
    KV_CUDA(cudaGetLastError());
    KV_CUDA(cudaMemcpyAsync(st, sc.stats.p, sizeof(st), cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaStreamSynchronize(s));
    struct Pass { int field, shift; unsigned long long base; };
    Pass passes[24];
    int n_passes = 0;
    const unsigned long long range[3] = {st[5] - st[4], st[3] - st[2], st[1] - st[0]};
    const unsigned long long base[3] = {st[4], st[3], st[0]};
    for (int f : {F_ROW, F_SCORE, F_QUERY})
      for (int sh = 0; sh < key_bits(range[f]); sh += 8) passes[n_passes++] = Pass{f, sh, base[f]};
    Rec *other = reinterpret_cast<Rec *>(sc.alt.p);
    for (int p = 0; p < n_passes; p++) {
      const Pass &P = passes[p];
      ro_count_kernel<Rec><<<(unsigned)n_tiles, RO_THREADS, 0, s>>>(cur, n, P.field, P.shift, P.base, sc.counts.p, n_tiles);
      ro_scan_reduce_kernel<<<(unsigned)n_part, RO_THREADS, 0, s>>>(sc.counts.p, m, sc.partials.p);
      ro_scan_partials_kernel<<<1, RO_THREADS, 0, s>>>(sc.partials.p, n_part);
      ro_scan_down_kernel<<<(unsigned)n_part, RO_THREADS, 0, s>>>(sc.counts.p, m, sc.partials.p);
      ro_scatter_kernel<Rec><<<(unsigned)n_tiles, RO_THREADS, 0, s>>>(cur, other, n, P.field, P.shift, P.base, sc.counts.p,
                                                                      n_tiles);
      KV_CUDA(cudaGetLastError());
      std::swap(cur, other);
    }
  }
  if (n > 0) {
    ro_emit_kernel<Rec><<<grid_for(n), RO_THREADS, 0, s>>>(cur, n, row_base, rows, scores, inter, uni);
    KV_CUDA(cudaGetLastError());
  }
  ro_indptr_kernel<Rec><<<grid_for(n_q + 1), RO_THREADS, 0, s>>>(cur, n, n_q, indptr);
  KV_CUDA(cudaGetLastError());
  return KV_OK;
}

namespace {
inline float host_score(const RangePair &p) { return p.score; }
inline float host_score(const JaccardPair &p) { return (float)p.inter / (float)p.uni; }  // IEEE: the bits of __fdiv_rn

// The ordering on one host core: a counting sort by query, then each query's segment by (score desc, row asc).
template <class Rec>
int host_order(const Rec *rec, int64_t n, int64_t n_q, int64_t row_base, int64_t *indptr, int64_t *rows, float *scores,
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
  for (int64_t q = 0; q < n_q; q++)
    std::sort(by_q.begin() + indptr[q], by_q.begin() + indptr[q + 1], [](const Rec &x, const Rec &y) {
      const float sx = host_score(x), sy = host_score(y);
      return sx != sy ? sx > sy : x.row < y.row;
    });
  for (int64_t i = 0; i < n; i++) {
    const Rec &p = by_q[(size_t)i];
    scores[i] = host_score(p);
    if constexpr (std::is_same_v<Rec, JaccardPair>) {
      rows[i] = row_base + p.row;
      inter[i] = p.inter;
      uni[i] = p.uni;
    } else {
      rows[i] = p.row;
    }
  }
  return KV_OK;
}

// range_order_device into sc.out, then the ordered arrays copied to the host
template <class Rec>
int device_order_to_host(Rec *rec, int64_t n, int64_t n_q, int64_t row_base, int64_t *indptr, int64_t *rows, float *scores,
                         int32_t *inter, int32_t *uni, RangeOrderScratch &sc, cudaStream_t s, const char *fn) {
  constexpr bool jac = std::is_same_v<Rec, JaccardPair>;
  const int64_t bytes = (n_q + 1) * 8 + n * (jac ? 20 : 12);
  if (sc.out.ensure(bytes) != cudaSuccess) {
    cudaGetLastError();
    return kv_fail(KV_ERR_NOMEM, "%s: %lld pairs: their ordered arrays do not fit in device memory", fn, (long long)n);
  }
  int64_t *d_indptr = reinterpret_cast<int64_t *>(sc.out.p), *d_rows = d_indptr + (n_q + 1);
  float *d_scores = reinterpret_cast<float *>(d_rows + n);
  int32_t *d_inter = jac ? reinterpret_cast<int32_t *>(d_scores + n) : nullptr, *d_uni = jac ? d_inter + n : nullptr;
  int rc = range_order_device(rec, n, n_q, row_base, d_indptr, d_rows, d_scores, d_inter, d_uni, sc, s, fn);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaMemcpyAsync(indptr, d_indptr, (size_t)(n_q + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  if (n > 0) {
    KV_CUDA(cudaMemcpyAsync(rows, d_rows, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaMemcpyAsync(scores, d_scores, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if constexpr (jac) {
      KV_CUDA(cudaMemcpyAsync(inter, d_inter, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
      KV_CUDA(cudaMemcpyAsync(uni, d_uni, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    }
  }
  KV_CUDA(cudaStreamSynchronize(s));
  return KV_OK;
}
}  // namespace

template <class Rec>
int range_order_to_host(Rec *rec, int64_t n, int64_t n_q, int64_t row_base, int64_t *indptr, int64_t *rows, float *scores,
                        int32_t *inter, int32_t *uni, RangeOrderScratch &sc, cudaStream_t s, const char *fn) {
  if (n + n_q >= RANGE_HOST_ORDER_MAX)
    return device_order_to_host(rec, n, n_q, row_base, indptr, rows, scores, inter, uni, sc, s, fn);
  // few pairs over few queries: the records come back (16 B each) and one host core orders them (work n + n_q) in less
  // time than the device ordering's fixed cost (a min/max read-back and some forty launches; DESIGN §6)
  if (sc.staged.ensure(std::max<int64_t>(n, 1)) != cudaSuccess) {
    cudaGetLastError();
    return kv_fail(KV_ERR_NOMEM, "%s: out of pinned host memory", fn);
  }
  if (n) KV_CUDA(cudaMemcpyAsync(sc.staged.p, rec, (size_t)n * sizeof(Rec), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  return host_order(reinterpret_cast<const Rec *>(sc.staged.p), n, n_q, row_base, indptr, rows, scores, inter, uni, fn);
}

template int range_order_device<RangePair>(RangePair *, int64_t, int64_t, int64_t, int64_t *, int64_t *, float *, int32_t *,
                                           int32_t *, RangeOrderScratch &, cudaStream_t, const char *);
template int range_order_device<JaccardPair>(JaccardPair *, int64_t, int64_t, int64_t, int64_t *, int64_t *, float *,
                                             int32_t *, int32_t *, RangeOrderScratch &, cudaStream_t, const char *);
template int range_order_to_host<RangePair>(RangePair *, int64_t, int64_t, int64_t, int64_t *, int64_t *, float *, int32_t *,
                                            int32_t *, RangeOrderScratch &, cudaStream_t, const char *);
template int range_order_to_host<JaccardPair>(JaccardPair *, int64_t, int64_t, int64_t, int64_t *, int64_t *, float *,
                                              int32_t *, int32_t *, RangeOrderScratch &, cudaStream_t, const char *);

extern "C" int kv_debug_range_order(int device, int jaccard, const void *records, int64_t n, int64_t n_q, int64_t row_base,
                                    int64_t *indptr, int64_t *rows, float *scores, int32_t *inter, int32_t *uni) {
  const char *fn = "kv_debug_range_order";
  if (n < 0 || n_q < 0 || n_q >= (1LL << 31) || !indptr || (n > 0 && (!records || !rows || !scores)) ||
      (jaccard && n > 0 && (!inter || !uni)))
    return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  // the records a scan emits: a query of the batch, a finite score (Jaccard: 0 <= inter <= uni, uni >= 1)
  for (int64_t i = 0; i < n; i++) {
    int32_t q;
    memcpy(&q, (const char *)records + i * 16, sizeof(q));
    if (q < 0 || q >= n_q) return kv_fail(KV_ERR_INVALID, "%s: record %lld: query %d outside 0..%lld", fn, (long long)i, q, (long long)n_q);
    if (jaccard) {
      JaccardPair p;
      memcpy(&p, (const char *)records + i * 16, sizeof(p));
      if (p.uni < 1 || p.inter < 0 || p.inter > p.uni) return kv_fail(KV_ERR_INVALID, "%s: record %lld: bad counts", fn, (long long)i);
    } else {
      RangePair p;
      memcpy(&p, (const char *)records + i * 16, sizeof(p));
      if (!(p.score == p.score)) return kv_fail(KV_ERR_INVALID, "%s: record %lld: NaN score", fn, (long long)i);
    }
  }
  int sm_count = 0;
  int rc = open_device(device, fn, &sm_count);
  if (rc != KV_OK) return rc;
  CudaStream s;
  KV_CUDA(s.create());
  DevBuf<int4> d_rec;
  RangeOrderScratch sc;
  if (d_rec.ensure(std::max<int64_t>(n, 1)) != cudaSuccess) {
    cudaGetLastError();
    return kv_fail(KV_ERR_NOMEM, "%s: %lld records do not fit in device memory", fn, (long long)n);
  }
  if (n) KV_CUDA(cudaMemcpyAsync(d_rec.p, records, (size_t)n * 16, cudaMemcpyHostToDevice, s));
  // always the device ordering, whatever the size
  if (jaccard)
    rc = device_order_to_host(reinterpret_cast<JaccardPair *>(d_rec.p), n, n_q, row_base, indptr, rows, scores, inter, uni, sc,
                              s, fn);
  else
    rc = device_order_to_host(reinterpret_cast<RangePair *>(d_rec.p), n, n_q, 0, indptr, rows, scores, nullptr, nullptr, sc, s,
                              fn);
  cudaStreamSynchronize(s);
  return rc;
}
