// K4: 64-bit fingerprint exact-match scan (SURVEY.md section 8 row a7, BASELINE "hash fingerprints").
//
// The reference defines fingerprint() = first 16 hex digits of sha256(signature_text)
// (services/shared/fingerprint.py:69-71) but never queries it; matching by it is an extension
// whose CPU oracle is plain integer equality (oracle/tfidf_oracle.py::fingerprint64; parity
// UNPINNED -- there is no reference output).  The index is one uint64 per row (8 B/row); a batch of
// query hashes is matched in passes of <= 4096 queries: their open-addressing set sits in shared
// memory and every CTA streams the whole hash column with 16-byte loads -- a pure HBM-bound scan.
// Matches (rare) are appended to a global list, then reduced per query to (count, first k rows).
#include "kv_cuda.cuh"

#include <algorithm>
#include <memory>
#include <mutex>
#include <vector>

namespace {

constexpr int HQ_TILE = 4096;        // queries per pass
constexpr int HQ_SLOTS = 8192;       // shared-memory table slots (64 KiB of keys + 32 KiB of ids)
// Prefilter: two bitmaps of 2^19 bits (64 KiB each), indexed by different hash bits.  One 16 KiB bitmap had 3 % of its
// bits set -- per key that is fine, per WARP it sent 62 % of the 32-key groups down the probe path (ncu: 42
// instructions per key).  <= 0.8 % set per bitmap -> the second test runs for ~22 % of the warps, the probe for ~0.2 %.
constexpr int HQ_BITS_LOG = 19;
constexpr int HQ_BIT_WORDS = 1 << (HQ_BITS_LOG - 5);  // words per bitmap; the two bitmaps are stored back to back
constexpr unsigned long long H_EMPTY = 0xFFFFFFFFFFFFFFFFULL;

__host__ __device__ __forceinline__ uint32_t hslot(unsigned long long h) {
  return (uint32_t)((h * 0x9E3779B97F4A7C15ULL) >> 51) & (HQ_SLOTS - 1);
}
// fingerprints are sha256 prefixes (uniform bits): the low bits index the prefilter directly
__host__ __device__ __forceinline__ uint32_t hbit(unsigned long long h) { return (uint32_t)h & ((1u << HQ_BITS_LOG) - 1); }
__host__ __device__ __forceinline__ uint32_t hbit2(unsigned long long h) { return (uint32_t)(h >> HQ_BITS_LOG) & ((1u << HQ_BITS_LOG) - 1); }

// table: keys[HQ_SLOTS] (global, built on the host), qidx[HQ_SLOTS] first query with that hash
__global__ void __launch_bounds__(1024) hash_scan_kernel(const ulonglong2 *__restrict__ rows2, int64_t n_rows,
                                                        const unsigned long long *__restrict__ t_keys,
                                                        const int *__restrict__ t_qidx,
                                                        const uint32_t *__restrict__ t_bits, unsigned long long *out_pairs,
                                                        unsigned int *out_count, unsigned int out_cap) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long *s_keys = (unsigned long long *)smem_raw;
  int *s_qidx = (int *)(s_keys + HQ_SLOTS);
  uint32_t *s_bits = (uint32_t *)(s_qidx + HQ_SLOTS);
  {
    const uint4 *src3 = (const uint4 *)t_bits;
    uint4 *dst3 = (uint4 *)s_bits;
    for (int i = threadIdx.x; i < 2 * HQ_BIT_WORDS / 4; i += blockDim.x) dst3[i] = src3[i];
    const uint4 *src = (const uint4 *)t_keys;
    uint4 *dst = (uint4 *)s_keys;
    for (int i = threadIdx.x; i < HQ_SLOTS / 2; i += blockDim.x) dst[i] = src[i];
    const uint4 *src2 = (const uint4 *)t_qidx;
    uint4 *dst2 = (uint4 *)s_qidx;
    for (int i = threadIdx.x; i < HQ_SLOTS / 4; i += blockDim.x) dst2[i] = src2[i];
  }
  __syncthreads();
  // persistent CTAs (one per SM); every thread keeps 4 independent 16-byte loads in flight
  const int64_t n2 = (n_rows + 1) / 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i0 < n2; i0 += 4 * stride) {
    ulonglong2 v[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int64_t i = i0 + u * stride;
      v[u].x = v[u].y = H_EMPTY;
      if (i < n2)
        asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(v[u].x), "=l"(v[u].y) : "l"(rows2 + i));
    }
#pragma unroll
    for (int x = 0; x < 8; x++) {
      const int u = x >> 1, h = x & 1;
      const unsigned long long key = h ? v[u].y : v[u].x;
      // No range or sentinel test per key: loads past the end deliver H_EMPTY, the slot after the last row is padded
      // with H_EMPTY (kv_hash_append), and H_EMPTY can never equal a stored query key -- a probe for it stops at the
      // first empty slot.  The common case is three 32-bit ALU ops, one LDS and one predicate per key.
      const uint32_t lo = (uint32_t)key;
      const uint32_t wd = s_bits[(lo >> 5) & (HQ_BIT_WORDS - 1)];
      if (!(wd & (1u << (lo & 31u)))) continue;  // > 99 % of the rows stop here (one 4-byte LDS)
      const uint32_t b2 = hbit2(key);
      if (!((s_bits[HQ_BIT_WORDS + (b2 >> 5)] >> (b2 & 31u)) & 1u)) continue;
      const int64_t row = 2 * (i0 + u * stride) + h;
      uint32_t s = hslot(key);
      for (;;) {
        unsigned long long k = s_keys[s];
        if (k == H_EMPTY) break;
        if (k == key) {
          unsigned int o = atomicAdd(out_count, 1u);
          if (o < out_cap) out_pairs[o] = ((unsigned long long)(unsigned)s_qidx[s] << 40) | (unsigned long long)row;
          break;
        }
        s = (s + 1) & (HQ_SLOTS - 1);
      }
    }
  }
}

}  // namespace

struct kv_hash_index {
  int device = 0;
  int64_t row_base = 0;
  CudaStream stream;
  CudaEvent ev[2];
  std::mutex mu;
  int sm_count = 132;
  DevVec<unsigned long long> rows;
  int64_t n_rows = 0;
  DevBuf<unsigned long long> d_keys, d_pairs;
  DevBuf<int> d_qidx;
  DevBuf<uint32_t> d_bits;
  DevBuf<unsigned int> d_count;
  float last_scan_ms = 0;
  int last_passes = 0;
};

extern "C" {

int kv_hash_create(int device, int64_t row_base, kv_hash_index **out) {
  if (!out) return kv_fail(KV_ERR_INVALID, "kv_hash_create: out is NULL");
  int sm_count = 0;
  int rc = open_device(device, "kv_hash_create", &sm_count);
  if (rc != KV_OK) return rc;
  std::unique_ptr<kv_hash_index> hx(new kv_hash_index());
  hx->device = device;
  hx->row_base = row_base;
  hx->sm_count = sm_count;
  KV_CUDA(hx->stream.create());
  for (auto &e : hx->ev) KV_CUDA(e.create());
  KV_CUDA(cudaFuncSetAttribute(hash_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, HQ_SLOTS * 12 + 2 * HQ_BIT_WORDS * 4));
  *out = hx.release();
  return KV_OK;
}

void kv_hash_destroy(kv_hash_index *hx) {
  if (!hx) return;
  cudaSetDevice(hx->device);
  cudaStreamSynchronize(hx->stream);
  delete hx;
}

int64_t kv_hash_rows(const kv_hash_index *hx) { return hx ? hx->n_rows : 0; }

int kv_hash_append(kv_hash_index *hx, const uint64_t *hashes, int64_t n) {
  if (!hx || n < 0 || (n > 0 && !hashes)) return kv_fail(KV_ERR_INVALID, "kv_hash_append: bad arguments");
  if (n == 0) return KV_OK;
  std::lock_guard<std::mutex> g(hx->mu);
  KV_CUDA(cudaSetDevice(hx->device));
  for (int64_t i = 0; i < n; i++)
    if (hashes[i] == H_EMPTY) return kv_fail(KV_ERR_INVALID, "kv_hash_append: hash 0xFFFFFFFFFFFFFFFF is reserved");
  KV_CUDA(hx->rows.reserve(hx->n_rows + n + 2, hx->stream));
  KV_CUDA(cudaMemcpyAsync(hx->rows.p + hx->n_rows, hashes, (size_t)n * 8, cudaMemcpyHostToDevice, hx->stream));
  KV_CUDA(cudaMemsetAsync(hx->rows.p + hx->n_rows + n, 0xFF, 16, hx->stream));  // H_EMPTY padding: the scan reads row pairs
  KV_CUDA(cudaStreamSynchronize(hx->stream));
  hx->n_rows += n;
  hx->rows.n = hx->n_rows;
  return KV_OK;
}

int kv_hash_match(kv_hash_index *hx, const uint64_t *q_hashes, int64_t n_q, int k, int64_t *out_rows,
                  int64_t *out_counts) {
  if (!hx || n_q < 0 || k < 1 || (n_q > 0 && (!q_hashes || !out_rows || !out_counts)))
    return kv_fail(KV_ERR_INVALID, "kv_hash_match: bad arguments");
  if (n_q >= (1LL << 23)) return kv_fail(KV_ERR_INVALID, "kv_hash_match: at most 2^23-1 queries per call");
  std::lock_guard<std::mutex> g(hx->mu);
  KV_CUDA(cudaSetDevice(hx->device));
  cudaStream_t s = hx->stream;
  for (int64_t i = 0; i < n_q * k; i++) out_rows[i] = -1;
  for (int64_t i = 0; i < n_q; i++) out_counts[i] = 0;
  if (n_q == 0 || hx->n_rows == 0) return KV_OK;
  KV_CUDA(hx->d_keys.ensure(HQ_SLOTS)); KV_CUDA(hx->d_qidx.ensure(HQ_SLOTS)); KV_CUDA(hx->d_count.ensure(1));
  KV_CUDA(hx->d_bits.ensure(2 * HQ_BIT_WORDS));
  std::vector<uint32_t> bits(2 * HQ_BIT_WORDS);
  unsigned int cap = 1u << 22;
  std::vector<unsigned long long> keys(HQ_SLOTS), pairs;
  std::vector<int> qidx(HQ_SLOTS);
  std::vector<std::vector<int>> same;  // per table entry: every query of the pass with that hash
  std::vector<std::pair<int64_t, int64_t>> all;  // (query, row)
  hx->last_scan_ms = 0;
  hx->last_passes = 0;
  for (int64_t q0 = 0; q0 < n_q; q0 += HQ_TILE) {
    const int64_t q1 = std::min(n_q, q0 + HQ_TILE);
    std::fill(keys.begin(), keys.end(), H_EMPTY);
    std::fill(qidx.begin(), qidx.end(), -1);
    std::fill(bits.begin(), bits.end(), 0u);
    same.assign((size_t)(q1 - q0), {});
    for (int64_t q = q0; q < q1; q++) {
      const unsigned long long h = q_hashes[q];
      if (h == H_EMPTY) continue;
      uint32_t sl = hslot(h);
      bits[hbit(h) >> 5] |= 1u << (hbit(h) & 31);
      bits[HQ_BIT_WORDS + (hbit2(h) >> 5)] |= 1u << (hbit2(h) & 31);
      while (keys[sl] != H_EMPTY && keys[sl] != h) sl = (sl + 1) & (HQ_SLOTS - 1);
      if (keys[sl] == H_EMPTY) { keys[sl] = h; qidx[sl] = (int)(q - q0); }
      same[(size_t)qidx[sl]].push_back((int)(q - q0));  // duplicates among the queries share one slot
    }
    for (;;) {
      KV_CUDA(hx->d_pairs.ensure(cap));
      KV_CUDA(cudaMemcpyAsync(hx->d_keys.p, keys.data(), HQ_SLOTS * 8, cudaMemcpyHostToDevice, s));
      KV_CUDA(cudaMemcpyAsync(hx->d_qidx.p, qidx.data(), HQ_SLOTS * 4, cudaMemcpyHostToDevice, s));
      KV_CUDA(cudaMemcpyAsync(hx->d_bits.p, bits.data(), 2 * HQ_BIT_WORDS * 4, cudaMemcpyHostToDevice, s));
      KV_CUDA(cudaMemsetAsync(hx->d_count.p, 0, 4, s));
      KV_CUDA(cudaEventRecord(hx->ev[0], s));
      hash_scan_kernel<<<hx->sm_count, 1024, HQ_SLOTS * 12 + 2 * HQ_BIT_WORDS * 4, s>>>((const ulonglong2 *)hx->rows.p, hx->n_rows,
                                                                    hx->d_keys.p, hx->d_qidx.p, hx->d_bits.p, hx->d_pairs.p,
                                                                    hx->d_count.p, cap);
      KV_CUDA(cudaGetLastError());
      KV_CUDA(cudaEventRecord(hx->ev[1], s));
      unsigned int cnt = 0;
      KV_CUDA(cudaMemcpyAsync(&cnt, hx->d_count.p, 4, cudaMemcpyDeviceToHost, s));
      KV_CUDA(cudaStreamSynchronize(s));
      if (cnt > cap) { cap = cnt; continue; }  // rare: more matches than the list holds -> rerun the pass
      float ms = 0;
      cudaEventElapsedTime(&ms, hx->ev[0], hx->ev[1]);
      hx->last_scan_ms += ms;
      hx->last_passes++;
      pairs.resize(cnt);
      if (cnt) KV_CUDA(cudaMemcpy(pairs.data(), hx->d_pairs.p, (size_t)cnt * 8, cudaMemcpyDeviceToHost));
      for (unsigned long long p : pairs) {
        int qi = (int)(p >> 40);
        int64_t row = (int64_t)(p & ((1ULL << 40) - 1));
        for (int dup : same[(size_t)qi]) all.emplace_back(q0 + dup, row);
      }
      break;
    }
  }
  std::sort(all.begin(), all.end());
  for (auto &m : all) {
    int64_t c = out_counts[m.first]++;
    if (c < k) out_rows[m.first * k + c] = hx->row_base + m.second;
  }
  return KV_OK;
}

int kv_hash_last_timing(const kv_hash_index *hx, float *scan_ms, int *passes) {
  if (!hx || !scan_ms || !passes) return kv_fail(KV_ERR_INVALID, "kv_hash_last_timing: bad arguments");
  *scan_ms = hx->last_scan_ms;
  *passes = hx->last_passes;
  return KV_OK;
}

}  // extern "C"
