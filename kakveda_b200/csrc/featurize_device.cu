// Device featuriser: kv_featurize(grow = 0) on the GPU, against a mirror of the vocabulary in HBM.
//
// The output is bit-identical to the host featuriser's (featurizer.cpp): the same tokens, the same MurmurHash3 keys,
// features in order of first appearance (t0, t0 t1, t1, t1 t2, ...), tf as counts and oov as the sum of tf^2 of the
// features the vocabulary lacks.  The batch is processed in flat arrays rather than one document per warp, so short and
// long documents take the same path:
//   1. tokens per document (one thread per document, a serial walk over its bytes; raw-mode non-ASCII detection);
//   2. an exclusive scan of the token counts; the token spans are written by a second walk;
//   3. occurrence g of the batch is token g/2 (g even) or the bigram of tokens g/2 and g/2+1 (g odd, when both belong
//      to one document), so occurrences are numbered in document order and, inside a document, in position order.
//      One thread per occurrence hashes it;
//   4. a batch-wide open-addressing table keyed by (document, key) counts the occurrences of every feature and keeps
//      the smallest occurrence number (atomicMin): that occurrence is the feature's first appearance;
//   5. the first occurrence of each feature looks its key up in the mirror: a hit keeps (id, tf), a miss adds tf^2 to
//      its document's oov (integer-valued doubles: the sum is exact in any order below 2^53);
//   6. an exclusive scan of the kept flags places the kept features; indptr is the scan at each document's first
//      occurrence.
#include "kv_cuda.cuh"

#include <chrono>
#include <memory>
#include <mutex>
#include <thread>
#include <utility>
#include <vector>

namespace {

constexpr uint32_t FZ_EMPTY = 0xFFFFFFFFu;
constexpr uint32_t TOK_RAW = 0x80000000u;  // tok_len flag: a raw-text token (A-Z are lower-cased when hashed)
constexpr int FZ_THREADS = 256;
constexpr uint64_t MURMUR_SEED = 0x6b616b76ULL;

inline unsigned fz_grid(int64_t n) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + FZ_THREADS - 1) / FZ_THREADS, (int64_t)1 << 20));
}

__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t fmix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return k;
}

__device__ __forceinline__ bool is_word(unsigned c) { return (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '_'; }

// The bytes of one feature without materialising it: token a, or token a + ' ' + token b.
struct FeatBytes {
  const uint8_t *a, *b;
  uint32_t la, lb;
  bool lower, bigram;
  __device__ __forceinline__ uint32_t len() const { return bigram ? la + 1 + lb : la; }
  __device__ __forceinline__ unsigned byte(uint32_t i) const {
    unsigned c;
    if (i < la) c = a[i];
    else if (i == la) return ' ';
    else c = b[i - la - 1];
    if (lower && c >= 'A' && c <= 'Z') c += 32;
    return c;
  }
  // little-endian load of n <= 8 bytes at i
  __device__ __forceinline__ uint64_t word(uint32_t i, uint32_t n) const {
    uint64_t w = 0;
    for (uint32_t k = 0; k < n; k++) w |= (uint64_t)byte(i + k) << (8 * k);
    return w;
  }
};

// MurmurHash3 x64 128 (featurizer.cpp hash128), seed 0x6b616b76 for both halves
__device__ ulonglong2 murmur128(const FeatBytes &f) {
  const uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
  const uint32_t len = f.len(), nblocks = len / 16;
  uint64_t h1 = MURMUR_SEED, h2 = MURMUR_SEED;
  for (uint32_t i = 0; i < nblocks; i++) {
    uint64_t k1 = f.word(16 * i, 8), k2 = f.word(16 * i + 8, 8);
    k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
    h1 = rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
    k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;
    h2 = rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
  }
  const uint32_t rem = len & 15, t0 = 16 * nblocks;
  if (rem > 8) {
    uint64_t k2 = f.word(t0 + 8, rem - 8);
    k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;
  }
  if (rem > 0) {
    uint64_t k1 = f.word(t0, rem < 8 ? rem : 8);
    k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
  }
  h1 ^= len; h2 ^= len; h1 += h2; h2 += h1;
  h1 = fmix64(h1); h2 = fmix64(h2);
  h1 += h2; h2 += h1;
  return make_ulonglong2(h1, h2);
}

// Walks document d (bytes [a, b) of the batch) the way featurizer.cpp tokenize() does.  WRITE = false: stores the token
// count in n_tok[d] and reports a non-ASCII raw document in *bad (the smallest such d).  WRITE = true: writes the spans
// from position n_tok[d] (the scanned counts).
template <bool WRITE>
__global__ void __launch_bounds__(FZ_THREADS) tokenize_kernel(const uint8_t *text, const int64_t *offsets, int64_t n_docs,
                                                              int mode, uint32_t *n_tok, uint32_t *tok_start,
                                                              uint32_t *tok_len, uint32_t *tok_doc,
                                                              unsigned long long *bad) {
  for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < n_docs; d += (int64_t)gridDim.x * blockDim.x) {
    uint32_t a = (uint32_t)(offsets[d] - offsets[0]), b = (uint32_t)(offsets[d + 1] - offsets[0]);
    bool pre = mode == KV_TEXT_TOKENS;
    if (mode == KV_TEXT_MIXED && b > a && text[a] == 0x1F) { pre = true; a++; }
    uint32_t k = WRITE ? n_tok[d] : 0;
    auto emit = [&](uint32_t s, uint32_t len, bool raw) {
      if (WRITE) {
        tok_start[k] = s;
        tok_len[k] = len | (raw ? TOK_RAW : 0u);
        tok_doc[k] = (uint32_t)d;
      }
      k++;
    };
    if (pre) {
      uint32_t s = a;
      for (uint32_t i = a; i <= b; i++)
        if (i == b || text[i] == 0x1F) {
          if (i > s) emit(s, i - s, false);
          s = i + 1;
        }
    } else {
      uint32_t run = 0;
      bool ascii = true;
      for (uint32_t i = a; i < b; i++) {
        unsigned c = text[i];
        if (c >= 0x80) { ascii = false; break; }
        if (c >= 'A' && c <= 'Z') c += 32;
        if (is_word(c)) {
          run++;
        } else {
          if (run >= 2) emit(i - run, run, true);
          run = 0;
        }
      }
      if (!ascii) {
        if (!WRITE) atomicMin(bad, (unsigned long long)d);
        k = WRITE ? n_tok[d] : 0;
        continue;
      }
      if (run >= 2) emit(b - run, run, true);
    }
    if (!WRITE) n_tok[d] = k;
  }
}

// Occurrence g exists: a unigram, or a bigram whose second token is in the same document.
__device__ __forceinline__ bool occ_exists(uint32_t g, uint32_t n_tok, const uint32_t *tok_doc) {
  const uint32_t t = g >> 1;
  return !(g & 1) || (t + 1 < n_tok && tok_doc[t + 1] == tok_doc[t]);
}

__global__ void __launch_bounds__(FZ_THREADS) hash_kernel(const uint8_t *text, uint32_t n_tok, const uint32_t *tok_start,
                                                          const uint32_t *tok_len, const uint32_t *tok_doc, ulonglong2 *occ_h) {
  for (int64_t gg = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; gg < 2 * (int64_t)n_tok; gg += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t g = (uint32_t)gg;
    if (!occ_exists(g, n_tok, tok_doc)) continue;
    const uint32_t t = g >> 1, la = tok_len[t];
    FeatBytes f;
    f.a = text + tok_start[t];
    f.la = la & ~TOK_RAW;
    f.lower = (la & TOK_RAW) != 0;
    f.bigram = (g & 1) != 0;
    f.b = f.bigram ? text + tok_start[t + 1] : nullptr;
    f.lb = f.bigram ? tok_len[t + 1] & ~TOK_RAW : 0;
    occ_h[g] = murmur128(f);
  }
}

__device__ __forceinline__ uint64_t dedup_home(ulonglong2 h, uint32_t doc) {
  const uint64_t x = h.x ^ ((uint64_t)doc * 0x9E3779B97F4A7C15ull);
  return x ^ (x >> 29);
}

__device__ __forceinline__ bool same_feature(uint32_t f, uint32_t doc, ulonglong2 h, const uint32_t *tok_doc,
                                             const ulonglong2 *occ_h) {
  if (tok_doc[f >> 1] != doc) return false;
  const ulonglong2 o = occ_h[f];
  return o.x == h.x && o.y == h.y;
}

// (document, feature) -> smallest occurrence number and count
__global__ void __launch_bounds__(FZ_THREADS) dedup_insert_kernel(uint32_t n_tok, const uint32_t *tok_doc,
                                                                  const ulonglong2 *occ_h, uint32_t *first, uint32_t *cnt,
                                                                  uint64_t mask) {
  for (int64_t gg = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; gg < 2 * (int64_t)n_tok; gg += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t g = (uint32_t)gg;
    if (!occ_exists(g, n_tok, tok_doc)) continue;
    const uint32_t doc = tok_doc[g >> 1];
    const ulonglong2 h = occ_h[g];
    for (uint64_t j = dedup_home(h, doc) & mask;; j = (j + 1) & mask) {
      uint32_t f = first[j];
      if (f == FZ_EMPTY) {
        f = atomicCAS(&first[j], FZ_EMPTY, g);
        if (f == FZ_EMPTY) { atomicAdd(&cnt[j], 1u); break; }
      }
      if (same_feature(f, doc, h, tok_doc, occ_h)) {  // any occurrence the slot names has the slot's feature
        atomicMin(&first[j], g);
        atomicAdd(&cnt[j], 1u);
        break;
      }
    }
  }
}

__device__ __forceinline__ uint32_t mirror_find(const ulonglong2 *keys, const uint32_t *ids, uint64_t mask, ulonglong2 h) {
  for (uint64_t j = h.x & mask;; j = (j + 1) & mask) {
    const uint32_t id = ids[j];
    if (id == FZ_EMPTY) return FZ_EMPTY;
    const ulonglong2 k = keys[j];
    if (k.x == h.x && k.y == h.y) return id;
  }
}

// keep[g] = 1 for the first occurrence of an in-vocabulary feature (with its id and tf); oov of the others
__global__ void __launch_bounds__(FZ_THREADS) resolve_kernel(uint32_t n_tok, const uint32_t *tok_doc, const ulonglong2 *occ_h,
                                                             const uint32_t *first, const uint32_t *cnt, uint64_t mask,
                                                             const ulonglong2 *vkeys, const uint32_t *vids, uint64_t vmask,
                                                             uint32_t *keep, uint32_t *occ_id, uint32_t *occ_tf, double *oov) {
  for (int64_t gg = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; gg <= 2 * (int64_t)n_tok; gg += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t g = (uint32_t)gg;
    uint32_t kept = 0;
    if (g < 2 * n_tok && occ_exists(g, n_tok, tok_doc)) {
      const uint32_t doc = tok_doc[g >> 1];
      const ulonglong2 h = occ_h[g];
      uint64_t j = dedup_home(h, doc) & mask;
      while (!same_feature(first[j], doc, h, tok_doc, occ_h)) j = (j + 1) & mask;
      if (first[j] == g) {
        const uint32_t tf = cnt[j], id = mirror_find(vkeys, vids, vmask, h);
        if (id != FZ_EMPTY) {
          kept = 1;
          occ_id[g] = id;
          occ_tf[g] = tf;
        } else {
          atomicAdd(&oov[doc], (double)tf * (double)tf);
        }
      }
    }
    keep[g] = kept;
  }
}

// pos = exclusive scan of keep (2 n_tok + 1 entries): kept features to their places, indptr from the documents' first
// occurrences (tok_off = exclusive scan of the token counts, n_docs + 1 entries)
__global__ void __launch_bounds__(FZ_THREADS) emit_kernel(uint32_t n_tok, const uint32_t *pos, const uint32_t *occ_id,
                                                          const uint32_t *occ_tf, uint32_t *ids, uint32_t *tf) {
  for (int64_t gg = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; gg < 2 * (int64_t)n_tok; gg += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t g = (uint32_t)gg;
    if (pos[g + 1] != pos[g]) {
      ids[pos[g]] = occ_id[g];
      tf[pos[g]] = occ_tf[g];
    }
  }
}

__global__ void __launch_bounds__(FZ_THREADS) indptr_kernel(int64_t n_docs, const uint32_t *tok_off, const uint32_t *pos,
                                                            int64_t *indptr) {
  for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d <= n_docs; d += (int64_t)gridDim.x * blockDim.x)
    indptr[d] = pos ? (int64_t)pos[2 * (uint64_t)tok_off[d]] : 0;
}

__global__ void __launch_bounds__(FZ_THREADS) mirror_insert_kernel(ulonglong2 *keys, uint32_t *ids, uint64_t mask,
                                                                   const ulonglong2 *src, const uint32_t *src_ids,
                                                                   uint32_t id0, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t id = src_ids ? src_ids[i] : id0 + (uint32_t)i;
    if (id == FZ_EMPTY) continue;
    const ulonglong2 k = src[i];
    uint64_t j = k.x & mask;
    while (atomicCAS(&ids[j], FZ_EMPTY, id) != FZ_EMPTY) j = (j + 1) & mask;  // keys are distinct: no comparison
    keys[j] = k;
  }
}

}  // namespace

struct kv_vocab_mirror {
  int device = 0;
  std::mutex mu;
  CudaStream stream;
  const kv_vocab *vocab = nullptr;  // the vocabulary this mirror follows (set by the first sync)
  // the table: keys and ids by slot, cap a power of two >= 2 n
  DevBuf<ulonglong2> keys;
  DevBuf<uint32_t> ids;
  int64_t cap = 0, n = 0;
  DevBuf<ulonglong2> staged;
  // featurisation scratch
  DevBuf<uint8_t> text;
  DevBuf<int64_t> offsets;
  DevBuf<uint32_t> tok_off, tok_start, tok_len, tok_doc, first, cnt, keep, occ_id, occ_tf;
  DevBuf<ulonglong2> occ_h;
  DevBuf<unsigned> part;
  DevBuf<unsigned long long> bad;
  // outputs of kv_featurize_device
  DevBuf<int64_t> o_indptr;
  DevBuf<uint32_t> o_ids, o_tf;
  DevBuf<double> o_oov;
};

int mirror_device(const kv_vocab_mirror *m) { return m->device; }
void mirror_lock(kv_vocab_mirror *m) { m->mu.lock(); }
void mirror_unlock(kv_vocab_mirror *m) { m->mu.unlock(); }

namespace {

// One sync attempt; the caller holds the lock and has made the mirror's device current.
int sync_once(kv_vocab_mirror *m, const kv_vocab *v) {
  if (m->vocab && m->vocab != v) return kv_fail(KV_ERR_INVALID, "kv_vocab_mirror_sync: the mirror follows another vocabulary");
  const int64_t n = kv_vocab_size(v);
  if (n < m->n) return kv_fail(KV_ERR_STATE, "kv_vocab_mirror_sync: the vocabulary has fewer features than its mirror");
  m->vocab = v;
  if (n == m->n && m->cap) return KV_OK;
  std::vector<uint64_t> keys((size_t)(2 * (n - m->n)));
  if (n > m->n) {
    const int rc = vocab_export_range(v, m->n, n, keys.data());
    if (rc != KV_OK) return rc;  // a concurrent grow or import: the mirror stays as it was
  }
  cudaStream_t s = m->stream;
  int64_t cap = std::max<int64_t>(m->cap, 1024);
  while (cap < 2 * n) cap *= 2;
  if (cap != m->cap) {  // grow: a new table, the old slots re-inserted
    DevBuf<ulonglong2> nk;
    DevBuf<uint32_t> ni;
    KV_CUDA(nk.ensure(cap));
    KV_CUDA(ni.ensure(cap));
    KV_CUDA(cudaMemsetAsync(ni.p, 0xFF, (size_t)cap * 4, s));
    if (m->n)
      mirror_insert_kernel<<<fz_grid(m->cap), FZ_THREADS, 0, s>>>(nk.p, ni.p, (uint64_t)cap - 1, m->keys.p, m->ids.p, 0, m->cap);
    KV_CUDA(cudaGetLastError());
    KV_CUDA(cudaStreamSynchronize(s));
    std::swap(m->keys.p, nk.p);  // the old table is freed with nk / ni
    std::swap(m->keys.cap, nk.cap);
    std::swap(m->ids.p, ni.p);
    std::swap(m->ids.cap, ni.cap);
    m->cap = cap;
  }
  if (n > m->n) {
    KV_CUDA(m->staged.ensure(n - m->n));
    KV_CUDA(cudaMemcpyAsync(m->staged.p, keys.data(), keys.size() * 8, cudaMemcpyHostToDevice, s));
    mirror_insert_kernel<<<fz_grid(n - m->n), FZ_THREADS, 0, s>>>(m->keys.p, m->ids.p, (uint64_t)m->cap - 1, m->staged.p,
                                                                  nullptr, (uint32_t)m->n, n - m->n);
    KV_CUDA(cudaGetLastError());
  }
  KV_CUDA(cudaStreamSynchronize(s));
  m->n = n;
  return KV_OK;
}

}  // namespace

// sync_once, retried for about a second while a concurrent grow or import keeps the vocabulary in motion
int mirror_sync_locked(kv_vocab_mirror *m, const kv_vocab *v) {
  KV_CUDA(cudaSetDevice(m->device));
  int rc = KV_OK;
  for (int attempt = 0; attempt < 1000; attempt++) {
    rc = sync_once(m, v);
    if (rc != KV_ERR_STATE) return rc;
    std::this_thread::sleep_for(std::chrono::milliseconds(1));
  }
  return rc;
}

int featurize_device(kv_vocab_mirror *m, cudaStream_t s, const char *bytes, const int64_t *offsets, int64_t n_docs, int mode,
                     DevBuf<int64_t> &indptr, DevBuf<uint32_t> &ids, DevBuf<uint32_t> &tf, DevBuf<double> &oov, int64_t *nnz,
                     int64_t *bad_doc) {
  if (n_docs < 0 || (n_docs > 0 && (!bytes || !offsets))) return kv_fail(KV_ERR_INVALID, "kv_featurize: bad arguments");
  if (mode != KV_TEXT_RAW_ASCII && mode != KV_TEXT_TOKENS && mode != KV_TEXT_MIXED)
    return kv_fail(KV_ERR_INVALID, "kv_featurize: unknown text mode");
  for (int64_t i = 0; i < n_docs; i++)
    if (offsets[i + 1] < offsets[i] || offsets[i + 1] - offsets[i] > 0x7fffffffLL)
      return kv_fail(KV_ERR_INVALID, "kv_featurize: offsets must be non-decreasing, docs < 2 GiB");
  const int64_t n_bytes = n_docs ? offsets[n_docs] - offsets[0] : 0;
  if (n_bytes >= (int64_t)FZ_EMPTY) return kv_fail(KV_ERR_INVALID, "kv_featurize: the device featuriser takes batches below 4 GiB of text");
  KV_CUDA(indptr.ensure(n_docs + 1));
  KV_CUDA(oov.ensure(std::max<int64_t>(n_docs, 1)));
  *nnz = 0;
  if (n_docs == 0) {
    KV_CUDA(cudaMemsetAsync(indptr.p, 0, 8, s));
    KV_CUDA(ids.ensure(1));
    KV_CUDA(tf.ensure(1));
    KV_CUDA(cudaStreamSynchronize(s));
    return KV_OK;
  }
  KV_CUDA(m->text.ensure(std::max<int64_t>(n_bytes, 1)));
  KV_CUDA(m->offsets.ensure(n_docs + 1));
  KV_CUDA(m->tok_off.ensure(n_docs + 1));
  KV_CUDA(m->bad.ensure(1));
  if (n_bytes) KV_CUDA(cudaMemcpyAsync(m->text.p, bytes + offsets[0], (size_t)n_bytes, cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemcpyAsync(m->offsets.p, offsets, (size_t)(n_docs + 1) * 8, cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemsetAsync(m->bad.p, 0xFF, 8, s));
  KV_CUDA(cudaMemsetAsync(m->tok_off.p + n_docs, 0, 4, s));
  KV_CUDA(cudaMemsetAsync(oov.p, 0, (size_t)n_docs * 8, s));
  tokenize_kernel<false><<<fz_grid(n_docs), FZ_THREADS, 0, s>>>(m->text.p, m->offsets.p, n_docs, mode, m->tok_off.p, nullptr,
                                                                nullptr, nullptr, m->bad.p);
  KV_CUDA(cudaGetLastError());
  unsigned long long bad = 0;
  KV_CUDA(cudaMemcpyAsync(&bad, m->bad.p, 8, cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  if (bad != ~0ull) {
    if (bad_doc) *bad_doc = (int64_t)bad;
    return kv_fail(KV_ERR_NONASCII, "kv_featurize: non-ASCII byte in raw-text document");
  }
  // token counts -> offsets; 2 n_tok + 1 occurrence flags are scanned below, so n_tok < 2^31
  {
    const int rc = exclusive_scan_u32(m->tok_off.p, n_docs + 1, m->part, s);
    if (rc != KV_OK) return rc;
  }
  uint32_t n_tok = 0;
  KV_CUDA(cudaMemcpyAsync(&n_tok, m->tok_off.p + n_docs, 4, cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  if (n_tok >= 0x7FFFFFF0u) return kv_fail(KV_ERR_INVALID, "kv_featurize: too many tokens for one device batch");
  if (n_tok == 0) {
    KV_CUDA(ids.ensure(1));
    KV_CUDA(tf.ensure(1));
    indptr_kernel<<<fz_grid(n_docs + 1), FZ_THREADS, 0, s>>>(n_docs, m->tok_off.p, nullptr, indptr.p);
    KV_CUDA(cudaGetLastError());
    KV_CUDA(cudaStreamSynchronize(s));
    return KV_OK;
  }
  const int64_t n_occ = 2 * (int64_t)n_tok;
  int64_t dcap = 1024;
  while (dcap < 2 * n_occ) dcap *= 2;
  KV_CUDA(m->tok_start.ensure(n_tok));
  KV_CUDA(m->tok_len.ensure(n_tok));
  KV_CUDA(m->tok_doc.ensure(n_tok));
  KV_CUDA(m->occ_h.ensure(n_occ));
  KV_CUDA(m->first.ensure(dcap));
  KV_CUDA(m->cnt.ensure(dcap));
  KV_CUDA(m->keep.ensure(n_occ + 1));
  KV_CUDA(m->occ_id.ensure(n_occ));
  KV_CUDA(m->occ_tf.ensure(n_occ));
  KV_CUDA(cudaMemsetAsync(m->first.p, 0xFF, (size_t)dcap * 4, s));
  KV_CUDA(cudaMemsetAsync(m->cnt.p, 0, (size_t)dcap * 4, s));
  tokenize_kernel<true><<<fz_grid(n_docs), FZ_THREADS, 0, s>>>(m->text.p, m->offsets.p, n_docs, mode, m->tok_off.p,
                                                               m->tok_start.p, m->tok_len.p, m->tok_doc.p, nullptr);
  hash_kernel<<<fz_grid(n_occ), FZ_THREADS, 0, s>>>(m->text.p, n_tok, m->tok_start.p, m->tok_len.p, m->tok_doc.p, m->occ_h.p);
  dedup_insert_kernel<<<fz_grid(n_occ), FZ_THREADS, 0, s>>>(n_tok, m->tok_doc.p, m->occ_h.p, m->first.p, m->cnt.p,
                                                            (uint64_t)dcap - 1);
  resolve_kernel<<<fz_grid(n_occ + 1), FZ_THREADS, 0, s>>>(n_tok, m->tok_doc.p, m->occ_h.p, m->first.p, m->cnt.p,
                                                           (uint64_t)dcap - 1, m->keys.p, m->ids.p, (uint64_t)m->cap - 1,
                                                           m->keep.p, m->occ_id.p, m->occ_tf.p, oov.p);
  KV_CUDA(cudaGetLastError());
  {
    const int rc = exclusive_scan_u32(m->keep.p, n_occ + 1, m->part, s);
    if (rc != KV_OK) return rc;
  }
  uint32_t kept = 0;
  KV_CUDA(cudaMemcpyAsync(&kept, m->keep.p + n_occ, 4, cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  KV_CUDA(ids.ensure(std::max<uint32_t>(kept, 1)));
  KV_CUDA(tf.ensure(std::max<uint32_t>(kept, 1)));
  emit_kernel<<<fz_grid(n_occ), FZ_THREADS, 0, s>>>(n_tok, m->keep.p, m->occ_id.p, m->occ_tf.p, ids.p, tf.p);
  indptr_kernel<<<fz_grid(n_docs + 1), FZ_THREADS, 0, s>>>(n_docs, m->tok_off.p, m->keep.p, indptr.p);
  KV_CUDA(cudaGetLastError());
  *nnz = kept;
  return KV_OK;
}

extern "C" {

int kv_vocab_mirror_create(int device, kv_vocab_mirror **out) {
  if (!out) return kv_fail(KV_ERR_INVALID, "kv_vocab_mirror_create: out is NULL");
  int sm = 0;
  int rc = open_device(device, "kv_vocab_mirror_create", &sm);
  if (rc != KV_OK) return rc;
  std::unique_ptr<kv_vocab_mirror> m;
  try {
    m.reset(new kv_vocab_mirror());
  } catch (const std::bad_alloc &) {
    return kv_fail(KV_ERR_NOMEM, "kv_vocab_mirror_create: out of memory");
  }
  m->device = device;
  KV_CUDA(m->stream.create());
  *out = m.release();
  return KV_OK;
}

void kv_vocab_mirror_destroy(kv_vocab_mirror *m) {
  if (!m) return;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(m->device);
  if (m->stream.s) cudaStreamSynchronize(m->stream);
  delete m;  // the buffers are freed with their device current
  cudaSetDevice(prev);
}

int kv_vocab_mirror_sync(kv_vocab_mirror *m, const kv_vocab *v, int64_t *n_mirrored) {
  if (!m || !v) return kv_fail(KV_ERR_INVALID, "kv_vocab_mirror_sync: NULL handle");
  std::lock_guard<std::mutex> g(m->mu);
  const int rc = mirror_sync_locked(m, v);
  if (n_mirrored) *n_mirrored = m->n;
  return rc;
}

int kv_featurize_device(kv_vocab_mirror *m, const kv_vocab *v, const char *bytes, const int64_t *offsets, int64_t n_docs,
                        int mode, kv_csr **out, int64_t *bad_doc) {
  if (!m || !v || !out) return kv_fail(KV_ERR_INVALID, "kv_featurize_device: bad arguments");
  std::lock_guard<std::mutex> g(m->mu);
  int rc = mirror_sync_locked(m, v);
  if (rc != KV_OK) return rc;
  cudaStream_t s = m->stream;
  int64_t nnz = 0;
  rc = featurize_device(m, s, bytes, offsets, n_docs, mode, m->o_indptr, m->o_ids, m->o_tf, m->o_oov, &nnz, bad_doc);
  if (rc != KV_OK) return rc;
  try {
    std::unique_ptr<kv_csr> res(new kv_csr());
    res->indptr.resize((size_t)n_docs + 1);
    res->ids.resize((size_t)nnz);
    res->tf.resize((size_t)nnz);
    res->oov.resize((size_t)n_docs);
    KV_CUDA(cudaMemcpyAsync(res->indptr.data(), m->o_indptr.p, (size_t)(n_docs + 1) * 8, cudaMemcpyDeviceToHost, s));
    if (nnz) {
      KV_CUDA(cudaMemcpyAsync(res->ids.data(), m->o_ids.p, (size_t)nnz * 4, cudaMemcpyDeviceToHost, s));
      KV_CUDA(cudaMemcpyAsync(res->tf.data(), m->o_tf.p, (size_t)nnz * 4, cudaMemcpyDeviceToHost, s));
    }
    if (n_docs) KV_CUDA(cudaMemcpyAsync(res->oov.data(), m->o_oov.p, (size_t)n_docs * 8, cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaStreamSynchronize(s));
    *out = res.release();
  } catch (const std::bad_alloc &) {
    return kv_fail(KV_ERR_NOMEM, "kv_featurize_device: out of memory");
  }
  return KV_OK;
}

}  // extern "C"
