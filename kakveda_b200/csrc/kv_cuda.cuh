// CUDA helpers shared by the kernel translation units.
#pragma once
#include "kv_internal.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <utility>

#define KV_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return kv_fail(KV_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),     \
                     __FILE__, __LINE__);                                                     \
  } while (0)

// Checks that `device` exists, makes it current and reads its SM count: the first step of every create function
// (`fn` names it in the error message).  No visible device is KV_ERR_CUDA ("no CUDA device visible").
int open_device(int device, const char *fn, int *sm_count);

// The buffers and handles below own what they hold: it is freed when they are destroyed, and they are move-only, so a
// copy (two owners) does not compile.  Destroy them with their device current.

// Growable device array (amortised doubling) -- the raw CSR of an append-only index.
template <typename T>
struct DevVec {
  T *p = nullptr;
  int64_t n = 0, cap = 0;
  DevVec() = default;
  DevVec(DevVec &&o) noexcept : p(std::exchange(o.p, nullptr)), n(std::exchange(o.n, 0)), cap(std::exchange(o.cap, 0)) {}
  DevVec(const DevVec &) = delete;
  ~DevVec() { cudaFree(p); }
  cudaError_t reserve(int64_t want, cudaStream_t s) {
    if (want <= cap) return cudaSuccess;
    int64_t nc = cap ? cap : 1024;
    while (nc < want) nc *= 2;
    T *q = nullptr;
    cudaError_t e = cudaMalloc(&q, (size_t)nc * sizeof(T));
    if (e != cudaSuccess) return e;
    if (n) {
      e = cudaMemcpyAsync(q, p, (size_t)n * sizeof(T), cudaMemcpyDeviceToDevice, s);
      if (e != cudaSuccess) { cudaFree(q); return e; }
      e = cudaStreamSynchronize(s);
      if (e != cudaSuccess) { cudaFree(q); return e; }
    }
    cudaFree(p);
    p = q;
    cap = nc;
    return cudaSuccess;
  }
};

// Fixed-size device buffer re-allocated only when it must grow (scratch reused across calls).
template <typename T>
struct DevBuf {
  T *p = nullptr;
  int64_t cap = 0;
  DevBuf() = default;
  DevBuf(DevBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  DevBuf(const DevBuf &) = delete;
  ~DevBuf() { cudaFree(p); }
  cudaError_t ensure(int64_t want) {
    if (want <= cap) return cudaSuccess;
    cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc(&p, (size_t)(want > 0 ? want : 1) * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
};

template <typename T>
struct PinnedBuf {
  T *p = nullptr;
  int64_t cap = 0;
  PinnedBuf() = default;
  PinnedBuf(PinnedBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  PinnedBuf(const PinnedBuf &) = delete;
  ~PinnedBuf() { cudaFreeHost(p); }
  cudaError_t ensure(int64_t want) {
    if (want <= cap) return cudaSuccess;
    cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaHostAlloc(&p, (size_t)(want > 0 ? want : 1) * sizeof(T), cudaHostAllocDefault);
    if (e == cudaSuccess) cap = want;
    return e;
  }
};

// One match of a threshold search (16 bytes): what the emitting scans (K1b-R, K2-R) append to their pair buffer
struct RangePair {
  int32_t q;    // query index within the search
  float score;  // the float32 score the top-k path reports for the pair
  int64_t row;  // global row
};

// One match of a Jaccard threshold search (16 bytes, what K3-R and its irregular-query fallback append).  The exact
// counts travel with the pair and the float32 score is their quotient, formed where the pairs are ordered: inter and
// union are integer-valued floats on the device, so the host's IEEE division gives the bits of the device's __fdiv_rn.
struct JaccardPair {
  int32_t q;      // original query
  int32_t row;    // local original row (below 2^31: the row permutation is int)
  int32_t inter;  // |q ∩ row|
  int32_t uni;    // |q ∪ row|
};

// Scratch of the device ordering of range records (range_order.cu), owned by an index handle: the buffers keep their
// capacity across calls, like the pair buffer itself.
struct RangeOrderScratch {
  DevBuf<int4> alt;                       // the records' second home during the radix passes
  DevBuf<unsigned int> counts, partials;  // per-tile digit counts (digit-major) and the sums of their scan tiles
  DevBuf<unsigned long long> stats;       // min / max of each key field
  DevBuf<unsigned char> out;              // the ordered arrays on their way to the host (host fetch only)
  PinnedBuf<int4> staged;                 // the records of a small result, ordered on the host (host fetch only)
};

// Host fetches whose pairs plus queries number fewer than this order them on one host core (range_order_to_host); the
// device fetches, and the host fetches of larger results, order on the device.  Measured in DESIGN §6.
constexpr int64_t RANGE_HOST_ORDER_MAX = 8192;

// Orders the n pairs of a threshold search over n_q queries (emit order, as the device left them; rec is reordered in
// place) into device arrays indptr[n_q+1] / rows[n] / scores[n] (and, for JaccardPair records, inter[n] / uni[n]) on
// stream s: per query by (score desc, row asc).  row_base is added to JaccardPair rows (RangePair rows are global
// already).  Returns once the work is enqueued.  KV_ERR_NOMEM (with the pair count) when the scratch does not fit.
// `fn` names the caller in error messages.  Defined for Rec = RangePair and JaccardPair.
template <class Rec>
int range_order_device(Rec *rec, int64_t n, int64_t n_q, int64_t row_base, int64_t *indptr, int64_t *rows, float *scores,
                       int32_t *inter, int32_t *uni, RangeOrderScratch &sc, cudaStream_t s, const char *fn);
// The same into host arrays, stream synchronised: ordered on the device into sc.out and copied back, or below
// RANGE_HOST_ORDER_MAX pairs plus queries copied back as records and ordered on the host (the same bits).
template <class Rec>
int range_order_to_host(Rec *rec, int64_t n, int64_t n_q, int64_t row_base, int64_t *indptr, int64_t *rows, float *scores,
                        int32_t *inter, int32_t *uni, RangeOrderScratch &sc, cudaStream_t s, const char *fn);

// Exclusive scan of x[0, m) in place on stream s (range_order.cu); `part` is scratch.  The sums must stay below 2^32.
int exclusive_scan_u32(unsigned *x, int64_t m, DevBuf<unsigned> &part, cudaStream_t s);

// Device featuriser (featurize_device.cu): kv_featurize(grow = 0) of a packed text batch against the device mirror of
// the vocabulary, into device CSR buffers (resized here: indptr n_docs + 1, ids / tf nnz, oov n_docs) on stream s, which
// must belong to the mirror's device.  The caller holds the mirror's lock (mirror_lock) from before this call until the
// stream has finished the work.  Returns with *nnz known and the last kernels enqueued.  KV_ERR_NONASCII sets *bad_doc.
int featurize_device(kv_vocab_mirror *m, cudaStream_t s, const char *bytes, const int64_t *offsets, int64_t n_docs, int mode,
                     DevBuf<int64_t> &indptr, DevBuf<uint32_t> &ids, DevBuf<uint32_t> &tf, DevBuf<double> &oov, int64_t *nnz,
                     int64_t *bad_doc);
// The mirror's device, and its lock (a std::mutex): featurize_device reads the table that kv_vocab_mirror_sync replaces.
int mirror_device(const kv_vocab_mirror *m);
// kv_vocab_mirror_sync with the mirror's lock held (makes the mirror's device current).
int mirror_sync_locked(kv_vocab_mirror *m, const kv_vocab *v);
void mirror_lock(kv_vocab_mirror *m);
void mirror_unlock(kv_vocab_mirror *m);

// KV_OK when p is device memory of `device` aligned to `align` bytes, else KV_ERR_INVALID naming `what` (a host pointer
// passed by mistake is an error, never a fault).
int check_device_ptr(const void *p, int device, size_t align, const char *what, const char *fn);

// Non-blocking stream; converts to cudaStream_t.
struct CudaStream {
  cudaStream_t s = nullptr;
  CudaStream() = default;
  CudaStream(CudaStream &&o) noexcept : s(std::exchange(o.s, nullptr)) {}
  CudaStream(const CudaStream &) = delete;
  ~CudaStream() { if (s) cudaStreamDestroy(s); }
  cudaError_t create() { return cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); }
  operator cudaStream_t() const { return s; }
};

// Event with timing; converts to cudaEvent_t.
struct CudaEvent {
  cudaEvent_t e = nullptr;
  CudaEvent() = default;
  CudaEvent(CudaEvent &&o) noexcept : e(std::exchange(o.e, nullptr)) {}
  CudaEvent(const CudaEvent &) = delete;
  ~CudaEvent() { if (e) cudaEventDestroy(e); }
  cudaError_t create() { return cudaEventCreate(&e); }
  operator cudaEvent_t() const { return e; }
};
