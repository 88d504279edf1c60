// Host-side state that both index handles (kv_index in tfidf_index.cu, kv_dense_index in dense_index.cu) keep the same
// way: the deleted rows, the result of the last threshold search and the checks of tag sets.  Each type owns the rules
// of its state; what a handle does in reaction (drop a batch, write NaN norms) stays with the handle.
#pragma once
#include "kv_cuda.cuh"
#include "tag_sets.cuh"

#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

// Checks a CSR of row tag sets, row r holding t[ip[r] .. ip[r+1]), for an index of n_rows rows (n sets given).
// *exact: every tag is < 64 (the 64-bit masks are the sets).
inline int check_row_tags(const int64_t *ip, const int32_t *t, int64_t n, int64_t n_rows, const char *fn, bool *exact) {
  if (n != n_rows) return kv_fail(KV_ERR_INVALID, "%s: %lld tag sets for an index of %lld rows", fn, (long long)n, (long long)n_rows);
  if (!ip) return kv_fail(KV_ERR_INVALID, "%s: NULL indptr", fn);
  if (ip[0] != 0) return kv_fail(KV_ERR_INVALID, "%s: indptr must start at 0", fn);
  for (int64_t r = 0; r < n; r++)
    if (ip[r + 1] < ip[r]) return kv_fail(KV_ERR_INVALID, "%s: indptr decreases at row %lld", fn, (long long)r);
  if (ip[n] > 0 && !t) return kv_fail(KV_ERR_INVALID, "%s: NULL tags", fn);
  *exact = true;
  for (int64_t r = 0; r < n; r++)
    for (int64_t i = ip[r]; i < ip[r + 1]; i++) {
      if (t[i] < 0) return kv_fail(KV_ERR_INVALID, "%s: tag %d of row %lld is negative", fn, t[i], (long long)r);
      *exact = *exact && t[i] < 64;
    }
  return KV_OK;
}

// One query's tag set (tags[0, n)) as a mask and an ascending list of MAX_QTAGS slots, -1 past the last tag
inline int parse_query_tags(const int32_t *t, int64_t n, int64_t q, const char *fn, unsigned long long *mask, int *list) {
  if (n > MAX_QTAGS) return kv_fail(KV_ERR_INVALID, "%s: query %lld has %lld tags (at most %d)", fn, (long long)q, (long long)n, MAX_QTAGS);
  std::vector<int> v(t, t + n);
  for (int x : v)
    if (x < 0) return kv_fail(KV_ERR_INVALID, "%s: tag %d of query %lld is negative", fn, x, (long long)q);
  std::sort(v.begin(), v.end());
  v.erase(std::unique(v.begin(), v.end()), v.end());
  *mask = 0;
  for (int j = 0; j < MAX_QTAGS; j++) list[j] = j < (int)v.size() ? v[(size_t)j] : -1;
  for (int x : v) *mask |= 1ull << (x & 63);
  return KV_OK;
}

// The tag sets of n_q queries, CSR ip[n_q+1] / t (parse_query_tags each): mask[n_q] and list[n_q * MAX_QTAGS].
// `ip_name` names the indptr in the errors.  *any: some query has a tag.
inline int parse_query_tag_csr(const int64_t *ip, const int32_t *t, int64_t n_q, const char *fn, const char *ip_name,
                               std::vector<unsigned long long> &mask, std::vector<int> &list, bool *any) {
  if (ip[0] != 0) return kv_fail(KV_ERR_INVALID, "%s: %s must start at 0", fn, ip_name);
  mask.assign((size_t)n_q, 0ull);
  list.assign((size_t)n_q * MAX_QTAGS, -1);
  *any = false;
  for (int64_t q = 0; q < n_q; q++) {
    const int64_t a = ip[q], e = ip[q + 1];
    if (e < a) return kv_fail(KV_ERR_INVALID, "%s: %s decreases at query %lld", fn, ip_name, (long long)q);
    if (e > a && !t) return kv_fail(KV_ERR_INVALID, "%s: NULL tags", fn);
    const int rc = parse_query_tags(t + a, e - a, q, fn, &mask[(size_t)q], &list[(size_t)q * MAX_QTAGS]);
    if (rc != KV_OK) return rc;
    *any = *any || mask[(size_t)q] != 0ull;
  }
  return KV_OK;
}

// Deleted rows (tombstones) by local row: no flags until the first deletion, then one per row.  A deleted row keeps
// its row id; an append extends the flags with live rows.
struct Tombstones {
  std::vector<uint8_t> flags;
  int64_t count = 0;

  bool any() const { return count != 0; }
  bool is_dead(int64_t r) const { return count && flags[(size_t)r]; }

  // Deletes rows[0, n) of an index of n_rows rows (any order; duplicates and rows deleted before are allowed).  Every
  // row is checked before any is marked; `fn` names the caller in the error.  *added = how many rows are newly deleted.
  int mark(const int64_t *rows, int64_t n, int64_t n_rows, const char *fn, int64_t *added) {
    for (int64_t i = 0; i < n; i++)
      if (rows[i] < 0 || rows[i] >= n_rows)
        return kv_fail(KV_ERR_INVALID, "%s: row %lld outside 0..%lld", fn, (long long)rows[i], (long long)n_rows - 1);
    *added = 0;
    for (int64_t i = 0; i < n; i++) {
      if (flags.empty()) flags.assign((size_t)n_rows, 0);
      uint8_t &d = flags[(size_t)rows[i]];
      if (!d) { d = 1; ++*added; }
    }
    count += *added;
    return KV_OK;
  }

  // The flags of all n == n_rows rows into out (0 live, 1 deleted).
  int copy_out(uint8_t *out, int64_t n, int64_t n_rows, const char *fn) const {
    if (n != n_rows)
      return kv_fail(KV_ERR_INVALID, "%s: %lld flags for an index of %lld rows", fn, (long long)n, (long long)n_rows);
    if (count) memcpy(out, flags.data(), (size_t)n);
    else if (n) memset(out, 0, (size_t)n);
    return KV_OK;
  }

  // After an append: the index now has n_rows rows, the new ones live.
  void extend(int64_t n_rows) {
    if (count) flags.resize((size_t)n_rows, 0);
  }
};

// The result of a handle's last threshold search, records Rec (RangePair, JaccardPair or ExactPair) in emit order: the pair buffer
// (65,536 records at first; it keeps its capacity across searches), the device pair count, and while the result is
// valid its query and pair counts.  It lives until a fetch consumes it or the handle drops it.
template <class Rec>
struct RangeResult {
  DevBuf<Rec> pairs;
  DevBuf<unsigned long long> d_count;
  bool valid = false;
  int64_t n_q = 0, n_pairs = 0;

  // Before a search: room for 65,536 records at least, and the device count zeroed on stream s.
  int prepare(cudaStream_t s) {
    KV_CUDA(pairs.ensure(65536));
    KV_CUDA(d_count.ensure(1));
    KV_CUDA(cudaMemsetAsync(d_count.p, 0, sizeof(unsigned long long), s));
    return KV_OK;
  }
  unsigned long long capacity() const { return (unsigned long long)pairs.cap; }
  // After a search found more pairs than fit: room for exactly `count`, and the device count zeroed again for the rerun.
  int grow(unsigned long long count, cudaStream_t s, const char *fn) {
    if (pairs.ensure((int64_t)count) != cudaSuccess) {
      cudaGetLastError();
      return kv_fail(KV_ERR_NOMEM, "%s: %llu pairs reach the threshold; their buffer does not fit in device memory "
                                   "(raise the threshold or split the query batch)", fn, count);
    }
    KV_CUDA(cudaMemsetAsync(d_count.p, 0, sizeof(unsigned long long), s));
    return KV_OK;
  }
  void commit(int64_t queries, int64_t pairs_found) {
    n_q = queries;
    n_pairs = pairs_found;
    valid = true;
  }
  void drop() { valid = false; }

  // The fetches order the pairs on the device in the pair buffer itself (range_order.cu), per query by (score desc, row
  // asc).  Once ordering has started the result is consumed whatever happens; a scratch allocation that fails first
  // (KV_ERR_NOMEM) leaves it for another try.  `search` names the entry point that makes a result, for the error of a
  // fetch without one; row_base is added to the local rows of JaccardPair and ExactPair records.  Scores are
  // RecScore<Rec>: float32, float64 for ExactPair.
  using Score = typename RecScore<Rec>::type;

  // Into host arrays.
  int fetch_host(const char *fn, const char *search, int device, cudaStream_t s, RangeOrderScratch &sc, int64_t row_base,
                 int64_t *indptr, int64_t *rows, Score *scores, int32_t *inter, int32_t *uni) {
    if (!valid) return kv_fail(KV_ERR_STATE, "%s: no threshold search result (%s first)", fn, search);
    if (n_pairs > 0 && (!rows || !scores)) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
    KV_CUDA(cudaSetDevice(device));
    const int rc = range_order_to_host(pairs.p, n_pairs, n_q, row_base, indptr, rows, scores, inter, uni, sc, s, fn);
    if (rc != KV_ERR_NOMEM) valid = false;
    return rc;
  }

  // Into caller-owned device memory of `device` (checked: a host pointer is an error, never a fault); returns with the
  // stream synchronised.
  int fetch_device(const char *fn, const char *search, int device, cudaStream_t s, RangeOrderScratch &sc, int64_t row_base,
                   void *d_indptr, void *d_rows, void *d_scores, void *d_inter, void *d_uni) {
    constexpr bool counts = std::is_same<Rec, JaccardPair>::value;
    if (!valid) return kv_fail(KV_ERR_STATE, "%s: no threshold search result (%s first)", fn, search);
    int rc = check_device_ptr(d_indptr, device, 8, "indptr", fn);
    if (rc == KV_OK && n_pairs > 0) rc = check_device_ptr(d_rows, device, 8, "rows", fn);
    if (rc == KV_OK && n_pairs > 0) rc = check_device_ptr(d_scores, device, sizeof(Score), "scores", fn);
    if (rc == KV_OK && n_pairs > 0 && counts) rc = check_device_ptr(d_inter, device, 4, "inter", fn);
    if (rc == KV_OK && n_pairs > 0 && counts) rc = check_device_ptr(d_uni, device, 4, "uni", fn);
    if (rc != KV_OK) return rc;
    KV_CUDA(cudaSetDevice(device));
    rc = range_order_device(pairs.p, n_pairs, n_q, row_base, (int64_t *)d_indptr, (int64_t *)d_rows, (Score *)d_scores,
                            (int32_t *)d_inter, (int32_t *)d_uni, sc, s, fn);
    if (rc != KV_ERR_NOMEM) valid = false;
    if (rc != KV_OK) return rc;
    KV_CUDA(cudaStreamSynchronize(s));
    return KV_OK;
  }
};
