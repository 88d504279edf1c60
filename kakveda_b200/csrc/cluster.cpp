// Connected components of the k-nearest-neighbour graph an all-pairs self-join returns (BASELINE configs[3]:
// "1M x 1M symmetric similarity + top-k=32 clustering").  Host side of the pattern-clustering extension: the
// reference's pattern_detector groups failures by failure_type equality only
// (services/pattern_detector/app.py:39-41); here rows are linked when their similarity reaches a threshold
// (the reference's failure_matching.similarity_threshold, services/warning_policy/app.py:22) and every connected
// component becomes one candidate pattern.  Union-find with the smaller row id as the root, so labels are
// deterministic: label[i] = smallest row id of i's component.
#include "kv_internal.h"

#include <cstdint>
#include <vector>

namespace {
inline int64_t find_root(std::vector<int64_t> &parent, int64_t x) {
  while (parent[(size_t)x] != x) {
    parent[(size_t)x] = parent[(size_t)parent[(size_t)x]];  // path halving
    x = parent[(size_t)x];
  }
  return x;
}

inline void unite(std::vector<int64_t> &parent, int64_t i, int64_t r) {
  const int64_t a = find_root(parent, i), b = find_root(parent, r);
  if (a == b) return;
  if (a < b) parent[(size_t)b] = a; else parent[(size_t)a] = b;
}

// parent := n singletons
int init_forest(std::vector<int64_t> &parent, int64_t n, const char *fn) {
  try {
    parent.resize((size_t)n);
  } catch (const std::bad_alloc &) {
    return kv_fail(KV_ERR_NOMEM, "%s: out of host memory", fn);
  }
  for (int64_t i = 0; i < n; i++) parent[(size_t)i] = i;
  return KV_OK;
}

// labels[i] = root of i, *n_clusters = number of roots
void write_labels(std::vector<int64_t> &parent, int64_t n, int64_t *labels, int64_t *n_clusters) {
  int64_t count = 0;
  for (int64_t i = 0; i < n; i++) {
    labels[i] = find_root(parent, i);
    count += labels[i] == i;
  }
  if (n_clusters) *n_clusters = count;
}
}  // namespace

extern "C" int kv_cluster_topk(int64_t n, int k, const int64_t *rows, const float *scores, float threshold,
                               int64_t *labels, int64_t *n_clusters) {
  if (n < 0 || k < 1 || (n > 0 && (!rows || !scores || !labels)))
    return kv_fail(KV_ERR_INVALID, "kv_cluster_topk: bad arguments");
  std::vector<int64_t> parent;
  int rc = init_forest(parent, n, "kv_cluster_topk");
  if (rc != KV_OK) return rc;
  for (int64_t i = 0; i < n; i++)
    for (int j = 0; j < k; j++) {
      const int64_t r = rows[i * k + j];
      if (r < 0) continue;
      if (r >= n) return kv_fail(KV_ERR_INVALID, "kv_cluster_topk: neighbour %lld of row %lld outside 0..%lld", (long long)r,
                                 (long long)i, (long long)n);
      if (!(scores[i * k + j] >= threshold)) continue;  // NaN never links
      unite(parent, i, r);
    }
  write_labels(parent, n, labels, n_clusters);
  return KV_OK;
}

// The same components for a graph given as adjacency lists (e.g. what a threshold search returns: every edge already
// reaches the threshold).
extern "C" int kv_cluster_csr(int64_t n, const int64_t *indptr, const int64_t *rows, int64_t *labels, int64_t *n_clusters) {
  if (n < 0 || (n > 0 && (!indptr || !labels))) return kv_fail(KV_ERR_INVALID, "kv_cluster_csr: bad arguments");
  for (int64_t i = 0; i < n; i++)
    if (indptr[i + 1] < indptr[i]) return kv_fail(KV_ERR_INVALID, "kv_cluster_csr: indptr not monotone");
  if (n > 0 && indptr[n] > indptr[0] && !rows) return kv_fail(KV_ERR_INVALID, "kv_cluster_csr: bad arguments");
  std::vector<int64_t> parent;
  int rc = init_forest(parent, n, "kv_cluster_csr");
  if (rc != KV_OK) return rc;
  for (int64_t i = 0; i < n; i++)
    for (int64_t j = indptr[i]; j < indptr[i + 1]; j++) {
      const int64_t r = rows[j];
      if (r < 0) continue;
      if (r >= n) return kv_fail(KV_ERR_INVALID, "kv_cluster_csr: neighbour %lld of row %lld outside 0..%lld", (long long)r,
                                 (long long)i, (long long)n);
      unite(parent, i, r);
    }
  write_labels(parent, n, labels, n_clusters);
  return KV_OK;
}
