// Tag sets, the same for both index handles (kv_index_set_row_tags / kv_query_set_tag_filter in tfidf_index.cu,
// kv_dense_set_row_tags / kv_dense_set_tag_filter in dense_index.cu).
// A row carries a set of tags >= 0, a query at most MAX_QTAGS of them; the query matches the rows whose set meets its
// own.  Both sides also carry a 64-bit mask, OR of 1 << (t & 63): a row whose mask misses the query's holds none of its
// tags, and when every tag of the index is < 64 a mask hit is the exact answer.  Otherwise the row's tags (CSR tag_ptr /
// tag_list, indexed by the handle's row layout: scan position or local row) are compared with the query's ascending
// list, -1 past its last tag.
#pragma once
#include <cstdint>

constexpr int MAX_QTAGS = 16;

__device__ __forceinline__ bool tags_meet(unsigned long long row_mask, unsigned long long q_mask, const int64_t *__restrict__ tag_ptr,
                                          const int *__restrict__ tag_list, int64_t pos, const int *__restrict__ q_tags) {
  if ((row_mask & q_mask) == 0ull) return false;
  if (!tag_ptr) return true;  // every tag < 64: the masks are the sets
  for (int64_t i = tag_ptr[pos], e = tag_ptr[pos + 1]; i < e; i++) {
    const int t = tag_list[i];
    if (!((q_mask >> (t & 63)) & 1ull)) continue;
    for (int j = 0; j < MAX_QTAGS; j++) {
      const int u = q_tags[j];
      if (u < 0 || u > t) break;
      if (u == t) return true;
    }
  }
  return false;
}
