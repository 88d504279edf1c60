// TF-IDF cosine index for the GFKB match path: the kv_index handle and its C ABI
// (include/kakveda_b200.h).  Device code lives in tfidf_kernels.cuh (scan, query preparation, merge) and
// bound_kernel.cuh (tensor-core chunk bounds); see there for the math and the HBM layout.  Host responsibilities: keep
// the append-only CSR, finalize (statistics on the device, (norm class, text) order of the rows and the column blocks
// on the host cores), per-batch query upload (text order of the queries, CSR -> device; tables are built by kernels)
// and kernel launches.
#include "block_builder.cuh"
#include "bound_kernel.cuh"
#include "index_state.cuh"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <limits>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

using namespace kvk;
using namespace kvh;  // parallel_for, stable_sort_indices, idf_host, build_blocks (block_builder.cuh)

// ----------------------------------------------------------------------------------------
// handle
// ----------------------------------------------------------------------------------------

// One integer >= 0 per local row (row labels, row groups).  It describes the rows it was set for: an append drops it.
// On the device, rebuilt by every finalize for the current scan layout: by row and by scan position.
struct RowSet {
  std::vector<int> h;
  bool has = false, on_device = false;
  DevBuf<int> d_row, d_pos;

  // v[0, n) for an index of n_rows rows; `what` names one value in the errors ("label", "group")
  int set(const int32_t *v, int64_t n, int64_t n_rows, const char *fn, const char *what) {
    if (n != n_rows) return kv_fail(KV_ERR_INVALID, "%s: %lld %ss for an index of %lld rows", fn, (long long)n, what, (long long)n_rows);
    for (int64_t i = 0; i < n; i++)
      if (v[i] < 0) return kv_fail(KV_ERR_INVALID, "%s: %s %d of row %lld is negative", fn, what, v[i], (long long)i);
    h.assign(v, v + n);
    has = true;
    return KV_OK;
  }
  void clear() {
    h.clear();
    has = on_device = false;
  }
  // set for the current n_rows rows and on the device for the current layout
  bool ready(int64_t n_rows) const { return has && on_device && (int64_t)h.size() == n_rows; }
  // The device copies for the layout whose scan position p holds row perm[p] (n_pos positions, n rows).
  int upload(const int *perm, int64_t n, int64_t n_pos, cudaStream_t s) {
    if (n == 0) return KV_OK;
    KV_CUDA(d_row.ensure(n));
    KV_CUDA(d_pos.ensure(n_pos));
    KV_CUDA(cudaMemcpyAsync(d_row.p, h.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    label_pos_kernel<<<(unsigned)((n_pos + 255) / 256), 256, 0, s>>>(perm, d_row.p, n, n_pos, d_pos.p);
    KV_CUDA(cudaGetLastError());
    KV_CUDA(cudaStreamSynchronize(s));  // h may change once this returns
    return KV_OK;
  }
};

// A set of tags >= 0 per local row (kv_index_set_row_tags), CSR on the host.  Like a RowSet it describes the rows it
// was set for (an append drops it) and every finalize rebuilds its device copies for the current scan layout: each
// row's mask (tags_meet) and, unless every tag is < 64, its tags, by scan position; and the chunk signatures over the
// live rows.
struct RowTags {
  std::vector<int64_t> indptr;
  std::vector<int> tags;
  bool has = false, on_device = false, masks_exact = true;  // masks_exact: every tag < 64
  DevBuf<unsigned long long> d_mask_pos, d_chunk_sig;
  DevBuf<int64_t> d_ptr_pos;
  DevBuf<int> d_list_pos;

  int set(const int64_t *ip, const int32_t *t, int64_t n, int64_t n_rows, const char *fn) {
    bool exact = true;
    const int rc = check_row_tags(ip, t, n, n_rows, fn, &exact);
    if (rc != KV_OK) return rc;
    indptr.assign(ip, ip + n + 1);
    tags.assign(t, t + ip[n]);
    masks_exact = exact;
    has = true;
    on_device = false;
    return KV_OK;
  }
  void clear() {
    indptr.clear();
    tags.clear();
    has = on_device = false;
  }
  bool ready(int64_t n_rows) const { return has && on_device && (int64_t)indptr.size() == n_rows + 1; }
};

// The tag filter of the resident batch (kv_query_set_tag_filter), while some query has tags: per query its mask (by
// original query on the host, for the fallbacks; on the device by original query and by sorted slot) and its
// ascending tags, -1 past the last (device: by original query for the fallbacks and the null fill, by sorted slot for
// the scan).
struct QueryTags {
  bool on = false;
  std::vector<unsigned long long> h_mask;
  DevBuf<unsigned long long> d_mask_orig, d_mask_sorted;
  DevBuf<int> d_tags_orig, d_tags_sorted;
};

// The irregular queries of the resident batch (see classify_queries), in sorted-slot order: their original index and
// CSR on the host, for the float64 full-scan fallback.
struct IrregularQueries {
  std::vector<int64_t> q, indptr{0};
  std::vector<uint32_t> ids, tf;
  std::vector<double> oov;

  void clear() {
    q.clear(); indptr.assign(1, 0); ids.clear(); tf.clear(); oov.clear();
  }
  void add(int64_t query, const uint32_t *q_ids, const uint32_t *q_tf, int64_t nnz, double q_oov) {
    q.push_back(query);
    ids.insert(ids.end(), q_ids, q_ids + nnz);
    tf.insert(tf.end(), q_tf, q_tf + nnz);
    indptr.push_back((int64_t)ids.size());
    oov.push_back(q_oov);
  }
};

struct kv_index {
  int device = 0;
  int64_t row_base = 0;
  CudaStream stream;
  CudaEvent ev[5];
  CudaEvent evk[6];  // bound/scan kernel boundaries of a batch
  CudaEvent evp2;    // start of phase 2 of a two-phase batch
  CudaEvent evq[4];  // stages of a text upload on the device (kv_query_upload_text)
  bool two_phase = false;
  std::mutex mu;
  int sm_count = 132;

  // raw CSR: device copy for the statistics kernels and K6, host copy for the sort and the column blocks
  DevVec<int64_t> indptr;  // n_rows + 1 entries once any row exists
  DevVec<uint32_t> ids;
  DevVec<uint16_t> tf;
  std::vector<int64_t> h_indptr{0};
  std::vector<uint32_t> h_ids;
  std::vector<uint16_t> h_tf;
  int64_t n_rows = 0, nnz = 0;

  bool has_gdf = false;
  std::vector<uint32_t> h_gdf;
  int64_t n_global = 0;

  bool finalized = false;
  int jaccard = 0;  // 0: TF-IDF cosine (the reference's measure), 1: token-set Jaccard (K3)
  int corpus_fit = 0;  // 1: TF-IDF fitted on the corpus only (self-join / pattern clustering); the query is just transformed
  int64_t V = 0, n_total = 0;
  DevBuf<uint32_t> d_df, d_cnt, d_tfmin, d_tfmax, d_utf;
  DevBuf<double> d_a64, d_d64, d_bb64, d_B64;
  DevBuf<float> d_B32, d_cminB;
  DevBuf<uint8_t> d_univ;
  DevBuf<int> d_perm, d_invperm;
  // scan layout currently on the device (perm, column blocks, dense matrix): which rows / universal set it was built for
  bool layout_valid = false;
  int64_t layout_rows = -1;
  std::vector<uint8_t> layout_univ;
  int last_finalize_kind = 0;  // 1: full rebuild, 2: statistics-only refresh
  DevBuf<uint32_t> d_blk;
  DevBuf<BlockInfo> d_binfo;
  DevBuf<__half> d_Uf;
  DevBuf<short> d_fslot;
  DevBuf<unsigned short> d_fslot2;
  DevBuf<uint32_t> d_ubt, d_rbloom, d_rt_off, d_rt_size;
  DevBuf<uint4> d_rt_slots;
  CUtensorMap map_u;
  DevBuf<unsigned long long> d_ovf_keys;
  DevBuf<uint32_t> d_ovf_vals;
  int n_ovf = 0;
  int64_t n_rt_slots = 0;  // slots of all blocks' rare tables
  int64_t rt_enlarged = 0;  // of those tables, the ones whose cuckoo insertion needed more than the initial size
  int64_t blk_words = 0, n_chunks = 0, n_chunks_pad = 0, n_entries = 0, n_rare_entries = 0;
  std::vector<uint32_t> h_df, h_tfmax;
  std::vector<short> h_fslot;
  std::vector<unsigned short> h_fslot2;
  std::vector<uint8_t> h_univ;
  std::vector<uint32_t> h_utf;
  int64_t n_univ = 0;
  // K6 scratch
  DevBuf<int64_t> d_rq_indptr;
  DevBuf<uint32_t> d_rq_ids, d_rq_tf;
  DevBuf<double> d_rq_const, d_rq_out;
  DevBuf<long long> d_rq_rows;

  // query batch: pinned staging + device copies of the CSR, per-query tables (built by kernels)
  PinnedBuf<int64_t> h_q_indptr;
  PinnedBuf<uint32_t> h_q_ids, h_q_tf;
  PinnedBuf<double> h_q_oov;
  PinnedBuf<int> h_qperm;     // 3 * n_q: sorted slot -> original query, null-query list, sorted slot -> row of the staged CSR
  PinnedBuf<uint8_t> h_flags;
  DevBuf<uint8_t> d_qflag_row;  // a text upload's classification by row, and its text order (two halves: merge passes)
  DevBuf<int> d_qorder;
  DevBuf<int64_t> d_q_indptr;
  DevBuf<uint32_t> d_q_ids, d_q_tf;
  DevBuf<double> d_q_oov;
  DevBuf<int> d_qperm;
  DevBuf<uint8_t> d_flags;
  DevBuf<float> d_qconst;     // 7 * n_q: nq, dotU, corrU, dotS, corrS, dotX, 1 / s_q (fixed-point unit of the bound kernel's R)
  DevBuf<unsigned long long> d_qfix;  // 2 * n_q: the universal features' fixed-point sums U_w, U_c (what the scan adds)
  DevBuf<unsigned char> d_qtab;
  DevBuf<uint2> d_q2list;
  DevBuf<uint32_t> d_q3id, d_q3w, d_d2col;  // rare lists (feature, weight); second-class dictionary of each tile
  DevBuf<__half> d_Wf, d_Wf2;
  DevBuf<unsigned long long> d_f2out;       // second-class listings left out of their tile's dictionary
  CUtensorMap map_w, map_w2;
  DevBuf<int> d_gthr;
  // candidate lists of a batch
  DevBuf<int> d_seeds;
  DevBuf<uint2> d_direct, d_pool;
  DevBuf<uint32_t> d_list_count, d_list_pages;
  DevBuf<unsigned int> d_pool_ctl;  // [0] pages handed out, [1] overflow flag
  DevBuf<unsigned char> d_ubq;      // 8-bit bound codes of a batch, [n_q][n_chunks_pad] (when they fit)
  DevBuf<int> d_tcode;              // threshold code per query of the scan of the codes (threshold_codes_kernel)
  int last_used_codes = 0;
  int64_t pool_pages = 0;
  // cross-GPU threshold exchange (row-sharded GFKB): d_gthr is exported over CUDA IPC, the peers' arrays are mapped here
  bool gthr_exported = false;
  int n_peers = 0;
  int *peer_gthr[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  int64_t peer_cap = 0;  // queries the exchanged arrays hold
  bool peers_borrowed = false;  // peer_gthr points at other handles' arrays in this process (kv_debug_thresholds_link)
  DevBuf<int> d_excl_sorted, d_excl_orig;  // self-join exclusions of the resident batch (by sorted slot / by original query)
  std::vector<int> h_excl_orig;
  bool has_excl = false;
  // row labels (kv_index_set_row_labels); besides the common device copies, the chunk label signatures and the first
  // LAB_FIRST rows of every label
  RowSet labels;
  DevBuf<int> d_lab_keys, d_lab_rows;
  DevBuf<unsigned long long> d_chunk_sig;
  int n_lab = 0;
  // label filter of the resident batch (kv_query_set_filter; by sorted slot / by original query), only while some
  // query is filtered
  DevBuf<int> d_filt_sorted, d_filt_orig;
  std::vector<int> h_filt_orig;
  bool has_filter = false;
  // row groups (kv_index_set_row_groups): by row for K5, the fallbacks and null queries, by scan position for the
  // scan.  Distinct mode of the resident batch (kv_query_set_distinct), cleared by the next upload; merged_seeds: the
  // caller merges the shards' seed lists group-aware (KV_DISTINCT_MERGED_SEEDS), so the two-phase top-k may run.
  RowSet groups;
  bool distinct = false, merged_seeds = false;
  // row tag sets (kv_index_set_row_tags) and the tag filter of the resident batch (kv_query_set_tag_filter, cleared by
  // the next upload); the fallbacks' per-query ineligible rows
  RowTags tags;
  QueryTags qtags;
  DevBuf<uint8_t> d_tagdead;
  // deleted rows (kv_index_delete_rows).  They keep their place in the scan layout.  On the device while any row is
  // deleted, rebuilt by every finalize: by row, the live word of every chunk (by scan position) and the first LAB_FIRST
  // live rows (null queries)
  Tombstones tomb;
  DevBuf<uint8_t> d_dead;
  DevBuf<uint32_t> d_alive, d_dcnt;
  DevBuf<int> d_dead_list, d_first_live;
  // threshold search over the resident batch (kv_range_resident): its own threshold array (not d_gthr, which peers push
  // into and a top-k raises) and the result of the index's mode -- on a Jaccard index (K3-R) the records carry the
  // exact counts and local rows.  Either result is dropped by the next upload, search, append, deletion or finalize.
  // An exact search (kv_range_resident_exact) leaves its result in xrange and consumes the float32 one it started from.
  DevBuf<int> d_rthr;
  RangeResult<RangePair> range;
  RangeResult<JaccardPair> jrange;
  RangeResult<ExactPair> xrange;
  RangeOrderScratch rsort;  // the fetches order the pairs on the device (range_order.cu)
  DevBuf<unsigned long long> d_stats;
  DevBuf<float> d_part_s, d_out_s;
  DevBuf<long long> d_part_r, d_out_r;
  // single-query scratch
  PinnedBuf<unsigned char> h_qtab;
  DevBuf<unsigned char> d_qtab1;
  DevBuf<double> d_scores;

  // query batch currently resident on the device (kv_query_upload and its variants)
  bool batch_valid = false;
  bool batch_selfjoin = false;  // the resident batch came from kv_selfjoin_upload (no exact threshold search)
  int64_t batch_q = 0, batch_tiles = 0, batch_h2d_bytes = 0, batch_null = 0, batch_f2_outside = 0;
  IrregularQueries irr;

  float *dbg_xs = nullptr;  // test hook (kv_debug_bound_numerators)
  float last_ms[4] = {0, 0, 0, 0};
  float last_prepare_ms[4] = {0, 0, 0, 0};  // host side of the last upload: staging, classification, text order, copies + table kernels
  float last_kernel_ms[5] = {0, 0, 0, 0, 0};  // bound pass 0, seed scan, bound pass 1, scan, merge
  float last_score_ms = 0;
  int64_t last_ctas = 0, last_tiles = 0, last_splits = 0, last_launches = 0;
  unsigned long long last_stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};

static void close_peers(kv_index *ix) {
  if (!ix->peers_borrowed)
    for (int i = 0; i < ix->n_peers; i++)
      if (ix->peer_gthr[i]) cudaIpcCloseMemHandle(ix->peer_gthr[i]);
  for (auto &p : ix->peer_gthr) p = nullptr;
  ix->n_peers = 0;
  ix->peer_cap = 0;
  ix->peers_borrowed = false;
}

static void drop_range(kv_index *ix) {
  ix->range.drop();
  ix->jrange.drop();
  ix->xrange.drop();
}

namespace {

// |q|^2 in float64, features in CSR order (the value K1a and the prep kernel compute)
double host_query_norm(const kv_index *ix, const uint32_t *ids, const uint32_t *tf, int64_t nnz, double oov_tf2) {
  const double idf0 = ix->jaccard ? 1.0 : (ix->corpus_fit ? 0.0 : std::log((double)(ix->n_total + 2) / 2.0) + 1.0);
  double nq = oov_tf2 * idf0 * idf0;
  for (int64_t i = 0; i < nnz; i++) {
    const uint32_t t = ids[i];
    const double f = (double)tf[i];
    if ((int64_t)t >= ix->V) { nq += f * f * idf0 * idf0; continue; }
    double a, d;
    idf_host(ix->n_total, ix->h_df[t], a, d, ix->jaccard, ix->corpus_fit);
    nq += f * f * a;
  }
  return nq;
}

// lexicographic order of two id sequences (shorter prefix first)
inline int cmp_seq(const uint32_t *a, int64_t na, const uint32_t *b, int64_t nb) {
  int64_t n = std::min(na, nb);
  for (int64_t i = 0; i < n; i++)
    if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  return na < nb ? -1 : (na > nb ? 1 : 0);
}

// perm := row indices sorted by (norm class, feature-id sequence).  The featuriser emits 1-grams in
// token order first, so the second key is text order up to the naming of tokens: rows with similar
// text become neighbours.  The first key groups rows whose norms B_c lie within a factor sqrt(2),
// which keeps the chunk bound (it uses the smallest norm of the chunk) tight.  Ties keep the
// original order.
void sort_rows_by_text(const std::vector<int64_t> &indptr, const std::vector<uint32_t> &ids, int64_t n,
                       const std::vector<float> &B, std::vector<int> &perm) {
  perm.resize((size_t)n);
  std::vector<short> cls((size_t)n);
  for (int64_t i = 0; i < n; i++) {
    perm[(size_t)i] = (int)i;
    cls[(size_t)i] = B[(size_t)i] > 0.f ? (short)std::floor(std::log2((double)B[(size_t)i]) * 2.0) : (short)-1000;
  }
  auto less = [&](int a, int b) {
    if (cls[(size_t)a] != cls[(size_t)b]) return cls[(size_t)a] < cls[(size_t)b];
    int c = cmp_seq(ids.data() + indptr[a], indptr[a + 1] - indptr[a], ids.data() + indptr[b],
                    indptr[b + 1] - indptr[b]);
    return c != 0 ? c < 0 : a < b;
  };
  int T = host_threads();
  if (n < 50000) T = 1;
  int parts = 1;
  while (parts * 2 <= T) parts *= 2;
  std::vector<int64_t> cut((size_t)parts + 1);
  for (int i = 0; i <= parts; i++) cut[(size_t)i] = n * i / parts;
  parallel_for(parts, parts, [&](int, int64_t a, int64_t b) {
    for (int64_t i = a; i < b; i++) std::sort(perm.begin() + cut[(size_t)i], perm.begin() + cut[(size_t)i + 1], less);
  });
  for (int width = 1; width < parts; width *= 2) {
    int merges = parts / (2 * width);
    parallel_for(merges, merges, [&](int, int64_t a, int64_t b) {
      for (int64_t m = a; m < b; m++) {
        int64_t lo = cut[(size_t)(m * 2 * width)], mid = cut[(size_t)(m * 2 * width + width)],
                hi = cut[(size_t)(m * 2 * width + 2 * width)];
        std::inplace_merge(perm.begin() + lo, perm.begin() + mid, perm.begin() + hi, less);
      }
    });
  }
}

// ---- the scan layout in host memory ----
// The arrays kv_index_finalize builds on the host cores (row order, column blocks, dense / bitmap / rare-table side
// structures) with the counts that size them.  A layout file (kv_index_layout_save) is this header followed by univ and
// then the arrays in each_array's order.
struct LayoutHeader {
  uint64_t magic, checksum;
  int64_t n_rows, nnz, V, n_chunks, n_chunks_pad, blk_words, n_entries, n_rare_entries, n_ovf, n_rt_slots, n_blocks, univ_len;
  int32_t jaccard, corpus_fit, threads, rt_enlarged;
};

struct ScanLayout {
  LayoutHeader H{};
  std::vector<uint8_t> univ;  // the universal features the layout folds into per-query constants (host only)
  std::vector<short> fslot;
  std::vector<unsigned short> fslot2;
  std::vector<int> perm;
  std::vector<BlockInfo> binfo;
  std::vector<uint32_t> blk;
  std::vector<__half> uf;
  std::vector<uint32_t> ubt, rbloom, rt_off, rt_size;
  std::vector<uint4> rt_slots;
  std::vector<unsigned long long> ovf_keys;
  std::vector<uint32_t> ovf_vals;
};

// f(host array, device buffer, entries) for every device array of the layout, in file order, until f returns false
template <class SL, class F>
bool each_array(SL &L, kv_index *ix, F &&f) {
  const LayoutHeader &H = L.H;
  const size_t V = (size_t)H.V, pad = (size_t)H.n_chunks_pad, nb = (size_t)H.n_blocks, slots = (size_t)H.n_rt_slots,
               n_ovf = (size_t)H.n_ovf;
  return f(L.fslot, ix->d_fslot, V) && f(L.fslot2, ix->d_fslot2, V) && f(L.perm, ix->d_perm, (size_t)H.n_rows) &&
         f(L.binfo, ix->d_binfo, pad) && f(L.blk, ix->d_blk, (size_t)H.blk_words) && f(L.uf, ix->d_Uf, pad * NF) &&
         f(L.ubt, ix->d_ubt, nb * NF2 * 4) && f(L.rbloom, ix->d_rbloom, nb * (RB_BITS / 32)) && f(L.rt_off, ix->d_rt_off, nb) &&
         f(L.rt_size, ix->d_rt_size, nb) && f(L.rt_slots, ix->d_rt_slots, slots) &&
         f(L.ovf_keys, ix->d_ovf_keys, n_ovf) && f(L.ovf_vals, ix->d_ovf_vals, n_ovf);
}

// Makes L the scan layout on the device: sizes the buffers, copies the arrays, builds invperm and the tensor map of the
// dense matrix, and takes L's counts.  Row norms and chunk minima are the caller's (they depend on the statistics).
int upload_layout(kv_index *ix, const ScanLayout &L) {
  cudaStream_t s = ix->stream;
  const LayoutHeader &H = L.H;
  const int64_t nz = std::max<int64_t>(H.n_rows, 1);
  KV_CUDA(ix->d_invperm.ensure(nz)); KV_CUDA(ix->d_B64.ensure(nz)); KV_CUDA(ix->d_B32.ensure(nz));
  KV_CUDA(ix->d_cminB.ensure(H.n_chunks_pad)); KV_CUDA(ix->d_blk.ensure(H.blk_words + 64));
  cudaError_t err = cudaSuccess;
  each_array(L, ix, [&](const auto &h, auto &d, size_t n) {
    err = d.ensure(std::max<int64_t>((int64_t)n, 1));
    if (err == cudaSuccess && n) err = cudaMemcpyAsync(d.p, h.data(), n * sizeof(h[0]), cudaMemcpyHostToDevice, s);
    return err == cudaSuccess;
  });
  KV_CUDA(err);
  if (H.n_rows) {
    invperm_kernel<<<(unsigned)((H.n_rows + 255) / 256), 256, 0, s>>>(ix->d_perm.p, H.n_rows, ix->d_invperm.p);
    KV_CUDA(cudaGetLastError());
  }
  KV_CUDA(cudaStreamSynchronize(s));  // the caller's staging vectors may go out of scope
  int rc = make_map_2d(&ix->map_u, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ix->d_Uf.p, H.n_chunks_pad, NF, B_BN);
  if (rc != KV_OK) return rc;
  ix->h_fslot = L.fslot; ix->h_fslot2 = L.fslot2;
  ix->n_chunks = H.n_chunks; ix->n_chunks_pad = H.n_chunks_pad; ix->blk_words = H.blk_words; ix->n_entries = H.n_entries;
  ix->n_rare_entries = H.n_rare_entries; ix->n_ovf = (int)H.n_ovf; ix->n_rt_slots = H.n_rt_slots;
  ix->rt_enlarged = H.rt_enlarged;
  ix->layout_valid = H.n_rows > 0; ix->layout_rows = H.n_rows; ix->layout_univ = L.univ;
  return KV_OK;
}

}  // namespace

extern "C" {

int kv_index_create(int device, int64_t row_base, kv_index **out) {
  if (!out) return kv_fail(KV_ERR_INVALID, "kv_index_create: out is NULL");
  int sm_count = 0;
  int rc = open_device(device, "kv_index_create", &sm_count);
  if (rc != KV_OK) return rc;
  std::unique_ptr<kv_index> ix(new kv_index());
  ix->device = device;
  ix->row_base = row_base;
  ix->sm_count = sm_count;
  KV_CUDA(ix->stream.create());
  for (auto &e : ix->ev) KV_CUDA(e.create());
  for (auto &e : ix->evk) KV_CUDA(e.create());
  for (auto &e : ix->evq) KV_CUDA(e.create());
  KV_CUDA(ix->evp2.create());
  constexpr auto smem_limit = cudaFuncAttributeMaxDynamicSharedMemorySize;
  KV_CUDA(cudaFuncSetAttribute(tfidf_score_kernel, smem_limit, 200 * 1024));
  KV_CUDA(cudaFuncSetAttribute(tfidf_scan_kernel<false, false>, smem_limit, (int)scan_smem_bytes(32)));
  KV_CUDA(cudaFuncSetAttribute(tfidf_scan_kernel<true, false>, smem_limit, (int)scan_smem_bytes(0)));
  KV_CUDA(cudaFuncSetAttribute(tfidf_scan_kernel<false, true>, smem_limit, (int)scan_smem_bytes(32, true)));
  KV_CUDA(cudaFuncSetAttribute(tfidf_scan_kernel<false, false, true>, smem_limit, (int)scan_smem_bytes(32, false, true)));
  KV_CUDA(cudaFuncSetAttribute(tfidf_scan_kernel<true, false, true>, smem_limit, (int)scan_smem_bytes(0, false, true)));
  KV_CUDA(cudaFuncSetAttribute(tfidf_scan_kernel<false, true, true>, smem_limit, (int)scan_smem_bytes(32, true, true)));
  KV_CUDA(cudaFuncSetAttribute(tfidf_bound_kernel<true>, smem_limit, 232448));
  KV_CUDA(cudaFuncSetAttribute(tfidf_bound_kernel<false>, smem_limit, 232448));
  KV_CUDA(cudaFuncSetAttribute(jaccard_scan_kernel<false>, smem_limit, (int)jaccard_smem_bytes(32)));
  KV_CUDA(cudaFuncSetAttribute(jaccard_scan_kernel<true>, smem_limit, (int)jaccard_smem_bytes(0)));
  *out = ix.release();
  return KV_OK;
}

void kv_index_destroy(kv_index *ix) {
  if (!ix) return;
  cudaSetDevice(ix->device);
  cudaStreamSynchronize(ix->stream);
  close_peers(ix);  // the peers' mapped threshold arrays: not memory this handle allocated
  delete ix;
}

int64_t kv_index_rows(const kv_index *ix) { return ix ? ix->n_rows : 0; }

int kv_index_append(kv_index *ix, const int64_t *indptr, const uint32_t *ids, const uint32_t *tf, int64_t n_rows) {
  if (!ix || n_rows < 0 || (n_rows > 0 && !indptr)) return kv_fail(KV_ERR_INVALID, "kv_index_append: bad arguments");
  if (n_rows == 0) return KV_OK;
  std::lock_guard<std::mutex> g(ix->mu);
  KV_CUDA(cudaSetDevice(ix->device));
  const int64_t add = indptr[n_rows] - indptr[0];
  if (add < 0 || (add > 0 && (!ids || !tf))) return kv_fail(KV_ERR_INVALID, "kv_index_append: bad CSR");
  if (ix->n_rows + n_rows >= (1LL << 31) - CHUNK_ROWS)
    return kv_fail(KV_ERR_INVALID, "kv_index_append: more than 2^31 rows in one shard");
  for (int64_t i = 1; i <= n_rows; i++)
    if (indptr[i] < indptr[i - 1]) return kv_fail(KV_ERR_INVALID, "kv_index_append: indptr not monotone");
  const uint32_t *tfs = tf + indptr[0];
  for (int64_t i = 0; i < add; i++)
    if (tfs[i] == 0 || tfs[i] > 65535u || (ix->jaccard && tfs[i] != 1))
      return kv_fail(KV_ERR_INVALID, "kv_index_append: term frequency %u outside 1..65535 (or != 1 in Jaccard mode)", tfs[i]);
  try {
    ix->h_indptr.reserve((size_t)(ix->n_rows + n_rows + 1));
    for (int64_t i = 1; i <= n_rows; i++) ix->h_indptr.push_back(indptr[i] - indptr[0] + ix->nnz);
    ix->h_ids.insert(ix->h_ids.end(), ids + indptr[0], ids + indptr[0] + add);
    ix->h_tf.resize((size_t)(ix->nnz + add));
    for (int64_t i = 0; i < add; i++) ix->h_tf[(size_t)(ix->nnz + i)] = (uint16_t)tfs[i];
  } catch (const std::bad_alloc &) {
    return kv_fail(KV_ERR_NOMEM, "kv_index_append: out of host memory");
  }
  KV_CUDA(ix->indptr.reserve(ix->n_rows + n_rows + 1, ix->stream));
  KV_CUDA(ix->ids.reserve(ix->nnz + add, ix->stream));
  KV_CUDA(ix->tf.reserve(ix->nnz + add, ix->stream));
  KV_CUDA(cudaMemcpyAsync(ix->indptr.p + ix->n_rows, ix->h_indptr.data() + ix->n_rows,
                          (size_t)(n_rows + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, ix->stream));
  if (add) {
    KV_CUDA(cudaMemcpyAsync(ix->ids.p + ix->nnz, ix->h_ids.data() + ix->nnz, (size_t)add * sizeof(uint32_t),
                            cudaMemcpyHostToDevice, ix->stream));
    KV_CUDA(cudaMemcpyAsync(ix->tf.p + ix->nnz, ix->h_tf.data() + ix->nnz, (size_t)add * sizeof(uint16_t),
                            cudaMemcpyHostToDevice, ix->stream));
  }
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  ix->n_rows += n_rows;
  ix->nnz += add;
  ix->indptr.n = ix->n_rows + 1;
  ix->ids.n = ix->nnz;
  ix->tf.n = ix->nnz;
  ix->finalized = false;
  drop_range(ix);
  // labels and groups describe the rows they were given for: a filtered or distinct query fails until they are set
  // again.  Deleted rows stay deleted.
  ix->labels.clear();
  ix->groups.clear();
  ix->tags.clear();
  ix->tomb.extend(ix->n_rows);
  return KV_OK;
}

int kv_index_set_mode(kv_index *ix, int mode) {
  if (!ix || (mode != KV_MODE_TFIDF_COSINE && mode != KV_MODE_JACCARD && mode != KV_MODE_TFIDF_CORPUS_FIT))
    return kv_fail(KV_ERR_INVALID, "kv_index_set_mode: mode must be KV_MODE_TFIDF_COSINE, KV_MODE_JACCARD or KV_MODE_TFIDF_CORPUS_FIT");
  std::lock_guard<std::mutex> g(ix->mu);
  if (mode == KV_MODE_JACCARD && ix->tomb.any())
    return kv_fail(KV_ERR_INVALID, "kv_index_set_mode: a Jaccard index (mode 1) has no row deletion, and rows are deleted");
  if (mode == KV_MODE_JACCARD)
    for (uint16_t f : ix->h_tf)
      if (f != 1) return kv_fail(KV_ERR_INVALID, "kv_index_set_mode: Jaccard rows are token SETS (every tf must be 1)");
  ix->jaccard = mode == KV_MODE_JACCARD;
  ix->corpus_fit = mode == KV_MODE_TFIDF_CORPUS_FIT;
  ix->finalized = false;
  ix->layout_valid = false;
  return KV_OK;
}

// |q ∩ row| and |q ∪ row| of already selected (query, row) pairs, exact integers (host; Q*k pairs)
int kv_jaccard_counts(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const double *q_oov_tf2, int64_t n_q,
                      int k, const int64_t *rows, int32_t *out_inter, int32_t *out_union) {
  if (!ix || n_q < 0 || k < 1 || (n_q > 0 && (!q_indptr || !rows || !out_inter || !out_union)))
    return kv_fail(KV_ERR_INVALID, "kv_jaccard_counts: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  std::vector<uint32_t> qs, rs;
  for (int64_t q = 0; q < n_q; q++) {
    qs.assign(q_ids + q_indptr[q], q_ids + q_indptr[q + 1]);
    std::sort(qs.begin(), qs.end());
    const int64_t nq = (int64_t)qs.size() + (q_oov_tf2 ? (int64_t)q_oov_tf2[q] : 0);
    for (int j = 0; j < k; j++) {
      const int64_t r = rows[q * k + j] - ix->row_base;
      if (rows[q * k + j] < 0 || r < 0 || r >= ix->n_rows) { out_inter[q * k + j] = out_union[q * k + j] = -1; continue; }
      rs.assign(ix->h_ids.begin() + ix->h_indptr[(size_t)r], ix->h_ids.begin() + ix->h_indptr[(size_t)r + 1]);
      std::sort(rs.begin(), rs.end());
      int32_t inter = 0;
      for (size_t a = 0, b = 0; a < qs.size() && b < rs.size();) {
        if (qs[a] == rs[b]) { inter++; a++; b++; }
        else if (qs[a] < rs[b]) a++;
        else b++;
      }
      out_inter[q * k + j] = inter;
      out_union[q * k + j] = (int32_t)(nq + (int64_t)rs.size() - inter);
    }
  }
  return KV_OK;
}

int kv_index_set_global_df(kv_index *ix, const uint32_t *df, int64_t vocab_size, int64_t n_rows_global) {
  if (!ix || !df || vocab_size < 0 || n_rows_global < 0)
    return kv_fail(KV_ERR_INVALID, "kv_index_set_global_df: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  ix->h_gdf.assign(df, df + vocab_size);
  ix->n_global = n_rows_global;
  ix->has_gdf = true;
  ix->finalized = false;
  return KV_OK;
}

// Document frequencies of the live rows: d_cnt (every row of the layout, already histogrammed) minus the entries of the
// deleted rows, in d_dcnt; *out = d_cnt itself when nothing is deleted.  Caller holds ix->mu.
static int live_counts(kv_index *ix, int64_t Vz, const uint32_t **out) {
  *out = ix->d_cnt.p;
  if (!ix->tomb.any()) return KV_OK;
  cudaStream_t s = ix->stream;
  std::vector<int> list;
  list.reserve((size_t)ix->tomb.count);
  for (int64_t r = 0; r < ix->n_rows; r++)
    if (ix->tomb.is_dead(r)) list.push_back((int)r);
  KV_CUDA(ix->d_dead_list.ensure((int64_t)list.size()));
  KV_CUDA(ix->d_dcnt.ensure(Vz));
  KV_CUDA(cudaMemcpyAsync(ix->d_dead_list.p, list.data(), list.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemsetAsync(ix->d_dcnt.p, 0, (size_t)Vz * sizeof(uint32_t), s));
  hist_rows_kernel<<<(unsigned)(((int64_t)list.size() * 32 + 255) / 256), 256, 0, s>>>(ix->indptr.p, ix->ids.p, ix->d_dead_list.p,
                                                                                       (int64_t)list.size(), ix->d_dcnt.p);
  KV_CUDA(cudaGetLastError());
  sub_count_kernel<<<(unsigned)((Vz + 255) / 256), 256, 0, s>>>(ix->d_cnt.p, ix->d_dcnt.p, Vz, ix->d_dcnt.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(s));  // the host list goes out of scope
  *out = ix->d_dcnt.p;
  return KV_OK;
}

int kv_index_local_df(kv_index *ix, uint32_t *df_out, int64_t vocab_size) {
  if (!ix || !df_out || vocab_size < 0) return kv_fail(KV_ERR_INVALID, "kv_index_local_df: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  KV_CUDA(cudaSetDevice(ix->device));
  for (uint32_t t : ix->h_ids)
    if ((int64_t)t >= vocab_size) return kv_fail(KV_ERR_INVALID, "kv_index_local_df: feature id %u outside vocabulary", t);
  KV_CUDA(ix->d_cnt.ensure(std::max<int64_t>(vocab_size, 1)));
  KV_CUDA(cudaMemsetAsync(ix->d_cnt.p, 0, (size_t)std::max<int64_t>(vocab_size, 1) * sizeof(uint32_t), ix->stream));
  if (ix->nnz) {
    hist_kernel<<<ix->sm_count * 8, 256, 0, ix->stream>>>(ix->ids.p, ix->tf.p, ix->nnz, ix->d_cnt.p, nullptr, nullptr);
    KV_CUDA(cudaGetLastError());
  }
  const uint32_t *live = nullptr;
  int rc = live_counts(ix, std::max<int64_t>(vocab_size, 1), &live);  // deleted rows do not count
  if (rc != KV_OK) return rc;
  if (vocab_size)
    KV_CUDA(cudaMemcpyAsync(df_out, live, (size_t)vocab_size * sizeof(uint32_t), cudaMemcpyDeviceToHost, ix->stream));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return KV_OK;
}

// a(t), d(t) as the HOST computes them (idf_host: the values every query table is built from) -> d_a64/d_d64, so
// that K6 multiplies the very same doubles as K1a
static int upload_idf_tables(kv_index *ix, int64_t V) {
  if (V <= 0) return KV_OK;
  std::vector<double> ha((size_t)V), hd((size_t)V);
  parallel_for(V, V >= 65536 ? host_threads() : 1, [&](int, int64_t a0, int64_t a1) {
    for (int64_t t = a0; t < a1; t++) idf_host(ix->n_total, ix->h_df[(size_t)t], ha[(size_t)t], hd[(size_t)t], ix->jaccard, ix->corpus_fit);
  });
  KV_CUDA(cudaMemcpyAsync(ix->d_a64.p, ha.data(), (size_t)V * 8, cudaMemcpyHostToDevice, ix->stream));
  KV_CUDA(cudaMemcpyAsync(ix->d_d64.p, hd.data(), (size_t)V * 8, cudaMemcpyHostToDevice, ix->stream));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return KV_OK;
}

// The device copies of one per-row set for the current layout (by row and by scan position); the labels add their
// chunk signatures (scan and selection) and the first LAB_FIRST live rows of every label (null queries).  Nothing to
// do until the index is finalized; every finalize calls it again.
static int upload_row_set(kv_index *ix, RowSet &rs) {
  rs.on_device = false;
  if (!rs.has || !ix->finalized) return KV_OK;
  cudaStream_t s = ix->stream;
  const int64_t n = ix->n_rows;
  int rc = rs.upload(ix->d_perm.p, n, ix->n_chunks_pad * CHUNK_ROWS, s);
  if (rc != KV_OK) return rc;
  if (&rs == &ix->labels) {
    std::vector<int> keys(rs.h);
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    std::vector<int> first(keys.size() * LAB_FIRST, -1), cnt(keys.size(), 0);
    for (int64_t r = 0; r < n; r++) {
      if (ix->tomb.is_dead(r)) continue;  // null queries get live rows only
      const size_t i = (size_t)(std::lower_bound(keys.begin(), keys.end(), rs.h[(size_t)r]) - keys.begin());
      if (cnt[i] < LAB_FIRST) first[i * LAB_FIRST + (size_t)cnt[i]++] = (int)r;
    }
    ix->n_lab = (int)keys.size();
    KV_CUDA(ix->d_lab_keys.ensure(std::max<int64_t>((int64_t)keys.size(), 1)));
    KV_CUDA(ix->d_lab_rows.ensure(std::max<int64_t>((int64_t)first.size(), 1)));
    if (!keys.empty()) {
      KV_CUDA(cudaMemcpyAsync(ix->d_lab_keys.p, keys.data(), keys.size() * sizeof(int), cudaMemcpyHostToDevice, s));
      KV_CUDA(cudaMemcpyAsync(ix->d_lab_rows.p, first.data(), first.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    }
    if (n > 0) {
      KV_CUDA(ix->d_chunk_sig.ensure(ix->n_chunks_pad));
      chunk_sig_kernel<<<(unsigned)((ix->n_chunks_pad + 255) / 256), 256, 0, s>>>(rs.d_pos.p, ix->n_chunks_pad, ix->d_chunk_sig.p);
      KV_CUDA(cudaGetLastError());
    }
    KV_CUDA(cudaStreamSynchronize(s));  // the host staging vectors go out of scope
  }
  rs.on_device = true;
  return KV_OK;
}

static const uint32_t *alive_words(const kv_index *ix);

// The device copies of the row tags for the current layout (d_perm, and d_alive when rows are deleted, must hold it):
// masks and tag lists by scan position, chunk signatures over the live rows.  Nothing until the index is finalized.
static int upload_row_tags(kv_index *ix) {
  RowTags &T = ix->tags;
  T.on_device = false;
  if (!T.has || !ix->finalized) return KV_OK;
  const int64_t n = ix->n_rows, n_pos = ix->n_chunks_pad * CHUNK_ROWS;
  if (n == 0) { T.on_device = true; return KV_OK; }
  cudaStream_t s = ix->stream;
  std::vector<int> perm((size_t)n);
  KV_CUDA(cudaMemcpyAsync(perm.data(), ix->d_perm.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  std::vector<unsigned long long> mask((size_t)n_pos, 0ull);
  std::vector<int64_t> ptr;
  std::vector<int> list;
  if (!T.masks_exact) { ptr.assign((size_t)n_pos + 1, 0); list.reserve(T.tags.size()); }
  for (int64_t p = 0; p < n_pos; p++) {
    if (p < n) {
      const int64_t r = perm[(size_t)p];
      for (int64_t i = T.indptr[(size_t)r]; i < T.indptr[(size_t)r + 1]; i++) {
        mask[(size_t)p] |= 1ull << (T.tags[(size_t)i] & 63);
        if (!T.masks_exact) list.push_back(T.tags[(size_t)i]);
      }
    }
    if (!T.masks_exact) ptr[(size_t)p + 1] = (int64_t)list.size();
  }
  KV_CUDA(T.d_mask_pos.ensure(n_pos));
  KV_CUDA(T.d_chunk_sig.ensure(ix->n_chunks_pad));
  KV_CUDA(cudaMemcpyAsync(T.d_mask_pos.p, mask.data(), mask.size() * 8, cudaMemcpyHostToDevice, s));
  if (!T.masks_exact) {
    KV_CUDA(T.d_ptr_pos.ensure(n_pos + 1));
    KV_CUDA(T.d_list_pos.ensure(std::max<int64_t>((int64_t)list.size(), 1)));
    KV_CUDA(cudaMemcpyAsync(T.d_ptr_pos.p, ptr.data(), ptr.size() * 8, cudaMemcpyHostToDevice, s));
    if (!list.empty()) KV_CUDA(cudaMemcpyAsync(T.d_list_pos.p, list.data(), list.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  chunk_tag_sig_kernel<<<(unsigned)((ix->n_chunks_pad + 255) / 256), 256, 0, s>>>(T.d_mask_pos.p, alive_words(ix), ix->n_chunks_pad,
                                                                                T.d_chunk_sig.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(s));  // the host staging vectors go out of scope
  T.on_device = true;
  return KV_OK;
}

// the per-row sets a finalize rebuilds on the device: labels, groups and tags
static int upload_row_sets(kv_index *ix) {
  int rc = upload_row_set(ix, ix->labels);
  if (rc == KV_OK) rc = upload_row_set(ix, ix->groups);
  return rc != KV_OK ? rc : upload_row_tags(ix);
}

// A filtered batch never runs on labels or tags that do not describe the current rows
static int check_filter(const kv_index *ix, const char *fn) {
  if (ix->has_filter && !ix->labels.ready(ix->n_rows))
    return kv_fail(KV_ERR_STATE, "%s: the batch is filtered but the row labels are missing or stale (set them again after an append)", fn);
  if (ix->qtags.on && !ix->tags.ready(ix->n_rows))
    return kv_fail(KV_ERR_STATE, "%s: the batch is tag-filtered but the row tags are missing or stale (set them again after an append)", fn);
  return KV_OK;
}

int kv_index_set_row_tags(kv_index *ix, const int64_t *indptr, const int32_t *tags, int64_t n_rows) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_tags: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!indptr) {
    ix->tags.clear();
    return KV_OK;
  }
  if (ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_tags: a Jaccard index (mode 1) has no tag filter");
  const int rc = ix->tags.set(indptr, tags, n_rows, ix->n_rows, "kv_index_set_row_tags");
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaSetDevice(ix->device));
  return upload_row_tags(ix);
}

int kv_index_set_row_labels(kv_index *ix, const int32_t *labels, int64_t n) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_labels: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!labels) {
    ix->labels.clear();
    return KV_OK;
  }
  const int rc = ix->labels.set(labels, n, ix->n_rows, "kv_index_set_row_labels", "label");
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaSetDevice(ix->device));
  return upload_row_set(ix, ix->labels);
}

int kv_index_set_row_groups(kv_index *ix, const int32_t *groups, int64_t n) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_groups: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!groups) {
    ix->groups.clear();
    return KV_OK;
  }
  if (ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_groups: a Jaccard index (mode 1) has no distinct top-k");
  const int rc = ix->groups.set(groups, n, ix->n_rows, "kv_index_set_row_groups", "group");
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaSetDevice(ix->device));
  return upload_row_set(ix, ix->groups);
}

// The device copies of the deletions for the current layout (d_perm must hold it): deleted flags by row, the live word
// of every chunk and the first LAB_FIRST live rows.  Nothing while no row is deleted: the kernels then get NULL.
static int upload_dead(kv_index *ix) {
  if (!ix->tomb.any() || ix->n_rows == 0) return KV_OK;
  cudaStream_t s = ix->stream;
  const int64_t n = ix->n_rows;
  std::vector<int> first(LAB_FIRST, -1);
  for (int64_t r = 0, c = 0; r < n && c < LAB_FIRST; r++)
    if (!ix->tomb.is_dead(r)) first[(size_t)c++] = (int)r;
  KV_CUDA(ix->d_dead.ensure(n));
  KV_CUDA(ix->d_alive.ensure(ix->n_chunks_pad));
  KV_CUDA(ix->d_first_live.ensure(LAB_FIRST));
  KV_CUDA(cudaMemcpyAsync(ix->d_dead.p, ix->tomb.flags.data(), (size_t)n, cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemcpyAsync(ix->d_first_live.p, first.data(), first.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  alive_kernel<<<(unsigned)((ix->n_chunks_pad + 255) / 256), 256, 0, s>>>(ix->d_perm.p, ix->d_dead.p, n, ix->n_chunks_pad, ix->d_alive.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(s));  // the host list goes out of scope
  return KV_OK;
}

// NULL while no row is deleted: the kernels' per-row and per-chunk tests are then skipped
static const uint8_t *dead_rows(const kv_index *ix) { return ix->tomb.any() ? ix->d_dead.p : nullptr; }
static const uint32_t *alive_words(const kv_index *ix) { return ix->tomb.any() ? ix->d_alive.p : nullptr; }

// The rows a query may not match in the float64 fallbacks (*out, NULL: none): the deleted rows and, when the query has
// tags (q_mask != 0, d_q_tags its MAX_QTAGS ascending tags on the device), the rows whose tag set misses its own --
// those are written to d_tagdead, which the launches that follow on the stream read.
static int fallback_dead(kv_index *ix, unsigned long long q_mask, const int *d_q_tags, const uint8_t **out) {
  *out = dead_rows(ix);
  if (q_mask == 0ull || ix->n_rows == 0) return KV_OK;
  const RowTags &T = ix->tags;
  KV_CUDA(ix->d_tagdead.ensure(ix->n_rows));
  tag_dead_kernel<<<(unsigned)((ix->n_rows + 255) / 256), 256, 0, ix->stream>>>(
      ix->d_invperm.p, ix->n_rows, T.d_mask_pos.p, T.masks_exact ? nullptr : T.d_ptr_pos.p,
      T.masks_exact ? nullptr : T.d_list_pos.p, q_mask, d_q_tags, dead_rows(ix), ix->d_tagdead.p);
  KV_CUDA(cudaGetLastError());
  *out = ix->d_tagdead.p;
  return KV_OK;
}

// fallback_dead for query q (original index) of the resident batch
static int batch_fallback_dead(kv_index *ix, int64_t q, const uint8_t **out) {
  if (!ix->qtags.on) { *out = dead_rows(ix); return KV_OK; }
  return fallback_dead(ix, ix->qtags.h_mask[(size_t)q], ix->qtags.d_tags_orig.p + q * MAX_QTAGS, out);
}

int kv_index_delete_rows(kv_index *ix, const int64_t *rows, int64_t n) {
  if (!ix || n < 0 || (n > 0 && !rows)) return kv_fail(KV_ERR_INVALID, "kv_index_delete_rows: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_index_delete_rows: a Jaccard index (mode 1) has no row deletion");
  int64_t added = 0;
  const int rc = ix->tomb.mark(rows, n, ix->n_rows, "kv_index_delete_rows", &added);
  if (rc != KV_OK || !added) return rc;  // duplicates and rows deleted before: nothing changes
  // like an append: statistics and the device copies are stale until the next finalize
  ix->finalized = false;
  ix->batch_valid = false;
  drop_range(ix);
  return KV_OK;
}

int64_t kv_index_live_rows(const kv_index *ix) { return ix ? ix->n_rows - ix->tomb.count : 0; }

int kv_index_deleted_rows(kv_index *ix, uint8_t *out, int64_t n) {
  if (!ix || n < 0 || (n > 0 && !out)) return kv_fail(KV_ERR_INVALID, "kv_index_deleted_rows: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  return ix->tomb.copy_out(out, n, ix->n_rows, "kv_index_deleted_rows");
}

// The end of both kinds of finalize (kind 1: full rebuild, 2: statistics-only refresh), once the scan layout is on the
// device: row norms in scan order, the deletions and the chunk minima.  The index is then finalized for a vocabulary of V
// features, the batch and the range result are dropped and the per-row sets are rebuilt for the layout.
static int finish_finalize(kv_index *ix, int64_t V, int kind) {
  cudaStream_t s = ix->stream;
  const int64_t n = ix->n_rows;
  if (n) {
    rownorm_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(ix->indptr.p, ix->ids.p, ix->tf.p, ix->d_perm.p, n,
                                                                    ix->d_bb64.p, ix->d_B64.p, ix->d_B32.p);
    KV_CUDA(cudaGetLastError());
  }
  const int rc = upload_dead(ix);
  if (rc != KV_OK) return rc;
  chunk_meta_kernel<<<(unsigned)((ix->n_chunks_pad + 255) / 256), 256, 0, s>>>(ix->d_B32.p, n, ix->n_chunks, ix->n_chunks_pad,
                                                                                alive_words(ix), ix->d_cminB.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(s));
  ix->V = V;
  ix->finalized = true;
  ix->batch_valid = false;
  drop_range(ix);
  ix->last_finalize_kind = kind;
  return upload_row_sets(ix);
}

int kv_index_finalize(kv_index *ix, int64_t vocab_size) {
  if (!ix || vocab_size < 0) return kv_fail(KV_ERR_INVALID, "kv_index_finalize: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  KV_CUDA(cudaSetDevice(ix->device));
  if (vocab_size >= (int64_t)FID_NONE)
    return kv_fail(KV_ERR_INVALID, "kv_index_finalize: vocabulary of %lld features exceeds the 2^26-1 the scan layout encodes",
                   (long long)vocab_size);
  if (ix->has_gdf && (int64_t)ix->h_gdf.size() != vocab_size)
    return kv_fail(KV_ERR_INVALID, "kv_index_finalize: global df has %lld entries, vocabulary %lld",
                   (long long)ix->h_gdf.size(), (long long)vocab_size);
  cudaStream_t s = ix->stream;
  const int64_t V = vocab_size, n = ix->n_rows;
  {
    uint32_t mx = 0;
    for (uint32_t t : ix->h_ids) mx = std::max(mx, t);
    if (ix->nnz && (int64_t)mx >= V)
      return kv_fail(KV_ERR_INVALID, "kv_index_finalize: feature id %u outside vocabulary of %lld", mx, (long long)V);
  }
  // ---- statistics on the device: df, idf tables, universal features ----
  const int64_t Vz = V > 0 ? V : 1;
  KV_CUDA(ix->d_df.ensure(Vz)); KV_CUDA(ix->d_cnt.ensure(Vz)); KV_CUDA(ix->d_tfmin.ensure(Vz));
  KV_CUDA(ix->d_tfmax.ensure(Vz)); KV_CUDA(ix->d_utf.ensure(Vz));
  KV_CUDA(ix->d_a64.ensure(Vz)); KV_CUDA(ix->d_d64.ensure(Vz)); KV_CUDA(ix->d_bb64.ensure(Vz));
  KV_CUDA(ix->d_univ.ensure(Vz));
  KV_CUDA(cudaMemsetAsync(ix->d_cnt.p, 0, (size_t)Vz * 4, s));
  KV_CUDA(cudaMemsetAsync(ix->d_tfmin.p, 0xFF, (size_t)Vz * 4, s));
  KV_CUDA(cudaMemsetAsync(ix->d_tfmax.p, 0, (size_t)Vz * 4, s));
  if (ix->nnz) {
    hist_kernel<<<ix->sm_count * 8, 256, 0, s>>>(ix->ids.p, ix->tf.p, ix->nnz, ix->d_cnt.p, ix->d_tfmin.p, ix->d_tfmax.p);
    KV_CUDA(cudaGetLastError());
  }
  if (ix->has_gdf) {
    if (V) KV_CUDA(cudaMemcpyAsync(ix->d_df.p, ix->h_gdf.data(), (size_t)V * 4, cudaMemcpyHostToDevice, s));
    ix->n_total = ix->n_global;
  } else {
    // N and df count live rows; d_cnt keeps counting every row of the layout, which is what decides a universal
    // feature (folded into per-query constants): a deletion alone therefore never changes the layout
    const uint32_t *live = nullptr;
    int rc = live_counts(ix, Vz, &live);
    if (rc != KV_OK) return rc;
    if (V) KV_CUDA(cudaMemcpyAsync(ix->d_df.p, live, (size_t)V * 4, cudaMemcpyDeviceToDevice, s));
    ix->n_total = n - ix->tomb.count;
  }
  if (V) {
    IdfTables T{ix->d_a64.p, ix->d_d64.p, ix->d_bb64.p, ix->d_univ.p, ix->d_utf.p};
    idf_kernel<<<(unsigned)((V + 255) / 256), 256, 0, s>>>(ix->d_df.p, ix->d_cnt.p, ix->d_tfmin.p, ix->d_tfmax.p, V,
                                                            ix->n_total, n, ix->jaccard, ix->corpus_fit, T);
    KV_CUDA(cudaGetLastError());
  }
  ix->h_df.assign((size_t)V, 0);
  ix->h_univ.assign((size_t)Vz, 0);
  ix->h_utf.assign((size_t)V, 0);
  ix->h_tfmax.assign((size_t)Vz, 0);
  if (V) {
    KV_CUDA(cudaMemcpyAsync(ix->h_df.data(), ix->d_df.p, (size_t)V * 4, cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaMemcpyAsync(ix->h_univ.data(), ix->d_univ.p, (size_t)V, cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaMemcpyAsync(ix->h_utf.data(), ix->d_utf.p, (size_t)V * 4, cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaMemcpyAsync(ix->h_tfmax.data(), ix->d_tfmax.p, (size_t)V * 4, cudaMemcpyDeviceToHost, s));
  }
  // row norms in original order (the sort key needs them)
  const int64_t nz = n > 0 ? n : 1;
  KV_CUDA(ix->d_perm.ensure(nz));
  KV_CUDA(ix->d_B64.ensure(nz)); KV_CUDA(ix->d_B32.ensure(nz));
  std::vector<float> hB((size_t)n);
  if (n) {
    rownorm_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(ix->indptr.p, ix->ids.p, ix->tf.p, nullptr, n,
                                                                    ix->d_bb64.p, ix->d_B64.p, ix->d_B32.p);
    KV_CUDA(cudaGetLastError());
    KV_CUDA(cudaMemcpyAsync(hB.data(), ix->d_B32.p, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  KV_CUDA(cudaStreamSynchronize(s));
  ix->n_univ = 0;
  for (int64_t t = 0; t < V; t++) ix->n_univ += ix->h_univ[(size_t)t];
  {
    int rc = upload_idf_tables(ix, V);
    if (rc != KV_OK) return rc;
  }
  // ---- statistics-only refresh: the rows (hence their order and the column blocks, which hold term frequencies and
  // row masks only) are the ones the device layout was built from and the set of folded universal features is
  // unchanged; only N / df moved (rows were appended to ANOTHER shard or segment of the same GFKB).  Row norms and chunk
  // minima are recomputed, nothing is re-sorted.
  if (ix->layout_valid && ix->layout_rows == n && n > 0 && !getenv("KAKVEDA_B200_FULL_FINALIZE")) {
    bool same = (int64_t)ix->layout_univ.size() <= Vz;
    for (size_t t = 0; same && t < ix->layout_univ.size(); t++) same = ix->layout_univ[t] == ix->h_univ[t];
    for (size_t t = ix->layout_univ.size(); same && t < (size_t)V; t++) same = ix->h_univ[t] == 0;
    if (same) {
      if ((int64_t)ix->h_fslot.size() < Vz) {  // new feature ids (rows of another segment): none of them is a dense column
        ix->h_fslot.resize((size_t)Vz, (short)-1);
        ix->h_fslot2.resize((size_t)Vz, (unsigned short)0xFFFF);
        KV_CUDA(ix->d_fslot.ensure(Vz));
        KV_CUDA(ix->d_fslot2.ensure(Vz));
        KV_CUDA(cudaMemcpyAsync(ix->d_fslot.p, ix->h_fslot.data(), (size_t)Vz * sizeof(short), cudaMemcpyHostToDevice, s));
        KV_CUDA(cudaMemcpyAsync(ix->d_fslot2.p, ix->h_fslot2.data(), (size_t)Vz * sizeof(short), cudaMemcpyHostToDevice, s));
      }
      return finish_finalize(ix, V, 2);
    }
  }
  ix->layout_valid = false;
  // ---- on the host cores: (norm class, text) order of the rows, then the column blocks ----
  ScanLayout SL;
  sort_rows_by_text(ix->h_indptr, ix->h_ids, n, hB, SL.perm);
  {
    BlockLayout L;
    build_blocks(ix->h_indptr.data(), ix->h_ids.data(), ix->h_tf.data(), SL.perm.data(), n, V, ix->h_univ.data(),
                 ix->h_tfmax.data(), host_threads(), L, /*linear_tables=*/false);
    LayoutHeader &H = SL.H;
    H.n_rows = n; H.V = Vz; H.n_chunks = L.n_chunks; H.n_chunks_pad = L.n_chunks_pad; H.n_blocks = L.n_chunks_pad / 64;
    H.blk_words = L.total_words; H.n_entries = L.n_entries; H.n_rare_entries = L.n_rare_entries;
    H.n_rt_slots = (int64_t)L.rt_slots.size(); H.rt_enlarged = (int32_t)L.rt_enlarged; H.n_ovf = (int64_t)L.ovf.size(); H.univ_len = Vz;
    SL.univ = ix->h_univ;
    SL.fslot = std::move(L.fslot); SL.fslot2 = std::move(L.fslot2); SL.binfo = std::move(L.binfo); SL.uf = std::move(L.Uf);
    SL.ubt = std::move(L.Ubt); SL.rbloom = std::move(L.rbloom); SL.rt_off = std::move(L.rt_off); SL.rt_size = std::move(L.rt_size);
    SL.rt_slots = std::move(L.rt_slots);
    SL.blk.reserve((size_t)L.total_words);
    for (auto &part : L.parts) {  // the blocks of each build thread, back to back
      SL.blk.insert(SL.blk.end(), part.begin(), part.end());
      std::vector<uint32_t>().swap(part);
    }
    for (const auto &o : L.ovf) { SL.ovf_keys.push_back(o.first); SL.ovf_vals.push_back(o.second); }
  }
  const int rc = upload_layout(ix, SL);
  return rc != KV_OK ? rc : finish_finalize(ix, V, 1);
}

int kv_index_last_finalize_kind(const kv_index *ix) { return ix ? ix->last_finalize_kind : 0; }

// caller holds ix->mu; scores land in ix->d_scores and, when out_scores != NULL, on the host
static int score_impl(kv_index *ix, const uint32_t *q_ids, const uint32_t *q_tf, int64_t q_nnz, double q_oov_tf2,
                      double *out_scores) {
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_score: index not finalized");
  if (ix->n_rows == 0) return KV_OK;
  if (ix->nnz == 0 && q_nnz == 0 && q_oov_tf2 == 0.0)
    return kv_fail(KV_ERR_EMPTY_VOCAB, "empty vocabulary; perhaps the documents only contain stop words");
  KV_CUDA(cudaSetDevice(ix->device));
  // per-query constants in float64 (features in CSR order)
  const double idf0 = ix->jaccard ? 1.0 : (ix->corpus_fit ? 0.0 : std::log((double)(ix->n_total + 2) / 2.0) + 1.0);
  double nq = q_oov_tf2 * idf0 * idf0, dotU = 0, corrU = 0, maxdot = 1.0, maxcorr = 1e-30;
  std::vector<uint32_t> fid, tfq;
  std::vector<double> fa, fd;
  for (int64_t i = 0; i < q_nnz; i++) {
    const uint32_t t = q_ids[i];
    const double f = (double)q_tf[i];
    if ((int64_t)t >= ix->V) { nq += f * f * idf0 * idf0; continue; }  // id issued after finalize: in no indexed row
    double a, d;
    idf_host(ix->n_total, ix->h_df[t], a, d, ix->jaccard, ix->corpus_fit);
    nq += f * f * a;
    if (ix->h_univ[t]) {
      const double u = (double)ix->h_utf[t];
      dotU += f * u * a;
      corrU += u * u * d;
    } else {
      fid.push_back(t); tfq.push_back(q_tf[i]); fa.push_back(a); fd.push_back(d);
      const double tm = (double)ix->h_tfmax[t];
      maxdot += f * a * tm;
      maxcorr += -d * tm * tm;
    }
  }
  int log_h = 6;
  while ((1 << log_h) < 2 * (int)fid.size() + 2) log_h++;
  if (log_h > 13) return kv_fail(KV_ERR_INVALID, "kv_score: query has too many distinct features");
  const int H = 1 << log_h;
  // fixed point: the largest power-of-two scales that keep every row sum below 2^62
  const int e_w = std::max(0, std::min(50, (int)std::floor(62.0 - std::log2(maxdot))));
  const int e_c = std::max(0, std::min(50, (int)std::floor(62.0 - std::log2(maxcorr))));
  const size_t tab_bytes = (size_t)H * (8 + 8 + 4);
  KV_CUDA(ix->h_qtab.ensure((int64_t)tab_bytes));
  KV_CUDA(ix->d_qtab1.ensure((int64_t)tab_bytes));
  unsigned long long *tw = (unsigned long long *)ix->h_qtab.p, *tc = tw + H;
  uint32_t *tk = (uint32_t *)(tc + H);
  for (int i = 0; i < H; i++) { tk[i] = KEY_EMPTY; tw[i] = 0; tc[i] = 0; }
  for (size_t i = 0; i < fid.size(); i++) {
    const uint32_t t = fid[i];
    uint32_t h = (t * 0x9E3779B1u) >> (32 - log_h);
    while (tk[h] != KEY_EMPTY) h = (h + 1) & (H - 1);
    tk[h] = t;
    tw[h] = (unsigned long long)std::llrint(std::ldexp((double)tfq[i] * fa[i], e_w));
    tc[h] = (unsigned long long)std::llrint(std::ldexp(-fd[i], e_c));
  }
  cudaStream_t s = ix->stream;
  KV_CUDA(cudaMemcpyAsync(ix->d_qtab1.p, ix->h_qtab.p, tab_bytes, cudaMemcpyHostToDevice, s));
  KV_CUDA(ix->d_scores.ensure(ix->n_rows));
  ScoreParams P;
  P.blk = ix->d_blk.p; P.binfo = ix->d_binfo.p; P.perm = ix->d_perm.p;
  P.n_chunks = ix->n_chunks; P.n_rows = ix->n_rows;
  P.B64 = ix->d_B64.p; P.ovf_keys = ix->d_ovf_keys.p; P.ovf_vals = ix->d_ovf_vals.p; P.n_ovf = ix->n_ovf;
  P.qw = (const unsigned long long *)ix->d_qtab1.p; P.qc = P.qw + H; P.qkeys = (const uint32_t *)(P.qc + H);
  P.log_h = log_h;
  P.w_unscale = std::ldexp(1.0, -e_w); P.c_unscale = std::ldexp(1.0, -e_c);
  P.nq = nq; P.dotU = dotU; P.corrU = corrU; P.jaccard = ix->jaccard; P.dead = dead_rows(ix); P.out = ix->d_scores.p;
  const size_t smem = tab_bytes + 8 * 32 * 24;
  int blocks = (int)std::min<int64_t>((ix->n_chunks + 7) / 8, (int64_t)ix->sm_count * 8);
  if (blocks < 1) blocks = 1;
  KV_CUDA(cudaEventRecord(ix->ev[1], s));
  tfidf_score_kernel<<<blocks, 256, smem, s>>>(P);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaEventRecord(ix->ev[2], s));
  if (out_scores)
    KV_CUDA(cudaMemcpyAsync(out_scores, ix->d_scores.p, (size_t)ix->n_rows * sizeof(double), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  cudaEventElapsedTime(&ix->last_score_ms, ix->ev[1], ix->ev[2]);
  return KV_OK;
}

int kv_score(kv_index *ix, const uint32_t *q_ids, const uint32_t *q_tf, int64_t q_nnz, double q_oov_tf2,
             double *out_scores) {
  if (!ix || q_nnz < 0 || (q_nnz > 0 && (!q_ids || !q_tf)))
    return kv_fail(KV_ERR_INVALID, "kv_score: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (ix->finalized && ix->n_rows > 0 && !out_scores) return kv_fail(KV_ERR_INVALID, "kv_score: out_scores is NULL");
  return score_impl(ix, q_ids, q_tf, q_nnz, q_oov_tf2, out_scores);
}

// ---- batched top-k, in two halves: prepare_batch (host work + H2D + table kernels) and run_batch (device only) ----
// A query batch arrives as one CSR or as several consecutive "runs" (a row-sharded GFKB featurises one slice of the
// batch per rank and exchanges the slices, kakveda_b200/dist.py); a run may bring its own classification flags and its
// own text order (kv_query_prepare_slice), which are then merged instead of recomputed.
struct QueryRun {
  const int64_t *indptr = nullptr;
  const uint32_t *ids = nullptr, *tf = nullptr;
  const double *oov = nullptr;
  // optional (kv_query_prepare_slice): the run's rows are stored SORTED by feature-id sequence (ties by original
  // index) and order[p] = original index, inside the run, of the query in row p -- merging then walks memory in order
  const int32_t *order = nullptr;
  const uint8_t *flags = nullptr;   // optional, by row: 0 regular, 1 null, 2 irregular, 3 off (a deleted row's self-join)
  int64_t n_q = 0;
};

// null: no feature of the query is in the index (every score is 0).  irregular: more features than a query table
// holds, or term frequencies so large that the 64-bit fixed-point sums or the fp16 bound weights could overflow --
// such a query takes the float64 full-scan path (K1a + selection).  The scan's sums, universal features included
// (their common tf u stands in for tfmax; prep_queries_kernel folds them as the integers their entries would add):
// a row's dot sum adds tf_c round(tf_q a 2^32) <= tfmax (tf_q a 2^32 + 1) per feature, below 2^32 amax s_dot + s_dot
// < 2^62 + 2^30; its correction sum adds tf_c^2 round(-d 2^24) with -d = (idf_b - idf_q)(idf_b + idf_q) < ln 2 x
// 2 sqrt(amax) < 32, below 2^29 s_corr + s_corr < 2^54.  Both fit 64 bits.
static void classify_queries(const kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                             int64_t n_q, uint8_t *flag, int T) {
  const double amax = ix->jaccard ? 1.0 : std::pow(std::log((double)(ix->n_total + 2)) + 1.0, 2.0);
  parallel_for(n_q, n_q >= 2048 ? T : 1, [&](int, int64_t a, int64_t b) {
    for (int64_t q = a; q < b; q++) {
      bool known = false;
      int feats = 0;
      double s_dot = 0, s_corr = 0, wmax = 0;
      for (int64_t p = q_indptr[q]; p < q_indptr[q + 1]; p++) {
        const uint32_t t = q_ids[p];
        if ((int64_t)t >= ix->V) continue;
        if (ix->corpus_fit && ix->h_df[t] == 0) continue;  // in no live row: ignored like an out-of-vocabulary feature
        known = true;
        if (ix->h_univ[t]) {  // folded into the query's constants, but summed in fixed point like the other terms
          const double u = (double)ix->h_utf[t], f = (double)q_tf[p];
          s_dot += f * u;
          s_corr += u * u;
          continue;
        }
        feats++;
        const double tm = (double)ix->h_tfmax[t], f = (double)q_tf[p];
        s_dot += f * tm;
        s_corr += tm * tm;
        wmax = std::max(wmax, f);
      }
      flag[q] = 0;
      if (!known) flag[q] = 1;
      else if (feats > QFEATS || s_dot * amax >= 1073741824.0 || s_corr * 32.0 >= 1073741824.0 || wmax * amax > 60000.0)
        flag[q] = 2;
    }
  });
}

static bool csr_ok(const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf, int64_t n_q) {
  for (int64_t q = 0; q < n_q; q++)
    if (q_indptr[q + 1] < q_indptr[q] || (q_indptr[q + 1] > q_indptr[q] && (!q_ids || !q_tf))) return false;
  return true;
}

static int build_query_tables(kv_index *ix, int64_t n_q);

// An upload replaces the resident batch: the old batch and the range result are dropped, and the exclusions, label
// filter, distinct mode and irregular queries of the old batch go with it.
static void start_batch(kv_index *ix) {
  ix->batch_valid = ix->batch_selfjoin = false;
  drop_range(ix);
  ix->has_excl = ix->has_filter = ix->distinct = ix->merged_seeds = false;
  ix->qtags.on = false;
  ix->irr.clear();
}

// The new batch of n_q queries (n_null of them null) is resident: what the upload recorded, and the batch is valid.
static void end_batch(kv_index *ix, int64_t n_q, int64_t n_null, int64_t h2d_bytes, unsigned long long f2_out) {
  ix->batch_f2_outside = (int64_t)f2_out;
  ix->batch_q = n_q;
  ix->batch_tiles = (n_q + TILE_Q - 1) / TILE_Q;
  ix->batch_null = n_null;
  ix->batch_h2d_bytes = h2d_bytes;
  ix->batch_valid = true;
}

static int prepare_batch_runs(kv_index *ix, const QueryRun *runs, int n_runs) {
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_query_upload: index not finalized");
  int64_t n_q = 0, nnz = 0;
  std::vector<int64_t> qb((size_t)n_runs + 1, 0), nb((size_t)n_runs + 1, 0);
  bool have_order = true, have_flags = true, any_order = false;
  for (int r = 0; r < n_runs; r++) {
    const QueryRun &R = runs[r];
    if (R.n_q < 0 || !R.indptr || !csr_ok(R.indptr, R.ids, R.tf, R.n_q)) return kv_fail(KV_ERR_INVALID, "kv_query_upload: bad query CSR");
    n_q += R.n_q;
    nnz += R.indptr[R.n_q] - R.indptr[0];
    qb[(size_t)r + 1] = n_q;
    nb[(size_t)r + 1] = nnz;
    have_order = have_order && (R.order || R.n_q == 0);
    have_flags = have_flags && (R.flags || R.n_q == 0);
    any_order = any_order || (R.order && R.n_q > 0);
  }
  // a run with an order stores its rows sorted: without the orders of ALL runs the rows cannot be mapped back
  if (any_order && !have_order) return kv_fail(KV_ERR_INVALID, "kv_query_upload_runs: slice orders must be given for all runs or for none");
  if (n_q < 1) return kv_fail(KV_ERR_INVALID, "kv_query_upload: empty query batch");
  if (n_q >= (1LL << 31) - TILE_Q) return kv_fail(KV_ERR_INVALID, "kv_query_upload: too many queries in one call");
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  start_batch(ix);
  const int T = host_threads();
  const auto t_begin = std::chrono::steady_clock::now();
  auto ms_since = [](std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
  };

  // ---- host: pinned staging of the CSR (the runs back to back), classification, text order ----
  KV_CUDA(ix->h_qperm.ensure(3 * n_q));
  KV_CUDA(ix->h_flags.ensure(n_q));
  KV_CUDA(ix->h_q_indptr.ensure(n_q + 1));
  KV_CUDA(ix->h_q_ids.ensure(std::max<int64_t>(nnz, 1)));
  KV_CUDA(ix->h_q_tf.ensure(std::max<int64_t>(nnz, 1)));
  KV_CUDA(ix->h_q_oov.ensure(n_q));
  auto stage_run = [&](int r, int Tr) {
    const QueryRun &R = runs[r];
    const int64_t base = R.indptr[0], rn = R.indptr[R.n_q] - base, q0 = qb[(size_t)r], p0 = nb[(size_t)r];
    parallel_for(R.n_q, R.n_q >= 65536 ? Tr : 1, [&](int, int64_t a, int64_t b) {
      for (int64_t q = a; q < b; q++) {
        ix->h_q_indptr.p[q0 + q] = R.indptr[q] - base + p0;
        ix->h_q_oov.p[q0 + q] = R.oov ? R.oov[q] : 0.0;
      }
    });
    parallel_for(rn, rn >= (1 << 18) ? Tr : 1, [&](int, int64_t a, int64_t b) {
      if (b > a) {
        memcpy(ix->h_q_ids.p + p0 + a, R.ids + base + a, (size_t)(b - a) * 4);
        memcpy(ix->h_q_tf.p + p0 + a, R.tf + base + a, (size_t)(b - a) * 4);
      }
    });
  };
  if (n_runs == 1) stage_run(0, T);
  else
    parallel_for(n_runs, std::min(n_runs, T), [&](int, int64_t a, int64_t b) {
      for (int64_t r = a; r < b; r++) stage_run((int)r, std::max(1, T / n_runs));
    });
  ix->h_q_indptr.p[n_q] = nnz;
  const int64_t *q_indptr = ix->h_q_indptr.p;
  const uint32_t *q_ids = ix->h_q_ids.p, *q_tf = ix->h_q_tf.p;
  const double *q_oov = ix->h_q_oov.p;
  ix->last_prepare_ms[0] = ms_since(t_begin);
  auto t_mark = std::chrono::steady_clock::now();

  std::vector<uint8_t> flag((size_t)n_q, 0);
  if (have_flags) {
    for (int r = 0; r < n_runs; r++)
      if (runs[r].n_q) memcpy(flag.data() + qb[(size_t)r], runs[r].flags, (size_t)runs[r].n_q);
  } else {
    classify_queries(ix, q_indptr, q_ids, q_tf, n_q, flag.data(), T);
  }
  ix->last_prepare_ms[1] = ms_since(t_mark);
  t_mark = std::chrono::steady_clock::now();
  // queries with similar text share a scan group and a bound tile (their candidates are largely the same chunks)
  std::vector<int> order((size_t)n_q);
  auto less_text = [&](int a, int b) {
    return cmp_seq(q_ids + q_indptr[a], q_indptr[a + 1] - q_indptr[a], q_ids + q_indptr[b], q_indptr[b + 1] - q_indptr[b]) < 0;
  };
  std::vector<int> orig;  // row -> original query (sorted slices only; identity otherwise)
  for (int64_t q = 0; q < n_q; q++) order[(size_t)q] = (int)q;
  if (have_order) {
    // the runs arrive sorted (row p of a run is its p-th smallest query): merge them.  A run's queries precede the next
    // run's and equal queries keep their original order inside a run, so the stable merge == the full stable sort.
    orig.resize((size_t)n_q);
    std::vector<uint8_t> seen((size_t)n_q, 0);
    for (int r = 0; r < n_runs; r++)
      for (int64_t i = 0; i < runs[r].n_q; i++) {
        const int32_t o = runs[r].order[i];
        if (o < 0 || o >= runs[r].n_q || seen[(size_t)(qb[(size_t)r] + o)]++)
          return kv_fail(KV_ERR_INVALID, "kv_query_upload_runs: a slice order is not a permutation");
        orig[(size_t)(qb[(size_t)r] + i)] = (int)(qb[(size_t)r] + o);
      }
    std::atomic<int> unsorted{0};
    parallel_for(n_q - 1, n_q >= 8192 ? T : 1, [&](int, int64_t a, int64_t b) {
      for (int64_t i = a; i < b; i++) {
        const int x = (int)i, y = x + 1;
        if (std::upper_bound(qb.begin(), qb.end(), (int64_t)x) != std::upper_bound(qb.begin(), qb.end(), (int64_t)y)) continue;  // run boundary
        const int c = cmp_seq(q_ids + q_indptr[x], q_indptr[x + 1] - q_indptr[x], q_ids + q_indptr[y], q_indptr[y + 1] - q_indptr[y]);
        if (c > 0 || (c == 0 && orig[(size_t)y] < orig[(size_t)x])) unsorted.store(1);
      }
    });
    if (unsorted.load()) return kv_fail(KV_ERR_INVALID, "kv_query_upload_runs: a slice is not stored in text order");
    if (n_runs > 1) merge_sorted_runs(order, qb, less_text, T);
  } else {
    stable_sort_indices(order, less_text, T);  // == std::stable_sort, on all host threads
  }
  ix->last_prepare_ms[2] = ms_since(t_mark);
  t_mark = std::chrono::steady_clock::now();
  int *qperm = ix->h_qperm.p, *null_list = qperm + n_q, *qsrc = qperm + 2 * n_q;
  int64_t n_null = 0;
  for (int64_t i = 0; i < n_q; i++) {
    const int64_t row = order[(size_t)i], q = have_order ? orig[(size_t)row] : row;
    qperm[i] = (int)q;
    qsrc[i] = (int)row;
    ix->h_flags.p[i] = flag[(size_t)row];
    if (flag[(size_t)row] == 1) {
      null_list[n_null++] = (int)q;
    } else if (flag[(size_t)row] == 2) {
      const int64_t a = q_indptr[row];
      ix->irr.add(q, q_ids + a, q_tf + a, q_indptr[row + 1] - a, q_oov[row]);
    }
  }

  KV_CUDA(ix->d_q_indptr.ensure(n_q + 1));
  KV_CUDA(ix->d_q_ids.ensure(std::max<int64_t>(nnz, 1)));
  KV_CUDA(ix->d_q_tf.ensure(std::max<int64_t>(nnz, 1)));
  KV_CUDA(ix->d_q_oov.ensure(n_q));
  KV_CUDA(ix->d_qperm.ensure(3 * n_q));
  KV_CUDA(ix->d_flags.ensure(n_q));
  KV_CUDA(cudaEventRecord(ix->ev[0], s));
  KV_CUDA(cudaMemcpyAsync(ix->d_q_indptr.p, ix->h_q_indptr.p, (size_t)(n_q + 1) * 8, cudaMemcpyHostToDevice, s));
  if (nnz) {
    KV_CUDA(cudaMemcpyAsync(ix->d_q_ids.p, ix->h_q_ids.p, (size_t)nnz * 4, cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaMemcpyAsync(ix->d_q_tf.p, ix->h_q_tf.p, (size_t)nnz * 4, cudaMemcpyHostToDevice, s));
  }
  KV_CUDA(cudaMemcpyAsync(ix->d_q_oov.p, ix->h_q_oov.p, (size_t)n_q * 8, cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemcpyAsync(ix->d_qperm.p, ix->h_qperm.p, (size_t)3 * n_q * sizeof(int), cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemcpyAsync(ix->d_flags.p, ix->h_flags.p, (size_t)n_q, cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaEventRecord(ix->ev[1], s));
  {
    const int rc = build_query_tables(ix, n_q);
    if (rc != KV_OK) return rc;
  }
  unsigned long long f2_out = 0;
  KV_CUDA(cudaMemcpyAsync(&f2_out, ix->d_f2out.p, sizeof(f2_out), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));  // the pinned staging buffers may be rewritten by the next call
  end_batch(ix, n_q, n_null, (n_q + 1) * 8 + nnz * 8 + n_q * 8 + 3 * n_q * (int64_t)sizeof(int) + n_q, f2_out);
  cudaEventElapsedTime(&ix->last_ms[0], ix->ev[0], ix->ev[1]);
  ix->last_prepare_ms[3] = ms_since(t_mark);
  return KV_OK;
}

// The device half of an upload, shared by the host and the text path: with the query CSR (by row), d_qperm (qsrc) and
// d_flags (by sorted slot) on the device, the per-query constants and tables and the per-tile rare-feature tables.
static int build_query_tables(kv_index *ix, int64_t n_q) {
  cudaStream_t s = ix->stream;
  const int64_t n_tiles = (n_q + TILE_Q - 1) / TILE_Q, n_q_pad = n_tiles * TILE_Q;
  KV_CUDA(ix->d_qconst.ensure(7 * n_q));
  KV_CUDA(ix->d_qfix.ensure(2 * n_q));
  KV_CUDA(ix->d_qtab.ensure(n_q * (int64_t)QTAB_BYTES));
  KV_CUDA(ix->d_Wf.ensure(n_q_pad * NF));
  KV_CUDA(ix->d_q2list.ensure(n_q_pad * Q2CAP));
  KV_CUDA(ix->d_q3id.ensure(n_q_pad * Q3CAP));
  KV_CUDA(ix->d_q3w.ensure(n_q_pad * Q3CAP));
  KV_CUDA(ix->d_Wf2.ensure(n_q_pad * KT2));
  KV_CUDA(ix->d_d2col.ensure(n_tiles * KT2));
  KV_CUDA(ix->d_f2out.ensure(1));
  // ---- device: per-query constants and tables, per-tile rare-feature tables ----
  KV_CUDA(cudaMemsetAsync(ix->d_Wf.p, 0, (size_t)n_q_pad * NF * sizeof(__half), s));
  KV_CUDA(cudaMemsetAsync(ix->d_Wf2.p, 0, (size_t)n_q_pad * KT2 * sizeof(__half), s));
  KV_CUDA(cudaMemsetAsync(ix->d_f2out.p, 0, sizeof(unsigned long long), s));
  // the lists of the padding queries of the last tile must be empty (weight 0 / no feature)
  KV_CUDA(cudaMemsetAsync(ix->d_q2list.p, 0, (size_t)n_q_pad * Q2CAP * sizeof(uint2), s));
  KV_CUDA(cudaMemsetAsync(ix->d_q3id.p, 0xFF, (size_t)n_q_pad * Q3CAP * sizeof(uint32_t), s));
  KV_CUDA(cudaMemsetAsync(ix->d_q3w.p, 0, (size_t)n_q_pad * Q3CAP * sizeof(uint32_t), s));
  PrepParams P;
  P.q_indptr = ix->d_q_indptr.p; P.q_ids = ix->d_q_ids.p; P.q_tf = ix->d_q_tf.p; P.q_oov = ix->d_q_oov.p;
  P.qsrc = ix->d_qperm.p + 2 * n_q; P.flags = ix->d_flags.p;
  P.n_q = n_q; P.V = ix->V; P.n_total = ix->n_total;
  P.a64 = ix->d_a64.p; P.d64 = ix->d_d64.p; P.univ = ix->d_univ.p; P.utf = ix->d_utf.p; P.tfmax = ix->d_tfmax.p;
  P.fslot = ix->d_fslot.p; P.fslot2 = ix->d_fslot2.p; P.q2list = ix->d_q2list.p; P.jaccard = ix->jaccard; P.corpus_fit = ix->corpus_fit;
  P.q_nq = ix->d_qconst.p; P.q_dotU = P.q_nq + n_q; P.q_corrU = P.q_nq + 2 * n_q; P.q_dotS = P.q_nq + 3 * n_q;
  P.q_corrS = P.q_nq + 4 * n_q; P.q_dotX = P.q_nq + 5 * n_q; P.q_rscale = P.q_nq + 6 * n_q;
  P.q_uw = ix->d_qfix.p; P.q_uc = ix->d_qfix.p + n_q;
  P.qtab = ix->d_qtab.p; P.Wf = ix->d_Wf.p; P.q3id = ix->d_q3id.p; P.q3w = ix->d_q3w.p;
  prep_queries_kernel<<<(unsigned)((n_q + 127) / 128), 128, 0, s>>>(P);
  KV_CUDA(cudaGetLastError());
  DictParams DP;
  DP.q2list = ix->d_q2list.p; DP.Wf2 = ix->d_Wf2.p; DP.d2col = ix->d_d2col.p; DP.n_outside = ix->d_f2out.p;
  f2_dict_kernel<<<(unsigned)n_tiles, DICT_THREADS, 0, s>>>(DP);
  KV_CUDA(cudaGetLastError());
  {
    int rc = make_map_2d(&ix->map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ix->d_Wf.p, n_q_pad, NF, TILE_Q);
    if (rc == KV_OK) rc = make_map_2d(&ix->map_w2, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ix->d_Wf2.p, n_q_pad, KT2, TILE_Q);
    if (rc != KV_OK) return rc;
  }
  return KV_OK;
}

static int prepare_batch(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                         const double *q_oov, int64_t n_q) {
  QueryRun R;
  R.indptr = q_indptr; R.ids = q_ids; R.tf = q_tf; R.oov = q_oov; R.n_q = n_q;
  return prepare_batch_runs(ix, &R, 1);
}

// ---- the upload of a text batch featurised on the device (kv_query_upload_text) ----
namespace {

constexpr int TQ_THREADS = 256;

inline unsigned tq_grid(int64_t n) { return (unsigned)std::max<int64_t>(1, (n + TQ_THREADS - 1) / TQ_THREADS); }

// classify_queries on the device, one thread per query, the same float64 operations in the same order (no contraction)
__global__ void __launch_bounds__(TQ_THREADS) classify_kernel(const int64_t *indptr, const uint32_t *ids, const uint32_t *tf,
                                                              int64_t n_q, int64_t V, int corpus_fit, const uint32_t *df,
                                                              const uint8_t *univ, const uint32_t *utf, const uint32_t *tfmax,
                                                              double amax, uint8_t *flag) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_q) return;
  bool known = false;
  int feats = 0;
  double s_dot = 0, s_corr = 0, wmax = 0;
  for (int64_t p = indptr[q]; p < indptr[q + 1]; p++) {
    const uint32_t t = ids[p];
    if ((int64_t)t >= V) continue;
    if (corpus_fit && df[t] == 0) continue;
    known = true;
    if (univ[t]) {
      const double u = (double)utf[t], f = (double)tf[p];
      s_dot = __dadd_rn(s_dot, __dmul_rn(f, u));
      s_corr = __dadd_rn(s_corr, __dmul_rn(u, u));
      continue;
    }
    feats++;
    const double tm = (double)tfmax[t], f = (double)tf[p];
    s_dot = __dadd_rn(s_dot, __dmul_rn(f, tm));
    s_corr = __dadd_rn(s_corr, __dmul_rn(tm, tm));
    wmax = fmax(wmax, f);
  }
  uint8_t c = 0;
  if (!known) c = 1;
  else if (feats > QFEATS || __dmul_rn(s_dot, amax) >= 1073741824.0 || __dmul_rn(s_corr, 32.0) >= 1073741824.0 ||
           __dmul_rn(wmax, amax) > 60000.0)
    c = 2;
  flag[q] = c;
}

// cmp_seq of queries a and b of the device CSR
__device__ __forceinline__ int cmp_queries(const int64_t *indptr, const uint32_t *ids, int a, int b) {
  const int64_t a0 = indptr[a], na = indptr[a + 1] - a0, b0 = indptr[b], nb = indptr[b + 1] - b0;
  const int64_t n = na < nb ? na : nb;
  for (int64_t i = 0; i < n; i++) {
    const uint32_t x = ids[a0 + i], y = ids[b0 + i];
    if (x != y) return x < y ? -1 : 1;
  }
  return na < nb ? -1 : (na > nb ? 1 : 0);
}

__global__ void __launch_bounds__(TQ_THREADS) iota_kernel(int *order, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) order[i] = (int)i;
}

// One pass of a stable bottom-up merge sort: the sorted runs [lo, lo + w) and [lo + w, lo + 2w) of `in` merge into
// `out`.  Every element finds its place by a binary search in the other run: an element of the left run goes after the
// right run's strictly smaller elements, one of the right run after the left run's smaller-or-equal elements, so equal
// sequences keep their input order (== std::stable_sort with cmp_seq).
__global__ void __launch_bounds__(TQ_THREADS) merge_pass_kernel(const int *in, int *out, int64_t n, int64_t w,
                                                                const int64_t *indptr, const uint32_t *ids) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t lo = i / (2 * w) * (2 * w), mid = min(lo + w, n), hi = min(lo + 2 * w, n);
  const int x = in[i];
  const bool left = i < mid;
  int64_t a = left ? mid : lo, b = left ? hi : mid;  // search [a, b) for the first element placed after x
  while (a < b) {
    const int64_t m = (a + b) >> 1;
    const int c = cmp_queries(indptr, ids, in[m], x);
    if (left ? c < 0 : c <= 0) a = m + 1;
    else b = m;
  }
  out[left ? i + (a - mid) : (i - mid) + a] = x;
}

// qperm / qsrc (the CSR rows are the original queries) and the flags by sorted slot
__global__ void __launch_bounds__(TQ_THREADS) slot_order_kernel(const int *order, const uint8_t *flag_row, int64_t n,
                                                                int *qperm, uint8_t *flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int row = order[i];
  qperm[i] = row;
  qperm[2 * n + i] = row;
  flags[i] = flag_row[row];
}

}  // namespace

static int prepare_batch_text(kv_index *ix, kv_vocab_mirror *m, const kv_vocab *v, const char *bytes,
                              const int64_t *offsets, int64_t n_q, int mode, int64_t *bad_doc) {
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_query_upload_text: index not finalized");
  if (n_q < 1) return kv_fail(KV_ERR_INVALID, "kv_query_upload_text: empty query batch");
  if (n_q >= (1LL << 31) - TILE_Q) return kv_fail(KV_ERR_INVALID, "kv_query_upload_text: too many queries in one call");
  if (mirror_device(m) != ix->device)
    return kv_fail(KV_ERR_INVALID, "kv_query_upload_text: the vocabulary mirror is on device %d, the index on device %d",
                   mirror_device(m), ix->device);
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  start_batch(ix);
  const auto t_begin = std::chrono::steady_clock::now();

  // ---- the text goes up and is featurised into the query CSR (by row) ----
  int64_t nnz = 0;
  {
    mirror_lock(m);
    int rc = mirror_sync_locked(m, v);
    if (rc == KV_OK) rc = featurize_device(m, s, bytes, offsets, n_q, mode, ix->d_q_indptr, ix->d_q_ids, ix->d_q_tf,
                                           ix->d_q_oov, &nnz, bad_doc);
    if (rc == KV_OK && cudaStreamSynchronize(s) != cudaSuccess)  // the mirror's scratch is read until here
      rc = kv_fail(KV_ERR_CUDA, "kv_query_upload_text: featurisation failed: %s", cudaGetErrorString(cudaGetLastError()));
    mirror_unlock(m);
    if (rc != KV_OK) return rc;
  }
  ix->last_prepare_ms[0] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_begin).count();

  // ---- classification and text order on the device ----
  KV_CUDA(ix->d_qflag_row.ensure(n_q));
  KV_CUDA(ix->d_qorder.ensure(2 * n_q));
  KV_CUDA(ix->d_qperm.ensure(3 * n_q));
  KV_CUDA(ix->d_flags.ensure(n_q));
  KV_CUDA(ix->h_qperm.ensure(3 * n_q));
  KV_CUDA(ix->h_flags.ensure(n_q));
  const double amax = ix->jaccard ? 1.0 : std::pow(std::log((double)(ix->n_total + 2)) + 1.0, 2.0);
  KV_CUDA(cudaEventRecord(ix->evq[0], s));
  classify_kernel<<<tq_grid(n_q), TQ_THREADS, 0, s>>>(ix->d_q_indptr.p, ix->d_q_ids.p, ix->d_q_tf.p, n_q, ix->V, ix->corpus_fit,
                                                     ix->d_df.p, ix->d_univ.p, ix->d_utf.p, ix->d_tfmax.p, amax, ix->d_qflag_row.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaEventRecord(ix->evq[1], s));
  int *cur = ix->d_qorder.p, *other = cur + n_q;
  iota_kernel<<<tq_grid(n_q), TQ_THREADS, 0, s>>>(cur, n_q);
  for (int64_t w = 1; w < n_q; w *= 2) {
    merge_pass_kernel<<<tq_grid(n_q), TQ_THREADS, 0, s>>>(cur, other, n_q, w, ix->d_q_indptr.p, ix->d_q_ids.p);
    std::swap(cur, other);
  }
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaEventRecord(ix->evq[2], s));
  slot_order_kernel<<<tq_grid(n_q), TQ_THREADS, 0, s>>>(cur, ix->d_qflag_row.p, n_q, ix->d_qperm.p, ix->d_flags.p);
  KV_CUDA(cudaGetLastError());
  {
    const int rc = build_query_tables(ix, n_q);
    if (rc != KV_OK) return rc;
  }
  // ---- back to the host: the order and flags (filters, exclusions and the test hooks read them), the null list ----
  unsigned long long f2_out = 0;
  KV_CUDA(cudaMemcpyAsync(ix->h_qperm.p, ix->d_qperm.p, (size_t)n_q * sizeof(int), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaMemcpyAsync(ix->h_flags.p, ix->d_flags.p, (size_t)n_q, cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaMemcpyAsync(&f2_out, ix->d_f2out.p, sizeof(f2_out), cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaEventRecord(ix->evq[3], s));
  KV_CUDA(cudaStreamSynchronize(s));
  int *qperm = ix->h_qperm.p, *null_list = qperm + n_q, *qsrc = qperm + 2 * n_q;
  int64_t n_null = 0, n_irr = 0;
  for (int64_t i = 0; i < n_q; i++) {
    qsrc[i] = qperm[i];
    if (ix->h_flags.p[i] == 1) null_list[n_null++] = qperm[i];
    else if (ix->h_flags.p[i] == 2) n_irr++;
  }
  if (n_null) KV_CUDA(cudaMemcpyAsync(ix->d_qperm.p + n_q, null_list, (size_t)n_null * sizeof(int), cudaMemcpyHostToDevice, s));
  // the irregular queries' CSR, for the float64 fallback (rare: one copy per query)
  if (n_irr) {
    KV_CUDA(ix->h_q_indptr.ensure(n_q + 1));
    KV_CUDA(ix->h_q_oov.ensure(n_q));
    KV_CUDA(cudaMemcpyAsync(ix->h_q_indptr.p, ix->d_q_indptr.p, (size_t)(n_q + 1) * 8, cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaMemcpyAsync(ix->h_q_oov.p, ix->d_q_oov.p, (size_t)n_q * 8, cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaStreamSynchronize(s));
    std::vector<uint32_t> ids, tf;
    for (int64_t i = 0; i < n_q; i++) {
      if (ix->h_flags.p[i] != 2) continue;
      const int64_t q = qperm[i], a = ix->h_q_indptr.p[q], nnz_q = ix->h_q_indptr.p[q + 1] - a;
      ids.resize((size_t)nnz_q);
      tf.resize((size_t)nnz_q);
      if (nnz_q) {
        KV_CUDA(cudaMemcpyAsync(ids.data(), ix->d_q_ids.p + a, (size_t)nnz_q * 4, cudaMemcpyDeviceToHost, s));
        KV_CUDA(cudaMemcpyAsync(tf.data(), ix->d_q_tf.p + a, (size_t)nnz_q * 4, cudaMemcpyDeviceToHost, s));
        KV_CUDA(cudaStreamSynchronize(s));
      }
      ix->irr.add(q, ids.data(), tf.data(), nnz_q, ix->h_q_oov.p[q]);
    }
  }
  KV_CUDA(cudaStreamSynchronize(s));
  end_batch(ix, n_q, n_null, (offsets[n_q] - offsets[0]) + (n_q + 1) * 8 + n_null * (int64_t)sizeof(int), f2_out);
  cudaEventElapsedTime(&ix->last_prepare_ms[1], ix->evq[0], ix->evq[1]);
  cudaEventElapsedTime(&ix->last_prepare_ms[2], ix->evq[1], ix->evq[2]);
  cudaEventElapsedTime(&ix->last_prepare_ms[3], ix->evq[2], ix->evq[3]);
  ix->last_ms[0] = 0;  // no CSR crossed the bus
  return KV_OK;
}

// Device-only half: bounds + scans + merge (+ fallback scans for irregular queries) of the uploaded batch.
// phase 0: the whole batch.  phase 1: up to the seed scan; the outputs receive the seed top-k (their k-th score is a
// lower bound of the final k-th score; a row-sharded GFKB exchanges it between the GPUs).  phase 2: the rest.
// Three device paths: pruned (bound pass 0 -> seed scan -> candidate selection -> scan of the candidates), exhaustive
// (small indexes, KAKVEDA_B200_NO_PRUNE=1: every chunk is a candidate of every query) and Jaccard (K3).
// A threshold search (kv_range_resident, range = true, k = 0) runs the second phase of the pruned path -- bound pass 1
// on the fixed threshold, then the scan -- or the exhaustive scan, with K1b-R as the scan.
struct Batch {
  int k, phase;
  float *out_s;  // the outputs, [n_q][k] by original query
  long long *out_r;
  int64_t n_q, n_tiles, n_groups, n_bsplits, n_ssplits, n_ssplits_a, n_csplits, n_parts;
  int max_pages, n_seed, n_peers;
  bool prune, use_codes, range = false;
  bool distinct = false;  // kv_query_set_distinct: the scans keep one row per group, K5 skips taken groups
  int64_t launches = 0;
};

// K5: the first n_lists partial lists of the batch, per query -> the outputs, by original query
static int launch_merge(kv_index *ix, const Batch &b, int64_t n_lists) {
  if (b.distinct)
    merge_topk_distinct_kernel<<<(unsigned)((b.n_q * 32 + 255) / 256), 256, 0, ix->stream>>>(
        ix->d_part_s.p, ix->d_part_r.p, (int)n_lists, b.n_q, b.k, b.n_q * b.k, b.n_q * b.k, ix->d_qperm.p, ix->groups.d_row.p,
        ix->row_base, ix->n_rows, nullptr, b.out_s, b.out_r);
  else
    merge_topk_kernel<<<(unsigned)((b.n_q * 32 + 255) / 256), 256, 0, ix->stream>>>(
        ix->d_part_s.p, ix->d_part_r.p, (int)n_lists, b.n_q, b.k, b.n_q * b.k, b.n_q * b.k, ix->d_qperm.p, b.out_s, b.out_r);
  KV_CUDA(cudaGetLastError());
  return KV_OK;
}

// K1b-S parameters shared by every scan of the batch (the caller sets the candidate lists and the splits)
static ScanParams scan_params(const kv_index *ix, const Batch &b) {
  const float *qc = ix->d_qconst.p;
  ScanParams SP{};
  SP.blk = ix->d_blk.p; SP.binfo = ix->d_binfo.p; SP.B32 = ix->d_B32.p; SP.perm = ix->d_perm.p;
  SP.n_chunks = ix->n_chunks; SP.n_rows = ix->n_rows; SP.row_base = ix->row_base;
  SP.ovf_keys = ix->d_ovf_keys.p; SP.ovf_vals = ix->d_ovf_vals.p; SP.n_ovf = ix->n_ovf;
  SP.qtab = ix->d_qtab.p; SP.q_nq = qc; SP.q_uw = ix->d_qfix.p; SP.q_uc = ix->d_qfix.p + b.n_q;
  SP.q_excl = ix->has_excl ? ix->d_excl_sorted.p : nullptr; SP.gthr = b.range ? ix->d_rthr.p : ix->d_gthr.p;
  if (ix->has_filter) { SP.q_label = ix->d_filt_sorted.p; SP.label_pos = ix->labels.d_pos.p; SP.chunk_sig = ix->d_chunk_sig.p; }
  SP.alive = alive_words(ix);
  for (int i = 0; i < 7; i++) SP.peer_gthr[i] = i < b.n_peers ? ix->peer_gthr[i] : nullptr;
  SP.n_peers = b.n_peers; SP.stats = ix->d_stats.p; SP.n_q = b.n_q; SP.k = b.k;
  SP.part_scores = ix->d_part_s.p; SP.part_rows = ix->d_part_r.p; SP.max_pages = b.max_pages;
  SP.qperm = ix->d_qperm.p; SP.range_out = ix->range.pairs.p; SP.range_count = ix->range.d_count.p;
  SP.range_cap = ix->range.capacity();
  SP.group_pos = b.distinct ? ix->groups.d_pos.p : nullptr;
  if (ix->qtags.on) {
    const RowTags &T = ix->tags;
    SP.q_tmask = ix->qtags.d_mask_sorted.p; SP.q_tags = ix->qtags.d_tags_sorted.p;
    SP.tag_mask_pos = T.d_mask_pos.p; SP.chunk_tsig = T.d_chunk_sig.p;
    SP.tag_ptr = T.masks_exact ? nullptr : T.d_ptr_pos.p; SP.tag_list = T.masks_exact ? nullptr : T.d_list_pos.p;
  }
  return SP;
}

// K1b-S (distinct or not), or K1b-R for a threshold search, over a grid of candidate lists; the tag-filtered
// instantiations when the batch has a tag filter
static int launch_scan(kv_index *ix, const Batch &b, const ScanParams &SP, dim3 grid) {
  if (ix->qtags.on) {
    if (b.range) tfidf_scan_kernel<true, false, true><<<grid, S_WARPS * 32, scan_smem_bytes(0, false, true), ix->stream>>>(SP);
    else if (b.distinct) tfidf_scan_kernel<false, true, true><<<grid, S_WARPS * 32, scan_smem_bytes(b.k, true, true), ix->stream>>>(SP);
    else tfidf_scan_kernel<false, false, true><<<grid, S_WARPS * 32, scan_smem_bytes(b.k, false, true), ix->stream>>>(SP);
  } else if (b.range) tfidf_scan_kernel<true, false><<<grid, S_WARPS * 32, scan_smem_bytes(0), ix->stream>>>(SP);
  else if (b.distinct) tfidf_scan_kernel<false, true><<<grid, S_WARPS * 32, scan_smem_bytes(b.k, true), ix->stream>>>(SP);
  else tfidf_scan_kernel<false, false><<<grid, S_WARPS * 32, scan_smem_bytes(b.k), ix->stream>>>(SP);
  KV_CUDA(cudaGetLastError());
  return KV_OK;
}

// The scan of the candidates: of the lists bound pass 1 built, or, when the bound codes were kept, of the chunks whose
// codes reach the threshold codes (selected in the scan kernel, n_csplits CTAs per group)
static int scan_candidates(kv_index *ix, Batch &b) {
  ScanParams SP = scan_params(ix, b);
  b.launches++;
  if (b.use_codes) {
    SP.list_mode = 3; SP.ubq = ix->d_ubq.p; SP.ubq_stride = ix->n_chunks_pad; SP.tcode = ix->d_tcode.p;
    SP.n_bsplits = 1; SP.n_ssplits = (int)b.n_csplits;
    return launch_scan(ix, b, SP, dim3((unsigned)b.n_groups, (unsigned)b.n_csplits));
  }
  SP.list_mode = 0; SP.list_count = ix->d_list_count.p + b.n_groups; SP.list_pages = ix->d_list_pages.p; SP.pool = ix->d_pool.p;
  SP.n_bsplits = (int)b.n_bsplits; SP.n_ssplits = (int)b.n_ssplits;
  return launch_scan(ix, b, SP, dim3((unsigned)(b.n_groups * b.n_bsplits), (unsigned)b.n_ssplits));
}

// Pruned path.  Phase 0 / 1: bound pass 0 (seeds and bound codes) -> seed scan; phase 1 ends with the seed top-k.
// Phase 0 / 2: the scan of the candidates into b.n_parts partial lists -- selected from the stored codes by the scan
// itself when they were kept (after a snapshot of the threshold codes), else listed by recomputing the bounds (pass 1).
static int run_pruned(kv_index *ix, Batch &b) {
  cudaStream_t s = ix->stream;
  const float *qc = ix->d_qconst.p; const int64_t n_q = b.n_q;
  if (b.phase != 2) KV_CUDA(cudaMemsetAsync(ix->d_pool_ctl.p, 0, 2 * sizeof(unsigned int), s));
  BoundParams BP;
  BP.blk = ix->d_blk.p; BP.binfo = ix->d_binfo.p; BP.chunk_minB = ix->d_cminB.p;
  BP.ovf_keys = ix->d_ovf_keys.p; BP.ovf_vals = ix->d_ovf_vals.p; BP.n_ovf = ix->n_ovf;
  BP.n_chunks = ix->n_chunks; BP.n_q = n_q; BP.q3id = ix->d_q3id.p; BP.q3w = ix->d_q3w.p; BP.d2col = ix->d_d2col.p; BP.q2list = ix->d_q2list.p; BP.ubt = ix->d_ubt.p;
  BP.rbloom = ix->d_rbloom.p; BP.rt_slots = ix->d_rt_slots.p; BP.rt_off = ix->d_rt_off.p; BP.rt_size = ix->d_rt_size.p;
  BP.q_nq = qc; BP.q_dotS = qc + 3 * n_q; BP.q_corrS = qc + 4 * n_q; BP.q_dotX = qc + 5 * n_q; BP.q_rscale = qc + 6 * n_q;
  BP.gthr = b.range ? ix->d_rthr.p : ix->d_gthr.p; BP.n_bsplits = (int)b.n_bsplits; BP.seeds = ix->d_seeds.p;
  BP.lists.count = ix->d_list_count.p + b.n_groups; BP.lists.pages = ix->d_list_pages.p; BP.lists.max_pages = b.max_pages;
  BP.lists.pool = ix->d_pool.p; BP.lists.pool_next = ix->d_pool_ctl.p; BP.lists.pool_pages = (unsigned int)ix->pool_pages;
  BP.lists.overflow = (int *)(ix->d_pool_ctl.p + 1); BP.stats = ix->d_stats.p;
  BP.dbg_xs = ix->dbg_xs; BP.dbg_stride = ix->n_chunks_pad; BP.ubq = b.use_codes ? ix->d_ubq.p : nullptr; BP.ubq_stride = ix->n_chunks_pad;
  const size_t b_smem = bound_smem_bytes(b.max_pages);
  const dim3 bgrid((unsigned)b.n_tiles, (unsigned)b.n_bsplits);
  ScanParams SP = scan_params(ix, b);
  if (b.phase != 2) {
    // pass 0: seeds
    KV_CUDA(cudaEventRecord(ix->evk[0], s));
    BP.pass = 0;
    // the headline configuration (bound codes kept, no test hook) runs the specialised instantiation
    if (BP.ubq && !BP.dbg_xs && !getenv("KAKVEDA_B200_GENERIC_BOUND"))
      tfidf_bound_kernel<true><<<bgrid, B_THREADS, b_smem, s>>>(ix->map_w, ix->map_w2, ix->map_u, BP);
    else
      tfidf_bound_kernel<false><<<bgrid, B_THREADS, b_smem, s>>>(ix->map_w, ix->map_w2, ix->map_u, BP);
    KV_CUDA(cudaGetLastError());
    seeds_to_lists_kernel<<<(unsigned)((b.n_groups * GROUP_Q * b.n_seed + 255) / 256), 256, 0, s>>>(
        ix->d_seeds.p, n_q, b.n_seed, ix->d_direct.p, ix->d_list_count.p);
    KV_CUDA(cudaGetLastError());
    KV_CUDA(cudaEventRecord(ix->evk[1], s));
    // seed scan: gives every query a lower bound of its k-th score
    SP.list_mode = 1; SP.list_count = ix->d_list_count.p; SP.direct = ix->d_direct.p; SP.direct_stride = GROUP_Q * b.n_seed;
    SP.n_bsplits = 1; SP.n_ssplits = (int)b.n_ssplits_a;
    const int rc = launch_scan(ix, b, SP, dim3((unsigned)b.n_groups, (unsigned)b.n_ssplits_a));
    if (rc != KV_OK) return rc;
    KV_CUDA(cudaEventRecord(ix->evk[2], s));
    b.launches += 3;
    if (b.phase == 1) {  // the seed top-k of this shard, by original query
      b.launches++;
      return launch_merge(ix, b, b.n_ssplits_a);
    }
  }
  if (b.phase == 2) KV_CUDA(cudaEventRecord(ix->evp2, s));  // the caller's threshold exchange sits between evk[2] and this point
  if (b.use_codes) {
    threshold_codes_kernel<<<(unsigned)((n_q + 255) / 256), 256, 0, s>>>(qc, ix->d_gthr.p, n_q, ix->d_tcode.p);
  } else {
    BP.pass = 1;
    tfidf_bound_kernel<false><<<bgrid, B_THREADS, b_smem, s>>>(ix->map_w, ix->map_w2, ix->map_u, BP);
  }
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaEventRecord(ix->evk[3], s));
  b.launches++;
  return scan_candidates(ix, b);
}

// Exhaustive path: every chunk of a list's chunk range x every query of the group
static int run_exhaustive(kv_index *ix, Batch &b) {
  ScanParams SP = scan_params(ix, b);
  SP.list_mode = 2; SP.n_bsplits = (int)b.n_bsplits; SP.n_ssplits = (int)b.n_ssplits;
  b.launches++;
  return launch_scan(ix, b, SP, dim3((unsigned)(b.n_groups * b.n_bsplits), (unsigned)b.n_ssplits));
}

// Jaccard path: token sets have no text structure to prune on -- the dense-regime kernel K3 scores every chunk for a
// whole scan group at once.  A threshold search runs K3-R, which appends to ix->jrange instead of filling lists.
static int run_jaccard(kv_index *ix, Batch &b) {
  const int64_t n_q = b.n_q, n_groups = b.n_groups;
  const int64_t jsplits = std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>((4LL * ix->sm_count + n_groups - 1) / n_groups, 256),
                                                                 std::max<int64_t>(1, ix->n_chunks / 64)));
  b.n_parts = jsplits * J_WARPS;
  if (!b.range) {
    KV_CUDA(ix->d_part_s.ensure(b.n_parts * n_q * b.k));
    KV_CUDA(ix->d_part_r.ensure(b.n_parts * n_q * b.k));
  }
  const float *qc = ix->d_qconst.p;
  JaccardParams JP;
  JP.blk = ix->d_blk.p; JP.binfo = ix->d_binfo.p; JP.B32 = ix->d_B32.p; JP.perm = ix->d_perm.p;
  JP.n_chunks = ix->n_chunks; JP.n_rows = ix->n_rows; JP.row_base = ix->row_base;
  JP.qtab = ix->d_qtab.p; JP.q_nq = qc; JP.q_dotU = qc + n_q; JP.q_excl = ix->has_excl ? ix->d_excl_sorted.p : nullptr;
  JP.gthr = b.range ? ix->d_rthr.p : ix->d_gthr.p; JP.stats = ix->d_stats.p;
  JP.n_q = n_q; JP.k = b.k; JP.n_splits = (int)jsplits; JP.part_scores = ix->d_part_s.p; JP.part_rows = ix->d_part_r.p;
  const dim3 grid((unsigned)n_groups, (unsigned)jsplits);
  if (b.range) {
    const JaccardRangeOut R{ix->d_qperm.p, ix->jrange.pairs.p, ix->jrange.d_count.p, ix->jrange.capacity()};
    jaccard_scan_kernel<true><<<grid, J_WARPS * 32, jaccard_smem_bytes(0), ix->stream>>>(JP, R);
  } else {
    jaccard_scan_kernel<false><<<grid, J_WARPS * 32, jaccard_smem_bytes(b.k), ix->stream>>>(JP, JaccardRangeOut{});
  }
  KV_CUDA(cudaGetLastError());
  b.launches++;
  return KV_OK;
}

// Scan of the stored codes: aim for this many CTAs per SM (32 waves at 2 CTAs/SM).  At the bench shape that is 3 CTAs
// per group; 5 and 8 were measured slower (DESIGN section 6): every CTA of a group starts with empty lists.
constexpr int64_t CODE_SPLIT_CTAS = 64;

// Splits of the resident batch, pruned or exhaustive path, and the buffers of the candidate lists: sets b's sizes,
// b.prune and the last_* launch counts.  Shared by the top-k batch and the threshold search.
static int size_batch(kv_index *ix, Batch &b) {
  const int64_t n_q = b.n_q = ix->batch_q, n_tiles = b.n_tiles = ix->batch_tiles;
  const int64_t n_groups = b.n_groups = (n_q + GROUP_Q - 1) / GROUP_Q;
  const int64_t n_blocks = (ix->n_chunks + B_BN - 1) / B_BN;
  const char *env = getenv("KAKVEDA_B200_NO_PRUNE");
  const bool prune = b.prune = !(env && env[0] == '1') && !ix->jaccard && ix->n_chunks >= 512;
  int64_t &n_bsplits = b.n_bsplits, &n_ssplits = b.n_ssplits;
  if (prune) {
    n_bsplits = std::max<int64_t>(1, std::min<int64_t>((ix->sm_count + n_tiles - 1) / n_tiles, n_blocks));
    // a bound CTA keeps the page table of its four candidate lists in shared memory: bound the chunks per row range
    while (n_bsplits < n_blocks && bound_smem_bytes((int)((((n_blocks + n_bsplits - 1) / n_bsplits + 1) * B_BN) / PAGE_RECS + 2)) > 232448)
      n_bsplits++;
    n_ssplits = std::max<int64_t>(1, std::min<int64_t>((4LL * ix->sm_count + n_groups * n_bsplits - 1) / (n_groups * n_bsplits), 8));
  } else {
    n_bsplits = std::max<int64_t>(1, std::min<int64_t>((8LL * ix->sm_count + n_groups - 1) / n_groups,
                                                        std::min<int64_t>(1024, std::max<int64_t>(1, ix->n_chunks / 4))));
    n_ssplits = 1;
  }
  const int64_t n_lists = n_groups * n_bsplits;
  b.n_parts = n_bsplits * n_ssplits;
  // scan of the stored codes (run_batch decides whether they are kept): CTAs per group over the group's windows of
  // chunks, so that the grid spans many waves and the groups with the most candidates do not form the tail
  const int64_t n_windows = (ix->n_chunks + S_WIN - 1) / S_WIN;
  b.n_csplits = std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>((CODE_SPLIT_CTAS * ix->sm_count + n_groups - 1) / n_groups, 8), n_windows));
  if (const char *e = getenv("KAKVEDA_B200_CODE_SPLITS")) b.n_csplits = std::max(1, atoi(e));  // tests: a forced split count
  b.n_ssplits_a = std::max<int64_t>(1, std::min<int64_t>((4LL * ix->sm_count + n_groups - 1) / n_groups, 8));
  ix->last_tiles = n_tiles; ix->last_splits = b.n_parts; ix->last_ctas = n_lists * n_ssplits;
  KV_CUDA(ix->d_stats.ensure(8));
  b.n_seed = (int)n_bsplits * B_SEEDS_PER_QUERY;
  const int64_t chunks_per_split = ((n_blocks + n_bsplits - 1) / n_bsplits + 1) * B_BN;
  b.max_pages = (int)(chunks_per_split / PAGE_RECS + 2);
  if (prune) {
    KV_CUDA(ix->d_tcode.ensure(n_q));
    KV_CUDA(ix->d_seeds.ensure(n_q * b.n_seed));
    KV_CUDA(ix->d_direct.ensure(n_groups * GROUP_Q * b.n_seed));
    // the bound kernel writes the lists of whole tiles (4 groups each), including the groups past the last query
    KV_CUDA(ix->d_list_count.ensure(n_groups + n_tiles * 4 * n_bsplits));
    KV_CUDA(ix->d_list_pages.ensure(n_tiles * 4 * n_bsplits * b.max_pages));
    const int64_t want_pages = std::min<int64_t>(n_lists * b.max_pages, 524288 + n_lists);  // up to 4 GiB of records
    if (want_pages > ix->pool_pages) {
      KV_CUDA(ix->d_pool.ensure(want_pages * PAGE_RECS));
      ix->pool_pages = want_pages;
    }
    KV_CUDA(ix->d_pool_ctl.ensure(2));
  }
  if (prune && bound_smem_bytes(b.max_pages) > 232448)
    return kv_fail(KV_ERR_INVALID, "kv_topk_resident: index too large for one bound-kernel row range (max_pages %d)", b.max_pages);
  return KV_OK;
}

// d_out_s / d_out_r: device outputs [n_q*k] (NULL: ix->d_out_s / d_out_r).  phase 0 = the whole top-k, 1 = bound pass +
// seed scan, 2 = the rest (kv_topk_resident_seed / _finish).
static int run_batch(kv_index *ix, int k, float *d_out_s, long long *d_out_r, int phase = 0) {
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_topk_resident: no query batch uploaded");
  if (k < 1 || k > 32) return kv_fail(KV_ERR_INVALID, "kv_topk_resident: k must be 1..32");
  int rc = check_filter(ix, "kv_topk_resident");
  if (rc != KV_OK) return rc;
  // Filtered and distinct batches may use the threshold exchange of a row-sharded GFKB: every rank holds the same batch
  // with the same filter and mode (kv_index_thresholds_peers), so a pushed threshold -- the k-th score of a list of the
  // query's label, of k distinct groups in distinct mode -- bounds the query's global k-th score.
  if (ix->distinct) {
    if (!ix->groups.ready(ix->n_rows))
      return kv_fail(KV_ERR_STATE, "kv_topk_resident: the batch is distinct but the row groups are missing or stale (set them again after an append)");
    // The raised seed threshold only bounds the global k-th GROUP score when the shards' seed lists were merged
    // group-aware: one group can count on several shards.  The caller declares it with KV_DISTINCT_MERGED_SEEDS.
    if (phase != 0 && !ix->merged_seeds)
      return kv_fail(KV_ERR_INVALID, "kv_topk_resident: the two-phase top-k of a distinct batch needs kv_query_set_distinct(ix, KV_DISTINCT_MERGED_SEEDS) "
                                     "(the seed k-th score is then taken over distinct groups)");
  }
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  if (!d_out_s) {  // results for a host read-back: the handle's own device outputs
    KV_CUDA(ix->d_out_s.ensure(ix->batch_q * k)); KV_CUDA(ix->d_out_r.ensure(ix->batch_q * k));
    d_out_s = ix->d_out_s.p; d_out_r = ix->d_out_r.p;
  }
  Batch b;
  b.k = k; b.phase = phase; b.out_s = d_out_s; b.out_r = d_out_r; b.distinct = ix->distinct;
  rc = size_batch(ix, b);
  if (rc != KV_OK) return rc;
  const int64_t n_q = b.n_q;
  const bool prune = b.prune;
  if (n_q > ix->d_gthr.cap && (ix->gthr_exported || ix->n_peers))
    return kv_fail(KV_ERR_STATE, "kv_topk_resident: the query batch outgrew the threshold array shared with the peer GPUs; exchange it again "
                                 "(kv_index_thresholds_export / kv_index_thresholds_peers)");
  KV_CUDA(ix->d_gthr.ensure(n_q));
  b.n_peers = (ix->n_peers > 0 && n_q <= ix->peer_cap) ? ix->n_peers : 0;
  const int64_t parts_alloc = std::max({b.n_parts, b.n_ssplits_a, b.n_csplits});
  KV_CUDA(ix->d_part_s.ensure(parts_alloc * n_q * k));
  KV_CUDA(ix->d_part_r.ensure(parts_alloc * n_q * k));
  // Second pass without recomputation: the first bound pass stores every bound as an 8-bit code (n_q x chunks bytes)
  // when that fits comfortably (KAKVEDA_B200_BOUND_CODES=0 forces the recomputing second pass).
  b.use_codes = false;
  if (prune) {
    const char *ce = getenv("KAKVEDA_B200_BOUND_CODES");
    const int64_t want = n_q * ix->n_chunks_pad;
    if (phase == 2) {
      b.use_codes = ix->last_used_codes != 0;
    } else if (!(ce && ce[0] == '0')) {
      b.use_codes = want <= ix->d_ubq.cap;
      if (!b.use_codes) {
        size_t free_b = 0, total_b = 0;
        cudaMemGetInfo(&free_b, &total_b);
        b.use_codes = want <= (int64_t)std::min<size_t>((size_t)64 << 30, free_b / 2);
        if (b.use_codes) KV_CUDA(ix->d_ubq.ensure(want));
      }
    }
  }
  if (phase != 2) ix->last_used_codes = b.use_codes ? 1 : 0;
  if (b.use_codes) {
    b.n_parts = b.n_csplits;
    ix->last_splits = b.n_parts; ix->last_ctas = b.n_groups * b.n_csplits;
  }

  if (phase != 2) {
    KV_CUDA(cudaEventRecord(ix->ev[1], s));
    for (auto &e : ix->evk) KV_CUDA(cudaEventRecord(e, s));
  }
  const int64_t prior_launches = phase == 2 ? ix->last_launches : 0;
  ix->two_phase = prune && phase == 2;
  if (ix->n_rows == 0) {
    KV_CUDA(cudaEventRecord(ix->ev[2], s));
    std::vector<float> es((size_t)(n_q * k), -INFINITY);
    std::vector<long long> er((size_t)(n_q * k), -1);
    KV_CUDA(cudaMemcpyAsync(d_out_s, es.data(), es.size() * 4, cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaMemcpyAsync(d_out_r, er.data(), er.size() * 8, cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaStreamSynchronize(s));
    ix->last_launches = prior_launches;
    KV_CUDA(cudaEventRecord(ix->ev[3], s));
    return KV_OK;
  }
  if (phase != 2) {  // global lower bounds of the k-th score start at -inf
    KV_CUDA(cudaMemsetAsync(ix->d_stats.p, 0, 8 * sizeof(unsigned long long), s));
    fill_int_kernel<<<(unsigned)((n_q + 255) / 256), 256, 0, s>>>(ix->d_gthr.p, n_q, (int)0xFF800000);
    KV_CUDA(cudaGetLastError());
    b.launches++;
  }
  if (phase == 1 && !prune) {  // the exhaustive and Jaccard paths have no seed phase: empty seed lists
    fill_int_kernel<<<(unsigned)((n_q * k + 255) / 256), 256, 0, s>>>((int *)d_out_s, n_q * k, (int)0xFF800000);
    fill_ll_kernel<<<(unsigned)((n_q * k + 255) / 256), 256, 0, s>>>(d_out_r, n_q * k, -1LL);
    KV_CUDA(cudaGetLastError());
    ix->last_launches = b.launches + 2;
    return KV_OK;
  }
  rc = prune ? run_pruned(ix, b) : ix->jaccard ? run_jaccard(ix, b) : run_exhaustive(ix, b);
  if (rc != KV_OK) return rc;
  if (phase == 1) { ix->last_launches = b.launches; return KV_OK; }
  KV_CUDA(cudaEventRecord(ix->evk[4], s));
  KV_CUDA(cudaEventRecord(ix->ev[2], s));
  if ((rc = launch_merge(ix, b, b.n_parts)) != KV_OK) return rc;
  KV_CUDA(cudaEventRecord(ix->evk[5], s));
  b.launches++;
  // queries no path scanned: null queries score 0 against every row, irregular ones take the float64 full scan
  if (ix->batch_null && b.distinct) {
    fill_null_distinct_kernel<<<(unsigned)((ix->batch_null * 32 + 255) / 256), 256, 0, s>>>(
        ix->d_qperm.p + n_q, (int)ix->batch_null, k, ix->n_rows, ix->row_base, ix->has_excl ? ix->d_excl_orig.p : nullptr,
        ix->has_filter ? ix->d_filt_orig.p : nullptr, ix->labels.d_row.p, dead_rows(ix), ix->groups.d_row.p, d_out_s, d_out_r);
    KV_CUDA(cudaGetLastError());
    b.launches++;
  } else if (ix->batch_null) {
    const LabelFirstRows L{ix->d_lab_keys.p, ix->d_lab_rows.p, ix->n_lab};
    fill_null_kernel<<<(unsigned)((ix->batch_null * k + 255) / 256), 256, 0, s>>>(ix->d_qperm.p + n_q, (int)ix->batch_null, k,
                                                                                  ix->n_rows, ix->row_base,
                                                                                  ix->has_excl ? ix->d_excl_orig.p : nullptr,
                                                                                  ix->has_filter ? ix->d_filt_orig.p : nullptr, L,
                                                                                  ix->tomb.any() ? ix->d_first_live.p : nullptr, d_out_s, d_out_r);
    KV_CUDA(cudaGetLastError());
    b.launches++;
  }
  if (ix->batch_null && ix->qtags.on) {  // the null queries with tags walk the index for their first eligible rows
    const RowTags &T = ix->tags;
    fill_null_tags_kernel<<<(unsigned)((ix->batch_null * 32 + 255) / 256), 256, 0, s>>>(
        ix->d_qperm.p + n_q, (int)ix->batch_null, k, ix->n_rows, ix->row_base, ix->has_excl ? ix->d_excl_orig.p : nullptr,
        ix->has_filter ? ix->d_filt_orig.p : nullptr, ix->labels.d_row.p, dead_rows(ix), b.distinct ? ix->groups.d_row.p : nullptr,
        ix->qtags.d_mask_orig.p, ix->qtags.d_tags_orig.p, ix->d_invperm.p, T.d_mask_pos.p, T.masks_exact ? nullptr : T.d_ptr_pos.p,
        T.masks_exact ? nullptr : T.d_list_pos.p, d_out_s, d_out_r);
    KV_CUDA(cudaGetLastError());
    b.launches++;
  }
  const IrregularQueries &irr = ix->irr;
  for (size_t i = 0; i < irr.q.size(); i++) {
    const int64_t q = irr.q[i], a = irr.indptr[i], e = irr.indptr[i + 1];
    rc = score_impl(ix, irr.ids.data() + a, irr.tf.data() + a, e - a, irr.oov[i], nullptr);
    if (rc != KV_OK) return rc;
    const uint8_t *dq = nullptr;
    if ((rc = batch_fallback_dead(ix, q, &dq)) != KV_OK) return rc;
    if (b.distinct)
      select_topk_distinct_kernel<float><<<1, 1024, 0, s>>>(ix->d_scores.p, ix->n_rows, ix->row_base, k,
                                                     ix->has_excl ? (int64_t)ix->h_excl_orig[(size_t)q] : -1, ix->labels.d_row.p,
                                                     ix->has_filter ? ix->h_filt_orig[(size_t)q] : -1, dq,
                                                     ix->groups.d_row.p, d_out_s + q * k, d_out_r + q * k);
    else
      select_topk_kernel<float><<<1, 1024, 0, s>>>(ix->d_scores.p, ix->n_rows, ix->row_base, k,
                                            ix->has_excl ? (int64_t)ix->h_excl_orig[(size_t)q] : -1, ix->labels.d_row.p,
                                            ix->has_filter ? ix->h_filt_orig[(size_t)q] : -1, dq, d_out_s + q * k,
                                            d_out_r + q * k);
    KV_CUDA(cudaGetLastError());
    b.launches += 2;
  }
  KV_CUDA(cudaMemcpyAsync(ix->last_stats, ix->d_stats.p, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  if (prune) KV_CUDA(cudaMemcpyAsync(&ix->last_stats[6], ix->d_pool_ctl.p, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
  ix->last_launches = prior_launches + b.launches;
  KV_CUDA(cudaEventRecord(ix->ev[3], s));
  return KV_OK;
}

// after the stream is synchronised: whether the last run's bound pass ran out of candidate-pool pages
static int check_pool(kv_index *ix) {
  const unsigned int *ctl = (const unsigned int *)&ix->last_stats[6];
  if (ix->n_rows > 0 && ctl[1] != 0) {
    ix->last_stats[6] = 0;
    return kv_fail(KV_ERR_NOMEM, "kv_topk_resident: the candidate pool (%lld pages) is exhausted; split the query batch",
                   (long long)ix->pool_pages);
  }
  return KV_OK;
}

// after the stream is synchronised: timings of the batch and the candidate-pool check
static int finish_batch(kv_index *ix) {
  for (int i = 1; i < 4; i++) cudaEventElapsedTime(&ix->last_ms[i], ix->ev[i], ix->ev[i + 1]);
  for (int i = 0; i < 5; i++) cudaEventElapsedTime(&ix->last_kernel_ms[i], ix->evk[i], ix->evk[i + 1]);
  if (ix->two_phase) cudaEventElapsedTime(&ix->last_kernel_ms[2], ix->evp2, ix->evk[3]);
  return check_pool(ix);
}

// Threshold search over the resident batch: every pair with score >= thr lands in ix->range (ix->jrange on a Jaccard
// index), *n_pairs = their count.  When they do not fit, the buffer grows to the exact count and only the scan and the
// fallbacks run again (the candidate lists depend on the threshold alone).  Events: evk[2] -> evk[3] bound pass 1,
// evk[3] -> evk[4] scan, evk[4] -> evk[5] irregular-query fallbacks.  `fn` names the entry point in errors.  Caller
// holds ix->mu.
static int run_range(kv_index *ix, float thr, int64_t *n_pairs, const char *fn) {
  drop_range(ix);
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "%s: no query batch uploaded", fn);
  int rc = check_filter(ix, fn);
  if (rc != KV_OK) return rc;
  const bool jac = ix->jaccard != 0;
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  Batch b;
  b.k = 0; b.phase = 2; b.out_s = nullptr; b.out_r = nullptr; b.range = true; b.use_codes = false; b.n_peers = 0;
  rc = size_batch(ix, b);  // a Jaccard index never prunes
  if (rc != KV_OK) return rc;
  const int64_t n_q = b.n_q;
  KV_CUDA(ix->d_rthr.ensure(n_q));
  rc = jac ? ix->jrange.prepare(s) : ix->range.prepare(s);
  if (rc != KV_OK) return rc;
  auto range_cap = [&] { return jac ? ix->jrange.capacity() : ix->range.capacity(); };
  unsigned long long *d_count = jac ? ix->jrange.d_count.p : ix->range.d_count.p;
  for (auto &e : ix->evk) KV_CUDA(cudaEventRecord(e, s));
  KV_CUDA(cudaMemsetAsync(ix->d_stats.p, 0, 8 * sizeof(unsigned long long), s));
  float ms[5] = {0, 0, 0, 0, 0};
  unsigned long long count = 0;
  if (ix->n_rows > 0) {
    int thr_bits;
    memcpy(&thr_bits, &thr, sizeof(thr_bits));
    fill_int_kernel<<<(unsigned)((n_q + 255) / 256), 256, 0, s>>>(ix->d_rthr.p, n_q, thr_bits);
    KV_CUDA(cudaGetLastError());
    b.launches++;
    for (int run = 0;; run++) {
      if (run == 0 && b.prune) {
        KV_CUDA(cudaMemsetAsync(ix->d_pool_ctl.p, 0, 2 * sizeof(unsigned int), s));
        KV_CUDA(cudaEventRecord(ix->evk[2], s));
        rc = run_pruned(ix, b);  // bound pass 1 (ends with evk[3]), then the scan
      } else {
        KV_CUDA(cudaEventRecord(ix->evk[3], s));
        rc = jac ? run_jaccard(ix, b) : b.prune ? scan_candidates(ix, b) : run_exhaustive(ix, b);
      }
      if (rc != KV_OK) return rc;
      KV_CUDA(cudaEventRecord(ix->evk[4], s));
      const IrregularQueries &irr = ix->irr;
      for (size_t i = 0; i < irr.q.size(); i++) {
        const int64_t q = irr.q[i], a = irr.indptr[i], e = irr.indptr[i + 1];
        rc = score_impl(ix, irr.ids.data() + a, irr.tf.data() + a, e - a, irr.oov[i], nullptr);
        if (rc != KV_OK) return rc;
        const unsigned grid = (unsigned)std::min<int64_t>((ix->n_rows + 255) / 256, 8LL * ix->sm_count);
        const int64_t excl = ix->has_excl ? (int64_t)ix->h_excl_orig[(size_t)q] : -1;
        if (jac) {
          const double nq = host_query_norm(ix, irr.ids.data() + a, irr.tf.data() + a, e - a, irr.oov[i]);  // |q|
          jaccard_select_range_kernel<<<grid, 256, 0, s>>>(ix->d_scores.p, ix->d_B64.p, ix->d_invperm.p, ix->n_rows, nq, thr, excl,
                                                           (int)q, ix->jrange.pairs.p, d_count, range_cap());
        } else {
          const uint8_t *dq = nullptr;
          if ((rc = batch_fallback_dead(ix, q, &dq)) != KV_OK) return rc;
          select_range_kernel<<<grid, 256, 0, s>>>(ix->d_scores.p, ix->n_rows, ix->row_base, thr, excl, ix->labels.d_row.p,
                                                   ix->has_filter ? ix->h_filt_orig[(size_t)q] : -1, dq, (int)q, ix->range.pairs.p,
                                                   d_count, range_cap());
        }
        KV_CUDA(cudaGetLastError());
        b.launches += 2;
      }
      KV_CUDA(cudaEventRecord(ix->evk[5], s));
      KV_CUDA(cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, s));
      KV_CUDA(cudaMemcpyAsync(ix->last_stats, ix->d_stats.p, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
      if (b.prune) KV_CUDA(cudaMemcpyAsync(&ix->last_stats[6], ix->d_pool_ctl.p, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
      KV_CUDA(cudaStreamSynchronize(s));
      if (run == 0 && b.prune) {
        cudaEventElapsedTime(&ms[2], ix->evk[2], ix->evk[3]);
        if ((rc = check_pool(ix)) != KV_OK) return rc;
      }
      float t_scan = 0, t_fallback = 0;
      cudaEventElapsedTime(&t_scan, ix->evk[3], ix->evk[4]);
      cudaEventElapsedTime(&t_fallback, ix->evk[4], ix->evk[5]);
      ms[3] += t_scan;
      ms[4] += t_fallback;
      if (count <= range_cap()) break;
      if ((rc = jac ? ix->jrange.grow(count, s, fn) : ix->range.grow(count, s, fn)) != KV_OK) return rc;
      // the counters describe one run: the bound pass's stay, the scan's start again
      KV_CUDA(cudaMemsetAsync(ix->d_stats.p, 0, 2 * sizeof(unsigned long long), s));
    }
  } else {
    for (auto &st : ix->last_stats) st = 0;
  }
  for (int i = 0; i < 5; i++) ix->last_kernel_ms[i] = ms[i];
  ix->last_launches = b.launches;
  if (jac) ix->jrange.commit(n_q, (int64_t)count);
  else ix->range.commit(n_q, (int64_t)count);
  *n_pairs = (int64_t)count;
  return KV_OK;
}

// One top-k run of the resident batch into device outputs (NULL: the handle's own), copied to h_scores / h_rows when
// given.  Returns once the stream is complete, with the batch's timings and the candidate-pool check.  Caller holds ix->mu.
static int topk_run(kv_index *ix, int k, int phase, void *d_scores, void *d_rows, float *h_scores, int64_t *h_rows) {
  int rc = run_batch(ix, k, (float *)d_scores, (long long *)d_rows, phase);
  if (rc != KV_OK) return rc;
  cudaStream_t s = ix->stream;
  if (h_scores) {
    const size_t n = (size_t)(ix->batch_q * k);
    KV_CUDA(cudaMemcpyAsync(h_scores, ix->d_out_s.p, n * sizeof(float), cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaMemcpyAsync(h_rows, ix->d_out_r.p, n * sizeof(long long), cudaMemcpyDeviceToHost, s));
  }
  KV_CUDA(cudaEventRecord(ix->ev[4], s));
  KV_CUDA(cudaStreamSynchronize(s));
  return finish_batch(ix);
}

int kv_query_upload(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                    const double *q_oov_tf2, int64_t n_q) {
  if (!ix || n_q < 1 || !q_indptr) return kv_fail(KV_ERR_INVALID, "kv_query_upload: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  return prepare_batch(ix, q_indptr, q_ids, q_tf, q_oov_tf2, n_q);
}

int kv_query_upload_text(kv_index *ix, kv_vocab_mirror *m, const kv_vocab *v, const char *bytes, const int64_t *offsets,
                         int64_t n_q, int mode, int64_t *bad_doc) {
  if (!ix || !m || !v || n_q < 1 || !offsets || !bytes) return kv_fail(KV_ERR_INVALID, "kv_query_upload_text: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  return prepare_batch_text(ix, m, v, bytes, offsets, n_q, mode, bad_doc);
}

int kv_debug_query_order(kv_index *ix, int32_t *qperm, uint8_t *flags, int64_t n_q) {
  if (!ix || !qperm || !flags) return kv_fail(KV_ERR_INVALID, "kv_debug_query_order: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_debug_query_order: no resident batch");
  if (n_q != ix->batch_q) return kv_fail(KV_ERR_INVALID, "kv_debug_query_order: the batch has %lld queries", (long long)ix->batch_q);
  memcpy(qperm, ix->h_qperm.p, (size_t)n_q * sizeof(int));
  memcpy(flags, ix->h_flags.p, (size_t)n_q);
  return KV_OK;
}

// A slice of a query batch prepared where it was featurised: the slice's CSR re-stored in text order (s_* outputs, row
// p = the p-th smallest query, equal queries in their original order), order_out[p] = original index of row p, and the
// classification flags by row.
int kv_query_prepare_slice(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                           const double *q_oov_tf2, int64_t n_q, int64_t *s_indptr, uint32_t *s_ids, uint32_t *s_tf,
                           double *s_oov_tf2, int32_t *order_out, uint8_t *flags_out) {
  if (!ix || n_q < 0 || !q_indptr || !s_indptr || !order_out || !flags_out || !s_oov_tf2)
    return kv_fail(KV_ERR_INVALID, "kv_query_prepare_slice: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_query_prepare_slice: index not finalized");
  if (n_q >= (1LL << 31) - TILE_Q || !csr_ok(q_indptr, q_ids, q_tf, n_q)) return kv_fail(KV_ERR_INVALID, "kv_query_prepare_slice: bad query CSR");
  const int64_t nnz = q_indptr[n_q] - q_indptr[0];
  if (nnz > 0 && (!s_ids || !s_tf)) return kv_fail(KV_ERR_INVALID, "kv_query_prepare_slice: bad arguments");
  const int T = host_threads();
  std::vector<int> order((size_t)n_q);
  for (int64_t q = 0; q < n_q; q++) order[(size_t)q] = (int)q;
  stable_sort_indices(order, [&](int a, int b) {
    return cmp_seq(q_ids + q_indptr[a], q_indptr[a + 1] - q_indptr[a], q_ids + q_indptr[b], q_indptr[b + 1] - q_indptr[b]) < 0;
  }, T);
  s_indptr[0] = 0;
  for (int64_t p = 0; p < n_q; p++) {
    const int64_t q = order[(size_t)p];
    s_indptr[p + 1] = s_indptr[p] + (q_indptr[q + 1] - q_indptr[q]);
    order_out[p] = (int32_t)q;
    s_oov_tf2[p] = q_oov_tf2 ? q_oov_tf2[q] : 0.0;
  }
  parallel_for(n_q, n_q >= 4096 ? T : 1, [&](int, int64_t a, int64_t b) {
    for (int64_t p = a; p < b; p++) {
      const int64_t q = order[(size_t)p], len = q_indptr[q + 1] - q_indptr[q];
      if (len) {
        memcpy(s_ids + s_indptr[p], q_ids + q_indptr[q], (size_t)len * 4);
        memcpy(s_tf + s_indptr[p], q_tf + q_indptr[q], (size_t)len * 4);
      }
    }
  });
  classify_queries(ix, s_indptr, s_ids, s_tf, n_q, flags_out, T);
  return KV_OK;
}

// kv_query_upload of a batch that arrives as n_runs consecutive slices (run r holds queries [sum n_q[<r], ...)).
int kv_query_upload_runs(kv_index *ix, int n_runs, const int64_t *const *q_indptr, const uint32_t *const *q_ids,
                         const uint32_t *const *q_tf, const double *const *q_oov_tf2, const int32_t *const *order,
                         const uint8_t *const *flags, const int64_t *n_q) {
  if (!ix || n_runs < 1 || !q_indptr || !q_ids || !q_tf || !n_q) return kv_fail(KV_ERR_INVALID, "kv_query_upload_runs: bad arguments");
  std::vector<QueryRun> runs((size_t)n_runs);
  for (int r = 0; r < n_runs; r++) {
    QueryRun &R = runs[(size_t)r];
    R.indptr = q_indptr[r]; R.ids = q_ids[r]; R.tf = q_tf[r]; R.n_q = n_q[r];
    R.oov = q_oov_tf2 ? q_oov_tf2[r] : nullptr;
    R.order = order ? order[r] : nullptr;
    R.flags = flags ? flags[r] : nullptr;
  }
  std::lock_guard<std::mutex> g(ix->mu);
  return prepare_batch_runs(ix, runs.data(), n_runs);
}

int kv_index_last_prepare_ms(const kv_index *ix, float ms[4]) {
  if (!ix || !ms) return kv_fail(KV_ERR_INVALID, "kv_index_last_prepare_ms: bad arguments");
  for (int i = 0; i < 4; i++) ms[i] = ix->last_prepare_ms[i];
  return KV_OK;
}

static int set_exclusions_locked(kv_index *ix, const int64_t *exclude_rows, int64_t n_q);

int kv_query_set_exclusions(kv_index *ix, const int64_t *exclude_rows, int64_t n_q) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_query_set_exclusions: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  return set_exclusions_locked(ix, exclude_rows, n_q);
}

int kv_selfjoin_upload(kv_index *ix, int64_t q_begin, int64_t q_end) {
  if (!ix || q_begin < 0 || q_end <= q_begin) return kv_fail(KV_ERR_INVALID, "kv_selfjoin_upload: bad row range");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_selfjoin_upload: index not finalized");
  if (q_end > ix->n_rows) return kv_fail(KV_ERR_INVALID, "kv_selfjoin_upload: row range outside the index");
  const int64_t n = q_end - q_begin, base = ix->h_indptr[(size_t)q_begin];
  std::vector<int64_t> ip((size_t)n + 1), ex((size_t)n);
  for (int64_t i = 0; i <= n; i++) ip[(size_t)i] = ix->h_indptr[(size_t)(q_begin + i)] - base;
  std::vector<uint32_t> tf32((size_t)ip[(size_t)n]);
  for (size_t i = 0; i < tf32.size(); i++) tf32[i] = ix->h_tf[(size_t)base + i];
  QueryRun R;
  R.indptr = ip.data(); R.ids = ix->h_ids.data() + base; R.tf = tf32.data(); R.n_q = n;
  std::vector<uint8_t> flags;
  if (ix->tomb.any()) {  // a deleted row's query is switched off (flag 3): no path answers it, its list stays (-inf, -1)
    flags.resize((size_t)n);
    classify_queries(ix, ip.data(), R.ids, R.tf, n, flags.data(), host_threads());
    for (int64_t i = 0; i < n; i++)
      if (ix->tomb.is_dead(q_begin + i)) flags[(size_t)i] = 3;
    R.flags = flags.data();
  }
  int rc = prepare_batch_runs(ix, &R, 1);
  if (rc != KV_OK) return rc;
  ix->batch_selfjoin = true;
  for (int64_t i = 0; i < n; i++) ex[(size_t)i] = ix->row_base + q_begin + i;
  return set_exclusions_locked(ix, ex.data(), n);
}

// caller holds ix->mu, the index is finalized and has rows: a query batch for K6 -- its CSR and |q|^2 exactly as K1a gets
// them (prep_query, float64) -- in ix->d_rq_*, and room for n_q * k pairs in d_rq_rows / d_rq_out
// (the copies read cst and ip, which the caller keeps until it synchronises the stream)
static int rescore_upload(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                          const double *q_oov_tf2, int64_t n_q, int k, std::vector<double> &cst, std::vector<int64_t> &ip) {
  const int64_t nnz = q_indptr[n_q] - q_indptr[0];
  cudaStream_t s = ix->stream;
  cst.resize((size_t)n_q);
  ip.resize((size_t)n_q + 1);
  for (int64_t q = 0; q <= n_q; q++) ip[(size_t)q] = q_indptr[q] - q_indptr[0];
  parallel_for(n_q, n_q >= 2048 ? host_threads() : 1, [&](int, int64_t a, int64_t b) {
    for (int64_t q = a; q < b; q++)
      cst[(size_t)q] = host_query_norm(ix, q_ids + q_indptr[q], q_tf + q_indptr[q], q_indptr[q + 1] - q_indptr[q], q_oov_tf2 ? q_oov_tf2[q] : 0.0);
  });
  KV_CUDA(ix->d_rq_indptr.ensure(n_q + 1)); KV_CUDA(ix->d_rq_ids.ensure(std::max<int64_t>(nnz, 1)));
  KV_CUDA(ix->d_rq_tf.ensure(std::max<int64_t>(nnz, 1))); KV_CUDA(ix->d_rq_const.ensure(n_q));
  KV_CUDA(ix->d_rq_out.ensure(n_q * k)); KV_CUDA(ix->d_rq_rows.ensure(n_q * k));
  KV_CUDA(cudaMemcpyAsync(ix->d_rq_indptr.p, ip.data(), (size_t)(n_q + 1) * 8, cudaMemcpyHostToDevice, s));
  if (nnz) {
    KV_CUDA(cudaMemcpyAsync(ix->d_rq_ids.p, q_ids + q_indptr[0], (size_t)nnz * 4, cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaMemcpyAsync(ix->d_rq_tf.p, q_tf + q_indptr[0], (size_t)nnz * 4, cudaMemcpyHostToDevice, s));
  }
  KV_CUDA(cudaMemcpyAsync(ix->d_rq_const.p, cst.data(), (size_t)n_q * 8, cudaMemcpyHostToDevice, s));
  return KV_OK;
}

// caller holds ix->mu, after rescore_upload: K6 of the pairs (query q, global row d_rq_rows[q * k + j]) into d_rq_out
static int rescore_launch(kv_index *ix, int64_t n_q, int k) {
  RescoreParams P;
  P.indptr = ix->indptr.p; P.ids = ix->ids.p; P.tf = ix->tf.p;
  P.a64 = ix->d_a64.p; P.d64 = ix->d_d64.p; P.B64 = ix->d_B64.p; P.invperm = ix->d_invperm.p;
  P.q_indptr = ix->d_rq_indptr.p; P.q_ids = ix->d_rq_ids.p; P.q_tf = ix->d_rq_tf.p;
  P.q_nq = ix->d_rq_const.p;
  P.rows = ix->d_rq_rows.p; P.n_q = n_q; P.n_rows = ix->n_rows; P.row_base = ix->row_base; P.V = ix->V;
  P.k = k; P.jaccard = ix->jaccard; P.dead = dead_rows(ix); P.out = ix->d_rq_out.p;
  rescore_kernel<<<(unsigned)((n_q * k * 32 + 255) / 256), 256, 0, ix->stream>>>(P);
  KV_CUDA(cudaGetLastError());
  return KV_OK;
}

int kv_rescore_pairs(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                     const double *q_oov_tf2, int64_t n_q, int k, const int64_t *rows, double *out_scores) {
  if (!ix || n_q < 0 || k < 1 || (n_q > 0 && (!q_indptr || !rows || !out_scores)))
    return kv_fail(KV_ERR_INVALID, "kv_rescore_pairs: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_rescore_pairs: index not finalized");
  if (n_q == 0) return KV_OK;
  const int64_t nnz = q_indptr[n_q] - q_indptr[0];
  if (nnz < 0 || (nnz > 0 && (!q_ids || !q_tf))) return kv_fail(KV_ERR_INVALID, "kv_rescore_pairs: bad query CSR");
  if (ix->n_rows == 0) {
    for (int64_t i = 0; i < n_q * k; i++) out_scores[i] = -INFINITY;
    return KV_OK;
  }
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  std::vector<double> cst;
  std::vector<int64_t> ip;
  int rc = rescore_upload(ix, q_indptr, q_ids, q_tf, q_oov_tf2, n_q, k, cst, ip);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaMemcpyAsync(ix->d_rq_rows.p, rows, (size_t)n_q * k * 8, cudaMemcpyHostToDevice, s));
  if ((rc = rescore_launch(ix, n_q, k)) != KV_OK) return rc;
  KV_CUDA(cudaMemcpyAsync(out_scores, ix->d_rq_out.p, (size_t)n_q * k * 8, cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  return KV_OK;
}

// kv_exact_topk and kv_exact_topk_tags (tag_indptr NULL: no query has tags; fn names the entry point)
static int exact_topk_impl(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                           const double *q_oov_tf2, const int32_t *labels, const int64_t *tag_indptr, const int32_t *tags,
                           int distinct, int64_t n_q, int k, int64_t *out_rows, double *out_scores, const char *fn) {
  if (!ix || n_q < 0 || k < 1 || k > 32 || (n_q > 0 && (!q_indptr || !out_rows || !out_scores)))
    return kv_fail(KV_ERR_INVALID, "%s: bad arguments (k must be 1..32)", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  if (tag_indptr && ix->jaccard) return kv_fail(KV_ERR_INVALID, "%s: a Jaccard index (mode 1) has no tag filter", fn);
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "%s: index not finalized", fn);
  if (n_q == 0) return KV_OK;
  const int64_t nnz = q_indptr[n_q] - q_indptr[0];
  if (nnz < 0 || (nnz > 0 && (!q_ids || !q_tf))) return kv_fail(KV_ERR_INVALID, "%s: bad query CSR", fn);
  bool filtered = false;
  for (int64_t q = 0; labels && q < n_q; q++) {
    if (labels[q] < -1) return kv_fail(KV_ERR_INVALID, "%s: label %d of query %lld is below -1", fn, labels[q], (long long)q);
    filtered |= labels[q] >= 0;
  }
  std::vector<unsigned long long> tmask;
  std::vector<int> tlist;
  bool tagged = false;
  if (tag_indptr) {
    const int rc = parse_query_tag_csr(tag_indptr, tags, n_q, fn, "tag indptr", tmask, tlist, &tagged);
    if (rc != KV_OK) return rc;
  }
  if (ix->n_rows == 0) {
    for (int64_t i = 0; i < n_q * k; i++) { out_rows[i] = -1; out_scores[i] = -INFINITY; }
    return KV_OK;
  }
  if (filtered && !ix->labels.ready(ix->n_rows))
    return kv_fail(KV_ERR_STATE, "%s: a filtered query needs row labels (kv_index_set_row_labels)", fn);
  if (distinct && !ix->groups.ready(ix->n_rows))
    return kv_fail(KV_ERR_STATE, "%s: distinct needs row groups (kv_index_set_row_groups)", fn);
  if (tagged && !ix->tags.ready(ix->n_rows))
    return kv_fail(KV_ERR_STATE, "%s: a query with tags needs row tags for the current rows (kv_index_set_row_tags)", fn);
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  std::vector<double> cst;
  std::vector<int64_t> ip;
  int rc = rescore_upload(ix, q_indptr, q_ids, q_tf, q_oov_tf2, n_q, k, cst, ip);
  if (rc != KV_OK) return rc;
  DevBuf<int> d_tlist;
  if (tagged) {
    KV_CUDA(d_tlist.ensure((int64_t)tlist.size()));
    KV_CUDA(cudaMemcpyAsync(d_tlist.p, tlist.data(), tlist.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  for (int64_t q = 0; q < n_q; q++) {
    // K1a into ix->d_scores, then the best k rows in float64 order into d_rq_rows (global) -- the K1a scores they come
    // with land in d_rq_out, which K6 overwrites below
    const int64_t a = q_indptr[q], e = q_indptr[q + 1];
    if ((rc = score_impl(ix, q_ids + a, q_tf + a, e - a, q_oov_tf2 ? q_oov_tf2[q] : 0.0, nullptr)) != KV_OK) return rc;
    const int lab = labels ? labels[q] : -1;
    const uint8_t *dq = dead_rows(ix);
    if (tagged && (rc = fallback_dead(ix, tmask[(size_t)q], d_tlist.p + q * MAX_QTAGS, &dq)) != KV_OK) return rc;
    if (distinct)
      select_topk_distinct_kernel<double><<<1, 1024, 0, s>>>(ix->d_scores.p, ix->n_rows, ix->row_base, k, -1, ix->labels.d_row.p,
                                                             lab, dq, ix->groups.d_row.p, ix->d_rq_out.p + q * k,
                                                             ix->d_rq_rows.p + q * k);
    else
      select_topk_kernel<double><<<1, 1024, 0, s>>>(ix->d_scores.p, ix->n_rows, ix->row_base, k, -1, ix->labels.d_row.p, lab,
                                                    dq, ix->d_rq_out.p + q * k, ix->d_rq_rows.p + q * k);
    KV_CUDA(cudaGetLastError());
  }
  if ((rc = rescore_launch(ix, n_q, k)) != KV_OK) return rc;
  KV_CUDA(cudaMemcpyAsync(out_rows, ix->d_rq_rows.p, (size_t)n_q * k * 8, cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaMemcpyAsync(out_scores, ix->d_rq_out.p, (size_t)n_q * k * 8, cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  return KV_OK;
}

int kv_exact_topk(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                  const double *q_oov_tf2, const int32_t *labels, int distinct, int64_t n_q, int k, int64_t *out_rows,
                  double *out_scores) {
  return exact_topk_impl(ix, q_indptr, q_ids, q_tf, q_oov_tf2, labels, nullptr, nullptr, distinct, n_q, k, out_rows,
                         out_scores, "kv_exact_topk");
}

int kv_exact_topk_tags(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                       const double *q_oov_tf2, const int32_t *labels, const int64_t *tag_indptr, const int32_t *tags,
                       int distinct, int64_t n_q, int k, int64_t *out_rows, double *out_scores) {
  return exact_topk_impl(ix, q_indptr, q_ids, q_tf, q_oov_tf2, labels, tag_indptr, tags, distinct, n_q, k, out_rows,
                         out_scores, "kv_exact_topk_tags");
}

static int set_exclusions_locked(kv_index *ix, const int64_t *exclude_rows, int64_t n_q) {
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_query_set_exclusions: no query batch uploaded");
  if (!exclude_rows) { ix->has_excl = false; return KV_OK; }
  if (n_q != ix->batch_q) return kv_fail(KV_ERR_INVALID, "kv_query_set_exclusions: %lld entries for a batch of %lld queries",
                                         (long long)n_q, (long long)ix->batch_q);
  KV_CUDA(cudaSetDevice(ix->device));
  // global row ids -> local original rows of this shard (-1: none, or the row lives on another shard)
  ix->h_excl_orig.assign((size_t)n_q, -1);
  for (int64_t q = 0; q < n_q; q++) {
    const int64_t r = exclude_rows[q] - ix->row_base;
    if (exclude_rows[q] >= 0 && r >= 0 && r < ix->n_rows) ix->h_excl_orig[(size_t)q] = (int)r;
  }
  std::vector<int> sorted((size_t)n_q);
  for (int64_t i = 0; i < n_q; i++) sorted[(size_t)i] = ix->h_excl_orig[(size_t)ix->h_qperm.p[i]];
  KV_CUDA(ix->d_excl_sorted.ensure(n_q)); KV_CUDA(ix->d_excl_orig.ensure(n_q));
  KV_CUDA(cudaMemcpyAsync(ix->d_excl_sorted.p, sorted.data(), (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice, ix->stream));
  KV_CUDA(cudaMemcpyAsync(ix->d_excl_orig.p, ix->h_excl_orig.data(), (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice, ix->stream));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  ix->has_excl = true;
  return KV_OK;
}

int kv_query_set_filter(kv_index *ix, const int32_t *labels, int64_t n_q) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_query_set_filter: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  if (labels && ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_query_set_filter: a Jaccard index (mode 1) has no label filter");
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_query_set_filter: no query batch uploaded");
  if (!labels) { ix->has_filter = false; return KV_OK; }
  if (n_q != ix->batch_q) return kv_fail(KV_ERR_INVALID, "kv_query_set_filter: %lld labels for a batch of %lld queries",
                                         (long long)n_q, (long long)ix->batch_q);
  bool any = false;
  for (int64_t q = 0; q < n_q; q++) {
    if (labels[q] < -1) return kv_fail(KV_ERR_INVALID, "kv_query_set_filter: label %d of query %lld is below -1", labels[q], (long long)q);
    any = any || labels[q] >= 0;
  }
  ix->has_filter = false;
  if (!any) return KV_OK;  // every query unfiltered: the unfiltered batch
  if (!ix->labels.ready(ix->n_rows))
    return kv_fail(KV_ERR_STATE, "kv_query_set_filter: the index has no row labels for its current rows (kv_index_set_row_labels)");
  KV_CUDA(cudaSetDevice(ix->device));
  ix->h_filt_orig.assign(labels, labels + n_q);
  std::vector<int> sorted((size_t)n_q);
  for (int64_t i = 0; i < n_q; i++) sorted[(size_t)i] = ix->h_filt_orig[(size_t)ix->h_qperm.p[i]];
  KV_CUDA(ix->d_filt_sorted.ensure(n_q)); KV_CUDA(ix->d_filt_orig.ensure(n_q));
  KV_CUDA(cudaMemcpyAsync(ix->d_filt_sorted.p, sorted.data(), (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice, ix->stream));
  KV_CUDA(cudaMemcpyAsync(ix->d_filt_orig.p, ix->h_filt_orig.data(), (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice, ix->stream));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  ix->has_filter = true;
  return KV_OK;
}

int kv_query_set_tag_filter(kv_index *ix, const int64_t *indptr, const int32_t *tags, int64_t n_q) {
  const char *fn = "kv_query_set_tag_filter";
  if (!ix) return kv_fail(KV_ERR_INVALID, "%s: NULL handle", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  if (indptr && ix->jaccard) return kv_fail(KV_ERR_INVALID, "%s: a Jaccard index (mode 1) has no tag filter", fn);
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "%s: no query batch uploaded", fn);
  if (!indptr) { ix->qtags.on = false; return KV_OK; }
  if (n_q != ix->batch_q)
    return kv_fail(KV_ERR_INVALID, "%s: %lld tag sets for a batch of %lld queries", fn, (long long)n_q, (long long)ix->batch_q);
  std::vector<unsigned long long> mask;
  std::vector<int> list;
  bool any = false;
  const int prc = parse_query_tag_csr(indptr, tags, n_q, fn, "indptr", mask, list, &any);
  if (prc != KV_OK) return prc;
  QueryTags &Q = ix->qtags;
  Q.on = false;
  if (!any) return KV_OK;  // no query has tags: the batch without a tag filter
  if (!ix->tags.ready(ix->n_rows))
    return kv_fail(KV_ERR_STATE, "%s: the index has no row tags for its current rows (kv_index_set_row_tags)", fn);
  KV_CUDA(cudaSetDevice(ix->device));
  std::vector<unsigned long long> mask_sorted((size_t)n_q);
  std::vector<int> list_sorted((size_t)n_q * MAX_QTAGS);
  for (int64_t i = 0; i < n_q; i++) {
    const int64_t q = ix->h_qperm.p[i];
    mask_sorted[(size_t)i] = mask[(size_t)q];
    std::copy_n(list.begin() + q * MAX_QTAGS, MAX_QTAGS, list_sorted.begin() + i * MAX_QTAGS);
  }
  KV_CUDA(Q.d_mask_orig.ensure(n_q)); KV_CUDA(Q.d_mask_sorted.ensure(n_q));
  KV_CUDA(Q.d_tags_orig.ensure(n_q * MAX_QTAGS)); KV_CUDA(Q.d_tags_sorted.ensure(n_q * MAX_QTAGS));
  cudaStream_t s = ix->stream;
  KV_CUDA(cudaMemcpyAsync(Q.d_mask_orig.p, mask.data(), mask.size() * 8, cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemcpyAsync(Q.d_mask_sorted.p, mask_sorted.data(), mask_sorted.size() * 8, cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemcpyAsync(Q.d_tags_orig.p, list.data(), list.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemcpyAsync(Q.d_tags_sorted.p, list_sorted.data(), list_sorted.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaStreamSynchronize(s));
  Q.h_mask = std::move(mask);
  Q.on = true;
  return KV_OK;
}

int kv_query_set_distinct(kv_index *ix, int on) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_query_set_distinct: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  if (on && ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_query_set_distinct: a Jaccard index (mode 1) has no distinct top-k");
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_query_set_distinct: no query batch uploaded");
  ix->distinct = ix->merged_seeds = false;
  if (!on) return KV_OK;
  if (!ix->groups.ready(ix->n_rows))
    return kv_fail(KV_ERR_STATE, "kv_query_set_distinct: the index has no row groups for its current rows (kv_index_set_row_groups)");
  ix->distinct = true;
  ix->merged_seeds = on == KV_DISTINCT_MERGED_SEEDS;
  return KV_OK;
}

int kv_topk_resident_host(kv_index *ix, int k, float *out_scores, int64_t *out_rows) {
  if (!ix || !out_scores || !out_rows) return kv_fail(KV_ERR_INVALID, "kv_topk_resident_host: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  return topk_run(ix, k, 0, nullptr, nullptr, out_scores, out_rows);
}

int kv_range_resident(kv_index *ix, float threshold, int64_t *n_pairs) {
  if (!ix || !n_pairs) return kv_fail(KV_ERR_INVALID, "kv_range_resident: bad arguments");
  if (!(threshold > 0.f && threshold <= 1.f)) return kv_fail(KV_ERR_INVALID, "kv_range_resident: threshold must be in (0, 1]");
  std::lock_guard<std::mutex> g(ix->mu);
  return run_range(ix, threshold, n_pairs, "kv_range_resident");
}

// The float32 threshold of an exact search's first stage: the largest float32 <= thr * (1 - KV_RANGE_EXACT_MARGIN),
// and at least the smallest positive float32 (the float32 search needs a positive threshold).
static float exact_prefilter_threshold(double thr) {
  const double t = thr * (1.0 - KV_RANGE_EXACT_MARGIN);
  float f = (float)t;
  if ((double)f > t) f = std::nextafter(f, 0.f);
  return std::max(f, std::numeric_limits<float>::denorm_min());
}

// K6-R of the ix->range records into ix->xrange (room for all of them): events evk[0] -> evk[1] around the kernel.
// Caller holds ix->mu, after rescore_upload.
static int rescore_range_launch(kv_index *ix, int64_t n, double thr) {
  RescoreRangeParams R;
  RescoreParams &P = R.K6;
  P.indptr = ix->indptr.p; P.ids = ix->ids.p; P.tf = ix->tf.p;
  P.a64 = ix->d_a64.p; P.d64 = ix->d_d64.p; P.B64 = ix->d_B64.p; P.invperm = ix->d_invperm.p;
  P.q_indptr = ix->d_rq_indptr.p; P.q_ids = ix->d_rq_ids.p; P.q_tf = ix->d_rq_tf.p;
  P.q_nq = ix->d_rq_const.p;
  P.rows = nullptr; P.n_q = ix->range.n_q; P.n_rows = ix->n_rows; P.row_base = ix->row_base; P.V = ix->V;
  P.k = 0; P.jaccard = ix->jaccard; P.dead = nullptr; P.out = nullptr;
  R.in = ix->range.pairs.p; R.n = n; R.thr = thr; R.out = ix->xrange.pairs.p; R.count = ix->xrange.d_count.p;
  const int64_t warps = (n + 31) / 32;
  KV_CUDA(cudaEventRecord(ix->evk[0], ix->stream));
  rescore_range_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, ix->stream>>>(R);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaEventRecord(ix->evk[1], ix->stream));
  return KV_OK;
}

int kv_range_resident_exact(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                            const double *q_oov_tf2, int64_t n_q, double threshold, int64_t *n_pairs,
                            int64_t *n_candidates) {
  const char *fn = "kv_range_resident_exact";
  if (!ix || !n_pairs || n_q < 1 || !q_indptr) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  if (!(threshold > 0.0 && threshold <= 1.0)) return kv_fail(KV_ERR_INVALID, "%s: threshold must be in (0, 1]", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  if (ix->jaccard) return kv_fail(KV_ERR_INVALID, "%s: a Jaccard index (mode 1) has no exact threshold search", fn);
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "%s: index not finalized", fn);
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "%s: no query batch uploaded", fn);
  if (ix->batch_selfjoin) return kv_fail(KV_ERR_INVALID, "%s: a self-join batch (kv_selfjoin_upload) has no exact threshold search", fn);
  if (n_q != ix->batch_q)
    return kv_fail(KV_ERR_INVALID, "%s: a query CSR of %lld queries for a batch of %lld", fn, (long long)n_q, (long long)ix->batch_q);
  const int64_t nnz = q_indptr[n_q] - q_indptr[0];
  if (nnz < 0 || (nnz > 0 && (!q_ids || !q_tf))) return kv_fail(KV_ERR_INVALID, "%s: bad query CSR", fn);
  int64_t cand = 0;
  int rc = run_range(ix, exact_prefilter_threshold(threshold), &cand, fn);
  if (rc != KV_OK) return rc;
  ix->range.valid = false;  // its records are K6-R's input now, not a result
  cudaStream_t s = ix->stream;
  unsigned long long kept = 0;
  float ms = 0.f;
  if ((rc = ix->xrange.prepare(s)) != KV_OK) return rc;
  if ((unsigned long long)cand > ix->xrange.capacity() && (rc = ix->xrange.grow((unsigned long long)cand, s, fn)) != KV_OK)
    return rc;
  if (cand > 0) {
    std::vector<double> cst;
    std::vector<int64_t> ip;
    if ((rc = rescore_upload(ix, q_indptr, q_ids, q_tf, q_oov_tf2, n_q, 1, cst, ip)) != KV_OK) return rc;
    if ((rc = rescore_range_launch(ix, cand, threshold)) != KV_OK) return rc;
    KV_CUDA(cudaMemcpyAsync(&kept, ix->xrange.d_count.p, sizeof(kept), cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaStreamSynchronize(s));
    cudaEventElapsedTime(&ms, ix->evk[0], ix->evk[1]);
  }
  ix->last_kernel_ms[0] = ms;
  ix->xrange.commit(n_q, (int64_t)kept);
  *n_pairs = (int64_t)kept;
  if (n_candidates) *n_candidates = cand;
  return KV_OK;
}

// The count outputs a fetch was given must fit the index's mode: required on a Jaccard index (like rows and scores, only
// when there are pairs), NULL on a TF-IDF index.  Checked before anything is consumed.
static int check_count_outputs(const kv_index *ix, const void *inter, const void *uni, const char *fn) {
  if (!ix->jaccard && (inter || uni))
    return kv_fail(KV_ERR_INVALID, "%s: a TF-IDF index has no count outputs (pass NULL for inter and uni)", fn);
  if (ix->jaccard && ix->jrange.valid && ix->jrange.n_pairs > 0 && (!inter || !uni))
    return kv_fail(KV_ERR_INVALID, "%s: a Jaccard index returns the exact counts (inter and uni are required)", fn);
  return KV_OK;
}

// The pairs come back in emit order, which the scan does not fix; scores are exact integer sums (Jaccard: the quotient
// inter / union) rounded once, so (score desc, row asc) is a total order of each query's pairs and the result is
// deterministic.  Both fetches order the pairs on the device and consume the result (RangeResult).
int kv_range_fetch(kv_index *ix, int64_t *indptr, int64_t *rows, float *scores, int32_t *inter, int32_t *uni) {
  const char *fn = "kv_range_fetch", *search = "kv_range_resident";
  if (!ix || !indptr) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  if (ix->xrange.valid) return kv_fail(KV_ERR_STATE, "%s: the last threshold search was exact (kv_range_fetch_exact)", fn);
  const int rc = check_count_outputs(ix, inter, uni, fn);
  if (rc != KV_OK) return rc;
  return ix->jaccard ? ix->jrange.fetch_host(fn, search, ix->device, ix->stream, ix->rsort, ix->row_base, indptr, rows, scores, inter, uni)
                     : ix->range.fetch_host(fn, search, ix->device, ix->stream, ix->rsort, ix->row_base, indptr, rows, scores, inter, uni);
}

// Device outputs: the same arrays, written to caller-owned device memory of the index's device.
int kv_range_fetch_device(kv_index *ix, void *d_indptr, void *d_rows, void *d_scores, void *d_inter, void *d_uni) {
  const char *fn = "kv_range_fetch_device", *search = "kv_range_resident";
  if (!ix) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  if (ix->xrange.valid)
    return kv_fail(KV_ERR_STATE, "%s: the last threshold search was exact (kv_range_fetch_exact_device)", fn);
  const int rc = check_count_outputs(ix, d_inter, d_uni, fn);
  if (rc != KV_OK) return rc;
  return ix->jaccard ? ix->jrange.fetch_device(fn, search, ix->device, ix->stream, ix->rsort, ix->row_base, d_indptr, d_rows,
                                               d_scores, d_inter, d_uni)
                     : ix->range.fetch_device(fn, search, ix->device, ix->stream, ix->rsort, ix->row_base, d_indptr, d_rows,
                                              d_scores, d_inter, d_uni);
}

// The exact result: the same CSR with float64 scores; a float32 result is not one (KV_ERR_STATE).
static int check_exact_result(const kv_index *ix, const char *fn) {
  if (!ix->xrange.valid && (ix->range.valid || ix->jrange.valid))
    return kv_fail(KV_ERR_STATE, "%s: the last threshold search was a float32 one (kv_range_fetch)", fn);
  return KV_OK;
}

int kv_range_fetch_exact(kv_index *ix, int64_t *indptr, int64_t *rows, double *scores) {
  const char *fn = "kv_range_fetch_exact", *search = "kv_range_resident_exact";
  if (!ix || !indptr) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  const int rc = check_exact_result(ix, fn);
  if (rc != KV_OK) return rc;
  return ix->xrange.fetch_host(fn, search, ix->device, ix->stream, ix->rsort, ix->row_base, indptr, rows, scores, nullptr,
                               nullptr);
}

int kv_range_fetch_exact_device(kv_index *ix, void *d_indptr, void *d_rows, void *d_scores) {
  const char *fn = "kv_range_fetch_exact_device", *search = "kv_range_resident_exact";
  if (!ix) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  const int rc = check_exact_result(ix, fn);
  if (rc != KV_OK) return rc;
  return ix->xrange.fetch_device(fn, search, ix->device, ix->stream, ix->rsort, ix->row_base, d_indptr, d_rows, d_scores,
                                 nullptr, nullptr);
}

int kv_index_thresholds_export(kv_index *ix, int64_t capacity, void *handle_out) {
  if (!ix || capacity < 1 || !handle_out) return kv_fail(KV_ERR_INVALID, "kv_index_thresholds_export: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "the C ABI documents a 64-byte handle");
  std::lock_guard<std::mutex> g(ix->mu);
  KV_CUDA(cudaSetDevice(ix->device));
  if (ix->n_peers) return kv_fail(KV_ERR_STATE, "kv_index_thresholds_export: clear the peer mapping first (n_peers = 0)");
  KV_CUDA(ix->d_gthr.ensure(capacity));
  cudaIpcMemHandle_t h;
  KV_CUDA(cudaIpcGetMemHandle(&h, ix->d_gthr.p));
  memcpy(handle_out, &h, sizeof(h));
  ix->gthr_exported = true;
  return KV_OK;
}

int kv_index_thresholds_peers(kv_index *ix, const void *handles, int n_peers, int64_t capacity) {
  if (!ix || n_peers < 0 || n_peers > 7 || (n_peers > 0 && (!handles || capacity < 1)))
    return kv_fail(KV_ERR_INVALID, "kv_index_thresholds_peers: bad arguments (at most 7 peers)");
  std::lock_guard<std::mutex> g(ix->mu);
  KV_CUDA(cudaSetDevice(ix->device));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  close_peers(ix);
  if (n_peers == 0) { ix->gthr_exported = false; return KV_OK; }
  for (int i = 0; i < n_peers; i++) {
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char *)handles + (size_t)i * sizeof(h), sizeof(h));
    void *p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      ix->n_peers = i;
      close_peers(ix);
      return kv_fail(KV_ERR_CUDA, "kv_index_thresholds_peers: cudaIpcOpenMemHandle failed for peer %d: %s", i, cudaGetErrorString(e));
    }
    ix->peer_gthr[i] = (int *)p;
  }
  ix->n_peers = n_peers;
  ix->peer_cap = capacity;
  return KV_OK;
}

// Test hook: the peer threshold pushes of kv_index_thresholds_peers between indexes of ONE process on one device, without
// CUDA IPC.  Every peer must already hold a threshold array of `capacity` queries (kv_index_thresholds_export); the
// arrays are borrowed, so unmapping never closes an IPC mapping.  n_peers = 0 unlinks.
int kv_debug_thresholds_link(kv_index *ix, kv_index *const *peers, int n_peers, int64_t capacity) {
  if (!ix || n_peers < 0 || n_peers > 7 || (n_peers > 0 && (!peers || capacity < 1)))
    return kv_fail(KV_ERR_INVALID, "kv_debug_thresholds_link: bad arguments (at most 7 peers)");
  std::lock_guard<std::mutex> g(ix->mu);
  KV_CUDA(cudaSetDevice(ix->device));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  close_peers(ix);
  for (int i = 0; i < n_peers; i++) {
    if (!peers[i] || peers[i] == ix || peers[i]->device != ix->device || peers[i]->d_gthr.cap < capacity)
      return kv_fail(KV_ERR_INVALID, "kv_debug_thresholds_link: peer %d is not another exported index on this device", i);
    ix->peer_gthr[i] = peers[i]->d_gthr.p;
  }
  ix->n_peers = n_peers;
  ix->peer_cap = n_peers ? capacity : 0;
  ix->peers_borrowed = n_peers > 0;
  return KV_OK;
}

int kv_topk_resident(kv_index *ix, int k, void *d_scores, void *d_rows) {
  if (!ix || !d_scores || !d_rows) return kv_fail(KV_ERR_INVALID, "kv_topk_resident: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  return topk_run(ix, k, 0, d_scores, d_rows, nullptr, nullptr);
}

// Two-phase form for a row-sharded GFKB: _seed runs the bound pass and the seed scan of the resident batch and returns
// this shard's seed top-k (device, by original query); the caller merges the shards' seed lists (one small all-gather)
// and feeds the GLOBAL k-th seed score of every query back with kv_index_raise_thresholds; _finish then selects and
// scans only the chunks that can still beat it.  Every shard prunes with the threshold a single index would have.
int kv_topk_resident_seed(kv_index *ix, int k, void *d_scores, void *d_rows) {
  if (!ix || !d_scores || !d_rows) return kv_fail(KV_ERR_INVALID, "kv_topk_resident_seed: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  int rc = run_batch(ix, k, (float *)d_scores, (long long *)d_rows, 1);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return KV_OK;
}

int kv_index_raise_thresholds(kv_index *ix, const void *d_kth_scores, int64_t n_q) {
  if (!ix || !d_kth_scores) return kv_fail(KV_ERR_INVALID, "kv_index_raise_thresholds: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->batch_valid || n_q != ix->batch_q) return kv_fail(KV_ERR_STATE, "kv_index_raise_thresholds: no matching resident batch");
  if (n_q > ix->d_gthr.cap) return kv_fail(KV_ERR_STATE, "kv_index_raise_thresholds: run kv_topk_resident_seed first");
  KV_CUDA(cudaSetDevice(ix->device));
  raise_thresholds_kernel<<<(unsigned)((n_q + 255) / 256), 256, 0, ix->stream>>>((const float *)d_kth_scores, ix->d_qperm.p, n_q,
                                                                                  ix->d_gthr.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return KV_OK;
}

int kv_topk_resident_finish(kv_index *ix, int k, void *d_scores, void *d_rows) {
  if (!ix || !d_scores || !d_rows) return kv_fail(KV_ERR_INVALID, "kv_topk_resident_finish: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  return topk_run(ix, k, 2, d_scores, d_rows, nullptr, nullptr);
}

int kv_merge_topk_device(int device, const void *d_scores_in, const void *d_rows_in, int n_lists, int64_t n_q, int k,
                         void *d_scores_out, void *d_rows_out) {
  return kv_merge_topk_device_on(device, d_scores_in, d_rows_in, n_lists, n_q, k, n_q * k, n_q * k, d_scores_out, d_rows_out,
                                 nullptr, 1);
}

// stream: the CUDA stream (cudaStream_t) the input lists were produced on -- e.g. the stream an NCCL all-gather was
// enqueued on -- or NULL for the legacy default stream; sync != 0 waits for the merge before returning.  stride_s /
// stride_r: float32 / int64 elements between consecutive lists (packed all-gather buffers interleave both arrays).
int kv_merge_topk_device_on(int device, const void *d_scores_in, const void *d_rows_in, int n_lists, int64_t n_q, int k,
                            int64_t stride_s, int64_t stride_r, void *d_scores_out, void *d_rows_out, void *stream, int sync) {
  if (n_lists < 1 || n_lists > 2048 || n_q < 0 || k < 1 || k > 255 || !d_scores_in || !d_rows_in || !d_scores_out || !d_rows_out ||
      stride_s < n_q * k || stride_r < n_q * k)
    return kv_fail(KV_ERR_INVALID, "kv_merge_topk_device: bad arguments");
  if (n_q == 0) return KV_OK;
  KV_CUDA(cudaSetDevice(device));
  cudaStream_t s = (cudaStream_t)stream;
  merge_topk_kernel<<<(unsigned)((n_q * 32 + 255) / 256), 256, 0, s>>>((const float *)d_scores_in, (const long long *)d_rows_in,
                                                                       n_lists, n_q, k, stride_s, stride_r, nullptr,
                                                                       (float *)d_scores_out, (long long *)d_rows_out);
  KV_CUDA(cudaGetLastError());
  if (sync) KV_CUDA(cudaStreamSynchronize(s));
  return KV_OK;
}

// K5 of a distinct batch over lists of several indexes (e.g. the row shards' lists after the all-gather): the kernel
// launch_merge runs for one index, with the groups of every global row.  Waits for the merge: whether a row had no
// group is only known then.  The 4-byte flag it is reported in is one per device, allocated by the first call and kept
// for the process, so that a call allocates nothing; calls on one device take turns on it.
int kv_merge_topk_distinct_device_on(int device, const void *d_scores_in, const void *d_rows_in, int n_lists, int64_t n_q,
                                     int k, int64_t stride_s, int64_t stride_r, const void *d_row_groups,
                                     int64_t n_group_rows, void *d_scores_out, void *d_rows_out, void *stream) {
  const char *fn = "kv_merge_topk_distinct_device";
  if (n_lists < 1 || n_lists > 2048 || n_q < 0 || k < 1 || k > 32 || n_group_rows < 0 || stride_s < n_q * k ||
      stride_r < n_q * k)
    return kv_fail(KV_ERR_INVALID, "%s: bad arguments (1 to 2048 lists, k 1..32, strides of at least n_q * k)", fn);
  if (n_q == 0) return KV_OK;
  int sm_count = 0;
  int rc = open_device(device, fn, &sm_count);
  if (rc != KV_OK) return rc;
  const struct { const void *p; size_t al; const char *what; } ptrs[] = {
      {d_scores_in, 4, "scores_in"}, {d_rows_in, 8, "rows_in"}, {d_scores_out, 4, "scores_out"}, {d_rows_out, 8, "rows_out"},
      {d_row_groups, 4, "row_groups"}};
  for (int j = 0; j < (n_group_rows > 0 ? 5 : 4); j++)
    if ((rc = check_device_ptr(ptrs[j].p, device, ptrs[j].al, ptrs[j].what, fn)) != KV_OK) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  static std::mutex mu;
  static unsigned *flags[256] = {};
  if (device >= 256) return kv_fail(KV_ERR_INVALID, "%s: device %d", fn, device);
  std::lock_guard<std::mutex> g(mu);
  unsigned *&d_bad = flags[device];
  if (!d_bad) KV_CUDA(cudaMalloc((void **)&d_bad, sizeof(unsigned)));
  unsigned bad = 0;
  cudaError_t e = cudaMemsetAsync(d_bad, 0, sizeof(unsigned), s);
  if (e == cudaSuccess) {
    merge_topk_distinct_kernel<<<(unsigned)((n_q * 32 + 255) / 256), 256, 0, s>>>(
        (const float *)d_scores_in, (const long long *)d_rows_in, n_lists, n_q, k, stride_s, stride_r, nullptr,
        (const int *)d_row_groups, 0, n_group_rows, d_bad, (float *)d_scores_out, (long long *)d_rows_out);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return kv_fail(KV_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(e));
  if (bad)
    return kv_fail(KV_ERR_INVALID, "%s: a row outside the %lld rows of the group table (the outputs are undefined)", fn,
                   (long long)n_group_rows);
  return KV_OK;
}

// Test hook: the numerators of the chunk bounds the bound kernel forms for the resident batch (sorted query slot i =
// query order[i]), [n_q][n_chunks] floats on the host, plus the slot -> query map.  Small indexes only.
int kv_debug_bound_numerators(kv_index *ix, int k, float *out, int32_t *slot_query) {
  if (!ix || !out || !slot_query) return kv_fail(KV_ERR_INVALID, "kv_debug_bound_numerators: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_debug_bound_numerators: no query batch uploaded");
  KV_CUDA(cudaSetDevice(ix->device));
  const int64_t n_q = ix->batch_q, stride = ix->n_chunks_pad;
  DevBuf<float> xs;
  KV_CUDA(xs.ensure(n_q * stride));
  KV_CUDA(cudaMemset(xs.p, 0, (size_t)(n_q * stride) * 4));
  ix->dbg_xs = xs.p;
  int rc = run_batch(ix, k, nullptr, nullptr);
  ix->dbg_xs = nullptr;
  if (rc == KV_OK) {
    KV_CUDA(cudaEventRecord(ix->ev[4], ix->stream));
    KV_CUDA(cudaStreamSynchronize(ix->stream));
    std::vector<float> h((size_t)(n_q * stride));
    KV_CUDA(cudaMemcpy(h.data(), xs.p, h.size() * 4, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n_q; i++) {
      memcpy(out + i * ix->n_chunks, h.data() + i * stride, (size_t)ix->n_chunks * 4);
      slot_query[i] = ix->h_qperm.p[i];
    }
  }
  return rc;
}

// Test hook: what bound pass 0 of the resident batch produced on the headline path (no dbg_xs, so the instantiation is
// the one kv_topk_resident picks): the 8-bit codes and threshold codes the candidate scan compared, the query constants
// and chunk minima the bounds were formed from, and the scan layout's row order.
int kv_debug_bound_codes(kv_index *ix, int k, uint8_t *codes, int32_t *slot_query, int32_t *tcode, float *q_terms,
                         float *chunk_minB, int32_t *row_at_pos) {
  if (!ix || !codes || !slot_query) return kv_fail(KV_ERR_INVALID, "kv_debug_bound_codes: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_debug_bound_codes: no query batch uploaded");
  KV_CUDA(cudaSetDevice(ix->device));
  const int64_t n_q = ix->batch_q;
  int rc = topk_run(ix, k, 0, nullptr, nullptr, nullptr, nullptr);
  if (rc != KV_OK) return rc;
  if (!ix->last_used_codes) {
    const char *np = getenv("KAKVEDA_B200_NO_PRUNE"), *ce = getenv("KAKVEDA_B200_BOUND_CODES");
    const char *why = ix->jaccard ? "a Jaccard index has no bound pass"
                      : (np && np[0] == '1') || ix->n_chunks < 512 ? "the exhaustive path ran (fewer than 512 chunks or KAKVEDA_B200_NO_PRUNE=1)"
                      : (ce && ce[0] == '0') ? "KAKVEDA_B200_BOUND_CODES=0: bound pass 1 recomputed the bounds"
                                             : "the codes did not fit in device memory";
    return kv_fail(KV_ERR_STATE, "kv_debug_bound_codes: the run kept no bound codes (%s)", why);
  }
  const int64_t nch = ix->n_chunks;
  KV_CUDA(cudaMemcpy2D(codes, (size_t)nch, ix->d_ubq.p, (size_t)ix->n_chunks_pad, (size_t)nch, (size_t)n_q, cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < n_q; i++) slot_query[i] = ix->h_qperm.p[i];
  if (tcode) KV_CUDA(cudaMemcpy(tcode, ix->d_tcode.p, (size_t)n_q * sizeof(int), cudaMemcpyDeviceToHost));
  if (q_terms) {
    std::vector<float> qc((size_t)(7 * n_q));
    KV_CUDA(cudaMemcpy(qc.data(), ix->d_qconst.p, qc.size() * sizeof(float), cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n_q; i++) {  // d_qconst: nq, dotU, corrU, dotS, corrS, dotX, 1 / s_q
      q_terms[4 * i] = qc[(size_t)i];
      q_terms[4 * i + 1] = qc[(size_t)(3 * n_q + i)];
      q_terms[4 * i + 2] = qc[(size_t)(5 * n_q + i)];
      q_terms[4 * i + 3] = qc[(size_t)(4 * n_q + i)];
    }
  }
  if (chunk_minB) KV_CUDA(cudaMemcpy(chunk_minB, ix->d_cminB.p, (size_t)nch * sizeof(float), cudaMemcpyDeviceToHost));
  if (row_at_pos && ix->n_rows) KV_CUDA(cudaMemcpy(row_at_pos, ix->d_perm.p, (size_t)ix->n_rows * sizeof(int), cudaMemcpyDeviceToHost));
  return KV_OK;
}

int kv_index_last_timing(const kv_index *ix, float ms[4]) {
  if (!ix || !ms) return kv_fail(KV_ERR_INVALID, "kv_index_last_timing: bad arguments");
  for (int i = 0; i < 4; i++) ms[i] = ix->last_ms[i];
  return KV_OK;
}

int kv_index_last_kernel_ms(const kv_index *ix, float ms[5]) {
  if (!ix || !ms) return kv_fail(KV_ERR_INVALID, "kv_index_last_kernel_ms: bad arguments");
  for (int i = 0; i < 5; i++) ms[i] = ix->last_kernel_ms[i];
  return KV_OK;
}

int kv_index_last_score_ms(const kv_index *ix, float *ms) {
  if (!ix || !ms) return kv_fail(KV_ERR_INVALID, "kv_index_last_score_ms: bad arguments");
  *ms = ix->last_score_ms;
  return KV_OK;
}

int kv_index_layout(const kv_index *ix, int64_t bytes[4], int64_t counts[20]) {
  if (!ix || !bytes || !counts) return kv_fail(KV_ERR_INVALID, "kv_index_layout: bad arguments");
  bytes[0] = ix->blk_words * 4;
  bytes[1] = ix->n_rows * 4;
  bytes[2] = ix->n_chunks_pad * (int64_t)sizeof(BlockInfo);
  const int64_t rare_table_bytes = ix->n_rt_slots * (int64_t)sizeof(uint4) + (ix->n_chunks_pad / 64) * (RB_BITS / 8);
  bytes[3] = ix->n_chunks_pad * (int64_t)(NF * sizeof(__half) + sizeof(float)) + rare_table_bytes + (ix->n_chunks_pad / 64) * (int64_t)(NF2 * 16);
  counts[0] = ix->n_entries; counts[1] = ix->n_univ; counts[2] = ix->n_rows;
  counts[3] = ix->last_ctas; counts[4] = ix->last_tiles; counts[5] = ix->last_splits;
  counts[6] = ix->batch_h2d_bytes; counts[7] = ix->n_ovf;
  counts[8] = ix->n_chunks;
  counts[9] = (int64_t)ix->last_stats[0];   // (query, chunk) pairs scored (seed scan + candidate scan)
  counts[10] = (int64_t)ix->last_stats[1];  // candidate records scanned
  counts[11] = (int64_t)ix->last_stats[2];  // (query, chunk) pairs whose bound passed
  counts[12] = (int64_t)ix->last_stats[3];  // candidate records written
  counts[13] = ix->last_launches;
  counts[14] = ix->n_rare_entries;
  counts[15] = (int64_t)(ix->last_stats[6] & 0xFFFFFFFFull);  // pool pages used
  counts[16] = ix->pool_pages;
  counts[17] = ix->batch_f2_outside;  // second-class (query, feature) listings of the batch left out of their tile's dictionary
  counts[18] = ix->n_rt_slots;
  counts[19] = ix->rt_enlarged;
  return KV_OK;
}

}  // extern "C"

// ----------------------------------------------------------------------------------------
// Persisted scan layout (SURVEY 8(f) rank 4): the arrays kv_index_finalize builds on the host cores (row order, column
// blocks, dense / bitmap / rare-table side structures) written to one file, so that a cold start of a large GFKB is
// "read + H2D + statistics kernels" instead of a 15 s sort and block build.  The file is tied to the rows by their
// count, entry count and a checksum of the CSR; a file that does not match is refused (the caller then finalizes the
// usual way).  kv_index_layout_load is called after the rows were appended and BEFORE kv_index_finalize, which then takes
// the statistics-only path (kv_index_last_finalize_kind == 2).
// ----------------------------------------------------------------------------------------
namespace {
constexpr uint64_t LAYOUT_MAGIC = 0x33594C42564B4B41ULL;  // "AKKVBLY3"

uint64_t csr_checksum(const kv_index *ix) {
  const int T = host_threads();
  std::vector<uint64_t> part((size_t)T, 0);
  parallel_for(ix->n_rows, T, [&](int t, int64_t a, int64_t b) {
    uint64_t h = 1469598103934665603ULL ^ (uint64_t)a;
    for (int64_t r = a; r < b; r++) {
      for (int64_t p = ix->h_indptr[(size_t)r]; p < ix->h_indptr[(size_t)r + 1]; p++) {
        h = (h ^ ix->h_ids[(size_t)p]) * 1099511628211ULL;
        h = (h ^ ix->h_tf[(size_t)p]) * 1099511628211ULL;
      }
      h = (h ^ 0xFFFFFFFFULL) * 1099511628211ULL;  // row boundary
    }
    part[(size_t)t] = h;
  });
  uint64_t h = 1469598103934665603ULL;
  for (uint64_t x : part) h = (h ^ x) * 1099511628211ULL;
  return h;
}

template <class T>
bool put(FILE *f, const std::vector<T> &v) { return v.empty() || fwrite(v.data(), sizeof(T), v.size(), f) == v.size(); }
template <class T>
bool get(FILE *f, std::vector<T> &v, size_t n) { v.resize(n); return n == 0 || fread(v.data(), sizeof(T), n, f) == n; }
}  // namespace

extern "C" int kv_index_layout_save(kv_index *ix, const char *path) {
  if (!ix || !path) return kv_fail(KV_ERR_INVALID, "kv_index_layout_save: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->finalized || !ix->layout_valid) return kv_fail(KV_ERR_STATE, "kv_index_layout_save: index has no built layout (finalize first)");
  KV_CUDA(cudaSetDevice(ix->device));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  ScanLayout SL;
  LayoutHeader &H = SL.H;
  H.magic = LAYOUT_MAGIC; H.checksum = csr_checksum(ix);
  H.n_rows = ix->n_rows; H.nnz = ix->nnz; H.V = (int64_t)ix->h_fslot.size(); H.n_chunks = ix->n_chunks; H.n_chunks_pad = ix->n_chunks_pad;
  H.blk_words = ix->blk_words; H.n_entries = ix->n_entries; H.n_rare_entries = ix->n_rare_entries; H.n_ovf = ix->n_ovf;
  H.n_rt_slots = ix->n_rt_slots; H.rt_enlarged = (int32_t)ix->rt_enlarged; H.n_blocks = ix->n_chunks_pad / 64; H.univ_len = (int64_t)ix->layout_univ.size();
  H.jaccard = ix->jaccard; H.corpus_fit = ix->corpus_fit;
  cudaError_t err = cudaSuccess;
  each_array(SL, ix, [&](auto &h, auto &d, size_t n) {
    h.resize(n);
    if (n) err = cudaMemcpy(h.data(), d.p, n * sizeof(h[0]), cudaMemcpyDeviceToHost);
    return err == cudaSuccess;
  });
  KV_CUDA(err);
  FILE *f = fopen(path, "wb");
  if (!f) return kv_fail(KV_ERR_INVALID, "kv_index_layout_save: cannot open %s", path);
  bool ok = fwrite(&H, sizeof(H), 1, f) == 1 && put(f, ix->layout_univ) &&
            each_array(SL, ix, [&](const auto &h, auto &, size_t) { return put(f, h); });
  ok = (fclose(f) == 0) && ok;
  if (!ok) return kv_fail(KV_ERR_INVALID, "kv_index_layout_save: short write to %s", path);
  return KV_OK;
}

extern "C" int kv_index_layout_load(kv_index *ix, const char *path) {
  if (!ix || !path) return kv_fail(KV_ERR_INVALID, "kv_index_layout_load: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  KV_CUDA(cudaSetDevice(ix->device));
  FILE *f = fopen(path, "rb");
  if (!f) return kv_fail(KV_ERR_INVALID, "kv_index_layout_load: cannot open %s", path);
  ScanLayout SL;
  const LayoutHeader &H = SL.H;
  bool ok = fread(&SL.H, sizeof(SL.H), 1, f) == 1 && H.magic == LAYOUT_MAGIC;
  if (ok && (H.n_rows != ix->n_rows || H.nnz != ix->nnz || H.jaccard != ix->jaccard || H.corpus_fit != ix->corpus_fit || H.checksum != csr_checksum(ix))) {
    fclose(f);
    return kv_fail(KV_ERR_STATE, "kv_index_layout_load: %s was built for other rows (or another mode)", path);
  }
  ok = ok && get(f, SL.univ, (size_t)H.univ_len) && each_array(SL, ix, [&](auto &h, auto &, size_t n) { return get(f, h, n); });
  fclose(f);
  if (!ok) return kv_fail(KV_ERR_INVALID, "kv_index_layout_load: %s is not a layout file of this version (or is truncated)", path);
  int rc = upload_layout(ix, SL);
  if (rc != KV_OK) return rc;
  ix->finalized = false;
  ix->labels.on_device = ix->groups.on_device = ix->tags.on_device = false;  // positions changed: the finalize that follows rebuilds them
  return KV_OK;
}

#ifdef KV_SCAN_CLOCKS
// Measuring build only (see KV_SCAN_CLOCKS in tfidf_kernels.cuh): copies the candidate scan's profile of the current
// device to out[0..n) and clears it.  n must be the profile's slot count, so a caller with another layout fails.
extern "C" int kv_debug_scan_profile(unsigned long long *out, int n) {
  static unsigned long long zero[KVP_TOTAL];
  if (!out || n != KVP_TOTAL) return kv_fail(KV_ERR_INVALID, "kv_debug_scan_profile: the profile has %d slots", (int)KVP_TOTAL);
  KV_CUDA(cudaDeviceSynchronize());
  KV_CUDA(cudaMemcpyFromSymbol(out, g_scan_prof, sizeof(zero)));
  KV_CUDA(cudaMemcpyToSymbol(g_scan_prof, zero, sizeof(zero)));
  return KV_OK;
}
#endif

#ifdef KV_BOUND_CLOCKS
// Measuring build only (see KV_BOUND_CLOCKS in bound_kernel.cuh): copies the bound kernel's profile of the current
// device to out[0..n) and clears it.  n must be the profile's slot count, so a caller with another layout fails.
extern "C" int kv_debug_bound_profile(unsigned long long *out, int n) {
  if (!out || n != KB_TOTAL) return kv_fail(KV_ERR_INVALID, "kv_debug_bound_profile: the profile has %d slots", (int)KB_TOTAL);
  KV_CUDA(cudaDeviceSynchronize());
  KV_CUDA(cudaMemcpyFromSymbol(out, g_bound_prof, sizeof(g_bound_prof)));
  void *p = nullptr;
  KV_CUDA(cudaGetSymbolAddress(&p, g_bound_prof));
  KV_CUDA(cudaMemset(p, 0, sizeof(g_bound_prof)));
  return KV_OK;
}
#endif
