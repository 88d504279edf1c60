// TF-IDF cosine index for the GFKB match path: the kv_index handle and its C ABI
// (include/kakveda_b200.h).  Device code lives in tfidf_kernels.cuh (scan, query preparation, merge) and
// bound_kernel.cuh (tensor-core chunk bounds); see there for the math and the HBM layout.  Host responsibilities: keep
// the append-only CSR, finalize (statistics on the device, (norm class, text) order of the rows and the column blocks
// on the host cores), per-batch query upload (text order of the queries, CSR -> device; tables are built by kernels)
// and kernel launches.
#include "block_builder.cuh"
#include "bound_kernel.cuh"

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
  DevBuf<uint32_t> d_ubt, d_rbloom, d_rt_keys, d_rt_off, d_rt_size;
  DevBuf<unsigned long long> d_rt_masks;
  CUtensorMap map_u;
  DevBuf<unsigned long long> d_ovf_keys;
  DevBuf<uint32_t> d_ovf_vals;
  int n_ovf = 0;
  int64_t n_rt_slots = 0;  // slots of all blocks' rare tables
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
  DevBuf<int> d_excl_sorted, d_excl_orig;  // self-join exclusions of the resident batch (by sorted slot / by original query)
  std::vector<int> h_excl_orig;
  bool has_excl = false;
  // row labels (kv_index_set_row_labels), by local row; dropped by an append.  On the device (rebuilt by every finalize):
  // by row, by scan position, the chunk label signatures and the first LAB_FIRST rows of every label
  std::vector<int> h_labels;
  bool has_labels = false, labels_on_device = false;
  DevBuf<int> d_labels_row, d_label_pos, d_lab_keys, d_lab_rows;
  DevBuf<unsigned long long> d_chunk_sig;
  int n_lab = 0;
  // label filter of the resident batch (kv_query_set_filter; by sorted slot / by original query), only while some
  // query is filtered
  DevBuf<int> d_filt_sorted, d_filt_orig;
  std::vector<int> h_filt_orig;
  bool has_filter = false;
  // row groups (kv_index_set_row_groups), by local row; dropped by an append.  On the device (rebuilt by every
  // finalize): by row (K5, fallbacks, null queries) and by scan position (scan).  Distinct mode of the resident batch
  // (kv_query_set_distinct), cleared by the next upload.
  std::vector<int> h_groups;
  bool has_groups = false, groups_on_device = false, distinct = false;
  DevBuf<int> d_groups_row, d_group_pos;
  // deleted rows (kv_index_delete_rows), by local row (empty until the first deletion; an append extends it).  They
  // keep their place in the scan layout.  On the device while any row is deleted, rebuilt by every finalize: by row,
  // the live word of every chunk (by scan position) and the first LAB_FIRST live rows (null queries)
  std::vector<uint8_t> h_dead;
  int64_t n_dead = 0;
  DevBuf<uint8_t> d_dead;
  DevBuf<uint32_t> d_alive, d_dcnt;
  DevBuf<int> d_dead_list, d_first_live;
  // threshold search over the resident batch (kv_range_resident): its own threshold array (not d_gthr, which peers push
  // into and a top-k raises), the pair buffer, the pair count, and the result until it is fetched
  DevBuf<int> d_rthr;
  DevBuf<RangePair> d_range;
  DevBuf<unsigned long long> d_range_count;
  bool range_valid = false;
  // the same on a Jaccard index (K3-R, kv_jaccard_range_resident): the records carry the exact counts and have a
  // result flag of their own, so kv_range_fetch never reads them
  DevBuf<JaccardPair> d_jrange;
  bool jrange_valid = false;
  int64_t range_q = 0, range_pairs = 0;
  RangeOrderScratch rsort;  // the fetches order the pairs on the device (range_order.cu)
  DevBuf<unsigned long long> d_stats;
  DevBuf<float> d_part_s, d_out_s;
  DevBuf<long long> d_part_r, d_out_r;
  PinnedBuf<float> h_out_s;
  PinnedBuf<long long> h_out_r;
  // single-query scratch
  PinnedBuf<unsigned char> h_qtab;
  DevBuf<unsigned char> d_qtab1;
  DevBuf<double> d_scores;

  // query batch currently resident on the device (kv_query_upload / first half of kv_topk)
  bool batch_valid = false;
  int64_t batch_q = 0, batch_tiles = 0, batch_h2d_bytes = 0, batch_null = 0, batch_f2_outside = 0;
  std::vector<int64_t> irr_q, irr_indptr;
  std::vector<uint32_t> irr_ids, irr_tf;
  std::vector<double> irr_oov;

  float *dbg_xs = nullptr;  // test hook (kv_debug_bound_numerators)
  float last_ms[4] = {0, 0, 0, 0};
  float last_prepare_ms[4] = {0, 0, 0, 0};  // host side of the last upload: staging, classification, text order, copies + table kernels
  float last_kernel_ms[5] = {0, 0, 0, 0, 0};  // bound pass 0, seed scan, bound pass 1, scan, merge
  float last_score_ms = 0;
  int64_t last_ctas = 0, last_tiles = 0, last_splits = 0, last_launches = 0;
  unsigned long long last_stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};

static void close_peers(kv_index *ix) {
  for (int i = 0; i < ix->n_peers; i++)
    if (ix->peer_gthr[i]) cudaIpcCloseMemHandle(ix->peer_gthr[i]);
  for (auto &p : ix->peer_gthr) p = nullptr;
  ix->n_peers = 0;
  ix->peer_cap = 0;
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
  int32_t jaccard, corpus_fit, threads, reserved;
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
  std::vector<uint32_t> ubt, rbloom, rt_off, rt_size, rt_keys;
  std::vector<unsigned long long> rt_masks, ovf_keys;
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
         f(L.rt_size, ix->d_rt_size, nb) && f(L.rt_keys, ix->d_rt_keys, slots) && f(L.rt_masks, ix->d_rt_masks, slots) &&
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
  ix->jrange_valid = false;
  // labels describe the rows they were given for: a filtered query fails until the rows are labelled again
  ix->h_labels.clear();
  ix->has_labels = ix->labels_on_device = false;
  ix->h_groups.clear();  // the same for groups: distinct mode fails until they are set again
  ix->has_groups = ix->groups_on_device = false;
  if (ix->n_dead) ix->h_dead.resize((size_t)ix->n_rows, 0);  // appended rows are live
  return KV_OK;
}

int kv_index_set_mode(kv_index *ix, int mode) {
  if (!ix || (mode != KV_MODE_TFIDF_COSINE && mode != KV_MODE_JACCARD && mode != KV_MODE_TFIDF_CORPUS_FIT))
    return kv_fail(KV_ERR_INVALID, "kv_index_set_mode: mode must be KV_MODE_TFIDF_COSINE, KV_MODE_JACCARD or KV_MODE_TFIDF_CORPUS_FIT");
  std::lock_guard<std::mutex> g(ix->mu);
  if (mode == KV_MODE_JACCARD && ix->n_dead)
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
  if (!ix->n_dead) return KV_OK;
  cudaStream_t s = ix->stream;
  std::vector<int> list;
  list.reserve((size_t)ix->n_dead);
  for (int64_t r = 0; r < ix->n_rows; r++)
    if (ix->h_dead[(size_t)r]) list.push_back((int)r);
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

// The device copies of the row labels for the current layout: by row (fallbacks), by scan position and as chunk
// signatures (scan and selection), and the first LAB_FIRST rows of every label (null queries).  Nothing to do until
// the index is finalized; every finalize calls it again.
static int upload_labels(kv_index *ix) {
  ix->labels_on_device = false;
  if (!ix->has_labels || !ix->finalized) return KV_OK;
  cudaStream_t s = ix->stream;
  const int64_t n = ix->n_rows, n_pos = ix->n_chunks_pad * CHUNK_ROWS;
  std::vector<int> keys(ix->h_labels);
  std::sort(keys.begin(), keys.end());
  keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
  std::vector<int> first(keys.size() * LAB_FIRST, -1), cnt(keys.size(), 0);
  for (int64_t r = 0; r < n; r++) {
    if (ix->n_dead && ix->h_dead[(size_t)r]) continue;  // null queries get live rows only
    const size_t i = (size_t)(std::lower_bound(keys.begin(), keys.end(), ix->h_labels[(size_t)r]) - keys.begin());
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
    KV_CUDA(ix->d_labels_row.ensure(n));
    KV_CUDA(ix->d_label_pos.ensure(n_pos));
    KV_CUDA(ix->d_chunk_sig.ensure(ix->n_chunks_pad));
    KV_CUDA(cudaMemcpyAsync(ix->d_labels_row.p, ix->h_labels.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    label_pos_kernel<<<(unsigned)((n_pos + 255) / 256), 256, 0, s>>>(ix->d_perm.p, ix->d_labels_row.p, n, n_pos, ix->d_label_pos.p);
    KV_CUDA(cudaGetLastError());
    chunk_sig_kernel<<<(unsigned)((ix->n_chunks_pad + 255) / 256), 256, 0, s>>>(ix->d_label_pos.p, ix->n_chunks_pad, ix->d_chunk_sig.p);
    KV_CUDA(cudaGetLastError());
  }
  KV_CUDA(cudaStreamSynchronize(s));  // the host staging vectors go out of scope
  ix->labels_on_device = true;
  return KV_OK;
}

static bool labels_ready(const kv_index *ix) {
  return ix->has_labels && ix->labels_on_device && (int64_t)ix->h_labels.size() == ix->n_rows;
}

// A filtered batch never runs on labels that do not describe the current rows
static int check_filter(const kv_index *ix, const char *fn) {
  if (ix->has_filter && !labels_ready(ix))
    return kv_fail(KV_ERR_STATE, "%s: the batch is filtered but the row labels are missing or stale (set them again after an append)", fn);
  return KV_OK;
}

int kv_index_set_row_labels(kv_index *ix, const int32_t *labels, int64_t n) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_labels: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!labels) {
    ix->h_labels.clear();
    ix->has_labels = ix->labels_on_device = false;
    return KV_OK;
  }
  if (n != ix->n_rows)
    return kv_fail(KV_ERR_INVALID, "kv_index_set_row_labels: %lld labels for an index of %lld rows", (long long)n,
                   (long long)ix->n_rows);
  for (int64_t i = 0; i < n; i++)
    if (labels[i] < 0) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_labels: label %d of row %lld is negative", labels[i], (long long)i);
  ix->h_labels.assign(labels, labels + n);
  ix->has_labels = true;
  KV_CUDA(cudaSetDevice(ix->device));
  return upload_labels(ix);
}

// The device copies of the row groups for the current layout: by row and by scan position.  Nothing to do until the
// index is finalized; every finalize calls it again.
static int upload_groups(kv_index *ix) {
  ix->groups_on_device = false;
  if (!ix->has_groups || !ix->finalized) return KV_OK;
  cudaStream_t s = ix->stream;
  const int64_t n = ix->n_rows, n_pos = ix->n_chunks_pad * CHUNK_ROWS;
  if (n > 0) {
    KV_CUDA(ix->d_groups_row.ensure(n));
    KV_CUDA(ix->d_group_pos.ensure(n_pos));
    KV_CUDA(cudaMemcpyAsync(ix->d_groups_row.p, ix->h_groups.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    label_pos_kernel<<<(unsigned)((n_pos + 255) / 256), 256, 0, s>>>(ix->d_perm.p, ix->d_groups_row.p, n, n_pos, ix->d_group_pos.p);
    KV_CUDA(cudaGetLastError());
    KV_CUDA(cudaStreamSynchronize(s));
  }
  ix->groups_on_device = true;
  return KV_OK;
}

// the per-row sets a finalize rebuilds on the device: labels and groups
static int upload_row_sets(kv_index *ix) {
  const int rc = upload_labels(ix);
  return rc != KV_OK ? rc : upload_groups(ix);
}

static bool groups_ready(const kv_index *ix) {
  return ix->has_groups && ix->groups_on_device && (int64_t)ix->h_groups.size() == ix->n_rows;
}

int kv_index_set_row_groups(kv_index *ix, const int32_t *groups, int64_t n) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_groups: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!groups) {
    ix->h_groups.clear();
    ix->has_groups = ix->groups_on_device = false;
    return KV_OK;
  }
  if (ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_groups: a Jaccard index (mode 1) has no distinct top-k");
  if (n != ix->n_rows)
    return kv_fail(KV_ERR_INVALID, "kv_index_set_row_groups: %lld groups for an index of %lld rows", (long long)n,
                   (long long)ix->n_rows);
  for (int64_t i = 0; i < n; i++)
    if (groups[i] < 0) return kv_fail(KV_ERR_INVALID, "kv_index_set_row_groups: group %d of row %lld is negative", groups[i], (long long)i);
  ix->h_groups.assign(groups, groups + n);
  ix->has_groups = true;
  KV_CUDA(cudaSetDevice(ix->device));
  return upload_groups(ix);
}

// The device copies of the deletions for the current layout (d_perm must hold it): deleted flags by row, the live word
// of every chunk and the first LAB_FIRST live rows.  Nothing while no row is deleted: the kernels then get NULL.
static int upload_dead(kv_index *ix) {
  if (!ix->n_dead || ix->n_rows == 0) return KV_OK;
  cudaStream_t s = ix->stream;
  const int64_t n = ix->n_rows;
  std::vector<int> first(LAB_FIRST, -1);
  for (int64_t r = 0, c = 0; r < n && c < LAB_FIRST; r++)
    if (!ix->h_dead[(size_t)r]) first[(size_t)c++] = (int)r;
  KV_CUDA(ix->d_dead.ensure(n));
  KV_CUDA(ix->d_alive.ensure(ix->n_chunks_pad));
  KV_CUDA(ix->d_first_live.ensure(LAB_FIRST));
  KV_CUDA(cudaMemcpyAsync(ix->d_dead.p, ix->h_dead.data(), (size_t)n, cudaMemcpyHostToDevice, s));
  KV_CUDA(cudaMemcpyAsync(ix->d_first_live.p, first.data(), first.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  alive_kernel<<<(unsigned)((ix->n_chunks_pad + 255) / 256), 256, 0, s>>>(ix->d_perm.p, ix->d_dead.p, n, ix->n_chunks_pad, ix->d_alive.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(s));  // the host list goes out of scope
  return KV_OK;
}

// NULL while no row is deleted: the kernels' per-row and per-chunk tests are then skipped
static const uint8_t *dead_rows(const kv_index *ix) { return ix->n_dead ? ix->d_dead.p : nullptr; }
static const uint32_t *alive_words(const kv_index *ix) { return ix->n_dead ? ix->d_alive.p : nullptr; }

int kv_index_delete_rows(kv_index *ix, const int64_t *rows, int64_t n) {
  if (!ix || n < 0 || (n > 0 && !rows)) return kv_fail(KV_ERR_INVALID, "kv_index_delete_rows: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_index_delete_rows: a Jaccard index (mode 1) has no row deletion");
  for (int64_t i = 0; i < n; i++)
    if (rows[i] < 0 || rows[i] >= ix->n_rows)
      return kv_fail(KV_ERR_INVALID, "kv_index_delete_rows: row %lld outside 0..%lld", (long long)rows[i], (long long)ix->n_rows - 1);
  int64_t added = 0;
  for (int64_t i = 0; i < n; i++) {
    if (ix->h_dead.empty()) ix->h_dead.assign((size_t)ix->n_rows, 0);
    uint8_t &d = ix->h_dead[(size_t)rows[i]];
    if (!d) { d = 1; added++; }
  }
  if (!added) return KV_OK;  // duplicates and rows deleted before: nothing changes
  ix->n_dead += added;
  // like an append: statistics and the device copies are stale until the next finalize
  ix->finalized = false;
  ix->batch_valid = ix->range_valid = ix->jrange_valid = false;
  return KV_OK;
}

int64_t kv_index_live_rows(const kv_index *ix) { return ix ? ix->n_rows - ix->n_dead : 0; }

int kv_index_deleted_rows(kv_index *ix, uint8_t *out, int64_t n) {
  if (!ix || n < 0 || (n > 0 && !out)) return kv_fail(KV_ERR_INVALID, "kv_index_deleted_rows: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (n != ix->n_rows)
    return kv_fail(KV_ERR_INVALID, "kv_index_deleted_rows: %lld flags for an index of %lld rows", (long long)n, (long long)ix->n_rows);
  if (ix->n_dead) memcpy(out, ix->h_dead.data(), (size_t)n);
  else if (n) memset(out, 0, (size_t)n);
  return KV_OK;
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
    ix->n_total = n - ix->n_dead;
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
      rownorm_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(ix->indptr.p, ix->ids.p, ix->tf.p, ix->d_perm.p, n,
                                                                      ix->d_bb64.p, ix->d_B64.p, ix->d_B32.p);
      KV_CUDA(cudaGetLastError());
      int rc = upload_dead(ix);
      if (rc != KV_OK) return rc;
      chunk_meta_kernel<<<(unsigned)((ix->n_chunks_pad + 255) / 256), 256, 0, s>>>(ix->d_B32.p, n, ix->n_chunks, ix->n_chunks_pad,
                                                                                    alive_words(ix), ix->d_cminB.p);
      KV_CUDA(cudaGetLastError());
      KV_CUDA(cudaStreamSynchronize(s));
      ix->V = V;
      ix->finalized = true;
      ix->batch_valid = ix->range_valid = ix->jrange_valid = false;
      ix->last_finalize_kind = 2;
      return upload_row_sets(ix);
    }
  }
  ix->layout_valid = false;
  // ---- on the host cores: (norm class, text) order of the rows, then the column blocks ----
  ScanLayout SL;
  sort_rows_by_text(ix->h_indptr, ix->h_ids, n, hB, SL.perm);
  {
    BlockLayout L;
    build_blocks(ix->h_indptr.data(), ix->h_ids.data(), ix->h_tf.data(), SL.perm.data(), n, V, ix->h_univ.data(),
                 ix->h_tfmax.data(), host_threads(), L);
    LayoutHeader &H = SL.H;
    H.n_rows = n; H.V = Vz; H.n_chunks = L.n_chunks; H.n_chunks_pad = L.n_chunks_pad; H.n_blocks = L.n_chunks_pad / 64;
    H.blk_words = L.total_words; H.n_entries = L.n_entries; H.n_rare_entries = L.n_rare_entries;
    H.n_rt_slots = (int64_t)L.rt_keys.size(); H.n_ovf = (int64_t)L.ovf.size(); H.univ_len = Vz;
    SL.univ = ix->h_univ;
    SL.fslot = std::move(L.fslot); SL.fslot2 = std::move(L.fslot2); SL.binfo = std::move(L.binfo); SL.uf = std::move(L.Uf);
    SL.ubt = std::move(L.Ubt); SL.rbloom = std::move(L.rbloom); SL.rt_off = std::move(L.rt_off); SL.rt_size = std::move(L.rt_size);
    SL.rt_keys = std::move(L.rt_keys); SL.rt_masks = std::move(L.rt_masks);
    SL.blk.reserve((size_t)L.total_words);
    for (auto &part : L.parts) {  // the blocks of each build thread, back to back
      SL.blk.insert(SL.blk.end(), part.begin(), part.end());
      std::vector<uint32_t>().swap(part);
    }
    for (const auto &o : L.ovf) { SL.ovf_keys.push_back(o.first); SL.ovf_vals.push_back(o.second); }
  }
  int rc = upload_layout(ix, SL);
  if (rc == KV_OK) rc = upload_dead(ix);
  if (rc != KV_OK) return rc;
  if (n) {
    rownorm_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(ix->indptr.p, ix->ids.p, ix->tf.p, ix->d_perm.p, n,
                                                                    ix->d_bb64.p, ix->d_B64.p, ix->d_B32.p);
    KV_CUDA(cudaGetLastError());
  }
  chunk_meta_kernel<<<(unsigned)((ix->n_chunks_pad + 255) / 256), 256, 0, s>>>(ix->d_B32.p, n, ix->n_chunks, ix->n_chunks_pad,
                                                                                alive_words(ix), ix->d_cminB.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(s));
  ix->V = V;
  ix->finalized = true;
  ix->batch_valid = ix->range_valid = ix->jrange_valid = false;
  ix->last_finalize_kind = 1;
  return upload_row_sets(ix);
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
// such a query takes the float64 full-scan path (K1a + selection).
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
        if (ix->h_univ[t]) continue;
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

static int prepare_batch_runs(kv_index *ix, const QueryRun *runs, int n_runs) {
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_topk: index not finalized");
  int64_t n_q = 0, nnz = 0;
  std::vector<int64_t> qb((size_t)n_runs + 1, 0), nb((size_t)n_runs + 1, 0);
  bool have_order = true, have_flags = true, any_order = false;
  for (int r = 0; r < n_runs; r++) {
    const QueryRun &R = runs[r];
    if (R.n_q < 0 || !R.indptr || !csr_ok(R.indptr, R.ids, R.tf, R.n_q)) return kv_fail(KV_ERR_INVALID, "kv_topk: bad query CSR");
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
  if (n_q < 1) return kv_fail(KV_ERR_INVALID, "kv_topk: empty query batch");
  if (n_q >= (1LL << 31) - TILE_Q) return kv_fail(KV_ERR_INVALID, "kv_topk: too many queries in one call");
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  ix->batch_valid = ix->range_valid = ix->jrange_valid = false;
  ix->has_excl = ix->has_filter = ix->distinct = false;
  ix->irr_q.clear(); ix->irr_indptr.assign(1, 0); ix->irr_ids.clear(); ix->irr_tf.clear(); ix->irr_oov.clear();
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
      const int64_t a = q_indptr[row], b = q_indptr[row + 1];
      ix->irr_q.push_back(q);
      ix->irr_ids.insert(ix->irr_ids.end(), q_ids + a, q_ids + b);
      ix->irr_tf.insert(ix->irr_tf.end(), q_tf + a, q_tf + b);
      ix->irr_indptr.push_back((int64_t)ix->irr_ids.size());
      ix->irr_oov.push_back(q_oov[row]);
    }
  }

  const int64_t n_tiles = (n_q + TILE_Q - 1) / TILE_Q;
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
  ix->batch_f2_outside = (int64_t)f2_out;
  ix->batch_q = n_q;
  ix->batch_tiles = n_tiles;
  ix->batch_null = n_null;
  ix->batch_h2d_bytes = (n_q + 1) * 8 + nnz * 8 + n_q * 8 + 3 * n_q * (int64_t)sizeof(int) + n_q;
  ix->batch_valid = true;
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
                                                              const uint8_t *univ, const uint32_t *tfmax, double amax,
                                                              uint8_t *flag) {
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
    if (univ[t]) continue;
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
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_topk: index not finalized");
  if (n_q < 1) return kv_fail(KV_ERR_INVALID, "kv_topk: empty query batch");
  if (n_q >= (1LL << 31) - TILE_Q) return kv_fail(KV_ERR_INVALID, "kv_topk: too many queries in one call");
  if (mirror_device(m) != ix->device)
    return kv_fail(KV_ERR_INVALID, "kv_query_upload_text: the vocabulary mirror is on device %d, the index on device %d",
                   mirror_device(m), ix->device);
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  ix->batch_valid = ix->range_valid = ix->jrange_valid = false;
  ix->has_excl = ix->has_filter = ix->distinct = false;
  ix->irr_q.clear(); ix->irr_indptr.assign(1, 0); ix->irr_ids.clear(); ix->irr_tf.clear(); ix->irr_oov.clear();
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
                                                     ix->d_df.p, ix->d_univ.p, ix->d_tfmax.p, amax, ix->d_qflag_row.p);
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
    for (int64_t i = 0; i < n_q; i++) {
      if (ix->h_flags.p[i] != 2) continue;
      const int64_t q = qperm[i], a = ix->h_q_indptr.p[q], b = ix->h_q_indptr.p[q + 1];
      const size_t at = ix->irr_ids.size();
      ix->irr_q.push_back(q);
      ix->irr_ids.resize(at + (size_t)(b - a));
      ix->irr_tf.resize(at + (size_t)(b - a));
      if (b > a) {
        KV_CUDA(cudaMemcpyAsync(ix->irr_ids.data() + at, ix->d_q_ids.p + a, (size_t)(b - a) * 4, cudaMemcpyDeviceToHost, s));
        KV_CUDA(cudaMemcpyAsync(ix->irr_tf.data() + at, ix->d_q_tf.p + a, (size_t)(b - a) * 4, cudaMemcpyDeviceToHost, s));
      }
      ix->irr_indptr.push_back((int64_t)ix->irr_ids.size());
      ix->irr_oov.push_back(ix->h_q_oov.p[q]);
    }
  }
  KV_CUDA(cudaStreamSynchronize(s));
  ix->batch_f2_outside = (int64_t)f2_out;
  ix->batch_q = n_q;
  ix->batch_tiles = (n_q + TILE_Q - 1) / TILE_Q;
  ix->batch_null = n_null;
  ix->batch_h2d_bytes = (offsets[n_q] - offsets[0]) + (n_q + 1) * 8 + n_null * (int64_t)sizeof(int);
  ix->batch_valid = true;
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
        ix->d_part_s.p, ix->d_part_r.p, (int)n_lists, b.n_q, b.k, b.n_q * b.k, ix->d_qperm.p, ix->d_groups_row.p, ix->row_base,
        b.out_s, b.out_r);
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
  SP.qtab = ix->d_qtab.p; SP.q_nq = qc; SP.q_dotU = qc + b.n_q; SP.q_corrU = qc + 2 * b.n_q;
  SP.q_excl = ix->has_excl ? ix->d_excl_sorted.p : nullptr; SP.gthr = b.range ? ix->d_rthr.p : ix->d_gthr.p;
  if (ix->has_filter) { SP.q_label = ix->d_filt_sorted.p; SP.label_pos = ix->d_label_pos.p; SP.chunk_sig = ix->d_chunk_sig.p; }
  SP.alive = alive_words(ix);
  for (int i = 0; i < 7; i++) SP.peer_gthr[i] = i < b.n_peers ? ix->peer_gthr[i] : nullptr;
  SP.n_peers = b.n_peers; SP.stats = ix->d_stats.p; SP.n_q = b.n_q; SP.k = b.k;
  SP.part_scores = ix->d_part_s.p; SP.part_rows = ix->d_part_r.p; SP.max_pages = b.max_pages;
  SP.qperm = ix->d_qperm.p; SP.range_out = ix->d_range.p; SP.range_count = ix->d_range_count.p;
  SP.range_cap = (unsigned long long)ix->d_range.cap;
  SP.group_pos = b.distinct ? ix->d_group_pos.p : nullptr;
  return SP;
}

// K1b-S (distinct or not), or K1b-R for a threshold search, over a grid of candidate lists
static int launch_scan(kv_index *ix, const Batch &b, const ScanParams &SP, dim3 grid) {
  if (b.range) tfidf_scan_kernel<true, false><<<grid, S_WARPS * 32, scan_smem_bytes(0), ix->stream>>>(SP);
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
  BP.rbloom = ix->d_rbloom.p; BP.rt_keys = ix->d_rt_keys.p; BP.rt_masks = ix->d_rt_masks.p; BP.rt_off = ix->d_rt_off.p;
  BP.rt_size = ix->d_rt_size.p; BP.tfmax = ix->d_tfmax.p;
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
// whole scan group at once.  A threshold search runs K3-R, which appends to d_jrange instead of filling lists.
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
    const JaccardRangeOut R{ix->d_qperm.p, ix->d_jrange.p, ix->d_range_count.p, (unsigned long long)ix->d_jrange.cap};
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
    return kv_fail(KV_ERR_INVALID, "kv_topk: index too large for one bound-kernel row range (max_pages %d)", b.max_pages);
  return KV_OK;
}

static int run_batch(kv_index *ix, int k, float *d_out_s, long long *d_out_r, int phase = 0) {
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_topk_resident: no query batch uploaded");
  if (k < 1 || k > 32) return kv_fail(KV_ERR_INVALID, "kv_topk: k must be 1..32");
  int rc = check_filter(ix, "kv_topk");
  if (rc != KV_OK) return rc;
  // the thresholds peers push are those of unfiltered queries: not a bound of a filtered query's k-th score
  if (ix->has_filter && (ix->gthr_exported || ix->n_peers))
    return kv_fail(KV_ERR_INVALID, "kv_topk: a label filter cannot be combined with the threshold exchange of a row-sharded GFKB");
  if (ix->distinct) {
    if (!groups_ready(ix))
      return kv_fail(KV_ERR_STATE, "kv_topk: the batch is distinct but the row groups are missing or stale (set them again after an append)");
    // a shard's seed k-th score is no lower bound of the global k-th GROUP score: one group can count on several shards
    if (phase != 0 || ix->gthr_exported || ix->n_peers)
      return kv_fail(KV_ERR_INVALID, "kv_topk: distinct mode cannot be combined with the two-phase top-k or the threshold exchange of a row-sharded GFKB");
  }
  ix->jrange_valid = false;
  KV_CUDA(cudaSetDevice(ix->device));
  cudaStream_t s = ix->stream;
  Batch b;
  b.k = k; b.phase = phase; b.out_s = d_out_s; b.out_r = d_out_r; b.distinct = ix->distinct;
  rc = size_batch(ix, b);
  if (rc != KV_OK) return rc;
  const int64_t n_q = b.n_q;
  const bool prune = b.prune;
  if (n_q > ix->d_gthr.cap && (ix->gthr_exported || ix->n_peers))
    return kv_fail(KV_ERR_STATE, "kv_topk: the query batch outgrew the threshold array shared with the peer GPUs; exchange it again "
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
        ix->has_filter ? ix->d_filt_orig.p : nullptr, ix->d_labels_row.p, dead_rows(ix), ix->d_groups_row.p, d_out_s, d_out_r);
    KV_CUDA(cudaGetLastError());
    b.launches++;
  } else if (ix->batch_null) {
    const LabelFirstRows L{ix->d_lab_keys.p, ix->d_lab_rows.p, ix->n_lab};
    fill_null_kernel<<<(unsigned)((ix->batch_null * k + 255) / 256), 256, 0, s>>>(ix->d_qperm.p + n_q, (int)ix->batch_null, k,
                                                                                  ix->n_rows, ix->row_base,
                                                                                  ix->has_excl ? ix->d_excl_orig.p : nullptr,
                                                                                  ix->has_filter ? ix->d_filt_orig.p : nullptr, L,
                                                                                  ix->n_dead ? ix->d_first_live.p : nullptr, d_out_s, d_out_r);
    KV_CUDA(cudaGetLastError());
    b.launches++;
  }
  for (size_t i = 0; i < ix->irr_q.size(); i++) {
    const int64_t q = ix->irr_q[i], a = ix->irr_indptr[i], e = ix->irr_indptr[i + 1];
    rc = score_impl(ix, ix->irr_ids.data() + a, ix->irr_tf.data() + a, e - a, ix->irr_oov[i], nullptr);
    if (rc != KV_OK) return rc;
    if (b.distinct)
      select_topk_distinct_kernel<<<1, 1024, 0, s>>>(ix->d_scores.p, ix->n_rows, ix->row_base, k,
                                                     ix->has_excl ? (int64_t)ix->h_excl_orig[(size_t)q] : -1, ix->d_labels_row.p,
                                                     ix->has_filter ? ix->h_filt_orig[(size_t)q] : -1, dead_rows(ix),
                                                     ix->d_groups_row.p, d_out_s + q * k, d_out_r + q * k);
    else
      select_topk_kernel<<<1, 1024, 0, s>>>(ix->d_scores.p, ix->n_rows, ix->row_base, k,
                                            ix->has_excl ? (int64_t)ix->h_excl_orig[(size_t)q] : -1, ix->d_labels_row.p,
                                            ix->has_filter ? ix->h_filt_orig[(size_t)q] : -1, dead_rows(ix), d_out_s + q * k,
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
    return kv_fail(KV_ERR_NOMEM, "kv_topk: the candidate pool (%lld pages) is exhausted; split the query batch",
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

// Threshold search over the resident batch: every pair with score >= thr lands in d_range (d_jrange on a Jaccard
// index), *n_pairs = their count.  When they do not fit, the buffer grows to the exact count and only the scan and the
// fallbacks run again (the candidate lists depend on the threshold alone).  Events: evk[2] -> evk[3] bound pass 1,
// evk[3] -> evk[4] scan, evk[4] -> evk[5] irregular-query fallbacks.  `fn` names the caller in error messages.
// Caller holds ix->mu.
static int run_range(kv_index *ix, float thr, int64_t *n_pairs, const char *fn) {
  ix->range_valid = ix->jrange_valid = false;
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
  if (jac) KV_CUDA(ix->d_jrange.ensure(65536));
  else KV_CUDA(ix->d_range.ensure(65536));
  auto range_cap = [&] { return (unsigned long long)(jac ? ix->d_jrange.cap : ix->d_range.cap); };
  KV_CUDA(ix->d_range_count.ensure(1));
  for (auto &e : ix->evk) KV_CUDA(cudaEventRecord(e, s));
  KV_CUDA(cudaMemsetAsync(ix->d_stats.p, 0, 8 * sizeof(unsigned long long), s));
  KV_CUDA(cudaMemsetAsync(ix->d_range_count.p, 0, sizeof(unsigned long long), s));
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
      for (size_t i = 0; i < ix->irr_q.size(); i++) {
        const int64_t q = ix->irr_q[i], a = ix->irr_indptr[i], e = ix->irr_indptr[i + 1];
        rc = score_impl(ix, ix->irr_ids.data() + a, ix->irr_tf.data() + a, e - a, ix->irr_oov[i], nullptr);
        if (rc != KV_OK) return rc;
        const unsigned grid = (unsigned)std::min<int64_t>((ix->n_rows + 255) / 256, 8LL * ix->sm_count);
        const int64_t excl = ix->has_excl ? (int64_t)ix->h_excl_orig[(size_t)q] : -1;
        if (jac) {
          const double nq = host_query_norm(ix, ix->irr_ids.data() + a, ix->irr_tf.data() + a, e - a, ix->irr_oov[i]);  // |q|
          jaccard_select_range_kernel<<<grid, 256, 0, s>>>(ix->d_scores.p, ix->d_B64.p, ix->d_invperm.p, ix->n_rows, nq, thr, excl,
                                                           (int)q, ix->d_jrange.p, ix->d_range_count.p, range_cap());
        } else {
          select_range_kernel<<<grid, 256, 0, s>>>(ix->d_scores.p, ix->n_rows, ix->row_base, thr, excl, ix->d_labels_row.p,
                                                   ix->has_filter ? ix->h_filt_orig[(size_t)q] : -1, dead_rows(ix), (int)q, ix->d_range.p,
                                                   ix->d_range_count.p, range_cap());
        }
        KV_CUDA(cudaGetLastError());
        b.launches += 2;
      }
      KV_CUDA(cudaEventRecord(ix->evk[5], s));
      KV_CUDA(cudaMemcpyAsync(&count, ix->d_range_count.p, sizeof(count), cudaMemcpyDeviceToHost, s));
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
      if ((jac ? ix->d_jrange.ensure((int64_t)count) : ix->d_range.ensure((int64_t)count)) != cudaSuccess) {
        cudaGetLastError();
        return kv_fail(KV_ERR_NOMEM, "%s: %llu pairs reach the threshold; their buffer does not fit in device memory "
                                     "(raise the threshold or split the query batch)", fn, count);
      }
      // the counters describe one run: the bound pass's stay, the scan's start again
      KV_CUDA(cudaMemsetAsync(ix->d_stats.p, 0, 2 * sizeof(unsigned long long), s));
      KV_CUDA(cudaMemsetAsync(ix->d_range_count.p, 0, sizeof(unsigned long long), s));
    }
  } else {
    for (auto &st : ix->last_stats) st = 0;
  }
  for (int i = 0; i < 5; i++) ix->last_kernel_ms[i] = ms[i];
  ix->last_launches = b.launches;
  ix->range_q = n_q;
  ix->range_pairs = (int64_t)count;
  (jac ? ix->jrange_valid : ix->range_valid) = true;
  *n_pairs = (int64_t)count;
  return KV_OK;
}

static int topk_impl(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                     const double *q_oov, int64_t n_q, int k, float *h_scores, int64_t *h_rows, void *d_scores_out,
                     void *d_rows_out) {
  if (!ix || n_q < 0 || k < 1 || k > 32 || (n_q > 0 && !q_indptr))
    return kv_fail(KV_ERR_INVALID, "kv_topk: bad arguments (k must be 1..32)");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->finalized) return kv_fail(KV_ERR_STATE, "kv_topk: index not finalized");
  if (n_q == 0) return KV_OK;
  int rc = prepare_batch(ix, q_indptr, q_ids, q_tf, q_oov, n_q);
  if (rc != KV_OK) return rc;
  cudaStream_t s = ix->stream;
  float *d_out_s = (float *)d_scores_out;
  long long *d_out_r = (long long *)d_rows_out;
  if (!d_out_s) {
    KV_CUDA(ix->d_out_s.ensure(n_q * k)); KV_CUDA(ix->d_out_r.ensure(n_q * k));
    d_out_s = ix->d_out_s.p; d_out_r = ix->d_out_r.p;
  }
  rc = run_batch(ix, k, d_out_s, d_out_r);
  if (rc != KV_OK) return rc;
  if (h_scores) {
    KV_CUDA(ix->h_out_s.ensure(n_q * k)); KV_CUDA(ix->h_out_r.ensure(n_q * k));
    KV_CUDA(cudaMemcpyAsync(ix->h_out_s.p, d_out_s, (size_t)n_q * k * sizeof(float), cudaMemcpyDeviceToHost, s));
    KV_CUDA(cudaMemcpyAsync(ix->h_out_r.p, d_out_r, (size_t)n_q * k * sizeof(long long), cudaMemcpyDeviceToHost, s));
  }
  KV_CUDA(cudaEventRecord(ix->ev[4], s));
  KV_CUDA(cudaStreamSynchronize(s));
  if (h_scores) {
    memcpy(h_scores, ix->h_out_s.p, (size_t)n_q * k * sizeof(float));
    memcpy(h_rows, ix->h_out_r.p, (size_t)n_q * k * sizeof(int64_t));
  }
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
  if (ix->n_dead) {  // a deleted row's query is switched off (flag 3): no path answers it, its list stays (-inf, -1)
    flags.resize((size_t)n);
    classify_queries(ix, ip.data(), R.ids, R.tf, n, flags.data(), host_threads());
    for (int64_t i = 0; i < n; i++)
      if (ix->h_dead[(size_t)(q_begin + i)]) flags[(size_t)i] = 3;
    R.flags = flags.data();
  }
  int rc = prepare_batch_runs(ix, &R, 1);
  if (rc != KV_OK) return rc;
  for (int64_t i = 0; i < n; i++) ex[(size_t)i] = ix->row_base + q_begin + i;
  return set_exclusions_locked(ix, ex.data(), n);
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
  // |q|^2 exactly as K1a gets it (prep_query, float64)
  std::vector<double> cst((size_t)n_q);
  std::vector<int64_t> ip((size_t)n_q + 1);
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
  KV_CUDA(cudaMemcpyAsync(ix->d_rq_rows.p, rows, (size_t)n_q * k * 8, cudaMemcpyHostToDevice, s));
  RescoreParams P;
  P.indptr = ix->indptr.p; P.ids = ix->ids.p; P.tf = ix->tf.p;
  P.a64 = ix->d_a64.p; P.d64 = ix->d_d64.p; P.B64 = ix->d_B64.p; P.invperm = ix->d_invperm.p;
  P.q_indptr = ix->d_rq_indptr.p; P.q_ids = ix->d_rq_ids.p; P.q_tf = ix->d_rq_tf.p;
  P.q_nq = ix->d_rq_const.p;
  P.rows = ix->d_rq_rows.p; P.n_q = n_q; P.n_rows = ix->n_rows; P.row_base = ix->row_base; P.V = ix->V;
  P.k = k; P.jaccard = ix->jaccard; P.dead = dead_rows(ix); P.out = ix->d_rq_out.p;
  rescore_kernel<<<(unsigned)((n_q * k * 32 + 255) / 256), 256, 0, s>>>(P);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaMemcpyAsync(out_scores, ix->d_rq_out.p, (size_t)n_q * k * 8, cudaMemcpyDeviceToHost, s));
  KV_CUDA(cudaStreamSynchronize(s));
  return KV_OK;
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
  if (!labels_ready(ix))
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

int kv_query_set_distinct(kv_index *ix, int on) {
  if (!ix) return kv_fail(KV_ERR_INVALID, "kv_query_set_distinct: NULL handle");
  std::lock_guard<std::mutex> g(ix->mu);
  if (on && ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_query_set_distinct: a Jaccard index (mode 1) has no distinct top-k");
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_query_set_distinct: no query batch uploaded");
  ix->distinct = false;
  if (!on) return KV_OK;
  if (!groups_ready(ix))
    return kv_fail(KV_ERR_STATE, "kv_query_set_distinct: the index has no row groups for its current rows (kv_index_set_row_groups)");
  ix->distinct = true;
  return KV_OK;
}

int kv_topk_resident_host(kv_index *ix, int k, float *out_scores, int64_t *out_rows) {
  if (!ix || !out_scores || !out_rows) return kv_fail(KV_ERR_INVALID, "kv_topk_resident_host: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->batch_valid) return kv_fail(KV_ERR_STATE, "kv_topk_resident_host: no query batch uploaded");
  if (k < 1 || k > 32) return kv_fail(KV_ERR_INVALID, "kv_topk: k must be 1..32");
  const int64_t n_q = ix->batch_q;
  KV_CUDA(cudaSetDevice(ix->device));
  KV_CUDA(ix->d_out_s.ensure(n_q * k)); KV_CUDA(ix->d_out_r.ensure(n_q * k));
  int rc = run_batch(ix, k, ix->d_out_s.p, ix->d_out_r.p);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaMemcpyAsync(out_scores, ix->d_out_s.p, (size_t)n_q * k * sizeof(float), cudaMemcpyDeviceToHost, ix->stream));
  KV_CUDA(cudaMemcpyAsync(out_rows, ix->d_out_r.p, (size_t)n_q * k * sizeof(long long), cudaMemcpyDeviceToHost, ix->stream));
  KV_CUDA(cudaEventRecord(ix->ev[4], ix->stream));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return finish_batch(ix);
}

int kv_range_resident(kv_index *ix, float threshold, int64_t *n_pairs) {
  if (!ix || !n_pairs) return kv_fail(KV_ERR_INVALID, "kv_range_resident: bad arguments");
  if (!(threshold > 0.f && threshold <= 1.f)) return kv_fail(KV_ERR_INVALID, "kv_range_resident: threshold must be in (0, 1]");
  std::lock_guard<std::mutex> g(ix->mu);
  if (ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_range_resident: a Jaccard index searches with kv_jaccard_range_resident");
  return run_range(ix, threshold, n_pairs, "kv_range_resident");
}

int kv_jaccard_range_resident(kv_index *ix, float threshold, int64_t *n_pairs) {
  if (!ix || !n_pairs) return kv_fail(KV_ERR_INVALID, "kv_jaccard_range_resident: bad arguments");
  if (!(threshold > 0.f && threshold <= 1.f))
    return kv_fail(KV_ERR_INVALID, "kv_jaccard_range_resident: threshold must be in (0, 1]");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_jaccard_range_resident: not a Jaccard index (kv_range_resident)");
  return run_range(ix, threshold, n_pairs, "kv_jaccard_range_resident");
}

// The pairs come back in emit order, which the scan does not fix; scores are exact integer sums rounded once, so
// (score desc, row asc) is a total order of each query's pairs and the result is deterministic.  Both fetches order the
// pairs on the device (range_order.cu, in the pair buffer itself: the fetch consumes the result) and copy the ordered
// arrays back.  Once ordering has started the result is gone whatever happens; a scratch allocation that fails first
// (KV_ERR_NOMEM) leaves it for another try.
int kv_range_fetch(kv_index *ix, int64_t *indptr, int64_t *rows, float *scores) {
  if (!ix || !indptr) return kv_fail(KV_ERR_INVALID, "kv_range_fetch: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->range_valid) return kv_fail(KV_ERR_STATE, "kv_range_fetch: no threshold search result (kv_range_resident first)");
  const int64_t n_q = ix->range_q, n = ix->range_pairs;
  if (n > 0 && (!rows || !scores)) return kv_fail(KV_ERR_INVALID, "kv_range_fetch: bad arguments");
  KV_CUDA(cudaSetDevice(ix->device));
  const int rc = range_order_to_host(ix->d_range.p, n, n_q, 0, indptr, rows, scores, nullptr, nullptr, ix->rsort, ix->stream,
                                     "kv_range_fetch");
  if (rc != KV_ERR_NOMEM) ix->range_valid = false;
  return rc;
}

// Same order as kv_range_fetch: the score is inter / union rounded to float32, and equal scores order by row.
int kv_jaccard_range_fetch(kv_index *ix, int64_t *indptr, int64_t *rows, float *scores, int32_t *inter, int32_t *uni) {
  if (!ix || !indptr) return kv_fail(KV_ERR_INVALID, "kv_jaccard_range_fetch: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->jaccard) return kv_fail(KV_ERR_INVALID, "kv_jaccard_range_fetch: not a Jaccard index (kv_range_fetch)");
  if (!ix->jrange_valid)
    return kv_fail(KV_ERR_STATE, "kv_jaccard_range_fetch: no threshold search result (kv_jaccard_range_resident first)");
  const int64_t n_q = ix->range_q, n = ix->range_pairs;
  if (n > 0 && (!rows || !scores || !inter || !uni)) return kv_fail(KV_ERR_INVALID, "kv_jaccard_range_fetch: bad arguments");
  KV_CUDA(cudaSetDevice(ix->device));
  const int rc = range_order_to_host(ix->d_jrange.p, n, n_q, ix->row_base, indptr, rows, scores, inter, uni, ix->rsort,
                                     ix->stream, "kv_jaccard_range_fetch");
  if (rc != KV_ERR_NOMEM) ix->jrange_valid = false;
  return rc;
}

// Device outputs: the same arrays, written to caller-owned device memory of the index's device.
int kv_range_fetch_device(kv_index *ix, void *d_indptr, void *d_rows, void *d_scores) {
  const char *fn = "kv_range_fetch_device";
  if (!ix) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  if (ix->jaccard) return kv_fail(KV_ERR_INVALID, "%s: a Jaccard index fetches with kv_jaccard_range_fetch_device", fn);
  if (!ix->range_valid) return kv_fail(KV_ERR_STATE, "%s: no threshold search result (kv_range_resident first)", fn);
  const int64_t n_q = ix->range_q, n = ix->range_pairs;
  int rc = check_device_ptr(d_indptr, ix->device, 8, "indptr", fn);
  if (rc == KV_OK && n > 0) rc = check_device_ptr(d_rows, ix->device, 8, "rows", fn);
  if (rc == KV_OK && n > 0) rc = check_device_ptr(d_scores, ix->device, 4, "scores", fn);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaSetDevice(ix->device));
  rc = range_order_device(ix->d_range.p, n, n_q, 0, (int64_t *)d_indptr, (int64_t *)d_rows, (float *)d_scores, nullptr, nullptr,
                          ix->rsort, ix->stream, fn);
  if (rc != KV_ERR_NOMEM) ix->range_valid = false;
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return KV_OK;
}

int kv_jaccard_range_fetch_device(kv_index *ix, void *d_indptr, void *d_rows, void *d_scores, void *d_inter, void *d_uni) {
  const char *fn = "kv_jaccard_range_fetch_device";
  if (!ix) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  std::lock_guard<std::mutex> g(ix->mu);
  if (!ix->jaccard) return kv_fail(KV_ERR_INVALID, "%s: not a Jaccard index (kv_range_fetch_device)", fn);
  if (!ix->jrange_valid) return kv_fail(KV_ERR_STATE, "%s: no threshold search result (kv_jaccard_range_resident first)", fn);
  const int64_t n_q = ix->range_q, n = ix->range_pairs;
  int rc = check_device_ptr(d_indptr, ix->device, 8, "indptr", fn);
  if (rc == KV_OK && n > 0) rc = check_device_ptr(d_rows, ix->device, 8, "rows", fn);
  if (rc == KV_OK && n > 0) rc = check_device_ptr(d_scores, ix->device, 4, "scores", fn);
  if (rc == KV_OK && n > 0) rc = check_device_ptr(d_inter, ix->device, 4, "inter", fn);
  if (rc == KV_OK && n > 0) rc = check_device_ptr(d_uni, ix->device, 4, "uni", fn);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaSetDevice(ix->device));
  rc = range_order_device(ix->d_jrange.p, n, n_q, ix->row_base, (int64_t *)d_indptr, (int64_t *)d_rows, (float *)d_scores,
                          (int32_t *)d_inter, (int32_t *)d_uni, ix->rsort, ix->stream, fn);
  if (rc != KV_ERR_NOMEM) ix->jrange_valid = false;
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return KV_OK;
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

int kv_topk_resident(kv_index *ix, int k, void *d_scores, void *d_rows) {
  if (!ix || !d_scores || !d_rows) return kv_fail(KV_ERR_INVALID, "kv_topk_resident: bad arguments");
  std::lock_guard<std::mutex> g(ix->mu);
  int rc = run_batch(ix, k, (float *)d_scores, (long long *)d_rows);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaEventRecord(ix->ev[4], ix->stream));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return finish_batch(ix);
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
  int rc = run_batch(ix, k, (float *)d_scores, (long long *)d_rows, 2);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaEventRecord(ix->ev[4], ix->stream));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  return finish_batch(ix);
}

int kv_topk(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
            const double *q_oov_tf2, int64_t n_q, int k, float *out_scores, int64_t *out_rows) {
  if (n_q > 0 && (!out_scores || !out_rows)) return kv_fail(KV_ERR_INVALID, "kv_topk: output buffers are NULL");
  return topk_impl(ix, q_indptr, q_ids, q_tf, q_oov_tf2, n_q, k, out_scores, out_rows, nullptr, nullptr);
}

int kv_topk_device(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                   const double *q_oov_tf2, int64_t n_q, int k, void *d_scores, void *d_rows) {
  if (n_q > 0 && (!d_scores || !d_rows)) return kv_fail(KV_ERR_INVALID, "kv_topk_device: output buffers are NULL");
  return topk_impl(ix, q_indptr, q_ids, q_tf, q_oov_tf2, n_q, k, nullptr, nullptr, d_scores, d_rows);
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
  KV_CUDA(ix->d_out_s.ensure(n_q * k)); KV_CUDA(ix->d_out_r.ensure(n_q * k));
  ix->dbg_xs = xs.p;
  int rc = run_batch(ix, k, ix->d_out_s.p, ix->d_out_r.p);
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
  KV_CUDA(ix->d_out_s.ensure(n_q * k)); KV_CUDA(ix->d_out_r.ensure(n_q * k));
  int rc = run_batch(ix, k, ix->d_out_s.p, ix->d_out_r.p);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaEventRecord(ix->ev[4], ix->stream));
  KV_CUDA(cudaStreamSynchronize(ix->stream));
  if ((rc = finish_batch(ix)) != KV_OK) return rc;
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

int kv_index_layout(const kv_index *ix, int64_t bytes[4], int64_t counts[18]) {
  if (!ix || !bytes || !counts) return kv_fail(KV_ERR_INVALID, "kv_index_layout: bad arguments");
  bytes[0] = ix->blk_words * 4;
  bytes[1] = ix->n_rows * 4;
  bytes[2] = ix->n_chunks_pad * (int64_t)sizeof(BlockInfo);
  const int64_t rare_table_bytes = ix->n_rt_slots * 12 + (ix->n_chunks_pad / 64) * (RB_BITS / 8);
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
constexpr uint64_t LAYOUT_MAGIC = 0x32594C42564B4B41ULL;  // "AKKVBLY2"

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
  H.n_rt_slots = ix->n_rt_slots; H.n_blocks = ix->n_chunks_pad / 64; H.univ_len = (int64_t)ix->layout_univ.size();
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
  ix->labels_on_device = ix->groups_on_device = false;  // positions changed: the finalize that follows rebuilds them
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
