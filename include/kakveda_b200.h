/*
 * kakveda_b200 -- C ABI of the H100-native GFKB fingerprint-match engine.
 *
 * The reference (prateekdevisingh/kakveda) is pure Python and has no FFI for this path;
 * its one similarity entry point is the method
 *     SimilarityEngine.score(self, query: str, corpus: List[str]) -> List[float]
 *                                      (services/shared/similarity.py:14-20)
 * called from the GFKB match handler (services/gfkb/app.py:86) which then takes a stable
 * top-5 (services/gfkb/app.py:89-91).  The entry points below are what a ctypes shim
 * backing that class binds (see INTEGRATION.md); each one names the reference code it
 * replaces.  Conventions: every function returns an int status (KV_OK == 0), the caller
 * owns every buffer it passes in, no callbacks, plain pointers and sizes only.  A handle
 * may be used from several threads (calls on one handle serialise on an internal mutex;
 * device work runs on the handle's own CUDA stream).
 */
#ifndef KAKVEDA_B200_H
#define KAKVEDA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KV_OK 0
#define KV_ERR_INVALID 1     /* bad argument / size limit exceeded              */
#define KV_ERR_CUDA 2        /* CUDA runtime error or no usable device          */
#define KV_ERR_EMPTY_VOCAB 3 /* sklearn's "empty vocabulary" ValueError         */
#define KV_ERR_NOMEM 4
#define KV_ERR_NONASCII 5    /* raw-text featurizer met a non-ASCII byte: the   */
                             /* caller must pre-tokenise that document itself   */
#define KV_ERR_STATE 6       /* call order violated (e.g. query before finalize)*/

/* Thread-local text of the last error raised on the calling thread ("" if none). */
const char *kv_last_error(void);
/* Library version string, and compile-time facts for the loader test. */
const char *kv_version(void);
/* Number of visible CUDA devices (0 when there is no driver/GPU); never fails. */
int kv_device_count(void);

/* ------------------------------------------------------------------------------------
 * Host featuriser: replaces TfidfVectorizer's analyzer + vocabulary
 * (sklearn/feature_extraction/text.py:1257 _count_vocab, :248 _word_ngrams, token
 * pattern (?u)\b\w\w+\b :1969, lowercase=True) as used by similarity.py:17-18.
 * Features are word 1-grams and 2-grams; a vocabulary maps feature -> dense uint32 id
 * (identity by a 128-bit hash of the feature bytes).
 * ---------------------------------------------------------------------------------- */
typedef struct kv_vocab kv_vocab;
typedef struct kv_csr kv_csr;

int kv_vocab_create(kv_vocab **out);
void kv_vocab_destroy(kv_vocab *v);
int64_t kv_vocab_size(const kv_vocab *v);

/* Persistence of a vocabulary (binary sidecar of failures.jsonl, so that a cold start does not re-tokenise the GFKB):
 * export writes the 128-bit key of every feature in id order (keys_out[2*id], keys_out[2*id+1]; capacity counts
 * features); import fills an EMPTY vocabulary so that feature id i has keys[2*i..2*i+1] again -- documents
 * featurised afterwards get the ids they had, new features continue the numbering. */
int kv_vocab_export(const kv_vocab *v, uint64_t *keys_out, int64_t capacity);
int kv_vocab_import(kv_vocab *v, const uint64_t *keys, int64_t n);

#define KV_TEXT_RAW_ASCII 0 /* docs are raw ASCII text: lower-cased + tokenised here       */
#define KV_TEXT_TOKENS 1    /* docs are tokens already lower-cased, separated by 0x1F (any  */
                            /* UTF-8): used by the Python shim for non-ASCII documents      */
#define KV_TEXT_MIXED 2     /* per document: a leading 0x1F byte marks a KV_TEXT_TOKENS     */
                            /* document (the marker is skipped), anything else is raw ASCII */

/* Featurise n_docs documents stored back to back in `bytes`; document i occupies
 * bytes[offsets[i] .. offsets[i+1]).  grow != 0 adds unseen features to the vocabulary
 * (corpus rows); grow == 0 leaves it untouched and reports, per document, the sum of
 * tf^2 over out-of-vocabulary features (needed for the query norm: such features have
 * corpus df == 0).  n_threads <= 0 picks hardware concurrency.  On KV_ERR_NONASCII
 * *bad_doc (if non-NULL) is the index of the first offending document. */
int kv_featurize(kv_vocab *v, const char *bytes, const int64_t *offsets, int64_t n_docs,
                 int mode, int grow, int n_threads, kv_csr **out, int64_t *bad_doc);

/* Borrow the arrays of a featurised batch (valid until kv_csr_destroy):
 * indptr[n_docs+1], ids[nnz], tf[nnz], oov_tf2[n_docs]. */
int kv_csr_view(const kv_csr *c, int64_t *n_docs, const int64_t **indptr, const uint32_t **ids,
                const uint32_t **tf, const double **oov_tf2);
void kv_csr_destroy(kv_csr *c);

/* Host-only helpers for sharding a GFKB by TEXT RANGE (kakveda_b200/dist.py, order="text"; no device involved):
 * kv_text_order: perm_out[i] = the row at position i when the rows are sorted by their feature-id sequence (the
 * text order the scan layout uses; equal rows by row index).  kv_csr_gather_rows: copy the rows `rows[0..n_sel)` of a
 * CSR into out_* (out_indptr[n_sel+1] prepared by the caller from the row lengths). */
int kv_text_order(const int64_t *indptr, const uint32_t *ids, int64_t n_rows, int32_t *perm_out, int n_threads);
int kv_csr_gather_rows(const int64_t *indptr, const uint32_t *ids, const uint32_t *tf, int64_t n_rows, const int64_t *rows,
                       int64_t n_sel, const int64_t *out_indptr, uint32_t *out_ids, uint32_t *out_tf, int n_threads);

/* ------------------------------------------------------------------------------------
 * TF-IDF cosine index (kernels K1a/K1b/K5): replaces the arithmetic of
 * SimilarityEngine.score -- TfidfTransformer.fit/transform (sklearn text.py:1650-1739),
 * cosine_similarity (sklearn/metrics/pairwise.py:1742-1752) -- with a resident, row-
 * sharded device index.  Rows are appended as CSR over vocabulary ids (append-only like
 * data/failures.jsonl, services/gfkb/app.py:49-51,132,146), then finalize() rebuilds the
 * query-independent statistics (df, idf tables, row norms) and the scan layout.
 * ---------------------------------------------------------------------------------- */
typedef struct kv_index kv_index;

/* device: CUDA ordinal.  row_base: global index of this shard's first row (row ids
 * reported by top-k are row_base + local row). */
int kv_index_create(int device, int64_t row_base, kv_index **out);
void kv_index_destroy(kv_index *ix);

int kv_index_append(kv_index *ix, const int64_t *indptr, const uint32_t *ids, const uint32_t *tf,
                    int64_t n_rows);

/* K3: switch the index to token-set Jaccard before finalize (default KV_MODE_TFIDF_COSINE).  Rows and
 * queries are then token-id SETS (every tf = 1; the id space is whatever the caller's vocabulary is),
 * score = |q ∩ row| / |q ∪ row| (0 for two empty sets).  The reference has no Jaccard path (its docs
 * list it as a possible measure, docs/failure-intelligence.md:43-46): parity UNPINNED, oracle = Python
 * sets.  kv_topk then ranks by float32 inter/union; kv_jaccard_counts returns the exact integers of the
 * selected pairs so that the caller can form the float64 ratio bit-exactly. */
#define KV_MODE_TFIDF_COSINE 0
#define KV_MODE_JACCARD 1
/* TF-IDF cosine with the vectoriser fitted on the corpus ALONE (idf = ln((1+N)/(1+df))+1 for both sides; query
 * features outside the vocabulary are ignored) -- sklearn's usual fit(corpus)/transform(query).  Symmetric, so it
 * is the measure of the all-pairs self-join that feeds pattern clustering (BASELINE configs[3]; the reference's
 * pattern_detector groups by failure_type only, services/pattern_detector/app.py:28-60 -- extension, oracle =
 * cosine_similarity(TfidfVectorizer(ngram_range=(1,2)).fit_transform(corpus))). */
#define KV_MODE_TFIDF_CORPUS_FIT 2
int kv_index_set_mode(kv_index *ix, int mode);
int kv_jaccard_counts(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const double *q_oov_tf2,
                      int64_t n_q, int k, const int64_t *rows, int32_t *out_inter, int32_t *out_union);

/* Optional, before finalize, for a corpus sharded over several GPUs: the GLOBAL document
 * frequency per feature id and the GLOBAL row count (else both come from the local rows). */
int kv_index_set_global_df(kv_index *ix, const uint32_t *df, int64_t vocab_size, int64_t n_rows_global);

/* Copy out the LOCAL document frequencies (length vocab_size) -- what a rank contributes
 * to the df all-reduce of a sharded corpus.  Valid after append, before or after finalize. */
int kv_index_local_df(kv_index *ix, uint32_t *df_out, int64_t vocab_size);

int kv_index_finalize(kv_index *ix, int64_t vocab_size);
/* What the last finalize did: 1 = full rebuild (text sort of the rows, scan stream, chunk summaries), 2 =
 * statistics-only refresh (the rows of THIS index are unchanged since its last full rebuild and only the global N /
 * df moved -- rows were appended to another shard or to the tail segment of a resident GFKB: idf tables, row norms
 * and chunk minima are recomputed on the device, nothing is re-sorted), 0 = never finalized. */
int kv_index_last_finalize_kind(const kv_index *ix);

int64_t kv_index_rows(const kv_index *ix);

/* Drop-in path (similarity.py:14-20): float64 cosine of one query against every local
 * row, in row order.  q_ids/q_tf: the query's in-vocabulary features; q_oov_tf2: sum of
 * tf^2 of its out-of-vocabulary features.  out_scores: host, length kv_index_rows().
 * Returns KV_ERR_EMPTY_VOCAB when neither the query nor any row has a feature. */
int kv_score(kv_index *ix, const uint32_t *q_ids, const uint32_t *q_tf, int64_t q_nnz,
             double q_oov_tf2, double *out_scores);

/* Batched scan with fused top-k (services/gfkb/app.py:88-89 generalised from 5 to k<=32):
 * for each query the k best rows ordered by (score desc, row asc) -- Python's stable
 * sort(reverse=True).  Outputs (host): out_scores[n_q*k] float32, out_rows[n_q*k] int64
 * (global row ids; unused tail slots: score -inf, row -1). */
int kv_topk(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
            const double *q_oov_tf2, int64_t n_q, int k, float *out_scores, int64_t *out_rows);

/* Same, results left on the device (d_scores float32[n_q*k], d_rows int64[n_q*k], device
 * pointers owned by the caller, e.g. torch tensors feeding the NCCL all-gather); the call
 * returns after the work is enqueued AND completed on the handle's stream. */
int kv_topk_device(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                   const double *q_oov_tf2, int64_t n_q, int k, void *d_scores, void *d_rows);

/* The two halves of kv_topk_device, for callers that keep a query batch resident:
 * kv_query_upload does the host-side preparation and the host->device copies of a batch;
 * kv_topk_resident runs scan + merge for the uploaded batch (device work only) and returns
 * when it has completed.  The batch stays valid until the next upload or finalize. */
int kv_query_upload(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                    const double *q_oov_tf2, int64_t n_q);
/* The same upload for a batch that arrives as n_runs consecutive slices (a row-sharded GFKB featurises one slice per
 * rank and exchanges them, kakveda_b200/dist.py).  kv_query_prepare_slice, on the rank that owns a slice, re-stores the
 * slice's CSR in text order (s_indptr[n_q+1] zero-based, s_ids/s_tf[nnz], s_oov_tf2[n_q]; row p = the p-th smallest
 * query, equal queries in their original order), with order_out[p] = original index of row p inside the slice and
 * flags_out[p] its classification.  kv_query_upload_runs takes per run a CSR and -- for all runs or for none -- these
 * orders and flags (then the rows must be stored sorted as above; the runs are merged instead of re-sorted; an order that
 * is not a permutation or rows out of order are rejected with KV_ERR_INVALID).  The resident batch and every result are
 * identical to kv_query_upload of the concatenated, unsorted CSR. */
int kv_query_prepare_slice(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                           const double *q_oov_tf2, int64_t n_q, int64_t *s_indptr, uint32_t *s_ids, uint32_t *s_tf,
                           double *s_oov_tf2, int32_t *order_out, uint8_t *flags_out);
int kv_query_upload_runs(kv_index *ix, int n_runs, const int64_t *const *q_indptr, const uint32_t *const *q_ids,
                         const uint32_t *const *q_tf, const double *const *q_oov_tf2, const int32_t *const *order,
                         const uint8_t *const *flags, const int64_t *n_q);
/* Host-side split of the last upload in ms: pinned staging, classification, text order, copies + table kernels. */
int kv_index_last_prepare_ms(const kv_index *ix, float ms[4]);
int kv_topk_resident(kv_index *ix, int k, void *d_scores, void *d_rows);
/* Same with host outputs (out_scores float32[n_q*k], out_rows int64[n_q*k]). */
int kv_topk_resident_host(kv_index *ix, int k, float *out_scores, int64_t *out_rows);
/* kv_topk_resident in two phases, for a row-sharded GFKB (kakveda_b200/dist.py): _seed = bound pass + seed scan, the
 * outputs receive this shard's seed top-k (device, [n_q*k], by original query); kv_index_raise_thresholds takes, per
 * query, a lower bound of the GLOBAL k-th score (device float32[n_q]; the k-th of the merged seed lists of all shards)
 * and raises the pruning thresholds of the resident batch; _finish = candidate selection + scan + merge. */
int kv_topk_resident_seed(kv_index *ix, int k, void *d_scores, void *d_rows);
int kv_index_raise_thresholds(kv_index *ix, const void *d_kth_scores, int64_t n_q);
int kv_topk_resident_finish(kv_index *ix, int k, void *d_scores, void *d_rows);
/* Self-join support: after kv_query_upload, query q never matches GLOBAL row exclude_rows[q] (-1: none; rows of
 * other shards are ignored).  Used when the queries ARE stored rows (all-pairs clustering: every row's k nearest
 * OTHER rows).  NULL clears; the next kv_query_upload clears too. */
int kv_query_set_exclusions(kv_index *ix, const int64_t *exclude_rows, int64_t n_q);
/* All-pairs on one index without re-featurising: local rows [q_begin, q_end) become the resident query batch, each
 * excluding itself (follow with kv_topk_resident / kv_topk_resident_host). */
int kv_selfjoin_upload(kv_index *ix, int64_t q_begin, int64_t q_end);

/* Label filter.  kv_index_set_row_labels gives every local row a label >= 0 (e.g. a failure-type id), labels[n] by
 * local row, n == kv_index_rows (else KV_ERR_INVALID, as for a negative label).  Labels may be set before or after
 * finalize and survive either kind of finalize and kv_index_layout_load; kv_index_append drops them.  NULL clears.
 * kv_query_set_filter restricts each query of the resident batch (kv_query_upload / kv_selfjoin_upload) to the rows
 * carrying labels[q] (by original query; -1: every row), with the lifetime of kv_query_set_exclusions; NULL clears.
 * A filtered query's top-k is the top-k over its label's rows -- (score desc, row asc), the same float32 scores as
 * unfiltered, the zero-score fill and null queries take the label's rows in ascending order, (-inf, -1) past its last
 * row -- and its threshold search returns the unfiltered pairs of its label.  The index statistics do not change.
 * KV_ERR_INVALID: wrong length, a label below -1, or a Jaccard index (mode 1).  KV_ERR_STATE: a filtered batch on an
 * index whose labels are missing or stale (appended rows), here or at the search.  Not combinable with the threshold
 * exchange of a row-sharded GFKB (kv_index_thresholds_*: KV_ERR_INVALID). */
int kv_index_set_row_labels(kv_index *ix, const int32_t *labels, int64_t n);
int kv_query_set_filter(kv_index *ix, const int32_t *labels, int64_t n_q);

/* Distinct top-k (field collapsing).  kv_index_set_row_groups gives every local row a group >= 0 (e.g. one id per
 * distinct text), groups[n] by local row; validation and lifetime as kv_index_set_row_labels: n == kv_index_rows and
 * every group >= 0 (else KV_ERR_INVALID), they survive either kind of finalize, kv_index_layout_load and deletions,
 * kv_index_append drops them, NULL clears.  Setting groups changes no result by itself.
 * kv_query_set_distinct(ix, 1) switches the resident batch (kv_query_upload / kv_selfjoin_upload) to distinct mode,
 * 0 back; the next upload switches it off.  A distinct query's top-k, for kv_topk_resident and kv_topk_resident_host:
 * of the rows it may match (live, not excluded, of its label when filtered) the best row of each group is the first in
 * (score desc, row asc) order; the groups are ranked by their best rows in that order and the first k best rows are
 * returned, (-inf, -1) past the last eligible group.  Scores are the float32 values of the non-distinct top-k, so
 * singleton groups give its result bit for bit, and the zero-score fill and null queries take the first row of each
 * new group in ascending row order.  kv_range_* ignores distinct mode: a threshold search already returns every pair.
 * KV_ERR_INVALID: a Jaccard index (mode 1), here or at kv_index_set_row_groups; kv_topk_resident_seed / _finish or
 * the threshold exchange of a row-sharded GFKB (kv_index_thresholds_*) in distinct mode -- a shard's seed scores are
 * no lower bound of the global k-th group score, since one group can count on several shards.  KV_ERR_STATE: distinct
 * mode on an index whose groups are missing or stale (appended rows), here or at the search. */
int kv_index_set_row_groups(kv_index *ix, const int32_t *groups, int64_t n);
int kv_query_set_distinct(kv_index *ix, int on);

/* Row deletion (tombstones).  rows[n]: local rows, any order; duplicates and rows already deleted are allowed (a call
 * that deletes no new row changes nothing).  A deleted row keeps its row id and its place in the scan layout but is
 * never returned again by any search on the handle: top-k (seed, candidate and exhaustive scans), threshold search,
 * self-joins, the float64 fallbacks of irregular queries and the null-query fill (a null query gets the first k LIVE
 * rows, a filtered one the first k live rows of its label).
 *   - Like an append, a deletion needs kv_index_finalize before the next search (until then: KV_ERR_STATE); the
 *     resident batch and any range result are dropped.  A finalize whose only change since the last full rebuild is
 *     deletions is a statistics-only refresh (kv_index_last_finalize_kind 2); after an append the full rebuild keeps
 *     the deleted rows deleted.
 *   - Statistics: N (without kv_index_set_global_df) and df count live rows, and so does kv_index_local_df, so the df
 *     all-reduce of a row-sharded or segmented GFKB stays right.  Universal-feature folding and the tf extremes stay
 *     properties of the layout rows, deleted ones included (a folded feature is still in every layout row).  A feature
 *     of the vocabulary that no live row holds (df 0) scores like an out-of-vocabulary feature: idf ln((N+2)/2)+1 in
 *     the query-inclusive mode, ignored in KV_MODE_TFIDF_CORPUS_FIT.
 *   - Outputs: kv_score writes -inf for a deleted row, kv_rescore_pairs -inf (as for a row of another shard); the
 *     kv_selfjoin_upload query of a deleted row has an empty list, (-inf, -1), and no threshold pairs -- it stays a
 *     singleton in kv_cluster_*.
 *   - Labels (kv_index_set_row_labels) survive deletions.  kv_index_layout_save / _load do not carry deletions (state
 *     of the handle, not of the file); a layout load keeps the handle's deletions.
 *   - KV_ERR_INVALID: a row outside 0..kv_index_rows-1, rows == NULL with n > 0, or a Jaccard index (mode 1).
 * kv_index_live_rows: kv_index_rows minus the deleted rows.  kv_index_deleted_rows: out[n] = 1 for a deleted local
 * row, 0 for a live one; n == kv_index_rows (else KV_ERR_INVALID). */
int kv_index_delete_rows(kv_index *ix, const int64_t *rows, int64_t n);
int64_t kv_index_live_rows(const kv_index *ix);
int kv_index_deleted_rows(kv_index *ix, uint8_t *out, int64_t n);

/* Threshold search over the resident batch (kv_query_upload / kv_selfjoin_upload; exclusions honoured): every
 * (query, row) pair whose score -- the float32 value kv_topk reports for that pair -- is >= threshold,
 * 0 < threshold <= 1.  *n_pairs receives the count; the pairs stay in the handle until kv_range_fetch, the next
 * upload, finalize or range call.  Extension for threshold consumers (services/warning_policy/app.py:22,52 compares
 * with failure_matching.similarity_threshold; kv_cluster_csr links on the exact threshold graph).  It runs bound pass 1
 * on the fixed threshold and the candidate scan with an emitting epilogue (the exhaustive scan on small indexes), then
 * the float64 full scan of irregular queries; the resident batch, its exclusions and the top-k thresholds are left as
 * they were, so a later kv_topk_resident* returns what it would have without it.  kv_index_last_kernel_ms: [0] = [1] =
 * 0, [2] = bound pass 1, [3] = the scan (including a re-run after the pair buffer grew), [4] = irregular-query
 * fallbacks; kv_index_layout counters [9]-[13] describe the run.  threshold NaN, <= 0 or > 1: KV_ERR_INVALID.
 * KV_ERR_NOMEM when the candidate pool is exhausted or the pairs do not fit in device memory (the message gives their
 * count).  Jaccard indexes: KV_ERR_INVALID (they search with kv_jaccard_range_resident). */
int kv_range_resident(kv_index *ix, float threshold, int64_t *n_pairs);
/* The last range result: indptr[n_q+1] by original query, rows[n_pairs] (global), scores[n_pairs]; per query
 * ordered by (score desc, row asc).  KV_ERR_STATE when there is none (always on a Jaccard index). */
int kv_range_fetch(kv_index *ix, int64_t *indptr, int64_t *rows, float *scores);
/* The threshold search of a Jaccard index (KV_MODE_JACCARD), over the batch uploaded by kv_query_upload or
 * kv_selfjoin_upload (exclusions honoured): every (query, row) pair whose float32 score -- the value kv_topk reports,
 * |q ∩ row| / |q ∪ row| rounded once -- is >= threshold, 0 < threshold <= 1 (else KV_ERR_INVALID).  K3-R scores every
 * chunk like the top-k scan and appends each match with its exact counts; queries of more than 64 tokens take the
 * float64 full scan, whose exact ratio gives the counts back.  The pair buffer starts at 65,536 records and grows to
 * the exact count when a search finds more (the scan then runs again; KV_ERR_NOMEM with the count when the pairs do
 * not fit in device memory).  The result stays until kv_jaccard_range_fetch or the next upload, top-k, range, append
 * or finalize call.  kv_index_last_kernel_ms: [3] = the scan (re-run included), [4] = irregular-query fallbacks.
 * Both functions return KV_ERR_INVALID on a TF-IDF index. */
int kv_jaccard_range_resident(kv_index *ix, float threshold, int64_t *n_pairs);
/* The last Jaccard range result: indptr[n_q+1] by original query, rows[n_pairs] (global), scores[n_pairs] (float32),
 * inter[n_pairs] = |q ∩ row| and uni[n_pairs] = |q ∪ row|; per query ordered by (score desc, row asc), as
 * kv_range_fetch.  scores[i] is the float32 quotient inter[i] / uni[i].  KV_ERR_STATE when there is none. */
int kv_jaccard_range_fetch(kv_index *ix, int64_t *indptr, int64_t *rows, float *scores, int32_t *inter, int32_t *uni);
/* Both fetches order the pairs on the device (an LSD radix sort of the records on (query, score desc, row)) and copy
 * the ordered arrays back; when pairs plus queries number below 8192 they copy the records back and order them on one
 * host core, which is faster there (the same bits either way).  The _device forms write the same arrays, bit for bit, to caller-owned device memory (e.g.
 * torch tensors) on the index's device: d_indptr int64[n_q+1], d_rows int64[n_pairs], d_scores float32[n_pairs], and
 * for Jaccard d_inter / d_uni int32[n_pairs].  They consume the result like the host fetch and return once the work on
 * the handle's stream is complete.  KV_ERR_STATE when there is no result (none computed, fetched already, or dropped by
 * a later upload); KV_ERR_INVALID on the other index kind, or when a pointer is not device memory of the index's device
 * aligned to its element size (the arrays of n_pairs elements are not looked at when n_pairs == 0).  KV_ERR_NOMEM (with
 * the pair count) when the ordering's scratch -- about the pair buffer's size again -- does not fit; the result then
 * stays for another try. */
int kv_range_fetch_device(kv_index *ix, void *d_indptr, void *d_rows, void *d_scores);
int kv_jaccard_range_fetch_device(kv_index *ix, void *d_indptr, void *d_rows, void *d_scores, void *d_inter, void *d_uni);

/* K6: float64 scores of selected (query, row) pairs: rows[n_q*k] are GLOBAL row ids (e.g. what kv_topk returned;
 * -1 = unused slot), out_scores[n_q*k] (host) receives the float64 cosine of SimilarityEngine.score
 * (similarity.py:14-20) for that row, -inf for unused slots and rows that live on another shard.  Summation follows
 * the row's stored feature order with nothing folded, so rows with identical text get identical bits on every shard /
 * segment and services/gfkb/app.py:89's stable sort is reproduced (ties -> lower row).  The batched match path ranks
 * candidates in float32 (K1b) and re-scores the survivors here. */
int kv_rescore_pairs(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                     const double *q_oov_tf2, int64_t n_q, int k, const int64_t *rows, double *out_scores);

/* Cross-GPU pruning thresholds for a row-sharded GFKB (one process per GPU, all ranks hold the SAME resident query
 * batch).  Block-max pruning needs a lower bound of every query's GLOBAL k-th score; a shard scanning alone only knows
 * its own.  export: make this index's threshold array (int32 float bits per sorted query slot, `capacity` queries)
 * visible to the other processes -- writes a 64-byte CUDA IPC handle.  peers: map the arrays the other ranks exported
 * (n_peers <= 7 handles of 64 bytes, same capacity); from then on every bound a scan CTA establishes is also pushed
 * into the peers' arrays with system-scope reductions over NVLink/NVSwitch peer memory while the kernels run, so all
 * shards prune with the best bound known anywhere (n_peers = 0 unmaps).  Results are unchanged -- a pushed value
 * always is a valid lower bound (k rows at least that good exist in some shard) -- only less is scanned.  Callers must
 * keep scans of different batches apart with a collective (the all-gather of partial top-k does that) and exchange
 * again after uploading a batch larger than `capacity` (kv_topk* returns KV_ERR_STATE otherwise). */
int kv_index_thresholds_export(kv_index *ix, int64_t capacity, void *handle_out);
int kv_index_thresholds_peers(kv_index *ix, const void *handles, int n_peers, int64_t capacity);

/* K5: merge n_lists partial top-k lists per query (device pointers; list l of query q at
 * [l*n_q*k + q*k], each sorted by (score desc,row asc)) into one [n_q*k] result with the
 * same ordering.  Used after the cross-GPU all-gather. */
int kv_merge_topk_device(int device, const void *d_scores_in, const void *d_rows_in, int n_lists,
                         int64_t n_q, int k, void *d_scores_out, void *d_rows_out);
/* The same on a caller-given CUDA stream (a cudaStream_t, e.g. the stream the all-gather that produced the lists
 * was enqueued on; NULL = legacy default stream); sync = 0 returns without waiting for the kernel.  stride_s /
 * stride_r: float32 / int64 elements between the starts of consecutive lists (n_q*k when contiguous; larger when
 * scores and rows travel in ONE packed all-gather buffer per rank). */
int kv_merge_topk_device_on(int device, const void *d_scores_in, const void *d_rows_in, int n_lists,
                            int64_t n_q, int k, int64_t stride_s, int64_t stride_r, void *d_scores_out,
                            void *d_rows_out, void *stream, int sync);

/* Timing of the last kv_topk / kv_topk_device call on this handle, CUDA-event
 * milliseconds on its stream:
 * ms[0] = H2D of the query batch, ms[1] = bound + scan kernels, ms[2] = merge (+ fallbacks), ms[3] = D2H. */
int kv_index_last_timing(const kv_index *ix, float ms[4]);
/* ... and of its kernels: ms[0] = bound pass 0 (seeds; wgmma GEMM + rare-feature join), ms[1] = seed scan,
 * ms[2] = bound pass 1 (candidate lists; when the bound codes of pass 0 were kept, only the snapshot of the
 * threshold codes: the scan selects its candidates from the codes), ms[3] = candidate scan, ms[4] = merge.
 * Exhaustive mode: only [3], [4].
 * After kv_range_resident: see there. */
int kv_index_last_kernel_ms(const kv_index *ix, float ms[5]);
/* Test hook: runs the resident batch once and returns the numerators (dot-product upper bounds) the bound kernel formed
 * for every (query slot, chunk): out[n_q][chunks] floats, slot_query[i] = original query of sorted slot i.  Needs an
 * index large enough for the pruned path (>= 512 chunks of 32 rows); tests/test_gpu_parity.py compares with NumPy. */
int kv_debug_bound_numerators(kv_index *ix, int k, float *out, int32_t *slot_query);
/* Test hook: runs the resident batch once, as kv_topk_resident does (same bound-kernel instantiation: the specialised
 * one, or the generic one under KAKVEDA_B200_GENERIC_BOUND=1), and returns what bound pass 0 produced, by sorted query
 * slot i (original query slot_query[i]):
 *   codes[n_q][chunks]    the 8-bit bound codes the candidate scan selected from;
 *   tcode[n_q]            the threshold codes it compared them with (256: the query takes no candidate);
 *   q_terms[n_q][4]       the query constants of the bound: |q|^2, dotS, dotX, corrS;
 *   chunk_minB[chunks]    the smallest positive live row norm per chunk (+inf: none);
 *   row_at_pos[n_rows]    the local row at each scan position (chunk c = positions 32c .. 32c + 31).
 * codes and slot_query are required, the other outputs may be NULL.  kv_index_layout describes this run afterwards.
 * KV_ERR_STATE when no batch is uploaded or the run kept no codes (exhaustive path below 512 chunks,
 * KAKVEDA_B200_BOUND_CODES=0, codes too large for the device, Jaccard mode). */
int kv_debug_bound_codes(kv_index *ix, int k, uint8_t *codes, int32_t *slot_query, int32_t *tcode, float *q_terms,
                         float *chunk_minB, int32_t *row_at_pos);
/* Test hook: orders n caller-built range records (host memory, 16 bytes each, the layout the range scans emit) on
 * `device` with the code the fetch functions use, so that inputs a real search cannot cheaply produce can be checked.
 * jaccard = 0: records {int32 q, float32 score, int64 row} (rows global, row_base ignored); jaccard != 0: {int32 q,
 * int32 local row, int32 inter, int32 uni}, rows + row_base, scores inter / uni in float32.  Outputs as
 * kv_jaccard_range_fetch (host); inter / uni are only written for Jaccard records.  Records with a query outside
 * 0..n_q-1, a NaN score or counts outside 0 <= inter <= uni, uni >= 1: KV_ERR_INVALID. */
int kv_debug_range_order(int device, int jaccard, const void *records, int64_t n, int64_t n_q, int64_t row_base,
                         int64_t *indptr, int64_t *rows, float *scores, int32_t *inter, int32_t *uni);
/* CUDA-event milliseconds of the scan kernel of the last kv_score call (K1a). */
int kv_index_last_score_ms(const kv_index *ix, float *ms);

/* Persisted scan layout (SURVEY 8(f) rank 4; the write side of services/gfkb/app.py:38-56 makes cold starts matter): _save
 * writes what kv_index_finalize built on the host cores (row order, column blocks, dense matrix, bitmaps, rare tables)
 * to one file; _load, called after the SAME rows were appended and before kv_index_finalize, restores it (the file is
 * tied to the rows by count + checksum; KV_ERR_STATE if it does not match), so that finalize only refreshes the
 * statistics (kv_index_last_finalize_kind == 2) instead of sorting and building (~15 s at 10M rows). */
int kv_index_layout_save(kv_index *ix, const char *path);
int kv_index_layout_load(kv_index *ix, const char *path);

/* Scan-layout facts for roofline accounting.
 * bytes[0] = column blocks, bytes[1] = row norms (float32), bytes[2] = block directory,
 * bytes[3] = dense frequent-feature matrix (fp16) + chunk min norms.
 * counts[0] = block entries, [1] = folded (universal) features, [2] = rows, [3] = CTAs of the
 * last candidate scan, [4] = its 128-query bound tiles, [5] = partial lists per query, [6] = host->device bytes of
 * the last query upload, [7] = tf-overflow entries, [8] = chunks (32 rows each), and for the last batch:
 * [9] = (query, chunk) pairs scored exactly (seed scan + candidate scan), [10] = candidate records scanned,
 * [11] = (query, chunk) pairs whose bound passed, [12] = candidate records written, [13] = kernels launched,
 * [14] = block entries of non-frequent features, [15] = candidate-pool pages used, [16] = pool pages allocated,
 * [17] = second-class (query, feature) listings of the last query upload left out of their bound tile's dictionary
 * (the bound kernel's epilogue adds those per block from the second-class bitmaps). */
int kv_index_layout(const kv_index *ix, int64_t bytes[4], int64_t counts[18]);

/* ------------------------------------------------------------------------------------
 * K2: dense-embedding cosine index (bf16 rows of `dim` elements, dim a multiple of 64) with the
 * top-k fused into a wgmma GEMM epilogue.  The reference has no embedding path (its docs list
 * embeddings as a possible extension, docs/failure-intelligence.md:43-46): parity UNPINNED, oracle =
 * float64 cosine of the same bf16 inputs.  Inputs are bfloat16 bit patterns (uint16), row-major.
 * kv_dense_topk: per query the k (<=32) best rows by (cosine desc, row asc); host outputs
 * float32[n_q*k] / int64[n_q*k]; unused slots (-inf, -1).
 * ---------------------------------------------------------------------------------- */
typedef struct kv_dense_index kv_dense_index;
int kv_dense_create(int device, int dim, int64_t row_base, kv_dense_index **out);
void kv_dense_destroy(kv_dense_index *dx);
int kv_dense_append(kv_dense_index *dx, const uint16_t *rows_bf16, int64_t n);
int kv_dense_finalize(kv_dense_index *dx);
int64_t kv_dense_rows(const kv_dense_index *dx);
int kv_dense_topk(kv_dense_index *dx, const uint16_t *q_bf16, int64_t n_q, int k, float *out_scores, int64_t *out_rows);
/* Device-side variants (pointers are device memory owned by the caller, e.g. torch tensors; bf16 data 16-byte
 * aligned): append rows that are already in HBM; scan with queries and results on the device -- what a rank of
 * a row-sharded GFKB calls before the NCCL all-gather of partial top-k (BASELINE configs[2]).  exclude_base >= 0:
 * query q must not match GLOBAL row exclude_base + q (the all-pairs self-join of BASELINE configs[3], where the
 * queries are the stored rows themselves); -1: no exclusion. */
int kv_dense_append_device(kv_dense_index *dx, const void *d_rows_bf16, int64_t n);
int kv_dense_topk_device(kv_dense_index *dx, const void *d_q_bf16, int64_t n_q, int k, int64_t exclude_base,
                         void *d_scores, void *d_rows);
/* All-pairs on one shard without copying: local rows [q_begin, q_end) are the queries, each row's own entry is
 * excluded, results (device) as above. */
int kv_dense_selfjoin_device(kv_dense_index *dx, int64_t q_begin, int64_t q_end, int k, void *d_scores, void *d_rows);
/* Threshold search (K2-R, the same GEMM with an emitting epilogue): every (query, row) pair whose cosine -- the float32
 * value kv_dense_topk reports for that pair, bit for bit -- is >= threshold, 0 < threshold <= 1.  Rows are global
 * (row_base applied); q is the query's index within the call (row - q_begin for the self-join, which excludes each
 * row's own entry; exclude_base as in kv_dense_topk_device).  *n_pairs receives the count; the pairs stay in the handle
 * until kv_dense_range_fetch or the next range, top-k, append or finalize call.  The pair buffer starts at 65,536
 * records and keeps its capacity; when a search finds more pairs it grows to the exact count and the whole kernel,
 * GEMM included, runs again.  threshold NaN, <= 0 or > 1, n_q >= 2^31, or device queries not 16-byte aligned:
 * KV_ERR_INVALID.  Index not finalized: KV_ERR_STATE.  KV_ERR_NOMEM when the pairs do not fit in device memory (the
 * message gives their count). */
int kv_dense_range(kv_dense_index *dx, const uint16_t *q_bf16, int64_t n_q, float threshold, int64_t *n_pairs);
int kv_dense_range_device(kv_dense_index *dx, const void *d_q_bf16, int64_t n_q, float threshold,
                          int64_t exclude_base, int64_t *n_pairs);
int kv_dense_selfjoin_range(kv_dense_index *dx, int64_t q_begin, int64_t q_end, float threshold, int64_t *n_pairs);
/* The last dense range result (host outputs): indptr[n_q+1] by query, rows[n_pairs], scores[n_pairs]; per query ordered
 * by (score desc, row asc).  KV_ERR_STATE when there is none. */
int kv_dense_range_fetch(kv_dense_index *dx, int64_t *indptr, int64_t *rows, float *scores);
/* The same arrays in caller-owned device memory, as kv_range_fetch_device (the host fetch orders on the device too). */
int kv_dense_range_fetch_device(kv_dense_index *dx, void *d_indptr, void *d_rows, void *d_scores);
/* CUDA-event milliseconds of the GEMM kernel of the last kv_dense_topk* / kv_dense_selfjoin_device or range call (a
 * range re-run after the pair buffer grew included) and its row splits. */
int kv_dense_last_timing(const kv_dense_index *dx, float *gemm_ms, int64_t *splits);
/* Dense row deletion (tombstones), as kv_index_delete_rows.  rows[n]: local rows, any order; duplicates and rows already
 * deleted are allowed (a call that deletes no new row changes nothing).  A deleted row keeps its row id and its position
 * but no top-k, threshold search or self-join returns it again; a self-join query whose own row is deleted gets an empty
 * list, (-inf, -1), and no threshold pairs.
 *   - Like an append, a deletion needs kv_dense_finalize before the next search (until then: KV_ERR_STATE) and drops
 *     any range result.  The finalize gives every deleted row a NaN inverse norm, which removes all its scores in the
 *     epilogue: the kernels themselves do not change.
 *   - The deleted set belongs to the handle: appends and finalizes keep it, appended rows are live.  Row labels
 *     (kv_dense_set_row_labels) survive deletions.
 *   - KV_ERR_INVALID: a row outside 0..kv_dense_rows-1, or rows == NULL with n > 0.
 * kv_dense_live_rows: kv_dense_rows minus the deleted rows.  kv_dense_deleted_rows: out[n] = 1 for a deleted local row,
 * 0 for a live one; n == kv_dense_rows (else KV_ERR_INVALID). */
int kv_dense_delete_rows(kv_dense_index *dx, const int64_t *rows, int64_t n);
int64_t kv_dense_live_rows(const kv_dense_index *dx);
int kv_dense_deleted_rows(kv_dense_index *dx, uint8_t *out, int64_t n);
/* Dense label filter.  kv_dense_set_row_labels gives every local row a label >= 0, labels[n] by local row, n ==
 * kv_dense_rows (else KV_ERR_INVALID, as for a negative label); NULL clears.  Labels may be set before or after
 * finalize; finalize and deletions keep them, an append drops them.
 * kv_dense_set_query_filter restricts each query of THE NEXT SEARCH CALL on the handle (kv_dense_topk, _topk_device,
 * _selfjoin_device, _range, _range_device or _selfjoin_range) to the rows carrying labels[q] (-1: every row); NULL
 * clears.  That call must have exactly n_q queries (else KV_ERR_INVALID) and clears the filter whether it succeeds or
 * fails; an append or a finalize clears it too.  A filtered query's top-k is the top-k over its label's live rows --
 * (score desc, row asc), the same float32 scores as unfiltered, (-inf, -1) past its label's last candidate -- and its
 * threshold search returns the unfiltered pairs of its label; a -1 query gets the unfiltered answer.  The kernel skips
 * every (128-query tile, 256-row tile) item whose row tile holds no live row of a label of the query tile.
 * KV_ERR_INVALID: a query label below -1 (here) or a query count that differs (at the search).  KV_ERR_STATE: a
 * filtered search on an index whose labels are missing or stale (appended rows). */
int kv_dense_set_row_labels(kv_dense_index *dx, const int32_t *labels, int64_t n);
int kv_dense_set_query_filter(kv_dense_index *dx, const int32_t *labels, int64_t n_q);
/* Measurement and test hook: the (query tile, row tile) items the last dense search's kernel skipped and its total
 * items (q_tiles x r_tiles; skipped is 0 for an unfiltered search). */
int kv_dense_last_skipped(const kv_dense_index *dx, int64_t *skipped, int64_t *items);

/* ------------------------------------------------------------------------------------
 * K4: 64-bit fingerprint exact-match index.  One uint64 per row = the leading 64 bits of
 * sha256(signature_text), i.e. int(fingerprint(), 16) of services/shared/fingerprint.py:69-71
 * (a function the reference defines but never queries: matching by it is an extension, its
 * oracle is integer equality).  kv_hash_match reports, per query hash, how many rows carry it
 * and the first k of them in ascending row order (unused slots -1).  Pure HBM-bound scan.
 * ---------------------------------------------------------------------------------- */
typedef struct kv_hash_index kv_hash_index;
int kv_hash_create(int device, int64_t row_base, kv_hash_index **out);
void kv_hash_destroy(kv_hash_index *hx);
int kv_hash_append(kv_hash_index *hx, const uint64_t *hashes, int64_t n);
int64_t kv_hash_rows(const kv_hash_index *hx);
int kv_hash_match(kv_hash_index *hx, const uint64_t *q_hashes, int64_t n_q, int k, int64_t *out_rows,
                  int64_t *out_counts);
/* CUDA-event milliseconds of the scan kernel launches of the last kv_hash_match, and their number
 * (one pass over all rows per 4096 queries). */
int kv_hash_last_timing(const kv_hash_index *hx, float *scan_ms, int *passes);

/* ------------------------------------------------------------------------------------
 * Pattern clustering on top of an all-pairs top-k (BASELINE configs[3]): rows[n*k] / scores[n*k] are every row's k
 * nearest OTHER rows (kv_selfjoin_upload + kv_topk_resident_host, or kv_dense_selfjoin_device); rows i and j are
 * linked when either lists the other with score >= threshold; labels[i] = smallest row id of i's connected
 * component, *n_clusters = number of components.  Host code (union-find).  Extension of
 * services/pattern_detector/app.py:39-41, which groups by failure_type equality only.
 * ---------------------------------------------------------------------------------- */
int kv_cluster_topk(int64_t n, int k, const int64_t *rows, const float *scores, float threshold, int64_t *labels,
                    int64_t *n_clusters);
/* Connected components of the graph whose edges are i -- rows[j] for j in [indptr[i], indptr[i+1]) (rows < 0
 * skipped, rows >= n rejected): labels[i] = smallest row of i's component (union-find of kv_cluster_topk).  With the
 * result of kv_selfjoin_upload + kv_range_resident these are the components of the exact threshold graph, which a
 * top-k list cannot give when a text is stored more than k times. */
int kv_cluster_csr(int64_t n, const int64_t *indptr, const int64_t *rows, int64_t *labels, int64_t *n_clusters);
/* kv_cluster_csr on the device: d_indptr int64[n+1], d_rows int64 (indexed absolutely by indptr, so indptr[0] may be
 * nonzero) and d_labels int64[n] are device memory of `device` (e.g. the output of kv_range_fetch_device); the same
 * labels, bit for bit.  A lock-free union-find (roots hooked under smaller roots with compare-and-swap), so labels do
 * not depend on thread timing.  Validation passes run before any hooking: indptr not monotone or indptr[0] < 0, or a
 * row >= n: KV_ERR_INVALID.  Pointers that are not device memory of `device` aligned to 8 bytes: KV_ERR_INVALID.
 * Runs on a stream of its own and returns when the labels are written; n_clusters (host, may be NULL). */
int kv_cluster_csr_device(int device, int64_t n, const void *d_indptr, const void *d_rows, void *d_labels,
                          int64_t *n_clusters);

/* ------------------------------------------------------------------------------------
 * Synthetic failures.jsonl-shaped signature_text generator (test / bench support; the
 * strings have the shape services/shared/fingerprint.py:51-66 produces).  Row i of a
 * stream is a pure function of (seed, i).  Writes rows [first, first+count) back to back
 * into `bytes` (capacity cap) with offsets[count+1]; returns KV_ERR_NOMEM if cap is too
 * small (needed size in offsets[count]).  dup_of_seed/dup_rows != 0 makes about half the
 * rows exact copies of rows of another stream (queries that hit stored failures). */
int kv_synth_signatures(uint64_t seed, int64_t first, int64_t count, uint64_t dup_of_seed,
                        int64_t dup_rows, char *bytes, int64_t cap, int64_t *offsets);

#ifdef __cplusplus
}
#endif
#endif /* KAKVEDA_B200_H */
