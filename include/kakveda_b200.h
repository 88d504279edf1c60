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

/* Device featuriser (featurize_device.cu).  A kv_vocab_mirror is an open-addressing table in the HBM of one device
 * that maps the 128-bit key of every feature of a kv_vocab to its id (load factor <= 0.5, home slot k0 & (cap - 1),
 * 40 bytes of HBM per feature at the largest load, 80 just after a growth).  kv_vocab_mirror_sync appends the ids
 * [mirrored, kv_vocab_size(v)) and grows the table when needed; a vocabulary only grows, so the mirror is a prefix of it.
 * A sync that meets a concurrent featurize(grow = 1) or import keeps the mirror as it was and returns KV_ERR_STATE (try
 * again later).  *n_mirrored (optional) receives the features mirrored after the call.
 * kv_featurize_device is kv_featurize(v, ..., grow = 0) computed on the device against the mirror (synced first), with
 * the same result bit for bit and the same errors; it returns an ordinary host kv_csr. */
typedef struct kv_vocab_mirror kv_vocab_mirror;
int kv_vocab_mirror_create(int device, kv_vocab_mirror **out);
void kv_vocab_mirror_destroy(kv_vocab_mirror *m);
int kv_vocab_mirror_sync(kv_vocab_mirror *m, const kv_vocab *v, int64_t *n_mirrored);
int kv_featurize_device(kv_vocab_mirror *m, const kv_vocab *v, const char *bytes, const int64_t *offsets, int64_t n_docs,
                        int mode, kv_csr **out, int64_t *bad_doc);

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
 * sets.  Top-k then ranks by float32 inter/union; kv_jaccard_counts returns the exact integers of the
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

/* Batched scan with fused top-k (services/gfkb/app.py:88-89 generalised from 5 to k<=32), in two steps:
 * kv_query_upload (or _runs, _text, kv_selfjoin_upload) does the host-side preparation and the host->device copies of
 * a query batch (n_q >= 1), which stays resident until the next upload or finalize; kv_topk_resident /
 * kv_topk_resident_host run scan + merge for it, as often as wanted.  For each query the k best rows ordered by
 * (score desc, row asc) -- Python's stable sort(reverse=True) -- as float32 scores[n_q*k] and int64 rows[n_q*k] by
 * original query (global row ids; unused tail slots: score -inf, row -1). */
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
/* kv_query_upload of the batch kv_featurize(v, bytes, offsets, n_q, mode, grow = 0) would give, built on the device:
 * the text goes up, is featurised there against the mirror m (synced first; m must live on the index's device), and
 * classification, text order and tables are computed there.  The resident batch is identical to the host path's.
 * Errors: those of kv_featurize (*bad_doc on KV_ERR_NONASCII) and of kv_query_upload. */
int kv_query_upload_text(kv_index *ix, kv_vocab_mirror *m, const kv_vocab *v, const char *bytes, const int64_t *offsets,
                         int64_t n_q, int mode, int64_t *bad_doc);
/* Host-side split of the last upload in ms: pinned staging, classification, text order, copies + table kernels.
 * After kv_query_upload_text: text upload + featurisation, classification, text order, tables + copies back. */
int kv_index_last_prepare_ms(const kv_index *ix, float ms[4]);
/* Test hook: the resident batch's query order and flags (qperm[i] = original query at sorted slot i, flags[i] its
 * class: 0 regular, 1 null, 2 irregular); n_q must be the batch size. */
int kv_debug_query_order(kv_index *ix, int32_t *qperm, uint8_t *flags, int64_t n_q);
/* Top-k of the resident batch into caller-owned device memory (d_scores, d_rows; e.g. torch tensors feeding the NCCL
 * all-gather); returns when the work on the handle's stream has completed.  k outside 1..32: KV_ERR_INVALID. */
int kv_topk_resident(kv_index *ix, int k, void *d_scores, void *d_rows);
/* Same with host outputs (out_scores, out_rows). */
int kv_topk_resident_host(kv_index *ix, int k, float *out_scores, int64_t *out_rows);
/* kv_topk_resident in two phases, for a row-sharded GFKB (kakveda_b200/dist.py): _seed = bound pass + seed scan, the
 * outputs receive this shard's seed top-k (device, [n_q*k], by original query); kv_index_raise_thresholds takes, per
 * query, a lower bound of the GLOBAL k-th score (device float32[n_q]; the k-th of the merged seed lists of all shards)
 * and raises the pruning thresholds of the resident batch; _finish = candidate selection + scan + merge.  The seed
 * lists honour the batch's filter and distinct mode.  _seed writes the slots of regular queries only: null and
 * irregular queries have no seed list, so a caller that merges the seed lists fills the outputs with (-inf, -1) first.
 * For a distinct batch the k-th seed score must be taken over distinct groups -- one group can appear in several
 * shards' seed lists: slot k-1 of kv_merge_topk_distinct_device_on over the gathered seed lists (global rows); the
 * batch must be switched on with kv_query_set_distinct(ix, KV_DISTINCT_MERGED_SEEDS), else KV_ERR_INVALID. */
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
 * index whose labels are missing or stale (appended rows), here or at the search.  A filtered batch may use
 * kv_topk_resident_seed / _finish and the threshold exchange of a row-sharded GFKB (kv_index_thresholds_*) when every
 * rank sets the same filter (see there). */
int kv_index_set_row_labels(kv_index *ix, const int32_t *labels, int64_t n);
int kv_query_set_filter(kv_index *ix, const int32_t *labels, int64_t n_q);

/* Tag filter (e.g. a failure's affected apps).  kv_index_set_row_tags gives every local row a SET of tags >= 0, any
 * number, possibly none: row r holds tags[indptr[r] .. indptr[r+1]), indptr[n_rows+1] starting at 0, n_rows ==
 * kv_index_rows.  Lifetime as row labels: they survive either kind of finalize, kv_index_layout_load and deletions,
 * kv_index_append drops them, NULL clears.  Tags touch no statistics, so setting them again on a finalized index needs
 * no finalize.  kv_query_set_tag_filter gives each query of the resident batch a set of at most 16 tags (same CSR form,
 * n_q == the batch; an empty set: no tag constraint), cleared by the next upload like kv_query_set_filter; NULL clears.
 * A query with tags matches only the rows whose set meets its own (any of its tags); the label filter, exclusions,
 * deletions and distinct mode apply as well, and scores, statistics and the order rules are those of the unfiltered
 * search.  The scans skip the chunks whose live rows carry none of the query's tags (a 64-bit signature per chunk of
 * bit t & 63 per tag), then test each row's mask and, when the index holds a tag >= 64, its exact set.  A null query
 * with tags walks the index in row order until it has k eligible rows (the whole index when it has fewer).
 * KV_ERR_INVALID: wrong lengths, indptr not starting at 0 or decreasing, a negative tag, more than 16 tags on a query,
 * or a Jaccard index (mode 1).  KV_ERR_STATE: a query with tags on an index whose tags are missing or stale (appended
 * rows), here or at the search. */
int kv_index_set_row_tags(kv_index *ix, const int64_t *indptr, const int32_t *tags, int64_t n_rows);
int kv_query_set_tag_filter(kv_index *ix, const int64_t *indptr, const int32_t *tags, int64_t n_q);

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
 * A row-sharded GFKB gives each shard the groups of its own rows (one group may span shards) and switches its batch on
 * with on = KV_DISTINCT_MERGED_SEEDS: distinct mode, plus the caller's promise that it merges the shards' seed lists
 * group-aware (kv_merge_topk_distinct_device_on) and raises the thresholds to slot k-1 of that merge.  Only then do
 * kv_topk_resident_seed / _finish run a distinct batch; with on = 1 they refuse it (KV_ERR_INVALID), since the k-th of
 * the shards' raw seed scores may count one group several times and is no lower bound of the global k-th group score.
 * The threshold exchange (kv_index_thresholds_*) takes distinct batches in either form.  The final merge of the
 * shards' lists is kv_merge_topk_distinct_device_on.
 * KV_ERR_INVALID: a Jaccard index (mode 1), here or at kv_index_set_row_groups.  KV_ERR_STATE: distinct mode on an
 * index whose groups are missing or stale (appended rows), here or at the search. */
#define KV_DISTINCT_MERGED_SEEDS 2
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
 * (query, row) pair whose score -- the float32 value the top-k reports for that pair -- is >= threshold,
 * 0 < threshold <= 1.  *n_pairs receives the count; the pairs stay in the handle until kv_range_fetch, the next
 * upload, range, append, deletion or finalize call.  Extension for threshold consumers (services/warning_policy/app.py:22,52 compares
 * with failure_matching.similarity_threshold; kv_cluster_csr links on the exact threshold graph).  It runs bound pass 1
 * on the fixed threshold and the candidate scan with an emitting epilogue (the exhaustive scan on small indexes), then
 * the float64 full scan of irregular queries; the resident batch, its exclusions and the top-k thresholds are left as
 * they were, so a later kv_topk_resident* returns what it would have without it.  kv_index_last_kernel_ms: [0] = [1] =
 * 0, [2] = bound pass 1, [3] = the scan (including a re-run after the pair buffer grew), [4] = irregular-query
 * fallbacks; kv_index_layout counters [9]-[13] describe the run.  threshold NaN, <= 0 or > 1: KV_ERR_INVALID.
 * KV_ERR_NOMEM when the candidate pool is exhausted or the pairs do not fit in device memory (the message gives their
 * count).
 * On a Jaccard index (KV_MODE_JACCARD) the score is |q ∩ row| / |q ∪ row| rounded once, and K3-R scores every chunk
 * like the top-k scan and appends each match with its exact counts; queries of more than 64 tokens take the float64
 * full scan, whose exact ratio gives the counts back.  Its pair buffer starts at 65,536 records and grows to the exact
 * count when a search finds more (the scan then runs again).  kv_index_last_kernel_ms: [3] = the scan (re-run
 * included), [4] = irregular-query fallbacks. */
int kv_range_resident(kv_index *ix, float threshold, int64_t *n_pairs);
/* The last range result: indptr[n_q+1] by original query, rows[n_pairs] (global), scores[n_pairs] (float32); per query
 * ordered by (score desc, row asc).  On a Jaccard index also inter[n_pairs] = |q ∩ row| and uni[n_pairs] = |q ∪ row|,
 * with scores[i] the float32 quotient inter[i] / uni[i]; a TF-IDF index has no counts.  inter and uni are required on
 * a Jaccard index (like rows and scores: when there are pairs) and must be NULL on a TF-IDF index; anything else is
 * KV_ERR_INVALID and leaves the result for a later fetch.  KV_ERR_STATE when there is no result. */
int kv_range_fetch(kv_index *ix, int64_t *indptr, int64_t *rows, float *scores, int32_t *inter, int32_t *uni);
/* Both fetches order the pairs on the device (an LSD radix sort of the records on (query, score desc, row)) and copy
 * the ordered arrays back; when pairs plus queries number below 8192 they copy the records back and order them on one
 * host core, which is faster there (the same bits either way).  The _device forms write the same arrays, bit for bit, to caller-owned device memory (e.g.
 * torch tensors) on the index's device: d_indptr int64[n_q+1], d_rows int64[n_pairs], d_scores float32[n_pairs], and
 * for Jaccard d_inter / d_uni int32[n_pairs] (NULL on a TF-IDF index, as for the host fetch).  They consume the result
 * like the host fetch and return once the work on the handle's stream is complete.  KV_ERR_STATE when there is no
 * result (none computed, fetched already, or dropped by a later upload); KV_ERR_INVALID for count outputs that do not
 * fit the index's mode, or when a pointer is not device memory of the index's device aligned to its element size (the
 * arrays of n_pairs elements are not looked at when n_pairs == 0).  KV_ERR_NOMEM (with the pair count) when the
 * ordering's scratch -- about the pair buffer's size again -- does not fit; the result then stays for another try. */
int kv_range_fetch_device(kv_index *ix, void *d_indptr, void *d_rows, void *d_scores, void *d_inter, void *d_uni);

/* The relative margin of the exact threshold search's float32 stage.  It rests on the assumption the store's
 * candidate check (AMBIGUITY_RTOL) makes too: the float32 score of a pair (K1b, and the float64 fallback of irregular
 * queries rounded once) lies within this relative distance of its K6 float64 score; DESIGN §3 reports 6e-8 observed.
 * So a float32 search at threshold * (1 - margin) finds every pair whose K6 score reaches threshold. */
#define KV_RANGE_EXACT_MARGIN 4e-6

/* Exact threshold search over the resident batch: every (query, row) pair whose K6 float64 score -- the value
 * kv_rescore_pairs gives the pair, bit for bit -- is >= threshold, 0 < threshold <= 1.  It decides membership with the
 * float64 arithmetic of the reference's scores, where kv_range_resident decides it with the float32 top-k score.
 *   1. The float32 search of kv_range_resident (label, tag and exclusion filters, deletions) at the largest float32
 *      <= threshold * (1 - KV_RANGE_EXACT_MARGIN): the candidates, *n_candidates (may be NULL) their count.
 *   2. K6-R: every candidate gets its K6 score on the device, one warp per pair, and the pairs whose score is
 *      >= threshold are kept: *n_pairs.  Rows with identical text tie exactly, on any index.
 * q_indptr / q_ids / q_tf / q_oov_tf2 (host, n_q queries) are the resident batch's query CSR, as kv_rescore_pairs gets
 * it; n_q must be the batch's query count.  The result stays in the handle until kv_range_fetch_exact(_device), the
 * next upload, search, append, deletion or finalize.  The resident batch, its filters, exclusions and top-k thresholds
 * are left as they were.  kv_index_last_kernel_ms: [0] = K6-R with its compaction, [2]-[4] as kv_range_resident.
 * KV_ERR_INVALID: threshold NaN, <= 0 or > 1, a Jaccard index (mode 1), a batch from kv_selfjoin_upload, n_q not the
 * batch's count, a bad CSR.  KV_ERR_STATE: not finalized, no resident batch.  KV_ERR_NOMEM as kv_range_resident. */
int kv_range_resident_exact(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                            const double *q_oov_tf2, int64_t n_q, double threshold, int64_t *n_pairs,
                            int64_t *n_candidates);
/* The exact result: indptr[n_q+1] by original query, rows[n_pairs] (global), scores[n_pairs] (float64, K6), per query
 * ordered by (score desc, row asc), on the device by the radix sort of the float32 results extended to a 64-bit score
 * key (on one host core below 8192 pairs plus queries, the same bits).  Consumption, KV_ERR_NOMEM, a second fetch and,
 * for the _device form, the device-pointer checks (d_scores aligned to 8 bytes) are those of kv_range_fetch /
 * kv_range_fetch_device.  A float32 result (kv_range_resident) is not fetched here, nor an exact one by the float32
 * fetches: KV_ERR_STATE, and the result stays. */
int kv_range_fetch_exact(kv_index *ix, int64_t *indptr, int64_t *rows, double *scores);
int kv_range_fetch_exact_device(kv_index *ix, void *d_indptr, void *d_rows, void *d_scores);

/* K6: float64 scores of selected (query, row) pairs: rows[n_q*k] are GLOBAL row ids (e.g. what a top-k returned;
 * -1 = unused slot), out_scores[n_q*k] (host) receives the float64 cosine of SimilarityEngine.score
 * (similarity.py:14-20) for that row, -inf for unused slots and rows that live on another shard.  Summation follows
 * the row's stored feature order with nothing folded, so rows with identical text get identical bits on every shard /
 * segment and services/gfkb/app.py:89's stable sort is reproduced (ties -> lower row).  The batched match path ranks
 * candidates in float32 (K1b) and re-scores the survivors here. */
int kv_rescore_pairs(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                     const double *q_oov_tf2, int64_t n_q, int k, const int64_t *rows, double *out_scores);

/* Exact top-k of this index alone, with no candidate stage: per query K1a scores every row in float64 on the device,
 * the block-wide selection of the irregular-query fallback takes the best k rows in (float64 score desc, row asc)
 * order -- labels[q] >= 0: rows of that label only (kv_index_set_row_labels; labels NULL or -1: any row); distinct:
 * the first row of each group (kv_index_set_row_groups); deleted rows never --, and K6 re-scores those rows.
 * out_rows[n_q*k] (host) receives GLOBAL rows in that order, -1 past the last eligible row, and out_scores[n_q*k] their
 * K6 float64 scores (-inf for unused slots).  Only the k rows of a query leave the device, not its score vector.  K6 and
 * not K1a gives the reported scores because K1a's bits depend on the index by about 2^-50 (its fixed-point scales and
 * folded features are per index) while K6's depend only on the row's text: identical texts on different shards or
 * segments then tie exactly, and a merge of several indexes' lists by (score desc, row asc) reproduces
 * services/gfkb/app.py:89's stable sort.  k 1..32; a filtered query without row labels, or distinct without row groups:
 * KV_ERR_STATE.  The resident batch is left as it was. */
int kv_exact_topk(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                  const double *q_oov_tf2, const int32_t *labels, int distinct, int64_t n_q, int k, int64_t *out_rows,
                  double *out_scores);
/* kv_exact_topk with a tag set per query (tag_indptr[n_q+1] from 0, tags; NULL: no query has tags), validated as by
 * kv_query_set_tag_filter: a query with tags takes only the rows whose tag set meets its own.  A query with tags on an
 * index without current row tags: KV_ERR_STATE. */
int kv_exact_topk_tags(kv_index *ix, const int64_t *q_indptr, const uint32_t *q_ids, const uint32_t *q_tf,
                       const double *q_oov_tf2, const int32_t *labels, const int64_t *tag_indptr, const int32_t *tags,
                       int distinct, int64_t n_q, int k, int64_t *out_rows, double *out_scores);

/* Cross-GPU pruning thresholds for a row-sharded GFKB (one process per GPU, all ranks hold the SAME resident query
 * batch).  Block-max pruning needs a lower bound of every query's GLOBAL k-th score; a shard scanning alone only knows
 * its own.  export: make this index's threshold array (int32 float bits per sorted query slot, `capacity` queries)
 * visible to the other processes -- writes a 64-byte CUDA IPC handle.  peers: map the arrays the other ranks exported
 * (n_peers <= 7 handles of 64 bytes, same capacity); from then on every bound a scan CTA establishes is also pushed
 * into the peers' arrays with system-scope reductions over NVLink/NVSwitch peer memory while the kernels run, so all
 * shards prune with the best bound known anywhere (n_peers = 0 unmaps).  Results are unchanged -- a pushed value
 * always is a valid lower bound (k rows at least that good exist in some shard) -- only less is scanned.  Callers must
 * keep scans of different batches apart with a collective (the all-gather of partial top-k does that) and exchange
 * again after uploading a batch larger than `capacity` (kv_topk_resident* returns KV_ERR_STATE otherwise).
 * Contract: every rank holds the same resident batch WITH THE SAME FILTER AND DISTINCT MODE (kv_query_set_filter,
 * kv_query_set_distinct).  Then a pushed value is the k-th score of a list of rows of the query's label -- of k distinct
 * groups in distinct mode -- and bounds the query's global (filtered, distinct) k-th score.  For a distinct batch the
 * seed k-th score given to kv_index_raise_thresholds is taken over distinct groups (kv_merge_topk_distinct_device_on). */
int kv_index_thresholds_export(kv_index *ix, int64_t capacity, void *handle_out);
int kv_index_thresholds_peers(kv_index *ix, const void *handles, int n_peers, int64_t capacity);
/* Test hook: what kv_index_thresholds_peers does, for indexes of one process on one device (no CUDA IPC): ix pushes
 * into the threshold arrays of `peers`, each exported before with at least `capacity` queries.  n_peers = 0 unlinks. */
int kv_debug_thresholds_link(kv_index *ix, kv_index *const *peers, int n_peers, int64_t capacity);

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
/* K5 of a distinct batch (kv_query_set_distinct) over lists of several indexes, e.g. the row shards' lists after the
 * all-gather, laid out as for kv_merge_topk_device_on (1..2048 lists, k 1..32, global rows, -1 = unused).
 * d_row_groups: device int32[n_group_rows], the group of every GLOBAL row (row_base 0), owned by the caller.  Output as
 * the single index's distinct top-k: in (score desc, row asc) order the first entry of each group, (-inf, -1) past the
 * last group; exact across shards, since a group of the merged top-k is in the top-k of the list holding its best row.
 * Runs on `stream` and returns once the outputs and their validity are known.  KV_ERR_INVALID for bad counts or
 * strides, pointers that are not device memory of `device` aligned to their element size, and -- after the fact, the
 * outputs then undefined -- a row outside [0, n_group_rows), whose group is never read. */
int kv_merge_topk_distinct_device_on(int device, const void *d_scores_in, const void *d_rows_in, int n_lists,
                                     int64_t n_q, int k, int64_t stride_s, int64_t stride_r,
                                     const void *d_row_groups, int64_t n_group_rows, void *d_scores_out,
                                     void *d_rows_out, void *stream);

/* Merge of n_runs (1..64) threshold-search results over disjoint rows -- e.g. the row shards' results after ONE
 * all-gather -- into the single result over all the rows.  Run w is a CSR as kv_range_fetch_device writes it:
 * indptr int64[n_q+1] at d_indptr + w*indptr_stride elements, with indptr[0] = 0 and indptr[n_q] = run_pairs[w] (host
 * array); rows int64 / scores float32 (and, for Jaccard results, inter / uni int32: both set or both NULL) at their
 * base + w*rec_stride_bytes bytes (a multiple of 8); each query's segment ordered by (score desc, row asc).  Writes
 * d_indptr_out int64[n_q+1] (the summed counts) and the pairs of every query, the union of its segments in the same
 * order, to d_rows_out / d_scores_out (/ d_inter_out / d_uni_out), all device memory of `device` (the record
 * arrays are not looked at when no run holds a pair).  Runs on `stream`
 * (a cudaStream_t, e.g. the all-gather's; NULL = legacy default stream) and returns once the outputs and their
 * validity are known.  KV_ERR_INVALID, after the fact, for a decreasing indptr, a count that does not match run_pairs,
 * a segment out of order or a (score, row) key present in two runs (the outputs are then undefined); for pointers
 * that are not device memory of `device` aligned to their element size.  KV_ERR_NOMEM for 2^32 - 1 pairs or more. */
int kv_merge_range_device_on(int device, int n_runs, int64_t n_q, const void *d_indptr, int64_t indptr_stride,
                             const void *d_rows, const void *d_scores, const void *d_inter, const void *d_uni,
                             int64_t rec_stride_bytes, const int64_t *run_pairs, void *d_indptr_out, void *d_rows_out,
                             void *d_scores_out, void *d_inter_out, void *d_uni_out, void *stream);

/* Timing of the last query upload and top-k (kv_topk_resident, _host or _finish) on this handle, CUDA-event
 * milliseconds on its stream:
 * ms[0] = H2D of the query batch, ms[1] = bound + scan kernels, ms[2] = merge (+ fallbacks), ms[3] = D2H of host
 * outputs. */
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
 * kv_range_fetch (host); inter / uni are only written for Jaccard records.  Records with a query outside
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
 * (the bound kernel's epilogue adds those per block from the second-class bitmaps), [18] = slots of the per-block rare
 * tables (16 bytes each), [19] = rare tables the finalize enlarged past load 0.4 because cuckoo insertion failed. */
int kv_index_layout(const kv_index *ix, int64_t bytes[4], int64_t counts[20]);

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
/* Dense tag filter (e.g. a failure's affected apps), with the semantics of kv_index_set_row_tags /
 * kv_query_set_tag_filter.  kv_dense_set_row_tags gives every local row a SET of tags >= 0, any number, possibly none:
 * row r holds tags[indptr[r] .. indptr[r+1]), indptr[n+1] starting at 0, n == kv_dense_rows; NULL clears.  Row tags
 * have the lifetime of the row labels: set before or after finalize, kept by finalize and deletions, dropped by an
 * append; setting them on a finalized index needs no finalize.
 * kv_dense_set_tag_filter gives each query of THE NEXT SEARCH CALL on the handle a set of at most 16 tags (same CSR
 * form; an empty set: no tag constraint), with the lifetime of kv_dense_set_query_filter: that call must have exactly
 * n_q queries (else KV_ERR_INVALID) and clears it whether it succeeds or fails; an append or a finalize clears it too;
 * NULL clears.  A query with tags matches only the rows whose set meets its own (any of its tags); the label filter,
 * deletions and self-join exclusions apply as well.  Its top-k is the top-k over its eligible live rows -- (score desc,
 * row asc), the same float32 scores as unfiltered, (-inf, -1) past the last eligible row -- and its threshold search
 * returns the unfiltered pairs whose rows are eligible.  The kernel skips every (128-query tile, 256-row tile) item
 * whose row tile carries no tag of a query of the query tile (a 64-bit signature of bit t & 63 per tag over the live
 * rows; a query tile holding a query without tags skips nothing this way, since that query matches untagged rows
 * too), then tests each row's mask and, when the index holds a tag >= 64, its exact set.
 * KV_ERR_INVALID: wrong counts, indptr not starting at 0 or decreasing, a negative tag, more than 16 tags on a query.
 * KV_ERR_STATE: a search with a tagged query on an index whose row tags are missing or stale (appended rows). */
int kv_dense_set_row_tags(kv_dense_index *dx, const int64_t *indptr, const int32_t *tags, int64_t n);
int kv_dense_set_tag_filter(kv_dense_index *dx, const int64_t *indptr, const int32_t *tags, int64_t n_q);
/* Measurement and test hook: the (query tile, row tile) items the last dense search's kernel skipped, by the label or
 * the tag signature, and its total items (q_tiles x r_tiles; skipped is 0 for an unfiltered search). */
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
