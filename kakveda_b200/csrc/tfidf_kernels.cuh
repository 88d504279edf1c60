// Device code of the TF-IDF cosine index: finalize kernels, query preparation, K1a (one query, float64 scores of
// every row), K1b-S (exact scan of candidate (query, chunk) pairs with fused top-k), K5 (list merge), K6 (float64
// re-scoring).  The bound kernel K1b-B (wgmma) lives in bound_kernel.cuh.  Included by tfidf_index.cu only.
//
// Math (SURVEY.md section 7, restating sklearn text.py:1650-1739 + pairwise.py:1742-1752 as called
// by services/shared/similarity.py:14-20).  The reference refits TF-IDF on [query]+corpus per
// call; with N corpus rows and corpus document frequency df(t):
//   idf_b(t) = ln((N+2)/(df(t)+1)) + 1      feature t of a row that is NOT in the query
//   idf_q(t) = ln((N+2)/(df(t)+2)) + 1      feature t that IS in the query (the fit saw it once more)
//   B_c      = sum_{t in c} (tf_c(t) idf_b(t))^2                        query independent
//   dot      = sum_{t in q∩c} tf_q(t) tf_c(t) a(t),          a(t) = idf_q(t)^2
//   corr     = sum_{t in q∩c} tf_c(t)^2 d(t),                d(t) = idf_q(t)^2 - idf_b(t)^2  (< 0)
//   |q|^2    = sum_{t in q} (tf_q(t) idf_q(t))^2   (out-of-vocabulary features: df = 0)
//   score    = dot / sqrt(|q|^2 (B_c + corr)),  0 when either side has no feature.
//
// Scan layout in HBM (built by finalize; "position" = index of a row in (norm class, text) order):
//   * rows are sorted by (norm class, feature-id sequence = token order): rows with similar text are neighbours;
//     perm[position] is the original row; a CHUNK is 32 consecutive positions (one row per lane);
//   * features present in EVERY local row with one common tf ("universal": the field names of signature_text,
//     fingerprint.py:60-65) are folded into per-query constants -- in fixed point, the exact integers the unfolded
//     entries would add (see below);
//   * per chunk one feature-major COLUMN BLOCK: the distinct (feature, tf) pairs of its rows, each with the 32-bit
//     mask of the rows that hold it:  words[E] = [31] every valid row holds it  [30:5] feature id  [4:0] tf (31 =
//     see overflow table), masks[E].  A query is scored against a chunk by probing the E words in its own hash table
//     and adding each hit's weight to the rows of its mask -- a third of the entries a row-major stream needs, and
//     the per-row sums are INTEGERS (fixed point, see below), so the order of the additions is irrelevant: rows
//     with identical text get identical bits wherever they sit -- in any row shard too, whichever features its index
//     folds, since a folded feature adds the same integer as its entries would -- and the (score desc, row asc) order
//     of services/gfkb/app.py:89 is reproduced for duplicate rows;
//   * entries of the NF = 256 features found in most chunks ("frequent") come last in a block; for them a dense
//     fp16 matrix Uf[chunk][256] holds the largest tf in the chunk -- the tensor-core part of the chunk bounds;
//   * B32/B64: row norms B_c by position, chunk_minB: smallest positive norm of a chunk.
//
// Fixed point: a query's weights are w(t) = round(tf_q a(t) 2^32) (64-bit) and c(t) = round(-d(t) 2^24); a row's sums
// are exact integer sums of tf_c w(t) and tf_c^2 c(t), the universal features' u w(t) and u^2 c(t) included (u: their
// common tf).  Relative resolution 2^-32 per term (float32 has 2^-24).
#pragma once
#include "kv_cuda.cuh"
#include "sm90.cuh"
#include "tag_sets.cuh"

#include <cuda_fp16.h>

namespace kvk {

constexpr int CHUNK_ROWS = 32;
constexpr int NF = 256;   // features evaluated densely (tensor cores) by the bound kernel
constexpr int NF2 = 1024; // the next most frequent features: per 64-chunk block two transposed bitmaps [NF2][tf >= 1, tf >= 2][64 bits]
constexpr int Q2CAP = 24; // features of that class a query keeps in its own list (further ones are treated as rare)
constexpr int KT2 = 256;  // columns of a bound tile's second-class dictionary (extra K of the bound GEMM)
constexpr uint32_t FID_BITS = 26;
constexpr uint32_t FID_MASK = (1u << FID_BITS) - 1;
constexpr uint32_t FID_NONE = FID_MASK;  // sentinel feature id (never in a table)
constexpr uint32_t KEY_EMPTY = 0xFFFFFFFFu;
constexpr uint32_t W_ALL = 0x80000000u;  // block word flag: every valid row of the chunk holds the entry
constexpr uint32_t TF_OVF = 31;
constexpr uint32_t FULL = 0xFFFFFFFFu;
constexpr uint32_t PAD_WORD = (FID_NONE << 5) | 1u;
constexpr int QKEYS = 128;   // hash slots of a query's own table (K1b-S)
constexpr int QFEATS = 64;   // features a query may hold in it (more: float64 full-scan path)
constexpr int QTAB_BYTES = QKEYS * 4 + QFEATS * 16;
constexpr int GROUP_Q = 32;  // queries per scan group (one candidate list, one K1b-S CTA)
constexpr int TILE_Q = 128;  // queries per bound tile (4 groups; the M of the bound GEMM)
constexpr int Q3CAP = 32;       // rare features a query keeps in its own list for the bound kernel (further ones: a constant)
constexpr int RB_BITS = 1 << 16;  // per 64-chunk block: presence bitmap of its rare features (one hash), probed before the block's table
constexpr float PRUNE_SLACK = 1.0005f;  // bounds: fp16 round-up of weights, fp32 tensor-core sums, constants rounded outwards
constexpr float FILTER_SLACK = 0.999996f;
constexpr int PAGE_RECS = 1024;  // candidate records per pool page

struct BlockInfo {
  uint32_t off4;       // offset of the block in 16-byte units
  uint16_t n_entries;  // entries of the block, ordered [rare][second class][frequent], each part sorted by (feature, tf)
  uint16_t n_rare;     // leading entries of features in neither dense class (what the bound kernel's join probes)
  uint16_t n_f2;       // following entries of second-class features (bitmaps in the bound kernel)
  uint16_t pad;
};

// ----------------------------------------------------------------------------------------
// finalize kernels
// ----------------------------------------------------------------------------------------
__global__ void hist_kernel(const uint32_t *__restrict__ ids, const uint16_t *__restrict__ tf, int64_t nnz,
                            uint32_t *cnt, uint32_t *tfmin, uint32_t *tfmax) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < nnz; p += (int64_t)gridDim.x * blockDim.x) {
    uint32_t t = ids[p], f = tf[p];
    atomicAdd(&cnt[t], 1u);
    if (tfmin) {
      atomicMin(&tfmin[t], f);
      atomicMax(&tfmax[t], f);
    }
  }
}

struct IdfTables {
  double *a64, *d64, *bb64;
  uint8_t *univ;
  uint32_t *utf;
};

__global__ void idf_kernel(const uint32_t *__restrict__ df, const uint32_t *__restrict__ cnt,
                           const uint32_t *__restrict__ tfmin, const uint32_t *__restrict__ tfmax, int64_t V,
                           int64_t n_total, int64_t n_local, int jaccard, int corpus_fit, IdfTables T) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= V) return;
  // corpus_fit: TF-IDF fitted on the corpus alone (the query is only transformed): one idf for both sides
  double num = (double)(n_total + (corpus_fit ? 1 : 2));
  double ib = jaccard ? 1.0 : log(num / ((double)df[t] + 1.0)) + 1.0;  // Jaccard: every token weighs 1
  double iq = jaccard ? 1.0 : (corpus_fit ? ib : log(num / ((double)df[t] + 2.0)) + 1.0);
  double a = iq * iq, bb = ib * ib;
  // corpus_fit: a feature no live row holds (all its rows deleted) is outside the vocabulary a fit on the corpus
  // would learn, so the query ignores it like an out-of-vocabulary feature (idf_host does the same)
  if (corpus_fit && !jaccard && df[t] == 0) a = bb = 0.0;
  T.a64[t] = a; T.d64[t] = a - bb; T.bb64[t] = ib * ib;
  bool u = n_local > 0 && (int64_t)cnt[t] == n_local && tfmin[t] == tfmax[t];
  T.univ[t] = u ? 1 : 0;
  T.utf[t] = u ? tfmin[t] : 0;
}

// Row deletion (kv_index_delete_rows): cnt[t] += entries of feature t in the listed rows -- one warp per listed row.
// cnt minus this histogram is the live document frequency.
__global__ void hist_rows_kernel(const int64_t *__restrict__ indptr, const uint32_t *__restrict__ ids,
                                 const int *__restrict__ rows, int64_t n, uint32_t *cnt) {
  const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;
  const int r = rows[i];
  for (int64_t p = indptr[r] + (threadIdx.x & 31); p < indptr[r + 1]; p += 32) atomicAdd(&cnt[ids[p]], 1u);
}

__global__ void sub_count_kernel(const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, int64_t n, uint32_t *out) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t < n) out[t] = a[t] - b[t];
}

// Live word of every chunk: bit i set when the row at position 32c + i exists and is not deleted (dead: by row)
__global__ void alive_kernel(const int *__restrict__ perm, const uint8_t *__restrict__ dead, int64_t n_rows,
                             int64_t n_chunks_pad, uint32_t *alive) {
  const int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (c >= n_chunks_pad) return;
  uint32_t m = 0;
  for (int i = 0; i < CHUNK_ROWS; i++) {
    const int64_t pos = c * CHUNK_ROWS + i;
    if (pos < n_rows && !dead[perm[pos]]) m |= 1u << i;
  }
  alive[c] = m;
}

// one warp per position: B_c
__global__ void rownorm_kernel(const int64_t *__restrict__ indptr, const uint32_t *__restrict__ ids,
                               const uint16_t *__restrict__ tf, const int *__restrict__ perm, int64_t n_rows,
                               const double *__restrict__ bb64, double *B64, float *B32) {
  int64_t pos = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (pos >= n_rows) return;
  const int64_t r = perm ? perm[pos] : pos;
  // B_c is summed in entry order by one lane-strided pass + a fixed shuffle tree: rows with equal
  // text get the same bits
  double b = 0.0;
  for (int64_t p = indptr[r] + lane; p < indptr[r + 1]; p += 32) {
    uint32_t t = ids[p];
    double f = (double)tf[p];
    b += f * f * bb64[t];
  }
  for (int o = 16; o; o >>= 1) b += __shfl_xor_sync(FULL, b, o);
  if (lane == 0) {
    B64[pos] = b;
    B32[pos] = (float)b;
  }
}

// chunk_minB[c] for c < n_chunks; +inf for the padding chunks up to n_pad (and for chunks without a positive norm:
// rows without features always score 0, they do not loosen a bound).  alive (NULL: no row deleted): deleted rows are
// never returned, so they do not loosen a bound either -- an all-deleted chunk's bound is 0.
__global__ void chunk_meta_kernel(const float *__restrict__ B32, int64_t n_rows, int64_t n_chunks, int64_t n_pad,
                                  const uint32_t *__restrict__ alive, float *chunk_minB) {
  int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (c >= n_pad) return;
  float m = INFINITY;
  if (c < n_chunks) {
    const int64_t r = c * CHUNK_ROWS;
    const uint32_t live = alive ? alive[c] : FULL;
    for (int64_t i = r; i < r + CHUNK_ROWS && i < n_rows; i++)
      if (B32[i] > 0.f && ((live >> (i - r)) & 1u)) m = fminf(m, B32[i]);
  }
  chunk_minB[c] = m;
}

__global__ void fill_int_kernel(int *p, int64_t n, int v) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void fill_ll_kernel(long long *p, int64_t n, long long v) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// gthr[slot] = max(gthr[slot], kth[query of the slot]) for positive scores (float bits order like ints)
__global__ void raise_thresholds_kernel(const float *__restrict__ kth, const int *__restrict__ qperm, int64_t n_q, int *gthr) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n_q) return;
  const float v = kth[qperm[i]];
  if (v > 0.f) atomicMax(&gthr[i], __float_as_int(v));
}

__global__ void invperm_kernel(const int *__restrict__ perm, int64_t n, int *invperm) {
  const int64_t pos = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (pos < n) invperm[perm[pos]] = (int)pos;
}

// Row labels in scan order (kv_index_set_row_labels): label_pos[pos] = label of the row at position pos, -1 past the
// last row (label_pos holds n_chunks_pad * 32 entries)
__global__ void label_pos_kernel(const int *__restrict__ perm, const int *__restrict__ labels, int64_t n_rows, int64_t n_pos,
                                 int *label_pos) {
  const int64_t pos = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (pos < n_pos) label_pos[pos] = pos < n_rows ? labels[perm[pos]] : -1;
}

// chunk label signature: bit (label & 63) of every label a row of the chunk carries.  No false negatives, so a chunk
// whose signature lacks a query's bit holds no row of that query's label.
__global__ void chunk_sig_kernel(const int *__restrict__ label_pos, int64_t n_chunks_pad, unsigned long long *sig) {
  const int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (c >= n_chunks_pad) return;
  unsigned long long m = 0;
  for (int i = 0; i < CHUNK_ROWS; i++) {
    const int l = label_pos[c * CHUNK_ROWS + i];
    if (l >= 0) m |= 1ull << (l & 63);
  }
  sig[c] = m;
}

// ---- tag sets (kv_index_set_row_tags / kv_query_set_tag_filter): MAX_QTAGS and tags_meet in tag_sets.cuh; here the
// rows' tags are indexed by scan position ----

// chunk tag signature: OR of the masks of the chunk's live rows (alive NULL: every row is live)
__global__ void chunk_tag_sig_kernel(const unsigned long long *__restrict__ mask_pos, const uint32_t *__restrict__ alive,
                                     int64_t n_chunks_pad, unsigned long long *sig) {
  const int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (c >= n_chunks_pad) return;
  const uint32_t live = alive ? alive[c] : FULL;
  unsigned long long m = 0;
  for (int i = 0; i < CHUNK_ROWS; i++)
    if ((live >> i) & 1u) m |= mask_pos[c * CHUNK_ROWS + i];
  sig[c] = m;
}

// The rows one tag-filtered query may not match, for the float64 fallbacks: out[row] = 1 when the row is deleted
// (dead, NULL: none) or its tag set misses the query's (q_mask, q_tags)
__global__ void tag_dead_kernel(const int *__restrict__ invperm, int64_t n_rows, const unsigned long long *__restrict__ mask_pos,
                                const int64_t *__restrict__ tag_ptr, const int *__restrict__ tag_list, unsigned long long q_mask,
                                const int *__restrict__ q_tags, const uint8_t *__restrict__ dead, uint8_t *out) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const int64_t pos = invperm[r];
  out[r] = (dead && dead[r]) || !tags_meet(mask_pos[pos], q_mask, tag_ptr, tag_list, pos, q_tags);
}

// ----------------------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t hash_fid(uint32_t fid, int log_h) { return (fid * 0x9E3779B1u) >> (32 - log_h); }

// tf of a block entry whose 5-bit field overflowed: sorted table keyed by (chunk << 32 | entry index)
__device__ uint32_t ovf_lookup(const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ vals,
                               int n, int64_t chunk, uint32_t entry) {
  unsigned long long key = ((unsigned long long)chunk << 32) | entry;
  int lo = 0, hi = n - 1;
  while (lo <= hi) {
    int mid = (lo + hi) >> 1;
    unsigned long long k = keys[mid];
    if (k == key) return vals[mid];
    if (k < key) lo = mid + 1; else hi = mid - 1;
  }
  return TF_OVF;  // unreachable for a consistent index
}

__device__ __forceinline__ uint32_t lanemask_lt() {
  uint32_t v;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(v));
  return v;
}

// ----------------------------------------------------------------------------------------
// K1a: one query against every row, float64 (the drop-in SimilarityEngine.score path).  One warp per chunk: the
// lanes probe the block's entries in the query table, every hit adds its fixed-point weight to the rows of its
// mask; lane = row.
// ----------------------------------------------------------------------------------------
struct ScoreParams {
  const uint32_t *blk;
  const BlockInfo *binfo;
  const int *perm;
  int64_t n_chunks, n_rows;
  const double *B64;
  const unsigned long long *ovf_keys;
  const uint32_t *ovf_vals;
  int n_ovf;
  // query table (global memory): keys[H], then w[H] = round(tf_q a(t) 2^e), c[H] = round(-d(t) 2^e2)  (64-bit)
  const uint32_t *qkeys;
  const unsigned long long *qw, *qc;
  int log_h;
  double w_unscale, c_unscale;  // 2^-e, 2^-e2
  double nq, dotU, corrU;
  int jaccard;
  const uint8_t *dead;  // by ORIGINAL row, NULL: no row deleted (a deleted row scores -inf)
  double *out;  // by ORIGINAL row
};

__global__ void __launch_bounds__(256) tfidf_score_kernel(ScoreParams P) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int H = 1 << P.log_h;
  unsigned long long *s_w = (unsigned long long *)smem_raw;
  unsigned long long *s_c = s_w + H;
  uint32_t *s_k = (uint32_t *)(s_c + H);
  // per-warp hit buffer: up to 32 hits of one probe round
  struct Hit { unsigned long long w, c; uint32_t m, pad; };
  Hit *s_hits = (Hit *)(s_k + H) + (threadIdx.x >> 5) * 32;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    s_k[i] = P.qkeys[i];
    s_w[i] = P.qw[i];
    s_c[i] = P.qc[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const uint32_t lt = lanemask_lt();
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp; c < P.n_chunks; c += n_warps) {
    const BlockInfo bi = P.binfo[c];
    const int E = bi.n_entries, E4 = (E + 3) & ~3;
    const uint32_t *words = P.blk + (size_t)bi.off4 * 4, *masks = words + E4;
    const int64_t pos0 = c * CHUNK_ROWS;
    const int rows = (int)min((int64_t)CHUNK_ROWS, P.n_rows - pos0);
    const uint32_t valid = rows == 32 ? FULL : ((1u << rows) - 1u);
    unsigned long long acc_w = 0, acc_c = 0;
    for (int e0 = 0; e0 < E; e0 += 32) {
      const int e = e0 + lane;
      const uint32_t w = e < E ? __ldg(words + e) : PAD_WORD;
      const uint32_t fid = (w >> 5) & FID_MASK;
      bool hit = false;
      uint32_t h = 0;
      if (fid != FID_NONE) {
        h = hash_fid(fid, P.log_h);
        for (;;) {
          const uint32_t k = s_k[h];
          if (k == KEY_EMPTY) break;
          if (k == fid) { hit = true; break; }
          h = (h + 1) & (H - 1);
        }
      }
      const uint32_t hm = __ballot_sync(FULL, hit);
      if (hm == 0) continue;
      if (hit) {
        uint32_t tf = w & 31u;
        if (tf == TF_OVF) tf = ovf_lookup(P.ovf_keys, P.ovf_vals, P.n_ovf, c, (uint32_t)e);
        Hit r;
        r.m = (w & W_ALL) ? valid : __ldg(masks + e);
        r.w = s_w[h] * (unsigned long long)tf;
        r.c = s_c[h] * (unsigned long long)tf * (unsigned long long)tf;
        r.pad = 0;
        s_hits[__popc(hm & lt)] = r;
      }
      __syncwarp();
      const int nh = __popc(hm);
      for (int i = 0; i < nh; i++) {
        const Hit r = s_hits[i];
        if ((r.m >> lane) & 1u) { acc_w += r.w; acc_c += r.c; }
      }
      __syncwarp();
    }
    if (lane < rows) {
      const double dot = P.dotU + (double)acc_w * P.w_unscale;
      const double corr = P.corrU - (double)acc_c * P.c_unscale;
      const double B = P.B64[pos0 + lane];
      double sc;
      if (P.jaccard) {
        const double den = P.nq + B - dot;
        sc = (den > 0.0 && dot != 0.0) ? dot / den : 0.0;
      } else {
        const double den = P.nq * (B + corr);
        sc = (den > 0.0 && dot != 0.0) ? dot / sqrt(den) : 0.0;
      }
      const int row = P.perm[pos0 + lane];
      P.out[row] = (P.dead && P.dead[row]) ? -INFINITY : sc;
    }
  }
}

// ----------------------------------------------------------------------------------------
// query batch preparation (device): per-query constants, the query's own hash table (K1b-S), its row of the dense
// weight matrix Wf (K1b-B), and its lists of second-class and rare features (K1b-B)
// ----------------------------------------------------------------------------------------
struct QFeat {
  uint32_t w_lo, w_hi;  // round(tf_q a(t) 2^32)
  uint32_t cq;          // round(-d(t) 2^24)
  uint32_t tfq;
};

struct PrepParams {
  const int64_t *q_indptr;  // [n_q + 1] by row of the uploaded CSR (device)
  const uint32_t *q_ids, *q_tf;
  const double *q_oov;      // [n_q] or NULL
  const int *qsrc;          // sorted slot -> row of the uploaded CSR
  const uint8_t *flags;     // by sorted slot: 0 regular, 1 null (every score is 0), 2 irregular (float64 full-scan path),
                            // 3 off (a deleted row's self-join query: answered by no path)
  int64_t n_q, V, n_total;
  const double *a64, *d64;
  const uint8_t *univ;
  const uint32_t *utf, *tfmax;
  const short *fslot;       // feature -> column of the dense matrices, -1: not a frequent feature
  const unsigned short *fslot2;  // feature -> bit row of the block bitmaps (second class), 0xFFFF: none
  int jaccard, corpus_fit;
  float *q_nq, *q_dotU, *q_corrU, *q_dotS, *q_corrS, *q_dotX;  // [n_q] by sorted slot
  unsigned long long *q_uw, *q_uc;  // [n_q] universal features in fixed point: sum u w(t), sum u^2 c(t) (the scan's constants)
  float *q_rscale;          // [n_q] 1 / s_q: fixed-point unit of the bound kernel's accumulator R (see below)
  unsigned char *qtab;      // [n_q][QTAB_BYTES]
  __half *Wf;               // [n_q_pad][NF], zeroed by the caller
  uint32_t *q3id, *q3w;     // [n_tiles][Q3CAP][TILE_Q] rare feature id, weight ceil(tf_q a(t) s_q) as an integer
  uint2 *q2list;            // [n_tiles][Q2CAP][TILE_Q] (bit row | (tfmax(t) - 1) << 16, weight tf_q a(t) as float bits)
};

__global__ void prep_queries_kernel(PrepParams P) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= P.n_q) return;
  uint32_t *keys = (uint32_t *)(P.qtab + (size_t)i * QTAB_BYTES);
  QFeat *feats = (QFeat *)(keys + QKEYS);
  for (int j = 0; j < QKEYS; j++) keys[j] = KEY_EMPTY;
  const int q = P.qsrc[i];
  const double idf0 = P.jaccard ? 1.0 : (P.corpus_fit ? 0.0 : log((double)(P.n_total + 2) / 2.0) + 1.0);
  double nq = (P.q_oov ? P.q_oov[q] : 0.0) * idf0 * idf0;
  double dotU = 0.0, corrU = 0.0, corrS = 0.0;
  unsigned long long uw = 0, uc = 0;
  int cnt = 0, c2 = 0;
  const bool regular = P.flags[i] == 0;
  uint2 *q2 = P.q2list + ((size_t)(i / TILE_Q) * Q2CAP) * TILE_Q + (i % TILE_Q);
  for (int j = 0; j < Q2CAP; j++) q2[(size_t)j * TILE_Q] = make_uint2(0u, 0u);
  const size_t q3o = ((size_t)(i / TILE_Q) * Q3CAP) * TILE_Q + (i % TILE_Q);
  uint32_t *q3id = P.q3id + q3o, *q3w = P.q3w + q3o;
  for (int j = 0; j < Q3CAP; j++) { q3id[(size_t)j * TILE_Q] = FID_NONE; q3w[(size_t)j * TILE_Q] = 0u; }
  int c3 = 0;
  float dotX = 0.f;
  double xmax = 0.0;  // upper bound of what the bound kernel sums into R for this query: frequent, listed second-class
                      // and listed rare terms
  for (int64_t p = P.q_indptr[q]; p < P.q_indptr[q + 1]; p++) {
    const uint32_t t = P.q_ids[p];
    const double f = (double)P.q_tf[p];
    if ((int64_t)t >= P.V) { nq += f * f * idf0 * idf0; continue; }  // id issued after finalize: in no indexed row
    const double a = P.a64[t], d = P.d64[t];
    nq += f * f * a;
    if (P.univ[t]) {
      const double u = (double)P.utf[t];
      dotU += f * u * a;
      corrU += u * u * d;
      // exactly what the feature's entries would add to the scan's integer sums (the weights are formed as below)
      const unsigned long long ut = P.utf[t];
      uw += (unsigned long long)__double2ll_rn(f * a * 4294967296.0) * ut;
      uc += (unsigned long long)(uint32_t)__double2ll_rn(-d * 16777216.0) * ut * ut;
    } else if (regular && cnt < QFEATS) {
      const double tm = (double)P.tfmax[t];
      corrS += tm * tm * d;
      uint32_t h = hash_fid(t, 7);
      while (keys[h] != KEY_EMPTY) h = (h + 1) & (QKEYS - 1);
      keys[h] = (t << 6) | (uint32_t)cnt;
      const unsigned long long w = (unsigned long long)__double2ll_rn(f * a * 4294967296.0);
      QFeat qf;
      qf.w_lo = (uint32_t)w; qf.w_hi = (uint32_t)(w >> 32);
      qf.cq = (uint32_t)__double2ll_rn(-d * 16777216.0);
      qf.tfq = P.q_tf[p];
      feats[cnt++] = qf;
      const int fs = P.fslot[t];
      if (fs >= 0) {
        const __half wf = __float2half_ru(__double2float_ru(f * a));
        P.Wf[(size_t)i * NF + fs] = wf;
        xmax += (double)__half2float(wf) * tm;
      } else if (P.fslot2[t] != 0xFFFFu && c2 < Q2CAP) {
        const uint32_t tm1 = min(P.tfmax[t] - 1u, 65535u);  // weight of the 'tf >= 2' plane: (largest tf - 1) more times
        const float w2 = __double2float_ru(f * a * (1.0 + 1e-6));
        q2[(size_t)c2 * TILE_Q] = make_uint2((uint32_t)P.fslot2[t] | (tm1 << 16), __float_as_uint(w2));
        // what a column of the tile's dictionary adds to R (f2_dict_kernel): fp16 weight x fp16 largest tf, both rounded
        // up (a largest tf beyond the fp16 range never takes a column)
        const float th = __half2float(__float2half_ru((float)(tm1 + 1u)));
        if (isfinite(th)) xmax += (double)__half2float(__float2half_ru(w2)) * (double)th;
        c2++;
      } else if (P.fslot2[t] == 0xFFFFu && c3 < Q3CAP) {  // rare: looked up per block of chunks by the bound kernel
        const float w3 = __double2float_ru(f * a * (1.0 + 1e-6));
        q3id[(size_t)c3 * TILE_Q] = t;
        q3w[(size_t)c3 * TILE_Q] = __float_as_uint(w3);  // scaled to an integer below, once s_q is known
        xmax += (double)w3 * tm;
        c3++;
      } else {  // no list slot left: assumed present in every chunk with its largest tf (a valid, loose bound)
        dotX = __fadd_ru(dotX, __double2float_ru(f * a * tm * (1.0 + 1e-6)));
      }
    }
  }
  // Fixed-point scale of R (the bound kernel's frequent + second-class + rare part, summed with integer shared atomics):
  // s_q = 2^(30 - e) with xmax < 2^e, so xmax s_q <= 2^30, and a power of two, so scaling is exact.  No wrap:
  // R[chunk][query] is one MMA term ceil(acc s_q) plus at most Q3CAP rare terms w3 tf with w3 = ceil(weight s_q) <=
  // weight s_q + 1.  The accumulator acc is the fp32 tensor-core sum of fp16 weights times fp16 B values: the chunk's
  // largest tf (frequent features, within 2^-11 of it) or 0 / 1 / the feature's largest tf rounded up to fp16 (the
  // tile's second-class dictionary), each product counted in xmax above with both factors as the GEMM sees them.  A
  // query lists only a subset of its second-class features in the dictionary, so acc <= 1.001 xmax; every tf is at
  // most tfmax(t) <= 65535, so R <= 1.001 xmax s_q + 1 + Q3CAP 65535 < 2^31.  A wrapped sum would LOWER a bound and
  // pruning would drop rows.  xmax < 2^31 for a regular query (classify_queries bounds the sum over every non-universal
  // feature, s_dot amax < 2^30, and fp16 rounding adds at most 2^-10 to each product) and 0 for the others, so s_q
  // and 1 / s_q are normal floats.
  int e = 0;
  frexp(xmax, &e);
  const double s_q = ldexp(1.0, 30 - e);
  for (int j = 0; j < c3; j++) {
    uint32_t &w = q3w[(size_t)j * TILE_Q];
    w = (uint32_t)ceil((double)__uint_as_float(w) * s_q);  // <= xmax s_q: fits
  }
  P.q_rscale[i] = (float)ldexp(1.0, e - 30);
  P.q_nq[i] = regular ? (float)nq : 0.f;  // nq == 0 switches the query off in the kernels
  P.q_dotU[i] = (float)dotU;
  P.q_corrU[i] = (float)corrU;
  P.q_uw[i] = uw;
  P.q_uc[i] = uc;
  P.q_dotS[i] = __double2float_ru(dotU * (1.0 + 1e-6));  // bounds may only err upwards
  P.q_corrS[i] = __double2float_rd(corrU + corrS);       // ... and their denominators downwards
  P.q_dotX[i] = dotX;
}

// ----------------------------------------------------------------------------------------
// second-class dictionary of a bound tile (after prep_queries_kernel): the KT2 bit rows most listed by the tile's 128
// queries (count descending, lower row first: deterministic) become extra K columns of the bound GEMM.  Per column the
// bit row and T = the feature's largest tf rounded up to fp16 (the bound kernel's B value is 0, 1 or T by the block's
// tf >= 1 / tf >= 2 bitmaps); per query its fp16 weight, rounded up, in the A operand Wf2.  The listed features left
// out (only tiles with more than KT2 distinct ones) stay in the query's list, moved to its front: the bound kernel's
// epilogue adds them from the block's bitmaps, as exactly as a dictionary column would.
// ----------------------------------------------------------------------------------------
struct DictParams {
  uint2 *q2list;                  // [n_tiles][Q2CAP][TILE_Q]; on return only the features left out of the dictionary
  __half *Wf2;                    // [n_q_pad][KT2], zeroed by the caller
  uint32_t *d2col;                // [n_tiles][KT2] bit row | fp16 bits of T << 16; 0: unused column
  unsigned long long *n_outside;  // listed (query, feature) incidences left out of their tile's dictionary
};

constexpr int DICT_THREADS = 256;

__global__ void __launch_bounds__(DICT_THREADS) f2_dict_kernel(DictParams P) {
  __shared__ uint32_t cnt[NF2];     // listings of each bit row in the tile
  __shared__ uint16_t th[NF2];      // fp16 bits of T of each listed row
  __shared__ int16_t col_of[NF2];   // column of a row, -1: none
  __shared__ uint32_t keys[NF2];    // listed rows, count << 10 | (NF2 - 1 - row): a larger key ranks first
  __shared__ uint32_t colw[KT2];
  __shared__ uint32_t n_keys;
  __shared__ unsigned int n_out;
  static_assert(NF2 == 1024 && Q2CAP * TILE_Q < (1 << 22), "dictionary key packing");
  const int tile = blockIdx.x;
  for (int r = threadIdx.x; r < NF2; r += DICT_THREADS) { cnt[r] = 0; col_of[r] = -1; }
  for (int c = threadIdx.x; c < KT2; c += DICT_THREADS) colw[c] = 0;
  if (threadIdx.x == 0) { n_keys = 0; n_out = 0; }
  __syncthreads();
  uint2 *q2 = P.q2list + (size_t)tile * Q2CAP * TILE_Q;
  for (int e = threadIdx.x; e < Q2CAP * TILE_Q; e += DICT_THREADS) {
    const uint2 f = q2[e];
    if (!(__uint_as_float(f.y) > 0.f)) continue;
    const __half T = __float2half_ru((float)((f.x >> 16) + 1u));
    if (!__hisinf(T)) {  // a B value of inf would turn the product with a zero weight into NaN
      atomicAdd(&cnt[f.x & 0xFFFFu], 1u);
      th[f.x & 0xFFFFu] = __half_as_ushort(T);  // the same value from every listing of the row
    }
  }
  __syncthreads();
  for (int r = threadIdx.x; r < NF2; r += DICT_THREADS)
    if (cnt[r]) keys[atomicAdd(&n_keys, 1u)] = cnt[r] << 10 | (uint32_t)(NF2 - 1 - r);
  __syncthreads();
  const int nk = (int)n_keys;
  for (int i = threadIdx.x; i < nk; i += DICT_THREADS) {
    const uint32_t k = keys[i];
    int rank = 0;
    for (int j = 0; j < nk; j++) rank += keys[j] > k;
    if (rank < KT2) {
      const int r = NF2 - 1 - (int)(k & (NF2 - 1));
      col_of[r] = (int16_t)rank;
      colw[rank] = (uint32_t)r | (uint32_t)th[r] << 16;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < KT2; c += DICT_THREADS) P.d2col[(size_t)tile * KT2 + c] = colw[c];
  if (threadIdx.x < TILE_Q) {
    const int64_t slot = (int64_t)tile * TILE_Q + threadIdx.x;
    __half *wrow = P.Wf2 + (size_t)slot * KT2;
    uint2 *ql = q2 + threadIdx.x;
    int used = 0, out = 0;
    for (; used < Q2CAP; used++) {  // the lists are filled from the front; padding queries have none
      const uint2 f = ql[(size_t)used * TILE_Q];
      const float w2 = __uint_as_float(f.y);
      if (!(w2 > 0.f)) break;
      const int c = col_of[f.x & 0xFFFFu];
      if (c >= 0) wrow[c] = __float2half_ru(__fadd_ru(__half2float(wrow[c]), w2));
      else ql[(size_t)(out++) * TILE_Q] = f;  // out <= used: never overwrites an entry still to be read
    }
    for (int j = out; j < used; j++) ql[(size_t)j * TILE_Q] = make_uint2(0u, 0u);
    if (out) atomicAdd(&n_out, (unsigned int)out);
  }
  __syncthreads();
  if (threadIdx.x == 0 && n_out) atomicAdd(P.n_outside, (unsigned long long)n_out);
}

__host__ __device__ __forceinline__ uint32_t rb_bit(uint32_t fid) { return (fid * 0x85EBCA6Bu) >> 16; }  // 16 bits: RB_BITS
// slot of a feature in a table of `size` slots (fast range reduction of a multiplicative hash): the first slot of the
// linear-probing tables build_blocks writes on request, and the first of a feature's two slots in a block's rare table
__host__ __device__ __forceinline__ uint32_t rt_slot(uint32_t fid, uint32_t size) {
  return (uint32_t)(((unsigned long long)(fid * 0x9E3779B1u) * (unsigned long long)size) >> 32);
}
__host__ __device__ __forceinline__ uint32_t rt_slot1(uint32_t fid, uint32_t size) { return rt_slot(fid, size); }
// the second slot: an independent multiplier.  A slot of a block's rare table is one uint4 {feature id (KEY_EMPTY: free),
// tf, chunk mask low, high}: tf = the feature's largest tf in the block, or tfmax[feature] when that reaches TF_OVF.
__host__ __device__ __forceinline__ uint32_t rt_slot2(uint32_t fid, uint32_t size) {
  return (uint32_t)(((unsigned long long)(fid * 0xC2B2AE35u) * (unsigned long long)size) >> 32);
}

// ----------------------------------------------------------------------------------------
// K1b-S: exact scan of candidate (query, chunk) pairs with fused top-k.  One CTA = one scan group (32 queries, their
// tables and top-k lists in shared memory) x one range of the group's candidate records {chunk, query mask}.  A warp
// takes a record, stages the chunk's column block into shared memory with a bulk-async copy (TMA, mbarrier
// completion; double buffered, so the next block lands while this one is scored) and scores it for each query of the
// mask: lanes probe 32 block entries at a time in the query's table, hits add their fixed-point weights to the rows
// of their masks, lane = row.  Survivors of the division-free pre-test enter the query's sorted list under a lock.
// In the codes mode (list_mode 3) the records are not read from a list: a warp takes a window of S_WIN chunks, each
// lane reads its query's S_WIN stored bound codes, and a ballot per chunk gives the chunk's query mask -- the warp
// loads the codes of its next window before it scores the records of this one, so the n_q x chunks bytes of codes
// stream in behind the scoring instead of in a separate selection pass that writes the lists to memory.
// K1b-R (RANGE = true) is the same scan for a threshold search: the filter is the query's fixed threshold and every
// row that reaches it is appended to a global pair buffer instead of a top-k list.
// TAGS: the batch has a tag filter.  A record drops the filtered queries whose tags no live row of the chunk carries
// (chunk signature), a (query, record) pair is skipped when no row's mask meets the query's, and a row enters only
// when its set meets the query's (tags_meet).  The instantiations without it compile as before.
// ----------------------------------------------------------------------------------------
struct ScanParams {
  const uint32_t *blk;
  const BlockInfo *binfo;
  const float *B32;
  const int *perm;
  int64_t n_chunks, n_rows, row_base;
  const unsigned long long *ovf_keys;
  const uint32_t *ovf_vals;
  int n_ovf;
  const unsigned char *qtab;              // [n_q][QTAB_BYTES]
  const float *q_nq;                      // [n_q] (sorted query order)
  const unsigned long long *q_uw, *q_uc;  // [n_q] universal features' fixed-point sums (prep_queries_kernel)
  const int *q_excl;                      // [n_q] or NULL: local ORIGINAL row a query must not match (self-join), -1 = none
  // label filter (kv_query_set_filter); q_label NULL: the batch has none and the other two are not read
  const int *q_label;                     // [n_q] label a query's rows must carry, -1 = any
  const int *label_pos;                   // [n_chunks_pad * 32] row label by scan position
  const unsigned long long *chunk_sig;    // [n_chunks_pad] chunk label signatures
  const uint32_t *alive;                  // [n_chunks_pad] live word per chunk (kv_index_delete_rows), NULL: none deleted
  int *gthr;                              // [n_q] float bits: lower bound of the global k-th score
  int *peer_gthr[7];                      // the same array on the other GPUs of a row-sharded GFKB (peer memory over
  int n_peers;                            //   NVLink): a raised bound is pushed to every shard, so all of them prune with it
  // candidate lists: list l = group * n_bsplits + bsplit.  mode 0: paged pool, 1: fixed stride (seed lists),
  // 2: every chunk of the list's chunk range x every query of the group (exhaustive), 3: built in the kernel from the
  // stored bound codes (top-k scan only; n_bsplits 1, the CTAs of a group split its windows of S_WIN chunks)
  int list_mode;
  const unsigned char *ubq;     // mode 3: [n_q][ubq_stride] 8-bit bound codes of bound pass 0
  int64_t ubq_stride;
  const int *tcode;             // mode 3: [n_q] code a chunk's bound needs for the query to take it, 256: none
                                //   (threshold_codes_kernel: a snapshot, fixed while the scan raises gthr)
  const uint32_t *list_count;   // [n_lists]
  const uint32_t *list_pages;   // [n_lists][max_pages]
  int max_pages;
  const uint2 *pool;            // {chunk, query mask}
  const uint2 *direct;          // mode 1: [n_lists][direct_stride]
  int direct_stride;
  int n_bsplits, n_ssplits;
  unsigned long long *stats;    // [0] (query, chunk) pairs scored, [1] records; mode 3 also [2] pairs and [3] records
                                //   that passed the bound (as list_append counts them)
  int64_t n_q;
  int k;
  float *part_scores;  // [n_bsplits * n_ssplits][n_q][k]
  long long *part_rows;
  // threshold search (tfidf_scan_kernel<true>): gthr holds the fixed threshold, k is 0, matches are appended here
  const int *qperm;                  // [n_q] sorted slot -> original query
  RangePair *range_out;              // [range_cap]
  unsigned long long *range_count;   // matches found (may exceed range_cap: those past it are not written)
  unsigned long long range_cap;
  // distinct top-k (tfidf_scan_kernel<false, true>, kv_query_set_distinct): row group by scan position
  const int *group_pos;              // [n_chunks_pad * 32], -1 past the last row
  // tag filter (tfidf_scan_kernel<..., true>, kv_query_set_tag_filter), see tags_meet.  By sorted slot: the query's
  // mask (0: no tag constraint) and ascending tags; by scan position: the row masks and, unless every tag is < 64
  // (tag_ptr NULL), the rows' tags; per chunk the OR of its live rows' masks
  const unsigned long long *q_tmask;     // [n_q]
  const int *q_tags;                     // [n_q][MAX_QTAGS]
  const unsigned long long *tag_mask_pos;  // [n_chunks_pad * 32], 0 past the last row
  const unsigned long long *chunk_tsig;  // [n_chunks_pad]
  const int64_t *tag_ptr;                // [n_chunks_pad * 32 + 1]
  const int *tag_list;
};

// Appends the pairs (*q, score, row) of the lanes with `hit` set: one reservation per warp
__device__ __forceinline__ void range_emit(RangePair *out, unsigned long long *count, unsigned long long cap, bool hit,
                                           const int *q, float score, int64_t row) {
  const uint32_t hm = __ballot_sync(FULL, hit);
  if (hm == 0) return;
  unsigned long long base = 0;
  if ((threadIdx.x & 31) == 0) base = atomicAdd(count, (unsigned long long)__popc(hm));
  base = __shfl_sync(FULL, base, 0);
  if (hit) {
    const unsigned long long o = base + (unsigned long long)__popc(hm & lanemask_lt());
    if (o < cap) out[o] = RangePair{*q, score, row};
  }
}

constexpr int S_WARPS = 12;
constexpr int S_BUF_ENTRIES = 256;  // a staged block holds up to this many entries (larger blocks are read in place)
constexpr int S_BUF_BYTES = S_BUF_ENTRIES * 8;
constexpr int S_WIN = 64;  // codes mode: chunks per window (a lane loads its query's S_WIN codes as four 16-byte loads)
constexpr unsigned long long KTH_NONE = 0xFF8000007FFFFFFFull;  // s_kth of a list that is not full: (-inf, INT_MAX)

// Measuring build of K1b-S (-DKV_SCAN_CLOCKS, profiles/run_scan_split.py): every warp of a codes-mode scan splits its
// life into spans with clock(), counts what it meets, and adds both to g_scan_prof, which kv_debug_scan_profile reads.
// The product build defines none of this and KV_SCAN_PROF(...) expands to nothing.
#ifdef KV_SCAN_CLOCKS
enum {
  KVP_SELECT, KVP_WAIT, KVP_HEAD, KVP_PROBE, KVP_HITPROD, KVP_HITACC, KVP_EPI, KVP_LOCKWAIT, KVP_INSERT, KVP_TAIL,  // cycles
  KVC_PAIRS, KVC_TRIPS, KVC_HITS, KVC_HITS_ALL, KVC_LOCKS, KVC_LOCKS_UNCHANGED, KVC_ROWS_PASSED, KVC_INPLACE, KVC_RECORDS,
  KVC_WARPS, KVC_CTAS, KVC_CTA_PAIRS_MAX, KVP_N,
  KVH_QUERIES = KVP_N,            // [33] records by queries in the mask
  KVH_CTA_PAIRS = KVH_QUERIES + 33,  // [64] CTAs by pairs scored / 512 (last bucket: the rest)
  KVP_TOTAL = KVH_CTA_PAIRS + 64
};
__device__ unsigned long long g_scan_prof[KVP_TOTAL];
#define KV_SCAN_PROF(...) __VA_ARGS__
// charges the cycles since the previous mark to a span (the warp is converged first, lane 0's clock is the warp's)
#define KV_SCAN_MARK(slot) { __syncwarp(); const unsigned int kvp_n = clock(); kvp[slot] += kvp_n - kvp_t; kvp_t = kvp_n; }
#else
#define KV_SCAN_PROF(...)
#define KV_SCAN_MARK(slot)
#endif

// 1-D bulk asynchronous copy global -> shared (TMA engine), completion counted in bytes on an mbarrier
__device__ __forceinline__ void bulk_copy_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst)),
               "l"(src), "r"(bytes), "r"(smem_addr(bar))
               : "memory");
}

// DISTINCT (top-k only): every list entry also carries its row's group (s_lgrp) and a list holds at most one row per
// group, the best one seen.  The warp first keeps the best survivor of each group of the chunk (__match_any_sync), so
// runs of copies -- neighbours in text order -- reach the lock once; under the lock an entry of the new row's group is
// found by a ballot and either kept (the new row is worse) or deleted before the new row is inserted.  A full list
// then holds k distinct groups, so its k-th score stays a lower bound of the k-th group score: the threshold, the
// codes snapshot and the bound passes are unchanged.
template <bool RANGE, bool DISTINCT, bool TAGS = false>
__global__ void __launch_bounds__(S_WARPS * 32, 2) tfidf_scan_kernel(ScanParams P) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int k = P.k;
  uint32_t *s_keys = (uint32_t *)smem_raw;                                  // [GROUP_Q][QKEYS]
  QFeat *s_feats = (QFeat *)(s_keys + GROUP_Q * QKEYS);                     // [GROUP_Q][QFEATS]
  unsigned char *s_buf = (unsigned char *)(s_feats + GROUP_Q * QFEATS);     // [S_WARPS][2][S_BUF_BYTES]
  uint64_t *s_bar = (uint64_t *)(s_buf + S_WARPS * 2 * S_BUF_BYTES);        // [S_WARPS][2]
  unsigned long long *s_kth = (unsigned long long *)(s_bar + S_WARPS * 2);  // [GROUP_Q] k-th entry of a full list
  unsigned long long *s_uw = s_kth + GROUP_Q, *s_uc = s_uw + GROUP_Q;       // [GROUP_Q] per-query fixed-point constants
  float *s_lscore = (float *)(s_uc + GROUP_Q);                              // [GROUP_Q][k]
  int *s_lrow = (int *)(s_lscore + GROUP_Q * k);                            // [GROUP_Q][k]
  int *s_cnt = s_lrow + GROUP_Q * k;                                        // [GROUP_Q]
  int *s_lock = s_cnt + GROUP_Q;                                            // [GROUP_Q]
  float *s_nq = (float *)(s_lock + GROUP_Q);                                // [GROUP_Q] per-query constants
  int *s_excl = (int *)(s_nq + GROUP_Q);
  int *s_qlab = s_excl + GROUP_Q;                                           // [GROUP_Q] label filter, -1 = any
  unsigned int *s_next = (unsigned int *)(s_qlab + GROUP_Q);                // [1] next record of this CTA's range
  unsigned int *s_stat = s_next + 1;                                        // [4]
  int *s_lgrp = (int *)(s_stat + 4);                                        // [GROUP_Q][k] (DISTINCT only)
  unsigned long long *s_qtm = nullptr;                                      // [GROUP_Q] tag masks (TAGS only)
  if constexpr (TAGS)
    s_qtm = (unsigned long long *)(((uintptr_t)(s_lgrp + (DISTINCT ? GROUP_Q * k : 0)) + 7) & ~(uintptr_t)7);

  const int list = blockIdx.x, ssplit = blockIdx.y;
  const int group = list / P.n_bsplits, bsplit = list - group * P.n_bsplits;
  const int64_t q0 = (int64_t)group * GROUP_Q;
  const int q_count = (int)min((int64_t)GROUP_Q, P.n_q - q0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = lanemask_lt();
  bool codes = false;  // list_mode 3
  if constexpr (!RANGE) codes = P.list_mode == 3;

  // record range of this CTA (codes mode: a range of windows)
  uint32_t n_rec;
  uint32_t c_lo = 0;  // chunk indices are 32-bit in this kernel (a chunk is 32 rows)
  if (codes) {
    n_rec = (uint32_t)((P.n_chunks + S_WIN - 1) / S_WIN);
  } else if (P.list_mode == 2) {
    c_lo = (uint32_t)(P.n_chunks * bsplit / P.n_bsplits);
    n_rec = (uint32_t)(P.n_chunks * (bsplit + 1) / P.n_bsplits - c_lo);
  } else {
    n_rec = P.list_count[list];
    if (P.list_mode == 1) n_rec = min(n_rec, (uint32_t)P.direct_stride);
  }
  const uint32_t r_lo = (uint32_t)((unsigned long long)n_rec * ssplit / P.n_ssplits);
  const uint32_t r_hi = (uint32_t)((unsigned long long)n_rec * (ssplit + 1) / P.n_ssplits);

  {  // stage the group's query tables and constants
    const uint4 *src = (const uint4 *)(P.qtab + (size_t)q0 * QTAB_BYTES);
    for (int i = threadIdx.x; i < q_count * (QTAB_BYTES / 16); i += blockDim.x) {
      const int q = i / (QTAB_BYTES / 16), o = i - q * (QTAB_BYTES / 16);
      const uint4 v = src[i];
      if (o < QKEYS / 4) ((uint4 *)(s_keys + q * QKEYS))[o] = v;
      else ((uint4 *)(s_feats + q * QFEATS))[o - QKEYS / 4] = v;
    }
    for (int i = threadIdx.x; i < GROUP_Q * k; i += blockDim.x) {
      s_lscore[i] = -INFINITY;
      s_lrow[i] = 0x7fffffff;
      if constexpr (DISTINCT) s_lgrp[i] = -1;
    }
    if (threadIdx.x < GROUP_Q) {
      const int qi = threadIdx.x;
      const bool ok = qi < q_count;
      s_kth[qi] = KTH_NONE;
      s_cnt[qi] = 0;
      s_lock[qi] = 0;
      s_nq[qi] = ok ? P.q_nq[q0 + qi] : 0.f;
      s_uw[qi] = ok ? P.q_uw[q0 + qi] : 0ull;
      s_uc[qi] = ok ? P.q_uc[q0 + qi] : 0ull;
      s_excl[qi] = (ok && P.q_excl) ? P.q_excl[q0 + qi] : -1;
      s_qlab[qi] = (ok && P.q_label) ? P.q_label[q0 + qi] : -1;
      if constexpr (TAGS) s_qtm[qi] = ok ? P.q_tmask[q0 + qi] : 0ull;
    }
    if (threadIdx.x == 0) { *s_next = r_lo; s_stat[0] = s_stat[1] = s_stat[2] = s_stat[3] = 0; }
    if (lane == 0) {
      mbar_init(&s_bar[warp * 2], 1);
      mbar_init(&s_bar[warp * 2 + 1], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // Publish a lower bound of a query's global k-th score: locally (the CTAs scanning other candidate ranges and the
  // bound kernel) and, when it raises the local value, on every peer GPU (fire-and-forget system-scope reductions
  // over NVLink peer memory).  Valid for all shards: k rows with at least this score exist somewhere in the GFKB.
  auto publish_threshold = [&](int64_t q, float ks) {
    const int v = __float_as_int(ks);
    if (v <= 0) return;  // only positive scores order like their bit patterns
    const int old = atomicMax(&P.gthr[q], v);
    if (old < v) {
#pragma unroll
      for (int p = 0; p < 7; p++)
        if (p < P.n_peers) atomicMax_system(P.peer_gthr[p] + q, v);
    }
  };

  auto fetch = [&](uint32_t r, uint32_t &chunk, uint32_t &mask) {
    if (P.list_mode == 2) {
      chunk = c_lo + r;
      mask = q_count == 32 ? FULL : ((1u << q_count) - 1u);
    } else {
      uint2 rec;
      if (P.list_mode == 1) rec = P.direct[(size_t)list * P.direct_stride + r];
      else rec = P.pool[(size_t)P.list_pages[(size_t)list * P.max_pages + (r / PAGE_RECS)] * PAGE_RECS + (r % PAGE_RECS)];
      chunk = rec.x;
      mask = rec.y;
    }
    if (P.q_label) {  // drop the filtered queries whose label no row of the chunk carries: an emptied record is never staged
      const unsigned long long sig = P.chunk_sig[chunk];
      const int lb = s_qlab[lane];
      mask &= __ballot_sync(FULL, lb < 0 || ((sig >> (lb & 63)) & 1ull));
    }
    if constexpr (TAGS) {  // the same for the tag-filtered queries
      const unsigned long long qm = s_qtm[lane];
      mask &= __ballot_sync(FULL, qm == 0ull || (P.chunk_tsig[chunk] & qm) != 0ull);
    }
    if (P.alive && P.alive[chunk] == 0u) mask = 0;  // every row of the chunk deleted: never staged
  };
  auto grab = [&]() -> uint32_t {
    uint32_t r = 0;
    if (lane == 0) r = atomicAdd(s_next, 1u);
    return __shfl_sync(FULL, r, 0);
  };

  unsigned char *my_buf = s_buf + warp * 2 * S_BUF_BYTES;
  uint64_t *my_bar = s_bar + warp * 2;
  uint32_t phases = 0;  // bit b: parity the next wait on buffer b expects

  // start the copy of a record's block (if it fits the staging buffer); returns whether it was staged
  auto issue = [&](uint32_t chunk, int b) -> bool {
    const BlockInfo bi = P.binfo[chunk];
    const int E4 = (bi.n_entries + 3) & ~3;
    if (E4 == 0 || E4 > S_BUF_ENTRIES) return false;
    if (lane == 0) {
      mbar_expect_tx(&my_bar[b], (uint32_t)E4 * 8u);
      bulk_copy_g2s(my_buf + b * S_BUF_BYTES, P.blk + (size_t)bi.off4 * 4, (uint32_t)E4 * 8u, &my_bar[b]);
    }
    return true;
  };

  // Codes mode: the warp's window state.  A lane reads the codes of query q0 + lane (lanes past the group read the
  // last query's row and take nothing); tq = 256 takes nothing.
  uint32_t tq = 256;
  uint4 wraw[S_WIN / 16];            // codes of window w_nxt (in flight while the current window's records are scored)
  uint32_t w_nxt = 0;
  uint32_t wbase = 0;                // first chunk of the current window
  uint32_t wm[S_WIN / 32] = {};      // lane j: query mask of chunk wbase + 32 i + j
  unsigned long long pend = 0;       // chunks of the current window with a record not yet taken
  auto load_window = [&](uint32_t w) {
    const unsigned char *crow = P.ubq + (size_t)(q0 + min(lane, q_count - 1)) * P.ubq_stride + (size_t)w * S_WIN;
#pragma unroll
    for (int i = 0; i < S_WIN / 16; i++) wraw[i] = __ldcs(reinterpret_cast<const uint4 *>(crow) + i);
  };
  if (codes) {
    if (lane < q_count) tq = (uint32_t)P.tcode[q0 + lane];
    w_nxt = grab();
    if (w_nxt < r_hi) load_window(w_nxt);
  }
  // Next record of a codes-mode warp.  When the current window is used up, window w_nxt becomes current: its codes are
  // compared with the threshold codes (the same test, in the same order, as bound pass 1's survivors: code >= tq, chunk
  // in range, label signature), the next window's loads are issued, and a ballot per chunk transposes the comparisons
  // into query masks.  Pairs and records are counted before the live-word test, as list_append counts them.
  auto next_code_record = [&](uint32_t &chunk, uint32_t &mask) -> bool {
    while (pend == 0) {
      if (w_nxt >= r_hi) return false;
      wbase = w_nxt * S_WIN;
      const uint32_t t4 = tq < 256 ? tq * 0x01010101u : 0u;
      uint32_t ge[S_WIN / 4];  // byte i of ge[j]: 0xFF when the code of chunk wbase + 4 j + i reaches tq
      bool any = false;
#pragma unroll
      for (int i = 0; i < S_WIN / 16; i++) {
        const uint32_t v[4] = {wraw[i].x, wraw[i].y, wraw[i].z, wraw[i].w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
          ge[4 * i + j] = tq < 256 ? __vcmpgeu4(v[j], t4) : 0u;
          any |= ge[4 * i + j] != 0u;
        }
      }
      w_nxt = grab();
      if (w_nxt < r_hi) load_window(w_nxt);
#pragma unroll
      for (int i = 0; i < S_WIN / 32; i++) wm[i] = 0;
      if (!__any_sync(FULL, any)) continue;
      if (P.q_label) {
        const int lb = s_qlab[lane];
        const unsigned long long qbit = lb >= 0 ? 1ull << (lb & 63) : ~0ull;  // the query's label bit, every bit when it is not filtered
#pragma unroll
        for (int i = 0; i < S_WIN / 32; i++) {
          const unsigned long long sig = P.chunk_sig[wbase + 32 * i + lane];
#pragma unroll
          for (int j = 0; j < 32; j++) {
            const unsigned long long sig_j = __shfl_sync(FULL, sig, j);
            const bool take = ((ge[8 * i + (j >> 2)] >> ((j & 3) * 8)) & 1u) && (sig_j & qbit) != 0ull;
            const uint32_t m = __ballot_sync(FULL, take);
            if (lane == j) wm[i] = m;
          }
        }
      } else {
#pragma unroll
        for (int i = 0; i < S_WIN / 32; i++)
#pragma unroll
          for (int j = 0; j < 32; j++) {
            const uint32_t m = __ballot_sync(FULL, (ge[8 * i + (j >> 2)] >> ((j & 3) * 8)) & 1u);
            if (lane == j) wm[i] = m;
          }
      }
      if constexpr (TAGS) {  // lane = query: its tag mask against each chunk's signature (one broadcast load each)
        const unsigned long long qm = s_qtm[lane];
        if (__any_sync(FULL, qm != 0ull)) {
          for (int i = 0; i < S_WIN / 32; i++) {
            uint32_t keep = 0;  // lane j: the queries chunk wbase + 32 i + j keeps
            for (int j = 0; j < 32; j++) {
              const uint32_t m = __ballot_sync(FULL, qm == 0ull || (P.chunk_tsig[wbase + 32 * i + j] & qm) != 0ull);
              if (lane == j) keep = m;
            }
            if (i == 0) wm[0] &= keep;
            else wm[1] &= keep;
          }
        }
      }
      pend = 0;
      unsigned int sel_pairs = 0, sel_recs = 0;
#pragma unroll
      for (int i = 0; i < S_WIN / 32; i++) {
        const uint32_t c = wbase + 32 * i + lane;
        if (c >= P.n_chunks) wm[i] = 0;
        sel_pairs += (unsigned int)__popc(wm[i]);
        sel_recs += wm[i] != 0u;
        if (P.alive && P.alive[c] == 0u) wm[i] = 0;  // every row of the chunk deleted: never staged
        pend |= (unsigned long long)__ballot_sync(FULL, wm[i] != 0u) << (32 * i);
      }
      sel_pairs = __reduce_add_sync(FULL, sel_pairs);
      sel_recs = __reduce_add_sync(FULL, sel_recs);
      if (lane == 0) {
        atomicAdd(&s_stat[2], sel_pairs);
        atomicAdd(&s_stat[3], sel_recs);
      }
    }
    const int i = __ffsll((long long)pend) - 1;
    pend &= pend - 1;
    chunk = wbase + i;
    uint32_t m = wm[0];
#pragma unroll
    for (int j = 1; j < S_WIN / 32; j++)
      if ((i >> 5) == j) m = wm[j];
    mask = __shfl_sync(FULL, m, i & 31);
    return true;
  };
  auto next_record = [&](uint32_t &chunk, uint32_t &mask) -> bool {
    if (codes) return next_code_record(chunk, mask);
    const uint32_t r = grab();
    if (r >= r_hi) return false;
    fetch(r, chunk, mask);
    return true;
  };

  unsigned int pairs_done = 0, recs_done = 0;
  KV_SCAN_PROF(unsigned int kvp[KVP_N] = {}; unsigned int kvp_t = clock();)
  uint32_t chunk_cur = 0, chunk_nxt = 0;
  uint32_t mask_cur = 0, mask_nxt = 0;
  bool staged_cur = false, staged_nxt = false;
  int b = 0;
  bool have_cur = next_record(chunk_cur, mask_cur);
  if (have_cur) staged_cur = mask_cur ? issue(chunk_cur, b) : false;
  while (have_cur) {
    const bool have_nxt = next_record(chunk_nxt, mask_nxt);
    if (have_nxt) staged_nxt = mask_nxt ? issue(chunk_nxt, b ^ 1) : false;
    KV_SCAN_MARK(KVP_SELECT)
    if (mask_cur) {
      const BlockInfo bi = P.binfo[chunk_cur];
      const int E = bi.n_entries, E4 = (E + 3) & ~3;
      const uint32_t *words, *masks;
      if (staged_cur) {
        mbar_wait(&my_bar[b], (phases >> b) & 1u);
        phases ^= 1u << b;
        words = (const uint32_t *)(my_buf + b * S_BUF_BYTES);
      } else {
        words = P.blk + (size_t)bi.off4 * 4;
        KV_SCAN_PROF(kvp[KVC_INPLACE]++;)
      }
      KV_SCAN_MARK(KVP_WAIT)
      KV_SCAN_PROF(kvp[KVC_RECORDS]++; if (codes && lane == 0) atomicAdd(&g_scan_prof[KVH_QUERIES + __popc(mask_cur)], 1ull);)
      masks = words + E4;
      const int64_t pos0 = (int64_t)chunk_cur * CHUNK_ROWS;
      const int rows = (int)min((int64_t)CHUNK_ROWS, P.n_rows - pos0);
      const float Bc = lane < rows ? P.B32[pos0 + lane] : 0.f;
      const int lpos = P.q_label ? P.label_pos[pos0 + lane] : -1;  // one 128-byte line per record
      const bool live = P.alive ? ((P.alive[chunk_cur] >> lane) & 1u) != 0u : true;
      int gpos = -1;
      if constexpr (DISTINCT) gpos = P.group_pos[pos0 + lane];  // one 128-byte line per record
      recs_done++;
      for (uint32_t qm = mask_cur; qm; qm &= qm - 1) {
        const int qi = __ffs(qm) - 1;
        const float nq = s_nq[qi];
        if (!(nq > 0.f)) continue;  // null / irregular query: answered elsewhere
        const int ql = s_qlab[qi];
        if (ql >= 0 && __ballot_sync(FULL, lpos == ql) == 0) continue;  // signature collision: no row of the label here
        if constexpr (TAGS) {  // the row masks are read again (L1) where needed rather than held across the probe loop
          const unsigned long long qtm = s_qtm[qi];
          if (qtm && __ballot_sync(FULL, (P.tag_mask_pos[pos0 + lane] & qtm) != 0ull) == 0) continue;  // no row's mask meets the query's
        }
        pairs_done++;
        const uint32_t *keys = s_keys + qi * QKEYS;
        const QFeat *feats = s_feats + qi * QFEATS;
        // Hits reach the rows in two ways.  An entry held by every row of the chunk (W_ALL: the common case in a
        // candidate chunk, whose rows are text neighbours) is summed by the lane that found it (lane = entry) and the
        // warp adds those sums to every row once, after the last trip.  An entry held by some rows is handed to the
        // row lanes by shuffle from the lane that found it.  64-bit integer sums: the order does not change a bit.
        unsigned long long acc_w = 0, acc_c = 0;  // lane = row
        unsigned long long all_w = 0, all_c = 0;  // lane = entry
        KV_SCAN_PROF(kvp[KVC_PAIRS]++;)
        KV_SCAN_MARK(KVP_HEAD)
        for (int e0 = 0; e0 < E; e0 += 32) {
          const int e = e0 + lane;
          const uint32_t w = e < E ? words[e] : PAD_WORD;
          const uint32_t fid = (w >> 5) & FID_MASK;
          int idx = -1;
          if (fid != FID_NONE) {
            uint32_t h = hash_fid(fid, 7);
            for (;;) {
              const uint32_t key = keys[h];
              if (key == KEY_EMPTY) break;
              if ((key >> 6) == fid) { idx = (int)(key & 63u); break; }
              h = (h + 1) & (QKEYS - 1);
            }
          }
          KV_SCAN_PROF(kvp[KVC_TRIPS]++; kvp[KVC_HITS] += __popc(__ballot_sync(FULL, idx >= 0));
                       kvp[KVC_HITS_ALL] += __popc(__ballot_sync(FULL, idx >= 0 && (w & W_ALL)));)
          KV_SCAN_MARK(KVP_PROBE)
          uint32_t hmask = 0;  // rows of a hit that is not W_ALL
          unsigned long long ww = 0, cc = 0;
          if (idx >= 0) {
            uint32_t tf = w & 31u;
            if (tf == TF_OVF) tf = ovf_lookup(P.ovf_keys, P.ovf_vals, P.n_ovf, chunk_cur, (uint32_t)e);
            const QFeat f = feats[idx];
            ww = ((unsigned long long)f.w_hi << 32) | f.w_lo;
            cc = (unsigned long long)f.cq;
            if (tf != 1u) { ww *= (unsigned long long)tf; cc *= (unsigned long long)tf * (unsigned long long)tf; }
            if (w & W_ALL) { all_w += ww; all_c += cc; }
            else hmask = masks[e];
          }
          KV_SCAN_MARK(KVP_HITPROD)
          for (uint32_t hm = __ballot_sync(FULL, hmask != 0u); hm; hm &= hm - 1) {
            const int j = __ffs(hm) - 1;
            const uint32_t m = __shfl_sync(FULL, hmask, j);
            const unsigned long long hw = __shfl_sync(FULL, ww, j), hc = __shfl_sync(FULL, cc, j);
            if ((m >> lane) & 1u) { acc_w += hw; acc_c += hc; }
          }
          KV_SCAN_MARK(KVP_HITACC)
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          all_w += __shfl_xor_sync(FULL, all_w, o);
          all_c += __shfl_xor_sync(FULL, all_c, o);
        }
        acc_w += all_w + s_uw[qi];  // + the folded universal features: exact, so a row's bits do not depend on the fold
        acc_c += all_c + s_uc[qi];
        // fused epilogue: pre-test without division, exact score for survivors; the warp then takes the query's lock
        // ONCE and inserts all surviving rows of the chunk into the sorted list held one entry per lane (k <= 32)
        float sc = -INFINITY;
        int row = 0x7fffffff;
        bool cand = false;
        if (lane < rows) {
          const float dot = __ull2float_rn(acc_w) * (1.f / 4294967296.f);
          const float corr = -(__ull2float_rn(acc_c) * (1.f / 16777216.f));
          const float t = Bc + corr;
          float filt, ks = -INFINITY;
          int kr = 0x7fffffff;
          if constexpr (RANGE) {
            filt = __int_as_float(P.gthr[q0 + qi]);  // the search threshold: fixed for the whole scan
          } else {
            // Filter read without the lock: the global lower bound of the k-th score (rows tying with it pass) and the
            // list's k-th ENTRY once it is full, score and row in one 64-bit word, so the two always belong together.
            // A row enters a full list only if it comes before that entry in (score desc, row asc) order, and the entry
            // only ever improves: a stale word lets a few more rows through to the exact comparison under the lock and
            // never keeps out a row that belongs.  DISTINCT has a second way in, replacing the entry of the row's own
            // group; that entry is in the list, so it is no worse than the k-th one, and a row that does not come
            // before the k-th entry does not come before its group's entry either.
            filt = __int_as_float(*(volatile int *)&P.gthr[q0 + qi]);
            const unsigned long long kth = *(volatile unsigned long long *)&s_kth[qi];
            ks = __int_as_float((int)(kth >> 32));
            kr = (int)(uint32_t)kth;
            filt = fmaxf(filt, ks);
          }
          bool pass = true;
          if (filt > 0.f) pass = dot * dot >= filt * filt * nq * FILTER_SLACK * t;
          if (pass) {
            const float den = nq * t;
            sc = den > 0.f ? __fdiv_rn(dot, __fsqrt_rn(den)) : 0.f;
            row = P.perm[pos0 + lane];
            cand = row != s_excl[qi] && sc >= filt && (sc > ks || row < kr) && (ql < 0 || lpos == ql) && live;
            if constexpr (TAGS) {
              const unsigned long long qtm = s_qtm[qi];
              if (cand && qtm)
                cand = tags_meet(P.tag_mask_pos[pos0 + lane], qtm, P.tag_ptr, P.tag_list, pos0 + lane, P.q_tags + (q0 + qi) * MAX_QTAGS);
            }
          }
        }
        if constexpr (RANGE) {
          range_emit(P.range_out, P.range_count, P.range_cap, cand, P.qperm + q0 + qi, sc, P.row_base + row);
          continue;
        }
        uint32_t cm = __ballot_sync(FULL, cand);
        KV_SCAN_PROF(kvp[KVC_ROWS_PASSED] += __popc(cm);)
        if constexpr (DISTINCT) {
          // the best survivor of each group of the chunk goes on (lanes without a survivor get keys of their own)
          const uint32_t peers = __match_any_sync(FULL, cand ? gpos : -1 - lane);
          bool keep = cand;
          for (uint32_t m = __ballot_sync(FULL, cand && peers != (1u << lane)); m; m &= m - 1) {
            const int j = __ffs(m) - 1;
            const float s2 = __shfl_sync(FULL, sc, j);
            const int r2 = __shfl_sync(FULL, row, j);
            if (((peers >> j) & 1u) && (s2 > sc || (s2 == sc && r2 < row))) keep = false;
          }
          cm = __ballot_sync(FULL, keep);
        }
        KV_SCAN_MARK(KVP_EPI)
        if (cm) {
          if (lane == 0) while (atomicCAS(&s_lock[qi], 0, 1) != 0) {}
          __syncwarp();
          KV_SCAN_MARK(KVP_LOCKWAIT)
          __threadfence_block();
          int cnt = *(volatile int *)&s_cnt[qi];
          float ls = lane < k ? *(volatile float *)&s_lscore[qi * k + lane] : -INFINITY;   // unused slots hold (-inf, INT_MAX)
          int lr = lane < k ? *(volatile int *)&s_lrow[qi * k + lane] : 0x7fffffff;
          int lg = -1;                                                                      // ... and group -1
          if constexpr (DISTINCT) lg = lane < k ? *(volatile int *)&s_lgrp[qi * k + lane] : -1;
          bool changed = false;
          for (uint32_t m = cm; m; m &= m - 1) {
            const int j = __ffs(m) - 1;
            const float ns = __shfl_sync(FULL, sc, j);
            const int nr = __shfl_sync(FULL, row, j);
            int ng = -1;
            if constexpr (DISTINCT) {
              ng = __shfl_sync(FULL, gpos, j);
              const uint32_t same = __ballot_sync(FULL, lane < k && lg == ng);  // at most one entry per group
              if (same) {
                const int p = __ffs(same) - 1;
                const float ps = __shfl_sync(FULL, ls, p);
                const int pr = __shfl_sync(FULL, lr, p);
                if (!(ns > ps || (ns == ps && nr < pr))) continue;  // the group's entry is better: the row is dropped
                // delete the group's entry: the entries after it move up by one, the last slot becomes unused
                const float ds = __shfl_down_sync(FULL, ls, 1);
                const int dr = __shfl_down_sync(FULL, lr, 1);
                const int dg = __shfl_down_sync(FULL, lg, 1);
                if (lane == k - 1) { ls = -INFINITY; lr = 0x7fffffff; lg = -1; }
                else if (lane >= p && lane < k) { ls = ds; lr = dr; lg = dg; }
                cnt--;
              }
            }
            // entries that stay ahead of the new one form a prefix of the sorted list
            const bool ahead = lane < k && (ls > ns || (ls == ns && lr < nr));
            const int pos = __popc(__ballot_sync(FULL, ahead));
            const float us = __shfl_up_sync(FULL, ls, 1);
            const int ur = __shfl_up_sync(FULL, lr, 1);
            int ug = -1;
            if constexpr (DISTINCT) ug = __shfl_up_sync(FULL, lg, 1);
            if (pos < k) {
              if (lane > pos) { ls = us; lr = ur; if constexpr (DISTINCT) lg = ug; }
              else if (lane == pos) { ls = ns; lr = nr; if constexpr (DISTINCT) lg = ng; }
              if (cnt < k) cnt++;
              changed = true;
            }
          }
          if (changed) {
            if (lane < k) { s_lscore[qi * k + lane] = ls; s_lrow[qi * k + lane] = lr; }
            if constexpr (DISTINCT) if (lane < k) s_lgrp[qi * k + lane] = lg;
            if (lane == 0) s_cnt[qi] = cnt;
            if (lane == k - 1 && cnt == k)  // one 64-bit store: a reader never pairs a new score with an old row
              s_kth[qi] = ((unsigned long long)(uint32_t)__float_as_int(ls) << 32) | (uint32_t)lr;
            const float ks = __shfl_sync(FULL, ls, k - 1);
            if (lane == 0 && cnt == k) publish_threshold(q0 + qi, ks);
          }
          __threadfence_block();
          __syncwarp();
          if (lane == 0) atomicExch(&s_lock[qi], 0);
          KV_SCAN_PROF(kvp[KVC_LOCKS]++; kvp[KVC_LOCKS_UNCHANGED] += !changed;)
          KV_SCAN_MARK(KVP_INSERT)
        }
        __syncwarp();
      }
    }
    __syncwarp();  // every lane is done with buffer b before a later copy may overwrite it
    have_cur = have_nxt;
    chunk_cur = chunk_nxt;
    mask_cur = mask_nxt;
    staged_cur = staged_nxt;
    b ^= 1;
  }
  if (lane == 0) {
    atomicAdd(&s_stat[0], pairs_done);
    atomicAdd(&s_stat[1], recs_done);
  }
  KV_SCAN_MARK(KVP_SELECT)
  __syncthreads();
  KV_SCAN_MARK(KVP_TAIL)
  KV_SCAN_PROF(if (codes && lane == 0) {
    kvp[KVC_WARPS] = 1;
    for (int i = 0; i < KVC_CTAS; i++) atomicAdd(&g_scan_prof[i], (unsigned long long)kvp[i]);
    if (warp == 0) {
      atomicAdd(&g_scan_prof[KVC_CTAS], 1ull);
      atomicMax(&g_scan_prof[KVC_CTA_PAIRS_MAX], (unsigned long long)s_stat[0]);
      atomicAdd(&g_scan_prof[KVH_CTA_PAIRS + min(s_stat[0] / 512u, 63u)], 1ull);
    }
  })
  if constexpr (!RANGE) {  // publish this CTA's partial lists (already ordered)
    const int part = bsplit * P.n_ssplits + ssplit;
    for (int i = threadIdx.x; i < q_count * k; i += blockDim.x) {
      const int qi = i / k, j = i - qi * k;
      const size_t o = ((size_t)part * P.n_q + (q0 + qi)) * k + j;
      const bool used = j < s_cnt[qi];
      P.part_scores[o] = used ? s_lscore[i] : -INFINITY;
      P.part_rows[o] = used ? (long long)(P.row_base + s_lrow[i]) : -1LL;
    }
  }
  if (threadIdx.x == 0 && P.stats) {
    atomicAdd(&P.stats[0], (unsigned long long)s_stat[0]);
    atomicAdd(&P.stats[1], (unsigned long long)s_stat[1]);
    if (codes) {
      atomicAdd(&P.stats[2], (unsigned long long)s_stat[2]);
      atomicAdd(&P.stats[3], (unsigned long long)s_stat[3]);
    }
  }
}

static inline size_t scan_smem_bytes(int k, bool distinct = false, bool tags = false) {
  return (size_t)GROUP_Q * QTAB_BYTES + (size_t)S_WARPS * 2 * S_BUF_BYTES + (size_t)S_WARPS * 2 * 8 + (size_t)GROUP_Q * 8 * 3 +
         (size_t)GROUP_Q * k * 8 + (size_t)GROUP_Q * 4 * 5 + 32 + (distinct ? (size_t)GROUP_Q * k * 4 : 0) +
         (tags ? (size_t)GROUP_Q * 8 + 8 : 0);
}

// ----------------------------------------------------------------------------------------
// K3: token-set Jaccard, dense regime.  Random token sets have no text structure, so chunk bounds prune nothing and
// the per-(query, chunk) scan would redo the probing for every query; here one warp scores a chunk for the 32 queries
// of its scan group AT ONCE (lane = query).  The group's union table (token -> mask of the queries holding it) sits in
// shared memory; the lanes probe 32 block entries at a time; every hit's row mask is spread into eight words of four
// 8-bit counters (lane-parallel) and added by the lanes whose query holds the token -- after the chunk a lane holds
// |q ∩ row| for all 32 rows as bytes.  Exact integers; score = |∩| / (|q| + |row| - |∩|); per-warp private top-k lists
// (no locks), merged by K5.  Queries are limited to 64 tokens like everywhere (more: float64 full-scan path).
// K3-R (RANGE = true) is the same scan for a threshold search: no lists; P.gthr holds the fixed threshold, and every
// (query, row) pair whose score reaches it is appended to R.out with its exact counts.
// ----------------------------------------------------------------------------------------
struct JaccardParams {
  const uint32_t *blk;
  const BlockInfo *binfo;
  const float *B32;
  const int *perm;
  int64_t n_chunks, n_rows, row_base;
  const unsigned char *qtab;
  const float *q_nq, *q_dotU;
  const int *q_excl;
  int *gthr;
  int64_t n_q;
  int k, n_splits;
  float *part_scores;  // [n_splits * J_WARPS][n_q][k]
  long long *part_rows;
  unsigned long long *stats;
};

constexpr int J_WARPS = 8;
constexpr int J_SLOTS = 4096;  // union table of a group: <= 32 x 64 tokens

static inline size_t jaccard_smem_bytes(int k) { return (size_t)J_SLOTS * 8 + (size_t)J_WARPS * 32 * 36 + (size_t)J_WARPS * k * 32 * 8; }

// Output of the threshold search (jaccard_scan_kernel<true>, which leaves k and the partial lists of JaccardParams
// unused; the top-k form ignores this argument).  A kernel argument of its own, so that the top-k form's parameter
// block stays as it was.
struct JaccardRangeOut {
  const int *qperm;           // [n_q] sorted slot -> original query
  JaccardPair *out;           // [cap]
  unsigned long long *count;  // pairs found (may exceed cap: those past it are not written)
  unsigned long long cap;
};

template <bool RANGE>
__global__ void __launch_bounds__(J_WARPS * 32, 2) jaccard_scan_kernel(JaccardParams P, JaccardRangeOut R) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t *s_keys = (uint32_t *)smem_raw;                 // [J_SLOTS]
  uint32_t *s_qm = s_keys + J_SLOTS;                       // [J_SLOTS] queries of the group holding the token
  uint32_t *s_hit = s_qm + J_SLOTS;                        // [J_WARPS][32][9]: query mask + 8 spread words
  float *s_ls = (float *)(s_hit + J_WARPS * 32 * 9);       // [J_WARPS][k][32]
  int *s_lr = (int *)(s_ls + J_WARPS * P.k * 32);          // [J_WARPS][k][32]
  const int group = blockIdx.x, split = blockIdx.y, k = P.k;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t q0 = (int64_t)group * GROUP_Q;
  const int q_count = (int)min((int64_t)GROUP_Q, P.n_q - q0);
  for (int i = threadIdx.x; i < J_SLOTS; i += blockDim.x) { s_keys[i] = KEY_EMPTY; s_qm[i] = 0; }
  __syncthreads();
  for (int i = threadIdx.x; i < q_count * QKEYS; i += blockDim.x) {
    const int qi = i / QKEYS, sl = i - qi * QKEYS;
    if (!(P.q_nq[q0 + qi] > 0.f)) continue;
    const uint32_t key = ((const uint32_t *)(P.qtab + (size_t)(q0 + qi) * QTAB_BYTES))[sl];
    if (key == KEY_EMPTY) continue;
    const uint32_t fid = key >> 6;
    uint32_t h = hash_fid(fid, 12);
    for (;;) {
      uint32_t cur = s_keys[h];
      if (cur == KEY_EMPTY) cur = atomicCAS(&s_keys[h], KEY_EMPTY, fid);
      if (cur == KEY_EMPTY || cur == fid) break;
      h = (h + 1) & (J_SLOTS - 1);
    }
    atomicOr(&s_qm[h], 1u << qi);
  }
  __syncthreads();
  const bool valid = lane < q_count && P.q_nq[q0 + (lane < q_count ? lane : 0)] > 0.f;
  const float nq = valid ? P.q_nq[q0 + lane] : 0.f;
  const float dotU = valid ? P.q_dotU[q0 + lane] : 0.f;
  const int excl = (valid && P.q_excl) ? P.q_excl[q0 + lane] : -1;
  // threshold search: this lane's fixed threshold and original query
  const float rthr = (RANGE && valid) ? __int_as_float(P.gthr[q0 + lane]) : 0.f;
  const int rq = (RANGE && valid) ? R.qperm[q0 + lane] : 0;
  float *ls = s_ls + (size_t)warp * k * 32 + lane;  // element j at ls[j * 32]
  int *lr = s_lr + (size_t)warp * k * 32 + lane;
  if constexpr (!RANGE)
    for (int j = 0; j < k; j++) { ls[j * 32] = -INFINITY; lr[j * 32] = 0x7fffffff; }
  int cnt = 0;
  float kth = -INFINITY;
  int kth_row = 0x7fffffff;
  uint32_t *hit = s_hit + warp * 32 * 9;
  const uint32_t lt = lanemask_lt();
  const int64_t c_lo = P.n_chunks * split / P.n_splits, c_hi = P.n_chunks * (split + 1) / P.n_splits;
  unsigned int done = 0;
  for (int64_t c = c_lo + warp; c < c_hi; c += J_WARPS) {
    const BlockInfo bi = P.binfo[c];
    const int E = bi.n_entries, E4 = (E + 3) & ~3;
    const uint32_t *words = P.blk + (size_t)bi.off4 * 4, *masks = words + E4;
    const int64_t pos0 = c * CHUNK_ROWS;
    const int rows = (int)min((int64_t)CHUNK_ROWS, P.n_rows - pos0);
    const uint32_t vmask = rows == 32 ? FULL : ((1u << rows) - 1u);
    const float myB = lane < rows ? P.B32[pos0 + lane] : 0.f;
    const int myrow = lane < rows ? P.perm[pos0 + lane] : 0x7fffffff;
    uint32_t cw[8];
#pragma unroll
    for (int i = 0; i < 8; i++) cw[i] = 0;
    for (int e0 = 0; e0 < E; e0 += 32) {
      const int e = e0 + lane;
      const uint32_t w = e < E ? __ldg(words + e) : PAD_WORD;
      const uint32_t fid = (w >> 5) & FID_MASK;
      uint32_t qm = 0;
      if (fid != FID_NONE) {
        uint32_t h = hash_fid(fid, 12);
        for (;;) {
          const uint32_t key = s_keys[h];
          if (key == KEY_EMPTY) break;
          if (key == fid) { qm = s_qm[h]; break; }
          h = (h + 1) & (J_SLOTS - 1);
        }
      }
      const uint32_t hm = __ballot_sync(FULL, qm != 0);
      if (hm == 0) continue;
      if (qm) {
        const uint32_t m = (w & W_ALL) ? vmask : __ldg(masks + e);
        uint32_t *o = hit + __popc(hm & lt) * 9;
        o[0] = qm;
#pragma unroll
        for (int i = 0; i < 8; i++) o[1 + i] = (((m >> (4 * i)) & 0xFu) * 0x00204081u) & 0x01010101u;  // 4 bits -> 4 bytes
      }
      __syncwarp();
      const int nh = __popc(hm);
      for (int hh = 0; hh < nh; hh++) {
        const uint32_t *o = hit + hh * 9;
        if ((o[0] >> lane) & 1u) {
#pragma unroll
          for (int i = 0; i < 8; i++) cw[i] += o[1 + i];
        }
      }
      __syncwarp();
    }
    done++;
    if constexpr (RANGE) {
      // this lane's hits among the chunk's 32 rows (the score is the top-k epilogue's expression), then one
      // reservation for the warp's hits from an inclusive prefix sum of the lanes' counts
      uint32_t hits = 0;
#pragma unroll
      for (int r = 0; r < 32; r++) {
        const float t = __shfl_sync(FULL, myB, r);
        const int row = __shfl_sync(FULL, myrow, r);
        if (r >= rows || !valid || row == excl) continue;
        const float inter = dotU + (float)((cw[r >> 2] >> ((r & 3) * 8)) & 0xFFu);
        const float uni = nq + t - inter;
        if (!(inter >= rthr * uni * FILTER_SLACK)) continue;  // pre-test without division, looser than the test below
        if (uni > 0.f && __fdiv_rn(inter, uni) >= rthr) hits |= 1u << r;
      }
      const int nh = __popc(hits);
      int incl = nh;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += v;
      }
      const int total = __shfl_sync(FULL, incl, 31);
      if (total == 0) continue;
      unsigned long long base = 0;
      if (lane == 31) base = atomicAdd(R.count, (unsigned long long)total);
      unsigned long long o = __shfl_sync(FULL, base, 31) + (unsigned long long)(incl - nh);
#pragma unroll
      for (int r = 0; r < 32; r++) {
        const float t = __shfl_sync(FULL, myB, r);
        const int row = __shfl_sync(FULL, myrow, r);
        if ((hits >> r) & 1u) {
          const float inter = dotU + (float)((cw[r >> 2] >> ((r & 3) * 8)) & 0xFFu);
          if (o < R.cap) R.out[o] = JaccardPair{rq, row, (int)inter, (int)(nq + t - inter)};
          o++;
        }
      }
      continue;
    }
    // 32 rows of the chunk for this lane's query
    float filt = kth;
    if (valid) filt = fmaxf(filt, __int_as_float(__ldcg(&P.gthr[q0 + lane])));
#pragma unroll
    for (int r = 0; r < 32; r++) {
      const float t = __shfl_sync(FULL, myB, r);
      const int row = __shfl_sync(FULL, myrow, r);
      if (r >= rows || !valid || row == excl) continue;
      const float inter = dotU + (float)((cw[r >> 2] >> ((r & 3) * 8)) & 0xFFu);
      const float uni = nq + t - inter;
      if (!(inter >= filt * uni * FILTER_SLACK)) continue;  // pre-test without division (filt = -inf passes everything)
      const float sc = uni > 0.f ? __fdiv_rn(inter, uni) : 0.f;
      bool take = cnt < k || sc > kth || (sc == kth && row < kth_row);
      if (!take || sc < filt) continue;
      int pos = cnt < k ? cnt++ : k - 1;
      while (pos > 0 && (ls[(pos - 1) * 32] < sc || (ls[(pos - 1) * 32] == sc && lr[(pos - 1) * 32] > row))) {
        ls[pos * 32] = ls[(pos - 1) * 32];
        lr[pos * 32] = lr[(pos - 1) * 32];
        pos--;
      }
      ls[pos * 32] = sc;
      lr[pos * 32] = row;
      if (cnt == k) {
        kth = ls[(k - 1) * 32];
        kth_row = lr[(k - 1) * 32];
        filt = fmaxf(filt, kth);
        if (kth > 0.f) atomicMax(&P.gthr[q0 + lane], __float_as_int(kth));
      }
    }
  }
  // publish this warp's partial lists
  const int part = split * J_WARPS + warp;
  if (!RANGE && lane < q_count) {
    for (int j = 0; j < k; j++) {
      const size_t o = ((size_t)part * P.n_q + (q0 + lane)) * k + j;
      const bool used = j < cnt;
      P.part_scores[o] = used ? ls[j * 32] : -INFINITY;
      P.part_rows[o] = used ? (long long)(P.row_base + lr[j * 32]) : -1LL;
    }
  }
  if (lane == 0 && P.stats) atomicAdd(&P.stats[0], (unsigned long long)done * (unsigned long long)q_count);
}

// seeds of the first bound pass -> fixed-stride candidate lists: query slot i holds n_seed chunk ids (-1: none)
__global__ void seeds_to_lists_kernel(const int *__restrict__ seeds, int64_t n_q, int n_seed, uint2 *direct,
                                      uint32_t *list_count) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t n_groups = (n_q + GROUP_Q - 1) / GROUP_Q;
  if (i < n_groups) list_count[i] = (uint32_t)(GROUP_Q * n_seed);
  if (i >= n_groups * GROUP_Q * n_seed) return;
  const int64_t q = i / n_seed;
  const int c = q < n_q ? seeds[i] : -1;
  uint2 rec;
  rec.x = c >= 0 ? (uint32_t)c : 0u;
  rec.y = c >= 0 ? (1u << (q % GROUP_Q)) : 0u;
  // seed-major inside a group: consecutive records belong to different queries, so the warps of a scan CTA do not
  // queue on one query's list lock
  const int64_t g = q / GROUP_Q, j = i - q * n_seed;
  direct[(g * n_seed + j) * GROUP_Q + (q % GROUP_Q)] = rec;
}

// ----------------------------------------------------------------------------------------
// K6: float64 re-scoring of selected (query, row) pairs -- one warp per pair.  Walks ALL of the row's raw CSR
// entries in their stored (text) order and sums with explicit round-to-nearest adds/multiplies (no fused
// multiply-add, no folded constants), so the bits depend only on the row's text, the query and the global
// statistics -- not on which segment or shard holds the row or which features that shard folded as universal.
// Rows with identical text therefore tie EXACTLY everywhere, and the (score desc, row asc) order of
// services/gfkb/app.py:89 is reproduced across segments.  Same formula as K1a (values agree to ~1e-12 relative).
// Used by the batched match path: K1b selects candidates in float32, K6 gives them float64 scores.
// ----------------------------------------------------------------------------------------
struct RescoreParams {
  const int64_t *indptr;   // raw CSR of the index (device)
  const uint32_t *ids;
  const uint16_t *tf;
  const double *a64, *d64;  // host-computed idf tables (the values K1a's query tables are built from)
  const double *B64;        // row norms by position
  const int *invperm;       // original row -> position
  const int64_t *q_indptr;  // query batch CSR (device)
  const uint32_t *q_ids, *q_tf;
  const double *q_nq;
  const long long *rows;    // [n_q * k] global row ids (-1: unused slot)
  int64_t n_q, n_rows, row_base, V;
  int k, jaccard;
  const uint8_t *dead;      // by local row, NULL: no row deleted
  double *out;              // [n_q * k]; -inf for unused slots, rows of other shards and deleted rows
};

// K6's body for one pair, shared by K6 and K6-R so that both give the same bits for the same pair: the whole warp
// walks local row r against query q, and the lanes with `finish` set return the float64 score (the others 0).
__device__ __forceinline__ double rescore_pair(const RescoreParams &P, int64_t q, int64_t r, int lane, bool finish) {
  const int64_t qa = P.q_indptr[q], qb = P.q_indptr[q + 1];
  double du = 0.0, dv = 0.0;
  const int64_t p1 = P.indptr[r + 1];
  for (int64_t p0 = P.indptr[r]; p0 < p1; p0 += 32) {
    const int64_t p = p0 + lane;
    bool hit = false;
    double wu = 0.0, wv = 0.0;
    if (p < p1) {
      const uint32_t t = P.ids[p];
      if ((int64_t)t < P.V) {
        for (int64_t j = qa; j < qb; j++)
          if (P.q_ids[j] == t) {
            const double f = (double)P.tf[p];
            wu = __dmul_rn(f, __dmul_rn((double)P.q_tf[j], P.a64[t]));
            wv = __dmul_rn(__dmul_rn(f, f), P.d64[t]);
            hit = true;
            break;
          }
      }
    }
    uint32_t hm = __ballot_sync(FULL, hit);
    while (hm) {
      const int j = __ffs(hm) - 1;
      hm &= hm - 1;
      du = __dadd_rn(du, __shfl_sync(FULL, wu, j));
      dv = __dadd_rn(dv, __shfl_sync(FULL, wv, j));
    }
  }
  if (!finish) return 0.0;
  const double B = P.B64[P.invperm[r]];
  const double dot = du;
  double sc;
  if (P.jaccard) {
    const double den = __dadd_rn(__dadd_rn(P.q_nq[q], B), -dot);
    sc = (den > 0.0 && dot != 0.0) ? dot / den : 0.0;
  } else {
    const double den = __dmul_rn(P.q_nq[q], __dadd_rn(B, dv));
    sc = (den > 0.0 && dot != 0.0) ? dot / sqrt(den) : 0.0;
  }
  return sc;
}

__global__ void __launch_bounds__(256) rescore_kernel(RescoreParams P) {
  const int64_t pair = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (pair >= P.n_q * P.k) return;
  const int64_t q = pair / P.k;
  const long long gr = P.rows[pair];
  const int64_t r = gr - P.row_base;
  if (gr < 0 || r < 0 || r >= P.n_rows || (P.dead && P.dead[r])) {
    if (lane == 0) P.out[pair] = -INFINITY;
    return;
  }
  const double sc = rescore_pair(P, q, r, lane, lane == 0);
  if (lane == 0) P.out[pair] = sc;
}

// ----------------------------------------------------------------------------------------
// K6-R: K6 of the pairs a threshold search emitted (kv_range_resident_exact).  It reads the search's records in place
// (emit order, global rows), gives each pair its K6 score through rescore_pair -- the bits K6 gives the same pair --
// and keeps the pairs whose score reaches the float64 threshold as ExactPair records (local rows).  A warp takes 32
// consecutive records and scores them one after the other with all its lanes, so that lane j ends with record j's
// score; the kept ones then take one reservation per warp, as range_emit and dense_emit do.  The output has room for
// every input record, so no pair is lost.
// ----------------------------------------------------------------------------------------
struct RescoreRangeParams {
  RescoreParams K6;          // the index and the query batch; rows, k and out are not used
  const RangePair *in;       // [n] the search's records
  int64_t n;
  double thr;
  ExactPair *out;            // [n]
  unsigned long long *count;  // kept records
};

__global__ void __launch_bounds__(256) rescore_range_kernel(RescoreRangeParams P) {
  const int64_t i0 = ((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5) * 32;
  const int lane = threadIdx.x & 31;
  if (i0 >= P.n) return;
  const int m = (int)min((int64_t)32, P.n - i0);
  RangePair rec{0, 0.f, 0};
  if (lane < m) rec = P.in[i0 + lane];
  double mine = 0.0;
  for (int j = 0; j < m; j++) {
    const int q = __shfl_sync(FULL, rec.q, j);
    const long long row = __shfl_sync(FULL, (long long)rec.row, j);
    const double sc = rescore_pair(P.K6, q, row - P.K6.row_base, lane, lane == j);
    if (lane == j) mine = sc;
  }
  const bool keep = lane < m && mine >= P.thr;
  const uint32_t hm = __ballot_sync(FULL, keep);
  if (hm == 0) return;
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(P.count, (unsigned long long)__popc(hm));
  base = __shfl_sync(FULL, base, 0);
  if (keep) P.out[base + __popc(hm & lanemask_lt())] = ExactPair{rec.q, (int)(rec.row - P.K6.row_base), mine};
}

// ----------------------------------------------------------------------------------------
// K5: merge n_lists ordered partial lists per query -- one warp per query
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ bool better(float s1, long long r1, float s2, long long r2) {
  // (score desc, row asc); unused slots (-inf, -1) lose against everything real
  if (s1 != s2) return s1 > s2;
  if (r1 < 0) return false;
  if (r2 < 0) return true;
  return r1 < r2;
}

// out_index: optional map from the list's query slot to the output slot (un-sorts the query batch)
// stride_s / stride_r: elements between the starts of consecutive lists (n_q * k when the lists are contiguous)
__global__ void merge_topk_kernel(const float *__restrict__ in_s, const long long *__restrict__ in_r, int n_lists,
                                  int64_t n_q, int k, int64_t stride_s, int64_t stride_r,
                                  const int *__restrict__ out_index, float *out_s, long long *out_r) {
  const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (q >= n_q) return;
  const int64_t oq = out_index ? out_index[q] : q;
  constexpr int MAXL = 64;  // lists per lane -> up to 2048 lists per launch
  unsigned char head[MAXL];
#pragma unroll
  for (int i = 0; i < MAXL; i++) head[i] = 0;
  for (int j = 0; j < k; j++) {
    float bs = -INFINITY;
    long long br = -1;
    int bl = -1;
    for (int i = 0; i < MAXL; i++) {
      int l = lane + 32 * i;
      if (l >= n_lists) break;
      int h = head[i];
      if (h >= k) continue;
      const size_t o = (size_t)q * k + h;
      float s = in_s[(size_t)l * stride_s + o];
      long long r = in_r[(size_t)l * stride_r + o];
      if (r >= 0 && (bl < 0 || better(s, r, bs, br))) { bs = s; br = r; bl = l; }
    }
    for (int o = 16; o; o >>= 1) {
      float s2 = __shfl_xor_sync(FULL, bs, o);
      long long r2 = __shfl_xor_sync(FULL, br, o);
      int l2 = __shfl_xor_sync(FULL, bl, o);
      if (l2 >= 0 && (bl < 0 || better(s2, r2, bs, br))) { bs = s2; br = r2; bl = l2; }
    }
    if (bl >= 0 && (bl & 31) == lane) head[bl >> 5]++;
    if (lane == 0) {
      out_s[oq * k + j] = bl >= 0 ? bs : -INFINITY;
      out_r[oq * k + j] = bl >= 0 ? br : -1LL;
    }
  }
}

// K5 of a distinct batch (kv_query_set_distinct).  Each partial list holds distinct groups; in the merged (score desc,
// row asc) order a group's first entry is its best row, and every later entry of a taken group is skipped.  Exact: a
// group of the global top-k is also in the top-k of the partial list that holds its best row -- inside one index and
// across the row shards of a sharded GFKB alike.  groups: by local row (global row - row_base), n_group_rows of them;
// a row outside them is never looked up: it ends its list and sets *bad (when given).  stride_s / stride_r as in
// merge_topk_kernel.  One warp per query, as merge_topk_kernel; 256 threads per block.
__global__ void merge_topk_distinct_kernel(const float *__restrict__ in_s, const long long *__restrict__ in_r, int n_lists,
                                           int64_t n_q, int k, int64_t stride_s, int64_t stride_r,
                                           const int *__restrict__ out_index, const int *__restrict__ groups, int64_t row_base,
                                           int64_t n_group_rows, unsigned *bad, float *out_s, long long *out_r) {
  __shared__ int s_taken[8][32];  // per warp: the groups taken so far
  const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (q >= n_q) return;
  int *taken = s_taken[threadIdx.x >> 5];
  const int64_t oq = out_index ? out_index[q] : q;
  constexpr int MAXL = 64;
  unsigned char head[MAXL];
#pragma unroll
  for (int i = 0; i < MAXL; i++) head[i] = 0;
  for (int j = 0; j < k; j++) {
    float bs = -INFINITY;
    long long br = -1;
    int bl = -1, bg = -1;
    for (int i = 0; i < MAXL; i++) {
      int l = lane + 32 * i;
      if (l >= n_lists) break;
      int h = head[i];
      float s = -INFINITY;
      long long r = -1;
      int g = -1;
      for (; h < k; h++) {  // skip the entries of taken groups
        const size_t o = (size_t)q * k + h;
        r = in_r[(size_t)l * stride_r + o];
        if (r < 0) break;
        const long long gr = r - row_base;
        if (gr < 0 || gr >= n_group_rows) {  // a row without a group: the list ends here, the caller reports it
          if (bad) *bad = 1u;
          r = -1;
          break;
        }
        g = groups[gr];
        bool seen = false;
        for (int t = 0; t < j; t++) seen |= taken[t] == g;
        if (!seen) { s = in_s[(size_t)l * stride_s + o]; break; }
        r = -1;
      }
      head[i] = (unsigned char)h;
      if (r >= 0 && (bl < 0 || better(s, r, bs, br))) { bs = s; br = r; bl = l; bg = g; }
    }
    for (int o = 16; o; o >>= 1) {
      float s2 = __shfl_xor_sync(FULL, bs, o);
      long long r2 = __shfl_xor_sync(FULL, br, o);
      int l2 = __shfl_xor_sync(FULL, bl, o);
      int g2 = __shfl_xor_sync(FULL, bg, o);
      if (l2 >= 0 && (bl < 0 || better(s2, r2, bs, br))) { bs = s2; br = r2; bl = l2; bg = g2; }
    }
    if (bl >= 0 && (bl & 31) == lane) head[bl >> 5]++;
    if (lane == 0) {
      out_s[oq * k + j] = bl >= 0 ? bs : -INFINITY;
      out_r[oq * k + j] = bl >= 0 ? br : -1LL;
      taken[j] = bg;  // -1 once the lists are exhausted: no group is -1
    }
    __syncwarp();
  }
}

constexpr int LAB_FIRST = 33;  // smallest rows kept per label: k <= 32 of them plus one a self-join excludes

// The rows of each label in ascending order, first LAB_FIRST of them (kv_index_set_row_labels): keys[n_lab] sorted,
// rows[n_lab][LAB_FIRST] local rows, -1 past the label's last row
struct LabelFirstRows {
  const int *keys, *rows;
  int n_lab;
};

// Null queries (no feature in common with any row: every score is 0): the stable sort keeps the
// first k live rows -- of the query's label when it is filtered (label_by_query: by ORIGINAL query, NULL: no filter).
// first_live: the first LAB_FIRST live rows, -1 past the last (NULL: no row deleted, rows 0, 1, ...).
// One thread per (query, slot).
__global__ void fill_null_kernel(const int *__restrict__ null_q, int n_null, int k, int64_t n_rows, int64_t row_base,
                                 const int *__restrict__ excl_by_query, const int *__restrict__ label_by_query,
                                 LabelFirstRows L, const int *__restrict__ first_live, float *out_s, long long *out_r) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_null * k) return;
  int q = null_q[i / k], j = i % k;
  const int ex = excl_by_query ? excl_by_query[q] : -1;  // by ORIGINAL query index
  const int lb = label_by_query ? label_by_query[q] : -1;
  if (lb >= 0 || first_live) {
    int idx = -1;
    const int *list = first_live;
    if (lb >= 0) {
      int lo = 0, hi = L.n_lab - 1;
      while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        if (L.keys[mid] == lb) { idx = mid; break; }
        if (L.keys[mid] < lb) lo = mid + 1; else hi = mid - 1;
      }
      list = idx >= 0 ? L.rows + (size_t)idx * LAB_FIRST : nullptr;
    }
    int r = -1;
    for (int t = 0, seen = 0; list && t < LAB_FIRST; t++) {  // the j-th listed row once the excluded one is skipped
      const int x = list[t];
      if (x < 0) break;
      if (x == ex) continue;
      if (seen++ == j) { r = x; break; }
    }
    out_s[(size_t)q * k + j] = r >= 0 ? 0.f : -INFINITY;
    out_r[(size_t)q * k + j] = r >= 0 ? row_base + r : -1LL;
    return;
  }
  const int64_t r = (ex >= 0 && j >= ex) ? j + 1 : j;     // the j-th row once the excluded one is skipped
  out_s[(size_t)q * k + j] = r < n_rows ? 0.f : -INFINITY;
  out_r[(size_t)q * k + j] = r < n_rows ? row_base + r : -1LL;
}

// Fallback selection for one (irregular) query: k passes of block-wide arg-best over float64 scores.  lab >= 0: only
// rows with labels[row] == lab (by original row) compete; dead (NULL: none) marks deleted rows, which never do.
// S: the precision the scores are compared and reported in -- float for the top-k (the float32 value K1b reports),
// double for kv_exact_topk, whose order is the float64 one.
template <typename S>
__global__ void select_topk_kernel(const double *__restrict__ scores, int64_t n, int64_t row_base, int k, int64_t excl,
                                   const int *__restrict__ labels, int lab, const uint8_t *__restrict__ dead,
                                   S *out_s, long long *out_r) {
  __shared__ S s_s[32];
  __shared__ long long s_r[32];
  __shared__ S prev_s;
  __shared__ long long prev_r;
  if (threadIdx.x == 0) { prev_s = INFINITY; prev_r = -1; }
  __syncthreads();
  for (int j = 0; j < k; j++) {
    S bs = -INFINITY;
    long long br = -1;
    const S ps = prev_s;
    const long long pr = prev_r;
    for (int64_t r = threadIdx.x; r < n; r += blockDim.x) {
      if (r == excl || (lab >= 0 && labels[r] != lab) || (dead && dead[r])) continue;
      S s = (S)scores[r];
      bool after = (s < ps) || (s == ps && r > pr);  // strictly after the previously selected pair
      if (after && (br < 0 || s > bs || (s == bs && r < br))) { bs = s; br = r; }
    }
    for (int o = 16; o; o >>= 1) {
      S s2 = __shfl_xor_sync(FULL, bs, o);
      long long r2 = __shfl_xor_sync(FULL, br, o);
      if (r2 >= 0 && (br < 0 || s2 > bs || (s2 == bs && r2 < br))) { bs = s2; br = r2; }
    }
    if ((threadIdx.x & 31) == 0) { s_s[threadIdx.x >> 5] = bs; s_r[threadIdx.x >> 5] = br; }
    __syncthreads();
    if (threadIdx.x < 32) {
      int nw = blockDim.x >> 5;
      bs = threadIdx.x < nw ? s_s[threadIdx.x] : -INFINITY;
      br = threadIdx.x < nw ? s_r[threadIdx.x] : -1;
      for (int o = 16; o; o >>= 1) {
        S s2 = __shfl_xor_sync(FULL, bs, o);
        long long r2 = __shfl_xor_sync(FULL, br, o);
        if (r2 >= 0 && (br < 0 || s2 > bs || (s2 == bs && r2 < br))) { bs = s2; br = r2; }
      }
      if (threadIdx.x == 0) {
        out_s[j] = br >= 0 ? bs : -INFINITY;
        out_r[j] = br >= 0 ? row_base + br : -1LL;
        if (br >= 0) { prev_s = bs; prev_r = br; } else { prev_s = -INFINITY; prev_r = (long long)n; }
      }
    }
    __syncthreads();
  }
}

// select_topk_kernel of a distinct batch: each pass takes the next row in (score desc, row asc) order whose group
// (groups: by local row) is not taken yet.  Every row before the previous pick is a pick or of a taken group, so
// "strictly after the previous pick" stays the only order constraint.  The <= k taken groups sit in shared memory and
// are only consulted for a row that would beat the thread's current best.  S as in select_topk_kernel.
template <typename S>
__global__ void select_topk_distinct_kernel(const double *__restrict__ scores, int64_t n, int64_t row_base, int k, int64_t excl,
                                            const int *__restrict__ labels, int lab, const uint8_t *__restrict__ dead,
                                            const int *__restrict__ groups, S *out_s, long long *out_r) {
  __shared__ S s_s[32];
  __shared__ long long s_r[32];
  __shared__ int s_taken[32];
  __shared__ S prev_s;
  __shared__ long long prev_r;
  if (threadIdx.x == 0) { prev_s = INFINITY; prev_r = -1; }
  __syncthreads();
  for (int j = 0; j < k; j++) {
    S bs = -INFINITY;
    long long br = -1;
    const S ps = prev_s;
    const long long pr = prev_r;
    for (int64_t r = threadIdx.x; r < n; r += blockDim.x) {
      if (r == excl || (lab >= 0 && labels[r] != lab) || (dead && dead[r])) continue;
      S s = (S)scores[r];
      bool after = (s < ps) || (s == ps && r > pr);
      if (after && (br < 0 || s > bs || (s == bs && r < br))) {
        const int g = groups[r];
        bool seen = false;
        for (int t = 0; t < j; t++) seen |= s_taken[t] == g;
        if (!seen) { bs = s; br = r; }
      }
    }
    for (int o = 16; o; o >>= 1) {
      S s2 = __shfl_xor_sync(FULL, bs, o);
      long long r2 = __shfl_xor_sync(FULL, br, o);
      if (r2 >= 0 && (br < 0 || s2 > bs || (s2 == bs && r2 < br))) { bs = s2; br = r2; }
    }
    if ((threadIdx.x & 31) == 0) { s_s[threadIdx.x >> 5] = bs; s_r[threadIdx.x >> 5] = br; }
    __syncthreads();
    if (threadIdx.x < 32) {
      int nw = blockDim.x >> 5;
      bs = threadIdx.x < nw ? s_s[threadIdx.x] : -INFINITY;
      br = threadIdx.x < nw ? s_r[threadIdx.x] : -1;
      for (int o = 16; o; o >>= 1) {
        S s2 = __shfl_xor_sync(FULL, bs, o);
        long long r2 = __shfl_xor_sync(FULL, br, o);
        if (r2 >= 0 && (br < 0 || s2 > bs || (s2 == bs && r2 < br))) { bs = s2; br = r2; }
      }
      if (threadIdx.x == 0) {
        out_s[j] = br >= 0 ? bs : -INFINITY;
        out_r[j] = br >= 0 ? row_base + br : -1LL;
        s_taken[j] = br >= 0 ? groups[br] : -1;
        if (br >= 0) { prev_s = bs; prev_r = br; } else { prev_s = -INFINITY; prev_r = (long long)n; }
      }
    }
    __syncthreads();
  }
}

// fill_null_kernel of a distinct batch: one warp per null query walks the rows it may match (not excluded, of its
// label when filtered -- labels by local row --, live) in ascending order and keeps the first row of each new group
// until it has k.  A query whose eligible rows hold fewer than k groups walks the whole index.
__global__ void fill_null_distinct_kernel(const int *__restrict__ null_q, int n_null, int k, int64_t n_rows, int64_t row_base,
                                          const int *__restrict__ excl_by_query, const int *__restrict__ label_by_query,
                                          const int *__restrict__ labels, const uint8_t *__restrict__ dead,
                                          const int *__restrict__ groups, float *out_s, long long *out_r) {
  const int w = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n_null) return;
  const int q = null_q[w];
  const int ex = excl_by_query ? excl_by_query[q] : -1;  // by ORIGINAL query index
  const int lb = label_by_query ? label_by_query[q] : -1;
  int tg = -1;  // lane t: group of the t-th row taken
  int n = 0;
  for (int64_t r0 = 0; r0 < n_rows && n < k; r0 += 32) {
    const int64_t r = r0 + lane;
    const bool elig = r < n_rows && r != ex && (lb < 0 || labels[r] == lb) && !(dead && dead[r]);
    const int g = elig ? groups[r] : -1 - lane;
    bool fresh = elig;
    for (int t = 0; t < n; t++) fresh &= __shfl_sync(FULL, tg, t) != g;
    const uint32_t peers = __match_any_sync(FULL, g);
    fresh = fresh && __ffs(peers) - 1 == lane;  // the lowest row of its group among these 32
    for (uint32_t fm = __ballot_sync(FULL, fresh); fm && n < k; fm &= fm - 1, n++) {
      const int j = __ffs(fm) - 1;
      const int gj = __shfl_sync(FULL, g, j);
      if (lane == n) {
        tg = gj;
        out_s[(size_t)q * k + n] = 0.f;
        out_r[(size_t)q * k + n] = row_base + r0 + j;
      }
    }
  }
  if (lane >= n && lane < k) {
    out_s[(size_t)q * k + lane] = -INFINITY;
    out_r[(size_t)q * k + lane] = -1LL;
  }
}

// The null queries of a tag-filtered batch whose own tag set is not empty (the others keep what fill_null_kernel or
// fill_null_distinct_kernel wrote): one warp per query walks the rows in ascending order and keeps the first k it may
// match -- not excluded, of its label when filtered, live, tag set meeting the query's (q_tmask / q_tags by ORIGINAL
// query, rows through invperm to their scan position) -- and in distinct mode (groups by local row, NULL: not
// distinct) only the first row of each new group.  A query with fewer than k such rows walks the whole index.
__global__ void fill_null_tags_kernel(const int *__restrict__ null_q, int n_null, int k, int64_t n_rows, int64_t row_base,
                                      const int *__restrict__ excl_by_query, const int *__restrict__ label_by_query,
                                      const int *__restrict__ labels, const uint8_t *__restrict__ dead,
                                      const int *__restrict__ groups, const unsigned long long *__restrict__ q_tmask,
                                      const int *__restrict__ q_tags, const int *__restrict__ invperm,
                                      const unsigned long long *__restrict__ mask_pos, const int64_t *__restrict__ tag_ptr,
                                      const int *__restrict__ tag_list, float *out_s, long long *out_r) {
  const int w = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n_null) return;
  const int q = null_q[w];
  const unsigned long long qm = q_tmask[q];
  if (qm == 0ull) return;
  const int *qt = q_tags + (size_t)q * MAX_QTAGS;
  const int ex = excl_by_query ? excl_by_query[q] : -1;
  const int lb = label_by_query ? label_by_query[q] : -1;
  int tg = -1;  // lane t: group of the t-th row taken
  int n = 0;
  for (int64_t r0 = 0; r0 < n_rows && n < k; r0 += 32) {
    const int64_t r = r0 + lane;
    bool elig = r < n_rows && r != ex && (lb < 0 || labels[r] == lb) && !(dead && dead[r]);
    if (elig) {
      const int64_t pos = invperm[r];
      elig = tags_meet(mask_pos[pos], qm, tag_ptr, tag_list, pos, qt);
    }
    const int g = elig ? (groups ? groups[r] : (int)r) : -1 - lane;
    bool fresh = elig;
    if (groups) {
      for (int t = 0; t < n; t++) fresh &= __shfl_sync(FULL, tg, t) != g;
      const uint32_t peers = __match_any_sync(FULL, g);
      fresh = fresh && __ffs(peers) - 1 == lane;  // the lowest row of its group among these 32
    }
    for (uint32_t fm = __ballot_sync(FULL, fresh); fm && n < k; fm &= fm - 1, n++) {
      const int j = __ffs(fm) - 1;
      const int gj = __shfl_sync(FULL, g, j);
      if (lane == n) {
        tg = gj;
        out_s[(size_t)q * k + n] = 0.f;
        out_r[(size_t)q * k + n] = row_base + r0 + j;
      }
    }
  }
  if (lane >= n && lane < k) {
    out_s[(size_t)q * k + lane] = -INFINITY;
    out_r[(size_t)q * k + lane] = -1LL;
  }
}

// Fallback of a threshold search for one (irregular) query: every row whose float64 score, rounded to the float32
// select_topk_kernel reports, reaches the threshold is appended to the pair buffer (lab >= 0: rows of that label only;
// deleted rows never).
__global__ void select_range_kernel(const double *__restrict__ scores, int64_t n, int64_t row_base, float thr, int64_t excl,
                                    const int *__restrict__ labels, int lab, const uint8_t *__restrict__ dead, int q,
                                    RangePair *out, unsigned long long *count, unsigned long long cap) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int qv = q;
  // whole warps step together (blockDim is a multiple of 32): range_emit needs every lane
  for (int64_t r0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) & ~31LL; r0 < n; r0 += stride) {
    const int64_t r = r0 + (threadIdx.x & 31);
    const float s = r < n ? (float)scores[r] : -INFINITY;
    range_emit(out, count, cap, r < n && r != excl && (lab < 0 || labels[r] == lab) && !(dead && dead[r]) && s >= thr, &qv, s,
               row_base + r);
  }
}

// The same fallback for a Jaccard threshold search: the test is the float32 rounding of K1a's float64 ratio, and each
// pair carries its exact counts.  K1a forms s = I / (T - I) from exact integers (T = |q| + |row|) with one rounding,
// so I = rint(s T / (1 + s)) recovers |q ∩ row|: the expression is off by a few ulps of I, far below 1/2.
__global__ void jaccard_select_range_kernel(const double *__restrict__ scores, const double *__restrict__ B64,
                                            const int *__restrict__ invperm, int64_t n, double nq, float thr, int64_t excl,
                                            int q, JaccardPair *out, unsigned long long *count, unsigned long long cap) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  // whole warps step together (blockDim is a multiple of 32): one reservation per warp and 32 rows
  for (int64_t r0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) & ~31LL; r0 < n; r0 += stride) {
    const int64_t r = r0 + lane;
    const double s = r < n ? scores[r] : 0.0;
    const bool hit = r < n && r != excl && (float)s >= thr;
    const uint32_t hm = __ballot_sync(FULL, hit);
    if (hm == 0) continue;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(count, (unsigned long long)__popc(hm));
    base = __shfl_sync(FULL, base, 0);
    if (hit) {
      const double T = nq + B64[invperm[r]], I = rint(s * T / (1.0 + s));
      const unsigned long long o = base + (unsigned long long)__popc(hm & lanemask_lt());
      if (o < cap) out[o] = JaccardPair{q, (int)r, (int)I, (int)(T - I)};
    }
  }
}

}  // namespace kvk
