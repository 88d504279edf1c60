// K2: dense-embedding cosine scan with fused top-k on the Hopper tensor cores (BASELINE configs[1]:
// "1M-entry GFKB, 768-d embedding cosine, 10k-query batch").
//
// The reference has no embedding path (SURVEY.md section 0: only TF-IDF exists, dense embeddings are a
// documented possible extension, docs/failure-intelligence.md:43-46) -- parity for this kernel is
// UNPINNED; its oracle is oracle/tfidf_oracle.py::dense_cosine (float64 on the same bf16 inputs).
//
// scores[q, r] = <Q[q,:], C[r,:]> / (|Q[q]| |C[r]|): a bf16 GEMM Q * C^T with fp32 accumulation, the
// norms applied as fp32 scales in the epilogue, and the top-k fused into the epilogue so that the
// [Q, N] score matrix never exists.  A work item is one (128-query tile, row split); items are ordered
// split-major so that the CTAs resident together (one per SM) stream the same corpus rows through L2.  Few, long
// row splits keep every list's k-th-score threshold high.  Per CTA (288 threads):
//   warps 0-7   two consumer warpgroups, one per 64-query half of the tile: wgmma.mma_async m64n256k16 (bf16 in,
//               fp32 accumulators in registers, 128 per thread), then the epilogue on those registers: one shuffle
//               per pair of values gives every thread ONE query and half of the 256 columns (interleaved in groups of
//               two); scale, threshold test, insertion into the thread's own sorted top-k list (k <= 32; ties keep
//               the lower row; a self-join skips the query's own row)
//   warp 8      TMA producer: K-slices (64 elements) of the query tile and of the row tile -> 3-stage
//               shared-memory ring (128B-swizzled), mbarrier expect_tx / complete_tx; a slot is refilled once both
//               warpgroups' MMAs have read it (empty barrier, one arrival per consumer warp)
// While the consumers run a tile's epilogue, the producer already fills the ring with the next tile's first slices.
// Each (query tile, split, column half) writes one partial list; K5 (kv_merge_topk_device) merges them.  CTAs
// working on the same queries exchange k-th-score lower bounds through global memory (gthr).
// K2-R (dense_topk_kernel<true>) is the same kernel for a threshold search: producer, ring, MMAs and register exchange
// are unchanged; the epilogue keeps no lists and appends every pair whose score (the same float32 expression) reaches
// the threshold to a global pair buffer, one reservation per warp and 16-column group (dense_emit).
// FILTER and TAGS add the label and tag filters of a search (DenseFilter): items no query of the tile can match are
// skipped, and an element outside its query's filter gets a NaN scale.
#include "index_state.cuh"
#include "kv_cuda.cuh"
#include "sm90.cuh"

#include <cuda_bf16.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

namespace {

constexpr int BM = 128;        // queries per CTA (two 64-row wgmma tiles)
constexpr int BN = 256;        // corpus rows per MMA tile (the N of the wgmma)
constexpr int BK = 64;         // K-slice: 64 bf16 = one 128-byte swizzle row
constexpr int UMMA_K = 16;
constexpr int STAGES = 3;       // 3 x 48 KiB ring + two list sets fit in 227 KiB
constexpr int A_BYTES = BM * BK * 2;  // 16 KiB
constexpr int B_BYTES = BN * BK * 2;  // 32 KiB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int MAXK = 32;       // per-query list slots: 2 x 32 x 128 x 8 B = 64 KiB beside the 3 x 48 KiB ring (k <= 32)
constexpr int EPI_THREADS = 256;  // the two consumer warpgroups
constexpr int N_THREADS = EPI_THREADS + 32;  // + the TMA producer warp

// D[64 x 256] (+)= A[64 x 16] * B[256 x 16]^T, bf16 in, fp32 accumulators in registers (both operands K-major)
__device__ __forceinline__ void wgmma_m64n256k16_bf16(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
      "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, "
      "%42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, "
      "%62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, "
      "%82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, "
      "%101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, "
      "%117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]),
        "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),
        "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]),
        "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]),
        "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]),
        "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]),
        "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]),
        "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]),
        "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d)
      : "memory");
}

struct DenseParams {
  int64_t n_rows, row_base, n_q;
  int64_t excl_base;        // self-join: query q must not match global row excl_base + q (-1: no exclusion)
  int64_t r_tiles, q_tiles;  // 256-row tiles, 128-query tiles
  int dim, k, n_lists, dbg;
  const float *inv_norm_c;  // [n_rows]
  const float *inv_norm_q;  // [n_q]
  unsigned int *gthr;       // [n_q] order-preserving key of a lower bound of the global k-th score (0 = none)
  float *part_scores;       // [n_lists][n_q][k]
  long long *part_rows;
};

// Output of the threshold search (dense_topk_kernel<true>, which leaves k, gthr and the partial lists of DenseParams
// unused; the top-k form ignores this argument).  A kernel argument of its own: added to DenseParams it changes the
// top-k form's register allocation.
struct DenseRangeOut {
  float thr;                  // every pair whose score is >= thr is appended
  RangePair *out;             // [cap]
  unsigned long long *count;  // pairs found (may exceed cap: those past it are not written)
  unsigned long long cap;
};

// Label filter of one search (dense_topk_kernel<*, true>; the unfiltered forms ignore this argument).  The queries
// are in kernel order: stable-sorted by label, so that a 128-query tile holds few labels.  Query p (kernel order) is
// the call's query qperm[p]: its partial lists, its range records and its self-join exclusion use that index.
struct DenseFilter {
  const int *lab_c;                     // [n_rows] row labels (>= 0)
  const int *lab_q;                     // [n_q] query labels, kernel order (-1: any row)
  const int64_t *qperm;                 // [n_q] original query index of kernel query p
  const unsigned long long *tile_sig;   // [r_tiles] OR of 1 << (label & 63) over the tile's live rows
  const unsigned long long *qsig;       // [q_tiles] the same over the tile's queries (all ones: an unfiltered query)
  unsigned long long *skipped;          // (query tile, row tile) items skipped, counted by the producers
  // Tag filter (dense_topk_kernel<*, true, true>; tags_meet): query p only matches the rows whose tag set meets its own
  // (q_tmask[p] == 0: any row).  A tag-filtered call without labels runs with every query label -1 and lab_c =
  // tile_sig = NULL.  Rows by local row, queries in kernel order (stable-sorted by (label, smallest tag)).
  const unsigned long long *tmask_c;    // [n_rows] OR of 1 << (t & 63) over the row's tags
  const int64_t *tag_ptr;               // [n_rows + 1] CSR of the rows' tags; NULL when every tag is < 64
  const int *tag_list;
  const unsigned long long *q_tmask;    // [n_q] the queries' masks (0: no tag constraint)
  const int *q_tags;                    // [n_q][MAX_QTAGS] ascending, -1 past the last
  const unsigned long long *tile_tsig;  // [r_tiles] OR of the masks of the tile's live rows
  const unsigned long long *qtsig;      // [q_tiles] OR of the tile's query masks (all ones: a query without tags; no tag skip)
};

// order-preserving float <-> unsigned key (cosines may be negative)
__device__ __forceinline__ unsigned int fkey(float f) {
  unsigned int b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

struct __align__(1024) DenseSmem {
  unsigned char stage[STAGES][STAGE_BYTES];
  uint64_t full_bar[STAGES], empty_bar[STAGES];
  __align__(16) float inv_c[2][BN];
  float lscore[2][MAXK][BM];  // [column half][slot][query]: the 32 lanes of a warp hit 32 different banks
  int lrow[2][MAXK][BM];
  int lab_c[2][BN];  // FILTER: this tile's row labels (-1 past the end); last, so the other members keep their offsets
  __align__(16) unsigned long long tmask_c[2][BN];  // TAGS: this tile's row tag masks (0 past the end); after lab_c for the same reason
};

// Whether the producer skips item (query tile qtile, row tile t): no live row of the tile carries a label (FILTER) or a
// tag (TAGS) of any query of the tile.  Each signature test alone has no false negatives.
template <bool TAGS>
__device__ __forceinline__ bool item_skipped(const DenseFilter &F, int64_t t, int qtile) {
  if constexpr (TAGS) {
    // a query without tags (qtsig all ones: a tagged query sets at most MAX_QTAGS bits) matches rows without tags too,
    // which tile_tsig does not record, so its tile takes no tag test
    if (F.qtsig[qtile] != ~0ull && (F.tile_tsig[t] & F.qtsig[qtile]) == 0) return true;
    if (!F.tile_sig) return false;  // no label filter in this call
  }
  return (F.tile_sig[t] & F.qsig[qtile]) == 0;
}

// K2-R: appends this thread's pairs of one 16-column group (columns c0 + {0, 1, 4, 5, 8, 9, 12, 13} of the tile at
// row0): (q, tv[e] * inv_q, global row) for each element whose score reaches R.thr, whose row exists, is not the
// excluded one and passes keep(local row).  All 32 lanes call it; the warp reserves its records with one atomic (none
// when no lane has a hit).
template <class Keep>
__device__ __forceinline__ void dense_emit(const DenseParams &P, const DenseRangeOut &R, const float (&tv)[8], float inv_q, int q,
                                           int64_t row0, int c0, int excl, Keep keep) {
  const int lane = threadIdx.x & 31;
  uint32_t hits = 0;
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const int64_t r = row0 + c0 + 8 * (e >> 2) + 4 * ((e >> 1) & 1) + (e & 1);
    if (tv[e] * inv_q >= R.thr && r < P.n_rows && (int)r != excl && keep(r)) hits |= 1u << e;
  }
  const int nh = __popc(hits);
  int incl = nh;  // inclusive prefix sum of the warp's hit counts: lane 31 holds the total
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if (lane >= o) incl += v;
  }
  unsigned long long base = 0;
  if (lane == 31 && incl > 0) base = atomicAdd(R.count, (unsigned long long)incl);
  unsigned long long o = __shfl_sync(0xFFFFFFFFu, base, 31) + (unsigned long long)(incl - nh);
#pragma unroll
  for (int e = 0; e < 8; e++) {
    if (hits & (1u << e)) {
      const int64_t r = row0 + c0 + 8 * (e >> 2) + 4 * ((e >> 1) & 1) + (e & 1);
      if (o < R.cap) R.out[o] = RangePair{q, tv[e] * inv_q, P.row_base + r};
      o++;
    }
  }
}

// FILTER: query p only matches rows labelled F.lab_q[p] (-1: any row).  An item whose row tile holds no live row of
// any label of its query tile (tile_sig & qsig == 0; a signature has no false negatives) is skipped by the producer
// (no loads) and by the consumers (no MMAs, ring waits or epilogue) alike, so the ring's stage and phase stay in step.
// TAGS (instantiated with FILTER only): query p also only matches rows whose tag set meets its own; the items whose row
// tile carries no tag of any query of the tile (tile_tsig & qtsig == 0) are skipped the same way.  An element whose row
// mask misses the query's gets a NaN scale; when some tag of the index is >= 64 a mask hit is confirmed on the row's
// tag list (tags_meet) where an element would enter a list or be emitted, the only places its eligibility matters.
template <bool RANGE, bool FILTER, bool TAGS = false>
__global__ void __launch_bounds__(N_THREADS, 1)
dense_topk_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c, DenseParams P,
                  DenseRangeOut R, DenseFilter F) {
  extern __shared__ unsigned char smem_raw[];
  DenseSmem &S = *reinterpret_cast<DenseSmem *>(smem_raw + smem_align1024(smem_raw));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // work item = (query tile, row split); consecutive CTAs take consecutive query tiles of the same split, so the
  // CTAs resident at one time stream the same corpus rows (B tiles are shared through L2)
  const int64_t item = blockIdx.x;
  const int64_t my_qtile = item % P.q_tiles, my_split = item / P.q_tiles;
  const int64_t L0 = my_qtile * P.r_tiles + P.r_tiles * my_split / P.n_lists;
  const int64_t L1 = my_qtile * P.r_tiles + P.r_tiles * (my_split + 1) / P.n_lists;
  const int n_kb = P.dim / BK;
  constexpr unsigned FULL_MASK = 0xFFFFFFFFu;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; i++) { mbar_init(&S.full_bar[i], 1); mbar_init(&S.empty_bar[i], EPI_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == EPI_THREADS / 32) {
    // ===== TMA producer =====
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      unsigned long long n_skip = 0;
      for (int64_t L = L0; L < L1; L++) {
        const int qtile = (int)(L / P.r_tiles);
        const int64_t t = L % P.r_tiles;
        if constexpr (FILTER) {
          if (item_skipped<TAGS>(F, t, qtile)) { n_skip++; continue; }
        }
        for (int kb = 0; kb < n_kb; kb++) {
          mbar_wait(&S.empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&S.full_bar[stage], STAGE_BYTES);
          tma_load_2d(S.stage[stage], &map_q, &S.full_bar[stage], kb * BK, qtile * BM);
          tma_load_2d(S.stage[stage] + A_BYTES, &map_c, &S.full_bar[stage], kb * BK, (int)(t * BN));
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      if constexpr (FILTER) {
        if (n_skip) atomicAdd(F.skipped, n_skip);
      }
    }
  } else {
    // ===== consumers: MMA, then epilogue on the accumulator registers =====
    // m64nNk16 accumulator fragment: warp w of the warpgroup holds rows 16 w + lane / 4 (register 4 j + e, e < 2) and
    // 16 w + lane / 4 + 8 (e >= 2), columns 8 j + 2 (lane % 4) + (e & 1).  After the exchange with lane ^ 2, lanes with
    // lane % 4 < 2 hold the first of those rows, the others the second, each for columns 8 j + 2 (lane & 1) + {0, 1}
    // ("lo") and 8 j + 4 + 2 (lane & 1) + {0, 1} ("hi"): one query, half of the columns, ascending in j.
    const int wg = warp >> 2, wq = warp & 3;
    const int quad = lane & 3;
    const bool upper = quad >= 2;
    const int qi = wg * 64 + wq * 16 + (lane >> 2) + (upper ? 8 : 0);  // query inside the tile
    const int et = threadIdx.x;                 // 0..255 among the epilogue threads
    const int half = quad & 1;                  // which interleaved half of every tile's columns this thread scans
    const int cofs = 2 * half;                  // column of register 4 j + m: 8 j + cofs + (m & 1) + 4 (m >> 1)
    const int k = P.k;
    float *ls = &S.lscore[half][0][qi];         // element j of this thread's list lives at ls[j * BM]
    int *lr = &S.lrow[half][0][qi];
    int cur_qtile = -1, cnt = 0;
    int excl = -1;          // local row this thread's query must not match (self-join)
    int64_t q = 0;
    bool q_ok = false;
    float inv_q = 0.f;
    float thr = -INFINITY;  // own k-th score: later rows must beat it strictly (rows ascend inside a CTA)
    float gth = -INFINITY;  // k-th score another CTA already secured for this query: ties may still win on row id
    float gth_pred = -INFINITY;  // largest float below gth (-0 is not below +0)
    float lo = INFINITY;         // a row enters the list iff its score > lo
    int qlab = -1;               // FILTER: this thread's query label (-1: any row)
    int64_t qo = 0;              // FILTER: the call's index of this thread's query, qperm[q]
    unsigned long long qtm = 0;  // TAGS: this thread's query mask (0: any row)
    const int *qtl = nullptr;    // TAGS: its ascending tags
    auto flush = [&]() {    // publish the list of (cur_qtile, this CTA)
      if (cur_qtile < 0 || !q_ok) return;
      const int slot = (int)my_split * 2 + half;
      for (int j = 0; j < k; j++) {
        const size_t o = ((size_t)slot * P.n_q + (FILTER ? qo : q)) * k + j;
        P.part_scores[o] = j < cnt ? ls[j * BM] : -INFINITY;
        P.part_rows[o] = j < cnt ? (long long)(P.row_base + lr[j * BM]) : -1LL;
      }
    };
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; i++) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    int64_t it = 0;
    for (int64_t L = L0; L < L1; L++, it++) {
      const int qtile = (int)(L / P.r_tiles);
      const int64_t t = L % P.r_tiles;
      bool skip = false;  // (CTA-uniform) the producer issued no loads for this item
      if constexpr (FILTER) skip = item_skipped<TAGS>(F, t, qtile);
      int prev = -1;
      if (!skip) {
        // ---- MMA over the K slices; a slice's ring slot is released once the next slice's MMAs are issued and the
        //      slice's own have completed ----
#pragma unroll
        for (int i = 0; i < 128; i++) wgmma_reg_fence(acc[i]);
        wgmma_fence();
        for (int kb = 0; kb < n_kb; kb++) {
          mbar_wait(&S.full_bar[stage], phase);
          const uint64_t da = wgmma_desc_sw128(S.stage[stage] + wg * (A_BYTES / 2));  // rows 64 wg .. 64 wg + 63 of the tile
          const uint64_t db = wgmma_desc_sw128(S.stage[stage] + A_BYTES);
#pragma unroll
          for (int kk = 0; kk < BK / UMMA_K; kk++)  // advance 32 bytes (2 x 16-byte units) per K=16 step inside the swizzle row
            wgmma_m64n256k16_bf16(acc, da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), (uint32_t)((kb | kk) != 0));
          wgmma_commit();
          if (prev >= 0) {
            wgmma_wait<1>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&S.empty_bar[prev]);
          }
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      // the query-tile switch runs for a skipped item too: a query tile whose first row tiles are all skipped must
      // still publish the previous tile's lists and start its own
      if (qtile != cur_qtile) {  // (CTA-uniform) next query tile: publish and restart the lists
        if constexpr (!RANGE) flush();
        cur_qtile = qtile;
        q = (int64_t)qtile * BM + qi;
        q_ok = q < P.n_q;
        inv_q = q_ok ? P.inv_norm_q[q] : 0.f;
        if constexpr (FILTER) {
          qlab = q_ok ? F.lab_q[q] : -1;
          qo = q_ok ? F.qperm[q] : q;
        }
        if constexpr (TAGS) {
          qtm = q_ok ? F.q_tmask[q] : 0ull;
          qtl = F.q_tags + (q_ok ? q : 0) * MAX_QTAGS;
        }
        {
          const int64_t e = P.excl_base >= 0 ? P.excl_base + (FILTER ? qo : q) - P.row_base : -1;
          excl = (e >= 0 && e < P.n_rows) ? (int)e : -1;
        }
        if constexpr (!RANGE) {
          cnt = 0;
          thr = gth = gth_pred = -INFINITY;
          lo = q_ok ? -INFINITY : INFINITY;
          for (int j = 0; j < k; j++) { ls[j * BM] = -INFINITY; lr[j * BM] = 0x7fffffff; }
        }
      }
      if constexpr (FILTER) {
        // `it` counts the tiles whose inverse norms and labels were staged: the double buffer alternates between
        // processed tiles only
        if (skip) { it--; continue; }
      }
      const int as = (int)(it & 1);
      // inverse norms of this tile's rows (0 past the end; such rows are rejected by index below)
      const int64_t row0 = t * BN;
      for (int c = et; c < BN; c += EPI_THREADS) S.inv_c[as][c] = (row0 + c < P.n_rows) ? P.inv_norm_c[row0 + c] : -INFINITY;  // 0 * -inf = NaN: never a candidate
      if constexpr (FILTER) {
        if (!TAGS || F.lab_c)
          for (int c = et; c < BN; c += EPI_THREADS) S.lab_c[as][c] = (row0 + c < P.n_rows) ? F.lab_c[row0 + c] : -1;
      }
      if constexpr (TAGS) {
        for (int c = et; c < BN; c += EPI_THREADS) S.tmask_c[as][c] = (row0 + c < P.n_rows) ? F.tmask_c[row0 + c] : 0ull;
      }
      if constexpr (!RANGE) {
        if (q_ok) {
          const unsigned int gk = *(volatile unsigned int *)&P.gthr[q];
          if (gk > fkey(-INFINITY) && fkey_inv(gk) > gth) {
            gth = fkey_inv(gk);
            // the order-preserving key makes "previous float" a decrement, except below +0: the key before it is -0,
            // which compares equal to +0 and would reject the rows scoring exactly 0 that tie with a k-th score of 0
            gth_pred = fkey_inv(gk - (gk == fkey(0.f) ? 2u : 1u));
            lo = fmaxf(thr, gth_pred);
          }
        }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < 128; i++) wgmma_reg_fence(acc[i]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&S.empty_bar[prev]);
      if (P.dbg == 1) continue;
      // one query per thread: swap the row this thread does not keep with lane ^ 2
#pragma unroll
      for (int j = 0; j < 32; j++) {
        const float s0 = upper ? acc[4 * j + 0] : acc[4 * j + 2], s1 = upper ? acc[4 * j + 1] : acc[4 * j + 3];
        const float m0 = upper ? acc[4 * j + 2] : acc[4 * j + 0], m1 = upper ? acc[4 * j + 3] : acc[4 * j + 1];
        const float g0 = __shfl_xor_sync(FULL_MASK, s0, 2), g1 = __shfl_xor_sync(FULL_MASK, s1, 2);
        acc[4 * j + 0] = upper ? g0 : m0;
        acc[4 * j + 1] = upper ? g1 : m1;
        acc[4 * j + 2] = upper ? m0 : g0;
        acc[4 * j + 3] = upper ? m1 : g1;
      }
      if (P.dbg == 2) { if (acc[0] == 1.2345678f && acc[127] == 9.87654321f) thr = 1.f; continue; }
      // per 8 values (16 columns): scale, max -> one branch; only groups where some query of the warp has a
      // candidate are walked element by element (`sc > lo` == `sc > thr && sc >= gth`, lo = max(thr, pred(gth)))
      // A NaN scale removes an element: a deleted row's inverse norm is NaN (kv_dense_finalize), and so is the scale of
      // a row outside a filtered query's label here, and a deleted self-join query's inv_q.  fmaxf drops NaN operands,
      // and NaN fails every `> lo` and `>= thr` test, so such an element is never a candidate and never emitted.  Neither
      // edge case turns NaN into a number: a zero query has inv_q = 0 and NaN * 0 is NaN; a padded row (past n_rows)
      // is never deleted and has the -inf scale, whose products are -inf or NaN (0 * -inf) and fail the same tests.
#pragma unroll
      for (int sb = 0; sb < 16; sb++) {
        float tv[8];
#pragma unroll
        for (int jj = 0; jj < 2; jj++) {
          const int j = 2 * sb + jj;
          float2 icl = *reinterpret_cast<const float2 *>(&S.inv_c[as][8 * j + cofs]);
          float2 ich = *reinterpret_cast<const float2 *>(&S.inv_c[as][8 * j + 4 + cofs]);
          if constexpr (FILTER) {
            if (qlab >= 0) {
              const int2 ll = *reinterpret_cast<const int2 *>(&S.lab_c[as][8 * j + cofs]);
              const int2 lh = *reinterpret_cast<const int2 *>(&S.lab_c[as][8 * j + 4 + cofs]);
              if (ll.x != qlab) icl.x = __int_as_float(0x7fc00000);
              if (ll.y != qlab) icl.y = __int_as_float(0x7fc00000);
              if (lh.x != qlab) ich.x = __int_as_float(0x7fc00000);
              if (lh.y != qlab) ich.y = __int_as_float(0x7fc00000);
            }
          }
          if constexpr (TAGS) {
            if (qtm) {
              const ulonglong2 ml = *reinterpret_cast<const ulonglong2 *>(&S.tmask_c[as][8 * j + cofs]);
              const ulonglong2 mh = *reinterpret_cast<const ulonglong2 *>(&S.tmask_c[as][8 * j + 4 + cofs]);
              if (!(ml.x & qtm)) icl.x = __int_as_float(0x7fc00000);
              if (!(ml.y & qtm)) icl.y = __int_as_float(0x7fc00000);
              if (!(mh.x & qtm)) ich.x = __int_as_float(0x7fc00000);
              if (!(mh.y & qtm)) ich.y = __int_as_float(0x7fc00000);
            }
          }
          tv[4 * jj + 0] = acc[4 * j + 0] * icl.x;
          tv[4 * jj + 1] = acc[4 * j + 1] * icl.y;
          tv[4 * jj + 2] = acc[4 * j + 2] * ich.x;
          tv[4 * jj + 3] = acc[4 * j + 3] * ich.y;
        }
        const float m01 = fmaxf(tv[0], tv[1]), m23 = fmaxf(tv[2], tv[3]);
        const float m45 = fmaxf(tv[4], tv[5]), m67 = fmaxf(tv[6], tv[7]);
        const float best = fmaxf(fmaxf(m01, m23), fmaxf(m45, m67)) * inv_q;
        if constexpr (RANGE) {
          // inv_q > 0 and rounding is monotone, so no score of the group reaches thr unless best does (zero and
          // padded queries have inv_q = 0: best is 0 or NaN)
          if (__any_sync(FULL_MASK, best >= R.thr)) {
            if constexpr (TAGS) {
              dense_emit(P, R, tv, inv_q, (int)qo, row0, 16 * sb + cofs, excl, [&](int64_t r) {
                return qtm == 0ull || tags_meet(S.tmask_c[as][r - row0], qtm, F.tag_ptr, F.tag_list, r, qtl);
              });
            } else {
              dense_emit(P, R, tv, inv_q, (int)(FILTER ? qo : q), row0, 16 * sb + cofs, excl, [](int64_t) { return true; });
            }
          }
        } else {
          if (best > lo) {
            if constexpr (TAGS) {
              auto insert = [&](float sc, int col) {
                int pos = cnt < k ? cnt++ : k - 1;
                while (pos > 0 && ls[(pos - 1) * BM] < sc) {
                  ls[pos * BM] = ls[(pos - 1) * BM];
                  lr[pos * BM] = lr[(pos - 1) * BM];
                  pos--;
                }
                ls[pos * BM] = sc;
                lr[pos * BM] = (int)(row0 + col);
                if (cnt == k) { thr = ls[(k - 1) * BM]; lo = fmaxf(thr, gth_pred); }
              };
              // the group's candidates by score and exclusion; when some tag is >= 64 a rolled loop confirms each on
              // its row's tag list, so that the list test is compiled once per group, not once per element
              uint32_t cb = 0;
#pragma unroll
              for (int e = 0; e < 8; e++) {
                const int col = 8 * (2 * sb + (e >> 2)) + cofs + (e & 1) + 4 * ((e >> 1) & 1);
                if (tv[e] * inv_q > lo && (int)(row0 + col) != excl) cb |= 1u << e;
              }
              if (cb && qtm && F.tag_ptr) {
                for (uint32_t m = cb; m; m &= m - 1) {
                  const int e = __ffs(m) - 1;
                  const int col = 8 * (2 * sb + (e >> 2)) + cofs + (e & 1) + 4 * ((e >> 1) & 1);
                  if (!tags_meet(S.tmask_c[as][col], qtm, F.tag_ptr, F.tag_list, row0 + col, qtl)) cb &= ~(1u << e);
                }
              }
#pragma unroll  // static indices keep tv[] in registers
              for (int e = 0; e < 8; e++) {
                const float sc = tv[e] * inv_q;
                const int col = 8 * (2 * sb + (e >> 2)) + cofs + (e & 1) + 4 * ((e >> 1) & 1);
                if (((cb >> e) & 1u) && sc > lo) insert(sc, col);  // lo may have risen since cb was formed
              }
            } else {
#pragma unroll  // static indices keep tv[] in registers
              for (int e = 0; e < 8; e++) {
                const float sc = tv[e] * inv_q;
                const int col = 8 * (2 * sb + (e >> 2)) + cofs + (e & 1) + 4 * ((e >> 1) & 1);
                if (sc > lo && (int)(row0 + col) != excl) {
                  int pos = cnt < k ? cnt++ : k - 1;
                  while (pos > 0 && ls[(pos - 1) * BM] < sc) {
                    ls[pos * BM] = ls[(pos - 1) * BM];
                    lr[pos * BM] = lr[(pos - 1) * BM];
                    pos--;
                  }
                  ls[pos * BM] = sc;
                  lr[pos * BM] = (int)(row0 + col);
                  if (cnt == k) { thr = ls[(k - 1) * BM]; lo = fmaxf(thr, gth_pred); }
                }
              }
            }
          }
        }
      }
      if constexpr (!RANGE) {
        if (q_ok && cnt == k && thr > gth) atomicMax(&P.gthr[q], fkey(thr));
      }
    }
    if constexpr (!RANGE) flush();
  }
}

// inverse L2 norms of bf16 rows (float64 accumulation); zero rows get 0 (their scores are 0)
__global__ void inv_norm_kernel(const __nv_bfloat16 *__restrict__ x, int64_t n, int dim, float *out) {
  const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  double s = 0.0;
  for (int i = lane; i < dim; i += 32) {
    double v = (double)__bfloat162float(x[r * dim + i]);
    s += v * v;
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
  if (lane == 0) out[r] = s > 0.0 ? (float)(1.0 / sqrt(s)) : 0.f;
}

// tombstones: x[idx[i]] = NaN (a deleted row's inverse norm, or a deleted self-join query's)
__global__ void nan_scatter_kernel(float *x, const int64_t *__restrict__ idx, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) x[idx[i]] = __int_as_float(0x7fc00000);
}

// one block of BN threads per 256-row tile: OR of 1 << (label & 63) over the tile's live rows (a deleted row has a NaN
// inverse norm); an all-deleted tile gets 0
__global__ void tile_sig_kernel(const int *__restrict__ lab, const float *__restrict__ inv_c, int64_t n,
                                unsigned long long *sig) {
  __shared__ unsigned long long s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  const int64_t r = blockIdx.x * (int64_t)BN + threadIdx.x;
  if (r < n && !isnan(inv_c[r])) atomicOr(&s, 1ull << (lab[r] & 63));
  __syncthreads();
  if (threadIdx.x == 0) sig[blockIdx.x] = s;
}

// the same for the tag filter: OR of the tag masks of the tile's live rows
__global__ void tile_tag_sig_kernel(const unsigned long long *__restrict__ mask, const float *__restrict__ inv_c, int64_t n,
                                    unsigned long long *sig) {
  __shared__ unsigned long long s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  const int64_t r = blockIdx.x * (int64_t)BN + threadIdx.x;
  if (r < n && !isnan(inv_c[r]) && mask[r]) atomicOr(&s, mask[r]);
  __syncthreads();
  if (threadIdx.x == 0) sig[blockIdx.x] = s;
}

// dst[p] = src[perm[p]], bf16 rows of dim elements (dim a multiple of 64: 16-byte vectors)
__global__ void gather_rows_kernel(const uint4 *__restrict__ src, const int64_t *__restrict__ perm, int64_t n, int vec_per_row,
                                   uint4 *dst) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n * vec_per_row) return;
  const int64_t p = i / vec_per_row;
  const int v = (int)(i % vec_per_row);
  dst[i] = src[perm[p] * vec_per_row + v];
}

}  // namespace

struct kv_dense_index {
  int device = 0, dim = 0;
  int64_t row_base = 0;
  CudaStream stream;
  CudaEvent ev[2];
  std::mutex mu;
  int sm_count = 132;
  DevVec<__nv_bfloat16> rows;
  int64_t n_rows = 0;
  DevBuf<float> d_inv_c, d_inv_q, d_part_s, d_out_s;
  DevBuf<long long> d_part_r, d_out_r;
  DevBuf<__nv_bfloat16> d_q;
  DevBuf<unsigned int> d_gthr;
  // last threshold search, kept until fetched or until the next range, top-k, append, deletion or finalize
  RangeResult<RangePair> range;
  RangeOrderScratch rsort;  // the fetches order the pairs on the device (range_order.cu)
  bool finalized = false;
  float last_ms = 0;
  int64_t last_splits = 0;
  // row deletion, applied as NaN inverse norms at every finalize
  Tombstones tomb;
  DevBuf<int64_t> d_dead;  // the deleted rows (finalize) or deleted self-join query positions (a search)
  // row labels: kept by finalize and deletions, dropped by an append; the device copy and the tile signatures are
  // rebuilt at every finalize and label upload
  std::vector<int> h_labels;
  bool has_labels = false;
  DevBuf<int> d_lab_c;
  DevBuf<unsigned long long> d_tile_sig;
  // query filter of the next search call (kv_dense_set_query_filter), and that call's device inputs
  std::vector<int> h_qfilter;
  bool has_qfilter = false;
  DevBuf<int> d_lab_q;
  DevBuf<int64_t> d_qperm;
  DevBuf<unsigned long long> d_qsig, d_skipped;
  DevBuf<__nv_bfloat16> d_qf;  // the filtered call's queries in kernel order (when that order is not the identity)
  int64_t last_skipped = 0, last_items = 0;
  // row tag sets (kv_dense_set_row_tags), with the lifetime of the row labels: uploaded when set (masks by local row,
  // and the CSR unless every tag is < 64); the tile tag signatures are rebuilt at every finalize and tag upload
  bool has_tags = false, tags_exact = true;
  int64_t tag_rows = 0;  // the row count they were set for
  DevBuf<unsigned long long> d_tmask_c, d_tile_tsig;
  DevBuf<int64_t> d_tag_ptr;
  DevBuf<int> d_tag_list;
  // tag filter of the next search call (kv_dense_set_tag_filter), by original query, and that call's device inputs
  std::vector<unsigned long long> h_qtmask;
  std::vector<int> h_qtlist;
  bool has_qtags = false;
  DevBuf<unsigned long long> d_q_tmask, d_qtsig;
  DevBuf<int> d_q_tags;
};

namespace {

// A search call's query filter, taken from the handle (which it leaves cleared) and then laid out in kernel order.
struct CallFilter {
  bool on = false;               // some query is filtered (label or tags): a FILTER kernel runs
  bool labels = false;           // some query has a label
  bool tags = false;             // some query has tags: the TAGS kernel runs
  std::vector<int> lab;          // [n_q] by original query (all -1 when only tags were given)
  std::vector<unsigned long long> tmask;  // tags: [n_q] by original query (0: no tag constraint)
  std::vector<int> tlist;                 // tags: [n_q][MAX_QTAGS] by original query, ascending, -1 past the last
  std::vector<int64_t> perm;     // [n_q] kernel order -> original query (stable sort by label, then smallest tag)
  bool identity = true;
};

// Takes (and clears) the handle's query label and tag filters for a call of n_q queries.  Caller holds dx->mu.
int take_filter(kv_dense_index *dx, int64_t n_q, const char *fn, CallFilter &cf) {
  const bool had_lab = dx->has_qfilter, had_tags = dx->has_qtags;
  dx->has_qfilter = dx->has_qtags = false;
  cf = CallFilter{};
  if (had_lab) {
    cf.lab.swap(dx->h_qfilter);
    if ((int64_t)cf.lab.size() != n_q)
      return kv_fail(KV_ERR_INVALID, "%s: the query filter has %lld labels for a call of %lld queries", fn, (long long)cf.lab.size(),
                     (long long)n_q);
    for (int l : cf.lab) cf.labels = cf.labels || l >= 0;
  }
  if (had_tags) {
    cf.tmask.swap(dx->h_qtmask);
    cf.tlist.swap(dx->h_qtlist);
    if ((int64_t)cf.tmask.size() != n_q)
      return kv_fail(KV_ERR_INVALID, "%s: the tag filter has %lld tag sets for a call of %lld queries", fn, (long long)cf.tmask.size(),
                     (long long)n_q);
    for (unsigned long long m : cf.tmask) cf.tags = cf.tags || m != 0ull;
  }
  cf.on = cf.labels || cf.tags;
  if (!cf.on) return KV_OK;  // every query unfiltered: the unfiltered call
  if (cf.labels && (!dx->has_labels || (int64_t)dx->h_labels.size() != dx->n_rows))
    return kv_fail(KV_ERR_STATE, "%s: the index has no row labels for its current rows (kv_dense_set_row_labels)", fn);
  if (cf.tags && (!dx->has_tags || dx->tag_rows != dx->n_rows))
    return kv_fail(KV_ERR_STATE, "%s: the index has no row tags for its current rows (kv_dense_set_row_tags)", fn);
  if (!cf.labels) cf.lab.assign((size_t)n_q, -1);
  cf.perm.resize((size_t)n_q);
  for (int64_t i = 0; i < n_q; i++) cf.perm[(size_t)i] = i;
  if (cf.tags) {  // (label, smallest tag): a query tile holds few apps; the queries without tags (-1) lead their label
    const auto key = [&](int64_t q) { return std::make_pair(cf.lab[(size_t)q], cf.tlist[(size_t)q * MAX_QTAGS]); };
    std::stable_sort(cf.perm.begin(), cf.perm.end(), [&](int64_t a, int64_t b) { return key(a) < key(b); });
  } else {
    std::stable_sort(cf.perm.begin(), cf.perm.end(), [&](int64_t a, int64_t b) { return cf.lab[(size_t)a] < cf.lab[(size_t)b]; });
  }
  for (int64_t i = 0; i < n_q && cf.identity; i++) cf.identity = cf.perm[(size_t)i] == i;
  return KV_OK;
}

// What an append of n rows changes besides the rows: the index needs a finalize, the row labels and tags and the query
// filters are dropped, the deleted rows stay deleted and the new rows are live.
void dense_rows_appended(kv_dense_index *dx, int64_t n) {
  dx->n_rows += n;
  dx->rows.n = dx->n_rows * dx->dim;
  dx->finalized = false;
  dx->has_labels = false;
  dx->h_labels.clear();
  dx->has_qfilter = false;
  dx->has_tags = false;
  dx->has_qtags = false;
  dx->tomb.extend(dx->n_rows);
}

// Rebuilds the tile signatures from the device labels and the inverse norms (NaN = deleted).  Needs a finalized index
// with labels on the device.
int build_tile_sig(kv_dense_index *dx) {
  const int64_t r_tiles = (dx->n_rows + BN - 1) / BN;
  if (!r_tiles) return KV_OK;
  KV_CUDA(dx->d_tile_sig.ensure(r_tiles));
  tile_sig_kernel<<<(unsigned)r_tiles, BN, 0, dx->stream>>>(dx->d_lab_c.p, dx->d_inv_c.p, dx->n_rows, dx->d_tile_sig.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(dx->stream));
  return KV_OK;
}

// Rebuilds the tile tag signatures from the device tag masks and the inverse norms.  Needs a finalized index with row
// tags on the device.
int build_tile_tsig(kv_dense_index *dx) {
  const int64_t r_tiles = (dx->n_rows + BN - 1) / BN;
  if (!r_tiles) return KV_OK;
  KV_CUDA(dx->d_tile_tsig.ensure(r_tiles));
  tile_tag_sig_kernel<<<(unsigned)r_tiles, BN, 0, dx->stream>>>(dx->d_tmask_c.p, dx->d_inv_c.p, dx->n_rows, dx->d_tile_tsig.p);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(dx->stream));
  return KV_OK;
}

// Writes NaN at x[idx[i]] for the host list idx (through dx->d_dead).
int scatter_nan(kv_dense_index *dx, float *x, const std::vector<int64_t> &idx) {
  if (idx.empty()) return KV_OK;
  const int64_t n = (int64_t)idx.size();
  KV_CUDA(dx->d_dead.ensure(n));
  KV_CUDA(cudaMemcpyAsync(dx->d_dead.p, idx.data(), (size_t)n * 8, cudaMemcpyHostToDevice, dx->stream));
  nan_scatter_kernel<<<(unsigned)((n + 255) / 256), 256, 0, dx->stream>>>(x, dx->d_dead.p, n);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaStreamSynchronize(dx->stream));  // idx may be freed once this returns
  return KV_OK;
}

}  // namespace

extern "C" {

int kv_dense_create(int device, int dim, int64_t row_base, kv_dense_index **out) {
  if (!out) return kv_fail(KV_ERR_INVALID, "kv_dense_create: out is NULL");
  if (dim < BK || dim % BK != 0 || dim > 8192) return kv_fail(KV_ERR_INVALID, "kv_dense_create: dim must be a multiple of 64 (64..8192)");
  int sm_count = 0;
  int rc = open_device(device, "kv_dense_create", &sm_count);
  if (rc != KV_OK) return rc;
  std::unique_ptr<kv_dense_index> dx(new kv_dense_index());
  dx->device = device;
  dx->dim = dim;
  dx->row_base = row_base;
  dx->sm_count = sm_count;
  KV_CUDA(dx->stream.create());
  for (auto &e : dx->ev) KV_CUDA(e.create());
  KV_CUDA(cudaFuncSetAttribute(dense_topk_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DenseSmem) + 1024));
  KV_CUDA(cudaFuncSetAttribute(dense_topk_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DenseSmem) + 1024));
  KV_CUDA(cudaFuncSetAttribute(dense_topk_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DenseSmem) + 1024));
  KV_CUDA(cudaFuncSetAttribute(dense_topk_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DenseSmem) + 1024));
  KV_CUDA(cudaFuncSetAttribute(dense_topk_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DenseSmem) + 1024));
  KV_CUDA(cudaFuncSetAttribute(dense_topk_kernel<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DenseSmem) + 1024));
  *out = dx.release();
  return KV_OK;
}

void kv_dense_destroy(kv_dense_index *dx) {
  if (!dx) return;
  cudaSetDevice(dx->device);
  cudaStreamSynchronize(dx->stream);
  delete dx;
}

int64_t kv_dense_rows(const kv_dense_index *dx) { return dx ? dx->n_rows : 0; }

// rows: n x dim bfloat16 (raw uint16 bit patterns), row-major, host memory
int kv_dense_append(kv_dense_index *dx, const uint16_t *rows_bf16, int64_t n) {
  if (!dx || n < 0 || (n > 0 && !rows_bf16)) return kv_fail(KV_ERR_INVALID, "kv_dense_append: bad arguments");
  if (n == 0) return KV_OK;
  std::lock_guard<std::mutex> g(dx->mu);
  dx->range.drop();
  KV_CUDA(cudaSetDevice(dx->device));
  if (dx->n_rows + n >= (1LL << 31) - BN) return kv_fail(KV_ERR_INVALID, "kv_dense_append: more than 2^31 rows in one shard");
  KV_CUDA(dx->rows.reserve((dx->n_rows + n) * dx->dim, dx->stream));
  KV_CUDA(cudaMemcpyAsync(dx->rows.p + dx->n_rows * dx->dim, rows_bf16, (size_t)n * dx->dim * 2, cudaMemcpyHostToDevice, dx->stream));
  KV_CUDA(cudaStreamSynchronize(dx->stream));
  dense_rows_appended(dx, n);
  return KV_OK;
}

int kv_dense_finalize(kv_dense_index *dx) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_finalize: NULL handle");
  std::lock_guard<std::mutex> g(dx->mu);
  dx->range.drop();
  dx->has_qfilter = dx->has_qtags = false;
  KV_CUDA(cudaSetDevice(dx->device));
  KV_CUDA(dx->d_inv_c.ensure(std::max<int64_t>(dx->n_rows, 1)));
  if (dx->n_rows) {
    inv_norm_kernel<<<(unsigned)((dx->n_rows * 32 + 255) / 256), 256, 0, dx->stream>>>(dx->rows.p, dx->n_rows, dx->dim, dx->d_inv_c.p);
    KV_CUDA(cudaGetLastError());
  }
  KV_CUDA(cudaStreamSynchronize(dx->stream));
  // tombstones: a deleted row's inverse norm is NaN, which removes every score of the row in the epilogue
  if (dx->tomb.any()) {
    std::vector<int64_t> dead;
    dead.reserve((size_t)dx->tomb.count);
    for (int64_t r = 0; r < dx->n_rows; r++)
      if (dx->tomb.is_dead(r)) dead.push_back(r);
    const int rc = scatter_nan(dx, dx->d_inv_c.p, dead);
    if (rc != KV_OK) return rc;
  }
  if (dx->has_labels) {
    const int rc = build_tile_sig(dx);
    if (rc != KV_OK) return rc;
  }
  if (dx->has_tags) {
    const int rc = build_tile_tsig(dx);
    if (rc != KV_OK) return rc;
  }
  dx->finalized = true;
  return KV_OK;
}

int kv_dense_delete_rows(kv_dense_index *dx, const int64_t *rows, int64_t n) {
  if (!dx || n < 0 || (n > 0 && !rows)) return kv_fail(KV_ERR_INVALID, "kv_dense_delete_rows: bad arguments");
  std::lock_guard<std::mutex> g(dx->mu);
  int64_t added = 0;
  const int rc = dx->tomb.mark(rows, n, dx->n_rows, "kv_dense_delete_rows", &added);
  if (rc != KV_OK || !added) return rc;  // duplicates and rows deleted before: nothing changes
  // like an append: the inverse norms and tile signatures are stale until the next finalize
  dx->finalized = false;
  dx->range.drop();
  return KV_OK;
}

int64_t kv_dense_live_rows(const kv_dense_index *dx) { return dx ? dx->n_rows - dx->tomb.count : 0; }

int kv_dense_deleted_rows(kv_dense_index *dx, uint8_t *out, int64_t n) {
  if (!dx || n < 0 || (n > 0 && !out)) return kv_fail(KV_ERR_INVALID, "kv_dense_deleted_rows: bad arguments");
  std::lock_guard<std::mutex> g(dx->mu);
  return dx->tomb.copy_out(out, n, dx->n_rows, "kv_dense_deleted_rows");
}

int kv_dense_set_row_labels(kv_dense_index *dx, const int32_t *labels, int64_t n) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_set_row_labels: NULL handle");
  std::lock_guard<std::mutex> g(dx->mu);
  if (!labels) {
    dx->h_labels.clear();
    dx->has_labels = false;
    return KV_OK;
  }
  if (n != dx->n_rows)
    return kv_fail(KV_ERR_INVALID, "kv_dense_set_row_labels: %lld labels for an index of %lld rows", (long long)n, (long long)dx->n_rows);
  for (int64_t i = 0; i < n; i++)
    if (labels[i] < 0) return kv_fail(KV_ERR_INVALID, "kv_dense_set_row_labels: label %d of row %lld is negative", labels[i], (long long)i);
  KV_CUDA(cudaSetDevice(dx->device));
  dx->has_labels = false;
  dx->h_labels.assign(labels, labels + n);
  KV_CUDA(dx->d_lab_c.ensure(std::max<int64_t>(n, 1)));
  KV_CUDA(cudaMemcpyAsync(dx->d_lab_c.p, labels, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, dx->stream));
  KV_CUDA(cudaStreamSynchronize(dx->stream));
  dx->has_labels = true;
  return dx->finalized ? build_tile_sig(dx) : KV_OK;  // else the next finalize builds the signatures
}

int kv_dense_set_query_filter(kv_dense_index *dx, const int32_t *labels, int64_t n_q) {
  if (!dx || n_q < 0) return kv_fail(KV_ERR_INVALID, "kv_dense_set_query_filter: bad arguments");
  std::lock_guard<std::mutex> g(dx->mu);
  dx->has_qfilter = false;
  if (!labels) return KV_OK;
  for (int64_t q = 0; q < n_q; q++)
    if (labels[q] < -1)
      return kv_fail(KV_ERR_INVALID, "kv_dense_set_query_filter: label %d of query %lld is below -1", labels[q], (long long)q);
  dx->h_qfilter.assign(labels, labels + n_q);
  dx->has_qfilter = true;
  return KV_OK;
}

int kv_dense_set_row_tags(kv_dense_index *dx, const int64_t *indptr, const int32_t *tags, int64_t n) {
  const char *fn = "kv_dense_set_row_tags";
  if (!dx) return kv_fail(KV_ERR_INVALID, "%s: NULL handle", fn);
  std::lock_guard<std::mutex> g(dx->mu);
  if (!indptr) {
    dx->has_tags = false;
    return KV_OK;
  }
  bool exact = true;
  const int rc = check_row_tags(indptr, tags, n, dx->n_rows, fn, &exact);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaSetDevice(dx->device));
  dx->has_tags = false;
  std::vector<unsigned long long> mask((size_t)n, 0ull);
  for (int64_t r = 0; r < n; r++)
    for (int64_t i = indptr[r]; i < indptr[r + 1]; i++) mask[(size_t)r] |= 1ull << (tags[i] & 63);
  cudaStream_t s = dx->stream;
  KV_CUDA(dx->d_tmask_c.ensure(std::max<int64_t>(n, 1)));
  if (n) KV_CUDA(cudaMemcpyAsync(dx->d_tmask_c.p, mask.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
  if (!exact) {
    KV_CUDA(dx->d_tag_ptr.ensure(n + 1));
    KV_CUDA(dx->d_tag_list.ensure(std::max<int64_t>(indptr[n], 1)));
    KV_CUDA(cudaMemcpyAsync(dx->d_tag_ptr.p, indptr, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, s));
    if (indptr[n]) KV_CUDA(cudaMemcpyAsync(dx->d_tag_list.p, tags, (size_t)indptr[n] * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  KV_CUDA(cudaStreamSynchronize(s));  // the caller's arrays and the staged masks may go once this returns
  dx->tags_exact = exact;
  dx->tag_rows = n;
  dx->has_tags = true;
  return dx->finalized ? build_tile_tsig(dx) : KV_OK;  // else the next finalize builds the signatures
}

int kv_dense_set_tag_filter(kv_dense_index *dx, const int64_t *indptr, const int32_t *tags, int64_t n_q) {
  const char *fn = "kv_dense_set_tag_filter";
  if (!dx || n_q < 0) return kv_fail(KV_ERR_INVALID, "%s: bad arguments", fn);
  std::lock_guard<std::mutex> g(dx->mu);
  dx->has_qtags = false;
  if (!indptr) return KV_OK;
  bool any = false;
  const int rc = parse_query_tag_csr(indptr, tags, n_q, fn, "indptr", dx->h_qtmask, dx->h_qtlist, &any);
  if (rc != KV_OK) return rc;
  dx->has_qtags = true;
  return KV_OK;
}

int kv_dense_last_skipped(const kv_dense_index *dx, int64_t *skipped, int64_t *items) {
  if (!dx || !skipped || !items) return kv_fail(KV_ERR_INVALID, "kv_dense_last_skipped: bad arguments");
  *skipped = dx->last_skipped;
  *items = dx->last_items;
  return KV_OK;
}

// What the top-k and the range scan of n_q queries already on the device (d_q: bf16 [n_q, dim], 16-byte aligned)
// share: the queries' inverse norms, both tensor maps, the row splits (dx->last_splits) and every DenseParams field but
// the epilogue's.  A filtered call (cf.on) runs on its queries in kernel order: d_q gathered into dx->d_qf unless that
// order is the identity, and F filled.  sj_begin >= 0: the queries are the local rows sj_begin.., and a deleted one
// gets a NaN inverse norm (an empty list, no pairs).  Needs n_rows > 0.
static int dense_setup(kv_dense_index *dx, const __nv_bfloat16 *d_q, int64_t n_q, int64_t excl_base, int64_t sj_begin,
                       const CallFilter &cf, CUtensorMap *map_q, CUtensorMap *map_c, DenseParams &P, DenseFilter &F) {
  cudaStream_t s = dx->stream;
  if (cf.on) {
    KV_CUDA(dx->d_qperm.ensure(n_q));
    KV_CUDA(cudaMemcpyAsync(dx->d_qperm.p, cf.perm.data(), (size_t)n_q * 8, cudaMemcpyHostToDevice, s));
    if (!cf.identity) {
      const int vpr = dx->dim / 8;  // 16-byte vectors per row
      KV_CUDA(dx->d_qf.ensure(n_q * dx->dim));
      gather_rows_kernel<<<(unsigned)((n_q * vpr + 255) / 256), 256, 0, s>>>((const uint4 *)d_q, dx->d_qperm.p, n_q, vpr,
                                                                                (uint4 *)dx->d_qf.p);
      KV_CUDA(cudaGetLastError());
      d_q = dx->d_qf.p;
    }
  }
  KV_CUDA(dx->d_inv_q.ensure(n_q));
  inv_norm_kernel<<<(unsigned)((n_q * 32 + 255) / 256), 256, 0, s>>>(d_q, n_q, dx->dim, dx->d_inv_q.p);
  KV_CUDA(cudaGetLastError());
  if (sj_begin >= 0 && dx->tomb.any()) {
    std::vector<int64_t> dead_q;  // kernel positions of the deleted query rows
    for (int64_t p = 0; p < n_q; p++)
      if (dx->tomb.is_dead(sj_begin + (cf.on ? cf.perm[(size_t)p] : p))) dead_q.push_back(p);
    const int rc = scatter_nan(dx, dx->d_inv_q.p, dead_q);
    if (rc != KV_OK) return rc;
  }
  int rc = make_map_2d(map_q, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, d_q, n_q, dx->dim, BM);
  if (rc != KV_OK) return rc;
  rc = make_map_2d(map_c, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, dx->rows.p, dx->n_rows, dx->dim, BN);
  if (rc != KV_OK) return rc;
  const int64_t q_tiles = (n_q + BM - 1) / BM, r_tiles = (dx->n_rows + BN - 1) / BN;
  // row splits: as few as possible (long row ranges keep the k-th-score thresholds high) while the CTA count
  // fills whole waves of SMs (one CTA per SM)
  int64_t n_lists = 1;
  {
    double best = 1e18;
    const int64_t lo = std::max<int64_t>(1, (dx->sm_count + q_tiles - 1) / q_tiles);
    for (int64_t sp = lo; sp <= std::min<int64_t>(r_tiles, lo + 16); sp++) {
      const int64_t ctas = q_tiles * sp, waves = (ctas + dx->sm_count - 1) / dx->sm_count;
      const double cost = (double)(waves * dx->sm_count) / (double)ctas * (1.0 + 0.01 * (double)sp);
      if (cost < best) { best = cost; n_lists = sp; }
    }
    n_lists = std::max<int64_t>(1, std::min<int64_t>(n_lists, r_tiles));
  }
  dx->last_splits = n_lists;
  P = DenseParams{};
  P.n_rows = dx->n_rows; P.row_base = dx->row_base; P.n_q = n_q; P.dim = dx->dim; P.n_lists = (int)n_lists;
  P.excl_base = excl_base;
  P.r_tiles = r_tiles; P.q_tiles = q_tiles;
  P.dbg = getenv("KAKVEDA_B200_DENSE_DBG") ? atoi(getenv("KAKVEDA_B200_DENSE_DBG")) : 0;
  P.inv_norm_c = dx->d_inv_c.p; P.inv_norm_q = dx->d_inv_q.p;
  dx->last_items = q_tiles * r_tiles;
  dx->last_skipped = 0;
  F = DenseFilter{};
  if (cf.on) {
    std::vector<int> lab_q((size_t)n_q);
    std::vector<unsigned long long> qsig((size_t)q_tiles, 0ull);
    for (int64_t p = 0; p < n_q; p++) {
      const int l = cf.lab[(size_t)cf.perm[(size_t)p]];
      lab_q[(size_t)p] = l;
      qsig[(size_t)(p / BM)] |= l < 0 ? ~0ull : 1ull << (l & 63);
    }
    KV_CUDA(dx->d_lab_q.ensure(n_q)); KV_CUDA(dx->d_qsig.ensure(q_tiles)); KV_CUDA(dx->d_skipped.ensure(1));
    KV_CUDA(cudaMemcpyAsync(dx->d_lab_q.p, lab_q.data(), (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaMemcpyAsync(dx->d_qsig.p, qsig.data(), (size_t)q_tiles * 8, cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaMemsetAsync(dx->d_skipped.p, 0, 8, s));
    F.lab_q = dx->d_lab_q.p; F.qperm = dx->d_qperm.p;
    F.qsig = dx->d_qsig.p; F.skipped = dx->d_skipped.p;
    if (cf.labels) { F.lab_c = dx->d_lab_c.p; F.tile_sig = dx->d_tile_sig.p; }
  }
  if (cf.tags) {
    std::vector<unsigned long long> q_tmask((size_t)n_q), qtsig((size_t)q_tiles, 0ull);
    std::vector<int> q_tags((size_t)n_q * MAX_QTAGS);
    for (int64_t p = 0; p < n_q; p++) {
      const int64_t q = cf.perm[(size_t)p];
      const unsigned long long m = cf.tmask[(size_t)q];
      q_tmask[(size_t)p] = m;
      std::copy_n(cf.tlist.begin() + q * MAX_QTAGS, MAX_QTAGS, q_tags.begin() + p * MAX_QTAGS);
      qtsig[(size_t)(p / BM)] |= m == 0ull ? ~0ull : m;
    }
    KV_CUDA(dx->d_q_tmask.ensure(n_q)); KV_CUDA(dx->d_q_tags.ensure(n_q * MAX_QTAGS)); KV_CUDA(dx->d_qtsig.ensure(q_tiles));
    KV_CUDA(cudaMemcpyAsync(dx->d_q_tmask.p, q_tmask.data(), (size_t)n_q * 8, cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaMemcpyAsync(dx->d_q_tags.p, q_tags.data(), q_tags.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaMemcpyAsync(dx->d_qtsig.p, qtsig.data(), (size_t)q_tiles * 8, cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaStreamSynchronize(s));  // the staged vectors go out of scope
    F.tmask_c = dx->d_tmask_c.p;
    F.tag_ptr = dx->tags_exact ? nullptr : dx->d_tag_ptr.p;
    F.tag_list = dx->tags_exact ? nullptr : dx->d_tag_list.p;
    F.q_tmask = dx->d_q_tmask.p; F.q_tags = dx->d_q_tags.p;
    F.tile_tsig = dx->d_tile_tsig.p; F.qtsig = dx->d_qtsig.p;
  }
  return KV_OK;
}

// launches the top-k or the threshold (range) form of K2, filtered when F.qperm is set, tag-filtered when F.q_tmask is
static void dense_launch(bool range, cudaStream_t s, int64_t grid, const CUtensorMap &map_q, const CUtensorMap &map_c,
                         const DenseParams &P, const DenseRangeOut &R, const DenseFilter &F) {
  const size_t smem = sizeof(DenseSmem) + 1024;
  if (range && F.q_tmask) dense_topk_kernel<true, true, true><<<(unsigned)grid, N_THREADS, smem, s>>>(map_q, map_c, P, R, F);
  else if (F.q_tmask) dense_topk_kernel<false, true, true><<<(unsigned)grid, N_THREADS, smem, s>>>(map_q, map_c, P, R, F);
  else if (range && F.qperm) dense_topk_kernel<true, true><<<(unsigned)grid, N_THREADS, smem, s>>>(map_q, map_c, P, R, F);
  else if (range) dense_topk_kernel<true, false><<<(unsigned)grid, N_THREADS, smem, s>>>(map_q, map_c, P, R, F);
  else if (F.qperm) dense_topk_kernel<false, true><<<(unsigned)grid, N_THREADS, smem, s>>>(map_q, map_c, P, R, F);
  else dense_topk_kernel<false, false><<<(unsigned)grid, N_THREADS, smem, s>>>(map_q, map_c, P, R, F);
}

// after a filtered kernel (stream synchronized): its skip count
static int read_skipped(kv_dense_index *dx, const DenseFilter &F) {
  if (!F.qperm) return KV_OK;
  unsigned long long v = 0;
  KV_CUDA(cudaMemcpy(&v, F.skipped, 8, cudaMemcpyDeviceToHost));
  dx->last_skipped = (int64_t)v;
  return KV_OK;
}

// scan + merge of n_q queries already on the device (d_q: bf16 [n_q, dim], 16-byte aligned) into device buffers
static int dense_run(kv_dense_index *dx, const __nv_bfloat16 *d_q, int64_t n_q, int k, int64_t excl_base, int64_t sj_begin,
                     const CallFilter &cf, float *d_out_s, long long *d_out_r) {
  cudaStream_t s = dx->stream;
  dx->last_items = dx->last_skipped = 0;
  if (dx->n_rows == 0) {
    KV_CUDA(cudaMemsetAsync(d_out_r, 0xFF, (size_t)n_q * k * 8, s));  // row -1
    std::vector<float> neg((size_t)(n_q * k), -INFINITY);
    KV_CUDA(cudaMemcpyAsync(d_out_s, neg.data(), neg.size() * 4, cudaMemcpyHostToDevice, s));
    KV_CUDA(cudaStreamSynchronize(s));
    return KV_OK;
  }
  CUtensorMap map_q, map_c;
  DenseParams P;
  DenseFilter F;
  int rc = dense_setup(dx, d_q, n_q, excl_base, sj_begin, cf, &map_q, &map_c, P, F);
  if (rc != KV_OK) return rc;
  const int64_t n_part = (int64_t)P.n_lists * 2;  // two epilogue threads (column halves) per query and CTA
  KV_CUDA(dx->d_part_s.ensure(n_part * n_q * k)); KV_CUDA(dx->d_part_r.ensure(n_part * n_q * k));
  KV_CUDA(dx->d_gthr.ensure(n_q));
  KV_CUDA(cudaMemsetAsync(dx->d_gthr.p, 0, (size_t)n_q * 4, s));
  // unused (query tile, slot) pairs stay "empty": row -1 (the merge ignores their scores)
  KV_CUDA(cudaMemsetAsync(dx->d_part_r.p, 0xFF, (size_t)n_part * n_q * k * 8, s));
  KV_CUDA(cudaMemsetAsync(dx->d_part_s.p, 0xFF, (size_t)n_part * n_q * k * 4, s));
  P.k = k;
  P.gthr = dx->d_gthr.p;
  P.part_scores = dx->d_part_s.p; P.part_rows = dx->d_part_r.p;
  const int64_t grid = P.q_tiles * P.n_lists;
  KV_CUDA(cudaEventRecord(dx->ev[0], s));
  dense_launch(false, s, grid, map_q, map_c, P, DenseRangeOut{}, F);
  KV_CUDA(cudaGetLastError());
  KV_CUDA(cudaEventRecord(dx->ev[1], s));
  KV_CUDA(cudaStreamSynchronize(s));
  cudaEventElapsedTime(&dx->last_ms, dx->ev[0], dx->ev[1]);
  rc = read_skipped(dx, F);
  if (rc != KV_OK) return rc;
  return kv_merge_topk_device(dx->device, dx->d_part_s.p, dx->d_part_r.p, (int)n_part, n_q, k, d_out_s, d_out_r);
}

// Threshold search of n_q queries already on the device (as dense_run): every pair whose score reaches thr lands in
// dx->range, in emit order, for kv_dense_range_fetch.  When a search finds more pairs than the buffer holds, it grows to
// the exact count and the kernel runs once more -- the whole GEMM again, since the pairs are only known in its epilogue.  last_ms sums
// both runs.  Caller holds dx->mu.
static int dense_range(kv_dense_index *dx, const __nv_bfloat16 *d_q, int64_t n_q, float thr, int64_t excl_base,
                       int64_t sj_begin, const CallFilter &cf, int64_t *n_pairs) {
  cudaStream_t s = dx->stream;
  unsigned long long count = 0;
  float total_ms = 0.f;
  dx->last_splits = 0;
  dx->last_items = dx->last_skipped = 0;
  if (dx->n_rows > 0 && n_q > 0) {
    CUtensorMap map_q, map_c;
    DenseParams P;
    DenseFilter F;
    int rc = dense_setup(dx, d_q, n_q, excl_base, sj_begin, cf, &map_q, &map_c, P, F);
    if (rc != KV_OK) return rc;
    if ((rc = dx->range.prepare(s)) != KV_OK) return rc;
    DenseRangeOut R;
    R.thr = thr;
    R.count = dx->range.d_count.p;
    const int64_t grid = P.q_tiles * P.n_lists;
    for (;;) {
      R.out = dx->range.pairs.p;
      R.cap = dx->range.capacity();
      if (F.qperm) KV_CUDA(cudaMemsetAsync(F.skipped, 0, 8, s));
      KV_CUDA(cudaEventRecord(dx->ev[0], s));
      dense_launch(true, s, grid, map_q, map_c, P, R, F);
      KV_CUDA(cudaGetLastError());
      KV_CUDA(cudaEventRecord(dx->ev[1], s));
      KV_CUDA(cudaMemcpyAsync(&count, R.count, sizeof(count), cudaMemcpyDeviceToHost, s));
      KV_CUDA(cudaStreamSynchronize(s));
      float ms = 0.f;
      cudaEventElapsedTime(&ms, dx->ev[0], dx->ev[1]);
      total_ms += ms;
      rc = read_skipped(dx, F);
      if (rc != KV_OK) return rc;
      if (count <= R.cap) break;
      if ((rc = dx->range.grow(count, s, "kv_dense_range")) != KV_OK) return rc;
    }
  }
  dx->last_ms = total_ms;
  dx->range.commit(n_q, (int64_t)count);
  *n_pairs = (int64_t)count;
  return KV_OK;
}

// The entry points below take the handle's query filter first and leave it cleared, whether they succeed or fail.

// q: n_q x dim bfloat16 bit patterns (host).  Outputs (host): scores float32[n_q*k], rows int64[n_q*k],
// ordered by (score desc, row asc); unused slots (-inf, -1).
int kv_dense_topk(kv_dense_index *dx, const uint16_t *q_bf16, int64_t n_q, int k, float *out_scores, int64_t *out_rows) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_topk: bad arguments (k must be 1..32)");
  std::lock_guard<std::mutex> g(dx->mu);
  CallFilter cf;
  const int frc = take_filter(dx, n_q, "kv_dense_topk", cf);
  if (n_q < 0 || k < 1 || k > MAXK || (n_q > 0 && (!q_bf16 || !out_scores || !out_rows)))
    return kv_fail(KV_ERR_INVALID, "kv_dense_topk: bad arguments (k must be 1..32)");
  dx->range.drop();
  if (!dx->finalized) return kv_fail(KV_ERR_STATE, "kv_dense_topk: index not finalized");
  if (frc != KV_OK) return frc;
  if (n_q == 0) return KV_OK;
  KV_CUDA(cudaSetDevice(dx->device));
  cudaStream_t s = dx->stream;
  KV_CUDA(dx->d_q.ensure(n_q * dx->dim));
  KV_CUDA(cudaMemcpyAsync(dx->d_q.p, q_bf16, (size_t)n_q * dx->dim * 2, cudaMemcpyHostToDevice, s));
  KV_CUDA(dx->d_out_s.ensure(n_q * k)); KV_CUDA(dx->d_out_r.ensure(n_q * k));
  int rc = dense_run(dx, dx->d_q.p, n_q, k, -1, -1, cf, dx->d_out_s.p, dx->d_out_r.p);
  if (rc != KV_OK) return rc;
  KV_CUDA(cudaMemcpy(out_scores, dx->d_out_s.p, (size_t)n_q * k * 4, cudaMemcpyDeviceToHost));
  KV_CUDA(cudaMemcpy(out_rows, dx->d_out_r.p, (size_t)n_q * k * 8, cudaMemcpyDeviceToHost));
  return KV_OK;
}

int kv_dense_topk_device(kv_dense_index *dx, const void *d_q_bf16, int64_t n_q, int k, int64_t exclude_base, void *d_scores,
                         void *d_rows) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_topk_device: bad arguments (k must be 1..32)");
  std::lock_guard<std::mutex> g(dx->mu);
  CallFilter cf;
  const int frc = take_filter(dx, n_q, "kv_dense_topk_device", cf);
  if (n_q < 0 || k < 1 || k > MAXK || (n_q > 0 && (!d_q_bf16 || !d_scores || !d_rows)))
    return kv_fail(KV_ERR_INVALID, "kv_dense_topk_device: bad arguments (k must be 1..32)");
  if (((uintptr_t)d_q_bf16 & 15) != 0) return kv_fail(KV_ERR_INVALID, "kv_dense_topk_device: queries must be 16-byte aligned");
  dx->range.drop();
  if (!dx->finalized) return kv_fail(KV_ERR_STATE, "kv_dense_topk_device: index not finalized");
  if (frc != KV_OK) return frc;
  if (n_q == 0) return KV_OK;
  KV_CUDA(cudaSetDevice(dx->device));
  return dense_run(dx, (const __nv_bfloat16 *)d_q_bf16, n_q, k, exclude_base, -1, cf, (float *)d_scores, (long long *)d_rows);
}

// rows already on the device (e.g. a torch tensor): device-to-device append
int kv_dense_append_device(kv_dense_index *dx, const void *d_rows_bf16, int64_t n) {
  if (!dx || n < 0 || (n > 0 && !d_rows_bf16)) return kv_fail(KV_ERR_INVALID, "kv_dense_append_device: bad arguments");
  if (n == 0) return KV_OK;
  std::lock_guard<std::mutex> g(dx->mu);
  dx->range.drop();
  KV_CUDA(cudaSetDevice(dx->device));
  if (dx->n_rows + n >= (1LL << 31) - BN) return kv_fail(KV_ERR_INVALID, "kv_dense_append_device: more than 2^31 rows in one shard");
  KV_CUDA(dx->rows.reserve((dx->n_rows + n) * dx->dim, dx->stream));
  KV_CUDA(cudaMemcpyAsync(dx->rows.p + dx->n_rows * dx->dim, d_rows_bf16, (size_t)n * dx->dim * 2, cudaMemcpyDeviceToDevice, dx->stream));
  KV_CUDA(cudaStreamSynchronize(dx->stream));
  dense_rows_appended(dx, n);
  return KV_OK;
}

// all-pairs (BASELINE configs[3]): local rows [q_begin, q_end) as queries against the whole shard, each row's own
// entry excluded; outputs on the device
int kv_dense_selfjoin_device(kv_dense_index *dx, int64_t q_begin, int64_t q_end, int k, void *d_scores, void *d_rows) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_selfjoin_device: bad arguments (k must be 1..32)");
  std::lock_guard<std::mutex> g(dx->mu);
  CallFilter cf;
  const int frc = take_filter(dx, q_end - q_begin, "kv_dense_selfjoin_device", cf);
  if (q_begin < 0 || q_end < q_begin || k < 1 || k > MAXK || !d_scores || !d_rows)
    return kv_fail(KV_ERR_INVALID, "kv_dense_selfjoin_device: bad arguments (k must be 1..32)");
  dx->range.drop();
  if (!dx->finalized) return kv_fail(KV_ERR_STATE, "kv_dense_selfjoin_device: index not finalized");
  if (q_end > dx->n_rows) return kv_fail(KV_ERR_INVALID, "kv_dense_selfjoin_device: row range outside the index");
  if (frc != KV_OK) return frc;
  if (q_end == q_begin) return KV_OK;
  KV_CUDA(cudaSetDevice(dx->device));
  return dense_run(dx, dx->rows.p + q_begin * dx->dim, q_end - q_begin, k, dx->row_base + q_begin, q_begin, cf,
                   (float *)d_scores, (long long *)d_rows);
}

static bool valid_threshold(float thr) { return thr > 0.f && thr <= 1.f; }  // false for NaN

int kv_dense_range(kv_dense_index *dx, const uint16_t *q_bf16, int64_t n_q, float threshold, int64_t *n_pairs) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_range: bad arguments (n_q must be below 2^31)");
  std::lock_guard<std::mutex> g(dx->mu);
  CallFilter cf;
  const int frc = take_filter(dx, n_q, "kv_dense_range", cf);
  if (!n_pairs || n_q < 0 || n_q >= (1LL << 31) || (n_q > 0 && !q_bf16))
    return kv_fail(KV_ERR_INVALID, "kv_dense_range: bad arguments (n_q must be below 2^31)");
  if (!valid_threshold(threshold)) return kv_fail(KV_ERR_INVALID, "kv_dense_range: threshold must be in (0, 1]");
  dx->range.drop();
  if (!dx->finalized) return kv_fail(KV_ERR_STATE, "kv_dense_range: index not finalized");
  if (frc != KV_OK) return frc;
  KV_CUDA(cudaSetDevice(dx->device));
  if (n_q > 0 && dx->n_rows > 0) {
    KV_CUDA(dx->d_q.ensure(n_q * dx->dim));
    KV_CUDA(cudaMemcpyAsync(dx->d_q.p, q_bf16, (size_t)n_q * dx->dim * 2, cudaMemcpyHostToDevice, dx->stream));
  }
  return dense_range(dx, dx->d_q.p, n_q, threshold, -1, -1, cf, n_pairs);
}

int kv_dense_range_device(kv_dense_index *dx, const void *d_q_bf16, int64_t n_q, float threshold, int64_t exclude_base,
                          int64_t *n_pairs) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_range_device: bad arguments (n_q must be below 2^31)");
  std::lock_guard<std::mutex> g(dx->mu);
  CallFilter cf;
  const int frc = take_filter(dx, n_q, "kv_dense_range_device", cf);
  if (!n_pairs || n_q < 0 || n_q >= (1LL << 31) || (n_q > 0 && !d_q_bf16))
    return kv_fail(KV_ERR_INVALID, "kv_dense_range_device: bad arguments (n_q must be below 2^31)");
  if (((uintptr_t)d_q_bf16 & 15) != 0) return kv_fail(KV_ERR_INVALID, "kv_dense_range_device: queries must be 16-byte aligned");
  if (!valid_threshold(threshold)) return kv_fail(KV_ERR_INVALID, "kv_dense_range_device: threshold must be in (0, 1]");
  dx->range.drop();
  if (!dx->finalized) return kv_fail(KV_ERR_STATE, "kv_dense_range_device: index not finalized");
  if (frc != KV_OK) return frc;
  KV_CUDA(cudaSetDevice(dx->device));
  return dense_range(dx, (const __nv_bfloat16 *)d_q_bf16, n_q, threshold, exclude_base, -1, cf, n_pairs);
}

int kv_dense_selfjoin_range(kv_dense_index *dx, int64_t q_begin, int64_t q_end, float threshold, int64_t *n_pairs) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_selfjoin_range: bad arguments");
  std::lock_guard<std::mutex> g(dx->mu);
  CallFilter cf;
  const int frc = take_filter(dx, q_end - q_begin, "kv_dense_selfjoin_range", cf);
  if (!n_pairs || q_begin < 0 || q_end < q_begin || q_end - q_begin >= (1LL << 31))
    return kv_fail(KV_ERR_INVALID, "kv_dense_selfjoin_range: bad arguments");
  if (!valid_threshold(threshold)) return kv_fail(KV_ERR_INVALID, "kv_dense_selfjoin_range: threshold must be in (0, 1]");
  dx->range.drop();
  if (!dx->finalized) return kv_fail(KV_ERR_STATE, "kv_dense_selfjoin_range: index not finalized");
  if (q_end > dx->n_rows) return kv_fail(KV_ERR_INVALID, "kv_dense_selfjoin_range: row range outside the index");
  if (frc != KV_OK) return frc;
  KV_CUDA(cudaSetDevice(dx->device));
  return dense_range(dx, dx->rows.p + q_begin * dx->dim, q_end - q_begin, threshold, dx->row_base + q_begin, q_begin, cf,
                     n_pairs);
}

// The pairs come back in emit order, which the kernel does not fix; (score desc, row asc) is a total order of each
// query's pairs, so the result is deterministic.  Both fetches order the pairs on the device and consume the result
// (RangeResult).
int kv_dense_range_fetch(kv_dense_index *dx, int64_t *indptr, int64_t *rows, float *scores) {
  if (!dx || !indptr) return kv_fail(KV_ERR_INVALID, "kv_dense_range_fetch: bad arguments");
  std::lock_guard<std::mutex> g(dx->mu);
  return dx->range.fetch_host("kv_dense_range_fetch", "kv_dense_range*", dx->device, dx->stream, dx->rsort, 0, indptr, rows,
                              scores, nullptr, nullptr);
}

// Device outputs: the same arrays, written to caller-owned device memory of the index's device.
int kv_dense_range_fetch_device(kv_dense_index *dx, void *d_indptr, void *d_rows, void *d_scores) {
  if (!dx) return kv_fail(KV_ERR_INVALID, "kv_dense_range_fetch_device: bad arguments");
  std::lock_guard<std::mutex> g(dx->mu);
  return dx->range.fetch_device("kv_dense_range_fetch_device", "kv_dense_range*", dx->device, dx->stream, dx->rsort, 0, d_indptr,
                                d_rows, d_scores, nullptr, nullptr);
}

int kv_dense_last_timing(const kv_dense_index *dx, float *gemm_ms, int64_t *splits) {
  if (!dx || !gemm_ms || !splits) return kv_fail(KV_ERR_INVALID, "kv_dense_last_timing: bad arguments");
  *gemm_ms = dx->last_ms;
  *splits = dx->last_splits;
  return KV_OK;
}

}  // extern "C"
