// K1b-B: upper bounds of every (query, chunk) score on the Hopper tensor cores, and the candidate lists they leave.
//
// For a query q and a chunk c (32 rows), with U_c(t) = largest tf of feature t in the chunk (0 if absent) and
// Bmin_c = smallest positive row norm of the chunk:
//     dot(q, r) <= dotS_q + dotX_q + sum_{t frequent} W_q(t) U_c(t) + sum_{t rare, in the chunk} w_tile(t) U_c(t)
//     B_r + corr(q, r) >= Bmin_c + corrS_q                                  (corrS_q: every d(t) of q at its largest tf)
// so  score(q, r) <= ub(q, c) = dot_bound / sqrt(|q|^2 (Bmin_c + corrS_q))  for every row r of c  (exact block-max
// pruning: a chunk whose bound is below a query's k-th best score cannot hold a top-k row for it).
//   * the sum over the NF = 256 FREQUENT features is a [128 queries x 256] x [256 x 64 chunks] fp16 GEMM (weights
//     rounded UP to fp16, tf exact): one MMA warpgroup issues wgmma.mma_async m64n64k16 (two per K step, one per
//     64-query half), fp32 accumulators in its registers, the query operand resident in shared memory for the CTA's
//     life, the chunk operand streamed by TMA (128B swizzle, mbarrier expect_tx; one thread of the warpgroup refills a
//     stage as soon as the warpgroup's MMAs have read it); the warpgroup adds its accumulators
//     into R (below) while the workers run the rare join of the same block, so the GEMM of block b + 1 overlaps the
//     epilogue of block b -- this only computes BOUNDS; scores stay exact integer sums (K1b-S);
//   * the next NF2 = 1024 features by chunk frequency ("second class": mid-frequency words and bigrams, each shared by
//     many queries of a tile) are kept per 64-chunk block as two TRANSPOSED presence bitmaps Ubt[feature][tf >= 1,
//     tf >= 2][64 chunk bits].  A tile's queries list <= Q2CAP of them each; the KT2 = 256 most listed form the tile's
//     dictionary (f2_dict_kernel) and are 256 more K of the same GEMM, into the same accumulators: A2 = the fp16
//     weights (resident, TMA), B2 = 0 / 1 / T (T = largest tf rounded up to fp16) by the block's two bitmap rows of
//     each column, built in shared memory by the MMA warpgroup after it has added the previous block into R.  A tile
//     listing more than KT2 distinct ones leaves the least listed in the queries' lists: the epilogue adds those from
//     the block's bitmap words in global memory (warps without such a feature skip that loop);
//   * the remaining RARE features are joined the other way round: every 64-chunk block carries (built at finalize) a
//     presence bitmap and a two-choice table of its rare features (feature -> mask of the block's chunks holding it,
//     largest tf, in one of two 16-byte slots); each query looks ITS OWN <= 32 rare features up -- one shared-memory bit
//     test per (query, feature, block), and only on a hit a lookup of the block's table in L2, the warp's hits spread
//     over its lanes -- and adds weight x tf into R[chunk][query] (shared memory).  1.8k bit tests per tile and block
//     instead of 5.4k entry probes;
//   * R is fixed point, uint32 in units of 1 / s_q per query (s_q: a power of two chosen by prep_queries_kernel so that
//     R cannot wrap), every term rounded up into it: the MMA warpgroup's and the rare join's adds are native integer
//     shared atomics (a float shared atomicAdd is a compare-and-swap loop on sm_90a);
//   * epilogue (16 warps, four threads per query, 16 chunk columns of R each): bound vs the query's threshold.
//     pass 0 keeps, per thread, the 4 best chunks by bound (16 seeds per query: K1b-S scores them first, which gives
//     every query a close lower bound theta0 of its k-th best score) and stores every bound as an 8-bit code rounded up
//     (the candidate scan selects its candidates from the codes, against threshold_codes_kernel's snapshot); pass 1 (only when the codes do not fit in
//     memory) recomputes the bounds and appends {chunk, mask of the group's surviving queries} to the scan group's
//     candidate list (paged pool) for every chunk with ub >= theta0.
// One CTA = one 128-query tile x one range of 64-chunk blocks; 20 warps: 16 workers (join + epilogue) and the MMA +
// TMA warpgroup (warps 16-19).
#pragma once
#include "tfidf_kernels.cuh"

namespace kvk {

constexpr int B_BN = 64;                     // chunks per block = N of the MMA tile
constexpr int B_BK = 64;                     // K slice: 64 fp16 = one 128-byte swizzle row
constexpr int B_KSLICES = NF / B_BK;         // 4
constexpr int B_KSLICES2 = KT2 / B_BK;       // 4: the second-class dictionary, one slice per warp of the MMA warpgroup
static_assert(KT2 == 2 * 128, "each thread of the MMA warpgroup builds two columns of the dictionary's B operand");
constexpr int B_STAGES = 2;
constexpr int B_A_SLICE_BYTES = TILE_Q * B_BK * 2;  // 16 KiB: one K slice of the query operand
constexpr int B_B_SLICE_BYTES = B_BN * B_BK * 2;    // 8 KiB: one K slice of the chunk operand
constexpr int B_WORKERS = 16;
constexpr int B_MMA_WARP = B_WORKERS;        // first warp of the MMA warpgroup (a warpgroup starts at a multiple of 4)
constexpr int B_THREADS = (B_WORKERS + 4) * 32;
// named barriers (0 is __syncthreads): R complete for the epilogue (workers wait, the MMA warpgroup arrives), R clean
// again for the next block's accumulators (the MMA warpgroup waits, the workers arrive), the workers among themselves,
// the MMA warpgroup among itself (a chunk slice has been read by all four warps and may be refilled)
constexpr int B_BAR_RFULL = 1, B_BAR_RCLEAN = 2, B_BAR_WORKERS = 3, B_BAR_MMA = 4;
constexpr int B_COLS = B_BN / 4;             // chunk columns per epilogue thread (four threads serve a query)
// Words per chunk row of R: the tile's queries and four of padding.  The MMA warpgroup's lanes add to chunks
// 2 (lane % 4) + const and queries lane / 4 + const: with 128-word rows those are 8 banks, four lanes each at different
// addresses; with 132-word rows the bank is 8 (lane % 4) + lane / 4 + const, 32 different ones.  The read-out (a warp =
// 32 consecutive queries of one chunk row) is conflict-free with either.
constexpr int B_RSTRIDE = TILE_Q + 4;
constexpr int B_SEEDS = 4;                   // seeds per worker thread
constexpr int B_SEEDS_PER_QUERY = 4 * B_SEEDS;
constexpr float UBQ_SCALE = 250.f;           // 8-bit bound code = ceil(bound * 250), saturating at 255 (bounds reach ~1.001)

// Measuring build of K1b-B (-DKV_BOUND_CLOCKS, profiles/run_bound_split.py): every warp splits each 64-chunk block of
// its loop into clock() spans and counts what the rare join meets, every CTA notes its start and end on the global
// timer, and all of it is added to g_bound_prof, which kv_debug_bound_profile reads.  The product build defines none
// of this: KV_BOUND_PROF(...) and KV_BOUND_MARK(...) expand to nothing.
#ifdef KV_BOUND_CLOCKS
constexpr int KB_MAX_CTAS = 4096;  // CTAs whose start and end are kept (the bench shape launches 782)
enum {
  // cycles, per worker warp
  KBW_BITMAP, KBW_JOIN_BITS, KBW_JOIN_COMPACT, KBW_JOIN_SLOTS, KBW_FANOUT, KBW_RFULL, KBW_READOUT, KBW_F2LEFT, KBW_BOUND,
  KBW_STORE, KBW_BARRIER, KBW_N,
  // cycles, per warp of the MMA warpgroup
  KBM_GEMM = KBW_N, KBM_RCLEAN, KBM_ADDS, KBM_B2, KB_NSPANS,
  // counters: the join's bitmap hits (= lookups), lookup rounds of a warp, (warp, block)s needing a second round, table
  // hits, hit-mask bits and fan-out iterations (largest lane per round); per block the slowest worker warp's join, and
  // which side reached RFULL last
  KBC_BIT_HITS = KB_NSPANS, KBC_ROUNDS, KBC_MULTI_ROUND, KBC_TABLE_HITS, KBC_MASK_BITS, KBC_FAN_ITERS, KBC_JOIN_SLOWEST,
  KBC_MMA_LAST, KBC_MMA_LAST_CYC, KBC_WORKERS_LAST_CYC, KBC_WORKER_WARP_BLOCKS, KBC_MMA_WARP_BLOCKS,
  KBC_CTA_BLOCKS, KBC_CTAS, KB_NSLOTS,
  KBT_START = KB_NSLOTS,               // [KB_MAX_CTAS] globaltimer ns, by blockIdx.y * gridDim.x + blockIdx.x
  KBT_END = KBT_START + KB_MAX_CTAS,   // [KB_MAX_CTAS]
  KB_TOTAL = KBT_END + KB_MAX_CTAS
};
__device__ unsigned long long g_bound_prof[KB_TOTAL];
__device__ __forceinline__ unsigned long long kb_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define KV_BOUND_PROF(...) __VA_ARGS__
// charges the cycles since the previous mark to a span (the warp is converged first, lane 0's clock is the warp's)
#define KV_BOUND_MARK(slot) { __syncwarp(); const unsigned int kbp_n = clock(); kbp[slot] += kbp_n - kbp_t; kbp_t = kbp_n; }
#else
#define KV_BOUND_PROF(...)
#define KV_BOUND_MARK(slot)
#endif

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, fp16 in, fp32 accumulators in registers (both operands K-major)
__device__ __forceinline__ void wgmma_m64n64k16_f16(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d)
      : "memory");
}

// wait of a single-lane role (TMA producer, MMA issuer): polls with a pause, so that the spinning lane does not
// take issue slots from the worker warps sharing its scheduler
__device__ __forceinline__ void mbar_wait_idle(uint64_t *bar, uint32_t parity) {
  uint32_t done;
  for (;;) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_addr(bar)), "r"(parity)
        : "memory");
    if (done) break;
    __nanosleep(64);
  }
}

// MUFU.RSQ without the denormal pre-/post-scaling rsqrtf() carries (the argument is |q|^2 x a row norm: far from denormal;
// for normal arguments the result is the same bit pattern)
__device__ __forceinline__ float rsqrt_approx(float x) {
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ceil(v) clamped to 0 .. 255 as an integer, v any float (NaN: 255): the same value as (uint32_t)fminf(255.f, ceilf(v))
// without the FRND and F2I of the conversion pipe.  At 2^23 one ulp of a float is 1, so adding 2^23 to a v in [0, 255]
// rounding up leaves ceil(v) in the low mantissa bits.
__device__ __forceinline__ uint32_t ceil_to_byte(float v) {
  return __float_as_uint(__fadd_ru(fmaxf(fminf(v, 255.f), 0.f), 8388608.f)) & 0xFFu;
}

// The candidate lists of a batch: list l = group * n_bsplits + bsplit holds records {chunk, mask of the group's queries}
// in pages of PAGE_RECS records taken from one pool.
struct CandLists {
  uint32_t *count;          // [n_lists]
  uint32_t *pages;          // [n_lists][max_pages]
  int max_pages;
  uint2 *pool;
  unsigned int *pool_next;  // pages handed out
  unsigned int pool_pages;  // capacity
  int *overflow;            // set when the pool ran out (the batch is rerun with a larger pool)
};

// Appends the {chunk, mask} of every lane with a non-empty mask to list `list`, warp-aggregated: lane 0 takes the
// warp's positions from the list's shared counter and allocates the pages its range crosses into, publishing each in the
// list's shared page table (warps sharing a list wait there for a page another warp is allocating).  All 32 lanes call.
__device__ __forceinline__ void list_append(const CandLists &L, int list, unsigned int *count, int *pages, uint32_t chunk,
                                            uint32_t mask, unsigned int &n_pairs, unsigned int &n_recs) {
  const uint32_t am = __ballot_sync(FULL, mask != 0);
  if (!am) return;
  const int n = __popc(am);
  unsigned int bpos = 0;
  if ((threadIdx.x & 31) == 0) {
    bpos = atomicAdd(count, (unsigned int)n);
    for (unsigned int pg = (bpos + PAGE_RECS - 1) / PAGE_RECS; pg * PAGE_RECS < bpos + n; pg++) {
      unsigned int np = atomicAdd(L.pool_next, 1u);
      if (np >= L.pool_pages) { *L.overflow = 1; np = 0; }
      L.pages[(size_t)list * L.max_pages + pg] = np;
      __threadfence_block();
      *(volatile int *)&pages[pg] = (int)np;
    }
  }
  bpos = __shfl_sync(FULL, bpos, 0);
  if (mask) {
    const unsigned int pos = bpos + (unsigned int)__popc(am & lanemask_lt());
    const unsigned int pg = pos / PAGE_RECS;
    int page;
    while ((page = *(volatile int *)&pages[pg]) < 0) {}
    uint2 rec;
    rec.x = chunk;
    rec.y = mask;
    L.pool[(size_t)page * PAGE_RECS + (pos % PAGE_RECS)] = rec;
    n_pairs += (unsigned int)__popc(mask);
    n_recs++;
  }
}

// adds a warp's appended pairs and records to stats[2] / stats[3]
__device__ __forceinline__ void flush_list_stats(unsigned long long *stats, unsigned int n_pairs, unsigned int n_recs) {
  if (!stats) return;
  for (int o = 16; o; o >>= 1) {
    n_pairs += __shfl_xor_sync(FULL, n_pairs, o);
    n_recs += __shfl_xor_sync(FULL, n_recs, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&stats[2], (unsigned long long)n_pairs);
    atomicAdd(&stats[3], (unsigned long long)n_recs);
  }
}

struct BoundParams {
  const uint32_t *blk;
  const BlockInfo *binfo;
  const float *chunk_minB;  // [n_chunks_pad]
  const unsigned long long *ovf_keys;
  const uint32_t *ovf_vals;
  int n_ovf;
  int64_t n_chunks, n_q;
  const uint32_t *q3id, *q3w;                             // [n_tiles][Q3CAP][TILE_Q] rare lists: feature, fixed-point weight
  const uint32_t *rbloom;                                 // [n_blocks][RB_BITS / 32]
  const uint4 *rt_slots;                                  // per-block two-choice rare tables (slot layout: rt_slot2)
  const uint32_t *rt_off, *rt_size;                       // [n_blocks]
  const uint32_t *d2col;                                  // [n_tiles][KT2] second-class dictionary (f2_dict_kernel)
  const uint2 *q2list;                                    // [n_tiles][Q2CAP][TILE_Q] second-class features left out of it
  const uint32_t *ubt;                                    // [n_blocks][NF2][2][B_BN / 32]
  const float *q_nq, *q_dotS, *q_dotX, *q_corrS;          // [n_q] (sorted query order)
  const float *q_rscale;                                  // [n_q] 1 / s_q, a power of two: the unit of R's fixed point
  const int *gthr;                                        // [n_q] float bits: lower bound of the k-th score
  int pass;                                               // 0: seeds, 1: candidate lists
  int n_bsplits;
  int *seeds;                                             // pass 0: [n_q][n_bsplits][B_SEEDS_PER_QUERY] chunk ids, -1 = none
  CandLists lists;                                        // pass 1 (max_pages also sizes the shared page tables)
  unsigned long long *stats;  // [2] surviving (query, chunk) pairs, [3] candidate records
  unsigned char *ubq;         // pass 0, optional: every bound as an 8-bit code (rounded up), [n_q][ubq_stride]
  int64_t ubq_stride;
  float *dbg_xs;              // test hook: when set, the numerator of every bound, [n_q][n_chunks_pad]
  int64_t dbg_stride;
};

struct __align__(1024) BoundSmem {
  unsigned char a[B_KSLICES][B_A_SLICE_BYTES];   // the tile's weight rows, resident
  unsigned char a2[B_KSLICES2][B_A_SLICE_BYTES]; // the tile's weights of its second-class dictionary, resident
  unsigned char b[B_STAGES][B_B_SLICE_BYTES];    // chunk slices in flight
  unsigned char b2[B_KSLICES2][B_B_SLICE_BYTES]; // the block's dictionary columns (0 / 1 / T), built by the MMA warpgroup
  uint32_t rbm[RB_BITS / 32];                    // rare-feature presence bitmap of the block
  uint32_t R[B_BN][B_RSTRIDE];                   // the dot bound without the query constants, units of 1 / s_q, [chunk][query]
  float minB[2][B_BN];
  uint64_t full_bar[B_STAGES], a_bar, blk_bar;
  unsigned int lcount[4];
  // of the block in hand, clocks relative to prof_t0: the longest join of a worker warp, the last worker warp's and
  // the MMA warpgroup's arrival at RFULL
  KV_BOUND_PROF(unsigned int prof_t0, prof_join_max, prof_w_arrive, prof_m_arrive;)
  int pages[1];  // [4][max_pages], sized at launch
};

static inline size_t bound_smem_bytes(int max_pages) { return sizeof(BoundSmem) + (size_t)4 * max_pages * sizeof(int) + 1024; }

// FAST = the configuration of the headline path fixed at compile time (pass 0 with bound codes, no test hook): the
// epilogue then holds no uniform branches, parameter reloads or dead variants.  FAST = false is the same code with
// those three switches read from the parameters.
template <bool FAST>
__global__ void __launch_bounds__(B_THREADS, 1)
tfidf_bound_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_w2,
                   const __grid_constant__ CUtensorMap map_u, BoundParams P) {
  extern __shared__ unsigned char smem_raw[];
  const int pass = FAST ? 0 : P.pass;
  const bool has_codes = FAST ? true : (P.ubq != nullptr);
  BoundSmem &S = *reinterpret_cast<BoundSmem *>(smem_raw + smem_align1024(smem_raw));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x, bsplit = blockIdx.y;
  const int64_t n_blocks = (P.n_chunks + B_BN - 1) / B_BN;
  const int64_t blk_lo = n_blocks * bsplit / P.n_bsplits, blk_hi = n_blocks * (bsplit + 1) / P.n_bsplits;

  if (threadIdx.x == 0) {
    for (int i = 0; i < B_STAGES; i++) mbar_init(&S.full_bar[i], 1);
    mbar_init(&S.a_bar, 1);
    mbar_init(&S.blk_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    KV_BOUND_PROF(S.prof_t0 = clock(); S.prof_join_max = S.prof_w_arrive = S.prof_m_arrive = 0;
                  const unsigned int cta = blockIdx.y * gridDim.x + blockIdx.x;
                  if (cta < KB_MAX_CTAS) g_bound_prof[KBT_START + cta] = kb_globaltimer();)
  }
  {  // R = 0, list state
    uint4 *r4 = (uint4 *)&S.R[0][0];
    for (int i = threadIdx.x; i < B_BN * B_RSTRIDE / 4; i += B_THREADS) r4[i] = make_uint4(0u, 0u, 0u, 0u);
    for (int i = threadIdx.x; i < 4 * P.lists.max_pages; i += B_THREADS) S.pages[i] = -1;
    if (threadIdx.x < 4) S.lcount[threadIdx.x] = 0;
  }
  __syncthreads();

  if (warp >= B_MMA_WARP) {
    // ===== MMA warpgroup: frequent and second-class part of the block's bounds, added into R =====
    // accumulator fragment of m64nNk16: warp w of the warpgroup holds rows 16 w + lane / 4 (+ 8) of each 64-query
    // half, register 4 j + e holds column 8 j + 2 (lane % 4) + (e & 1) of row + 8 (e >> 1)
    const int wq = warp - B_MMA_WARP;
    const bool producer = wq == 0 && lane == 0;
    // 32-bit block and slice counters (fewer registers next to the 64 accumulators): the TMA coordinates are 32-bit
    const int b0 = (int)blk_lo, n_blk = (int)(blk_hi - blk_lo);
    // chunk slices in global order g = (block - blk_lo) * B_KSLICES + slice; slice g goes to stage g % B_STAGES
    const int n_slices = n_blk * B_KSLICES;
    auto load_slice = [&](int g) {
      const int st = g % B_STAGES;
      mbar_expect_tx(&S.full_bar[st], B_B_SLICE_BYTES);
      tma_load_2d(S.b[st], &map_u, &S.full_bar[st], (g % B_KSLICES) * B_BK, (b0 + g / B_KSLICES) * B_BN);
    };
    if (producer) {
      mbar_expect_tx(&S.a_bar, (B_KSLICES + B_KSLICES2) * B_A_SLICE_BYTES);
      for (int s = 0; s < B_KSLICES; s++) tma_load_2d(S.a[s], &map_w, &S.a_bar, s * B_BK, tile * TILE_Q);
      for (int s = 0; s < B_KSLICES2; s++) tma_load_2d(S.a2[s], &map_w2, &S.a_bar, s * B_BK, tile * TILE_Q);
      for (int g = 0; g < B_STAGES && g < n_slices; g++) load_slice(g);
    }
    // Second-class dictionary: thread t of the warpgroup owns columns 2 t, 2 t + 1 (warp wq: K slice wq).  Their
    // 16-byte bitmap rows (tf >= 1, tf >= 2 over the block's 64 chunks) are loaded one block ahead into registers.
    const uint32_t dc0 = P.d2col[(size_t)tile * KT2 + 2 * (wq * 32 + lane)];
    const uint32_t dc1 = P.d2col[(size_t)tile * KT2 + 2 * (wq * 32 + lane) + 1];
    uint4 u0 = make_uint4(0u, 0u, 0u, 0u), u1 = u0;
    auto fetch_rows = [&](int i) {  // block blk_lo + i
      const uint4 *src = reinterpret_cast<const uint4 *>(P.ubt) + (size_t)(b0 + i) * NF2;
      if (dc0) u0 = __ldg(src + (dc0 & 0xFFFFu));  // dc == 0: unused column, stays 0
      if (dc1) u1 = __ldg(src + (dc1 & 0xFFFFu));
    };
    // B2 (K-major like the chunk slices: chunk n's 128-byte row, 16-byte units swizzled by n % 8) = 0, 1 (fp16 0x3C00)
    // or T: one 4-byte store per chunk, a warp's 32 stores fill one row (no bank conflicts)
    auto build_b2 = [&]() {
      unsigned char *dst = S.b2[wq] + (lane & 3) * 4;
#pragma unroll
      for (int n = 0; n < B_BN; n++) {
        const uint32_t w1a = n < 32 ? u0.x : u0.y, w2a = n < 32 ? u0.z : u0.w;
        const uint32_t w1b = n < 32 ? u1.x : u1.y, w2b = n < 32 ? u1.z : u1.w;
        const uint32_t lo = (w2a >> (n & 31)) & 1u ? dc0 >> 16 : ((w1a >> (n & 31)) & 1u ? 0x3C00u : 0u);
        const uint32_t hi = (w2b >> (n & 31)) & 1u ? dc1 >> 16 : ((w1b >> (n & 31)) & 1u ? 0x3C00u : 0u);
        *reinterpret_cast<uint32_t *>(dst + n * 128 + ((((uint32_t)lane >> 2) ^ (uint32_t)(n & 7)) << 4)) = lo | hi << 16;
      }
    };
    // generic-proxy stores of B2 -> visible to the wgmmas (async proxy) of every warp of the warpgroup
    auto publish_b2 = [&]() {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("bar.sync %0, 128;" ::"n"(B_BAR_MMA) : "memory");
    };
    if (n_blk > 0) {
      fetch_rows(0);
      build_b2();
      if (n_blk > 1) fetch_rows(1);
      publish_b2();
    }
    // refill the stage of slice g (read by every warp of the warpgroup: wgmma_wait done) with slice g + B_STAGES
    auto release = [&](int g) {
      asm volatile("bar.sync %0, 128;" ::"n"(B_BAR_MMA) : "memory");
      if (producer && g + B_STAGES < n_slices) load_slice(g + B_STAGES);
    };
    float acc[2][32] = {};
    // s_q of the four query rows this thread holds (1 / a power of two: exact); padding rows have zero weights
    float sq[2][2];
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int r = 0; r < 2; r++) {
        const int64_t sl = (int64_t)tile * TILE_Q + h * 64 + wq * 16 + (lane >> 2) + 8 * r;
        sq[h][r] = sl < P.n_q ? __frcp_rn(P.q_rscale[sl]) : 1.f;
      }
    mbar_wait_idle(&S.a_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    int g = 0;
    KV_BOUND_PROF(unsigned int kbp[KB_NSPANS] = {}; unsigned int kbp_t = clock(); const unsigned int kb_t0 = S.prof_t0;)
    for (int it = 0; it < n_blk; it++) {
#pragma unroll
      for (int h = 0; h < 2; h++)
#pragma unroll
        for (int i = 0; i < 32; i++) wgmma_reg_fence(acc[h][i]);
      wgmma_fence();
      // the second-class dictionary first: its operands are resident, so these issue while the chunk slices land
#pragma unroll
      for (int s = 0; s < B_KSLICES2; s++) {
        const uint64_t db = wgmma_desc_sw128(S.b2[s]);
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const uint64_t da = wgmma_desc_sw128(S.a2[s] + h * (B_A_SLICE_BYTES / 2));
#pragma unroll
          for (int kk = 0; kk < B_BK / 16; kk++)
            wgmma_m64n64k16_f16(acc[h], da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), (uint32_t)((s | kk) != 0));
        }
      }
      for (int s = 0; s < B_KSLICES; s++, g++) {
        mbar_wait_idle(&S.full_bar[stage], phase);
        const uint64_t db = wgmma_desc_sw128(S.b[stage]);
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const uint64_t da = wgmma_desc_sw128(S.a[s] + h * (B_A_SLICE_BYTES / 2));  // rows 64 h .. 64 h + 63
#pragma unroll
          for (int kk = 0; kk < B_BK / 16; kk++)  // advance 32 bytes (2 x 16-byte units) per K=16 step inside the swizzle row
            wgmma_m64n64k16_f16(acc[h], da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), 1u);
        }
        wgmma_commit();
        if (s > 0) {  // the previous slice's group is done: its stage may be refilled
          wgmma_wait<1>();
          release(g - 1);
        }
        if (++stage == B_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < 2; h++)
#pragma unroll
        for (int i = 0; i < 32; i++) wgmma_reg_fence(acc[h][i]);
      release(g - 1);
      KV_BOUND_MARK(KBM_GEMM)
      // R holds the previous block's values until the workers' epilogue has read and cleared them
      if (it > 0) asm volatile("bar.sync %0, %1;" ::"n"(B_BAR_RCLEAN), "n"(B_THREADS) : "memory");
      KV_BOUND_MARK(KBM_RCLEAN)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int q0 = h * 64 + wq * 16 + (lane >> 2);
#pragma unroll
        for (int i = 0; i < 32; i++) {
          const int c = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
          // rounded up into R's fixed point; the workers' rare join adds to R concurrently
          atomicAdd(&S.R[c][q0 + 8 * ((i >> 1) & 1)], __float2uint_ru(acc[h][i] * sq[h][(i >> 1) & 1]));
        }
      }
      KV_BOUND_PROF(if (wq == 0 && lane == 0) S.prof_m_arrive = clock() - kb_t0;)
      asm volatile("bar.arrive %0, %1;" ::"n"(B_BAR_RFULL), "n"(B_THREADS) : "memory");
      KV_BOUND_MARK(KBM_ADDS)
      // the GEMM of this block is done (wgmma_wait above): B2 takes the next block's columns
      if (it + 1 < n_blk) {
        build_b2();
        if (it + 2 < n_blk) fetch_rows(it + 2);
        publish_b2();
      }
      KV_BOUND_MARK(KBM_B2)
    }
    KV_BOUND_PROF(if (lane == 0) {
      _Pragma("unroll")
      for (int i = KBM_GEMM; i < KB_NSPANS; i++) atomicAdd(&g_bound_prof[i], (unsigned long long)kbp[i]);
      atomicAdd(&g_bound_prof[KBC_MMA_WARP_BLOCKS], (unsigned long long)n_blk);
    })
    if (n_blk > 0) asm volatile("bar.sync %0, %1;" ::"n"(B_BAR_RCLEAN), "n"(B_THREADS) : "memory");  // the last block's
  } else {
    // ===== workers: join, then epilogue, per block =====
    const int qtr = warp & 3;   // quarter of the tile's queries = scan group of the tile
    const int cs = warp >> 2;   // which B_COLS chunk columns of a block this warp's epilogue covers
    const int qi = qtr * 32 + lane;
    const int64_t slot = (int64_t)tile * TILE_Q + qi;
    const bool q_in = slot < P.n_q;
    const float nq = q_in ? P.q_nq[slot] : 0.f;
    const bool q_ok = nq > 0.f;
    const float base = q_ok ? P.q_dotS[slot] + P.q_dotX[slot] : 0.f;
    const float corrS = q_ok ? P.q_corrS[slot] : 0.f;
    const float rs = q_in ? P.q_rscale[slot] : 0.f;  // a power of two: R x rs is exact
    const int list = (tile * 4 + qtr) * P.n_bsplits + bsplit;
    int *my_pages = S.pages + qtr * P.lists.max_pages;
    float sm[B_SEEDS];
    int sc[B_SEEDS];
#pragma unroll
    for (int i = 0; i < B_SEEDS; i++) { sm[i] = -1.f; sc[i] = -1; }
    unsigned int n_pairs = 0, n_recs = 0;
    // the rare join's thread = (query jq, quarter `part` of its rare list): the list's feature ids stay in registers
    constexpr int NR = Q3CAP / 4;  // list entries of a thread
    const int jq = threadIdx.x & (TILE_Q - 1), part = threadIdx.x >> 7;  // 512 worker threads = 128 queries x 4
    const size_t q3o = (size_t)tile * Q3CAP * TILE_Q + (size_t)part * TILE_Q + jq;  // entry part + 4 k: + 4 k TILE_Q
    uint32_t fid[NR];
#pragma unroll
    for (int k = 0; k < NR; k++) fid[k] = P.q3id[q3o + (size_t)k * 4 * TILE_Q];  // FID_NONE past the end of the list
    // rare presence bitmap of the block: one bulk-async copy, issued for block b + 1 as soon as the join of block b has
    // read the buffer (after the RFULL barrier); it lands while block b's epilogue runs
    auto fetch_bitmap = [&](int64_t bk2) {
      mbar_expect_tx(&S.blk_bar, (uint32_t)sizeof(S.rbm));
      bulk_copy_g2s(&S.rbm[0], P.rbloom + (size_t)bk2 * (RB_BITS / 32), sizeof(S.rbm), &S.blk_bar);
    };
    if (threadIdx.x == 0 && blk_lo < blk_hi) fetch_bitmap(blk_lo);
    // second-class features of the warp's queries left out of the tile's dictionary (only tiles listing more than KT2
    // distinct ones): added per block from the bitmaps in global memory; most warps have none and skip the loop
    const uint2 *ql2 = P.q2list + (size_t)tile * Q2CAP * TILE_Q + qi;
    const bool warp_left = __any_sync(FULL, q_ok && __uint_as_float(ql2[0].y) > 0.f);
    // size and offset of the block's rare table, loaded one block ahead: the first-slot key loads need them at once,
    // and loaded in the join they were a third dependent L2 round trip of every block
    uint32_t tsize_n = 0, toff_n = 0;
    if (blk_lo < blk_hi) { tsize_n = P.rt_size[blk_lo]; toff_n = P.rt_off[blk_lo]; }
    int64_t it = 0;
    KV_BOUND_PROF(unsigned int kbp[KB_NSPANS] = {}; unsigned int kbp_t = clock(); const unsigned int kb_t0 = S.prof_t0;
                  unsigned int kbc_bit = 0, kbc_rounds = 0, kbc_multi = 0, kbc_tab = 0, kbc_bits = 0, kbc_fan = 0;
                  unsigned long long kbc_slowest = 0, kbc_mma_last = 0, kbc_mma_cyc = 0, kbc_w_cyc = 0;)
    for (int64_t bk = blk_lo; bk < blk_hi; bk++, it++) {
      const int as = (int)(it & 1);
      const int64_t c0 = bk * B_BN;
      mbar_wait(&S.blk_bar, (uint32_t)(it & 1));
      KV_BOUND_MARK(KBW_BITMAP)
      KV_BOUND_PROF(const unsigned int kb_join0 = kbp_t;)
      // ---- rare join, inverted: thread (query, quarter of its rare list) tests each feature in the block's presence
      //      bitmap; the warp's hits are then spread over its lanes, 32 per round, and each lane looks its hit up in the
      //      block's two-choice table (both slots and the weight loaded together: one L2 round trip, hit or miss) and
      //      adds weight x tf to R[chunk][query] for every chunk of the mask.  Rows are text-sorted, so one feature can
      //      sit in most chunks of a block: R is dense. ----
      {
        const uint32_t *bm = S.rbm;
        const uint32_t tsize = tsize_n, toff = toff_n;
        if (bk + 1 < blk_hi) { tsize_n = P.rt_size[bk + 1]; toff_n = P.rt_off[bk + 1]; }
        // the warp's hits, numbered entry-major: the hit of entry k at lane l is number pre_k + popc(ball[k] below l)
        uint32_t ball[NR], n_hits = 0;
#pragma unroll
        for (int k = 0; k < NR; k++) {
          const uint32_t bb = rb_bit(fid[k]);
          ball[k] = __ballot_sync(FULL, fid[k] < FID_NONE && ((bm[bb >> 5] >> (bb & 31u)) & 1u));
          n_hits += __popc(ball[k]);
        }
        KV_BOUND_MARK(KBW_JOIN_BITS)
        KV_BOUND_PROF(kbc_bit += n_hits; kbc_rounds += (n_hits + 31) / 32; kbc_multi += n_hits > 32;)
        const uint4 *tab = P.rt_slots + toff;
        for (uint32_t g = (uint32_t)lane; g - (uint32_t)lane < n_hits; g += 32) {  // round: hit g goes to lane g % 32
          // entry k and source lane of hit g: the last k with pre_k <= g, then the (g - pre_k)-th set bit of ball[k]
          uint32_t kk = 0, bk_bits = 0, rank = 0, pre = 0;
#pragma unroll
          for (int k = 0; k < NR; k++) {
            if (g >= pre) { kk = (uint32_t)k; bk_bits = ball[k]; rank = g - pre; }
            pre += __popc(ball[k]);
          }
          const bool has = g < n_hits;
          uint32_t src = 0;  // binary search for the set bit with `rank` set bits below it (lane 0 for a lane without a hit)
#pragma unroll
          for (uint32_t s = 16; s; s >>= 1) {
            const uint32_t c = (uint32_t)__popc((bk_bits >> src) & ((1u << s) - 1u));
            if (rank >= c) { rank -= c; src += s; }
          }
          if (!has) src = 0;
          uint32_t f = FID_NONE;
#pragma unroll
          for (int k = 0; k < NR; k++)
            if (ball[k]) {
              const uint32_t v = __shfl_sync(FULL, fid[k], src);
              if (kk == (uint32_t)k) f = v;
            }
          const uint32_t jsrc = (uint32_t)(jq & (TILE_Q - 32)) | src;  // the source lane's query
          KV_BOUND_MARK(KBW_JOIN_COMPACT)
          uint4 s1 = make_uint4(KEY_EMPTY, 0u, 0u, 0u), s2 = s1;
          uint32_t w = 0;
          if (has) {
            s1 = __ldg(tab + rt_slot1(f, tsize));
            s2 = __ldg(tab + rt_slot2(f, tsize));
            w = __ldg(P.q3w + (q3o - (size_t)jq + jsrc) + (size_t)kk * 4 * TILE_Q);
          }
          const uint4 s = s1.x == f ? s1 : s2;
          unsigned long long m = has && s.x == f ? ((unsigned long long)s.w << 32 | s.z) : 0ull;
          const uint32_t x = w * s.y;  // fixed point, <= 2^30 + tf (prep_queries_kernel)
          KV_BOUND_MARK(KBW_JOIN_SLOTS)
          KV_BOUND_PROF({
            const unsigned int nb = (unsigned int)__popcll(m);
            kbc_tab += m != 0; kbc_bits += nb; kbc_fan += __reduce_max_sync(FULL, nb);
          })
          for (; m; m &= m - 1) atomicAdd(&S.R[__ffsll((long long)m) - 1][jsrc], x);
          KV_BOUND_MARK(KBW_FANOUT)
        }
        KV_BOUND_PROF(if (lane == 0) atomicMax(&S.prof_join_max, kbp_t - kb_join0);)
      }
      if (threadIdx.x < B_BN) S.minB[as][threadIdx.x] = P.chunk_minB[c0 + threadIdx.x];
      // this block's threshold of the query (pass 1: theta0 from the seed scan, possibly raised by peers meanwhile)
      float tq = 0.f;
      if (pass == 1 && q_ok) {
        const float th = __int_as_float(__ldcg(&P.gthr[slot]));
        if (th > 0.f) tq = th * th * nq / (PRUNE_SLACK * PRUNE_SLACK);
      }
      // R complete: the workers' rare join and the MMA warpgroup's frequent + second-class part of this block
      KV_BOUND_PROF(if (lane == 0) atomicMax(&S.prof_w_arrive, clock() - kb_t0);)
      asm volatile("bar.sync %0, %1;" ::"n"(B_BAR_RFULL), "n"(B_THREADS) : "memory");
      if (threadIdx.x == 0 && bk + 1 < blk_hi) fetch_bitmap(bk + 1);  // every join has read this block's bitmap
      KV_BOUND_MARK(KBW_RFULL)
      KV_BOUND_PROF(if (threadIdx.x == 0) {  // the next block's values are written after this thread's RCLEAN / WORKERS arrival
        const unsigned int ta = S.prof_w_arrive, tm = S.prof_m_arrive;
        if ((int)(tm - ta) > 0) { kbc_mma_last++; kbc_mma_cyc += tm - ta; } else { kbc_w_cyc += ta - tm; }
        kbc_slowest += S.prof_join_max;
        S.prof_join_max = S.prof_w_arrive = 0;
      })
      // ---- epilogue, thread = query, B_COLS chunk columns: R + second-class features outside the dictionary -> bound
      //      -> seed / candidate ----
      float x[B_COLS];
      {
        uint32_t *Rcol = &S.R[cs * B_COLS][qi];
#pragma unroll
        for (int j = 0; j < B_COLS; j++) { x[j] = __uint2float_ru(Rcol[j * B_RSTRIDE]) * rs; Rcol[j * B_RSTRIDE] = 0u; }
      }
      KV_BOUND_MARK(KBW_READOUT)
      if (warp_left) {
        const uint32_t bsh = (uint32_t)((cs * B_COLS) & 31), bword = (uint32_t)((cs * B_COLS) >> 5);
        constexpr uint32_t CMASK = B_COLS == 32 ? 0xFFFFFFFFu : ((1u << B_COLS) - 1u);
        const uint32_t *ub = P.ubt + (size_t)bk * NF2 * 4 + bword;  // [feature][tf >= 1, tf >= 2][2 words]
#pragma unroll 1
        for (int i = 0; i < Q2CAP; i++) {
          const uint2 f2 = __ldg(ql2 + (size_t)i * TILE_Q);
          const float w2 = q_ok ? __uint_as_float(f2.y) : 0.f;
          if (!__any_sync(FULL, w2 > 0.f)) break;  // the lists are filled from the front
          const uint32_t row2 = f2.x & 0xFFFFu, tm1 = f2.x >> 16;
          const uint32_t m = w2 > 0.f ? ((__ldg(ub + row2 * 4) >> bsh) & CMASK) : 0u;
          if (m) {
#pragma unroll
            for (int j = 0; j < B_COLS; j++)
              if ((m >> j) & 1u) x[j] += w2;
            const uint32_t mm = tm1 ? ((__ldg(ub + row2 * 4 + 2) >> bsh) & CMASK) : 0u;  // tf >= 2: up to tfmax - 1 more
            if (mm) {
              const float wex = __fmul_ru(w2, (float)tm1);
#pragma unroll
              for (int j = 0; j < B_COLS; j++)
                if ((mm >> j) & 1u) x[j] += wex;
            }
          }
        }
      }
      KV_BOUND_MARK(KBW_F2LEFT)
      const float *mb = &S.minB[as][cs * B_COLS];
      const int64_t cbase = c0 + cs * B_COLS;
      uint32_t mymask = 0;
      const bool dbg = FAST ? false : (P.dbg_xs != nullptr);
      const int nv = (int)min((int64_t)B_COLS, P.n_chunks - cbase);  // chunk columns of this thread that exist
      uint32_t codes[B_COLS / 4];
#pragma unroll
      for (int j = 0; j < B_COLS / 4; j++) codes[j] = 0;
#pragma unroll
      for (int j = 0; j < B_COLS; j++) {
        const float xs = base + x[j];
        const bool c_ok = j < nv;
        if (dbg && q_in && c_ok) P.dbg_xs[(size_t)slot * P.dbg_stride + cbase + j] = xs;
        const float den = mb[j] + corrS;
        if (pass == 1) {
          const bool sv = q_ok && c_ok && (tq <= 0.f || den <= 0.f || xs * xs >= tq * den);
          const uint32_t m = __ballot_sync(FULL, sv);
          if (lane == j) mymask = m;
        } else if (q_ok && c_ok) {
          // the bound itself (slack included): seeds are ranked by it, and it is stored as a code that only errs upwards
          float metric = den > 0.f ? xs * rsqrt_approx(nq * den) * (PRUNE_SLACK * 1.00001f) : INFINITY;
          if (has_codes) codes[j >> 2] |= ceil_to_byte(metric * UBQ_SCALE) << ((j & 3) * 8);
          if (metric > sm[B_SEEDS - 1]) {
            int cc = (int)(cbase + j);
#pragma unroll
            for (int i = 0; i < B_SEEDS; i++)
              if (metric > sm[i]) {
                const float tm = sm[i]; sm[i] = metric; metric = tm;
                const int tc = sc[i]; sc[i] = cc; cc = tc;
              }
          }
        }
      }
      KV_BOUND_MARK(KBW_BOUND)
      if (pass == 0 && has_codes && q_in)
        *reinterpret_cast<uint4 *>(P.ubq + (size_t)slot * P.ubq_stride + cbase) = make_uint4(codes[0], codes[1], codes[2], codes[3]);
      // four warps (one per chunk-column quarter) share the group's list
      if (pass == 1) list_append(P.lists, list, &S.lcount[qtr], my_pages, (uint32_t)(cbase + lane), mymask, n_pairs, n_recs);
      KV_BOUND_MARK(KBW_STORE)
      // R is clean again: the MMA warpgroup and, once all workers are here, the next block's join may add to it
      asm volatile("bar.arrive %0, %1;" ::"n"(B_BAR_RCLEAN), "n"(B_THREADS) : "memory");
      asm volatile("bar.sync %0, %1;" ::"n"(B_BAR_WORKERS), "n"(B_WORKERS * 32) : "memory");
      KV_BOUND_MARK(KBW_BARRIER)
    }
    KV_BOUND_PROF({
      // kbc_bit, kbc_rounds, kbc_multi and kbc_fan are the warp's (lane 0 adds them); the table hits and mask bits are
      // per lane
      kbc_tab = __reduce_add_sync(FULL, kbc_tab); kbc_bits = __reduce_add_sync(FULL, kbc_bits);
      if (lane == 0) {
        _Pragma("unroll")
        for (int i = 0; i < KBW_N; i++) atomicAdd(&g_bound_prof[i], (unsigned long long)kbp[i]);
        atomicAdd(&g_bound_prof[KBC_BIT_HITS], (unsigned long long)kbc_bit);
        atomicAdd(&g_bound_prof[KBC_ROUNDS], (unsigned long long)kbc_rounds);
        atomicAdd(&g_bound_prof[KBC_MULTI_ROUND], (unsigned long long)kbc_multi);
        atomicAdd(&g_bound_prof[KBC_TABLE_HITS], (unsigned long long)kbc_tab);
        atomicAdd(&g_bound_prof[KBC_MASK_BITS], (unsigned long long)kbc_bits);
        atomicAdd(&g_bound_prof[KBC_FAN_ITERS], (unsigned long long)kbc_fan);
        atomicAdd(&g_bound_prof[KBC_WORKER_WARP_BLOCKS], (unsigned long long)it);
      }
      if (threadIdx.x == 0) {
        atomicAdd(&g_bound_prof[KBC_JOIN_SLOWEST], kbc_slowest);
        atomicAdd(&g_bound_prof[KBC_MMA_LAST], kbc_mma_last);
        atomicAdd(&g_bound_prof[KBC_MMA_LAST_CYC], kbc_mma_cyc);
        atomicAdd(&g_bound_prof[KBC_WORKERS_LAST_CYC], kbc_w_cyc);
        atomicAdd(&g_bound_prof[KBC_CTA_BLOCKS], (unsigned long long)it);
        atomicAdd(&g_bound_prof[KBC_CTAS], 1ull);
        const unsigned int cta = blockIdx.y * gridDim.x + blockIdx.x;
        if (cta < KB_MAX_CTAS) g_bound_prof[KBT_END + cta] = kb_globaltimer();
      }
    })
    if (pass == 0) {
      if (q_in) {
        int *o = P.seeds + ((size_t)slot * P.n_bsplits + bsplit) * B_SEEDS_PER_QUERY + cs * B_SEEDS;
#pragma unroll
        for (int i = 0; i < B_SEEDS; i++) o[i] = sc[i];
      }
    } else {
      if (cs == 0 && lane == 0) P.lists.count[list] = S.lcount[qtr];
      flush_list_stats(P.stats, n_pairs, n_recs);
    }
  }
}

// ----------------------------------------------------------------------------------------
// K1b-B2: threshold codes of the candidate scan's codes mode (second pass without recomputing the bounds).  A chunk is
// a candidate of a query when its stored bound code reaches floor(UBQ_SCALE x the query's threshold) -- the threshold
// as it stands after the seed scan (and the threshold exchange of a two-phase batch), snapshotted here because the scan
// raises gthr while it selects: every CTA of a group then selects the same candidates, run after run.  256: the query
// takes no candidate (null or irregular: answered elsewhere).
// ----------------------------------------------------------------------------------------
__global__ void threshold_codes_kernel(const float *__restrict__ q_nq, const int *__restrict__ gthr, int64_t n_q, int *tcode) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n_q) return;
  uint32_t t = 256;
  if (q_nq[i] > 0.f) {
    const float th = __int_as_float(gthr[i]);
    t = th > 0.f ? (uint32_t)fminf(255.f, floorf(th * UBQ_SCALE)) : 0u;
  }
  tcode[i] = (int)t;
}

}  // namespace kvk
