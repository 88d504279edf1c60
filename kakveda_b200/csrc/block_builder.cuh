// Host-side construction of the scan layout (column blocks, dense frequent-feature matrix) and small host helpers.
// Pure host code without CUDA calls, so that it can be unit-tested on a box without a GPU
// (tests/cpp/block_builder_check.cu, run by tests/test_host.py): decoding the blocks must give back the rows.
#pragma once
#include "tfidf_kernels.cuh"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>
#include <thread>
#include <utility>
#include <vector>

namespace kvh {

using namespace kvk;

template <class F>
void parallel_for(int64_t n, int T, F &&body) {  // body(t, begin, end); thread t owns [n*t/T, n*(t+1)/T)
  T = (int)std::max<int64_t>(1, std::min<int64_t>(T, n));
  std::vector<std::thread> th;
  for (int t = 1; t < T; t++) th.emplace_back([&, t] { body(t, n * t / T, n * (t + 1) / T); });
  body(0, 0, n / T);
  for (auto &x : th) x.join();
}

// idf-derived weights of one feature as every query table uses them (see the header of tfidf_kernels.cuh)
inline void idf_host(int64_t n_total, uint32_t df, double &a, double &d, int jaccard, int corpus_fit) {
  if (jaccard) { a = 1.0; d = 0.0; return; }
  double num = (double)(n_total + (corpus_fit ? 1 : 2));
  double ib = std::log(num / ((double)df + 1.0)) + 1.0;
  double iq = corpus_fit ? ib : std::log(num / ((double)df + 2.0)) + 1.0;
  if (corpus_fit && df == 0) { a = d = 0.0; return; }  // in no live row: ignored like an out-of-vocabulary feature
  a = iq * iq;
  d = a - ib * ib;
}

// ---- index sort: result == std::stable_sort(order = 0..n-1, less) for any strict weak ordering `less` ----
// Two adjacent sorted runs first[0, n1) and first[n1, n1 + n2) merged on P threads: the first run is cut into P
// pieces, each piece merges with the elements of the second run that fall between its end points.  `total` is a
// total order (no two elements compare equal), so the cut points are unambiguous.
template <class Total>
void parallel_merge(int *first, int64_t n1, int64_t n2, int *tmp, Total total, int P) {
  if (n1 == 0 || n2 == 0) return;
  P = (int)std::max<int64_t>(1, std::min<int64_t>(P, n1 / 2048));
  std::vector<int64_t> s1((size_t)P + 1), s2((size_t)P + 1);
  for (int p = 0; p <= P; p++) {
    s1[(size_t)p] = n1 * p / P;
    s2[(size_t)p] = p == 0 ? 0 : (p == P ? n2 : std::lower_bound(first + n1, first + n1 + n2, first[s1[(size_t)p]], total) - (first + n1));
  }
  parallel_for(P, P, [&](int, int64_t a, int64_t b) {
    for (int64_t p = a; p < b; p++) {
      std::merge(first + s1[(size_t)p], first + s1[(size_t)p + 1], first + n1 + s2[(size_t)p], first + n1 + s2[(size_t)p + 1],
                 tmp + s1[(size_t)p] + s2[(size_t)p], total);
    }
  });
  parallel_for(n1 + n2, P, [&](int, int64_t a, int64_t b) { std::copy(tmp + a, tmp + b, first + a); });  // after ALL merges
}

// order holds consecutive runs [cut[i], cut[i+1]) that are each sorted by (less, index): merged pairwise, every level on
// all T threads.
template <class Less>
void merge_sorted_runs(std::vector<int> &order, const std::vector<int64_t> &cut, Less less, int T) {
  auto total = [&](int a, int b) { return less(a, b) || (!less(b, a) && a < b); };  // ties by index == stability
  const int runs = (int)cut.size() - 1;
  std::vector<int> tmp(order.size());
  for (int width = 1; width < runs; width *= 2) {
    const int merges = (runs + 2 * width - 1) / (2 * width);
    const int per = std::max(1, T / merges);
    parallel_for(merges, std::min(merges, std::max(T, 1)), [&](int, int64_t a, int64_t b) {
      for (int64_t m = a; m < b; m++) {
        const int lo = (int)(m * 2 * width), mid = std::min(runs, lo + width), hi = std::min(runs, lo + 2 * width);
        if (mid < hi)
          parallel_merge(order.data() + cut[(size_t)lo], cut[(size_t)mid] - cut[(size_t)lo], cut[(size_t)hi] - cut[(size_t)mid],
                         tmp.data() + cut[(size_t)lo], total, per);
      }
    });
  }
}

template <class Less>
void stable_sort_indices(std::vector<int> &order, Less less, int T) {
  const int64_t n = (int64_t)order.size();
  auto total = [&](int a, int b) { return less(a, b) || (!less(b, a) && a < b); };
  int parts = 1;
  if (n >= 8192) while (parts * 2 <= T && parts < 64) parts *= 2;
  std::vector<int64_t> cut((size_t)parts + 1);
  for (int i = 0; i <= parts; i++) cut[(size_t)i] = n * i / parts;
  parallel_for(parts, parts, [&](int, int64_t a, int64_t b) {
    for (int64_t i = a; i < b; i++) std::sort(order.begin() + cut[(size_t)i], order.begin() + cut[(size_t)i + 1], total);
  });
  merge_sorted_runs(order, cut, less, T);
}

// ---- column blocks ----
struct BlockLayout {
  int64_t n_chunks = 0, n_chunks_pad = 0;     // pad: multiple of 128 (the bound kernel's block of chunks)
  std::vector<std::vector<uint32_t>> parts;   // thread t built the blocks of chunks [n_chunks*t/T, n_chunks*(t+1)/T)
  std::vector<int64_t> part_off;              // offset (in 32-bit words) of each part in the concatenated array
  int64_t total_words = 0;
  std::vector<BlockInfo> binfo;               // [n_chunks_pad] (padding chunks: empty blocks)
  std::vector<std::pair<unsigned long long, uint32_t>> ovf;  // (chunk << 32 | entry) -> tf, sorted
  std::vector<short> fslot;                   // [V] column of a frequent feature, -1 otherwise
  std::vector<uint32_t> frequent;             // the frequent features by column
  std::vector<__half> Uf;                     // [n_chunks_pad][NF] largest tf of the frequent features per chunk
  std::vector<unsigned short> fslot2;         // [V] bit row of a second-class feature, 0xFFFF otherwise
  std::vector<uint32_t> Ubt;                  // [n_chunks_pad / 64][NF2][2][2]: bit c % 64 of plane 0 / 1 = present in chunk c with tf >= 1 / >= 2
  // rare features per 64-chunk block (the bound kernel's inverted join): presence bitmap + two-choice table
  std::vector<uint32_t> rbloom;               // [n_blocks][RB_BITS / 32]
  std::vector<uint4> rt_slots;                // all tables (slot layout: rt_slot2), a feature in slot rt_slot1 or rt_slot2 of its block's
  std::vector<uint32_t> rt_off, rt_size;      // [n_blocks] first slot / slots of a block's table
  int64_t rt_enlarged = 0;                    // tables whose cuckoo insertion failed at the first size and were enlarged
  // Only with build_blocks(..., linear_tables = true), for the host layout checks: the same entries placed by linear
  // probing from rt_slot in tables of the same offsets and sizes, feature id << 5 | largest 5-bit tf (31: see tfmax) and
  // the chunk mask in separate arrays (the rare-table format before the two-choice slots).  The index never builds them.
  std::vector<uint32_t> rt_keys;
  std::vector<unsigned long long> rt_masks;
  int64_t n_entries = 0, n_rare_entries = 0, n_f2_entries = 0;
};

// Places `n` entries (slots as in rt_slot2) in a two-choice table of *size slots (KEY_EMPTY-initialised by the caller) at tab:
// cuckoo insertion in the given order with at most RT_MAX_KICKS evictions per entry.  Returns false when an entry found
// no place; the caller then enlarges the table and starts over.  Deterministic: the same entries in the same order give
// the same bytes.
constexpr int RT_MAX_KICKS = 256;
inline bool rt_cuckoo(const uint4 *entries, size_t n, uint4 *tab, uint32_t size) {
  for (size_t i = 0; i < n; i++) {
    uint4 e = entries[i];
    uint32_t pos = rt_slot1(e.x, size);
    if (tab[pos].x != KEY_EMPTY) {
      const uint32_t p2 = rt_slot2(e.x, size);
      if (tab[p2].x == KEY_EMPTY) pos = p2;
    }
    for (int kick = 0;; kick++) {
      std::swap(e, tab[pos]);
      if (e.x == KEY_EMPTY) break;
      if (kick == RT_MAX_KICKS) return false;
      const uint32_t a = rt_slot1(e.x, size);  // the evicted entry moves to its other slot
      pos = pos == a ? rt_slot2(e.x, size) : a;
    }
  }
  return true;
}

// Slots of a block's table for n entries: load factor <= 0.4, at least 4
inline uint32_t rt_initial_size(size_t n) { return (uint32_t)std::max<size_t>(4, (n * 5 + 1) / 2); }

// the sorted (feature, tf, row-in-chunk) keys of a chunk's non-universal entries
inline void chunk_keys(const int64_t *indptr, const uint32_t *ids, const uint16_t *tf, const int *perm, int64_t n,
                       const uint8_t *univ, int64_t c, std::vector<unsigned long long> &keys) {
  keys.clear();
  const int64_t pos0 = c * CHUNK_ROWS, pos1 = std::min<int64_t>(n, pos0 + CHUNK_ROWS);
  for (int64_t pos = pos0; pos < pos1; pos++) {
    const int64_t r = perm[pos];
    for (int64_t p = indptr[r]; p < indptr[r + 1]; p++) {
      const uint32_t f = ids[p];
      if (!univ[f]) keys.push_back(((unsigned long long)f << 21) | ((unsigned long long)tf[p] << 5) | (unsigned long long)(pos - pos0));
    }
  }
  std::sort(keys.begin(), keys.end());
}

inline void build_blocks(const int64_t *indptr, const uint32_t *ids, const uint16_t *tf, const int *perm, int64_t n,
                         int64_t V, const uint8_t *univ, const uint32_t *tfmaxg, int T, BlockLayout &L,
                         bool linear_tables = true) {
  L.n_chunks = (n + CHUNK_ROWS - 1) / CHUNK_ROWS;
  L.n_chunks_pad = std::max<int64_t>(128, (L.n_chunks + 127) / 128 * 128);
  T = (int)std::max<int64_t>(1, std::min<int64_t>(T, std::max<int64_t>(1, L.n_chunks)));
  const int64_t Vz = std::max<int64_t>(V, 1);
  // pass 1: in how many chunks does a feature occur
  std::unique_ptr<std::atomic<uint32_t>[]> cnt(new std::atomic<uint32_t>[(size_t)Vz]);
  parallel_for(Vz, T, [&](int, int64_t a0, int64_t a1) {
    for (int64_t i = a0; i < a1; i++) cnt[(size_t)i].store(0, std::memory_order_relaxed);
  });
  parallel_for(L.n_chunks, T, [&](int, int64_t c0, int64_t c1) {
    std::vector<unsigned long long> keys;
    for (int64_t c = c0; c < c1; c++) {
      chunk_keys(indptr, ids, tf, perm, n, univ, c, keys);
      uint32_t prev = 0xFFFFFFFFu;
      for (unsigned long long k : keys) {
        const uint32_t f = (uint32_t)(k >> 21);
        if (f != prev) cnt[f].fetch_add(1, std::memory_order_relaxed);
        prev = f;
      }
    }
  });
  // the NF features found in most chunks (ties: lower id); a feature with huge term frequencies stays "rare" (fp16)
  L.fslot.assign((size_t)Vz, (short)-1);
  L.frequent.clear();
  {
    std::vector<std::pair<uint32_t, uint32_t>> cand;  // (chunks, feature)
    for (int64_t f = 0; f < V; f++) {
      const uint32_t cfreq = cnt[(size_t)f].load(std::memory_order_relaxed);
      if (cfreq > 0 && tfmaxg[f] <= 2048u) cand.emplace_back(cfreq, (uint32_t)f);
    }
    const size_t keep = std::min<size_t>(NF, cand.size());
    std::partial_sort(cand.begin(), cand.begin() + (std::ptrdiff_t)keep, cand.end(),
                      [](const std::pair<uint32_t, uint32_t> &a, const std::pair<uint32_t, uint32_t> &b) {
                        return a.first != b.first ? a.first > b.first : a.second < b.second;
                      });
    for (size_t i = 0; i < keep; i++) {
      L.fslot[cand[i].second] = (short)i;
      L.frequent.push_back(cand[i].second);
    }
    // second class: the next NF2 features by chunk frequency (any tf: the bound uses the feature's largest tf)
    L.fslot2.assign((size_t)Vz, (unsigned short)0xFFFF);
    std::vector<std::pair<uint32_t, uint32_t>> rest;
    for (int64_t f = 0; f < V; f++) {
      const uint32_t cfreq = cnt[(size_t)f].load(std::memory_order_relaxed);
      if (cfreq > 0 && L.fslot[(size_t)f] < 0) rest.emplace_back(cfreq, (uint32_t)f);
    }
    const size_t keep2 = std::min<size_t>(NF2, rest.size());
    std::partial_sort(rest.begin(), rest.begin() + (std::ptrdiff_t)keep2, rest.end(),
                      [](const std::pair<uint32_t, uint32_t> &a, const std::pair<uint32_t, uint32_t> &b) {
                        return a.first != b.first ? a.first > b.first : a.second < b.second;
                      });
    for (size_t i = 0; i < keep2; i++) L.fslot2[rest[i].second] = (unsigned short)i;
  }
  L.Ubt.assign((size_t)(L.n_chunks_pad / 64) * NF2 * 4, 0u);
  // pass 2: the blocks
  L.parts.assign((size_t)T, {});
  L.binfo.assign((size_t)L.n_chunks_pad, BlockInfo{0, 0, 0, 0, 0});
  L.Uf.assign((size_t)L.n_chunks_pad * NF, __float2half(0.f));
  std::vector<std::vector<std::pair<unsigned long long, uint32_t>>> povf((size_t)T);
  std::vector<int64_t> words_of((size_t)L.n_chunks, 0);
  std::vector<int64_t> ent((size_t)T, 0), rare((size_t)T, 0), sec((size_t)T, 0);
  parallel_for(L.n_chunks, T, [&](int t, int64_t c0, int64_t c1) {
    std::vector<unsigned long long> keys;
    std::vector<uint32_t> w_r, m_r, w_2, m_2, w_f, m_f;  // rare / second-class / frequent entries of the chunk: words and masks
    std::vector<uint32_t> tf_r, tf_2, tf_f;              // full term frequencies (overflow table)
    auto &out = L.parts[(size_t)t];
    for (int64_t c = c0; c < c1; c++) {
      chunk_keys(indptr, ids, tf, perm, n, univ, c, keys);
      const int rows = (int)std::min<int64_t>(CHUNK_ROWS, n - c * CHUNK_ROWS);
      const uint32_t valid = rows == 32 ? 0xFFFFFFFFu : ((1u << rows) - 1u);
      w_r.clear(); m_r.clear(); w_2.clear(); m_2.clear(); w_f.clear(); m_f.clear(); tf_r.clear(); tf_2.clear(); tf_f.clear();
      __half *urow = L.Uf.data() + (size_t)c * NF;
      for (size_t i = 0; i < keys.size();) {
        const unsigned long long ft = keys[i] >> 5;  // (feature, tf)
        uint32_t mask = 0;
        while (i < keys.size() && (keys[i] >> 5) == ft) { mask |= 1u << (keys[i] & 31u); i++; }
        const uint32_t f = (uint32_t)(ft >> 16), tfv = (uint32_t)(ft & 0xFFFFu);
        uint32_t word = (f << 5) | (tfv >= TF_OVF ? TF_OVF : tfv);
        if (mask == valid) word |= W_ALL;
        const int fs = L.fslot[f];
        if (fs >= 0) {
          w_f.push_back(word); m_f.push_back(mask); tf_f.push_back(tfv);
          urow[fs] = __float2half((float)tfv);  // keys ascend in tf: the last one is the largest (exact: tf <= 2048)
        } else if (L.fslot2[f] != 0xFFFFu) {
          w_2.push_back(word); m_2.push_back(mask); tf_2.push_back(tfv);
          const unsigned short f2 = L.fslot2[f];  // chunks of one 64-chunk block may belong to different threads: atomic OR
          uint32_t *w0 = &L.Ubt[((size_t)(c >> 6) * NF2 + f2) * 4 + ((c & 63) >> 5)];
          __atomic_fetch_or(w0, 1u << (c & 31), __ATOMIC_RELAXED);
          if (tfv >= 2) __atomic_fetch_or(w0 + 2, 1u << (c & 31), __ATOMIC_RELAXED);
        } else {
          w_r.push_back(word); m_r.push_back(mask); tf_r.push_back(tfv);
        }
      }
      const size_t E = w_r.size() + w_2.size() + w_f.size(), E4 = (E + 3) & ~(size_t)3;
      const size_t before = out.size();
      out.insert(out.end(), w_r.begin(), w_r.end());
      out.insert(out.end(), w_2.begin(), w_2.end());
      out.insert(out.end(), w_f.begin(), w_f.end());
      out.resize(before + E4, PAD_WORD);
      out.insert(out.end(), m_r.begin(), m_r.end());
      out.insert(out.end(), m_2.begin(), m_2.end());
      out.insert(out.end(), m_f.begin(), m_f.end());
      out.resize(before + 2 * E4, 0u);
      for (size_t i = 0; i < tf_r.size(); i++)
        if (tf_r[i] >= TF_OVF) povf[(size_t)t].emplace_back(((unsigned long long)c << 32) | (unsigned long long)i, tf_r[i]);
      for (size_t i = 0; i < tf_2.size(); i++)
        if (tf_2[i] >= TF_OVF) povf[(size_t)t].emplace_back(((unsigned long long)c << 32) | (unsigned long long)(w_r.size() + i), tf_2[i]);
      for (size_t i = 0; i < tf_f.size(); i++)
        if (tf_f[i] >= TF_OVF) povf[(size_t)t].emplace_back(((unsigned long long)c << 32) | (unsigned long long)(w_r.size() + w_2.size() + i), tf_f[i]);
      BlockInfo bi;
      bi.off4 = 0;
      bi.n_entries = (uint16_t)E;
      bi.n_rare = (uint16_t)w_r.size();
      bi.n_f2 = (uint16_t)w_2.size();
      bi.pad = 0;
      L.binfo[(size_t)c] = bi;
      words_of[(size_t)c] = (int64_t)(2 * E4);
      ent[(size_t)t] += (int64_t)E;
      rare[(size_t)t] += (int64_t)w_r.size();
      sec[(size_t)t] += (int64_t)w_2.size();
    }
  });
  int64_t off = 0;
  for (int64_t c = 0; c < L.n_chunks; c++) {
    L.binfo[(size_t)c].off4 = (uint32_t)(off / 4);
    off += words_of[(size_t)c];
  }
  for (int64_t c = L.n_chunks; c < L.n_chunks_pad; c++) L.binfo[(size_t)c].off4 = (uint32_t)(off / 4);
  L.total_words = off;
  L.part_off.assign((size_t)T, 0);
  {
    int64_t o = 0;
    for (int t = 0; t < T; t++) { L.part_off[(size_t)t] = o; o += (int64_t)L.parts[(size_t)t].size(); }
  }
  // pass 3: per 64-chunk block the inverted index of its rare entries
  {
    const int64_t n_blocks = L.n_chunks_pad / 64;
    L.rbloom.assign((size_t)n_blocks * (RB_BITS / 32), 0u);
    L.rt_off.assign((size_t)n_blocks, 0);
    L.rt_size.assign((size_t)n_blocks, 1);
    auto word_ptr = [&](int64_t off_words) -> const uint32_t * {  // position in the per-thread parts
      size_t tt = (size_t)(std::upper_bound(L.part_off.begin(), L.part_off.end(), off_words) - L.part_off.begin()) - 1;
      return L.parts[tt].data() + (off_words - L.part_off[tt]);
    };
    std::vector<std::vector<uint4>> tabs((size_t)n_blocks);  // the block's entries as slots, by feature
    std::vector<int64_t> enlarged((size_t)T, 0);
    parallel_for(n_blocks, T, [&](int t, int64_t b0, int64_t b1) {
      std::vector<unsigned long long> es;  // fid << 16 | tf5 << 8 | chunk in block
      std::vector<uint4> scratch;
      for (int64_t b = b0; b < b1; b++) {
        es.clear();
        for (int64_t c = b * 64; c < std::min<int64_t>(L.n_chunks, b * 64 + 64); c++) {
          const BlockInfo bi = L.binfo[(size_t)c];
          const uint32_t *w = word_ptr((int64_t)bi.off4 * 4);
          for (int e = 0; e < bi.n_rare; e++)
            es.push_back(((unsigned long long)((w[e] >> 5) & FID_MASK) << 16) | ((unsigned long long)(w[e] & 31u) << 8) | (unsigned long long)(c - b * 64));
        }
        std::sort(es.begin(), es.end());
        auto &tab = tabs[(size_t)b];
        for (size_t i = 0; i < es.size();) {
          const uint32_t f = (uint32_t)(es[i] >> 16);
          uint32_t tfm = 0;
          unsigned long long mask = 0;
          while (i < es.size() && (uint32_t)(es[i] >> 16) == f) { tfm = std::max<uint32_t>(tfm, (uint32_t)((es[i] >> 8) & 31u)); mask |= 1ULL << (es[i] & 63u); i++; }
          // the tf the bound kernel multiplies by: an overflowed 5-bit tf stands for the feature's global largest tf
          tab.push_back(make_uint4(f, tfm == TF_OVF ? tfmaxg[f] : tfm, (uint32_t)mask, (uint32_t)(mask >> 32)));
          const uint32_t bb = rb_bit(f);
          L.rbloom[(size_t)b * (RB_BITS / 32) + (bb >> 5)] |= 1u << (bb & 31u);
        }
        // the size at which the cuckoo insertion succeeds: load <= 0.4, + 25 % per failure
        uint32_t size = rt_initial_size(tab.size());
        for (;;) {
          scratch.assign(size, make_uint4(KEY_EMPTY, 0u, 0u, 0u));
          if (rt_cuckoo(tab.data(), tab.size(), scratch.data(), size)) break;
          size += size / 4;
          enlarged[(size_t)t]++;
        }
        L.rt_size[(size_t)b] = size;
      }
    });
    int64_t total = 0;
    for (int64_t b = 0; b < n_blocks; b++) { L.rt_off[(size_t)b] = (uint32_t)total; total += L.rt_size[(size_t)b]; }
    L.rt_slots.assign((size_t)total, make_uint4(KEY_EMPTY, 0u, 0u, 0u));
    L.rt_enlarged = 0;
    for (int64_t e : enlarged) L.rt_enlarged += e;
    L.rt_keys.assign(linear_tables ? (size_t)total : 0, KEY_EMPTY);
    L.rt_masks.assign(linear_tables ? (size_t)total : 0, 0ULL);
    parallel_for(n_blocks, T, [&](int, int64_t b0, int64_t b1) {
      for (int64_t b = b0; b < b1; b++) {
        const auto &tab = tabs[(size_t)b];
        const uint32_t size = L.rt_size[(size_t)b];
        rt_cuckoo(tab.data(), tab.size(), L.rt_slots.data() + L.rt_off[(size_t)b], size);  // succeeds at this size
        if (linear_tables) {
          uint32_t *keys = L.rt_keys.data() + L.rt_off[(size_t)b];
          unsigned long long *masks = L.rt_masks.data() + L.rt_off[(size_t)b];
          for (const uint4 &e : tab) {
            uint32_t h = rt_slot(e.x, size);
            while (keys[h] != KEY_EMPTY) h = h + 1 == size ? 0 : h + 1;
            keys[h] = (e.x << 5) | std::min<uint32_t>(e.y, TF_OVF);
            masks[h] = (unsigned long long)e.z | ((unsigned long long)e.w << 32);
          }
        }
        std::vector<uint4>().swap(tabs[(size_t)b]);
      }
    });
  }
  L.ovf.clear();
  L.n_entries = L.n_rare_entries = L.n_f2_entries = 0;
  for (int t = 0; t < T; t++) {
    L.ovf.insert(L.ovf.end(), povf[(size_t)t].begin(), povf[(size_t)t].end());
    L.n_entries += ent[(size_t)t];
    L.n_rare_entries += rare[(size_t)t];
    L.n_f2_entries += sec[(size_t)t];
  }
  std::sort(L.ovf.begin(), L.ovf.end());
}

}  // namespace kvh
