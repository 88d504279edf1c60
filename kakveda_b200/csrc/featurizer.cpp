// Host featuriser: word 1,2-gram counting over a shared vocabulary (SURVEY.md section 8 row a2).
//
// Replaces, for the GFKB match path, what TfidfVectorizer does before any arithmetic:
//   lowercase=True, token_pattern (?u)\b\w\w+\b   (sklearn/feature_extraction/text.py:1969)
//   _word_ngrams with ngram_range=(1,2)            (text.py:248)
//   _count_vocab: per-document feature counts      (text.py:1257)
// as invoked by services/shared/similarity.py:17-18.  The vocabulary identifies a feature by
// a 128-bit hash of its bytes (collision probability < 1e-20 at 1e8 features), so no strings
// are retained; ids are dense uint32 in order of first insertion.  Insertion is lock-free so
// that millions of rows can be featurised on all host cores.
#include "kv_internal.h"

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <vector>

namespace {

inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
inline uint64_t fmix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return k;
}

// MurmurHash3 x64 128-bit (public-domain algorithm by Austin Appleby), little-endian loads.
void hash128(const char *data, size_t len, uint64_t seed, uint64_t out[2]) {
  const uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
  uint64_t h1 = seed, h2 = seed;
  const size_t nblocks = len / 16;
  for (size_t i = 0; i < nblocks; i++) {
    uint64_t k1, k2;
    memcpy(&k1, data + i * 16, 8);
    memcpy(&k2, data + i * 16 + 8, 8);
    k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
    h1 = rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
    k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;
    h2 = rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
  }
  const unsigned char *tail = (const unsigned char *)(data + nblocks * 16);
  uint64_t k1 = 0, k2 = 0;
  switch (len & 15) {
    case 15: k2 ^= (uint64_t)tail[14] << 48; [[fallthrough]];
    case 14: k2 ^= (uint64_t)tail[13] << 40; [[fallthrough]];
    case 13: k2 ^= (uint64_t)tail[12] << 32; [[fallthrough]];
    case 12: k2 ^= (uint64_t)tail[11] << 24; [[fallthrough]];
    case 11: k2 ^= (uint64_t)tail[10] << 16; [[fallthrough]];
    case 10: k2 ^= (uint64_t)tail[9] << 8; [[fallthrough]];
    case 9:  k2 ^= (uint64_t)tail[8];
             k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2; [[fallthrough]];
    case 8:  k1 ^= (uint64_t)tail[7] << 56; [[fallthrough]];
    case 7:  k1 ^= (uint64_t)tail[6] << 48; [[fallthrough]];
    case 6:  k1 ^= (uint64_t)tail[5] << 40; [[fallthrough]];
    case 5:  k1 ^= (uint64_t)tail[4] << 32; [[fallthrough]];
    case 4:  k1 ^= (uint64_t)tail[3] << 24; [[fallthrough]];
    case 3:  k1 ^= (uint64_t)tail[2] << 16; [[fallthrough]];
    case 2:  k1 ^= (uint64_t)tail[1] << 8; [[fallthrough]];
    case 1:  k1 ^= (uint64_t)tail[0];
             k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
  }
  h1 ^= len; h2 ^= len; h1 += h2; h2 += h1;
  h1 = fmix64(h1); h2 = fmix64(h2);
  h1 += h2; h2 += h1;
  out[0] = h1; out[1] = h2;
}

constexpr uint32_t SLOT_EMPTY = 0xFFFFFFFFu;
constexpr uint32_t SLOT_LOCKED = 0xFFFFFFFEu;
constexpr uint32_t SLOT_PENDING = 0xFFFFFFFDu;  // created in the current epoch, final id not assigned yet
constexpr uint64_t PENDING_FLAG = 1ULL << 63;

struct Slot {
  uint64_t k0, k1;
  std::atomic<uint64_t> first;  // smallest (doc << 24 | position) that produced this feature in its epoch
  std::atomic<uint32_t> id;
};

struct Feat {
  uint64_t h0, h1;
  uint32_t tf;
  uint32_t pos;  // order of first appearance inside the document
};

}  // namespace

struct kv_vocab {
  std::unique_ptr<Slot[]> slots;
  uint64_t cap = 0;  // power of two
  std::atomic<uint32_t> count{0};

  void alloc(uint64_t c) {
    slots.reset(new Slot[c]);
    cap = c;
    for (uint64_t i = 0; i < c; i++) slots[i].id.store(SLOT_EMPTY, std::memory_order_relaxed);
  }
  void reserve(uint64_t want_entries) {  // single-threaded; keeps load factor <= 0.5
    uint64_t need = 1024;
    while (need < 2 * want_entries) need <<= 1;
    if (need <= cap) return;
    std::unique_ptr<Slot[]> old = std::move(slots);
    uint64_t old_cap = cap;
    alloc(need);
    for (uint64_t i = 0; i < old_cap; i++) {
      uint32_t id = old[i].id.load(std::memory_order_relaxed);
      if (id == SLOT_EMPTY) continue;
      uint64_t j = old[i].k0 & (cap - 1);
      while (slots[j].id.load(std::memory_order_relaxed) != SLOT_EMPTY) j = (j + 1) & (cap - 1);
      slots[j].k0 = old[i].k0; slots[j].k1 = old[i].k1;
      slots[j].first.store(0, std::memory_order_relaxed);
      slots[j].id.store(id, std::memory_order_relaxed);
    }
  }
  // Returns the feature id; SLOT_EMPTY when absent and !grow; or PENDING_FLAG|slot for a feature
  // first seen in the current epoch (ids are handed out after the epoch, ordered by first
  // appearance, so the numbering does not depend on thread timing).  `created` collects the
  // slots this thread claimed.
  uint64_t find_or_add(uint64_t h0, uint64_t h1, bool grow, uint64_t where, std::vector<uint64_t> &created) {
    uint64_t j = h0 & (cap - 1);
    for (;;) {
      uint32_t id = slots[j].id.load(std::memory_order_acquire);
      if (id == SLOT_EMPTY) {
        if (!grow) return SLOT_EMPTY;
        uint32_t expect = SLOT_EMPTY;
        if (slots[j].id.compare_exchange_strong(expect, SLOT_LOCKED, std::memory_order_acq_rel)) {
          slots[j].k0 = h0; slots[j].k1 = h1;
          slots[j].first.store(where, std::memory_order_relaxed);
          slots[j].id.store(SLOT_PENDING, std::memory_order_release);
          created.push_back(j);
          return PENDING_FLAG | j;
        }
        continue;  // somebody else took this slot: re-read it
      }
      if (id == SLOT_LOCKED) { std::this_thread::yield(); continue; }
      if (slots[j].k0 == h0 && slots[j].k1 == h1) {
        if (id != SLOT_PENDING) return id;
        uint64_t cur = slots[j].first.load(std::memory_order_relaxed);
        while (where < cur && !slots[j].first.compare_exchange_weak(cur, where, std::memory_order_relaxed)) {}
        return PENDING_FLAG | j;
      }
      j = (j + 1) & (cap - 1);
    }
  }
};

int vocab_export_range(const kv_vocab *v, int64_t lo, int64_t hi, uint64_t *keys) {
  int64_t found = 0;
  for (uint64_t i = 0; i < v->cap; i++) {
    const uint32_t id = v->slots[i].id.load(std::memory_order_acquire);
    if (id >= SLOT_PENDING || (int64_t)id < lo || (int64_t)id >= hi) continue;  // empty, being created, or outside
    keys[2 * (size_t)(id - lo)] = v->slots[i].k0;
    keys[2 * (size_t)(id - lo) + 1] = v->slots[i].k1;
    found++;
  }
  if (found != hi - lo) return kv_fail(KV_ERR_STATE, "vocabulary is being modified");
  return KV_OK;
}

namespace {

inline bool is_word(unsigned char c) {
  return (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '_';
}

// Tokenise one document into [begin,end) spans over `buf` (a lower-cased private copy for raw text).
// Returns false on a non-ASCII byte in raw mode.
bool tokenize(const char *doc, int64_t len, int mode, std::string &buf,
              std::vector<std::pair<uint32_t, uint32_t>> &spans) {
  spans.clear();
  if (mode == KV_TEXT_MIXED) {
    if (len > 0 && doc[0] == '\x1f') { doc++; len--; mode = KV_TEXT_TOKENS; }
    else mode = KV_TEXT_RAW_ASCII;
  }
  buf.assign(doc, (size_t)len);
  if (mode == KV_TEXT_TOKENS) {
    uint32_t b = 0;
    for (uint32_t i = 0; i <= (uint32_t)len; i++) {
      if (i == (uint32_t)len || buf[i] == '\x1f') {
        if (i > b) spans.emplace_back(b, i);
        b = i + 1;
      }
    }
    return true;
  }
  uint32_t run = 0;
  for (uint32_t i = 0; i < (uint32_t)len; i++) {
    unsigned char c = (unsigned char)buf[i];
    if (c >= 0x80) return false;
    if (c >= 'A' && c <= 'Z') { c = (unsigned char)(c + 32); buf[i] = (char)c; }
    if (is_word(c)) {
      run++;
    } else {
      if (run >= 2) spans.emplace_back(i - run, i);
      run = 0;
    }
  }
  if (run >= 2) spans.emplace_back((uint32_t)len - run, (uint32_t)len);
  return true;
}

// Distinct features of one document with counts, in order of first appearance in the text.
// Positions interleave 1-grams and 2-grams in token order (t0, t0 t1, t1, t1 t2, ...): rows that share a text prefix
// share a prefix of their feature lists, which the device index factors out per chunk.
void doc_features(const std::string &buf, const std::vector<std::pair<uint32_t, uint32_t>> &spans,
                  std::string &scratch, std::vector<Feat> &occ, std::vector<Feat> &out) {
  uint64_t h[2];
  const size_t n_occ = spans.empty() ? 0 : 2 * spans.size() - 1;
  constexpr size_t LT = 1024;  // slots of the per-document table (load <= 0.5)
  if (n_occ <= LT / 2) {
    // common case (a signature_text has ~40 tokens): walk the occurrences in position order and count them in a small
    // open-addressing table on the stack -- the first occurrence appends the feature, so `out` is already ordered
    uint32_t slot[LT];  // index into out (relative to w) + 1, 0 = empty
    memset(slot, 0, sizeof(slot));
    const size_t w = out.size();
    auto add = [&](uint64_t h0, uint64_t h1, uint32_t pos) {
      size_t j = (size_t)h0 & (LT - 1);
      for (;;) {
        const uint32_t s = slot[j];
        if (s == 0) {
          out.push_back({h0, h1, 1, pos});
          slot[j] = (uint32_t)(out.size() - w);
          return;
        }
        Feat &f = out[w + s - 1];
        if (f.h0 == h0 && f.h1 == h1) { f.tf++; return; }
        j = (j + 1) & (LT - 1);
      }
    };
    for (size_t i = 0; i < spans.size(); i++) {
      hash128(buf.data() + spans[i].first, spans[i].second - spans[i].first, 0x6b616b76ULL, h);
      add(h[0], h[1], (uint32_t)(2 * i));
      if (i + 1 < spans.size()) {
        scratch.assign(buf, spans[i].first, spans[i].second - spans[i].first);
        scratch.push_back(' ');
        scratch.append(buf, spans[i + 1].first, spans[i + 1].second - spans[i + 1].first);
        hash128(scratch.data(), scratch.size(), 0x6b616b76ULL, h);
        add(h[0], h[1], (uint32_t)(2 * i + 1));
      }
    }
    return;
  }
  // long documents: sort the occurrences by key, count runs, restore the order of first appearance
  occ.clear();
  for (size_t i = 0; i < spans.size(); i++) {
    hash128(buf.data() + spans[i].first, spans[i].second - spans[i].first, 0x6b616b76ULL, h);
    occ.push_back({h[0], h[1], 1, (uint32_t)(2 * i)});
  }
  for (size_t i = 0; i + 1 < spans.size(); i++) {
    scratch.assign(buf, spans[i].first, spans[i].second - spans[i].first);
    scratch.push_back(' ');
    scratch.append(buf, spans[i + 1].first, spans[i + 1].second - spans[i + 1].first);
    hash128(scratch.data(), scratch.size(), 0x6b616b76ULL, h);
    occ.push_back({h[0], h[1], 1, (uint32_t)(2 * i + 1)});
  }
  std::sort(occ.begin(), occ.end(), [](const Feat &a, const Feat &b) {
    if (a.h0 != b.h0) return a.h0 < b.h0;
    if (a.h1 != b.h1) return a.h1 < b.h1;
    return a.pos < b.pos;
  });
  size_t w = out.size();
  for (size_t i = 0; i < occ.size();) {
    size_t j = i + 1;
    while (j < occ.size() && occ[j].h0 == occ[i].h0 && occ[j].h1 == occ[i].h1) j++;
    Feat f = occ[i];
    f.tf = (uint32_t)(j - i);
    out.push_back(f);
    i = j;
  }
  std::sort(out.begin() + w, out.end(), [](const Feat &a, const Feat &b) { return a.pos < b.pos; });
}

}  // namespace

extern "C" {

int kv_vocab_create(kv_vocab **out) {
  if (!out) return kv_fail(KV_ERR_INVALID, "kv_vocab_create: out is NULL");
  try {
    kv_vocab *v = new kv_vocab();
    v->alloc(1 << 16);
    *out = v;
    return KV_OK;
  } catch (const std::bad_alloc &) {
    return kv_fail(KV_ERR_NOMEM, "kv_vocab_create: out of memory");
  }
}

void kv_vocab_destroy(kv_vocab *v) { delete v; }

int64_t kv_vocab_size(const kv_vocab *v) { return v ? (int64_t)v->count.load() : 0; }

// Sidecar support (SURVEY.md section 8(f) rank 4): the vocabulary is fully described by the 128-bit key of every
// feature in id order.
int kv_vocab_export(const kv_vocab *v, uint64_t *keys_out, int64_t capacity) {
  if (!v || (!keys_out && capacity > 0)) return kv_fail(KV_ERR_INVALID, "kv_vocab_export: bad arguments");
  const int64_t n = (int64_t)v->count.load();
  if (capacity < n) return kv_fail(KV_ERR_INVALID, "kv_vocab_export: room for %lld features needed, %lld given", (long long)n,
                                   (long long)capacity);
  for (uint64_t i = 0; i < v->cap; i++) {
    const uint32_t id = v->slots[i].id.load(std::memory_order_relaxed);
    if (id == SLOT_EMPTY) continue;
    if (id >= (uint32_t)n) return kv_fail(KV_ERR_STATE, "kv_vocab_export: vocabulary is being modified");
    keys_out[2 * (size_t)id] = v->slots[i].k0;
    keys_out[2 * (size_t)id + 1] = v->slots[i].k1;
  }
  return KV_OK;
}

int kv_vocab_import(kv_vocab *v, const uint64_t *keys, int64_t n) {
  if (!v || n < 0 || (n > 0 && !keys)) return kv_fail(KV_ERR_INVALID, "kv_vocab_import: bad arguments");
  if (v->count.load() != 0) return kv_fail(KV_ERR_STATE, "kv_vocab_import: the vocabulary must be empty");
  if (n >= (int64_t)SLOT_PENDING) return kv_fail(KV_ERR_INVALID, "kv_vocab_import: too many features");
  try {
    v->reserve((uint64_t)n + 1024);
  } catch (const std::bad_alloc &) {
    return kv_fail(KV_ERR_NOMEM, "kv_vocab_import: out of memory");
  }
  for (int64_t id = 0; id < n; id++) {
    const uint64_t k0 = keys[2 * id], k1 = keys[2 * id + 1];
    uint64_t j = k0 & (v->cap - 1);
    for (;;) {
      const uint32_t cur = v->slots[j].id.load(std::memory_order_relaxed);
      if (cur == SLOT_EMPTY) break;
      if (v->slots[j].k0 == k0 && v->slots[j].k1 == k1) {
        v->alloc(1 << 16);
        v->count.store(0);
        return kv_fail(KV_ERR_INVALID, "kv_vocab_import: features %u and %lld have the same key", cur, (long long)id);
      }
      j = (j + 1) & (v->cap - 1);
    }
    v->slots[j].k0 = k0; v->slots[j].k1 = k1;
    v->slots[j].first.store(0, std::memory_order_relaxed);
    v->slots[j].id.store((uint32_t)id, std::memory_order_relaxed);
  }
  v->count.store((uint32_t)n);
  return KV_OK;
}

int kv_featurize(kv_vocab *v, const char *bytes, const int64_t *offsets, int64_t n_docs, int mode,
                 int grow, int n_threads, kv_csr **out, int64_t *bad_doc) {
  if (!v || !out || n_docs < 0 || (n_docs > 0 && (!bytes || !offsets)))
    return kv_fail(KV_ERR_INVALID, "kv_featurize: bad arguments");
  if (mode != KV_TEXT_RAW_ASCII && mode != KV_TEXT_TOKENS && mode != KV_TEXT_MIXED)
    return kv_fail(KV_ERR_INVALID, "kv_featurize: unknown text mode");
  for (int64_t i = 0; i < n_docs; i++)
    if (offsets[i + 1] < offsets[i] || offsets[i + 1] - offsets[i] > 0x7fffffffLL)
      return kv_fail(KV_ERR_INVALID, "kv_featurize: offsets must be non-decreasing, docs < 2 GiB");
  int T = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
  if (n_threads <= 0)  // several ranks share one host: their launcher sets the per-process thread budget
    if (const char *e = getenv("KAKVEDA_B200_THREADS")) T = atoi(e);
  if (T < 1) T = 1;
  if (T > 256) T = 256;
  try {
    std::unique_ptr<kv_csr> res(new kv_csr());
    res->indptr.assign((size_t)n_docs + 1, 0);
    res->oov.assign((size_t)n_docs, 0.0);
    const int64_t GROUP = 1 << 17;  // documents per vocabulary-capacity epoch
    std::atomic<int64_t> first_bad{-1};
    struct Work {
      std::vector<Feat> feats;       // all features of this thread's docs in the group
      std::vector<uint32_t> counts;  // per doc
    };
    for (int64_t g0 = 0; g0 < n_docs; g0 += GROUP) {
      const int64_t g1 = std::min(n_docs, g0 + GROUP);
      const int64_t gn = g1 - g0;
      const int Tg = (int)std::min<int64_t>(T, std::max<int64_t>(1, gn / 64));
      std::vector<Work> work((size_t)Tg);
      auto range = [&](int t, int64_t &a, int64_t &b) {
        a = g0 + gn * t / Tg;
        b = g0 + gn * (t + 1) / Tg;
      };
      // phase 1: tokenise + hash + count, thread-private
      auto phase1 = [&](int t) {
        int64_t a, b;
        range(t, a, b);
        Work &w = work[(size_t)t];
        w.counts.resize((size_t)(b - a));
        std::string buf, scratch;
        std::vector<std::pair<uint32_t, uint32_t>> spans;
        std::vector<Feat> occ;
        for (int64_t d = a; d < b; d++) {
          if (!tokenize(bytes + offsets[d], offsets[d + 1] - offsets[d], mode, buf, spans)) {
            int64_t cur = first_bad.load();
            while ((cur < 0 || d < cur) && !first_bad.compare_exchange_weak(cur, d)) {}
            w.counts[(size_t)(d - a)] = 0;
            continue;
          }
          size_t before = w.feats.size();
          doc_features(buf, spans, scratch, occ, w.feats);
          w.counts[(size_t)(d - a)] = (uint32_t)(w.feats.size() - before);
        }
      };
      {
        std::vector<std::thread> th;
        for (int t = 1; t < Tg; t++) th.emplace_back(phase1, t);
        phase1(0);
        for (auto &x : th) x.join();
      }
      if (first_bad.load() >= 0) {
        if (bad_doc) *bad_doc = first_bad.load();
        return kv_fail(KV_ERR_NONASCII, "kv_featurize: non-ASCII byte in raw-text document");
      }
      uint64_t occ_total = 0;
      for (auto &w : work) occ_total += w.feats.size();
      if (grow) {
        if ((uint64_t)v->count.load() + occ_total >= 0xFFFFFFF0ULL)
          return kv_fail(KV_ERR_INVALID, "kv_featurize: vocabulary would exceed 2^32 features");
        v->reserve((uint64_t)v->count.load() + occ_total);
      }
      // phase 2: resolve ids (lock-free inserts) in place; in-vocab features compacted to the front
      std::vector<std::vector<uint32_t>> kept((size_t)Tg);  // per doc kept count
      std::vector<std::vector<uint64_t>> created((size_t)Tg);
      auto phase2 = [&](int t) {
        int64_t a, b;
        range(t, a, b);
        Work &w = work[(size_t)t];
        kept[(size_t)t].resize((size_t)(b - a));
        size_t r = 0, wr = 0;
        for (int64_t d = a; d < b; d++) {
          uint32_t c = w.counts[(size_t)(d - a)], k = 0;
          double oov = 0.0;
          for (uint32_t i = 0; i < c; i++, r++) {
            Feat f = w.feats[r];
            uint64_t where = ((uint64_t)(d - g0) << 24) | (f.pos < 0xFFFFFFu ? f.pos : 0xFFFFFFu);
            uint64_t id = v->find_or_add(f.h0, f.h1, grow != 0, where, created[(size_t)t]);
            if (id == SLOT_EMPTY) { oov += (double)f.tf * (double)f.tf; continue; }
            w.feats[wr].h0 = id; w.feats[wr].tf = f.tf;
            wr++; k++;
          }
          kept[(size_t)t][(size_t)(d - a)] = k;
          res->oov[(size_t)d] = oov;
        }
      };
      {
        std::vector<std::thread> th;
        for (int t = 1; t < Tg; t++) th.emplace_back(phase2, t);
        phase2(0);
        for (auto &x : th) x.join();
      }
      // hand out ids to this epoch's new features in order of first appearance (deterministic)
      {
        std::vector<std::pair<uint64_t, uint64_t>> fresh;  // (first, slot)
        for (auto &c : created)
          for (uint64_t j : c) fresh.emplace_back(v->slots[j].first.load(std::memory_order_relaxed), j);
        std::sort(fresh.begin(), fresh.end());
        uint32_t base = v->count.load(std::memory_order_relaxed);
        for (size_t i = 0; i < fresh.size(); i++)
          v->slots[fresh[i].second].id.store(base + (uint32_t)i, std::memory_order_relaxed);
        v->count.store(base + (uint32_t)fresh.size(), std::memory_order_relaxed);
      }
      // assemble CSR for this group
      int64_t nnz0 = res->indptr[(size_t)g0];
      {
        int64_t p = nnz0;
        for (int t = 0; t < Tg; t++) {
          int64_t a, b;
          range(t, a, b);
          for (int64_t d = a; d < b; d++) {
            p += kept[(size_t)t][(size_t)(d - a)];
            res->indptr[(size_t)d + 1] = p;
          }
        }
        res->ids.resize((size_t)p);
        res->tf.resize((size_t)p);
      }
      auto phase3 = [&](int t) {
        int64_t a, b;
        range(t, a, b);
        if (a == b) return;
        Work &w = work[(size_t)t];
        int64_t p = res->indptr[(size_t)a];
        int64_t n = res->indptr[(size_t)b] - p;
        for (int64_t i = 0; i < n; i++) {
          uint64_t id = w.feats[(size_t)i].h0;
          if (id & PENDING_FLAG) id = v->slots[id & ~PENDING_FLAG].id.load(std::memory_order_relaxed);
          res->ids[(size_t)(p + i)] = (uint32_t)id;
          res->tf[(size_t)(p + i)] = w.feats[(size_t)i].tf;
        }
      };
      {
        std::vector<std::thread> th;
        for (int t = 1; t < Tg; t++) th.emplace_back(phase3, t);
        phase3(0);
        for (auto &x : th) x.join();
      }
    }
    *out = res.release();
    return KV_OK;
  } catch (const std::bad_alloc &) {
    return kv_fail(KV_ERR_NOMEM, "kv_featurize: out of memory");
  }
}

int kv_csr_view(const kv_csr *c, int64_t *n_docs, const int64_t **indptr, const uint32_t **ids,
                const uint32_t **tf, const double **oov_tf2) {
  if (!c) return kv_fail(KV_ERR_INVALID, "kv_csr_view: NULL handle");
  if (n_docs) *n_docs = (int64_t)c->indptr.size() - 1;
  if (indptr) *indptr = c->indptr.data();
  if (ids) *ids = c->ids.data();
  if (tf) *tf = c->tf.data();
  if (oov_tf2) *oov_tf2 = c->oov.data();
  return KV_OK;
}

void kv_csr_destroy(kv_csr *c) { delete c; }

}  // extern "C"
