// CPU check (no GPU needed) of the per-block two-choice rare tables build_blocks writes (block_builder.cuh, pass 3):
//   1. every rare (block, feature) of the CSR sits in exactly one of its two slots, rt_slot1 or rt_slot2, with the exact
//      mask of the block's chunks holding it and the tf the bound kernel multiplies by (the block's largest tf, or the
//      feature's global largest tf once that reaches TF_OVF); no other key is present; the presence bitmap holds its bit;
//   2. the tables' offsets and sizes tile the slot array, at load factor <= 0.4;
//   3. the threaded build equals the sequential one byte for byte;
// on random corpora and on crafted ones: feature ids that share a first slot, or both slots, in one block (kicks and
// enlargements), ids next to FID_NONE, empty and padding blocks, and one block with tens of thousands of rare entries.
// Exit code 0 = all good.  Run by tests/test_host_rare_table.py.
#include "../../kakveda_b200/csrc/block_builder.cuh"

#include <cstdio>
#include <map>
#include <random>

using namespace kvh;

static int fails = 0;
#define CHECK(c, ...) do { if (!(c)) { if (fails < 20) { printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } fails++; } } while (0)

struct Corpus {
  std::vector<int64_t> indptr{0};
  std::vector<uint32_t> ids;
  std::vector<uint16_t> tf;
  std::vector<uint8_t> univ;
  std::vector<uint32_t> tfmax;
  std::vector<int> perm;
  int64_t n = 0, V = 0;
  void add_row(std::map<uint32_t, uint16_t> row) {
    for (auto &kv : row) {
      ids.push_back(kv.first);
      tf.push_back(kv.second);
    }
    indptr.push_back((int64_t)ids.size());
    n++;
  }
  void finish(int64_t vocab, unsigned seed) {
    V = vocab;
    univ.assign((size_t)V, 0);
    tfmax.assign((size_t)V, 0);
    for (size_t p = 0; p < ids.size(); p++) tfmax[ids[p]] = std::max<uint32_t>(tfmax[ids[p]], tf[p]);
    perm.resize((size_t)n);
    for (int64_t i = 0; i < n; i++) perm[(size_t)i] = (int)i;
    std::mt19937 rng(seed);
    std::shuffle(perm.begin(), perm.end(), rng);
  }
};

static void check_layout(const Corpus &c, const char *name) {
  BlockLayout L1, L4;
  build_blocks(c.indptr.data(), c.ids.data(), c.tf.data(), c.perm.data(), c.n, c.V, c.univ.data(), c.tfmax.data(), 1, L1, false);
  build_blocks(c.indptr.data(), c.ids.data(), c.tf.data(), c.perm.data(), c.n, c.V, c.univ.data(), c.tfmax.data(), 4, L4, false);
  CHECK(L1.rt_slots.size() == L4.rt_slots.size() &&
            memcmp(L1.rt_slots.data(), L4.rt_slots.data(), L1.rt_slots.size() * sizeof(uint4)) == 0 &&
            L1.rt_off == L4.rt_off && L1.rt_size == L4.rt_size && L1.rbloom == L4.rbloom && L1.rt_enlarged == L4.rt_enlarged,
        "%s: threaded build differs", name);
  CHECK(L1.rt_keys.empty() && L1.rt_masks.empty(), "%s: linear tables built without being asked for", name);
  const int64_t n_blocks = L1.n_chunks_pad / 64;
  CHECK((int64_t)L1.rt_off.size() == n_blocks && (int64_t)L1.rt_size.size() == n_blocks, "%s: table directory size", name);
  // 2: tiling
  int64_t at = 0;
  for (int64_t b = 0; b < n_blocks; b++) {
    CHECK(L1.rt_off[(size_t)b] == (uint32_t)at && L1.rt_size[(size_t)b] >= 4, "%s: table %lld offset / size", name, (long long)b);
    at += L1.rt_size[(size_t)b];
  }
  CHECK(at == (int64_t)L1.rt_slots.size(), "%s: tables do not tile the slot array", name);
  // what the tables must hold: per block, feature -> (mask, largest tf), from the CSR and the row order alone
  std::vector<std::map<uint32_t, std::pair<unsigned long long, uint32_t>>> want((size_t)n_blocks);
  for (int64_t pos = 0; pos < c.n; pos++) {
    const int64_t r = c.perm[(size_t)pos], ch = pos / 32, b = ch / 64;
    for (int64_t p = c.indptr[(size_t)r]; p < c.indptr[(size_t)r + 1]; p++) {
      const uint32_t f = c.ids[(size_t)p];
      if (L1.fslot[f] >= 0 || L1.fslot2[f] != 0xFFFF) continue;
      auto &e = want[(size_t)b][f];
      e.first |= 1ULL << (ch & 63);
      e.second = std::max<uint32_t>(e.second, c.tf[(size_t)p]);
    }
  }
  int64_t entries = 0;
  for (int64_t b = 0; b < n_blocks; b++) {
    const uint4 *tab = L1.rt_slots.data() + L1.rt_off[(size_t)b];
    const uint32_t size = L1.rt_size[(size_t)b];
    const auto &w = want[(size_t)b];
    entries += (int64_t)w.size();
    CHECK(w.size() == 0 || 5 * w.size() <= 2 * (size_t)size, "%s: block %lld above load 0.4", name, (long long)b);
    size_t keys = 0;
    for (uint32_t s = 0; s < size; s++) {
      if (tab[s].x == KEY_EMPTY) continue;
      keys++;
      const auto it = w.find(tab[s].x);
      CHECK(it != w.end(), "%s: block %lld holds feature %u that is not rare in it", name, (long long)b, tab[s].x);
      if (it != w.end()) CHECK(s == rt_slot1(tab[s].x, size) || s == rt_slot2(tab[s].x, size), "%s: feature %u outside its two slots", name, tab[s].x);
    }
    CHECK(keys == w.size(), "%s: block %lld holds %zu keys, %zu rare features", name, (long long)b, keys, w.size());
    for (const auto &kv : w) {
      const uint32_t f = kv.first, s1 = rt_slot1(f, size), s2 = rt_slot2(f, size);
      const int in = (tab[s1].x == f) + (s2 != s1 && tab[s2].x == f);
      CHECK(in == 1, "%s: feature %u of block %lld in %d of its slots", name, f, (long long)b, in);
      const uint4 e = tab[s1].x == f ? tab[s1] : tab[s2];
      const unsigned long long mask = (unsigned long long)e.z | ((unsigned long long)e.w << 32);
      const uint32_t tf_kernel = kv.second.second >= TF_OVF ? c.tfmax[f] : kv.second.second;
      CHECK(mask == kv.second.first, "%s: mask of feature %u in block %lld", name, f, (long long)b);
      CHECK(e.y == tf_kernel, "%s: tf of feature %u in block %lld: %u, want %u", name, f, (long long)b, e.y, tf_kernel);
      const uint32_t bb = rb_bit(f);
      CHECK((L1.rbloom[(size_t)b * (RB_BITS / 32) + (bb >> 5)] >> (bb & 31u)) & 1u, "%s: bitmap bit of feature %u", name, f);
    }
  }
  printf("%s: %lld rows, %lld blocks, %lld rare (block, feature) entries, %zu slots (%.1f B per entry), %lld tables enlarged\n",
         name, (long long)c.n, (long long)n_blocks, (long long)entries, L1.rt_slots.size(),
         entries ? 16.0 * (double)L1.rt_slots.size() / (double)entries : 0.0, (long long)L1.rt_enlarged);
}

// NF + NF2 features more widespread than any crafted one: they fill both dense classes, so that every crafted feature
// is rare (ids 0 .. NF + NF2 - 1, in 40 rows each)
constexpr uint32_t N_FILL = NF + NF2;
static void add_fillers(Corpus &c) {
  std::map<uint32_t, uint16_t> row;
  for (uint32_t f = 0; f < N_FILL; f++) row[f] = 1;
  for (int r = 0; r < 40; r++) c.add_row(row);
}

// a Zipf-like random corpus: a few common features, many rare ones, some tf beyond the 5-bit field
static Corpus random_corpus(int64_t n, int64_t V, unsigned seed) {
  Corpus c;
  std::mt19937 rng(seed);
  for (int64_t r = 0; r < n; r++) {
    std::map<uint32_t, uint16_t> row;
    const int len = (r % 13 == 4) ? 0 : 2 + (int)(rng() % 25);
    for (int j = 0; j < len; j++) {
      const uint32_t f = (rng() % 4 == 0) ? (uint32_t)(rng() % 30) : (uint32_t)(rng() % V);
      row[f] = (uint16_t)(rng() % 29 == 0 ? 31 + rng() % 500 : 1 + rng() % 4);
    }
    c.add_row(row);
  }
  c.finish(V, seed);
  return c;
}

// feature ids >= `from` with the same first slot (both = true: the same first AND second slot) in a table of `size`
static std::vector<uint32_t> colliding(uint32_t from, uint32_t size, bool both, size_t count) {
  std::vector<uint32_t> out;
  const uint32_t h1 = rt_slot1(from, size), h2 = rt_slot2(from, size);
  for (uint32_t f = from; out.size() < count && f < FID_NONE; f++)
    if (rt_slot1(f, size) == h1 && (!both || rt_slot2(f, size) == h2)) out.push_back(f);
  return out;
}

int main() {
  check_layout(random_corpus(1000, 5000, 1), "random-small");
  check_layout(random_corpus(9000, 200000, 2), "random-many-blocks");
  check_layout(random_corpus(31, 300, 3), "one-partial-chunk");
  {  // only empty rows: every table empty
    Corpus c;
    for (int r = 0; r < 70; r++) c.add_row({});
    c.finish(10, 4);
    check_layout(c, "empty-rows");
  }
  {  // one row holds 9 features sharing both slots and 9 sharing the first slot of its block's table at the initial
     // size: kicks, and enlargements (nine ids cannot share two slots)
    Corpus c;
    add_fillers(c);
    std::map<uint32_t, uint16_t> row;
    for (uint32_t f : colliding(5000, rt_initial_size(18), true, 9)) row[f] = 1;
    for (uint32_t f : colliding(9000000, rt_initial_size(18), false, 9)) row[f] = 2;
    CHECK(row.size() == 18, "could not craft the colliding ids");
    c.add_row(row);
    c.finish(FID_NONE - 1, 5);
    check_layout(c, "colliding-ids");
  }
  {  // three ids sharing both slots of the initial size force at least one enlargement
    Corpus c;
    add_fillers(c);
    std::vector<uint32_t> tri = colliding(5000, rt_initial_size(3), true, 3);
    CHECK(tri.size() == 3, "could not craft three ids sharing both slots");
    std::map<uint32_t, uint16_t> row;
    for (uint32_t f : tri) row[f] = 3;
    c.add_row(row);
    c.finish((int64_t)tri.back() + 1, 6);
    BlockLayout L;
    build_blocks(c.indptr.data(), c.ids.data(), c.tf.data(), c.perm.data(), c.n, c.V, c.univ.data(), c.tfmax.data(), 2, L, false);
    const int64_t b = std::find(c.perm.begin(), c.perm.end(), 40) - c.perm.begin();  // the crafted row's position
    CHECK(L.rt_enlarged >= 1 && L.rt_size[(size_t)(b / 2048)] > rt_initial_size(3), "three ids sharing both slots: no enlargement");
    check_layout(c, "forced-enlargement");
  }
  {  // ids next to FID_NONE, with large tf
    Corpus c;
    add_fillers(c);
    for (int r = 0; r < 100; r++) c.add_row({{FID_NONE - 1 - (uint32_t)(r % 7), (uint16_t)(1 + r % 40)}, {(uint32_t)r, 1}});
    c.finish(FID_NONE, 7);
    check_layout(c, "ids-near-FID_NONE");
  }
  {  // one block (2048 rows) with tens of thousands of rare entries
    Corpus c;
    add_fillers(c);
    std::mt19937 rng(8);
    for (int r = 0; r < 2000; r++) {
      std::map<uint32_t, uint16_t> row;
      for (int j = 0; j < 30; j++) row[(uint32_t)(2000 + r * 30 + j)] = (uint16_t)(1 + rng() % 3);
      c.add_row(row);
    }
    c.finish(2000 + 2000 * 30, 8);
    check_layout(c, "dense-block");
  }
  if (fails) { printf("%d check(s) failed\n", fails); return 1; }
  printf("all rare-table cases passed\n");
  return 0;
}
