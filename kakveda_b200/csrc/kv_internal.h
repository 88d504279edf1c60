// Shared internals of libkakveda_b200 (error reporting, small helpers).
#pragma once
#include "../../include/kakveda_b200.h"

#include <cstdarg>
#include <cstdio>
#include <vector>

// A featurised batch (kv_featurize, kv_featurize_device).
struct kv_csr {
  std::vector<int64_t> indptr;
  std::vector<uint32_t> ids, tf;
  std::vector<double> oov;
};

// The keys of the features with ids [lo, hi) into keys[2 * (id - lo)], keys[2 * (id - lo) + 1].  KV_ERR_STATE when one
// of them is not (yet) in the table: a featurize(grow = 1) or an import is running.  hi <= kv_vocab_size(v).
int vocab_export_range(const kv_vocab *v, int64_t lo, int64_t hi, uint64_t *keys);

// Records a thread-local message and returns `code` (so call sites read `return kv_fail(..)`).
int kv_fail(int code, const char *fmt, ...);
void kv_clear_error();

// Host threads for the parallel host stages: the hardware's, or KAKVEDA_B200_THREADS; 1..64.
int host_threads();
