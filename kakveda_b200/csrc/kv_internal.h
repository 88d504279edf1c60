// Shared internals of libkakveda_b200 (error reporting, small helpers).
#pragma once
#include "../../include/kakveda_b200.h"

#include <cstdarg>
#include <cstdio>

// Records a thread-local message and returns `code` (so call sites read `return kv_fail(..)`).
int kv_fail(int code, const char *fmt, ...);
void kv_clear_error();

// Host threads for the parallel host stages: the hardware's, or KAKVEDA_B200_THREADS; 1..64.
int host_threads();
