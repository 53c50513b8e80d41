// Host-side checks and copies of the streaming engines with per-row state (the resampler, time-stretch, limiter and
// codec encoder stream).  Host-only.
#pragma once
#include "common.cuh"

#include <vector>

// a list of n rows of an owner of `rows` rows: n in [0, rows], every row in range and listed once.  `what` is the
// operation ("reset", "save", ...) and `owner` the owner's name ("resampler", ...), as the messages read them.
static inline int check_row_list(int rows, int n, const int32_t* list, const char* what, const char* owner) {
  Q3_REQUIRE(n >= 0 && n <= rows, "%d rows to %s, the %s has %d", n, what, owner, rows);
  Q3_REQUIRE(n == 0 || list, "null argument");
  for (int i = 0; i < n; ++i) {
    Q3_REQUIRE(list[i] >= 0 && list[i] < rows, "%s row %d out of range [0, %d)", what, list[i], rows);
    for (int j = 0; j < i; ++j) Q3_REQUIRE(list[i] != list[j], "%s row %d listed twice", what, list[i]);
  }
  return 0;
}

// the headers (the first `head_bytes` bytes: the fields before the record's device state) of the n records at src_dev,
// copied back to the host on `st` and waited for, so that a loaded row's counters size its outputs at every later step
// without a sync
template <class Record>
int read_headers(std::vector<Record>& rec, const void* src_dev, int n, size_t head_bytes, cudaStream_t st) {
  rec.resize(n);
  for (int i = 0; i < n; ++i)
    Q3_CUDA(cudaMemcpyAsync(&rec[i], (const Record*)src_dev + i, head_bytes, cudaMemcpyDeviceToHost, st));
  Q3_CUDA(cudaStreamSynchronize(st));
  return 0;
}
