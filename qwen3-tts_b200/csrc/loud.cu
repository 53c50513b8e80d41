// Streaming loudness normaliser (q3_loud_*): a gain towards the client's target integrated loudness (BS.1770 K-weighting,
// 100 ms segments, gated blocks) at the codec's 24 kHz, over many rows with their own targets and counters in one launch.
//
// The gain is decided while the audio streams: a sample of segment k takes a gain ramped from A_{k-2} to A_{k-1}, the
// gains measured when segments k-2 and k-1 completed, so no output waits for a later input (DESIGN §4.9).  A row's state
// lives on the device in its record layout (LoudRecord): the gains of its last two segments, the filter state, the last
// three segment sums, the partial segment's inputs and the clip's block mean squares.  One CTA per row with inputs reads
// and writes its own record, so the state needs no second half.  The filter runs over whole segments only, each in the
// same order whatever the pushes were, so a streamed clip equals the one-shot bit for bit.
#include "common.cuh"
#include "dev_store.h"
#include "row_state.h"

#include <cmath>
#include <cstddef>
#include <vector>

#include "../../include/qwen3tts_b200.h"
#include "loud_kernels.cuh"

struct q3_loudness {
  int rows = 0, max_in = 0, max_out = 0, device = 0;
  bool filter = false;
  LoudFilter f{};
  std::vector<double> target;     // per row; NaN until the row is reset
  std::vector<long long> n_in;    // inputs of the row's clip so far
  std::vector<LoudJob> jobs_h;
  LoudRecord* st = nullptr;       // [rows]
  LoudJob* jobs = nullptr;        // [rows]
  DevStore store{"loudness"};
};

static bool target_ok(double t) { return std::isfinite(t); }

extern "C" int q3_loud_open(int32_t rows, int32_t max_in, int32_t max_out, int32_t device, q3_loudness** out) {
  Q3_REQUIRE(out, "null argument");
  Q3_REQUIRE(rows >= 1 && rows <= 4096, "rows %d outside [1, 4096]", rows);
  Q3_REQUIRE(max_in >= 1 && max_in <= kLdMaxIn, "max_in %d outside [1, %d]", max_in, kLdMaxIn);
  Q3_REQUIRE(max_out >= max_in, "max_out %d below max_in %d", max_out, max_in);
  Q3_CUDA(cudaSetDevice(device));
  q3_loudness* s = new q3_loudness();
  s->rows = rows; s->max_in = max_in; s->max_out = max_out; s->device = device;
  s->target.assign(rows, NAN); s->n_in.assign(rows, 0);
  s->jobs_h.resize(rows);
  int rc = s->store.alloc(&s->st, (size_t)rows, true);
  if (!rc) rc = s->store.alloc(&s->jobs, (size_t)rows, true);
  if (rc) { delete s; return 1; }
  *out = s;
  return 0;
}

extern "C" void q3_loud_close(q3_loudness* s) { delete s; }

extern "C" int q3_loud_set_filter(q3_loudness* s, const float* sos) {
  Q3_REQUIRE(s && sos, "null argument");
  for (int i = 0; i < 12; ++i) Q3_REQUIRE(std::isfinite(sos[i]), "sos[%d] = %g is not finite", i, sos[i]);
  Q3_REQUIRE(sos[3] == 1.f && sos[9] == 1.f, "a0 of each section must be 1");
  s->f = loud_filter(sos);
  s->filter = true;
  return 0;
}

extern "C" int q3_loud_reset_rows(q3_loudness* s, int32_t n, const int32_t* rows_host, const double* targets_host) {
  Q3_REQUIRE(s, "null loudness normaliser");
  if (check_row_list(s->rows, n, rows_host, "reset", "loudness normaliser")) return 1;
  Q3_REQUIRE(n == 0 || targets_host, "null argument");
  for (int i = 0; i < n; ++i)
    Q3_REQUIRE(target_ok(targets_host[i]), "row %d: target %g is not finite", rows_host[i], targets_host[i]);
  // a fresh row (n_in = 0) reads nothing of its record, so a reset is host state only
  for (int i = 0; i < n; ++i) {
    s->target[rows_host[i]] = targets_host[i];
    s->n_in[rows_host[i]] = 0;
  }
  return 0;
}

extern "C" int q3_loud_step_rows(q3_loudness* s, const float* in_dev, int64_t ld, const int32_t* counts_host,
                                 const int32_t* end_host, float* out_dev, int32_t* nout_host, void* stream_) {
  Q3_REQUIRE(s && counts_host && end_host && nout_host, "null argument");
  Q3_REQUIRE(s->filter, "the K-weighting filter is not set");
  const int R = s->rows;
  int jobs = 0;
  for (int r = 0; r < R; ++r) {
    const int c = counts_host[r], e = end_host[r];
    Q3_REQUIRE(c >= 0 && c <= s->max_in, "row %d: count %d outside [0, %d]", r, c, s->max_in);
    Q3_REQUIRE(c <= ld, "row %d: count %d exceeds the row stride %lld", r, c, (long long)ld);
    Q3_REQUIRE(target_ok(s->target[r]) || (c == 0 && !e), "row %d was never reset", r);
    Q3_REQUIRE(s->n_in[r] + c <= (long long)kLdSeg * kLdMaxBlocks,
               "row %d: a clip of %lld samples passes the %d segments a row measures", r, s->n_in[r] + c, kLdMaxBlocks);
    if (c > 0) s->jobs_h[jobs++] = LoudJob{s->n_in[r], s->target[r], r, c};
  }
  Q3_REQUIRE(jobs == 0 || in_dev, "null input");
  Q3_REQUIRE(jobs == 0 || out_dev, "null output");
  for (int r = 0; r < R; ++r) nout_host[r] = counts_host[r];
  if (jobs > 0) {
    Q3_CUDA(cudaSetDevice(s->device));
    cudaStream_t st = (cudaStream_t)stream_;
    Q3_CUDA(cudaMemcpyAsync(s->jobs, s->jobs_h.data(), (size_t)jobs * sizeof(LoudJob), cudaMemcpyHostToDevice, st));
    loud_kernel<<<jobs, kLdThreads, 0, st>>>(s->jobs, s->f, in_dev, ld, s->st, out_dev, s->max_out);
    Q3_CUDA(cudaGetLastError());
  }
  for (int r = 0; r < R; ++r)
    s->n_in[r] = end_host[r] ? 0 : s->n_in[r] + counts_host[r];   // an ended row's next clip reads nothing
  return 0;
}

static int move_rows(q3_loudness* s, int n, const int32_t* rows_host, void* rec, int dir, cudaStream_t st) {
  Q3_CUDA(cudaSetDevice(s->device));
  for (int i = 0; i < n; ++i) {
    const int r = rows_host[i];
    s->jobs_h[i] = LoudJob{s->n_in[r], s->target[r], r, 0};
  }
  Q3_CUDA(cudaMemcpyAsync(s->jobs, s->jobs_h.data(), (size_t)n * sizeof(LoudJob), cudaMemcpyHostToDevice, st));
  loud_move_kernel<<<n, kLdThreads, 0, st>>>(s->jobs, s->st, (LoudRecord*)rec, dir);
  Q3_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int q3_loud_save_rows(q3_loudness* s, int32_t n, const int32_t* rows_host, void* dst_dev, void* stream) {
  Q3_REQUIRE(s, "null loudness normaliser");
  if (check_row_list(s->rows, n, rows_host, "save", "loudness normaliser")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(dst_dev, "null argument");
  for (int i = 0; i < n; ++i)
    Q3_REQUIRE(target_ok(s->target[rows_host[i]]), "save row %d was never reset", rows_host[i]);
  return move_rows(s, n, rows_host, dst_dev, 0, (cudaStream_t)stream);
}

extern "C" int q3_loud_load_rows(q3_loudness* s, int32_t n, const int32_t* rows_host, const void* src_dev, void* stream) {
  Q3_REQUIRE(s, "null loudness normaliser");
  if (check_row_list(s->rows, n, rows_host, "load", "loudness normaliser")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(src_dev, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Q3_CUDA(cudaSetDevice(s->device));
  std::vector<LoudRecord> rec;   // only the headers are read back
  if (read_headers(rec, src_dev, n, offsetof(LoudRecord, part), st)) return 1;
  for (int i = 0; i < n; ++i)
    Q3_REQUIRE(target_ok(rec[i].target) && rec[i].n_in >= 0 && rec[i].n_in <= (long long)kLdSeg * kLdMaxBlocks,
               "load row %d: record %d is not a saved row of a loudness normaliser", rows_host[i], i);
  for (int i = 0; i < n; ++i) {
    s->target[rows_host[i]] = rec[i].target;
    s->n_in[rows_host[i]] = rec[i].n_in;
  }
  return move_rows(s, n, rows_host, const_cast<void*>(src_dev), 1, st);
}
