// Streaming look-ahead limiter (q3_limit_*): the client's volume at the codec's 24 kHz with peaks held at -1 dBFS, over
// many rows with their own gains and counters in one launch.
//
// Row gain g, u = g*x; a[n] = 1 where |u[n]| <= c = 10^(-1/20), else c/|u[n]|; b[m] = min a[m .. m+119] (5 ms
// look-ahead); s[n] = min(a[n], mean of b[n-119 .. n]) (a 5 ms attack ramp that reaches each peak's a at the peak);
// G[n] = min over m in [max(0, n-1200), n] of s[m] + (n-m)/1200 (a linear release of at most 50 ms); y = u*G.  Every
// output is a windowed min of the inputs around it, so outputs are computed independently, one per thread, with no
// recursion across them.  Output n reads inputs up to n + 119, so after n inputs a row has emitted max(0, n - 119) and
// an end emits the rest (x = 0 past the clip); the first pending output reads 1438 inputs back, so a row keeps its last
// Q3_LIMIT_HIST.  The history is double-buffered as the resampler's is: a launch reads the current half and writes the
// other.  Every output is computed by the same code whatever the push sizes were, so a streamed clip equals the
// one-shot bit for bit.
#include "common.cuh"
#include "dev_store.h"
#include "row_state.h"

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <vector>

#include "../../include/qwen3tts_b200.h"
#include "limit_kernels.cuh"

namespace {

long long emitted(long long n) { return n < kLimL - 1 ? 0 : n - (kLimL - 1); }

}  // namespace

struct q3_limiter {
  int rows = 0, max_in = 0, max_out = 0, device = 0;
  std::vector<float> gain;        // per row; 0 until the row is reset
  std::vector<int> cur;
  std::vector<long long> n_in;    // inputs since the row's reset; it has emitted emitted(n_in) outputs
  std::vector<LimitJob> jobs_h;
  std::vector<int> rows_h;
  float* hist = nullptr;          // [2][rows][kLimHist]
  LimitJob* jobs = nullptr;       // [rows]
  int* rows_dev = nullptr;        // [rows]
  DevStore store{"limiter"};
};

extern "C" int q3_limit_open(int32_t rows, int32_t max_in, int32_t max_out, int32_t device, q3_limiter** out) {
  Q3_REQUIRE(out, "null argument");
  Q3_REQUIRE(rows >= 1 && rows <= 4096, "rows %d outside [1, 4096]", rows);
  Q3_REQUIRE(max_in >= 1, "max_in %d must be positive", max_in);
  Q3_REQUIRE(max_out >= max_in + kLimL - 1, "max_out %d below %d, the most one push of %d inputs and its end emit",
             max_out, max_in + kLimL - 1, max_in);
  Q3_CUDA(cudaSetDevice(device));
  q3_limiter* s = new q3_limiter();
  s->rows = rows; s->max_in = max_in; s->max_out = max_out; s->device = device;
  s->gain.assign(rows, 0.f); s->cur.assign(rows, 0); s->n_in.assign(rows, 0);
  s->jobs_h.resize(rows); s->rows_h.resize(rows);
  int rc = s->store.alloc(&s->hist, (size_t)2 * rows * kLimHist, true);
  if (!rc) rc = s->store.alloc(&s->jobs, (size_t)rows, true);
  if (!rc) rc = s->store.alloc(&s->rows_dev, (size_t)rows, true);
  if (rc) { delete s; return 1; }
  *out = s;
  return 0;
}

extern "C" void q3_limit_close(q3_limiter* s) { delete s; }

static bool gain_ok(float g) { return std::isfinite(g) && g > 0.f; }

extern "C" int q3_limit_reset_rows(q3_limiter* s, int32_t n, const int32_t* rows_host, const float* gains_host) {
  Q3_REQUIRE(s, "null limiter");
  if (check_row_list(s->rows, n, rows_host, "reset", "limiter")) return 1;
  Q3_REQUIRE(n == 0 || gains_host, "null argument");
  for (int i = 0; i < n; ++i)
    Q3_REQUIRE(gain_ok(gains_host[i]), "row %d: gain %g is not a positive finite number", rows_host[i], gains_host[i]);
  // a fresh row reads no history (its first outputs read inputs from 0 on), so a reset is host state only
  for (int i = 0; i < n; ++i) {
    s->gain[rows_host[i]] = gains_host[i];
    s->n_in[rows_host[i]] = 0;
  }
  return 0;
}

extern "C" int q3_limit_step_rows(q3_limiter* s, const float* in_dev, int64_t ld, const int32_t* counts_host,
                                  const int32_t* end_host, float* out_dev, int32_t* nout_host, void* stream_) {
  Q3_REQUIRE(s && counts_host && end_host && nout_host, "null argument");
  const int R = s->rows;
  int blocks = 0;
  bool any_in = false, any_out = false;
  for (int r = 0; r < R; ++r) {
    const int c = counts_host[r], e = end_host[r];
    Q3_REQUIRE(c >= 0 && c <= s->max_in, "row %d: count %d outside [0, %d]", r, c, s->max_in);
    Q3_REQUIRE(c <= ld, "row %d: count %d exceeds the row stride %lld", r, c, (long long)ld);
    Q3_REQUIRE(s->gain[r] > 0.f || (c == 0 && !e), "row %d was never reset", r);
    any_in |= c > 0;
    LimitJob& jb = s->jobs_h[r];
    const long long n = s->n_in[r] + c;
    jb = LimitJob{s->n_in[r], emitted(s->n_in[r]), c, 0, e ? 1 : 0, s->cur[r], s->gain[r], 0};
    if (c == 0 && !e) continue;
    const long long nout = (e ? n : emitted(n)) - jb.out0;
    Q3_REQUIRE(nout >= 0 && nout <= s->max_out, "row %d: %lld outputs outside [0, %d]", r, nout, s->max_out);
    jb.nout = (int)nout;
    any_out |= nout > 0;
    blocks = std::max(blocks, (jb.nout + kLimTile - 1) / kLimTile + (c > 0 && !e ? kLimHistTiles : 0));
  }
  Q3_REQUIRE(!any_in || in_dev, "null input");
  Q3_REQUIRE(!any_out || out_dev, "null output");
  for (int r = 0; r < R; ++r) nout_host[r] = s->jobs_h[r].nout;
  if (blocks == 0) return 0;
  Q3_CUDA(cudaSetDevice(s->device));
  cudaStream_t st = (cudaStream_t)stream_;
  Q3_CUDA(cudaMemcpyAsync(s->jobs, s->jobs_h.data(), (size_t)R * sizeof(LimitJob), cudaMemcpyHostToDevice, st));
  limit_kernel<<<dim3(blocks, R), kLimThreads, 0, st>>>(s->jobs, in_dev, ld, s->hist, R, out_dev, s->max_out);
  Q3_CUDA(cudaGetLastError());
  for (int r = 0; r < R; ++r) {
    const LimitJob& jb = s->jobs_h[r];
    if (jb.count == 0 && !jb.end) continue;
    if (jb.end) {
      s->n_in[r] = 0;   // a new clip reads no history
    } else {
      s->cur[r] ^= 1;
      s->n_in[r] += jb.count;
    }
  }
  return 0;
}

static int move_rows(q3_limiter* s, int n, const int32_t* rows_host, void* rec, int dir, cudaStream_t st) {
  Q3_CUDA(cudaSetDevice(s->device));
  for (int i = 0; i < n; ++i) {
    const int r = rows_host[i];
    s->jobs_h[i] = LimitJob{s->n_in[r], 0, 0, 0, 0, s->cur[r], s->gain[r], 0};
    s->rows_h[i] = r;
  }
  Q3_CUDA(cudaMemcpyAsync(s->jobs, s->jobs_h.data(), (size_t)n * sizeof(LimitJob), cudaMemcpyHostToDevice, st));
  Q3_CUDA(cudaMemcpyAsync(s->rows_dev, s->rows_h.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  limit_move_kernel<<<n, kLimThreads, 0, st>>>(s->jobs, s->rows_dev, s->hist, s->rows, (LimitRecord*)rec, dir);
  Q3_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int q3_limit_save_rows(q3_limiter* s, int32_t n, const int32_t* rows_host, void* dst_dev, void* stream) {
  Q3_REQUIRE(s, "null limiter");
  if (check_row_list(s->rows, n, rows_host, "save", "limiter")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(dst_dev, "null argument");
  for (int i = 0; i < n; ++i) Q3_REQUIRE(s->gain[rows_host[i]] > 0.f, "save row %d was never reset", rows_host[i]);
  return move_rows(s, n, rows_host, dst_dev, 0, (cudaStream_t)stream);
}

extern "C" int q3_limit_load_rows(q3_limiter* s, int32_t n, const int32_t* rows_host, const void* src_dev, void* stream) {
  Q3_REQUIRE(s, "null limiter");
  if (check_row_list(s->rows, n, rows_host, "load", "limiter")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(src_dev, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Q3_CUDA(cudaSetDevice(s->device));
  std::vector<LimitRecord> rec;
  if (read_headers(rec, src_dev, n, offsetof(LimitRecord, hist), st)) return 1;
  for (int i = 0; i < n; ++i)
    Q3_REQUIRE(gain_ok(rec[i].gain) && rec[i].n_in >= 0, "load row %d: record %d is not a saved row of a limiter",
               rows_host[i], i);
  for (int i = 0; i < n; ++i) {
    s->gain[rows_host[i]] = rec[i].gain;
    s->n_in[rows_host[i]] = rec[i].n_in;
  }
  return move_rows(s, n, rows_host, const_cast<void*>(src_dev), 1, st);
}
