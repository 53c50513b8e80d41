// Streaming polyphase resampler with an encoding epilogue (q3_resample_*): the rate conversion of
// scipy.signal.resample_poly (the reference's librosa.resample / resample_poly, qwen3_tts_tokenizer.py:156,204), one
// output sample per thread, over many rows with their own filters, encodings and counters in one launch.
//
// For a rate pair up/down with taps h[0..2*hl] (ntaps = 2*hl + 1), output j of a clip x[0..n) is
//   y[j] = sum over m of x[m] * h[hl + j*down - m*up],  0 <= m < n,  0 <= hl + j*down - m*up <= 2*hl,
// summed in fp32 in ascending m from the first product.  Output j needs inputs up to floor((hl + j*down) / up), so a row
// emits it as soon as that input has arrived; its earliest input is at least n_in - floor(2*hl / up) for the first
// output not yet emitted, so a row keeps its last kHist inputs.  The history is double-buffered: a launch reads the
// row's current half and writes the other, so the rows' histories need neither a second launch nor a host sync.  A row
// that ends its clip emits its remaining outputs with x = 0 past its end, and starts a new clip.  Every output is
// computed by the same loop whether its inputs came in one push or many, so a streamed clip equals the one-shot bit for
// bit.
#include "common.cuh"
#include "dev_store.h"
#include "row_state.h"

#include <algorithm>
#include <cstddef>
#include <vector>

#include "../../include/qwen3tts_b200.h"
#include "resample_kernels.cuh"

namespace {

long long emitted(long long n, int up, int down, int hl) {
  const long long a = n * up - 1 - hl;
  return a < 0 ? 0 : a / down + 1;
}
long long total_out(long long n, int up, int down) { return (n * up + down - 1) / down; }

}  // namespace

struct q3_resampler {
  int rows = 0, max_in = 0, max_out = 0, device = 0;
  std::vector<Filter> filters;
  std::vector<int> fid, enc, cur;  // per row; fid -1 until the row is reset
  std::vector<long long> n_in;  // inputs since the row's reset; it has emitted emitted(n_in) outputs
  std::vector<RowJob> jobs_h;
  std::vector<int> rows_h;
  float* hist = nullptr;      // [2][rows][kHist]
  RowJob* jobs = nullptr;     // [rows]
  int* rows_dev = nullptr;    // [rows]
  DevStore store{"resampler"};
};

extern "C" int q3_resample_open(int32_t rows, int32_t max_in, int32_t max_out, int32_t device, q3_resampler** out) {
  Q3_REQUIRE(out, "null argument");
  Q3_REQUIRE(rows >= 1 && rows <= 4096, "rows %d outside [1, 4096]", rows);
  Q3_REQUIRE(max_in >= 1 && max_out >= 1, "max_in %d and max_out %d must be positive", max_in, max_out);
  Q3_CUDA(cudaSetDevice(device));
  q3_resampler* s = new q3_resampler();
  s->rows = rows; s->max_in = max_in; s->max_out = max_out; s->device = device;
  s->fid.assign(rows, -1); s->enc.assign(rows, 0); s->cur.assign(rows, 0);
  s->n_in.assign(rows, 0);
  s->jobs_h.resize(rows); s->rows_h.resize(rows);
  int rc = s->store.alloc(&s->hist, (size_t)2 * rows * kHist, true);
  if (!rc) rc = s->store.alloc(&s->jobs, (size_t)rows, true);
  if (!rc) rc = s->store.alloc(&s->rows_dev, (size_t)rows, true);
  if (rc) { delete s; return 1; }
  *out = s;
  return 0;
}

extern "C" void q3_resample_close(q3_resampler* s) { delete s; }

// a filter id in use: added and not dropped (a dropped id keeps a null taps pointer until it is reused)
static bool filter_live(const q3_resampler* s, int id) {
  return id >= 0 && id < (int)s->filters.size() && s->filters[id].taps != nullptr;
}

extern "C" int q3_resample_add_filter(q3_resampler* s, int32_t up, int32_t down, const float* taps_dev, int32_t ntaps,
                                      int32_t* id_out) {
  Q3_REQUIRE(s && taps_dev && id_out, "null argument");
  int id = 0;
  while (id < (int)s->filters.size() && s->filters[id].taps) ++id;   // the lowest free id, reused after a drop
  Q3_REQUIRE(id < kMaxFilters, "a resampler holds at most %d filters", kMaxFilters);
  Q3_REQUIRE(up >= 1 && down >= 1, "up %d and down %d must be positive", up, down);
  Q3_REQUIRE(ntaps >= 1 && ntaps % 2 == 1, "a filter has an odd number of taps, got %d", ntaps);
  const int hl = ntaps / 2;
  Q3_REQUIRE(2 * hl / up <= kHist, "filter of %d taps at up %d reads %d past inputs, the history holds %d", ntaps, up,
             2 * hl / up, kHist);
  const long long worst = total_out(s->max_in, up, down) + (hl + down - 1) / down + 1;
  Q3_REQUIRE(worst <= s->max_out, "filter %d/%d may emit %lld samples per push of %d inputs, the rows hold %d", up, down,
             worst, s->max_in, s->max_out);
  Q3_CUDA(cudaSetDevice(s->device));
  const int64_t shape[1] = {ntaps};
  const std::string name = "filter." + std::to_string(id);
  if (s->store.load(name, taps_dev, shape, 1, DT_F32)) return 1;
  const float* p = s->store.need<float>(name, ntaps);
  if (!p) return 1;
  if (id == (int)s->filters.size()) s->filters.push_back(Filter{});
  s->filters[id] = Filter{p, up, down, hl};
  *id_out = id;
  return 0;
}

extern "C" int q3_resample_drop_filter(q3_resampler* s, int32_t id) {
  Q3_REQUIRE(s, "null resampler");
  Q3_REQUIRE(filter_live(s, id), "filter %d not added", id);
  for (int r = 0; r < s->rows; ++r) Q3_REQUIRE(s->fid[r] != id, "filter %d is in use by row %d", id, r);
  Q3_CUDA(cudaSetDevice(s->device));
  Q3_CUDA(cudaDeviceSynchronize());   // launches queued on any stream may still read its taps
  if (s->store.drop("filter." + std::to_string(id))) return 1;
  s->filters[id] = Filter{};
  return 0;
}

extern "C" int q3_resample_reset_rows(q3_resampler* s, int32_t n, const int32_t* rows_host, const int32_t* filters_host,
                                      const int32_t* encodings_host) {
  Q3_REQUIRE(s, "null resampler");
  if (check_row_list(s->rows, n, rows_host, "reset", "resampler")) return 1;
  Q3_REQUIRE(n == 0 || (filters_host && encodings_host), "null argument");
  for (int i = 0; i < n; ++i) {
    Q3_REQUIRE(filter_live(s, filters_host[i]), "row %d: filter %d not added", rows_host[i], filters_host[i]);
    Q3_REQUIRE(encodings_host[i] >= Q3_RESAMPLE_F32 && encodings_host[i] <= Q3_RESAMPLE_ULAW, "row %d: encoding %d unknown",
               rows_host[i], encodings_host[i]);
  }
  // a fresh row reads no history (its first outputs need inputs from 0 on), so a reset is host state only
  for (int i = 0; i < n; ++i) {
    const int r = rows_host[i];
    s->fid[r] = filters_host[i]; s->enc[r] = encodings_host[i];
    s->n_in[r] = 0;
  }
  return 0;
}

extern "C" int q3_resample_release_rows(q3_resampler* s, int32_t n, const int32_t* rows_host) {
  Q3_REQUIRE(s, "null resampler");
  if (check_row_list(s->rows, n, rows_host, "release", "resampler")) return 1;
  for (int i = 0; i < n; ++i) {
    s->fid[rows_host[i]] = -1;
    s->n_in[rows_host[i]] = 0;
  }
  return 0;
}

extern "C" int q3_resample_step_rows(q3_resampler* s, const float* in_dev, int64_t ld, const int32_t* counts_host,
                                     const int32_t* end_host, void* out_dev, int32_t* nout_host, void* stream_) {
  Q3_REQUIRE(s && counts_host && end_host && nout_host, "null argument");
  const int R = s->rows;
  int max_work = 0;
  bool any_in = false;
  for (int r = 0; r < R; ++r) {
    const int c = counts_host[r], e = end_host[r];
    Q3_REQUIRE(c >= 0 && c <= s->max_in, "row %d: count %d outside [0, %d]", r, c, s->max_in);
    Q3_REQUIRE(c <= ld, "row %d: count %d exceeds the row stride %lld", r, c, (long long)ld);
    Q3_REQUIRE(s->fid[r] >= 0 || (c == 0 && !e), "row %d was never reset", r);
    any_in |= c > 0;
    RowJob& jb = s->jobs_h[r];
    jb = RowJob{s->n_in[r], 0, c, 0, e ? 1 : 0, s->fid[r] < 0 ? 0 : s->fid[r], s->enc[r], s->cur[r]};
    if (s->fid[r] >= 0) {
      const Filter& f = s->filters[s->fid[r]];
      const long long n = s->n_in[r] + c;
      const long long upto = e ? total_out(n, f.up, f.down) : emitted(n, f.up, f.down, f.hl);
      jb.out0 = emitted(s->n_in[r], f.up, f.down, f.hl);
      jb.nout = (int)(upto - jb.out0);
      Q3_REQUIRE(jb.nout >= 0 && jb.nout <= s->max_out, "row %d: %d outputs outside [0, %d]", r, jb.nout, s->max_out);
    }
    if (c > 0 || e) max_work = std::max(max_work, jb.nout + kHist);
  }
  Q3_REQUIRE(!any_in || in_dev, "null input");
  Q3_REQUIRE(max_work == 0 || out_dev, "null output");
  for (int r = 0; r < R; ++r) nout_host[r] = s->jobs_h[r].nout;
  if (max_work == 0) return 0;
  Q3_CUDA(cudaSetDevice(s->device));
  cudaStream_t st = (cudaStream_t)stream_;
  Q3_CUDA(cudaMemcpyAsync(s->jobs, s->jobs_h.data(), (size_t)R * sizeof(RowJob), cudaMemcpyHostToDevice, st));
  FilterTable ft{};
  for (size_t i = 0; i < s->filters.size(); ++i) ft.f[i] = s->filters[i];
  const dim3 grid((max_work + kThreads - 1) / kThreads, R);
  resample_poly_kernel<<<grid, kThreads, 0, st>>>(ft, s->jobs, in_dev, ld, s->hist, R, (uint8_t*)out_dev,
                                             (long long)s->max_out * 4);
  Q3_CUDA(cudaGetLastError());
  for (int r = 0; r < R; ++r) {
    const RowJob& jb = s->jobs_h[r];
    if (jb.count == 0 && !jb.end) continue;
    s->cur[r] ^= 1;
    s->n_in[r] = jb.end ? 0 : s->n_in[r] + jb.count;
  }
  return 0;
}

static int move_rows(q3_resampler* s, int n, const int32_t* rows_host, void* rec, int dir, cudaStream_t st) {
  Q3_CUDA(cudaSetDevice(s->device));
  for (int i = 0; i < n; ++i) {
    const int r = rows_host[i];
    s->jobs_h[i] = RowJob{s->n_in[r], 0, 0, 0, 0, s->fid[r], s->enc[r], s->cur[r]};
    s->rows_h[i] = r;
  }
  Q3_CUDA(cudaMemcpyAsync(s->jobs, s->jobs_h.data(), (size_t)n * sizeof(RowJob), cudaMemcpyHostToDevice, st));
  Q3_CUDA(cudaMemcpyAsync(s->rows_dev, s->rows_h.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  resample_move_kernel<<<n, kHist, 0, st>>>(s->jobs, s->rows_dev, s->hist, s->rows, (RowRecord*)rec, dir);
  Q3_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int q3_resample_save_rows(q3_resampler* s, int32_t n, const int32_t* rows_host, void* dst_dev, void* stream) {
  Q3_REQUIRE(s, "null resampler");
  if (check_row_list(s->rows, n, rows_host, "save", "resampler")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(dst_dev, "null argument");
  for (int i = 0; i < n; ++i) Q3_REQUIRE(s->fid[rows_host[i]] >= 0, "save row %d was never reset", rows_host[i]);
  return move_rows(s, n, rows_host, dst_dev, 0, (cudaStream_t)stream);
}

extern "C" int q3_resample_load_rows(q3_resampler* s, int32_t n, const int32_t* rows_host, const void* src_dev, void* stream) {
  Q3_REQUIRE(s, "null resampler");
  if (check_row_list(s->rows, n, rows_host, "load", "resampler")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(src_dev, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Q3_CUDA(cudaSetDevice(s->device));
  std::vector<RowRecord> rec;
  if (read_headers(rec, src_dev, n, offsetof(RowRecord, hist), st)) return 1;
  for (int i = 0; i < n; ++i) {
    Q3_REQUIRE(filter_live(s, rec[i].fid) && rec[i].enc >= Q3_RESAMPLE_F32 &&
                   rec[i].enc <= Q3_RESAMPLE_ULAW && rec[i].n_in >= 0,
               "load row %d: record %d is not a saved row of this resampler", rows_host[i], i);
  }
  for (int i = 0; i < n; ++i) {
    const int r = rows_host[i];
    s->fid[r] = rec[i].fid; s->enc[r] = rec[i].enc; s->n_in[r] = rec[i].n_in;
  }
  return move_rows(s, n, rows_host, const_cast<void*>(src_dev), 1, st);
}
