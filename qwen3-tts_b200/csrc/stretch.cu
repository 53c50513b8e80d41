// Streaming WSOLA time-stretch (q3_stretch_*): the client's speaking rate at the codec's 24 kHz, pitch kept, over many
// rows with their own analysis hops and counters in one launch.
//
// Frame k of a clip sits at p_k = k*Ha + d_k, d_0 = 0, where d_k in [-240, 240] maximises the correlation of
// x[p_k .. p_k + 480) with the natural continuation x[p_{k-1} + 480 ..) of the previous frame; output block k is the
// overlap-add of frame k's first half and frame k-1's second half under a sin^2 window of 960 samples (block 0 is x
// itself).  Frame k needs inputs up to k*Ha + 1199, and the frames of a row follow one another, so one CTA runs a
// row's frames in order.  A row keeps its last Q3_STRETCH_HIST inputs, the windowed second half of its last frame and
// that frame's position on the device; its input count, hop and frames done stay on the host, so output counts need no
// sync.  Every frame is computed by the same code whatever the push sizes were, so a streamed clip equals the one-shot
// bit for bit.
#include "common.cuh"
#include "dev_store.h"
#include "row_state.h"

#include <algorithm>
#include <cstddef>
#include <vector>

#include "../../include/qwen3tts_b200.h"
#include "stretch_kernels.cuh"

namespace {

// frame k is done once input k*ha + 240 + 959 has arrived
long long frames_done(long long n, int ha) { return n < kStN + kStDelta ? 0 : (n - kStN - kStDelta) / ha + 1; }
long long total_out(long long n, int ha) { return (n * kStHs + ha - 1) / ha; }
size_t smem_bytes(int max_in) { return (size_t)(kStHist + max_in + kStPad) * sizeof(float); }

}  // namespace

struct q3_stretcher {
  int rows = 0, max_in = 0, max_out = 0, device = 0;
  bool window_set = false;
  std::vector<int> ha;          // per row; 0 until the row is reset
  std::vector<long long> n_in;  // inputs since the row's reset; it has done frames_done(n_in) frames
  std::vector<StretchJob> jobs_h;
  float* hist = nullptr;        // [rows][kStHist]
  float* tail = nullptr;        // [rows][480]
  long long* plast = nullptr;   // [rows]
  StretchJob* jobs = nullptr;   // [rows]
  const float* window = nullptr;
  DevStore store{"stretcher"};
};

extern "C" int q3_stretch_open(int32_t rows, int32_t max_in, int32_t max_out, int32_t device, q3_stretcher** out) {
  Q3_REQUIRE(out, "null argument");
  Q3_REQUIRE(rows >= 1 && rows <= 4096, "rows %d outside [1, 4096]", rows);
  Q3_REQUIRE(max_in >= 1 && max_in <= kStMaxIn, "max_in %d outside [1, %d]", max_in, kStMaxIn);
  const long long need = total_out((long long)max_in + 1199, kStDelta);
  Q3_REQUIRE(max_out >= need, "max_out %d below %lld, the most one push of %d inputs and its end emit at speed 0.5",
             max_out, need, max_in);
  Q3_CUDA(cudaSetDevice(device));
  // the attribute is the function's, shared by every stretcher: set it for the largest max_in any of them may have
  Q3_CUDA(cudaFuncSetAttribute(wsola_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes(kStMaxIn)));
  q3_stretcher* s = new q3_stretcher();
  s->rows = rows; s->max_in = max_in; s->max_out = max_out; s->device = device;
  s->ha.assign(rows, 0); s->n_in.assign(rows, 0);
  s->jobs_h.resize(rows);
  int rc = s->store.alloc(&s->hist, (size_t)rows * kStHist, true);
  if (!rc) rc = s->store.alloc(&s->tail, (size_t)rows * kStHs, true);
  if (!rc) rc = s->store.alloc(&s->plast, (size_t)rows, true);
  if (!rc) rc = s->store.alloc(&s->jobs, (size_t)rows, true);
  if (rc) { delete s; return 1; }
  *out = s;
  return 0;
}

extern "C" void q3_stretch_close(q3_stretcher* s) { delete s; }

extern "C" int q3_stretch_set_window(q3_stretcher* s, const float* window_dev) {
  Q3_REQUIRE(s && window_dev, "null argument");
  Q3_CUDA(cudaSetDevice(s->device));
  const int64_t shape[1] = {kStN};
  if (s->store.load("window", window_dev, shape, 1, DT_F32)) return 1;
  s->window = s->store.need<float>("window", kStN);
  if (!s->window) return 1;
  s->window_set = true;
  return 0;
}

extern "C" int q3_stretch_reset_rows(q3_stretcher* s, int32_t n, const int32_t* rows_host, const int32_t* hops_host) {
  Q3_REQUIRE(s, "null stretcher");
  if (check_row_list(s->rows, n, rows_host, "reset", "stretcher")) return 1;
  Q3_REQUIRE(n == 0 || hops_host, "null argument");
  for (int i = 0; i < n; ++i)
    Q3_REQUIRE(hops_host[i] >= kStDelta && hops_host[i] <= 2 * kStHs, "row %d: hop %d outside [%d, %d]", rows_host[i],
               hops_host[i], kStDelta, 2 * kStHs);
  // a fresh row reads none of its device state (frame 0 sits at 0, the first search reads from Ha - 240 >= 0)
  for (int i = 0; i < n; ++i) {
    s->ha[rows_host[i]] = hops_host[i];
    s->n_in[rows_host[i]] = 0;
  }
  return 0;
}

extern "C" int q3_stretch_step_rows(q3_stretcher* s, const float* in_dev, int64_t ld, const int32_t* counts_host,
                                    const int32_t* end_host, float* out_dev, int32_t* nout_host, void* stream_) {
  Q3_REQUIRE(s && counts_host && end_host && nout_host, "null argument");
  const int R = s->rows;
  int njobs = 0, max_count = 0;
  bool any_in = false, any_out = false;
  for (int r = 0; r < R; ++r) {
    const int c = counts_host[r], e = end_host[r];
    Q3_REQUIRE(c >= 0 && c <= s->max_in, "row %d: count %d outside [0, %d]", r, c, s->max_in);
    Q3_REQUIRE(c <= ld, "row %d: count %d exceeds the row stride %lld", r, c, (long long)ld);
    Q3_REQUIRE(s->ha[r] > 0 || (c == 0 && !e), "row %d was never reset", r);
    any_in |= c > 0;
    if (c == 0 && !e) continue;
    const int ha = s->ha[r];
    const long long n = s->n_in[r] + c, f0 = frames_done(s->n_in[r], ha);
    const long long upto = e ? total_out(n, ha) : kStHs * frames_done(n, ha);
    const long long f1 = e ? (upto + kStHs - 1) / kStHs : frames_done(n, ha);
    const long long nout = upto - kStHs * f0;
    Q3_REQUIRE(nout >= 0 && nout <= s->max_out, "row %d: %lld outputs outside [0, %d]", r, nout, s->max_out);
    s->jobs_h[njobs++] = StretchJob{s->n_in[r], f0, r, c, (int)(f1 - f0), (int)nout, e ? 1 : 0, ha};
    any_out |= nout > 0;
    max_count = std::max(max_count, c);
  }
  Q3_REQUIRE(!any_in || in_dev, "null input");
  Q3_REQUIRE(!any_out || out_dev, "null output");
  Q3_REQUIRE(njobs == 0 || s->window_set, "the window was never set");
  for (int r = 0; r < R; ++r) nout_host[r] = 0;
  for (int i = 0; i < njobs; ++i) nout_host[s->jobs_h[i].row] = s->jobs_h[i].nout;
  if (njobs == 0) return 0;
  Q3_CUDA(cudaSetDevice(s->device));
  cudaStream_t st = (cudaStream_t)stream_;
  Q3_CUDA(cudaMemcpyAsync(s->jobs, s->jobs_h.data(), (size_t)njobs * sizeof(StretchJob), cudaMemcpyHostToDevice, st));
  wsola_kernel<<<njobs, kStThreads, smem_bytes(max_count), st>>>(s->jobs, s->window, in_dev, ld, s->hist, s->tail,
                                                                 s->plast, out_dev, s->max_out);
  Q3_CUDA(cudaGetLastError());
  for (int i = 0; i < njobs; ++i) {
    const StretchJob& jb = s->jobs_h[i];
    s->n_in[jb.row] = jb.end ? 0 : jb.n_in + jb.count;
  }
  return 0;
}

static int move_rows(q3_stretcher* s, int n, const int32_t* rows_host, void* rec, int dir, cudaStream_t st) {
  Q3_CUDA(cudaSetDevice(s->device));
  for (int i = 0; i < n; ++i) {
    const int r = rows_host[i];
    s->jobs_h[i] = StretchJob{s->n_in[r], frames_done(s->n_in[r], s->ha[r]), r, 0, 0, 0, 0, s->ha[r]};
  }
  Q3_CUDA(cudaMemcpyAsync(s->jobs, s->jobs_h.data(), (size_t)n * sizeof(StretchJob), cudaMemcpyHostToDevice, st));
  stretch_move_kernel<<<n, kStThreads, 0, st>>>(s->jobs, s->hist, s->tail, s->plast, (StretchRecord*)rec, dir);
  Q3_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int q3_stretch_save_rows(q3_stretcher* s, int32_t n, const int32_t* rows_host, void* dst_dev, void* stream) {
  Q3_REQUIRE(s, "null stretcher");
  if (check_row_list(s->rows, n, rows_host, "save", "stretcher")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(dst_dev, "null argument");
  for (int i = 0; i < n; ++i) Q3_REQUIRE(s->ha[rows_host[i]] > 0, "save row %d was never reset", rows_host[i]);
  return move_rows(s, n, rows_host, dst_dev, 0, (cudaStream_t)stream);
}

extern "C" int q3_stretch_load_rows(q3_stretcher* s, int32_t n, const int32_t* rows_host, const void* src_dev,
                                    void* stream) {
  Q3_REQUIRE(s, "null stretcher");
  if (check_row_list(s->rows, n, rows_host, "load", "stretcher")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(src_dev, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Q3_CUDA(cudaSetDevice(s->device));
  std::vector<StretchRecord> rec;
  if (read_headers(rec, src_dev, n, offsetof(StretchRecord, tail), st)) return 1;
  for (int i = 0; i < n; ++i) {
    Q3_REQUIRE(rec[i].ha >= kStDelta && rec[i].ha <= 2 * kStHs && rec[i].n_in >= 0 &&
                   rec[i].frames == frames_done(rec[i].n_in, rec[i].ha),
               "load row %d: record %d is not a saved row of a stretcher", rows_host[i], i);
  }
  for (int i = 0; i < n; ++i) {
    s->ha[rows_host[i]] = rec[i].ha;
    s->n_in[rows_host[i]] = rec[i].n_in;
  }
  return move_rows(s, n, rows_host, const_cast<void*>(src_dev), 1, st);
}
