// Test-only C entry points around the streaming resampler's kernels (qwen3-tts_b200/csrc/resample_kernels.cuh), so
// that tests/test_gpu_resample_kernels.py can run them on rows, histories and counters it chooses instead of the ones
// a stream of pushes reaches.  The RowJob and FilterTable arguments are built here from plain arrays, so Python never
// restates a struct.  Like the other shims this file compiles its own copy of the kernels from the shipped source under
// the library's flags and links against nothing.  Return codes: 0 ok, 1 arguments the library never passes, 2 a CUDA
// error.
#include "resample_kernels.cuh"

#include <algorithm>
#include <vector>

namespace {
// per row: n_in, out0 (int64) and count, nout, end, fid, enc, cur (int32) -> a device RowJob array (freed by the caller)
RowJob* upload_jobs(int rows, const long long* n_in, const long long* out0, const int* f) {
  std::vector<RowJob> h(rows);
  for (int r = 0; r < rows; ++r)
    h[r] = RowJob{n_in[r], out0[r], f[6 * r], f[6 * r + 1], f[6 * r + 2], f[6 * r + 3], f[6 * r + 4], f[6 * r + 5]};
  RowJob* d = nullptr;
  if (cudaMalloc(&d, rows * sizeof(RowJob)) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, h.data(), rows * sizeof(RowJob), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
  return d;
}
}  // namespace

// one resample_poly_kernel launch with the geometry q3_resample_step_rows uses; filters: nf device tap pointers with
// their up / down / hl; x fp32 [rows][ld]; hist fp32 [2][rows][Q3_RESAMPLE_HIST]; out bytes [rows][cap]
extern "C" int resample_shim_poly(int nf, const float* const* taps, const int* up, const int* down, const int* hl, int rows,
                                  const long long* n_in, const long long* out0, const int* fields, const float* x,
                                  long long ld, float* hist, void* out, long long cap) {
  if (nf < 1 || nf > kMaxFilters || rows < 1) return 1;
  FilterTable ft{};
  for (int i = 0; i < nf; ++i) ft.f[i] = Filter{taps[i], up[i], down[i], hl[i]};
  int work = 0;
  for (int r = 0; r < rows; ++r) work = std::max(work, fields[6 * r + 1] + kHist);
  RowJob* jobs = upload_jobs(rows, n_in, out0, fields);
  if (!jobs) return 2;
  resample_poly_kernel<<<dim3((work + kThreads - 1) / kThreads, rows), kThreads>>>(ft, jobs, x, ld, hist, rows,
                                                                                   (uint8_t*)out, cap);
  const int rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
  cudaFree(jobs);
  return rc;
}

// one resample_move_kernel launch (dir 0 save, 1 load) over n listed rows, as q3_resample_save_rows / load_rows launch it
extern "C" int resample_shim_move(int n, const int* rows_host, const long long* n_in, const int* fields, float* hist,
                                  int rows, void* rec, int dir) {
  if (n < 1 || n > rows) return 1;
  RowJob* jobs = upload_jobs(n, n_in, n_in, fields);
  int* rd = nullptr;
  if (!jobs || cudaMalloc(&rd, n * sizeof(int)) != cudaSuccess) return 2;
  cudaMemcpy(rd, rows_host, n * sizeof(int), cudaMemcpyHostToDevice);
  resample_move_kernel<<<n, kHist>>>(jobs, rd, hist, rows, (RowRecord*)rec, dir);
  const int rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
  cudaFree(jobs);
  cudaFree(rd);
  return rc;
}
