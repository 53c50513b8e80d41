// Test-only C entry points around the streaming limiter's kernels (qwen3-tts_b200/csrc/limit_kernels.cuh), so that
// tests/test_gpu_limit_kernels.py can run them on rows, histories and counters it chooses instead of the ones a stream
// of pushes reaches.  The LimitJob array is built here from plain arrays, so Python never restates a struct.  Like the
// other shims this file compiles its own copy of the kernels from the shipped source under the library's flags and
// links against nothing.  Return codes: 0 ok, 1 arguments the library never passes, 2 a CUDA error.
#include "limit_kernels.cuh"

#include <algorithm>
#include <vector>

namespace {
// per row: n_in, out0 (int64), count, nout, end, cur (int32) and gain -> a device LimitJob array (freed by the caller)
LimitJob* upload_jobs(int n, const long long* n_in, const long long* out0, const int* f, const float* gain) {
  std::vector<LimitJob> h(n);
  for (int i = 0; i < n; ++i) h[i] = LimitJob{n_in[i], out0[i], f[4 * i], f[4 * i + 1], f[4 * i + 2], f[4 * i + 3], gain[i], 0};
  LimitJob* d = nullptr;
  if (cudaMalloc(&d, n * sizeof(LimitJob)) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, h.data(), n * sizeof(LimitJob), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
  return d;
}
}  // namespace

// one limit_kernel launch over every row with the geometry q3_limit_step_rows uses; x fp32 [rows][ld];
// hist fp32 [2][rows][Q3_LIMIT_HIST]; out fp32 [rows][cap]
extern "C" int limit_shim_step(int rows, const long long* n_in, const long long* out0, const int* fields,
                               const float* gain, const float* x, long long ld, float* hist, float* out, long long cap) {
  if (rows < 1) return 1;
  int blocks = 0;
  for (int r = 0; r < rows; ++r) {
    const int c = fields[4 * r], nout = fields[4 * r + 1], end = fields[4 * r + 2];
    if (nout > cap) return 1;
    blocks = std::max(blocks, (nout + kLimTile - 1) / kLimTile + (c > 0 && !end ? kLimHistTiles : 0));
  }
  if (blocks == 0) return 0;
  LimitJob* jobs = upload_jobs(rows, n_in, out0, fields, gain);
  if (!jobs) return 2;
  limit_kernel<<<dim3(blocks, rows), kLimThreads>>>(jobs, x, ld, hist, rows, out, cap);
  const int rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
  cudaFree(jobs);
  return rc;
}

// one limit_move_kernel launch (dir 0 save, 1 load) over n listed rows, as q3_limit_save_rows / load_rows launch it
extern "C" int limit_shim_move(int n, const int* rows_host, const long long* n_in, const int* fields, const float* gain,
                               float* hist, int rows, void* rec, int dir) {
  if (n < 1 || n > rows) return 1;
  LimitJob* jobs = upload_jobs(n, n_in, n_in, fields, gain);
  int* rd = nullptr;
  if (!jobs || cudaMalloc(&rd, n * sizeof(int)) != cudaSuccess) return 2;
  cudaMemcpy(rd, rows_host, n * sizeof(int), cudaMemcpyHostToDevice);
  limit_move_kernel<<<n, kLimThreads>>>(jobs, rd, hist, rows, (LimitRecord*)rec, dir);
  const int rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
  cudaFree(jobs);
  cudaFree(rd);
  return rc;
}
