// Test-only C entry points around the streaming time-stretch's kernels (qwen3-tts_b200/csrc/stretch_kernels.cuh), so
// that tests/test_gpu_stretch_kernels.py can run them on rows, histories, tails and counters it chooses instead of the
// ones a stream of pushes reaches.  The StretchJob array is built here from plain arrays, so Python never restates a
// struct.  Like the other shims this file compiles its own copy of the kernels from the shipped source under the
// library's flags and links against nothing.  Return codes: 0 ok, 1 arguments the library never passes, 2 a CUDA error.
#include "stretch_kernels.cuh"

#include <algorithm>
#include <vector>

namespace {
// per job: n_in, f0 (int64) and row, count, nf, nout, end, ha (int32) -> a device StretchJob array (freed by the caller)
StretchJob* upload_jobs(int n, const long long* n_in, const long long* f0, const int* f) {
  std::vector<StretchJob> h(n);
  for (int i = 0; i < n; ++i)
    h[i] = StretchJob{n_in[i], f0[i], f[6 * i], f[6 * i + 1], f[6 * i + 2], f[6 * i + 3], f[6 * i + 4], f[6 * i + 5]};
  StretchJob* d = nullptr;
  if (cudaMalloc(&d, n * sizeof(StretchJob)) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, h.data(), n * sizeof(StretchJob), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
  return d;
}
}  // namespace

// one wsola_kernel launch over n jobs with the geometry q3_stretch_step_rows uses; window fp32 [960]; x fp32
// [rows][ld]; hist fp32 [rows][Q3_STRETCH_HIST]; tail fp32 [rows][480]; plast int64 [rows]; out fp32 [rows][cap]
extern "C" int stretch_shim_wsola(int n, const long long* n_in, const long long* f0, const int* fields, const float* window,
                                  const float* x, long long ld, float* hist, float* tail, long long* plast, float* out,
                                  long long cap) {
  if (n < 1) return 1;
  int max_count = 0;
  for (int i = 0; i < n; ++i) max_count = std::max(max_count, fields[6 * i + 1]);
  if (max_count > kStMaxIn) return 1;
  const size_t smem = (size_t)(kStHist + max_count + kStPad) * sizeof(float);
  if (cudaFuncSetAttribute(wsola_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return 2;
  StretchJob* jobs = upload_jobs(n, n_in, f0, fields);
  if (!jobs) return 2;
  wsola_kernel<<<n, kStThreads, smem>>>(jobs, window, x, ld, hist, tail, plast, out, cap);
  const int rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
  cudaFree(jobs);
  return rc;
}

// one stretch_move_kernel launch (dir 0 save, 1 load) over n listed rows, as q3_stretch_save_rows / load_rows launch it
extern "C" int stretch_shim_move(int n, const long long* n_in, const long long* f0, const int* fields, float* hist,
                                 float* tail, long long* plast, void* rec, int dir) {
  if (n < 1) return 1;
  StretchJob* jobs = upload_jobs(n, n_in, f0, fields);
  if (!jobs) return 2;
  stretch_move_kernel<<<n, kStThreads>>>(jobs, hist, tail, plast, (StretchRecord*)rec, dir);
  const int rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
  cudaFree(jobs);
  return rc;
}
