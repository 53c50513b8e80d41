// Test-only C entry points around the streaming loudness normaliser's kernels (qwen3-tts_b200/csrc/loud_kernels.cuh),
// so that tests/test_gpu_loudness_kernels.py can run them on rows, records and counters it chooses instead of the ones a
// stream of pushes reaches.  The LoudJob array and the filter are built here from plain arrays, so Python never restates
// a struct.  Like the other shims this file compiles its own copy of the kernels from the shipped source under the
// library's flags and links against nothing.  Return codes: 0 ok, 1 arguments the library never passes, 2 a CUDA error.
#include "loud_kernels.cuh"

#include <vector>

namespace {
// per job: n_in (int64), row, count (int32) and target -> a device LoudJob array (freed by the caller)
LoudJob* upload_jobs(int n, const long long* n_in, const int* rows, const int* counts, const double* targets) {
  std::vector<LoudJob> h(n);
  for (int i = 0; i < n; ++i) h[i] = LoudJob{n_in[i], targets[i], rows[i], counts[i]};
  LoudJob* d = nullptr;
  if (cudaMalloc(&d, n * sizeof(LoudJob)) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, h.data(), n * sizeof(LoudJob), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
  return d;
}
}  // namespace

// one loud_kernel launch over n jobs as q3_loud_step_rows makes it; sos fp32 [12] on the host; x fp32 [rows][ld];
// st the rows' records [rows][Q3_LOUD_ROW_BYTES]; out fp32 [rows][cap]
extern "C" int loud_shim_step(int n, const long long* n_in, const int* rows, const int* counts, const double* targets,
                              const float* sos, const float* x, long long ld, void* st, float* out, long long cap) {
  if (n < 1) return 1;
  for (int i = 0; i < n; ++i)
    if (counts[i] < 1 || counts[i] > kLdMaxIn || counts[i] > cap || counts[i] > ld ||
        n_in[i] + counts[i] > (long long)kLdSeg * kLdMaxBlocks)
      return 1;
  LoudJob* jobs = upload_jobs(n, n_in, rows, counts, targets);
  if (!jobs) return 2;
  loud_kernel<<<n, kLdThreads>>>(jobs, loud_filter(sos), x, ld, (LoudRecord*)st, out, cap);
  const int rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
  cudaFree(jobs);
  return rc;
}

// one loud_move_kernel launch (dir 0 save, 1 load) over n listed rows, as q3_loud_save_rows / load_rows launch it
extern "C" int loud_shim_move(int n, const int* rows, const long long* n_in, const double* targets, void* st, void* rec,
                              int dir) {
  if (n < 1) return 1;
  std::vector<int> zero(n, 0);
  LoudJob* jobs = upload_jobs(n, n_in, rows, zero.data(), targets);
  if (!jobs) return 2;
  loud_move_kernel<<<n, kLdThreads>>>(jobs, (LoudRecord*)st, (LoudRecord*)rec, dir);
  const int rc = cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
  cudaFree(jobs);
  return rc;
}
