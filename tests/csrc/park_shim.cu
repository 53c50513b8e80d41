// Test-only C entry points around the parked-row kernel (row_move_kernel, ar_prefill.cuh), so that
// tests/test_gpu_row_move.py can run its gather (park) and scatter (resume) on buffers it chooses and check every byte.
// The shim owns one DevState whose per-row fields are copied in and out in the record's order (len0, finished,
// n_valid, n_gen, c0, trailing_len, cur[0..]); the RowMove argument is built here from plain arrays.  Like rows_shim.cu
// this file compiles its own copy of the kernel from the shipped source under the library's flags and links against
// nothing.  Return codes: 0 ok, 1 arguments the engine never passes, 2 a CUDA launch error.
#include "common.cuh"
#include "gemm_sm90.cuh"
#include "../../include/qwen3tts_b200.h"

#include <algorithm>
#include <stddef.h>

#include "ar_ring.cuh"
#include "ar_program.cuh"
#include "ar_gemv.cuh"
#include "ar_attention.cuh"
#include "ar_sampler.cuh"
#include "ar_prefill.cuh"

namespace {
DevState* shim_state() {
  static DevState* d = nullptr;
  if (!d && cudaMalloc(&d, sizeof(DevState)) != cudaSuccess) return nullptr;
  return d;
}
int* row_field(DevState& s, int b, int k) {
  int* p[6] = {s.len0, s.finished, s.n_valid, s.n_gen, s.c0, s.trailing_len};
  return k < 6 ? p[k] + b : &s.cur[b][k - 6];
}
}  // namespace

extern "C" int park_shim_row_ints(void) { return kRowInts; }
extern "C" int park_shim_row_spans(void) { return kRowSpans; }

// set = 1 writes vals[kRowInts] into row `slot` of the shim's DevState, set = 0 reads them back.  Synchronous.
extern "C" int park_shim_state(int set, int slot, int* vals) {
  DevState* d = shim_state();
  if (!d || slot < 0 || slot >= MAXB) return 1;
  if (cudaDeviceSynchronize() != cudaSuccess) return 2;
  DevState h;
  if (cudaMemcpy(&h, d, sizeof(DevState), cudaMemcpyDeviceToHost) != cudaSuccess) return 2;
  for (int k = 0; k < kRowInts; ++k) {
    if (set) *row_field(h, slot, k) = vals[k];
    else vals[k] = *row_field(h, slot, k);
  }
  if (set && cudaMemcpy(d, &h, sizeof(DevState), cudaMemcpyHostToDevice) != cudaSuccess) return 2;
  return 0;
}

// One park (resume = 0) or resume (resume = 1) of row `slot`: span s is chunks[s] 16-byte chunks at slot_ptrs[s] and
// rec_ptrs[s]; the talker caches kc / vc are [seq][lh][cap][HD] bf16, the record's K/V kv [2][lh][pos][HD]; ints is
// the record's int block (device).  `grid` blocks of 256 threads.
extern "C" int park_shim_row_move(int resume, void* const* slot_ptrs, void* const* rec_ptrs, const int* chunks, void* kc,
                                  void* vc, void* kv, int lh, int cap, int pos, int slot, int* ints, int grid, void* stream) {
  DevState* d = shim_state();
  if (!d || grid < 1 || pos < 0 || pos > cap || slot < 0 || slot >= MAXB) return 1;
  RowMove M{};
  for (int s = 0; s < kRowSpans; ++s)
    M.span[s] = RowSpan{static_cast<uint4*>(slot_ptrs[s]), static_cast<uint4*>(rec_ptrs[s]), chunks[s]};
  M.kc = static_cast<uint4*>(kc); M.vc = static_cast<uint4*>(vc); M.kv = static_cast<uint4*>(kv);
  M.lh = lh; M.cap = cap; M.pos = pos; M.slot = slot; M.ints = ints;
  // ar_engine.cu launch_row_move: min(work / 256, 8 * SMs) blocks of 256 threads; every grid covers every piece
  if (resume) row_move_kernel<true><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(M, d);
  else row_move_kernel<false><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(M, d);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
