// Test-only C entry points that run programs of GEMV phases through the production frame-step kernel
// (qwen3-tts_b200/csrc/ar_step.cuh: q3_step_kernel<NT, VAR>), so that tests/test_gpu_gemv.py can check the GEMV phase on
// weights and inputs it chooses.  The package headers are included in ar_engine.cu's order; the program is planned with
// the engine's own host functions (assign_tiles, make_smem_plan, build_run_table, step_kernels_set_max_dyn_smem) and
// launched cooperatively as the engine's launch_program does.  The shim compiles its own copy of the kernel from the
// shipped source under the library's flags and links against nothing.
//
// Every argument is checked before anything is launched: a bad one returns 1 and the reason in gemv_shim_last_error(),
// so no test can reach a kernel trap or a grid-barrier timeout.
#include "common.cuh"
#include "gemm_sm90.cuh"
#include "../../include/qwen3tts_b200.h"

#include <stdarg.h>
#include <stddef.h>

thread_local std::string g_q3_err;
int q3_set_err(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_q3_err = buf;
  return 1;
}

#include "ar_ring.cuh"
#include "ar_program.cuh"
#include "ar_gemv.cuh"
#include "ar_attention.cuh"
#include "ar_sampler.cuh"
#include "ar_step.cuh"
#include "ar_prefill.cuh"

namespace {

bool aligned(const void* p, size_t a) { return ((uintptr_t)p % a) == 0; }

// the dynamic shared-memory budget of this copy of the kernels (set once, as q3_engine_finalize does)
int device_max_dyn_smem(int* out) {
  static int v = 0;
  if (!v && step_kernels_set_max_dyn_smem(&v)) return 1;
  *out = v;
  return 0;
}

// The GEMV phases of a program from per-phase arrays; only the fields the plan reads when pointers are null.
int make_program(int n, const void* const* w, const int* N, const int* K, const void* const* src, const int* src_ld,
                 const void* const* norm_w, const float* eps, void* const* dst, const int* dst_ld, const int* epi,
                 const int* ncmode, const void* const* bias, void* const* save_normed, int B, int nt,
                 std::vector<Phase>* prog) {
  Q3_REQUIRE(n >= 1 && n <= MAX_PHASES, "program of %d phases: need 1..%d", n, MAX_PHASES);
  Q3_REQUIRE(B >= 1 && B <= MAXB, "batch %d out of range [1, %d]", B, MAXB);
  Q3_REQUIRE(nt == 1 || nt == 2 || nt == 4, "batch class nt = %d must be 1, 2 or 4", nt);
  prog->assign(n, Phase{});
  for (int i = 0; i < n; ++i) {
    Phase& p = (*prog)[i];
    Q3_REQUIRE(N[i] > 0 && N[i] % 16 == 0, "phase %d: N = %d must be a positive multiple of 16", i, N[i]);
    Q3_REQUIRE(K[i] > 0 && K[i] % 32 == 0, "phase %d: K = %d must be a positive multiple of 32", i, K[i]);
    Q3_REQUIRE(N[i] / 16 < 65536, "phase %d: N = %d has too many tiles", i, N[i]);
    Q3_REQUIRE(ncmode[i] == NC_B || ncmode[i] == NC_2B, "phase %d: ncmode %d must be 0 (B columns) or 1 (2B)", i, ncmode[i]);
    const int nc = ncmode[i] == NC_B ? B : 2 * B;
    Q3_REQUIRE(nc <= MAXCOLS, "phase %d: %d columns exceed %d", i, nc, MAXCOLS);
    Q3_REQUIRE(nt * 8 >= nc, "phase %d: batch class nt = %d holds %d columns, the phase has nc = %d (nt < ceil(nc/8))", i, nt,
               nt * 8, nc);
    const bool normed = norm_w && norm_w[i];
    Q3_REQUIRE(!normed || K[i] <= 2048, "phase %d: normed input with K = %d > 2048", i, K[i]);
    p.type = PH_GEMV;
    p.epi = epi ? epi[i] : EPI_STORE;
    p.ncmode = ncmode[i];
    p.n_tiles = N[i] / 16;
    p.kb = K[i] / 32;
    p.norm_w = normed ? static_cast<const bf16*>(norm_w[i]) : nullptr;
    if (!w) continue;  // plan only
    Q3_REQUIRE(p.epi >= EPI_STORE && p.epi <= EPI_LOGITS, "phase %d: unknown epilogue %d", i, p.epi);
    const int rows = p.epi == EPI_SWIGLU ? N[i] / 2 : N[i];
    Q3_REQUIRE(w[i] && aligned(w[i], 16), "phase %d: packed weight pointer null or not 16-byte aligned", i);
    Q3_REQUIRE(src[i] && aligned(src[i], 16), "phase %d: src pointer null or not 16-byte aligned", i);
    Q3_REQUIRE(src_ld[i] >= K[i] && src_ld[i] % 8 == 0, "phase %d: src_ld = %d must be >= K = %d and a multiple of 8", i,
               src_ld[i], K[i]);
    Q3_REQUIRE(!normed || aligned(norm_w[i], 16), "phase %d: norm weight pointer not 16-byte aligned", i);
    Q3_REQUIRE(dst[i] && aligned(dst[i], p.epi == EPI_LOGITS ? 4 : 2), "phase %d: dst pointer null or unaligned", i);
    Q3_REQUIRE(dst_ld[i] >= rows, "phase %d: dst_ld = %d below the %d output rows", i, dst_ld[i], rows);
    const bool has_bias = bias && bias[i];
    Q3_REQUIRE(has_bias == (p.epi == EPI_BIAS), "phase %d: a bias goes with the BIAS epilogue and only with it", i);
    Q3_REQUIRE(!has_bias || aligned(bias[i], 2), "phase %d: bias pointer unaligned", i);
    const bool has_save = save_normed && save_normed[i];
    Q3_REQUIRE(!has_save || normed, "phase %d: save_normed needs a normed input", i);
    Q3_REQUIRE(!has_save || aligned(save_normed[i], 16), "phase %d: save_normed pointer not 16-byte aligned", i);
    p.w = static_cast<const uint4*>(w[i]);
    p.src = static_cast<const bf16*>(src[i]);
    p.src_ld = src_ld[i];
    p.eps = eps ? eps[i] : 0.f;
    p.dst = dst[i];
    p.dst_ld = dst_ld[i];
    p.bias = has_bias ? static_cast<const bf16*>(bias[i]) : nullptr;
    p.save_normed = has_save ? static_cast<bf16*>(save_normed[i]) : nullptr;
  }
  return 0;
}

}  // namespace

extern "C" const char* gemv_shim_last_error(void) { return g_q3_err.c_str(); }

// Sizes and offsets of the device state and the kernel's limits.  -1 for an unknown name.
extern "C" long long gemv_shim_layout(const char* name) {
  const std::string n(name);
  if (n == "sizeof_state") return (long long)sizeof(DevState);
  if (n == "bar_count") return (long long)offsetof(DevState, bar_count);
  if (n == "error") return (long long)offsetof(DevState, error);
  if (n == "step") return (long long)offsetof(DevState, step);
  if (n == "finished") return (long long)offsetof(DevState, finished);
  if (n == "sizeof_phase") return (long long)sizeof(Phase);
  if (n == "max_phases") return MAX_PHASES;
  if (n == "max_batch") return MAXB;
  if (n == "max_dyn_smem") {
    int v = 0;
    return device_max_dyn_smem(&v) ? -1 : v;
  }
  return -1;
}

// Packs a row-major bf16 [N][K] weight into the kernel's 1 KB blocks (pack_weight_kernel, as q3_engine_load_tensor does).
extern "C" int gemv_shim_pack(const void* src, void* dst, int N, int K, void* stream) {
  Q3_REQUIRE(N > 0 && N % 16 == 0 && K > 0 && K % 32 == 0, "pack: [%d][%d] must be [16a][32b]", N, K);
  Q3_REQUIRE(src && dst && aligned(src, 16) && aligned(dst, 16), "pack: pointers must be 16-byte aligned");
  pack_weight_kernel<<<1024, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const bf16*>(src), static_cast<uint4*>(dst),
                                                                          N, K);
  Q3_CUDA(cudaGetLastError());
  return 0;
}

// The shared-memory plan the engine would choose for GEMV phases of these shapes at batch B and class nt, within
// max_dyn_smem bytes (<= 0: the device budget).  staged[i] = phase i stages its input; plan_out = {slot_blocks,
// nslots, total, x_bytes}.
extern "C" int gemv_shim_plan(int n, const int* N, const int* K, const int* normed, const int* ncmode, int B, int nt,
                              int max_dyn_smem, int* staged, int* plan_out) {
  std::vector<const void*> nw(n > 0 ? n : 0);
  for (int i = 0; i < n; ++i) nw[i] = normed[i] ? reinterpret_cast<const void*>(16) : nullptr;
  std::vector<Phase> prog;
  if (make_program(n, nullptr, N, K, nullptr, nullptr, nw.data(), nullptr, nullptr, nullptr, nullptr, ncmode, nullptr, nullptr,
                   B, nt, &prog))
    return 1;
  int dev_max = 0;
  if (device_max_dyn_smem(&dev_max)) return 1;
  const int cap = max_dyn_smem > 0 ? std::min(max_dyn_smem, dev_max) : dev_max;
  SmemPlan pl;
  if (make_smem_plan(prog, B, nt, cap, &pl)) return 1;
  for (int i = 0; i < n; ++i) staged[i] = prog[i].staged;
  plan_out[0] = pl.slot_blocks; plan_out[1] = pl.nslots; plan_out[2] = pl.total; plan_out[3] = pl.x_bytes;
  return 0;
}

// One cooperative launch of q3_step_kernel<nt, var> over a program of n GEMV phases (per-phase arrays; norm_w, bias and
// save_normed entries may be null).  mode 0: one pass; mode 1: max_iters passes (DevState.step advances).  frame0[B],
// admit_mask, hid_out / hid_stride as in KParams.  prog_dev, runs_dev, off_dev and state are caller-owned device
// buffers of the given byte sizes (the state is read as is: the caller zeroes `finished`, sets `step`).
extern "C" int gemv_shim_run(int n, const void* const* w, const int* N, const int* K, const void* const* src, const int* src_ld,
                             const void* const* norm_w, const float* eps, void* const* dst, const int* dst_ld, const int* epi,
                             const int* ncmode, const void* const* bias, void* const* save_normed, int grid, int B, int nt,
                             int var, int mode, int max_iters, unsigned int admit_mask, const int* frame0, void* hid_out,
                             int hid_stride, int max_dyn_smem, void* prog_dev, long long prog_bytes, void* runs_dev,
                             long long runs_bytes, void* off_dev, long long off_bytes, void* state, void* stream_) {
  Q3_REQUIRE(w && N && K && src && src_ld && dst && dst_ld && ncmode && frame0 && state && prog_dev && runs_dev && off_dev,
             "null argument");
  std::vector<Phase> prog;
  if (make_program(n, w, N, K, src, src_ld, norm_w, eps, dst, dst_ld, epi, ncmode, bias, save_normed, B, nt, &prog)) return 1;
  Q3_REQUIRE(var == 0 || var == 1, "var = %d: only the production (0) and hidden-capture (1) instantiations", var);
  Q3_REQUIRE(mode == 0 || mode == 1, "mode = %d must be 0 or 1", mode);
  Q3_REQUIRE(max_iters >= 1 && max_iters <= 64, "max_iters = %d out of range [1, 64]", max_iters);
  Q3_REQUIRE(!hid_out || (var == 1 && hid_stride > 0 && aligned(hid_out, 16)),
             "hid_out needs var = 1, hid_stride > 0 and a 16-byte aligned pointer");
  Q3_REQUIRE(aligned(state, 16) && aligned(prog_dev, 16) && aligned(runs_dev, 16) && aligned(off_dev, 16),
             "device scratch pointers must be 16-byte aligned");
  int dev;
  Q3_CUDA(cudaGetDevice(&dev));
  int sms = 0;
  Q3_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  Q3_REQUIRE(grid >= 1 && grid <= sms, "grid = %d out of range [1, %d SMs]", grid, sms);
  int dev_max = 0;
  if (device_max_dyn_smem(&dev_max)) return 1;
  const int cap = max_dyn_smem > 0 ? std::min(max_dyn_smem, dev_max) : dev_max;
  SmemPlan plan;
  if (make_smem_plan(prog, B, nt, cap, &plan)) return 1;
  assign_tiles(prog, grid);
  const char* wbase = reinterpret_cast<const char*>(prog[0].w);
  for (const Phase& p : prog) wbase = std::min(wbase, reinterpret_cast<const char*>(p.w));
  std::vector<uint2> runs;
  std::vector<uint32_t> off;
  if (build_run_table(prog, grid, wbase, 0, &runs, &off)) return 1;
  Q3_REQUIRE((long long)(prog.size() * sizeof(Phase)) <= prog_bytes, "program needs %zu B of scratch, %lld given",
             prog.size() * sizeof(Phase), prog_bytes);
  Q3_REQUIRE((long long)((runs.size() + 8) * sizeof(uint2)) <= runs_bytes, "run table needs %zu B of scratch, %lld given",
             (runs.size() + 8) * sizeof(uint2), runs_bytes);
  Q3_REQUIRE((long long)(off.size() * sizeof(uint32_t)) <= off_bytes, "run offsets need %zu B of scratch, %lld given",
             off.size() * sizeof(uint32_t), off_bytes);
  const int ni = nt == 1 ? 0 : nt == 2 ? 1 : 2;
  const void* fn = kStepKernels[var][ni];
  int per_sm = 0;
  Q3_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, CTA_THREADS, (size_t)plan.total));
  Q3_REQUIRE(per_sm >= 1, "plan of %d B does not fit one CTA per SM", plan.total);

  KParams P{};
  P.prog = static_cast<const Phase*>(prog_dev);
  P.n_phases = n;
  P.mode = mode;
  P.max_iters = max_iters;
  P.st = static_cast<DevState*>(state);
  P.B = B;
  for (int b = 0; b < B; ++b) P.frame0[b] = frame0[b];
  P.admit_mask = admit_mask;
  P.hid_out = static_cast<bf16*>(hid_out);
  P.hid_stride = hid_out ? hid_stride : 0;
  P.keep_fraction = 0.5f;
  P.plan = plan;
  P.wbase = wbase;
  P.runs = static_cast<const uint2*>(runs_dev);
  P.run_off = static_cast<const uint32_t*>(off_dev);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Q3_CUDA(cudaMemcpyAsync(prog_dev, prog.data(), prog.size() * sizeof(Phase), cudaMemcpyHostToDevice, stream));
  Q3_CUDA(cudaMemcpyAsync(runs_dev, runs.data(), runs.size() * sizeof(uint2), cudaMemcpyHostToDevice, stream));
  Q3_CUDA(cudaMemcpyAsync(off_dev, off.data(), off.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
  Q3_CUDA(cudaMemsetAsync(&P.st->bar_count, 0, sizeof(unsigned int), stream));
  void* args[] = {&P};
  Q3_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(CTA_THREADS), args, (size_t)plan.total, stream));
  // the host vectors above die with this call: the copies must have left them
  Q3_CUDA(cudaStreamSynchronize(stream));
  return 0;
}
