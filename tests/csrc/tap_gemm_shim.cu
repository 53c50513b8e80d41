// Test-only C entry points around the shipped tap-GEMM (qwen3-tts_b200/csrc/gemm_sm90.cu).  Every GemmPlan, GemmEpilogue
// and GemmViews field is a plain argument, so tests/test_gpu_tap_gemm.py can drive gemm_make_plan_v + gemm_launch through
// ctypes.  This file is linked against libqwen3tts_b200.so rather than compiled together with gemm_sm90.cu: the test runs
// the exact kernels the engine loads, and no second copy of the gemm_* / q3_set_err symbols exists in the process.
// Error text of a non-zero return is the library's q3_last_error().
#include "gemm_sm90.cuh"

extern "C" int tap_gemm_shim_init() { return gemm_init(); }

extern "C" int tap_gemm_shim_run(const void* a, int B, int T, int K, long long lda, long long a_bs, const void* w, int N,
                                 int Kp, int ntaps, const int* shifts, int bn, const float* bias, const float* scale,
                                 const void* resid, const float* snake_ea, const float* snake_ib, int cmod, int act,
                                 void* out_raw, void* out_act, int a_rows, int a_row0, long long raw_bs, long long act_bs,
                                 long long resid_bs, void* stream) {
  GemmEpilogue ep{};
  ep.bias = bias;
  ep.scale = scale;
  ep.resid = static_cast<const bf16*>(resid);
  ep.snake_ea = snake_ea;
  ep.snake_ib = snake_ib;
  ep.cmod = cmod;
  ep.act = act;
  ep.out_raw = static_cast<bf16*>(out_raw);
  ep.out_act = static_cast<bf16*>(out_act);
  GemmViews v;
  v.a_rows = a_rows;
  v.a_row0 = a_row0;
  v.raw_bs = raw_bs;
  v.act_bs = act_bs;
  v.resid_bs = resid_bs;
  GemmPlan plan;
  if (gemm_make_plan_v(&plan, static_cast<const bf16*>(a), B, T, K, lda, a_bs, static_cast<const bf16*>(w), N, Kp, ntaps,
                       shifts, bn, ep, v))
    return 1;
  return gemm_launch(plan, static_cast<cudaStream_t>(stream));
}
