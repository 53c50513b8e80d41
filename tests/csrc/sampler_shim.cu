// Test-only C entry points around the frame-step kernel's sample phase (qwen3-tts_b200/csrc/ar_sampler.cuh), so that
// tests/test_gpu_sampler.py can run it on logits it chooses.  The package headers are included in ar_engine.cu's order
// and the kernel below calls sample_phase() exactly as q3_step_kernel does: one CTA of NTHREADS per row, SAMPLER_SMEM
// bytes of dynamic shared memory.  Every KParams / Phase / q3_sampling field the phase reads is filled here from plain
// arguments, and the DevState layout is exported (sampler_shim_layout), so Python never restates a struct.
//
// Unlike tap_gemm_shim.cu this file compiles its own copy of the sample phase from the shipped source, under the
// library's flags; it links against nothing.  The instantiation inside q3_step_kernel is covered by
// tests/test_gpu_ar.py::test_sampler_against_oracle_on_engine_logits.
#include "common.cuh"
#include "gemm_sm90.cuh"
#include "../../include/qwen3tts_b200.h"

#include <stddef.h>

#include "ar_ring.cuh"
#include "ar_program.cuh"
#include "ar_gemv.cuh"
#include "ar_attention.cuh"
#include "ar_sampler.cuh"

namespace {
__global__ void __launch_bounds__(NTHREADS, 1) sampler_shim_kernel(const __grid_constant__ KParams P, const Phase ph,
                                                                     int frame, int in_prefill) {
  extern __shared__ __align__(1024) unsigned char smem[];
  sample_phase(ph, P, smem, frame, in_prefill != 0);
}
}  // namespace

// Sizes and offsets the test needs to read and write the device state: sizeof(DevState), offsetof its fields, the
// row stride of cur[][] and the kernel's limits.  -1 for an unknown name.
extern "C" long long sampler_shim_layout(const char* name) {
  const std::string n(name);
  if (n == "sizeof") return (long long)sizeof(DevState);
  if (n == "finished") return (long long)offsetof(DevState, finished);
  if (n == "n_valid") return (long long)offsetof(DevState, n_valid);
  if (n == "n_gen") return (long long)offsetof(DevState, n_gen);
  if (n == "c0") return (long long)offsetof(DevState, c0);
  if (n == "cur") return (long long)offsetof(DevState, cur);
  if (n == "cur_stride") return Q3_NUM_GROUPS_MAX;
  if (n == "max_batch") return MAXB;
  if (n == "max_vocab") return MAXV;
  return -1;
}

// One launch of the sample phase for rows 0..B-1 of phase `group` (0 = talker codebook 0, j >= 1 = code-predictor
// codebook j).  Host arrays: frame0, row_key, trailing_len [B].  Device pointers as in KParams (ar_program.cuh).
extern "C" int sampler_shim_run(int group, int B, int V, int Vc, int H, int G, int eos,
                                const float* talker_logits, const float* cp_logits, void* state,
                                const int* frame0, const unsigned int* row_key, unsigned int admit_mask,
                                const int* trailing_len,
                                int do_sample, int top_k, float top_p, float temperature, float repetition_penalty,
                                int subtalker_dosample, int subtalker_top_k, float subtalker_top_p,
                                float subtalker_temperature, int min_new_tokens, int suppress_eos,
                                unsigned long long seed,
                                unsigned char* seen, const void* emb_t, const void* emb_cp, void* x_cp,
                                const void* cp_next, void* cp_next_dst, int cp_next_w, const void* past_hidden,
                                const void* trailing, int trailing_stride, const void* tts_pad, void* talker_h,
                                int* codes_out, int codes_stride, const int* forced, int n_forced,
                                int frame, int in_prefill, void* stream) {
  if (B < 1 || B > MAXB || V > MAXV || Vc > MAXV || G > Q3_NUM_GROUPS_MAX || group < 0 || group >= G) return 1;
  KParams P{};
  P.st = static_cast<DevState*>(state);
  P.talker.vocab = V;
  P.talker.hidden = H;
  P.talker.logits = const_cast<float*>(talker_logits);
  P.talker.h = static_cast<bf16*>(talker_h);
  P.cp.vocab = Vc;
  P.cp.logits = const_cast<float*>(cp_logits);
  P.G = G;
  P.eos = eos;
  P.B = B;
  for (int b = 0; b < B; ++b) {
    P.frame0[b] = frame0[b];
    P.row_key[b] = row_key[b];
    P.trailing_len[b] = trailing_len[b];
  }
  P.admit_mask = admit_mask;
  q3_sampling sp{};
  sp.do_sample = do_sample;
  sp.top_k = top_k;
  sp.top_p = top_p;
  sp.temperature = temperature;
  sp.repetition_penalty = repetition_penalty;
  sp.subtalker_dosample = subtalker_dosample;
  sp.subtalker_top_k = subtalker_top_k;
  sp.subtalker_top_p = subtalker_top_p;
  sp.subtalker_temperature = subtalker_temperature;
  sp.min_new_tokens = min_new_tokens;
  sp.suppress_eos = suppress_eos;
  sp.seed = seed;
  P.sp = sp;
  P.emb_t = static_cast<const bf16*>(emb_t);
  P.emb_cp = static_cast<const bf16*>(emb_cp);
  P.x_cp = static_cast<bf16*>(x_cp);
  P.cp_next = static_cast<const bf16*>(cp_next);
  P.cp_next_dst = static_cast<bf16*>(cp_next_dst);
  P.cp_next_w = cp_next_w;
  P.past_hidden = static_cast<bf16*>(const_cast<void*>(past_hidden));
  P.trailing = static_cast<const bf16*>(trailing);
  P.trailing_stride = trailing_stride;
  P.tts_pad = static_cast<const bf16*>(tts_pad);
  P.seen = seen;
  P.codes_out = codes_out;
  P.codes_stride = codes_stride;
  P.forced = forced;
  P.n_forced = n_forced;
  Phase ph{};
  ph.type = PH_SAMPLE;
  ph.group = group;
  sampler_shim_kernel<<<B, NTHREADS, SAMPLER_SMEM, static_cast<cudaStream_t>(stream)>>>(P, ph, frame, in_prefill);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
