// Test-only C entry points around the three attention paths, so that tests/test_gpu_attention.py can run them on inputs
// it chooses:
//   - the frame-step kernel's attention phase (qwen3-tts_b200/csrc/ar_attention.cuh): attn_prefetch, a CTA-wide sync,
//     then attn_phase, the order q3_step_kernel uses around the grid barrier that precedes an attention phase;
//   - the prefill pair pf_qkv_post_kernel + pf_attention_kernel (ar_prefill.cuh), with prefill_rows' launch geometry;
//   - the codec decoder's rope_append_kernel + swa_stream_kernel (codec_kernels.cuh), with decode_frames' geometry.
// The package headers are included in ar_engine.cu's order.  Every KParams / Phase / StackDev field the attention phase
// reads is filled here from plain arguments, and the DevState layout is exported (attn_shim_layout), so Python never
// restates a struct.  Like sampler_shim.cu this file compiles its own copy of the kernels from the shipped source under
// the library's flags and links against nothing.
#include "common.cuh"
#include "gemm_sm90.cuh"
#include "../../include/qwen3tts_b200.h"

#include <stddef.h>

#include "ar_ring.cuh"
#include "ar_program.cuh"
#include "ar_gemv.cuh"
#include "ar_attention.cuh"
#include "ar_sampler.cuh"
#include "ar_prefill.cuh"
#include "codec_kernels.cuh"

namespace {
// The engine runs the phase on its x area, which is at least X_MIN_BYTES (>= ATT_SMEM); the shim gives it the same.
constexpr int SHIM_ATT_SMEM = X_MIN_BYTES;
static_assert(SHIM_ATT_SMEM >= ATT_SMEM, "attention shared memory");

__global__ void __launch_bounds__(NTHREADS, 1) attn_shim_kernel(const __grid_constant__ KParams P, const Phase ph, int frame) {
  extern __shared__ __align__(1024) unsigned char smem[];
  attn_prefetch(ph, P, smem, frame);
  cta_sync();
  attn_phase<false>(ph, P, smem, frame);
}
}  // namespace

// Sizes and limits the test needs; -1 for an unknown name.
extern "C" long long attn_shim_layout(const char* name) {
  const std::string n(name);
  if (n == "sizeof") return (long long)sizeof(DevState);
  if (n == "split_cnt") return (long long)offsetof(DevState, split_cnt);
  if (n == "split_cnt_len") return (long long)(sizeof(DevState::split_cnt) / sizeof(unsigned int));
  if (n == "att_smem") return ATT_SMEM;
  if (n == "kvwin") return KVWIN;
  if (n == "maxsplit") return MAXSPLIT;
  if (n == "rmax") return RMAX;
  if (n == "maxb") return MAXB;
  if (n == "hd") return HD;
  return -1;
}

// One attention phase over `grid` CTAs: layer `layer` of the talker (stack 0) or code-predictor (stack 1) cache.
// seqmode 1 (SEQ_DECODE): row b's context is max(1, min(len0[b] + frame + 1, cap)); seqmode 0 (SEQ_CP): nq query
// tokens at context ctx_end, column b + j*B of qkv / attn for token j.  Device pointers as in StackDev / KParams.
extern "C" int attn_shim_phase(int grid, int B, const int* len0, int max_len0, void* state, float* split_buf, int stack,
                               int nh, int nkv, int layers, int cap, float eps, void* qkv, void* attn, void* kc, void* vc,
                               const void* rope_cos, const void* rope_sin, const void* qn, const void* kn, int layer,
                               int seqmode, int nq, int ctx_end, int frame, void* stream) {
  if (grid < 1 || B < 1 || B > MAXB || nkv < 1 || nh % nkv || nh / nkv > RMAX || B * nkv > MAXB * 16 || nq < 1 || nq > 2 ||
      (stack != 0 && stack != 1))
    return 1;
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(attn_shim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SHIM_ATT_SMEM) != cudaSuccess) return 3;
    attr = true;
  }
  KParams P{};
  P.st = static_cast<DevState*>(state);
  P.B = B;
  for (int b = 0; b < B; ++b) P.len0[b] = len0[b];
  P.max_len0 = max_len0;
  P.split_buf = split_buf;
  StackDev S{};
  S.nh = nh; S.nkv = nkv; S.layers = layers; S.cap = cap; S.eps = eps;
  S.qkv = static_cast<bf16*>(qkv);
  S.attn = static_cast<bf16*>(attn);
  S.kc = static_cast<bf16*>(kc);
  S.vc = static_cast<bf16*>(vc);
  S.rope_cos = static_cast<const bf16*>(rope_cos);
  S.rope_sin = static_cast<const bf16*>(rope_sin);
  (stack == 0 ? P.talker : P.cp) = S;
  Phase ph{};
  ph.type = PH_ATTN;
  ph.stack = stack;
  ph.layer = layer;
  ph.seqmode = seqmode;
  ph.nq = nq;
  ph.ctx_end = ctx_end;
  ph.qn = static_cast<const bf16*>(qn);
  ph.kn = static_cast<const bf16*>(kn);
  attn_shim_kernel<<<grid, NTHREADS, SHIM_ATT_SMEM, static_cast<cudaStream_t>(stream)>>>(P, ph, frame);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

// prefill_rows' per-layer attention: q/k norm + RoPE and the K/V cache write of `ntok` packed tokens (token i is position
// tok_pos[i] of cache slot tok_seq[i]), then causal attention of every token over its slot's cache rows [0, pos].
extern "C" int attn_shim_prefill(void* qkv, void* attn, int ntok, const int* tok_seq, const int* tok_pos, int nh, int nkv,
                                 const void* qn, const void* kn, float eps, const void* rope_cos, const void* rope_sin,
                                 void* kc, void* vc, int layer, int layers, int cap, void* stream) {
  if (ntok < 1 || nkv < 1 || nh % nkv) return 1;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  pf_qkv_post_kernel<<<(ntok * (nh + 2 * nkv) + 7) / 8, 256, 0, s>>>(
      static_cast<bf16*>(qkv), ntok, tok_seq, tok_pos, nh, nkv, static_cast<const bf16*>(qn), static_cast<const bf16*>(kn), eps,
      static_cast<const bf16*>(rope_cos), static_cast<const bf16*>(rope_sin), static_cast<bf16*>(kc), static_cast<bf16*>(vc),
      layer, layers, cap);
  pf_attention_kernel<<<(ntok * nh + 7) / 8, 256, 0, s>>>(static_cast<const bf16*>(qkv), static_cast<bf16*>(attn), ntok,
                                                          tok_seq, tok_pos, nh, nkv, static_cast<const bf16*>(kc),
                                                          static_cast<const bf16*>(vc), layer, layers, cap);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

// decode_frames' attention of one codec transformer layer on qkv [B][n][3*nh*hd].  kvbuf == nullptr: the one-shot view
// (keys and values are qkv's own k and v heads, every row at position 0 with all n frames; rp and hist are ignored).
// Otherwise the stream view: kvbuf is a window buffer [B][kv_bs_rows][2*nh*hd] whose first `hist` rows per batch row are
// history, and rp (device int32 [2][B]) holds every row's position and count.
extern "C" int attn_shim_codec(void* qkv, const void* rope_cos, const void* rope_sin, void* kvbuf, int B, int n, int nh, int hd,
                               const int* rp, int hist, int kv_bs_rows, void* out, int window, void* stream) {
  if (B < 1 || n < 1 || hd % 2 || hd > 64 || window > 96) return 1;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  bf16* q = static_cast<bf16*>(qkv);
  const bool one_shot = kvbuf == nullptr;
  bf16* kv = one_shot ? q + nh * hd : static_cast<bf16*>(kvbuf);
  const int ld = one_shot ? 3 * nh * hd : 2 * nh * hd;
  if (one_shot) { rp = nullptr; hist = 0; kv_bs_rows = n; }
  rope_append_kernel<<<296, 256, 0, s>>>(q, static_cast<const bf16*>(rope_cos), static_cast<const bf16*>(rope_sin),
                                         one_shot ? nullptr : kv, B, n, nh, hd, rp, hist, kv_bs_rows);
  swa_stream_kernel<<<(B * n * nh + 7) / 8, 256, 0, s>>>(q, kv, ld, kv_bs_rows, hist, static_cast<bf16*>(out), B, n, nh, hd,
                                                         window, rp);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
