// Test-only C entry points around the row-wise kernels that have no other direct test, so that
// tests/test_gpu_row_kernels.py can run them on inputs it chooses:
//   - the codec decoder's RVQ gather, RMSNorm, depthwise conv + LayerNorm, final conv and history roll / reset / copy
//     (qwen3-tts_b200/csrc/codec_kernels.cuh);
//   - the prefill's RMSNorm, token index, prefix index, last-row gather, release and bf16 -> fp32 widening
//     (ar_prefill.cuh);
//   - the streaming codec encoder's waveform load, replicate seed, code mask and history reset
//     (codec_encoder_kernels.cuh).
// Each kernel is launched with the geometry its engine uses (cited beside every launch).  The RollTable, CopyTable,
// EncRollTable, PfLens, PfRows, PfPrefix and SlotList arguments are built here from plain arrays, and the shim owns one
// DevState whose per-slot fields are copied in and out as int arrays, so Python never restates a struct.  Like
// attention_shim.cu this file compiles its own copy of the kernels from the shipped source under the library's flags
// and links against nothing.  Return codes: 0 ok, 1 arguments the engine never passes, 2 a CUDA launch error.
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
#include "codec_kernels.cuh"
#include "codec_encoder_kernels.cuh"

namespace {
int launched() { return cudaGetLastError() == cudaSuccess ? 0 : 2; }
cudaStream_t st(void* s) { return static_cast<cudaStream_t>(s); }

DevState* shim_state() {
  static DevState* d = nullptr;
  if (!d && cudaMalloc(&d, sizeof(DevState)) != cudaSuccess) return nullptr;
  return d;
}
constexpr int kStateFields = 6;  // finished, n_valid, n_gen, c0, len0, trailing_len
int* state_field(DevState& s, int f) {
  int* p[kStateFields] = {s.finished, s.n_valid, s.n_gen, s.c0, s.len0, s.trailing_len};
  return p[f];
}
}  // namespace

extern "C" int rows_shim_layout(const char* name) {
  const std::string n(name);
  if (n == "maxb") return MAXB;
  if (n == "hd") return HD;
  if (n == "roll_max") return kRollMax;
  if (n == "enc_roll_max") return kEncRollMax;
  return -1;
}

// The shim's DevState: set = 1 writes fields [6][MAXB] (finished, n_valid, n_gen, c0, len0, trailing_len) into it,
// set = 0 reads them back.  Synchronous on the default stream after the device has finished.
extern "C" int rows_shim_state(int set, int* fields) {
  DevState* d = shim_state();
  if (!d || cudaDeviceSynchronize() != cudaSuccess) return 2;
  DevState h;
  if (cudaMemcpy(&h, d, sizeof(DevState), cudaMemcpyDeviceToHost) != cudaSuccess) return 2;
  for (int f = 0; f < kStateFields; ++f) {
    int* p = state_field(h, f);
    for (int b = 0; b < MAXB; ++b) {
      if (set) p[b] = fields[f * MAXB + b];
      else fields[f * MAXB + b] = p[b];
    }
  }
  if (set && cudaMemcpy(d, &h, sizeof(DevState), cudaMemcpyHostToDevice) != cudaSuccess) return 2;
  return 0;
}

// ---------------------------------------------------------------------------------------------- codec decoder
extern "C" int rows_shim_rvq_gather(const int* codes, const void* table, void* e, int B, int K, int T, int D, int bins,
                                    const int* rp, void* stream) {
  // codec_engine.cu decode_frames: B * n blocks, 128 threads
  rvq_gather_kernel<<<B * T, 128, 0, st(stream)>>>(codes, static_cast<const bf16*>(table), static_cast<bf16*>(e), B, K, T, D,
                                                   bins, rp);
  return launched();
}

extern "C" int rows_shim_rmsnorm_rows(const void* x, const void* w, void* y, int rows, int C, float eps, void* stream) {
  // decode_frames: (rows + 7) / 8 blocks, 256 threads (one warp per row)
  rmsnorm_rows_kernel<<<(rows + 7) / 8, 256, 0, st(stream)>>>(static_cast<const bf16*>(x), static_cast<const bf16*>(w),
                                                              static_cast<bf16*>(y), rows, C, eps);
  return launched();
}

extern "C" int rows_shim_dwconv_ln(const void* x, const float* w, const float* bias, const float* lnw, const float* lnb, void* y,
                                   int B, int T, int C, int x_bs_rows, int hist, void* stream) {
  // decode_frames: B * Tc blocks, 256 threads, (Cl + 64) * 4 bytes
  dwconv_ln_kernel<<<B * T, 256, (C + 64) * sizeof(float), st(stream)>>>(static_cast<const bf16*>(x), w, bias, lnw, lnb,
                                                                         static_cast<bf16*>(y), B, T, C, x_bs_rows, hist);
  return launched();
}

extern "C" int rows_shim_final_conv(const void* x, const float* w, const float* bias, float* wav, int B, int T, int C, int x_bs_rows,
                                    int hist, const int* rp, int up, void* stream) {
  if (C % 8) return 1;
  // decode_frames: 1184 blocks, 256 threads (grid-stride over B * Tc samples)
  final_conv_kernel<<<1184, 256, 0, st(stream)>>>(static_cast<const bf16*>(x), w, bias, wav, B, T, C, x_bs_rows, hist, rp, up);
  return launched();
}

namespace {
int roll_table(RollTable* tb, void* const* p, const int* hist, const int* factor, const int* C, const int* bs_rows, int n) {
  if (n < 1 || n > kRollMax) return 1;
  tb->n = n;
  for (int i = 0; i < n; ++i) {
    if (C[i] % 16) return 1;
    tb->e[i] = RollEntry{static_cast<bf16*>(p[i]), hist[i], factor[i], C[i], bs_rows[i]};
  }
  return 0;
}
}  // namespace

// n history buffers {p, hist, factor, C, bs_rows}
extern "C" int rows_shim_roll(void* const* p, const int* hist, const int* factor, const int* C, const int* bs_rows, int n,
                              const int* rp, int B, void* stream) {
  RollTable tb{};
  if (roll_table(&tb, p, hist, factor, C, bs_rows, n)) return 1;
  // codec_engine.cu q3_codec_stream_step_rows: roll.n * B blocks, 128 threads
  roll_history_kernel<<<tb.n * B, 128, 0, st(stream)>>>(tb, rp, B);
  return launched();
}

extern "C" int rows_shim_reset(void* const* p, const int* hist, const int* factor, const int* C, const int* bs_rows, int n,
                               const int* rp, int B, void* stream) {
  RollTable tb{};
  if (roll_table(&tb, p, hist, factor, C, bs_rows, n)) return 1;
  // codec_engine.cu q3_codec_stream_reset_rows: tb.n * B blocks, 128 threads
  reset_history_kernel<<<tb.n * B, 128, 0, st(stream)>>>(tb, rp, B);
  return launched();
}

// n buffer pairs {dst, src, hist, C, dst_bs_rows, src_bs_rows}; rows[i] / rows[ld + i]: source / destination row of pair i
extern "C" int rows_shim_copy(void* const* dst, void* const* src, const int* hist, const int* C, const int* dst_bs_rows,
                              const int* src_bs_rows, int n, const int* rows, int ld, int pairs, void* stream) {
  if (n < 1 || n > kRollMax || pairs < 1 || pairs > ld) return 1;
  CopyTable tb{};
  tb.n = n;
  for (int i = 0; i < n; ++i) {
    if (C[i] % 16) return 1;
    tb.e[i] = CopyEntry{static_cast<bf16*>(dst[i]), static_cast<const bf16*>(src[i]), hist[i], C[i], dst_bs_rows[i], src_bs_rows[i]};
  }
  // codec_engine.cu q3_codec_stream_copy_rows: tb.n * n blocks, 256 threads
  copy_rows_kernel<<<tb.n * pairs, 256, 0, st(stream)>>>(tb, rows, ld, pairs);
  return launched();
}

// ---------------------------------------------------------------------------------------------- prefill
extern "C" int rows_shim_pf_rmsnorm(const void* x, const void* w, void* y, int rows, int C, float eps, void* stream) {
  if (C % 8) return 1;
  // ar_engine.cu prefill_layers: (ntok + rows_per_blk - 1) / rows_per_blk blocks (rows_per_blk = 8), 256 threads
  pf_rmsnorm_kernel<<<(rows + 7) / 8, 256, 0, st(stream)>>>(static_cast<const bf16*>(x), static_cast<const bf16*>(w),
                                                            static_cast<bf16*>(y), rows, C, eps);
  return launched();
}

// Admission of n packed rows into the shim's DevState: row r has lens[r] packed tokens and lives in slot slots[r];
// prefix_kv[r] (null: none) holds its p0[r]-position prefix K then V, [lh][p0[r]][HD] each; trailing_len[r] rows of
// trailing text [r][stride][H] in src go to dst [slot][cap][H].
extern "C" int rows_shim_pf_index(int n, const int* lens, const int* slots, const int* p0, const int* trailing_len,
                                  const void* src, void* dst, int stride, int cap, int H, const void* const* prefix_kv,
                                  void* kc, void* vc, int lh, int kcap, unsigned char* seen, int V, int* tok_seq, int* tok_pos,
                                  void* stream) {
  if (n < 1 || n > MAXB) return 1;
  DevState* d = shim_state();
  if (!d) return 2;
  PfLens pl{};
  PfRows pr{};
  PfPrefix px{};
  pl.B = n;
  pr.src = static_cast<const bf16*>(src); pr.dst = static_cast<bf16*>(dst); pr.stride = stride; pr.cap = cap; pr.H = H;
  px.kc = static_cast<uint4*>(kc); px.vc = static_cast<uint4*>(vc); px.lh = lh; px.cap = kcap;
  // prefill_rows: row_work = max(V, trailing_len * H, lh * p0 * (HD / 8) of a row with a prefix)
  int row_work = V;
  for (int r = 0; r < n; ++r) {
    if ((p0[r] > 0) != (prefix_kv[r] != nullptr)) return 1;  // the engine sets p0 exactly for the rows with a prefix
    pl.start[r + 1] = pl.start[r] + lens[r]; pl.slot[r] = slots[r];
    pr.trailing_len[r] = trailing_len[r];
    row_work = std::max(row_work, trailing_len[r] * H);
    if (prefix_kv[r]) {
      pl.p0[r] = p0[r];
      px.kv[r] = static_cast<const uint4*>(prefix_kv[r]);
      row_work = std::max(row_work, lh * p0[r] * (HD / 8));
    }
  }
  const int ntok = pl.start[n];
  // prefill_rows: dim3((max(ntok, row_work) + 255) / 256, n), 256 threads
  pf_index_kernel<<<dim3((std::max(ntok, row_work) + 255) / 256, n), 256, 0, st(stream)>>>(pl, pr, px, d, seen, V, tok_seq, tok_pos);
  return launched();
}

extern "C" int rows_shim_pf_prefix_index(int n, int* tok_seq, int* tok_pos, void* stream) {
  // ar_engine.cu q3_prefix_create: (len + 255) / 256 blocks, 256 threads
  pf_prefix_index_kernel<<<(n + 255) / 256, 256, 0, st(stream)>>>(n, tok_seq, tok_pos);
  return launched();
}

extern "C" int rows_shim_pf_gather_last(int n, const int* lens, const int* slots, const void* x, void* h_last, int H, void* stream) {
  if (n < 1 || n > MAXB || H % 8) return 1;
  PfLens pl{};
  pl.B = n;
  for (int r = 0; r < n; ++r) { pl.start[r + 1] = pl.start[r] + lens[r]; pl.slot[r] = slots[r]; }
  // prefill_rows: n blocks, 128 threads
  pf_gather_last_kernel<<<n, 128, 0, st(stream)>>>(pl, static_cast<const bf16*>(x), static_cast<bf16*>(h_last), H);
  return launched();
}

extern "C" int rows_shim_release(int n, const int* slots, void* stream) {
  if (n < 1 || n > MAXB) return 1;
  DevState* d = shim_state();
  if (!d) return 2;
  SlotList A{};
  A.n = n;
  for (int i = 0; i < n; ++i) A.slot[i] = slots[i];
  // ar_engine.cu q3_release_slots: 1 block, 32 threads
  release_state_kernel<<<1, 32, 0, st(stream)>>>(d, A);
  return launched();
}

extern "C" int rows_shim_bf16_to_f32(const void* src, float* dst, int n, void* stream) {
  // ar_engine.cu q3_engine_finalize (projection bias): (Hc + 255) / 256 blocks, 256 threads
  bf16_to_f32_kernel<<<(n + 255) / 256, 256, 0, st(stream)>>>(static_cast<const bf16*>(src), dst, n);
  return launched();
}

// ---------------------------------------------------------------------------------------------- streaming encoder
extern "C" int rows_shim_load_wav(const float* src, int src_ld, float* dst, int dst_ld, int n, const int* rp, int B, int factor,
                                  void* stream) {
  // codec_encoder.cu q3_codec_enc_stream_step_rows: dim3((T + 1023) / 1024, B), 256 threads
  load_wav_kernel<<<dim3((n + 1023) / 1024, B), 256, 0, st(stream)>>>(src, src_ld, dst, dst_ld, n, rp, B, factor);
  return launched();
}

extern "C" int rows_shim_seed_replicate(float* h, int C, int hist, int ld, const int* rp, int B, void* stream) {
  // codec_encoder.cu encode_segment: dim3((C + 255) / 256, B), 256 threads
  seed_replicate_kernel<<<dim3((C + 255) / 256, B), 256, 0, st(stream)>>>(h, C, hist, ld, rp, B);
  return launched();
}

extern "C" int rows_shim_mask_codes(int* codes, int nq, int T, const int* rp, int B, int ds, void* stream) {
  // codec_encoder.cu encode_segment: (B * nq * t3 + 255) / 256 blocks, 256 threads
  mask_codes_kernel<<<(B * nq * T + 255) / 256, 256, 0, st(stream)>>>(codes, nq, T, rp, B, ds);
  return launched();
}

// n history buffers {p, hist, factor, C, ld}
extern "C" int rows_shim_enc_reset(float* const* p, const int* hist, const int* factor, const int* C, const int* ld, int n,
                                   const int* rp, int B, void* stream) {
  if (n < 1 || n > kEncRollMax) return 1;
  EncRollTable tb{};
  tb.n = n;
  for (int i = 0; i < n; ++i) tb.e[i] = EncRollEntry{p[i], hist[i], factor[i], C[i], ld[i]};
  // codec_encoder.cu enc_reset: dim3(tb.n * B, 16), 256 threads
  enc_reset_kernel<<<dim3(tb.n * B, 16), 256, 0, st(stream)>>>(tb, rp, B);
  return launched();
}
