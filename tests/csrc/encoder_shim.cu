// Test-only C entry points around the fp32 encoder kernels, so that tests/test_gpu_encoder_kernels.py can run them on
// inputs it chooses:
//   - conv_f32 through the library's own conv_f32_launch (qwen3-tts_b200/csrc/conv_f32.cu): this file is linked against
//     libqwen3tts_b200.so, so the convolution that runs is the binary both encoders load, and a refused launch reports
//     its reason through the library's q3_last_error();
//   - the codec encoder's per-column kernels and stream roll (codec_encoder_kernels.cuh) and the speaker encoder's small
//     kernels (speaker_kernels.cuh), compiled here from the shipped headers under the library's flags, each launched with
//     the geometry its engine uses (cited beside every launch).
// Every ConvF32Args field is a plain argument and the RvqArgs / EncRollTable pointer tables are built here, so Python
// never restates a struct.  Return codes: 0 ok, 1 the library refused the launch, 2 a CUDA launch error.
#include "common.cuh"
#include "conv_f32.cuh"
#include "codec_encoder_kernels.cuh"
#include "speaker_kernels.cuh"

namespace {
int launched() { return cudaGetLastError() == cudaSuccess ? 0 : 2; }
}  // namespace

// conv_f32_init (the 96 KB attribute of conv_f32_kernel) and the one q3_spk_create sets on melspec_kernel
extern "C" int enc_shim_init() {
  if (conv_f32_init()) return 1;
  return cudaFuncSetAttribute(melspec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024) == cudaSuccess ? 0 : 2;
}

extern "C" int enc_shim_conv(const float* x, const float* x2, const float* w, const float* bias, const float* scale,
                             const float* res, float* y, int xC, int x_off, int x2C, int x2_off, int yC, int y_off, int Cin,
                             int Cout, int Tin, int Tout, int k, int stride, int dil, int pad_left, int pad, int act_in,
                             int act_out, int B, int xT, int yT, void* stream) {
  ConvF32Args a{};
  a.x = x; a.x2 = x2; a.w = w; a.bias = bias; a.scale = scale; a.res = res; a.y = y;
  a.xC = xC; a.x_off = x_off; a.x2C = x2C; a.x2_off = x2_off; a.yC = yC; a.y_off = y_off;
  a.Cin = Cin; a.Cout = Cout; a.Tin = Tin; a.Tout = Tout; a.k = k; a.stride = stride; a.dil = dil; a.pad_left = pad_left;
  a.pad = pad; a.act_in = act_in; a.act_out = act_out;
  if (conv_f32_launch(a, B, static_cast<cudaStream_t>(stream), xT, yT)) return 1;
  return launched();
}

extern "C" int enc_shim_layernorm(const float* x, int ldx, const float* w, const float* b, float* y, int ldy, int C, int T,
                                  float eps, int B, void* stream) {
  // codec_encoder.cu encode_segment: lg((t + 31) / 32, B), 256 threads
  layernorm_ct_kernel<<<dim3((T + 31) / 32, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, ldx, w, b, y, ldy, C, T, eps);
  return launched();
}

// kv == nullptr: the one-shot (in place on the q and k thirds); otherwise the stream's window buffer, grid.y covering v
extern "C" int enc_shim_rope(float* qkv, const float* cosT, const float* sinT, int C, int T, int nh, int hd, const int* rp, int B,
                             float* kv, long long kv_bs, int kv_ld, void* stream) {
  const bool own_kv = kv != nullptr;
  // encode_segment: dim3((t + 127) / 128, (own_kv ? 3 : 2) * nh * (hd / 2), B), 128 threads
  rope_ct_kernel<<<dim3((T + 127) / 128, (own_kv ? 3 : 2) * nh * (hd / 2), B), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      qkv, cosT, sinT, C, T, nh, hd, rp, B, kv, kv_bs, kv_ld);
  return launched();
}

extern "C" int enc_shim_swa(const float* qkv, const float* kv, long long kv_bs, int kv_ld, int kv_hist, float* out, int C, int T,
                            int nh, int hd, int window, float scale, const int* rp, int B, void* stream) {
  if (hd > 64) return 1;
  // encode_segment: swa_ct_kernel<64><<<dim3((t + 127) / 128, nh, B), 128>>>
  swa_ct_kernel<64><<<dim3((T + 127) / 128, nh, B), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      qkv, kv, kv_bs, kv_ld, kv_hist, out, C, T, hd, window, scale, rp);
  return launched();
}

// E, ET, E2: host arrays of nq device pointers (as q3_codec_enc_finalize tabulates them)
extern "C" int enc_shim_rvq(const float* r_sem, const float* r_ac, const float* const* E, const float* const* ET,
                            const float* const* E2, int* codes, int D, int K, int T, int nq, int nsem, int B, void* stream) {
  if (nq < 1 || nq > 64) return 1;
  const float* tab[3 * 64];
  for (int q = 0; q < nq; ++q) { tab[q] = E[q]; tab[nq + q] = ET[q]; tab[2 * nq + q] = E2[q]; }
  static const float** d_tab = nullptr;
  if (!d_tab && cudaMalloc(&d_tab, sizeof(tab)) != cudaSuccess) return 2;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (cudaStreamSynchronize(st) != cudaSuccess) return 2;  // the previous call's launch may still read the table
  if (cudaMemcpy(d_tab, tab, 3 * nq * sizeof(float*), cudaMemcpyHostToDevice) != cudaSuccess) return 2;
  RvqArgs ra{};
  ra.r_sem = r_sem; ra.r_ac = r_ac; ra.E = d_tab; ra.ET = d_tab + nq; ra.E2 = d_tab + 2 * nq;
  ra.codes = codes; ra.D = D; ra.K = K; ra.T = T; ra.nq = nq; ra.nsem = nsem;
  // encode_segment: dim3(t3, B), 256 threads, (D + 16) * 4 bytes
  rvq_encode_kernel<<<dim3(T, B), 256, (size_t)(D + 16) * sizeof(float), st>>>(ra);
  return launched();
}

// n history buffers {p, hist, factor, C, ld}; q3_codec_enc_stream_step_rows: dim3(tb.n * B, 16), 256 threads
extern "C" int enc_shim_roll(float* const* p, const int* hist, const int* factor, const int* C, const int* ld, int n,
                             const int* rp, int B, void* stream) {
  if (n < 1 || n > kEncRollMax) return 1;
  EncRollTable tb{};
  tb.n = n;
  for (int i = 0; i < n; ++i) tb.e[i] = EncRollEntry{p[i], hist[i], factor[i], C[i], ld[i]};
  enc_roll_kernel<<<dim3(tb.n * B, 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(tb, rp, B);
  return launched();
}

extern "C" int enc_shim_melspec(const float* wav, int T, const float* window, const float* twc, const float* tws,
                                const float* fbT, float* out, int n_fft, int hop, int n_mels, int frames, int B, void* stream) {
  // speaker_encoder.cu run_mel: dim3(frames, B), 256 threads, (3 * n_fft + n_fft / 2 + 1) * 4 bytes
  const size_t smem = (size_t)(3 * n_fft + n_fft / 2 + 1) * sizeof(float);
  melspec_kernel<<<dim3(frames, B), 256, smem, static_cast<cudaStream_t>(stream)>>>(wav, T, window, twc, tws, fbT, out, n_fft,
                                                                                    hop, n_mels, frames);
  return launched();
}

extern "C" int enc_shim_mean_t(const float* x, int xC, int c_off, int C, int T, float* m, int B, void* stream) {
  // q3_spk_embed: dim3(C, B), 32 threads
  mean_t_kernel<<<dim3(C, B), 32, 0, static_cast<cudaStream_t>(stream)>>>(x, xC, c_off, C, T, m);
  return launched();
}

extern "C" int enc_shim_se_apply(const float* h, const float* gate, const float* res, int rC, int r_off, float* y, int yC,
                                 int y_off, int C, int T, int B, void* stream) {
  // q3_spk_embed: dim3((L + 127) / 128, C, B), 128 threads
  se_apply_kernel<<<dim3((T + 127) / 128, C, B), 128, 0, static_cast<cudaStream_t>(stream)>>>(h, gate, res, rC, r_off, y, yC,
                                                                                             y_off, C, T);
  return launched();
}

extern "C" int enc_shim_copy_ch(const float* x, int xC, int x_off, float* y, int yC, int y_off, int C, int T, int B,
                                void* stream) {
  // q3_spk_embed: dim3((L + 127) / 128, Cs, B), 128 threads
  copy_ch_kernel<<<dim3((T + 127) / 128, C, B), 128, 0, static_cast<cudaStream_t>(stream)>>>(x, xC, x_off, y, yC, y_off, T);
  return launched();
}

extern "C" int enc_shim_asp_cat(const float* x, float* cat, int C, int T, float eps, int B, void* stream) {
  // q3_spk_embed: dim3(Ccat, B), 32 threads
  asp_cat_kernel<<<dim3(C, B), 32, 0, static_cast<cudaStream_t>(stream)>>>(x, cat, C, T, eps);
  return launched();
}

extern "C" int enc_shim_asp_pool(const float* x, const float* att, float* pooled, int C, int T, float eps, int B, void* stream) {
  // q3_spk_embed: dim3(Ccat, B), 32 threads
  asp_pool_kernel<<<dim3(C, B), 32, 0, static_cast<cudaStream_t>(stream)>>>(x, att, pooled, C, T, eps);
  return launched();
}
