// Speaker x-vector path of voice cloning on H100 (sm_90a): 24 kHz waveform -> log-mel -> ECAPA-TDNN -> (enc_dim,) embedding.
// Replaces Qwen3TTSForConditionalGeneration.extract_speaker_embedding (qwen_tts/core/models/modeling_qwen3_tts.py:1941-1954):
// mel_spectrogram (:396-448) + Qwen3TTSSpeakerEncoder.forward (:371-393) with TimeDelayNetBlock :229-250, Res2NetBlock
// :95-126, SqueezeExcitationBlock :129-157, SqueezeExcitationRes2NetBlock :253-297, AttentiveStatisticsPooling :160-226.
//
// Checked against the CPU oracle by tests/test_gpu_speaker_encoder.py (log-mel, ECAPA embedding and the
// waveform-to-embedding path at tiny and default shapes, golden vectors).
//
// fp32 throughout, activations [B][C][T] (time contiguous).  Every Conv1d is one launch of the direct convolution of
// conv_f32.cu, which the codec encoder shares: reflect "same" padding with dilation, channel-sliced input/output (Res2Net
// chunks and the multi-layer feature concatenation are views into one buffer, never copies), an optional second input
// added on load (Res2Net's `part + previous output`), tanh-on-load, ReLU / sigmoid epilogues.  The STFT is a direct 1024-point DFT per frame
// against an exact periodic twiddle table (the Hann window is applied on load) fused with the mel projection and log.
#include "common.cuh"
#include "conv_f32.cuh"
#include "dev_store.h"
#include "../../include/qwen3tts_b200.h"

#include <string>

#include "speaker_kernels.cuh"

struct q3_spk {
  q3_spk_cfg cfg;
  DevStore store{"speaker encoder"};
  float* ws = nullptr;
  size_t ws_elems = 0;
  bool finalized = false;
  int launches = 0;
};

extern "C" int q3_spk_create(const q3_spk_cfg* cfg, q3_spk** out) {
  Q3_REQUIRE(cfg && out, "null argument");
  Q3_CUDA(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  Q3_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  Q3_REQUIRE(prop.major == 9 && prop.minor == 0, "this library is built for sm_90a (H100); device is sm_%d%d", prop.major, prop.minor);
  Q3_REQUIRE(cfg->n_blocks >= 3 && cfg->n_blocks <= 8, "3..8 encoder stages (enc_channels entries)");
  Q3_REQUIRE(cfg->n_fft >= 64 && (cfg->n_fft & (cfg->n_fft - 1)) == 0 && cfg->n_fft <= 4096, "n_fft must be a power of two <= 4096");
  Q3_REQUIRE(cfg->hop >= 1 && cfg->hop <= cfg->n_fft && cfg->win == cfg->n_fft, "win_size must equal n_fft; 1 <= hop <= n_fft");
  Q3_REQUIRE(cfg->res2net_scale >= 2, "res2net scale must be >= 2");
  int cat = 0;
  for (int i = 1; i < cfg->n_blocks - 1; ++i) {
    Q3_REQUIRE(cfg->channels[i] % cfg->res2net_scale == 0, "enc_channels[%d] must be divisible by the res2net scale", i);
    Q3_REQUIRE(cfg->channels[i] == cfg->channels[i - 1], "SE-Res2Net blocks need equal in/out channels (residual add)");
    cat += cfg->channels[i];
  }
  Q3_REQUIRE(cat == cfg->channels[cfg->n_blocks - 1], "enc_channels[-1] must equal the sum of the SE-Res2Net block widths");
  if (conv_f32_init()) return 1;
  Q3_CUDA(cudaFuncSetAttribute(melspec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  q3_spk* e = new q3_spk();
  e->cfg = *cfg;
  *out = e;
  return 0;
}

extern "C" void q3_spk_destroy(q3_spk* e) { delete e; }

extern "C" int q3_spk_load_tensor(q3_spk* e, const char* name, const float* dev, const int64_t* shape, int32_t ndim) {
  Q3_REQUIRE(e && name && dev && shape, "null argument");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  return e->store.load(name, dev, shape, ndim, DT_F32);
}

extern "C" int q3_spk_finalize(q3_spk* e) {
  Q3_REQUIRE(e, "null speaker encoder");
  const q3_spk_cfg& g = e->cfg;
  const DevStore& S = e->store;
  if (!S.need<float>("mel.window", g.n_fft) || !S.need<float>("mel.cos", g.n_fft) || !S.need<float>("mel.sin", g.n_fft) ||
      !S.need<float>("mel.fbT", (int64_t)(g.n_fft / 2 + 1) * g.mel_dim))
    return 1;
  e->finalized = true;
  return 0;
}

extern "C" int q3_spk_frames(q3_spk* e, int32_t T) {
  if (!e || T <= 0) return 0;
  const int padded = T + 2 * ((e->cfg.n_fft - e->cfg.hop) / 2);
  return padded < e->cfg.n_fft ? 0 : 1 + (padded - e->cfg.n_fft) / e->cfg.hop;
}
extern "C" int q3_spk_last_launch_count(q3_spk* e) { return e ? e->launches : 0; }

namespace {

struct SpkRunner {
  q3_spk* e;
  cudaStream_t st;
  int B, T;

  int conv(const std::string& name, const float* x, int xC, int x_off, const float* x2, int x2C, int x2_off, float* y, int yC,
           int y_off, int Cin, int Cout, int k, int dil, ConvActIn act_in, ConvActOut act_out, int T_) {
    ConvF32Args a{};
    if (!(a.w = e->store.need<float>(name + ".weight", (int64_t)Cout * Cin * k)) || !(a.bias = e->store.need<float>(name + ".bias", Cout)))
      return 1;
    Q3_REQUIRE(dil * (k - 1) / 2 < T_ || k == 1, "input too short (%d frames) for reflect padding of %s", T_, name.c_str());
    // nn.Conv1d(padding="same", padding_mode="reflect"): total pad dil*(k-1), left = total / 2
    a.x = x; a.x2 = x2; a.y = y;
    a.xC = xC; a.x_off = x_off; a.x2C = x2C; a.x2_off = x2_off; a.yC = yC; a.y_off = y_off;
    a.Cin = Cin; a.Cout = Cout; a.Tin = T_; a.Tout = T_; a.k = k; a.stride = 1; a.dil = dil; a.pad_left = dil * (k - 1) / 2;
    a.pad = PAD_REFLECT; a.act_in = act_in; a.act_out = act_out;
    if (conv_f32_launch(a, B, st)) return 1;
    ++e->launches;
    return 0;
  }
};

}  // namespace

// mel only (tests): wav fp32 [B][T] -> mel fp32 [B][mel_dim][frames]
static int run_mel(q3_spk* e, const float* wav, int B, int T, float* mel, int frames, cudaStream_t st) {
  const q3_spk_cfg& g = e->cfg;
  Q3_REQUIRE(frames >= 1, "waveform too short for one STFT frame");
  Q3_REQUIRE((g.n_fft - g.hop) / 2 < T, "waveform shorter than the reflect padding");
  const DevStore& S = e->store;
  const float *window = S.need<float>("mel.window", g.n_fft), *twc = S.need<float>("mel.cos", g.n_fft),
              *tws = S.need<float>("mel.sin", g.n_fft), *fbT = S.need<float>("mel.fbT", (int64_t)(g.n_fft / 2 + 1) * g.mel_dim);
  if (!window || !twc || !tws || !fbT) return 1;
  const size_t smem = (size_t)(3 * g.n_fft + g.n_fft / 2 + 1) * sizeof(float);
  melspec_kernel<<<dim3(frames, B), 256, smem, st>>>(wav, T, window, twc, tws, fbT, mel, g.n_fft, g.hop, g.mel_dim, frames);
  ++e->launches;
  return 0;
}

extern "C" int q3_spk_mel(q3_spk* e, const float* wav_dev, int32_t B, int32_t T, float* mel_dev, void* stream_) {
  Q3_REQUIRE(e && e->finalized && wav_dev && mel_dev && B >= 1 && T >= 1, "bad arguments");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  e->launches = 0;
  if (run_mel(e, wav_dev, B, T, mel_dev, q3_spk_frames(e, T), (cudaStream_t)stream_)) return 1;
  Q3_CUDA(cudaGetLastError());
  return 0;
}

// mel [B][mel_dim][frames] (device) -> emb [B][enc_dim]; mel_dev == NULL: computed from wav_dev [B][T] first
extern "C" int q3_spk_embed(q3_spk* e, const float* wav_dev, int32_t B, int32_t T, const float* mel_dev, int32_t frames_in,
                            float* emb_dev, void* stream_) {
  Q3_REQUIRE(e && e->finalized && emb_dev && B >= 1, "bad arguments");
  Q3_REQUIRE((wav_dev && T >= 1) || (mel_dev && frames_in >= 1), "need a waveform or a mel spectrogram");
  const q3_spk_cfg& g = e->cfg;
  Q3_CUDA(cudaSetDevice(g.device));
  cudaStream_t st = (cudaStream_t)stream_;
  e->launches = 0;
  const int L = mel_dev ? frames_in : q3_spk_frames(e, T);
  Q3_REQUIRE(L >= 1, "waveform too short for one STFT frame");
  const int nb = g.n_blocks, C = g.channels[1], Ccat = g.channels[nb - 1], S = g.res2net_scale, Cs = C / S;
  const int C0 = g.channels[0];
  // workspace (floats): mel | F0 | CAT | H | R | H2 | M | ACAT | AH | ATT | small (means, gates, pooled)
  const size_t nMel = (size_t)B * g.mel_dim * L, nF0 = (size_t)B * C0 * L, nC = (size_t)B * C * L, nCat = (size_t)B * Ccat * L;
  const size_t nAH = (size_t)B * g.attention_channels * L;
  const size_t small = (size_t)B * (C + g.se_channels + C + 2 * Ccat);
  const size_t need = nMel + nF0 + nCat + 3 * nC + nCat + 3 * nCat + nAH + nCat + small;
  if (need > e->ws_elems) {
    e->ws_elems = 0;
    if (e->store.grow(&e->ws, need * 4, st)) return 1;
    e->ws_elems = need;
  }
  float* p = e->ws;
  float* MEL = p; p += nMel;
  float* F0 = p; p += nF0;
  float* CAT = p; p += nCat;
  float* H = p; p += nC;
  float* R = p; p += nC;
  float* H2 = p; p += nC;
  float* M = p; p += nCat;
  float* ACAT = p; p += 3 * nCat;
  float* AH = p; p += nAH;
  float* ATT = p; p += nCat;
  float* MEAN = p; p += (size_t)B * C;
  float* SE1 = p; p += (size_t)B * g.se_channels;
  float* GATE = p; p += (size_t)B * C;
  float* POOL = p; p += (size_t)B * 2 * Ccat;
  const float* mel = mel_dev;
  if (!mel) {
    if (run_mel(e, wav_dev, B, T, MEL, L, st)) return 1;
    mel = MEL;
  }
  SpkRunner r{e, st, B, L};
  // blocks.0: TDNN(mel_dim -> C0, k0, d0)
  if (r.conv("blocks.0.conv", mel, g.mel_dim, 0, nullptr, 0, 0, F0, C0, 0, g.mel_dim, C0, g.kernel_sizes[0], g.dilations[0], IN_NONE, OUT_RELU, L)) return 1;
  // SE-Res2Net blocks (:253-297); block i reads its input from F0 (i == 1) or from CAT slice i-2 and writes CAT slice i-1
  for (int i = 1; i < nb - 1; ++i) {
    const std::string pfx = "blocks." + std::to_string(i);
    const float* xin = (i == 1) ? F0 : CAT;
    const int xinC = (i == 1) ? C0 : Ccat, xoff = (i == 1) ? 0 : (i - 2) * C;
    if (r.conv(pfx + ".tdnn1.conv", xin, xinC, xoff, nullptr, 0, 0, H, C, 0, g.channels[i - 1], C, 1, 1, IN_NONE, OUT_RELU, L)) return 1;
    // Res2Net (:114-126): chunk 0 passes through; chunk j = TDNN_j(chunk j [+ output j-1])
    copy_ch_kernel<<<dim3((L + 127) / 128, Cs, B), 128, 0, st>>>(H, C, 0, R, C, 0, L);
    ++e->launches;
    for (int j = 1; j < S; ++j) {
      const std::string bn = pfx + ".res2net_block.blocks." + std::to_string(j - 1) + ".conv";
      if (r.conv(bn, H, C, j * Cs, j >= 2 ? R : nullptr, C, (j - 1) * Cs, R, C, j * Cs, Cs, Cs, g.kernel_sizes[i], g.dilations[i], IN_NONE, OUT_RELU, L))
        return 1;
    }
    if (r.conv(pfx + ".tdnn2.conv", R, C, 0, nullptr, 0, 0, H2, C, 0, C, C, 1, 1, IN_NONE, OUT_RELU, L)) return 1;
    // squeeze-excitation gate (:150-157) and the residual (:296-297)
    mean_t_kernel<<<dim3(C, B), 32, 0, st>>>(H2, C, 0, C, L, MEAN);
    ++e->launches;
    SpkRunner r1{e, st, B, 1};
    if (r1.conv(pfx + ".se_block.conv1", MEAN, C, 0, nullptr, 0, 0, SE1, g.se_channels, 0, C, g.se_channels, 1, 1, IN_NONE, OUT_RELU, 1)) return 1;
    if (r1.conv(pfx + ".se_block.conv2", SE1, g.se_channels, 0, nullptr, 0, 0, GATE, C, 0, g.se_channels, C, 1, 1, IN_NONE, OUT_SIGMOID, 1)) return 1;
    se_apply_kernel<<<dim3((L + 127) / 128, C, B), 128, 0, st>>>(H2, GATE, xin, xinC, xoff, CAT, Ccat, (i - 1) * C, C, L);
    ++e->launches;
  }
  // multi-layer feature aggregation (:381-383) on the concatenation of the SE-Res2Net outputs
  if (r.conv("mfa.conv", CAT, Ccat, 0, nullptr, 0, 0, M, Ccat, 0, Ccat, Ccat, g.kernel_sizes[nb - 1], g.dilations[nb - 1], IN_NONE, OUT_RELU, L)) return 1;
  // attentive statistics pooling (:203-226)
  asp_cat_kernel<<<dim3(Ccat, B), 32, 0, st>>>(M, ACAT, Ccat, L, 1e-12f);
  ++e->launches;
  if (r.conv("asp.tdnn.conv", ACAT, 3 * Ccat, 0, nullptr, 0, 0, AH, g.attention_channels, 0, 3 * Ccat, g.attention_channels, 1, 1, IN_NONE, OUT_RELU, L)) return 1;
  if (r.conv("asp.conv", AH, g.attention_channels, 0, nullptr, 0, 0, ATT, Ccat, 0, g.attention_channels, Ccat, 1, 1, IN_TANH, OUT_NONE, L)) return 1;
  asp_pool_kernel<<<dim3(Ccat, B), 32, 0, st>>>(M, ATT, POOL, Ccat, L, 1e-12f);
  ++e->launches;
  // final 1x1 conv (:384-393)
  SpkRunner r1{e, st, B, 1};
  if (r1.conv("fc", POOL, 2 * Ccat, 0, nullptr, 0, 0, emb_dev, g.enc_dim, 0, 2 * Ccat, g.enc_dim, 1, 1, IN_NONE, OUT_NONE, 1)) return 1;
  Q3_CUDA(cudaGetLastError());
  return 0;
}
