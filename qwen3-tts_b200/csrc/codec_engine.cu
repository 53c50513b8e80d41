// Qwen3-TTS-Tokenizer-12Hz codec DECODER on H100 (sm_90a): codes -> 24 kHz waveform.
// Replaces Qwen3TTSTokenizerV2Decoder.forward (qwen_tts/core/tokenizer_12hz/modeling_qwen3_tts_tokenizer_v2.py:869-884).
//
// Layout: every activation is channels-last bf16 [B][T][C]; every Conv1d / ConvTranspose1d / Linear is ONE
// wgmma tap-GEMM launch (gemm_sm90.cu) whose A tiles are TMA-loaded with a per-tap row shift — no im2col
// buffer — with bias, LayerScale, residual add and the *next* layer's SnakeBeta fused into the epilogue.
// Small row-wise ops (RVQ gather, RMSNorm, RoPE, 72-frame sliding-window attention, depthwise conv + LayerNorm,
// the final 96->1 conv + clamp) are plain CUDA kernels: they are <2 % of the FLOPs and HBM-trivial.
#include "common.cuh"
#include "dev_store.h"
#include "gemm_sm90.cuh"
#include "../../include/qwen3tts_b200.h"

#include <algorithm>
#include <string>
#include <vector>

#include "codec_kernels.cuh"

// per-(row, frame) element high-water mark of the decoder's scratch tensors over all stages
static size_t scratch_per_frame(const q3_codec_cfg& g) {
  size_t per_frame = std::max<size_t>({(size_t)3 * g.num_heads * g.head_dim, (size_t)2 * g.intermediate_size, (size_t)g.latent_dim,
                                       (size_t)g.codebook_dim});
  size_t up = 1;
  for (int i = 0; i < g.n_upsampling_ratios; ++i) { up *= g.upsampling_ratios[i]; per_frame = std::max(per_frame, up * 4 * g.latent_dim); }
  per_frame = std::max(per_frame, up * (size_t)g.decoder_dim);
  int ch = g.decoder_dim;
  for (int i = 0; i < g.n_upsample_rates; ++i) { up *= g.upsample_rates[i]; ch /= 2; per_frame = std::max(per_frame, up * (size_t)ch); }
  return per_frame;
}

// (re)allocate the decoder's four scratch buffers X, Y, Z, W to `elems` bf16 each
static int alloc_scratch(DevStore& store, bf16* buf[4], size_t elems, cudaStream_t stream) {
  for (int i = 0; i < 4; ++i)
    if (store.grow(&buf[i], elems * 2 + 1024, stream)) return 1;
  return 0;
}

struct q3_codec {
  q3_codec_cfg cfg;
  DevStore store{"codec"};
  bf16* buf[4] = {nullptr, nullptr, nullptr, nullptr};
  size_t buf_elems = 0;
  bool finalized = false;
  int total_up = 1;
  int launches = 0;
  struct Capture { int stage; bf16* dst; int64_t capacity; };
  std::vector<Capture> captures;  // test hook (q3_codec_debug_capture): stage ordinal -> destination of the next forward
};

extern "C" int q3_codec_create(const q3_codec_cfg* cfg, q3_codec** out) {
  Q3_REQUIRE(cfg && out, "null argument");
  Q3_CUDA(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  Q3_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  Q3_REQUIRE(prop.major == 9 && prop.minor == 0, "this library is built for sm_90a (H100); device is sm_%d%d", prop.major, prop.minor);
  Q3_REQUIRE(cfg->head_dim % 2 == 0 && cfg->head_dim <= 64, "codec head_dim must be even and <= 64");
  // a window below 1 would leave a query no key (and a stream a history of -1 rows)
  Q3_REQUIRE(cfg->sliding_window >= 1 && cfg->sliding_window <= 96, "sliding_window must be in [1, 96]");
  Q3_REQUIRE(cfg->num_heads == cfg->num_kv_heads, "codec transformer is MHA in the reference config");
  Q3_REQUIRE(cfg->codebook_dim % 32 == 0 && cfg->latent_dim % 16 == 0 && cfg->hidden_size % 16 == 0 &&
                 cfg->intermediate_size % 16 == 0 && cfg->decoder_dim % 16 == 0,
             "channel counts must be multiples of 16");
  Q3_REQUIRE(cfg->n_upsample_rates >= 0 && cfg->n_upsample_rates <= 8 && cfg->n_upsampling_ratios >= 0 &&
                 cfg->n_upsampling_ratios <= 8,
             "n_upsample_rates and n_upsampling_ratios must be in [0, 8]");
  Q3_REQUIRE((cfg->decoder_dim >> cfg->n_upsample_rates) % 16 == 0, "final channel count must be a multiple of 16");
  if (gemm_init()) return 1;
  q3_codec* c = new q3_codec();
  c->cfg = *cfg;
  c->total_up = 1;
  for (int i = 0; i < cfg->n_upsample_rates; ++i) c->total_up *= cfg->upsample_rates[i];
  for (int i = 0; i < cfg->n_upsampling_ratios; ++i) c->total_up *= cfg->upsampling_ratios[i];
  *out = c;
  return 0;
}

extern "C" void q3_codec_destroy(q3_codec* c) { delete c; }

extern "C" int q3_codec_total_upsample(q3_codec* c) { return c ? c->total_up : 0; }
extern "C" int q3_codec_last_launch_count(q3_codec* c) { return c ? c->launches : 0; }

// Test hook (tests/ only): the next q3_codec_forward calls copy the bf16 [B][T_stage][C_stage] tensor of `stage` into
// dst_dev (at most `capacity` elements).  Stages: 0 pre_conv output, 1 pre-transformer output (after output_proj), 2 output
// of the upsample stack, 3 SnakeBeta(decoder.0 conv output) as fed to block 0, 4+i output of decoder block i.
// stage < 0 clears all captures.
extern "C" int q3_codec_debug_capture(q3_codec* c, int32_t stage, void* dst_dev, int64_t capacity) {
  Q3_REQUIRE(c, "null codec");
  if (stage < 0) { c->captures.clear(); return 0; }
  Q3_REQUIRE(dst_dev && capacity > 0, "bad capture destination");
  c->captures.push_back({stage, reinterpret_cast<bf16*>(dst_dev), capacity});
  return 0;
}

// Engine-native tensors (converted from the reference state_dict by the Python host, see INTEGRATION.md):
// shape[] / ndim describe the tensor; dtype is inferred from the name suffix: names ending in ".w" / "table" /
// "proj" / "norm" / "ln1" / "ln2" / "cos" / "sin" are bf16, everything else fp32.
static bool name_is_bf16(const std::string& n) {
  auto ends = [&](const char* s) { size_t l = strlen(s); return n.size() >= l && n.compare(n.size() - l, l, s) == 0; };
  if (ends(".dw.w") || ends("dec.out.w")) return false;
  return ends(".w") || ends(".table") || ends(".proj") || ends(".norm") || ends(".ln1") || ends(".ln2") || ends(".cos") ||
         ends(".sin");
}

extern "C" int q3_codec_load_tensor(q3_codec* c, const char* name, const void* dev, const int64_t* shape, int32_t ndim) {
  Q3_REQUIRE(c && name && dev && shape, "null argument");
  Q3_CUDA(cudaSetDevice(c->cfg.device));
  return c->store.load(name, dev, shape, ndim, name_is_bf16(name) ? DT_BF16 : DT_F32);
}

static int kpad(int k) { return (k + 63) / 64 * 64; }

extern "C" int q3_codec_finalize(q3_codec* c) {
  Q3_REQUIRE(c, "null codec");
  const q3_codec_cfg& g = c->cfg;
  // spot-check the tensors whose absence would otherwise only surface mid-forward
  if (!c->store.need<bf16>("rvq.table", (int64_t)g.num_quantizers * g.codebook_size * (g.codebook_dim / 2)) ||
      !c->store.need<bf16>("rvq.proj", (int64_t)g.codebook_dim * kpad(g.codebook_dim)) ||
      !c->store.need<float>("dec.out.w", (int64_t)7 * (g.decoder_dim >> g.n_upsample_rates)))
    return 1;
  c->finalized = true;
  return 0;
}

namespace {

struct Runner {
  q3_codec* c;
  cudaStream_t stream;
  int B;
  int err = 0;

  // one tap-GEMM: a [B][T][K] -> [B][T][N]; a: row 0 of the A map (history rows included), a_bs: its batch stride in
  // elements, v: the A map's rows and the output / residual batch strides
  void gemm(const bf16* a, int T, int K, int64_t a_bs, const char* wname, int N, int ntaps, const int* shifts, GemmEpilogue ep,
            const GemmViews& v) {
    if (err) return;
    const int Kp = kpad(K);
    const bf16* w = need<bf16>(wname, (int64_t)N * ntaps * Kp);
    if (!w) return;
    if (ep.cmod == 0) ep.cmod = N;
    GemmPlan plan;
    const int mt = (T + 127) / 128;
    if (gemm_make_plan_v(&plan, a, B, T, K, K, a_bs, w, N, Kp, ntaps, shifts,
                         gemm_pick_bn(N, mt, B), ep, v)) { err = 1; return; }
    if (gemm_launch(plan, stream)) { err = 1; return; }
    c->launches++;
  }
  // test hook: copy a stage's [B][T][C] bf16 tensor to every destination registered for `stage` (no launch, no sync)
  void capture(int stage, const bf16* x, int64_t elems) {
    if (err) return;
    for (const auto& cp : c->captures)
      if (cp.stage == stage) {
        const int64_t n = elems < cp.capacity ? elems : cp.capacity;
        if (cudaMemcpyAsync(cp.dst, x, (size_t)n * 2, cudaMemcpyDeviceToDevice, stream) != cudaSuccess)
          err = q3_set_err("codec: capture of stage %d failed", stage);
      }
  }
  // a tensor of the store; a missing or ill-shaped one fails the forward
  template <class T>
  const T* need(const std::string& n, int64_t cnt) {
    const T* p = c->store.need<T>(n, cnt);
    if (!p) err = 1;
    return p;
  }
};

}  // namespace

// A tensor that a layer reads back in time: [B][hist + cap][C], the new rows behind `hist` rows of history.  The
// streaming decoder keeps one per such layer; the one-shot forward views a scratch buffer as {p, 0, C, T}.
struct HistBuf {
  bf16* p = nullptr;
  int hist = 0, C = 0, cap = 0;                 // rows of history, channels, capacity in new rows
  int bs_rows() const { return hist + cap; }
  long long bs() const { return (long long)bs_rows() * C; }
  bf16* cur() const { return p + (size_t)hist * C; }  // first new row of batch row 0
};

// =================================================================================================
// Stateful streaming decoder (SURVEY §8f-2, §8b: q3_codec_stream_*).  Equal to the full causal forward over everything
// pushed so far (oracle/codec.py::StreamingDecoder is the spec; the reference's chunked_decode instead re-decodes 25
// frames of left context per chunk, …v2.py:886-896).  State per row: the last (k-1)*dilation input rows of every
// convolution with taps, the last input row of every k=2r ConvTranspose, and per transformer layer the rotated K and V
// of the last window-1 frames.  Every such tensor lives in a history-prefixed buffer [B][hist + T_cap][C]: its producer
// GEMM writes the new rows behind the history, its consumer GEMM reads through a TMA map whose taps reach back into the
// history (GemmViews), and one roll kernel per packet moves the last `hist` rows to the front.  Every row has its own
// position and may take fewer frames than the packet (its count) or be reset alone, so rows that start and end at
// different frames share one stream (a continuous-batching session).
// =================================================================================================
struct q3_codec_stream {
  q3_codec* c = nullptr;
  int B = 0, nmax = 0;
  std::vector<int> pos;       // frames pushed per row since its last reset
  std::vector<int32_t> rp_h;  // host image of rp: [0, B) positions, [B, 2B) counts of the next step (reset mask of a reset)
  int32_t* rp = nullptr;      // device int32 [2][B], uploaded with one copy per step or reset
  DevStore store{"codec stream"};
  HistBuf pre, in, out;
  std::vector<HistBuf> dw, ct, kv;
  std::vector<std::vector<HistBuf>> c1;
  bf16* buf[4] = {nullptr, nullptr, nullptr, nullptr};
};

// every history buffer of a stream, for the roll after a packet and for reset
template <class F>
static void for_each_hist(const q3_codec_stream* s, F f) {
  f(s->pre); f(s->in); f(s->out);
  for (const HistBuf& h : s->kv) f(h);
  for (const HistBuf& h : s->dw) f(h);
  for (const HistBuf& h : s->ct) f(h);
  for (const auto& v : s->c1) for (const HistBuf& h : v) f(h);
}

// The decoder's layer sequence for n new frames of every row, frame t of row b at position rp[b] + t, of which the first
// rp[B + b] are the row's (see row_pos; rp == nullptr: position 0, all n): codes int32 [B][K][n] -> wav fp32
// [B][n * total_upsample], zero past each row's count.  The tensors that a layer reads back in time (pre, kv, dw, in, ct, c1, out) are
// HistBuf views: with a stream state `s` its history-prefixed buffers; without one (the one-shot forward, rp = nullptr)
// plain views of the scratch buffers, where the TMA zero fill of negative rows is the causal left padding.  Scratch
// X, Y, Z, W (`scratch`, per_frame * B * n elements each) hold everything else.  One-shot mapping: pre, dw -> Y;
// in -> Z; ct, out -> X; c1 -> W.  No GEMM's A operand aliases one of its outputs.  Every layer is causal and row-local, so
// the frames past a row's count change nothing before them; they only never reach the history, the RoPE table or the codes.
static int decode_frames(q3_codec* c, const q3_codec_stream* s, const int32_t* codes, int B, int n, const int* rp,
                         bf16* const scratch[4], float* wav, cudaStream_t stream) {
  const q3_codec_cfg& g = c->cfg;
  const int Cl = g.latent_dim, Hh = g.hidden_size, nh = g.num_heads, hd = g.head_dim, I = g.intermediate_size;
  const int nr = g.n_upsample_rates;
  bf16 *X = scratch[0], *Y = scratch[1], *Z = scratch[2], *W = scratch[3];
  Runner R{c, stream, B};
  c->launches = 0;
  const int zero = 0;
  GemmEpilogue none{};
  auto view_in = [](const HistBuf& h, int T) { GemmViews v; v.a_rows = h.hist + T; v.a_row0 = h.hist; return v; };
  // stream views are strided: only the one-shot forward captures
  auto capture = [&](int stage, const bf16* x, int64_t elems) { if (!s) R.capture(stage, x, elems); };
  // input of decoder block bi's ConvTranspose (bi == nr: of the final conv), and of unit u's dilated conv
  auto block_in = [&](int bi, int C, int T) { return s ? (bi < nr ? s->ct[bi] : s->out) : HistBuf{X, 0, C, T}; };
  auto unit_in = [&](int bi, int u, int C, int T) { return s ? s->c1[bi][u] : HistBuf{W, 0, C, T}; };

  // ---- RVQ decode -> X [B][n][codebook_dim]; projection -> pre_conv's input
  const int D = g.codebook_dim / 2;
  rvq_gather_kernel<<<B * n, 128, 0, stream>>>(codes, R.need<bf16>("rvq.table", (int64_t)g.num_quantizers * g.codebook_size * D), X, B,
                                               g.num_quantizers, n, D, g.codebook_size, rp);
  c->launches++;
  if (R.err) return 1;
  const HistBuf pre = s ? s->pre : HistBuf{Y, 0, g.codebook_dim, n};
  { GemmEpilogue e = none; e.out_raw = pre.cur(); GemmViews v; v.raw_bs = pre.bs();
    R.gemm(X, n, g.codebook_dim, (int64_t)n * g.codebook_dim, "rvq.proj", g.codebook_dim, 1, &zero, e, v); }
  // ---- pre_conv k=3 (…v2.py:839-843,874)
  { const int sh[3] = {-2, -1, 0}; GemmEpilogue e = none; e.bias = R.need<float>("pre_conv.b", Cl); e.out_raw = X;
    R.gemm(pre.p, n, g.codebook_dim, pre.bs(), "pre_conv.w", Cl, 3, sh, e, view_in(pre, n)); }
  capture(0, X, (int64_t)B * n * Cl);
  // ---- pre_transformer (…v2.py:501-575); the stream keeps a K/V window per layer
  { GemmEpilogue e = none; e.bias = R.need<float>("tr.in.b", Hh); e.out_raw = Y; R.gemm(X, n, Cl, (int64_t)n * Cl, "tr.in.w", Hh, 1, &zero, e, {}); }
  bf16* xres = Y;  // residual stream [B][n][Hh]
  const int rows = B * n;
  const bf16* cosT = R.need<bf16>("rope.cos", (int64_t)g.max_frames * (hd / 2));
  const bf16* sinT = R.need<bf16>("rope.sin", (int64_t)g.max_frames * (hd / 2));
  for (int l = 0; l < g.num_layers && !R.err; ++l) {
    const std::string p = "tr." + std::to_string(l);
    rmsnorm_rows_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(xres, R.need<bf16>(p + ".ln1", Hh), X, rows, Hh, g.rms_eps);
    { GemmEpilogue e = none; e.out_raw = Z; R.gemm(X, n, Hh, (int64_t)n * Hh, (p + ".qkv.w").c_str(), 3 * nh * hd, 1, &zero, e, {}); }
    // keys and values: the stream appends them to the layer's window buffer, the one-shot attends over qkv itself
    const HistBuf kv = s ? s->kv[l] : HistBuf{Z + nh * hd, 0, 3 * nh * hd, n};
    rope_append_kernel<<<296, 256, 0, stream>>>(Z, cosT, sinT, s ? kv.p : nullptr, B, n, nh, hd, rp, kv.hist, kv.bs_rows());
    swa_stream_kernel<<<(rows * nh + 7) / 8, 256, 0, stream>>>(Z, kv.p, kv.C, kv.bs_rows(), kv.hist, X, B, n, nh, hd,
                                                                g.sliding_window, rp);
    { GemmEpilogue e = none; e.scale = R.need<float>(p + ".ls1", Hh); e.resid = xres; e.out_raw = W;
      R.gemm(X, n, nh * hd, (int64_t)n * nh * hd, (p + ".o.w").c_str(), Hh, 1, &zero, e, {}); }
    rmsnorm_rows_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(W, R.need<bf16>(p + ".ln2", Hh), X, rows, Hh, g.rms_eps);
    { GemmEpilogue e = none; e.act = ACT_SWIGLU_PAIR; e.out_act = Z;
      R.gemm(X, n, Hh, (int64_t)n * Hh, (p + ".gate_up.w").c_str(), 2 * I, 1, &zero, e, {}); }
    { GemmEpilogue e = none; e.scale = R.need<float>(p + ".ls2", Hh); e.resid = W; e.out_raw = xres;
      R.gemm(Z, n, I, (int64_t)n * I, (p + ".down.w").c_str(), Hh, 1, &zero, e, {}); }
    c->launches += 4;
  }
  rmsnorm_rows_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(xres, R.need<bf16>("tr.norm", Hh), X, rows, Hh, g.rms_eps);
  c->launches++;
  { GemmEpilogue e = none; e.bias = R.need<float>("tr.out.b", Cl); e.out_raw = Z; R.gemm(X, n, Hh, (int64_t)n * Hh, "tr.out.w", Cl, 1, &zero, e, {}); }
  capture(1, Z, (int64_t)B * n * Cl);
  // ---- upsample: ConvT(k=s=f) (no overlap) + ConvNeXt (depthwise k7) (…v2.py:845-855,878-880)
  bf16* cur = Z;  // [B][Tc][Cl] contiguous
  int Tc = n;
  for (int i = 0; i < g.n_upsampling_ratios && !R.err; ++i) {
    const int f = g.upsampling_ratios[i];
    const std::string p = "up." + std::to_string(i);
    const HistBuf dw = s ? s->dw[i] : HistBuf{Y, 0, Cl, Tc * f};
    { GemmEpilogue e = none; e.bias = R.need<float>(p + ".ct.b", Cl); e.cmod = Cl; e.out_raw = dw.cur(); GemmViews v; v.raw_bs = dw.bs();
      R.gemm(cur, Tc, Cl, (int64_t)Tc * Cl, (p + ".ct.w").c_str(), f * Cl, 1, &zero, e, v); }
    Tc *= f;
    const float *dww = R.need<float>(p + ".dw.w", (int64_t)Cl * 7), *dwb = R.need<float>(p + ".dw.b", Cl), *lw = R.need<float>(p + ".ln_g", Cl),
                *lb = R.need<float>(p + ".ln_beta", Cl);
    if (R.err) break;
    dwconv_ln_kernel<<<B * Tc, 256, (Cl + 64) * sizeof(float), stream>>>(dw.p, dww, dwb, lw, lb, X, B, Tc, Cl, dw.bs_rows(), dw.hist);
    c->launches++;
    { GemmEpilogue e = none; e.bias = R.need<float>(p + ".pw1.b", 4 * Cl); e.act = ACT_GELU; e.out_act = W;
      R.gemm(X, Tc, Cl, (int64_t)Tc * Cl, (p + ".pw1.w").c_str(), 4 * Cl, 1, &zero, e, {}); }
    // the stream's last stage writes decoder.0's input; every other stage writes Z, whose input `cur` is consumed
    const HistBuf o = (s && i + 1 == g.n_upsampling_ratios) ? s->in : HistBuf{Z, 0, Cl, Tc};
    { GemmEpilogue e = none; e.bias = R.need<float>(p + ".pw2.b", Cl); e.scale = R.need<float>(p + ".gamma", Cl); e.resid = dw.cur(); e.out_raw = o.cur();
      GemmViews v; v.resid_bs = dw.bs(); v.raw_bs = o.bs();
      R.gemm(W, Tc, 4 * Cl, (int64_t)Tc * 4 * Cl, (p + ".pw2.w").c_str(), Cl, 1, &zero, e, v); }
    cur = o.cur();
  }
  const HistBuf in = s ? s->in : HistBuf{Z, 0, Cl, Tc};
  capture(2, in.cur(), (int64_t)B * Tc * Cl);
  // ---- decoder.0: conv k7 latent -> decoder_dim; epilogue applies block 0's SnakeBeta (…v2.py:857,646)
  int C = g.decoder_dim;
  {
    const HistBuf o = block_in(0, C, Tc);
    const int sh[7] = {-6, -5, -4, -3, -2, -1, 0};
    GemmEpilogue e = none; e.bias = R.need<float>("dec.in.b", C); e.act = ACT_SNAKE; e.snake_ea = R.need<float>("dec.0.snake_ea", C);
    e.snake_ib = R.need<float>("dec.0.snake_ib", C); e.out_act = o.cur();
    GemmViews v = view_in(in, Tc); v.act_bs = o.bs();
    R.gemm(in.p, Tc, Cl, in.bs(), "dec.in.w", C, 7, sh, e, v);
    capture(3, o.cur(), (int64_t)B * Tc * C);  // SnakeBeta(decoder.0 output) with block 0's leading activation
  }
  // ---- decoder blocks (…v2.py:638-658, :619-635): residual stream y = Y, updated in place by every unit's c2
  for (int bi = 0; bi < nr && !R.err; ++bi) {
    const int r = g.upsample_rates[bi];
    const int Co = C / 2;
    const std::string p = "dec." + std::to_string(bi);
    {
      const HistBuf a = block_in(bi, C, Tc), o = unit_in(bi, 0, Co, Tc * r);
      const int sh[2] = {0, -1};
      GemmEpilogue e = none; e.bias = R.need<float>(p + ".ct.b", Co); e.cmod = Co; e.out_raw = Y; e.act = ACT_SNAKE;
      e.snake_ea = R.need<float>(p + ".0.s1_ea", Co); e.snake_ib = R.need<float>(p + ".0.s1_ib", Co); e.out_act = o.cur();
      GemmViews v = view_in(a, Tc); v.act_bs = o.bs();
      R.gemm(a.p, Tc, C, a.bs(), (p + ".ct.w").c_str(), r * Co, 2, sh, e, v);
    }
    Tc *= r;
    C = Co;
    for (int u = 0; u < 3 && !R.err; ++u) {
      const int dil = u == 0 ? 1 : (u == 1 ? 3 : 9);
      const std::string q = p + "." + std::to_string(u);
      {
        const HistBuf a = unit_in(bi, u, C, Tc);
        int sh[7];
        for (int j = 0; j < 7; ++j) sh[j] = -(6 - j) * dil;
        GemmEpilogue e = none; e.bias = R.need<float>(q + ".c1.b", C); e.act = ACT_SNAKE; e.snake_ea = R.need<float>(q + ".s2_ea", C);
        e.snake_ib = R.need<float>(q + ".s2_ib", C); e.out_act = Z;
        R.gemm(a.p, Tc, C, a.bs(), (q + ".c1.w").c_str(), C, 7, sh, e, view_in(a, Tc));
      }
      {
        // next activation: next unit's act1, or the next block's leading snake, or the final snake
        std::string nx = (u < 2) ? (p + "." + std::to_string(u + 1) + ".s1")
                                 : (bi + 1 < nr ? ("dec." + std::to_string(bi + 1) + ".snake") : std::string("dec.out.snake"));
        const HistBuf o = (u < 2) ? unit_in(bi, u + 1, C, Tc) : block_in(bi + 1, C, Tc);
        // in place: the epilogue thread that writes a residual element has read it first
        GemmEpilogue e = none; e.bias = R.need<float>(q + ".c2.b", C); e.resid = Y; e.out_raw = Y; e.act = ACT_SNAKE;
        e.snake_ea = R.need<float>(nx + "_ea", C); e.snake_ib = R.need<float>(nx + "_ib", C); e.out_act = o.cur();
        GemmViews v; v.act_bs = o.bs();
        R.gemm(Z, Tc, C, (int64_t)Tc * C, (q + ".c2.w").c_str(), C, 1, &zero, e, v);
      }
    }
    capture(4 + bi, Y, (int64_t)B * Tc * C);  // the block's output (residual stream after its three units)
  }
  if (R.err) return 1;
  // ---- final conv k7 + clamp
  {
    const HistBuf a = block_in(nr, C, Tc);
    const float* w = R.need<float>("dec.out.w", (int64_t)7 * C);
    const float* bsrc = R.need<float>("dec.out.b", 1);
    if (R.err) return 1;
    final_conv_kernel<<<1184, 256, 0, stream>>>(a.p, w, bsrc, wav, B, Tc, C, a.bs_rows(), a.hist, rp, c->total_up);  // bias read on the device
    c->launches++;
  }
  Q3_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int q3_codec_forward(q3_codec* c, const int32_t* codes_dev, int32_t B, int32_t T, float* wav_dev, void* stream_) {
  Q3_REQUIRE(c && c->finalized, "codec not finalized");
  Q3_REQUIRE(codes_dev && wav_dev && B >= 1 && T >= 1, "bad arguments");
  Q3_REQUIRE(T <= c->cfg.max_frames, "T=%d exceeds max_frames=%d", T, c->cfg.max_frames);
  Q3_CUDA(cudaSetDevice(c->cfg.device));
  const size_t need = scratch_per_frame(c->cfg) * (size_t)B * T;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (need > c->buf_elems) {
    c->buf_elems = 0;
    if (alloc_scratch(c->store, c->buf, need, stream)) return 1;
    c->buf_elems = need;
  }
  return decode_frames(c, nullptr, codes_dev, B, T, nullptr, c->buf, wav_dev, stream);
}

static int hist_alloc(q3_codec_stream* s, HistBuf* h, int hist, int C, int cap) {
  *h = HistBuf{nullptr, hist, C, cap};
  void* p = nullptr;
  // zero history == the causal left padding of a fresh stream
  if (s->store.alloc(&p, (size_t)s->B * h->bs_rows() * C * 2 + 256, true)) return 1;
  h->p = reinterpret_cast<bf16*>(p);
  return 0;
}

extern "C" int q3_codec_stream_open(q3_codec* c, int32_t B, int32_t max_packet_frames, q3_codec_stream** out) {
  Q3_REQUIRE(c && c->finalized && out, "codec not finalized");
  Q3_REQUIRE(B >= 1 && B <= c->cfg.max_batch && max_packet_frames >= 1 && max_packet_frames <= c->cfg.max_frames, "bad arguments");
  const q3_codec_cfg& g = c->cfg;
  Q3_REQUIRE(g.n_upsampling_ratios >= 1, "streaming decoder expects at least one upsampling stage");
  const int nhist = 3 + g.num_layers + g.n_upsampling_ratios + 4 * g.n_upsample_rates;  // pre, in, out; kv; dw; ct + 3 c1
  Q3_REQUIRE(nhist <= kRollMax, "streaming decoder needs %d history buffers, at most %d supported", nhist, kRollMax);
  Q3_CUDA(cudaSetDevice(g.device));
  q3_codec_stream* s = new q3_codec_stream();
  s->c = c; s->B = B; s->nmax = max_packet_frames;
  const int n = max_packet_frames, Cl = g.latent_dim, nh = g.num_heads, hd = g.head_dim;
  int rc = hist_alloc(s, &s->pre, 2, g.codebook_dim, n);
  s->kv.resize(g.num_layers);
  for (int l = 0; l < g.num_layers && !rc; ++l) rc = hist_alloc(s, &s->kv[l], g.sliding_window - 1, 2 * nh * hd, n);
  int Tc = n;
  s->dw.resize(g.n_upsampling_ratios);
  for (int i = 0; i < g.n_upsampling_ratios && !rc; ++i) { Tc *= g.upsampling_ratios[i]; rc = hist_alloc(s, &s->dw[i], 6, Cl, Tc); }
  if (!rc) rc = hist_alloc(s, &s->in, 6, Cl, Tc);
  int C = g.decoder_dim;
  s->ct.resize(g.n_upsample_rates);
  s->c1.resize(g.n_upsample_rates);
  for (int bi = 0; bi < g.n_upsample_rates && !rc; ++bi) {
    rc = hist_alloc(s, &s->ct[bi], 1, C, Tc);
    Tc *= g.upsample_rates[bi];
    C /= 2;
    s->c1[bi].resize(3);
    const int dil[3] = {1, 3, 9};
    for (int u = 0; u < 3 && !rc; ++u) rc = hist_alloc(s, &s->c1[bi][u], 6 * dil[u], C, Tc);
  }
  if (!rc) rc = hist_alloc(s, &s->out, 6, C, Tc);
  if (!rc) rc = alloc_scratch(s->store, s->buf, scratch_per_frame(g) * (size_t)B * n, nullptr);
  void* rp = nullptr;
  if (!rc) rc = s->store.alloc(&rp, (size_t)2 * B * sizeof(int32_t), true);
  s->rp = reinterpret_cast<int32_t*>(rp);
  s->pos.assign(B, 0);
  s->rp_h.assign(2 * B, 0);
  if (rc) { delete s; return 1; }
  Q3_CUDA(cudaDeviceSynchronize());
  *out = s;
  return 0;
}

extern "C" void q3_codec_stream_close(q3_codec_stream* s) { delete s; }

// the history buffers of a stream as a table for the roll and reset kernels.  A buffer's capacity is max_packet_frames
// times its stage's rows per frame, so its factor is cap / nmax.  q3_codec_stream_open bounds the number of buffers.
static RollTable hist_table(const q3_codec_stream* s) {
  RollTable tb{};
  for_each_hist(s, [&](const HistBuf& h) {
    if (h.hist > 0) tb.e[tb.n++] = RollEntry{h.p, h.hist, h.cap / s->nmax, h.C, h.bs_rows()};
  });
  return tb;
}

// frames pushed to `row` since its last reset; -1 for a bad row
extern "C" int q3_codec_stream_row_position(q3_codec_stream* s, int32_t row) {
  if (!s || row < 0 || row >= s->B) { q3_set_err("row %d out of range [0, %d)", row, s ? s->B : 0); return -1; }
  return s->pos[row];
}

// next frames of every row: codes_dev int32 [B][K][n]; row b takes the first counts_host[b] of them -> wav_dev fp32
// [B][n * total_upsample], zero past each row's count.  Every argument is checked before any device work.
extern "C" int q3_codec_stream_step_rows(q3_codec_stream* s, const int32_t* codes_dev, int32_t n, const int32_t* counts_host,
                                         float* wav_dev, void* stream_) {
  Q3_REQUIRE(s && codes_dev && counts_host && wav_dev, "null argument");
  const q3_codec_cfg& g = s->c->cfg;
  for (int b = 0; b < s->B; ++b) {
    Q3_REQUIRE((int64_t)s->pos[b] + counts_host[b] <= g.max_frames,
               "row %d: position %d + %d frames exceeds the RoPE table (max_frames %d)", b, s->pos[b], counts_host[b], g.max_frames);
    Q3_REQUIRE(counts_host[b] >= 0 && counts_host[b] <= n, "row %d: count %d outside [0, %d]", b, counts_host[b], n);
  }
  Q3_REQUIRE(n >= 1 && n <= s->nmax, "packet of %d frames (max %d)", n, s->nmax);
  Q3_CUDA(cudaSetDevice(g.device));
  cudaStream_t stream = (cudaStream_t)stream_;
  for (int b = 0; b < s->B; ++b) { s->rp_h[b] = s->pos[b]; s->rp_h[s->B + b] = counts_host[b]; }
  Q3_CUDA(cudaMemcpyAsync(s->rp, s->rp_h.data(), (size_t)2 * s->B * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  if (decode_frames(s->c, s, codes_dev, s->B, n, s->rp, s->buf, wav_dev, stream)) return 1;
  const RollTable roll = hist_table(s);
  roll_history_kernel<<<roll.n * s->B, 128, 0, stream>>>(roll, s->rp, s->B);
  s->c->launches++;
  Q3_CUDA(cudaGetLastError());
  for (int b = 0; b < s->B; ++b) s->pos[b] += counts_host[b];
  return 0;
}

// forget the listed rows: their next packet starts a new utterance at position 0; the other rows are untouched
extern "C" int q3_codec_stream_reset_rows(q3_codec_stream* s, int32_t n, const int32_t* rows_host, void* stream_) {
  Q3_REQUIRE(s && rows_host, "null argument");
  for (int i = 0; i < n; ++i) Q3_REQUIRE(rows_host[i] >= 0 && rows_host[i] < s->B, "reset row %d out of range [0, %d)", rows_host[i], s->B);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < i; ++j) Q3_REQUIRE(rows_host[i] != rows_host[j], "reset row %d listed twice", rows_host[i]);
  Q3_REQUIRE(n >= 0 && n <= s->B, "%d rows to reset, the stream has %d", n, s->B);
  if (n == 0) return 0;
  std::vector<int32_t> mask(s->B, 0);
  for (int i = 0; i < n; ++i) mask[rows_host[i]] = 1;
  Q3_CUDA(cudaSetDevice(s->c->cfg.device));
  cudaStream_t stream = (cudaStream_t)stream_;
  for (int b = 0; b < s->B; ++b) { s->rp_h[b] = mask[b] ? 0 : s->pos[b]; s->rp_h[s->B + b] = mask[b]; }
  Q3_CUDA(cudaMemcpyAsync(s->rp, s->rp_h.data(), (size_t)2 * s->B * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  const RollTable tb = hist_table(s);
  reset_history_kernel<<<tb.n * s->B, 128, 0, stream>>>(tb, s->rp, s->B);
  Q3_CUDA(cudaGetLastError());
  for (int b = 0; b < s->B; ++b) if (mask[b]) s->pos[b] = 0;
  return 0;
}

// row dst_rows[i] of dst becomes row src_rows[i] of src: every history buffer's `hist` rows and the position.  Used to
// seed a row with a reference prefix decoded elsewhere (qwen3_tts_model.py:612-631 decodes cat(ref_code, codes)).  The
// source rows' pairs go up through dst's rp buffer ([0, n) source rows, [B, B + n) destination rows).
extern "C" int q3_codec_stream_copy_rows(q3_codec_stream* dst, const q3_codec_stream* src, int32_t n, const int32_t* src_rows_host,
                                         const int32_t* dst_rows_host, void* stream_) {
  Q3_REQUIRE(dst && src, "null stream");
  Q3_REQUIRE(src != dst, "source and destination are the same stream");
  Q3_REQUIRE(src->c == dst->c, "source and destination streams belong to different codecs");
  Q3_REQUIRE(n >= 0 && n <= dst->B, "%d rows to copy, the destination stream has %d", n, dst->B);
  if (n == 0) return 0;
  Q3_REQUIRE(src_rows_host && dst_rows_host, "null argument");
  for (int i = 0; i < n; ++i) {
    Q3_REQUIRE(src_rows_host[i] >= 0 && src_rows_host[i] < src->B, "source row %d out of range [0, %d)", src_rows_host[i], src->B);
    Q3_REQUIRE(dst_rows_host[i] >= 0 && dst_rows_host[i] < dst->B, "destination row %d out of range [0, %d)", dst_rows_host[i], dst->B);
    for (int j = 0; j < i; ++j) Q3_REQUIRE(dst_rows_host[i] != dst_rows_host[j], "destination row %d listed twice", dst_rows_host[i]);
  }
  const RollTable td = hist_table(dst), ts = hist_table(src);
  Q3_REQUIRE(td.n == ts.n, "history tables differ (%d and %d buffers)", td.n, ts.n);
  CopyTable tb{};
  tb.n = td.n;
  for (int k = 0; k < td.n; ++k) {
    Q3_REQUIRE(td.e[k].hist == ts.e[k].hist && td.e[k].C == ts.e[k].C, "history buffer %d differs between the streams", k);
    tb.e[k] = CopyEntry{td.e[k].p, ts.e[k].p, td.e[k].hist, td.e[k].C, td.e[k].bs_rows, ts.e[k].bs_rows};
  }
  Q3_CUDA(cudaSetDevice(dst->c->cfg.device));
  cudaStream_t stream = (cudaStream_t)stream_;
  for (int i = 0; i < n; ++i) { dst->rp_h[i] = src_rows_host[i]; dst->rp_h[dst->B + i] = dst_rows_host[i]; }
  Q3_CUDA(cudaMemcpyAsync(dst->rp, dst->rp_h.data(), (size_t)2 * dst->B * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  copy_rows_kernel<<<tb.n * n, 256, 0, stream>>>(tb, dst->rp, dst->B, n);
  Q3_CUDA(cudaGetLastError());
  for (int i = 0; i < n; ++i) dst->pos[dst_rows_host[i]] = src->pos[src_rows_host[i]];
  return 0;
}
