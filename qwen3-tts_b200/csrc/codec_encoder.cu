// Qwen3-TTS-Tokenizer-12Hz codec ENCODER on H100 (sm_90a): 24 kHz waveform -> 16 x 12.5 Hz codes.
// Replaces Qwen3TTSTokenizerV2Model.encode (qwen_tts/core/tokenizer_12hz/modeling_qwen3_tts_tokenizer_v2.py:961-991),
// i.e. transformers' MimiModel._encode_frame (modeling_mimi.py:1455-1488): SEANet encoder (:454-496) -> 8-layer
// sliding-window transformer (:926-993, :1015-1140) -> stride-2 downsample (:1420-1430) -> split RVQ encode (:1311-1338).
//
// The output is DISCRETE (argmin over 2048 centroids, 16 residual levels deep), so this path computes in fp32 end to
// end: a bf16 tensor-core pipeline would flip nearest-centroid decisions relative to the fp32 reference and every
// flip cascades down the residual chain.  Activations are [B][C][T] fp32 (time contiguous, the reference's own
// layout); every Conv1d / Linear is one launch of the register-tiled direct convolution of conv_f32.cu, which the
// speaker encoder shares, with the preceding ELU, the bias, GELU, LayerScale and the residual add fused in.  It is a
// first correct version: ~12 GFLOP per 3 s of audio on CUDA cores; moving the strided convolutions onto wgmma (tf32) is
// the follow-up once parity is pinned.
//
// One layer walker (encode_segment) serves the one-shot q3_codec_enc_encode and the stateful stream
// (q3_codec_enc_stream_*): the one-shot passes plain views of its scratch, the stream history-prefixed buffers that carry
// each row's causal state, so a streamed frame runs the same kernels on the same values as the one-shot and its codes
// are bit-identical (DESIGN.md §4.4).
#include "common.cuh"
#include "conv_f32.cuh"
#include "dev_store.h"
#include "row_state.h"
#include "../../include/qwen3tts_b200.h"

#include <algorithm>
#include <string>
#include <vector>

#include "codec_encoder_kernels.cuh"

struct q3_codec_enc {
  q3_codec_enc_cfg cfg;
  DevStore store{"codec encoder"};
  float* buf[3] = {nullptr, nullptr, nullptr};
  size_t buf_elems = 0;
  const float** d_ptrs = nullptr;  // [3][nq] device pointer tables (E, ET, E2)
  std::vector<std::pair<int, std::pair<float*, int64_t>>> captures;  // stage ordinal -> (dst, capacity)
  bool finalized = false;
  int launches = 0;
  int hop = 1;
};

extern "C" int q3_codec_enc_create(const q3_codec_enc_cfg* cfg, q3_codec_enc** out) {
  Q3_REQUIRE(cfg && out, "null argument");
  Q3_CUDA(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  Q3_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  Q3_REQUIRE(prop.major == 9 && prop.minor == 0, "this library is built for sm_90a (H100); device is sm_%d%d", prop.major, prop.minor);
  Q3_REQUIRE(cfg->n_ratios >= 1 && cfg->n_ratios <= 8, "1..8 downsampling ratios");
  Q3_REQUIRE(cfg->head_dim % 2 == 0 && cfg->head_dim <= 64, "encoder head_dim must be even and <= 64");
  Q3_REQUIRE(cfg->num_heads * cfg->head_dim == cfg->hidden_size, "num_heads * head_dim must equal hidden_size");
  Q3_REQUIRE(cfg->num_quantizers >= cfg->num_semantic_quantizers && cfg->num_semantic_quantizers >= 1 &&
                 cfg->num_quantizers <= 64, "bad quantizer counts");
  Q3_REQUIRE(cfg->codebook_dim <= 1024, "codebook_dim > 1024 unsupported");
  Q3_REQUIRE(cfg->max_frames >= 1, "max_frames (rope table rows) must be positive");
  if (conv_f32_init()) return 1;
  q3_codec_enc* e = new q3_codec_enc();
  e->cfg = *cfg;
  e->hop = cfg->downsample_stride;
  for (int i = 0; i < cfg->n_ratios; ++i) e->hop *= cfg->ratios[i];
  *out = e;
  return 0;
}

extern "C" void q3_codec_enc_destroy(q3_codec_enc* e) { delete e; }

extern "C" int q3_codec_enc_hop(q3_codec_enc* e) { return e ? e->hop : 0; }
extern "C" int q3_codec_enc_last_launch_count(q3_codec_enc* e) { return e ? e->launches : 0; }

extern "C" int q3_codec_enc_load_tensor(q3_codec_enc* e, const char* name, const float* dev, const int64_t* shape, int32_t ndim) {
  Q3_REQUIRE(e && name && dev && shape, "null argument");
  Q3_CUDA(cudaSetDevice(e->cfg.device));
  return e->store.load(name, dev, shape, ndim, DT_F32);
}

extern "C" int q3_codec_enc_finalize(q3_codec_enc* e) {
  Q3_REQUIRE(e, "null encoder");
  const q3_codec_enc_cfg& g = e->cfg;
  Q3_CUDA(cudaSetDevice(g.device));
  const int nq = g.num_quantizers, K = g.codebook_size, D = g.codebook_dim;
  std::vector<const float*> tab(3 * nq);
  const DevStore& S = e->store;
  for (int q = 0; q < nq; ++q) {
    const std::string p = "rvq." + std::to_string(q);
    if (!(tab[q] = S.need<float>(p + ".e", (int64_t)K * D)) || !(tab[nq + q] = S.need<float>(p + ".et", (int64_t)K * D)) ||
        !(tab[2 * nq + q] = S.need<float>(p + ".e2", K)))
      return 1;
  }
  if (!S.need<float>("rope.cos", (int64_t)g.max_frames * (g.head_dim / 2)) ||
      !S.need<float>("rope.sin", (int64_t)g.max_frames * (g.head_dim / 2)) || !S.need<float>("rvq.sem.proj.w", (int64_t)D * g.hidden_size) ||
      !S.need<float>("rvq.ac.proj.w", (int64_t)D * g.hidden_size) ||
      !S.need<float>("down.w", (int64_t)g.hidden_size * g.hidden_size * 2 * g.downsample_stride))
    return 1;
  void* p = nullptr;
  if (e->store.alloc(&p, tab.size() * sizeof(float*))) return 1;
  e->d_ptrs = reinterpret_cast<const float**>(p);
  Q3_CUDA(cudaMemcpy(p, tab.data(), tab.size() * sizeof(float*), cudaMemcpyHostToDevice));
  e->finalized = true;
  return 0;
}

// Test hook: after stage `stage` of the next q3_codec_enc_encode (ordinals: conv0, then per ratio [res, down], conv_last,
// one per transformer layer, downsample) copy its activation [B][C][T] to dst (fp32, up to `capacity` floats).
extern "C" int q3_codec_enc_debug_capture(q3_codec_enc* e, int32_t stage, float* dst_dev, int64_t capacity) {
  Q3_REQUIRE(e, "null encoder");
  if (stage < 0) { e->captures.clear(); return 0; }
  e->captures.push_back({stage, {dst_dev, capacity}});
  return 0;
}

namespace {

// One activation of the layer walker: [B][C][ld] fp32, `hist` columns of history before the segment's first column.
// The one-shot views its scratch buffers with hist 0 (the convolutions' zero padding is the causal left padding); a
// stream's history-prefixed buffers carry the previous segments' last columns instead.
struct EncBuf {
  float* p = nullptr;
  int C = 0, hist = 0, ld = 0;
  float* cur() const { return p + hist; }
  size_t bs() const { return (size_t)C * ld; }
  EncBuf row(int b) const { EncBuf r = *this; r.p += (size_t)b * bs(); return r; }
};

// Every tensor of the walker.  x[i]: input of ratio i's residual block (x[n_ratios]: conv_last's input); y[i]: its k3
// conv's output; z[i]: the block's output = the downsample's input; h: the transformer's residual stream, read back by
// the final downsample; kv[l]: layer l's rotated keys and values (k channels [0, C), v [C, 2C) from `cur`); a: normed
// activations / attention output / downsample output; q: qkv / MLP hidden / RVQ projections.
struct EncViews {
  EncBuf wav, x[9], y[8], z[8], h, a, q;
  std::vector<EncBuf> kv;
  EncViews row(int b) const {  // batch row b of every history buffer as a one-row view; scratch stays at row 0
    EncViews v = *this;
    v.wav = wav.row(b); v.h = h.row(b);
    for (EncBuf& t : v.x) t = t.row(b);
    for (EncBuf& t : v.z) t = t.row(b);
    for (EncBuf& t : v.kv) t = t.row(b);
    return v;
  }
};

struct EncRunner {
  q3_codec_enc* e;
  cudaStream_t st;
  int B;
  bool capturing;
  int stage = 0;

  // y = conv(x) over the segment's Tin valid input columns; the causal left padding (k - stride columns) comes from x's
  // history when it has one, else from the kernel's zero / replicate padding.  Columns past Tin are padded on the right
  // ("extra padding", modeling_mimi.py:273-285).  res (optional) has y's layout.
  int conv(const std::string& wname, const EncBuf& x, const EncBuf& y, int Cin, int Cout, int Tin, int k, int stride,
           int replicate, bool elu_in, bool gelu_out, const EncBuf* res, const std::string& scale_name, bool has_bias, int* Tout_) {
    const DevStore& S = e->store;
    ConvF32Args a{};
    if (!(a.w = S.need<float>(wname + ".w", (int64_t)Cout * Cin * k))) return 1;
    if (has_bias && !(a.bias = S.need<float>(wname + ".b", Cout))) return 1;
    if (!scale_name.empty() && !(a.scale = S.need<float>(scale_name, Cout))) return 1;
    const int pad_left = k - stride;               // causal: padding_total on the left (modeling_mimi.py:343-345)
    const int from_hist = x.hist > 0 ? pad_left : 0;
    Q3_REQUIRE(x.hist == 0 || x.hist >= pad_left, "%s: %d history columns, the conv reads back %d", wname.c_str(), x.hist, pad_left);
    Q3_REQUIRE(x.C == Cin && y.C == Cout, "%s: views of %d and %d channels for a %d -> %d conv", wname.c_str(), x.C, y.C, Cin, Cout);
    Q3_REQUIRE(!res || (res->ld == y.ld && res->C == y.C), "%s: residual view differs from the output's", wname.c_str());
    a.x = x.cur() - from_hist; a.y = y.cur(); a.res = res ? res->cur() : nullptr;
    a.xC = x.C; a.yC = y.C;
    a.Cin = Cin; a.Cout = Cout; a.Tin = Tin + from_hist; a.k = k; a.stride = stride; a.dil = 1;
    a.pad_left = pad_left - from_hist;
    a.Tout = (Tin + stride - 1) / stride;          // right "extra padding" up to a stride multiple (:273-285)
    a.pad = replicate ? PAD_REPLICATE : PAD_ZERO;
    a.act_in = elu_in ? IN_ELU : IN_NONE;
    a.act_out = gelu_out ? OUT_GELU : OUT_NONE;
    if (conv_f32_launch(a, B, st, x.ld, y.ld)) return 1;
    ++e->launches;
    if (Tout_) *Tout_ = a.Tout;
    return 0;
  }
  void capture(const EncBuf& x, int C, int T) {
    if (!capturing) return;
    for (auto& c : e->captures)
      if (c.first == stage) {
        const int64_t n = std::min<int64_t>((int64_t)B * C * T, c.second.second);
        cudaMemcpyAsync(c.second.first, x.cur(), (size_t)n * 4, cudaMemcpyDeviceToDevice, st);
      }
    ++stage;
  }
};

// The encoder's layer sequence over a segment of T samples of every row (the one-shot: the whole clip; a stream: a
// packet of whole frames, or a row's final partial frame), frames of row b at 25 Hz positions rp[b] + t of which the
// first rp[B + b] are the row's (rp == nullptr: position 0, all).  Writes codes [B][nq][frames(T)].  Every layer is
// causal and row-local, so a row's frames past its count change nothing before them; the stream never lets them reach
// its history and masks their codes to -1.  Each output column is computed by the same instruction sequence whether it
// is streamed or not: the convolutions accumulate in an order independent of t, LayerNorm and RVQ work per column, and
// attention walks the same keys in the same order.
int encode_segment(q3_codec_enc* e, const EncViews& v, int B, int T, const int* rp, int32_t* codes_dev, cudaStream_t st) {
  const q3_codec_enc_cfg& g = e->cfg;
  EncRunner r{e, st, B, rp == nullptr};
  // ---- SEANet encoder (modeling_mimi.py:454-496)
  int t = T, c = g.num_filters, to = 0;
  if (r.conv("enc.conv0", v.wav, v.x[0], 1, c, t, g.kernel_size, 1, 0, false, false, nullptr, "", true, &to)) return 1;
  r.capture(v.x[0], c, t);
  for (int i = 0; i < g.n_ratios; ++i) {
    const std::string p = "enc.res" + std::to_string(i);
    // x + conv_k1(ELU(conv_k3(ELU(x))))  (:437-451)
    if (r.conv(p + ".a", v.x[i], v.y[i], c, c / g.compress, t, g.residual_kernel_size, 1, 0, true, false, nullptr, "", true, &to))
      return 1;
    if (r.conv(p + ".b", v.y[i], v.z[i], c / g.compress, c, t, 1, 1, 0, true, false, &v.x[i], "", true, &to)) return 1;
    r.capture(v.z[i], c, t);
    if (r.conv("enc.down" + std::to_string(i), v.z[i], v.x[i + 1], c, 2 * c, t, 2 * g.ratios[i], g.ratios[i], 0, true, false,
               nullptr, "", true, &to))
      return 1;
    t = to; c *= 2;
    r.capture(v.x[i + 1], c, t);
  }
  const EncBuf& H = v.h;
  const EncBuf& A = v.a;
  const EncBuf& Z = v.q;
  const EncBuf F{Z.p, g.intermediate_size, 0, Z.ld};  // the MLP hidden, in Z's scratch
  if (r.conv("enc.conv_last", v.x[g.n_ratios], H, c, g.hidden_size, t, g.last_kernel_size, 1, 0, true, false, nullptr, "", true, &to))
    return 1;
  r.capture(H, g.hidden_size, t);
  // ---- transformer (:926-993): h lives in H; A = normed / attention output, Z = qkv / mlp hidden
  const int C = g.hidden_size, nh = g.num_heads, hd = g.head_dim, I = g.intermediate_size;
  const float* cosT = e->store.need<float>("rope.cos", (int64_t)g.max_frames * (hd / 2));
  const float* sinT = e->store.need<float>("rope.sin", (int64_t)g.max_frames * (hd / 2));
  if (!cosT || !sinT) return 1;
  for (int l = 0; l < g.num_layers; ++l) {
    const std::string p = "tr." + std::to_string(l);
    const DevStore& S = e->store;
    const float *l1w = S.need<float>(p + ".ln1.w", C), *l1b = S.need<float>(p + ".ln1.b", C), *l2w = S.need<float>(p + ".ln2.w", C),
                *l2b = S.need<float>(p + ".ln2.b", C);
    if (!l1w || !l1b || !l2w || !l2b) return 1;
    const EncBuf& KV = v.kv[l];
    const bool own_kv = rp != nullptr;  // a stream's window buffer (the one-shot's KV views the k and v thirds of qkv)
    dim3 lg((t + 31) / 32, B);
    layernorm_ct_kernel<<<lg, 256, 0, st>>>(H.cur(), H.ld, l1w, l1b, A.cur(), A.ld, C, t, g.norm_eps);
    if (r.conv(p + ".qkv", A, Z, C, 3 * C, t, 1, 1, 0, false, false, nullptr, "", false, &to)) return 1;
    rope_ct_kernel<<<dim3((t + 127) / 128, (own_kv ? 3 : 2) * nh * (hd / 2), B), 128, 0, st>>>(
        Z.cur(), cosT, sinT, C, t, nh, hd, rp, B, own_kv ? KV.cur() : nullptr, (long long)KV.bs(), KV.ld);
    swa_ct_kernel<64><<<dim3((t + 127) / 128, nh, B), 128, 0, st>>>(Z.cur(), KV.p, (long long)KV.bs(), KV.ld, KV.hist, A.cur(), C,
                                                                     t, hd, g.sliding_window, 1.0f / sqrtf((float)hd), rp);
    if (r.conv(p + ".o", A, H, C, C, t, 1, 1, 0, false, false, &H, p + ".ls1", false, &to)) return 1;  // h += ls1 * o_proj(attn)
    layernorm_ct_kernel<<<lg, 256, 0, st>>>(H.cur(), H.ld, l2w, l2b, A.cur(), A.ld, C, t, g.norm_eps);
    if (r.conv(p + ".fc1", A, F, C, I, t, 1, 1, 0, false, true, nullptr, "", false, &to)) return 1;
    if (r.conv(p + ".fc2", F, H, I, C, t, 1, 1, 0, false, false, &H, p + ".ls2", false, &to)) return 1;  // h += ls2 * fc2(gelu(fc1))
    e->launches += 4;
    r.capture(H, C, t);
  }
  // ---- 25 Hz -> 12.5 Hz (:1420-1430: k = 2*stride, no bias, replicate padding)
  if (H.hist > 0) {
    seed_replicate_kernel<<<dim3((C + 255) / 256, B), 256, 0, st>>>(H.p, C, H.hist, H.ld, rp, B);
    ++e->launches;
  }
  const int t3 = (t + g.downsample_stride - 1) / g.downsample_stride;
  const EncBuf A3{A.p, C, 0, t3};  // the 12.5 Hz activations, in A's scratch
  if (r.conv("down", H, A3, C, C, t, 2 * g.downsample_stride, g.downsample_stride, 1, false, false, nullptr, "", false, &to)) return 1;
  r.capture(A3, C, t3);
  // ---- split RVQ (:1311-1338)
  const int D = g.codebook_dim, nq = g.num_quantizers;
  const EncBuf Rs{Z.p, D, 0, t3}, Ra{Z.p + (size_t)B * D * t3, D, 0, t3};
  if (r.conv("rvq.sem.proj", A3, Rs, C, D, t3, 1, 1, 0, false, false, nullptr, "", false, &to)) return 1;
  if (r.conv("rvq.ac.proj", A3, Ra, C, D, t3, 1, 1, 0, false, false, nullptr, "", false, &to)) return 1;
  RvqArgs ra{};
  ra.r_sem = Rs.p; ra.r_ac = Ra.p; ra.E = e->d_ptrs; ra.ET = e->d_ptrs + nq; ra.E2 = e->d_ptrs + 2 * nq;
  ra.codes = codes_dev; ra.D = D; ra.K = g.codebook_size; ra.T = t3; ra.nq = nq; ra.nsem = g.num_semantic_quantizers;
  rvq_encode_kernel<<<dim3(t3, B), 256, (size_t)(D + 16) * sizeof(float), st>>>(ra);
  ++e->launches;
  if (rp) {
    const int total = B * nq * t3;
    mask_codes_kernel<<<(total + 255) / 256, 256, 0, st>>>(codes_dev, nq, t3, rp, B, g.downsample_stride);
    ++e->launches;
  }
  Q3_CUDA(cudaGetLastError());
  return 0;
}

// scratch elements of the walker per batch row over a segment of T samples: the one-shot's ping-pong buffers each hold
// the largest [C][T] activation (the stream keeps its history-prefixed tensors elsewhere and needs less, but shares the
// same three buffers)
size_t scratch_per_row(const q3_codec_enc_cfg& g, int T) {
  int t = T, c = g.num_filters;
  size_t need = (size_t)c * t;
  for (int i = 0; i < g.n_ratios; ++i) { t = (t + g.ratios[i] - 1) / g.ratios[i]; c *= 2; need = std::max(need, (size_t)c * t); }
  need = std::max(need, (size_t)std::max(3 * g.hidden_size, g.intermediate_size) * t);
  const int t3 = (t + g.downsample_stride - 1) / g.downsample_stride;
  return std::max(need, (size_t)2 * g.codebook_dim * t3);  // both RVQ projections
}

int grow_scratch(q3_codec_enc* e, size_t need, cudaStream_t st) {
  if (need <= e->buf_elems) return 0;
  e->buf_elems = 0;
  for (float*& b : e->buf)
    if (e->store.grow(&b, need * 4, st)) return 1;
  e->buf_elems = need;
  return 0;
}

}  // namespace

extern "C" int q3_codec_enc_frames(q3_codec_enc* e, int32_t T) {
  if (!e || T <= 0) return 0;
  int t = T;
  for (int i = 0; i < e->cfg.n_ratios; ++i) t = (t + e->cfg.ratios[i] - 1) / e->cfg.ratios[i];
  return (t + e->cfg.downsample_stride - 1) / e->cfg.downsample_stride;
}

// 25 Hz frames (transformer columns) of a T-sample segment
static int frames25(const q3_codec_enc_cfg& g, int T) {
  int t = T;
  for (int i = 0; i < g.n_ratios; ++i) t = (t + g.ratios[i] - 1) / g.ratios[i];
  return t;
}

extern "C" int q3_codec_enc_encode(q3_codec_enc* e, const float* wav_dev, int32_t B, int32_t T, int32_t* codes_dev, void* stream_) {
  Q3_REQUIRE(e && e->finalized, "codec encoder not finalized");
  Q3_REQUIRE(wav_dev && codes_dev && B >= 1 && T >= 1, "bad arguments");
  const q3_codec_enc_cfg& g = e->cfg;
  Q3_CUDA(cudaSetDevice(g.device));
  cudaStream_t st = (cudaStream_t)stream_;
  e->launches = 0;
  const int t25 = frames25(g, T);
  Q3_REQUIRE(t25 <= g.max_frames, "%d transformer frames exceed max_frames %d", t25, g.max_frames);
  // ---- workspace: three ping-pong buffers sized for the largest [C][T] activation of this request
  if (grow_scratch(e, scratch_per_row(g, T) * (size_t)B, st)) return 1;
  float *X = e->buf[0], *Y = e->buf[1], *Z = e->buf[2];
  // every view is a plain [B][C][T] scratch tensor: the walker's one-shot mapping
  EncViews v;
  v.wav = EncBuf{const_cast<float*>(wav_dev), 1, 0, T};
  int t = T, c = g.num_filters;
  for (int i = 0; i < g.n_ratios; ++i) {
    v.x[i] = EncBuf{X, c, 0, t};
    v.y[i] = EncBuf{Y, c / g.compress, 0, t};
    v.z[i] = EncBuf{Z, c, 0, t};
    t = (t + g.ratios[i] - 1) / g.ratios[i];
    c *= 2;
  }
  v.x[g.n_ratios] = EncBuf{X, c, 0, t};
  const int C = g.hidden_size;
  v.h = EncBuf{Y, C, 0, t};
  v.a = EncBuf{X, C, 0, t};
  v.q = EncBuf{Z, 3 * C, 0, t};
  v.kv.assign(g.num_layers, EncBuf{Z + (size_t)C * t, 3 * C, 0, t});  // the k and v thirds of qkv
  return encode_segment(e, v, B, T, nullptr, codes_dev, st);
}

// =================================================================================================
// Stateful streaming encoder (q3_codec_enc_stream_*): packets of whole 1920-sample frames through the same walker as
// the one-shot, with each tensor that a layer reads back in time kept in a history-prefixed buffer per row:
//   waveform (conv0's k - 1), x[i] and z[i] (max(residual k - 1, ratio) each: the k3 conv and the downsample read them,
//   and the residual add reads x[i] in z[i]'s layout), conv_last's input (k - 1), the transformer's residual stream h
//   (the final downsample's stride), and each layer's rotated K and V (window - 1).
// Zero history after a reset is the causal zero padding (ELU(0) = 0); the final downsample's replicate padding is
// seeded from the row's first 25 Hz column.  A row's final partial frame (finish) runs the walker once more on that row
// alone with the one-shot's right padding, so the codes of a whole clip equal the one-shot encode of the clip alone.
// =================================================================================================
struct q3_codec_enc_stream {
  q3_codec_enc* e = nullptr;
  int B = 0, nmax = 0;
  std::vector<int> pos;       // 12.5 Hz frames since each row's reset
  std::vector<int32_t> rp_h;  // host image of rp
  int32_t* rp = nullptr;      // device int32: [0, B) 25 Hz positions, [B, 2B) 25 Hz frames of the next segment (or a
                              // reset mask), then {position, frames} of every finishing row
  DevStore store{"codec encoder stream"};
  EncViews hv;                // the history buffers (scratch views are filled per segment)
};

static int enc_hist_alloc(q3_codec_enc_stream* s, EncBuf* h, int C, int hist, int cap) {
  *h = EncBuf{nullptr, C, hist, hist + cap};
  // zero history == the causal left padding of a fresh stream
  return s->store.alloc(&h->p, (size_t)s->B * h->bs(), true);
}

// every history buffer with its columns per 25 Hz frame, for the roll after a packet and for reset
static EncRollTable enc_hist_table(const q3_codec_enc_stream* s) {
  const q3_codec_enc_cfg& g = s->e->cfg;
  EncRollTable tb{};
  auto add = [&](const EncBuf& h, int factor) { if (h.hist > 0) tb.e[tb.n++] = EncRollEntry{h.p, h.hist, factor, h.C, h.ld}; };
  int f = s->e->hop / g.downsample_stride;
  add(s->hv.wav, f);
  for (int i = 0; i < g.n_ratios; ++i) { add(s->hv.x[i], f); add(s->hv.z[i], f); f /= g.ratios[i]; }
  add(s->hv.x[g.n_ratios], 1);
  add(s->hv.h, 1);
  for (const EncBuf& k : s->hv.kv) add(k, 1);
  return tb;
}

// scratch views of the walker over a segment of T samples of B rows (the encoder's three ping-pong buffers)
static EncViews enc_stream_views(const q3_codec_enc_stream* s, int T) {
  const q3_codec_enc* e = s->e;
  const q3_codec_enc_cfg& g = e->cfg;
  EncViews v = s->hv;
  int t = T, c = g.num_filters;
  for (int i = 0; i < g.n_ratios; ++i) {
    v.y[i] = EncBuf{e->buf[1], c / g.compress, 0, t};
    t = (t + g.ratios[i] - 1) / g.ratios[i];
    c *= 2;
  }
  v.a = EncBuf{e->buf[0], g.hidden_size, 0, t};
  v.q = EncBuf{e->buf[2], 3 * g.hidden_size, 0, t};
  return v;
}

extern "C" int q3_codec_enc_stream_open(q3_codec_enc* e, int32_t B, int32_t max_packet_frames, q3_codec_enc_stream** out) {
  Q3_REQUIRE(e && e->finalized && out, "codec encoder not finalized");
  const q3_codec_enc_cfg& g = e->cfg;
  Q3_REQUIRE(B >= 1 && B <= Q3_MAX_BATCH, "batch %d outside [1, %d]", B, Q3_MAX_BATCH);
  Q3_REQUIRE(max_packet_frames >= 1 && (int64_t)max_packet_frames * g.downsample_stride <= g.max_frames,
             "max_packet_frames %d outside [1, max_frames / %d]", max_packet_frames, g.downsample_stride);
  Q3_REQUIRE(g.sliding_window >= 1, "sliding_window must be positive");
  const int nhist = 2 * g.n_ratios + 3 + g.num_layers;
  Q3_REQUIRE(nhist <= kEncRollMax, "streaming encoder needs %d history buffers, at most %d supported", nhist, kEncRollMax);
  Q3_CUDA(cudaSetDevice(g.device));
  q3_codec_enc_stream* s = new q3_codec_enc_stream();
  s->e = e; s->B = B; s->nmax = max_packet_frames;
  const int n = max_packet_frames;
  int cap = n * e->hop, c = g.num_filters;
  int rc = enc_hist_alloc(s, &s->hv.wav, 1, g.kernel_size - 1, cap);
  for (int i = 0; i < g.n_ratios && !rc; ++i) {
    const int hist = std::max(g.residual_kernel_size - 1, g.ratios[i]);
    rc = enc_hist_alloc(s, &s->hv.x[i], c, hist, cap);
    if (!rc) rc = enc_hist_alloc(s, &s->hv.z[i], c, hist, cap);
    cap /= g.ratios[i];
    c *= 2;
  }
  if (!rc) rc = enc_hist_alloc(s, &s->hv.x[g.n_ratios], c, g.last_kernel_size - 1, cap);
  if (!rc) rc = enc_hist_alloc(s, &s->hv.h, g.hidden_size, g.downsample_stride, cap);
  s->hv.kv.resize(g.num_layers);
  for (int l = 0; l < g.num_layers && !rc; ++l) rc = enc_hist_alloc(s, &s->hv.kv[l], 2 * g.hidden_size, g.sliding_window - 1, cap);
  void* rp = nullptr;
  if (!rc) rc = s->store.alloc(&rp, (size_t)4 * B * sizeof(int32_t), true);
  s->rp = reinterpret_cast<int32_t*>(rp);
  // packet scratch: the encoder's ping-pong buffers, grown (never shrunk) to a full packet of B rows
  if (!rc) {
    const cudaError_t ce = cudaDeviceSynchronize();
    rc = ce != cudaSuccess ? q3_set_err("codec encoder stream: %s", cudaGetErrorString(ce))
                           : grow_scratch(e, scratch_per_row(g, n * e->hop) * (size_t)B, nullptr);
  }
  s->pos.assign(B, 0);
  s->rp_h.assign(4 * B, 0);
  if (rc) { delete s; return 1; }
  *out = s;
  return 0;
}

extern "C" void q3_codec_enc_stream_close(q3_codec_enc_stream* s) { delete s; }

// 12.5 Hz frames encoded for `row` since its last reset; -1 for a bad row
extern "C" int q3_codec_enc_stream_row_position(q3_codec_enc_stream* s, int32_t row) {
  if (!s || row < 0 || row >= s->B) { q3_set_err("row %d out of range [0, %d)", row, s ? s->B : 0); return -1; }
  return s->pos[row];
}

// the next n frames of every row: wav_dev fp32 [B][n * hop]; row b takes the first counts_host[b] -> codes_dev int32
// [B][nq][n], -1 past each row's count.  Every argument is checked before any device work.
extern "C" int q3_codec_enc_stream_step_rows(q3_codec_enc_stream* s, const float* wav_dev, int32_t n, const int32_t* counts_host,
                                             int32_t* codes_dev, void* stream_) {
  Q3_REQUIRE(s && wav_dev && counts_host && codes_dev, "null argument");
  q3_codec_enc* e = s->e;
  const q3_codec_enc_cfg& g = e->cfg;
  Q3_REQUIRE(n >= 1 && n <= s->nmax, "packet of %d frames (max %d)", n, s->nmax);
  for (int b = 0; b < s->B; ++b) {
    Q3_REQUIRE(counts_host[b] >= 0 && counts_host[b] <= n, "row %d: count %d outside [0, %d]", b, counts_host[b], n);
    Q3_REQUIRE((int64_t)(s->pos[b] + counts_host[b]) * g.downsample_stride <= g.max_frames,
               "row %d: 25 Hz position %d + %d frames exceeds the RoPE table (max_frames %d)", b, s->pos[b] * g.downsample_stride,
               counts_host[b] * g.downsample_stride, g.max_frames);
  }
  Q3_CUDA(cudaSetDevice(g.device));
  cudaStream_t st = (cudaStream_t)stream_;
  const int B = s->B, T = n * e->hop;
  if (grow_scratch(e, scratch_per_row(g, T) * (size_t)B, st)) return 1;
  for (int b = 0; b < B; ++b) { s->rp_h[b] = s->pos[b] * g.downsample_stride; s->rp_h[B + b] = counts_host[b] * g.downsample_stride; }
  Q3_CUDA(cudaMemcpyAsync(s->rp, s->rp_h.data(), (size_t)2 * B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  const EncViews v = enc_stream_views(s, T);
  e->launches = 0;
  const int per25 = e->hop / g.downsample_stride;
  load_wav_kernel<<<dim3((T + 1023) / 1024, B), 256, 0, st>>>(wav_dev, T, v.wav.cur(), v.wav.ld, T, s->rp, B, per25);
  ++e->launches;
  if (encode_segment(e, v, B, T, s->rp, codes_dev, st)) return 1;
  const EncRollTable tb = enc_hist_table(s);
  enc_roll_kernel<<<dim3(tb.n * B, 16), 256, 0, st>>>(tb, s->rp, B);
  ++e->launches;
  Q3_CUDA(cudaGetLastError());
  for (int b = 0; b < B; ++b) s->pos[b] += counts_host[b];
  return 0;
}

static int enc_reset(q3_codec_enc_stream* s, int n, const int32_t* rows, cudaStream_t st) {
  const int B = s->B;
  for (int b = 0; b < B; ++b) s->rp_h[B + b] = 0;
  for (int i = 0; i < n; ++i) s->rp_h[B + rows[i]] = 1;
  Q3_CUDA(cudaMemcpyAsync(s->rp + B, s->rp_h.data() + B, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  const EncRollTable tb = enc_hist_table(s);
  enc_reset_kernel<<<dim3(tb.n * B, 16), 256, 0, st>>>(tb, s->rp, B);
  Q3_CUDA(cudaGetLastError());
  for (int i = 0; i < n; ++i) s->pos[rows[i]] = 0;
  return 0;
}

// forget the listed rows: their next packet starts a new clip at position 0; the other rows are untouched
extern "C" int q3_codec_enc_stream_reset_rows(q3_codec_enc_stream* s, int32_t n, const int32_t* rows_host, void* stream_) {
  Q3_REQUIRE(s, "null stream");
  if (check_row_list(s->B, n, rows_host, "reset", "stream")) return 1;
  if (n == 0) return 0;
  Q3_CUDA(cudaSetDevice(s->e->cfg.device));
  return enc_reset(s, n, rows_host, (cudaStream_t)stream_);
}

// end the clips of the listed rows with their final partial frames: row rows_host[i] takes tail_host[i] samples of
// wav_dev [n][hop] row i and gets its last frame's codes at codes_dev [n][nq] row i (-1 when the tail is empty).  Each
// row runs the walker alone over its tail, every layer padded on the right exactly as the one-shot pads the clip's end.
extern "C" int q3_codec_enc_stream_finish_rows(q3_codec_enc_stream* s, int32_t n, const int32_t* rows_host, const int32_t* tail_host,
                                               const float* wav_dev, int32_t* codes_dev, void* stream_) {
  Q3_REQUIRE(s, "null stream");
  if (check_row_list(s->B, n, rows_host, "finish", "stream")) return 1;
  if (n == 0) return 0;
  Q3_REQUIRE(tail_host && wav_dev && codes_dev, "null argument");
  q3_codec_enc* e = s->e;
  const q3_codec_enc_cfg& g = e->cfg;
  for (int i = 0; i < n; ++i) {
    const int r = rows_host[i], tail = tail_host[i];
    Q3_REQUIRE(tail >= 0 && tail < e->hop, "row %d: tail of %d samples outside [0, %d)", r, tail, e->hop);
    const int t25 = tail ? frames25(g, tail) : 0;
    Q3_REQUIRE((int64_t)s->pos[r] * g.downsample_stride + t25 <= g.max_frames,
               "row %d: 25 Hz position %d + %d frames exceeds the RoPE table (max_frames %d)", r, s->pos[r] * g.downsample_stride,
               t25, g.max_frames);
  }
  Q3_CUDA(cudaSetDevice(g.device));
  cudaStream_t st = (cudaStream_t)stream_;
  const int B = s->B, nq = g.num_quantizers;
  for (int i = 0; i < n; ++i) {
    s->rp_h[2 * B + 2 * i] = s->pos[rows_host[i]] * g.downsample_stride;
    s->rp_h[2 * B + 2 * i + 1] = tail_host[i] ? frames25(g, tail_host[i]) : 0;
  }
  Q3_CUDA(cudaMemcpyAsync(s->rp + 2 * B, s->rp_h.data() + 2 * B, (size_t)2 * n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  e->launches = 0;
  for (int i = 0; i < n; ++i) {
    const int r = rows_host[i], tail = tail_host[i];
    int32_t* codes = codes_dev + (size_t)i * nq;
    if (tail == 0) { Q3_CUDA(cudaMemsetAsync(codes, 0xff, (size_t)nq * sizeof(int32_t), st)); continue; }
    EncViews v = enc_stream_views(s, tail).row(r);
    Q3_CUDA(cudaMemcpyAsync(v.wav.cur(), wav_dev + (size_t)i * e->hop, (size_t)tail * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (encode_segment(e, v, 1, tail, s->rp + 2 * B + 2 * i, codes, st)) return 1;
  }
  return enc_reset(s, n, rows_host, st);
}
