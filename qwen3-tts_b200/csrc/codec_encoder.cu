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
#include "common.cuh"
#include "conv_f32.cuh"
#include "dev_store.h"
#include "../../include/qwen3tts_b200.h"

#include <algorithm>
#include <string>
#include <vector>

namespace {

// LayerNorm over channels of x [B][C][T] (nn.LayerNorm(hidden), modeling_mimi.py:933-934).  Block = 32 time steps x 8
// channel groups: loads stay coalesced along t, each thread reduces C/8 channels, groups combine through shared memory.
__global__ void __launch_bounds__(256) layernorm_ct_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                           const float* __restrict__ bb, float* __restrict__ y, int C, int T,
                                                           float eps) {
  __shared__ float red[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int t = blockIdx.x * 32 + tx, b = blockIdx.y;
  const bool ok = t < T;
  const float* xp = x + (size_t)b * C * T + (ok ? t : 0);
  float s = 0.f;
  if (ok) {
#pragma unroll 8
    for (int c = ty; c < C; c += 8) s += xp[(size_t)c * T];
  }
  red[ty][tx] = s;
  __syncthreads();
  float mean = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) mean += red[i][tx];
  mean /= (float)C;
  __syncthreads();
  float v = 0.f;
  if (ok) {
#pragma unroll 8
    for (int c = ty; c < C; c += 8) { const float d = xp[(size_t)c * T] - mean; v = fmaf(d, d, v); }
  }
  red[ty][tx] = v;
  __syncthreads();
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) var += red[i][tx];
  const float rstd = rsqrtf(var / (float)C + eps);
  if (!ok) return;
  float* yp = y + (size_t)b * C * T + t;
#pragma unroll 8
  for (int c = ty; c < C; c += 8) yp[(size_t)c * T] = (xp[(size_t)c * T] - mean) * rstd * w[c] + bb[c];
}

// RoPE on the q and k thirds of qkv [B][3C][T] (apply_rotary_pos_emb, modeling_mimi.py:589-611; rotate_half pairs
// (i, i + hd/2)); cos/sin: [Tmax][hd/2] fp32 tables computed by the host exactly as MimiRotaryEmbedding does
__global__ void rope_ct_kernel(float* __restrict__ qkv, const float* __restrict__ cosT, const float* __restrict__ sinT, int C,
                               int T, int nh, int hd) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int half = hd >> 1;
  const int pr = blockIdx.y;          // (which in {q,k}) x head x i
  const int i = pr % half, h = (pr / half) % nh, which = pr / (half * nh);
  const int b = blockIdx.z;
  float* base = qkv + ((size_t)b * 3 * C + (size_t)which * C + h * hd) * T;
  const float c = cosT[(size_t)t * half + i], s = sinT[(size_t)t * half + i];
  const float x1 = base[(size_t)i * T + t], x2 = base[(size_t)(i + half) * T + t];
  base[(size_t)i * T + t] = x1 * c - x2 * s;
  base[(size_t)(i + half) * T + t] = x2 * c + x1 * s;
}

// causal sliding-window attention (eager path, modeling_mimi.py:683-738; mask = create_sliding_window_causal_mask:
// key j visible to query t iff j <= t and t - j < window).  One thread per (b, head, t); fp32 online softmax.
template <int HD>
__global__ void __launch_bounds__(128) swa_ct_kernel(const float* __restrict__ qkv, float* __restrict__ out, int C, int T, int hd,
                                                     int window, float scale) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, h = blockIdx.y, b = blockIdx.z;
  if (t >= T) return;
  const float* q = qkv + ((size_t)b * 3 * C + h * hd) * T;
  const float* k = q + (size_t)C * T;
  const float* v = k + (size_t)C * T;
  float qr[HD], acc[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) { qr[d] = d < hd ? q[(size_t)d * T + t] : 0.f; acc[d] = 0.f; }
  float m = -INFINITY, l = 0.f;
  const int j0 = max(0, t - window + 1);
  for (int j = j0; j <= t; ++j) {
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < HD; ++d) if (d < hd) s = fmaf(qr[d], k[(size_t)d * T + j], s);
    s *= scale;
    const float mn = fmaxf(m, s);
    const float corr = __expf(m - mn), p = __expf(s - mn);
    l = l * corr + p;
#pragma unroll
    for (int d = 0; d < HD; ++d) if (d < hd) acc[d] = acc[d] * corr + p * v[(size_t)d * T + j];
    m = mn;
  }
  float* o = out + ((size_t)b * C + h * hd) * T;
  const float inv = 1.f / l;
#pragma unroll
  for (int d = 0; d < HD; ++d) if (d < hd) o[(size_t)d * T + t] = acc[d] * inv;
}

// split residual VQ encode (modeling_mimi.py:1311-1338, :1262-1280, :1197-1203): one block per (frame, batch row).
// level 0..nsem-1 quantise the semantic projection, the rest the acoustic one; per level: nearest centroid
// (argmin_c |r - e_c|^2 = argmin_c |e_c|^2 - 2 r.e_c, ties -> lowest index), then r -= e_c.
struct RvqArgs {
  const float* r_sem;   // [B][D][T]
  const float* r_ac;    // [B][D][T]
  const float* const* E;   // [nq] -> [K][D]
  const float* const* ET;  // [nq] -> [D][K]
  const float* const* E2;  // [nq] -> [K]
  int* codes;           // [B][nq][T]
  int D, K, T, nq, nsem;
};

__global__ void __launch_bounds__(256) rvq_encode_kernel(const RvqArgs a) {
  extern __shared__ float sm[];
  float* r = sm;                                   // [D]
  float* bestv = sm + a.D;                         // [8]
  int* besti = reinterpret_cast<int*>(bestv + 8);  // [8]
  __shared__ int s_code;
  const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  for (int q = 0; q < a.nq; ++q) {
    if (q == 0 || q == a.nsem) {
      const float* src = (q < a.nsem ? a.r_sem : a.r_ac) + (size_t)b * a.D * a.T + t;
      __syncthreads();
      for (int d = tid; d < a.D; d += 256) r[d] = src[(size_t)d * a.T];
    }
    __syncthreads();
    const float* ET = a.ET[q];
    const float* E2 = a.E2[q];
    float bv = INFINITY;
    int bi = 0x7fffffff;
    // 4 codes per thread and pass, d unrolled by 4: 16 independent coalesced loads in flight per thread (the loop is
    // otherwise one exposed L2 round trip per FMA)
    for (int c0 = tid; c0 < a.K; c0 += 4 * 256) {
      float dot[4] = {0.f, 0.f, 0.f, 0.f};
      const bool ok1 = c0 + 256 < a.K, ok2 = c0 + 512 < a.K, ok3 = c0 + 768 < a.K;
#pragma unroll 4
      for (int d = 0; d < a.D; ++d) {
        const float rd = r[d];
        const float* row = ET + (size_t)d * a.K + c0;
        dot[0] = fmaf(rd, row[0], dot[0]);
        if (ok1) dot[1] = fmaf(rd, row[256], dot[1]);
        if (ok2) dot[2] = fmaf(rd, row[512], dot[2]);
        if (ok3) dot[3] = fmaf(rd, row[768], dot[3]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = c0 + 256 * i;
        if (c < a.K) {
          const float dist = E2[c] - 2.f * dot[i];
          if (dist < bv) { bv = dist; bi = c; }   // ascending c: the first minimum wins
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov < bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if ((tid & 31) == 0) { bestv[tid >> 5] = bv; besti[tid >> 5] = bi; }
    __syncthreads();
    if (tid == 0) {
      float v = bestv[0];
      int i = besti[0];
      for (int w = 1; w < 8; ++w)
        if (bestv[w] < v || (bestv[w] == v && besti[w] < i)) { v = bestv[w]; i = besti[w]; }
      s_code = i;
      a.codes[((size_t)b * a.nq + q) * a.T + t] = i;
    }
    __syncthreads();
    const float* e = a.E[q] + (size_t)s_code * a.D;
    for (int d = tid; d < a.D; d += 256) r[d] -= e[d];
  }
}

}  // namespace

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

struct EncRunner {
  q3_codec_enc* e;
  cudaStream_t st;
  int B;
  int stage = 0;
  int rc = 0;

  int conv(const std::string& wname, const float* x, float* y, int Cin, int Cout, int Tin, int k, int stride, int replicate,
           bool elu_in, bool gelu_out, const float* res, const std::string& scale_name, bool has_bias, int* Tout_) {
    const DevStore& S = e->store;
    ConvF32Args a{};
    if (!(a.w = S.need<float>(wname + ".w", (int64_t)Cout * Cin * k))) return 1;
    if (has_bias && !(a.bias = S.need<float>(wname + ".b", Cout))) return 1;
    if (!scale_name.empty() && !(a.scale = S.need<float>(scale_name, Cout))) return 1;
    a.x = x; a.res = res; a.y = y;
    a.xC = Cin; a.yC = Cout;
    a.Cin = Cin; a.Cout = Cout; a.Tin = Tin; a.k = k; a.stride = stride; a.dil = 1;
    a.pad_left = k - stride;                       // causal: padding_total on the left (modeling_mimi.py:343-345)
    a.Tout = (Tin + stride - 1) / stride;          // right "extra padding" up to a stride multiple (:273-285)
    a.pad = replicate ? PAD_REPLICATE : PAD_ZERO;
    a.act_in = elu_in ? IN_ELU : IN_NONE;
    a.act_out = gelu_out ? OUT_GELU : OUT_NONE;
    if (conv_f32_launch(a, B, st)) return 1;
    ++e->launches;
    if (Tout_) *Tout_ = a.Tout;
    return 0;
  }
  void capture(const float* x, int C, int T) {
    for (auto& c : e->captures)
      if (c.first == stage) {
        const int64_t n = std::min<int64_t>((int64_t)B * C * T, c.second.second);
        cudaMemcpyAsync(c.second.first, x, (size_t)n * 4, cudaMemcpyDeviceToDevice, st);
      }
    ++stage;
  }
};

}  // namespace

extern "C" int q3_codec_enc_frames(q3_codec_enc* e, int32_t T) {
  if (!e || T <= 0) return 0;
  int t = T;
  for (int i = 0; i < e->cfg.n_ratios; ++i) t = (t + e->cfg.ratios[i] - 1) / e->cfg.ratios[i];
  return (t + e->cfg.downsample_stride - 1) / e->cfg.downsample_stride;
}

extern "C" int q3_codec_enc_encode(q3_codec_enc* e, const float* wav_dev, int32_t B, int32_t T, int32_t* codes_dev, void* stream_) {
  Q3_REQUIRE(e && e->finalized, "codec encoder not finalized");
  Q3_REQUIRE(wav_dev && codes_dev && B >= 1 && T >= 1, "bad arguments");
  const q3_codec_enc_cfg& g = e->cfg;
  Q3_CUDA(cudaSetDevice(g.device));
  cudaStream_t st = (cudaStream_t)stream_;
  e->launches = 0;
  // ---- workspace: three ping-pong buffers sized for the largest [C][T] activation of this request
  size_t need = 0;
  {
    int t = T, c = g.num_filters;
    need = (size_t)c * t;
    for (int i = 0; i < g.n_ratios; ++i) { t = (t + g.ratios[i] - 1) / g.ratios[i]; c *= 2; need = std::max(need, (size_t)c * t); }
    need = std::max(need, (size_t)std::max(3 * g.hidden_size, g.intermediate_size) * t);
    Q3_REQUIRE(t <= g.max_frames, "%d transformer frames exceed max_frames %d", t, g.max_frames);
    need *= (size_t)B;
  }
  if (need > e->buf_elems) {
    e->buf_elems = 0;
    for (float*& b : e->buf)
      if (e->store.grow(&b, need * 4, st)) return 1;
    e->buf_elems = need;
  }
  float *X = e->buf[0], *Y = e->buf[1], *Z = e->buf[2];
  EncRunner r{e, st, B};
  // ---- SEANet encoder (modeling_mimi.py:454-496)
  int t = T, c = g.num_filters, to = 0;
  if (r.conv("enc.conv0", wav_dev, X, 1, c, t, g.kernel_size, 1, 0, false, false, nullptr, "", true, &to)) return 1;
  r.capture(X, c, t);
  for (int i = 0; i < g.n_ratios; ++i) {
    const std::string p = "enc.res" + std::to_string(i);
    // x + conv_k1(ELU(conv_k3(ELU(x))))  (:437-451)
    if (r.conv(p + ".a", X, Y, c, c / g.compress, t, g.residual_kernel_size, 1, 0, true, false, nullptr, "", true, &to)) return 1;
    if (r.conv(p + ".b", Y, Z, c / g.compress, c, t, 1, 1, 0, true, false, X, "", true, &to)) return 1;
    r.capture(Z, c, t);
    if (r.conv("enc.down" + std::to_string(i), Z, X, c, 2 * c, t, 2 * g.ratios[i], g.ratios[i], 0, true, false, nullptr, "", true, &to))
      return 1;
    t = to; c *= 2;
    r.capture(X, c, t);
  }
  if (r.conv("enc.conv_last", X, Y, c, g.hidden_size, t, g.last_kernel_size, 1, 0, true, false, nullptr, "", true, &to)) return 1;
  r.capture(Y, g.hidden_size, t);
  // ---- transformer (:926-993): h lives in Y; X = normed / attention output, Z = qkv / mlp hidden
  const int C = g.hidden_size, nh = g.num_heads, hd = g.head_dim, I = g.intermediate_size;
  const float* cosT = e->store.need<float>("rope.cos", (int64_t)g.max_frames * (hd / 2));
  const float* sinT = e->store.need<float>("rope.sin", (int64_t)g.max_frames * (hd / 2));
  if (!cosT || !sinT) return 1;
  float* H = Y;
  float* A = X;
  for (int l = 0; l < g.num_layers; ++l) {
    const std::string p = "tr." + std::to_string(l);
    const DevStore& S = e->store;
    const float *l1w = S.need<float>(p + ".ln1.w", C), *l1b = S.need<float>(p + ".ln1.b", C), *l2w = S.need<float>(p + ".ln2.w", C),
                *l2b = S.need<float>(p + ".ln2.b", C);
    if (!l1w || !l1b || !l2w || !l2b) return 1;
    dim3 lg((t + 31) / 32, B);
    layernorm_ct_kernel<<<lg, 256, 0, st>>>(H, l1w, l1b, A, C, t, g.norm_eps);
    if (r.conv(p + ".qkv", A, Z, C, 3 * C, t, 1, 1, 0, false, false, nullptr, "", false, &to)) return 1;
    rope_ct_kernel<<<dim3((t + 127) / 128, 2 * nh * (hd / 2), B), 128, 0, st>>>(Z, cosT, sinT, C, t, nh, hd);
    swa_ct_kernel<64><<<dim3((t + 127) / 128, nh, B), 128, 0, st>>>(Z, A, C, t, hd, g.sliding_window, 1.0f / sqrtf((float)hd));
    if (r.conv(p + ".o", A, H, C, C, t, 1, 1, 0, false, false, H, p + ".ls1", false, &to)) return 1;  // h += ls1 * o_proj(attn)
    layernorm_ct_kernel<<<lg, 256, 0, st>>>(H, l2w, l2b, A, C, t, g.norm_eps);
    if (r.conv(p + ".fc1", A, Z, C, I, t, 1, 1, 0, false, true, nullptr, "", false, &to)) return 1;
    if (r.conv(p + ".fc2", Z, H, I, C, t, 1, 1, 0, false, false, H, p + ".ls2", false, &to)) return 1;  // h += ls2 * fc2(gelu(fc1))
    e->launches += 4;
    r.capture(H, C, t);
  }
  // ---- 25 Hz -> 12.5 Hz (:1420-1430: k = 2*stride, no bias, replicate padding)
  if (r.conv("down", H, A, C, C, t, 2 * g.downsample_stride, g.downsample_stride, 1, false, false, nullptr, "", false, &to)) return 1;
  const int t3 = to;
  r.capture(A, C, t3);
  // ---- split RVQ (:1311-1338)
  const int D = g.codebook_dim, nq = g.num_quantizers;
  float* Rs = Z;
  float* Ra = Z + (size_t)B * D * t3;
  Q3_REQUIRE((size_t)2 * B * D * t3 <= e->buf_elems, "workspace too small for the RVQ projections");
  if (r.conv("rvq.sem.proj", A, Rs, C, D, t3, 1, 1, 0, false, false, nullptr, "", false, &to)) return 1;
  if (r.conv("rvq.ac.proj", A, Ra, C, D, t3, 1, 1, 0, false, false, nullptr, "", false, &to)) return 1;
  RvqArgs ra{};
  ra.r_sem = Rs; ra.r_ac = Ra; ra.E = e->d_ptrs; ra.ET = e->d_ptrs + nq; ra.E2 = e->d_ptrs + 2 * nq;
  ra.codes = codes_dev; ra.D = D; ra.K = g.codebook_size; ra.T = t3; ra.nq = nq; ra.nsem = g.num_semantic_quantizers;
  rvq_encode_kernel<<<dim3(t3, B), 256, (size_t)(D + 16) * sizeof(float), st>>>(ra);
  ++e->launches;
  Q3_CUDA(cudaGetLastError());
  return 0;
}
