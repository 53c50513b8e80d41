// Row-wise kernels around the wgmma prefill GEMMs, and the weight re-packing kernels.
// Part of the ar_engine.cu translation unit (include order: ar_program, ar_gemv, ar_attention, ar_sampler,
// the persistent kernel in ar_step, ar_prefill).
#pragma once

namespace {

// ------------------------------------------------------------------------------------------------
// PREFILL on tensor cores: talker linears are wgmma tap-GEMMs (gemm_sm90.cu) over all prompt tokens at once
// (M = sum of prompt lengths); the row-wise pieces around them are the small kernels below.
// ------------------------------------------------------------------------------------------------
__global__ void pf_rmsnorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y, int rows, int C,
                                  float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * C);
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  float ss = 0.f;
  for (int i = lane; i < C / 8; i += 32) {
    const uint4 v = xr[i];
    float f;
    f = bf16lo(v.x); ss += f * f; f = bf16hi(v.x); ss += f * f;
    f = bf16lo(v.y); ss += f * f; f = bf16hi(v.y); ss += f * f;
    f = bf16lo(v.z); ss += f * f; f = bf16hi(v.z); ss += f * f;
    f = bf16lo(v.w); ss += f * f; f = bf16hi(v.w); ss += f * f;
  }
  ss = warp_sum(ss);
  const float inv = rsqrtf(ss / (float)C + eps);
  uint4* yr = reinterpret_cast<uint4*>(y + (size_t)row * C);
  for (int i = lane; i < C / 8; i += 32) {
    const uint4 v = xr[i], wv = wr[i];
    uint4 o;
    o.x = pack_bf16(rbf(bf16lo(v.x) * inv) * bf16lo(wv.x), rbf(bf16hi(v.x) * inv) * bf16hi(wv.x));
    o.y = pack_bf16(rbf(bf16lo(v.y) * inv) * bf16lo(wv.y), rbf(bf16hi(v.y) * inv) * bf16hi(wv.y));
    o.z = pack_bf16(rbf(bf16lo(v.z) * inv) * bf16lo(wv.z), rbf(bf16hi(v.z) * inv) * bf16hi(wv.z));
    o.w = pack_bf16(rbf(bf16lo(v.w) * inv) * bf16lo(wv.w), rbf(bf16hi(v.w) * inv) * bf16hi(wv.w));
    yr[i] = o;
  }
}

// packed-token index (row, position) of all prompt tokens, built on the device from the prompt lengths (passed by
// value: no host staging buffer, no synchronisation), and the gather of every row's last hidden state
// row r of the packed prompt batch lives in engine slot slot[r]; its packed rows are the suffix of a prompt whose first
// p0[r] positions (a prefix, 0: none) are already in the slot's K/V cache
struct PfLens { int B; int start[MAXB + 1]; int slot[MAXB]; int p0[MAXB]; };
// the admitted rows' trailing lengths and text [r][stride][H], gathered into the engine's copy [slot][cap][H]
struct PfRows {
  int trailing_len[MAXB];
  const bf16* src; bf16* dst; int stride, cap, H;
};
// the prefix K/V of the admitted rows (null: none), each [lh = layers * nkv][p0[r]][HD] for K and then for V, copied
// into the slots' caches [slot][lh][cap][HD] at positions [0, p0[r])
struct PfPrefix {
  const uint4* kv[MAXB];
  uint4 *kc, *vc;
  int lh, cap;
};
// Talker K/V of sequence b at positions [0, len) between the caches kc / vc ([seq][lh][cap][HD]) and a block in the
// registered-prefix layout ([2 (K, V)][lh][len][HD]), in 16-byte chunks: thread i of `stride` threads copies chunks i,
// i + stride, ... of K and of V, into the caches (kToCache) or out of them into the block
template <bool kToCache>
__device__ __forceinline__ void kv_block_copy(uint4* blk, uint4* kc, uint4* vc, int lh, int cap, int b, int len, size_t i,
                                              size_t stride) {
  const int row = len * (HD / 8);
  const size_t n = (size_t)lh * row;
  for (size_t j = i; j < n; j += stride) {
    const size_t l = j / row, c = j - l * row, d = ((size_t)b * lh + l) * cap * (HD / 8) + c;
    if (kToCache) {
      kc[d] = blk[j];
      vc[d] = blk[n + j];
    } else {
      blk[j] = kc[d];
      blk[n + j] = vc[d];
    }
  }
}

// grid (x, row r): slice r resets row r's device state and seen bytes, gathers its trailing text (element-wise: the
// source may be any bf16 pointer) and copies its prefix K/V; slice 0 also writes the token index
__global__ void pf_index_kernel(PfLens L, PfRows R, PfPrefix X, DevState* st, unsigned char* seen, int V, int* tok_seq, int* tok_pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y, b = L.slot[r];
  if (r == 0 && i < L.start[L.B]) {
    int s = 0;
    while (i >= L.start[s + 1]) ++s;
    tok_seq[i] = L.slot[s];
    tok_pos[i] = L.p0[s] + i - L.start[s];
  }
  if (i == 0) {
    st->finished[b] = 0; st->n_valid[b] = 0; st->n_gen[b] = 0; st->c0[b] = 0;
    st->len0[b] = L.p0[r] + L.start[r + 1] - L.start[r]; st->trailing_len[b] = R.trailing_len[r];
  }
  if (i < V) seen[(size_t)b * V + i] = 0;
  if (i < R.trailing_len[r] * R.H) R.dst[(size_t)b * R.cap * R.H + i] = R.src[(size_t)r * R.stride * R.H + i];
  if (X.kv[r])  // one 16-byte chunk of K and one of V per thread and step; a position is HD / 8 chunks
    kv_block_copy<true>(const_cast<uint4*>(X.kv[r]), X.kc, X.vc, X.lh, X.cap, b, L.p0[r], i, (size_t)gridDim.x * blockDim.x);
}

// A parked row (q3_row_park / q3_row_resume): its talker K/V at positions [0, pos) go to or come from the record's block
// kv (kv_block_copy, the layout of a registered prefix); every other piece of its state that a frame-step reads before
// it writes it is a span of 16-byte chunks on the slot's side and in the record, and its DevState fields are ints
constexpr int kRowSpans = 6;                        // x_cp rows of blocks 0 and 1, past_hidden, past_keep, trailing text, seen
constexpr int kRowInts = 6 + Q3_NUM_GROUPS_MAX;     // len0, finished, n_valid, n_gen, c0, trailing_len, cur[0..]
struct RowSpan { uint4* slot; uint4* rec; int n; };
struct RowMove {
  RowSpan span[kRowSpans];
  uint4 *kc, *vc, *kv;
  int lh, cap, pos, slot;
  int* ints;
};
// kResume = false (park): gather the slot into the record, then mark the slot's row finished as release_state_kernel
// does; kResume = true: scatter the record into the slot.  Any grid: every thread strides over every piece.
template <bool kResume>
__global__ void row_move_kernel(RowMove M, DevState* st) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  kv_block_copy<kResume>(M.kv, M.kc, M.vc, M.lh, M.cap, M.slot, M.pos, i, stride);
#pragma unroll 1
  for (int s = 0; s < kRowSpans; ++s) {
    const RowSpan& S = M.span[s];
    for (size_t j = i; j < (size_t)S.n; j += stride) {
      if (kResume) S.slot[j] = S.rec[j];
      else S.rec[j] = S.slot[j];
    }
  }
  if (i == 0) {
    const int b = M.slot;
    int* f[kRowInts];
    f[0] = &st->len0[b]; f[1] = &st->finished[b]; f[2] = &st->n_valid[b]; f[3] = &st->n_gen[b]; f[4] = &st->c0[b];
    f[5] = &st->trailing_len[b];
    for (int g = 0; g < Q3_NUM_GROUPS_MAX; ++g) f[6 + g] = &st->cur[b][g];
    for (int k = 0; k < kRowInts; ++k) {
      if (kResume) *f[k] = M.ints[k];
      else M.ints[k] = *f[k];
    }
    if (!kResume && !st->finished[b]) {
      st->finished[b] = 1;
      st->n_valid[b] = 0x3fffffff;
    }
  }
}
// token index of a prefix computed alone: its n rows are positions 0..n-1 of sequence 0 of the prefix's K/V block
__global__ void pf_prefix_index_kernel(int n, int* tok_seq, int* tok_pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { tok_seq[i] = 0; tok_pos[i] = i; }
}
__global__ void pf_gather_last_kernel(PfLens L, const bf16* __restrict__ x, bf16* __restrict__ h_last, int H) {
  const int b = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)(L.start[b + 1] - 1) * H);
  uint4* dst = reinterpret_cast<uint4*>(h_last + (size_t)L.slot[b] * H);
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) dst[i] = src[i];
}

// a row that is abandoned at its frame horizon: mark it finished (it keeps stepping like any finished row)
struct SlotList { int n; int slot[MAXB]; };
__global__ void release_state_kernel(DevState* st, SlotList A) {
  if ((int)threadIdx.x < A.n && !st->finished[A.slot[threadIdx.x]]) {
    st->finished[A.slot[threadIdx.x]] = 1;
    st->n_valid[A.slot[threadIdx.x]] = 0x3fffffff;  // "never sampled EOS": the host caps it at the frames it asked for
  }
}

// per (token, head-vector): q heads RMSNorm+RoPE in place; k head -> K cache (normed, roped); v head -> V cache
__global__ void pf_qkv_post_kernel(bf16* __restrict__ qkv, int ntok, const int* __restrict__ tok_seq, const int* __restrict__ tok_pos,
                                   int nh, int nkv, const bf16* __restrict__ qn, const bf16* __restrict__ kn, float eps,
                                   const bf16* __restrict__ cosT, const bf16* __restrict__ sinT, bf16* __restrict__ kc,
                                   bf16* __restrict__ vc, int layer, int layers, int cap) {
  const int nvec = nh + 2 * nkv;
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= ntok * nvec) return;
  const int lane = threadIdx.x & 31;
  const int tok = wid / nvec, v = wid - tok * nvec;
  const int seq = tok_seq[tok], pos = tok_pos[tok];
  bf16* src = qkv + (size_t)tok * (size_t)(nvec * HD) + (size_t)v * HD;
  const bf16* cosr = cosT + (size_t)pos * 64;
  const bf16* sinr = sinT + (size_t)pos * 64;
  if (v < nh) {
    norm_rope_vec(src, qn, eps, cosr, sinr, nullptr, src);
  } else if (v < nh + nkv) {
    const int kvh = v - nh;
    norm_rope_vec(src, kn, eps, cosr, sinr, nullptr, kc + ((((size_t)seq * layers + layer) * nkv + kvh) * cap + pos) * HD);
  } else {
    const int kvh = v - nh - nkv;
    bf16* d = vc + ((((size_t)seq * layers + layer) * nkv + kvh) * cap + pos) * HD;
#pragma unroll
    for (int i = 0; i < 4; ++i) d[lane + 32 * i] = src[lane + 32 * i];
  }
}

// causal attention over the KV cache, one warp per (token, q head); keys in blocks of 32 with an online softmax
__global__ void pf_attention_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ attn, int ntok, const int* __restrict__ tok_seq,
                                    const int* __restrict__ tok_pos, int nh, int nkv, const bf16* __restrict__ kc,
                                    const bf16* __restrict__ vc, int layer, int layers, int cap) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= ntok * nh) return;
  const int lane = threadIdx.x & 31;
  const int tok = wid / nh, h = wid - tok * nh;
  const int seq = tok_seq[tok], pos = tok_pos[tok];
  const int kvh = h / (nh / nkv);
  const bf16* q = qkv + (size_t)tok * (size_t)((nh + 2 * nkv) * HD) + (size_t)h * HD;
  const bf16* K = kc + (((size_t)seq * layers + layer) * nkv + kvh) * (size_t)cap * HD;
  const bf16* V = vc + (((size_t)seq * layers + layer) * nkv + kvh) * (size_t)cap * HD;
  const float scale = rsqrtf((float)HD);
  float m = -INFINITY, l = 0.f, o[4] = {0.f, 0.f, 0.f, 0.f};
  for (int kb = 0; kb <= pos; kb += 32) {
    const int key = kb + lane;
    float sc = -INFINITY;
    if (key <= pos) {
      const uint4* kr = reinterpret_cast<const uint4*>(K + (size_t)key * HD);
      const uint4* qr = reinterpret_cast<const uint4*>(q);
      float d = 0.f;
#pragma unroll 4
      for (int i = 0; i < HD / 8; ++i) {
        const uint4 a = qr[i], b = kr[i];
        d += bf16lo(a.x) * bf16lo(b.x) + bf16hi(a.x) * bf16hi(b.x) + bf16lo(a.y) * bf16lo(b.y) + bf16hi(a.y) * bf16hi(b.y) +
             bf16lo(a.z) * bf16lo(b.z) + bf16hi(a.z) * bf16hi(b.z) + bf16lo(a.w) * bf16lo(b.w) + bf16hi(a.w) * bf16hi(b.w);
      }
      sc = d * scale;
    }
    const float mn = fmaxf(m, warp_max(sc));
    const float corr = __expf(m - mn);
    const float p = (key <= pos) ? __expf(sc - mn) : 0.f;
    l = l * corr + warp_sum(p);
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] *= corr;
    const int nk = min(32, pos - kb + 1);
    for (int j = 0; j < nk; ++j) {
      const float pj = __shfl_sync(0xffffffffu, p, j);
      const uint2 vv = *reinterpret_cast<const uint2*>(V + (size_t)(kb + j) * HD + lane * 4);
      o[0] += pj * bf16lo(vv.x); o[1] += pj * bf16hi(vv.x); o[2] += pj * bf16lo(vv.y); o[3] += pj * bf16hi(vv.y);
    }
    m = mn;
  }
  const float inv = 1.f / l;
  uint2 r;
  r.x = pack_bf16(o[0] * inv, o[1] * inv);
  r.y = pack_bf16(o[2] * inv, o[3] * inv);
  *reinterpret_cast<uint2*>(attn + (size_t)tok * (size_t)(nh * HD) + (size_t)h * HD + lane * 4) = r;
}

// ------------------------------------------------------------------------------------------------
// weight packing: row-major [N][K] bf16 -> stream of (16 rows x 32 k) 1 KB blocks, each two 8x32 halves
// ------------------------------------------------------------------------------------------------
__global__ void bf16_to_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = bf2f(src[i]);
}

__global__ void pack_weight_kernel(const bf16* __restrict__ src, uint4* __restrict__ dst, int N, int K) {
  // one thread per 16-byte chunk of the destination.  Block (tile, kb) = 16 rows x 32 k = 1 KB = two 512-byte halves;
  // chunk `lane` (g = lane/4, t = lane%4) of half h holds the four A registers of MMA h of that lane:
  //   { W[g][k0..k0+1], W[g+8][k0..k0+1], W[g][k0+2..k0+3], W[g+8][k0+2..k0+3] },  k0 = kb*32 + t*8 + h*4
  // (the K permutation "lane t owns k t*8..t*8+7" is shared with the B fragments, which read 16 contiguous bytes of x)
  const size_t total = (size_t)N * K / 8;
  const int KB = K / 32;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t blk = i / 64;         // (tile, kb)
    const int within = (int)(i % 64);
    const int h = within / 32, g = (within % 32) / 4, t = within % 4;
    const size_t tile = blk / KB;
    const int kb = (int)(blk % KB);
    const int k0 = kb * 32 + t * 8 + h * 4;
    const bf16* r0 = src + (tile * 16 + g) * K + k0;
    const bf16* r1 = src + (tile * 16 + g + 8) * K + k0;
    uint4 o;
    o.x = *reinterpret_cast<const uint32_t*>(r0);
    o.y = *reinterpret_cast<const uint32_t*>(r1);
    o.z = *reinterpret_cast<const uint32_t*>(r0 + 2);
    o.w = *reinterpret_cast<const uint32_t*>(r1 + 2);
    dst[i] = o;
  }
}

}  // namespace
