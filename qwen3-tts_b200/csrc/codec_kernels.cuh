// Small row-wise kernels of the codec decoder (RVQ gather, RMSNorm, RoPE + K/V append, sliding-window attention,
// depthwise conv + LayerNorm, history roll / reset / copy, final conv).  Part of the codec_engine.cu translation unit;
// tests/csrc/attention_shim.cu includes it too, to run the RoPE and attention kernels on inputs a test chooses.
#pragma once

namespace {

// ---------------------------------------------------------------------------------------------- small kernels
// Per-row frame window of a decode of n frames per row: rp[b] is row b's position (of its frame 0) and rp[B + b] its
// count, the frames [0, count) that are its own; frames past the count are computed but are not part of the row's
// stream.  rp == nullptr: every row at position 0 with all n frames (the one-shot forward).
__device__ __forceinline__ int row_pos(const int* rp, int b) { return rp ? rp[b] : 0; }
__device__ __forceinline__ int row_count(const int* rp, int B, int b, int n) { return rp ? rp[B + b] : n; }

// RVQ decode (…v2.py:815-821, :721-727, :676-679): e[b][t][0:D] = table[0][c0]; e[b][t][D:2D] = sum_{k>=1} table[k][c_k].
// A frame past its row's count reads no code and gets a zero embedding.
__global__ void rvq_gather_kernel(const int* __restrict__ codes, const bf16* __restrict__ table, bf16* __restrict__ e,
                                  int B, int K, int T, int D, int bins, const int* __restrict__ rp) {
  const int bt = blockIdx.x;  // b*T + t
  const int b = bt / T, t = bt % T;
  if (t >= row_count(rp, B, b, T)) {
    for (int d = threadIdx.x; d < 2 * D; d += blockDim.x) e[(size_t)bt * 2 * D + d] = f2bf(0.f);
    return;
  }
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const int c0 = codes[((size_t)b * K + 0) * T + t];
    e[(size_t)bt * 2 * D + d] = table[((size_t)0 * bins + c0) * D + d];
    float acc = 0.f;
    for (int k = 1; k < K; ++k) {
      const int c = codes[((size_t)b * K + k) * T + t];
      const float v = bf2f(table[((size_t)k * bins + c) * D + d]);
      acc = (k == 1) ? v : rbf(acc + v);  // the reference accumulates in the model dtype
    }
    e[(size_t)bt * 2 * D + D + d] = f2bf(acc);
  }
}

// RMSNorm over the last dim (…v2.py:383-388): one warp per row
__global__ void rmsnorm_rows_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y, int rows,
                                    int C, float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const bf16* xr = x + (size_t)row * C;
  float ss = 0.f;
  for (int i = lane; i < C; i += 32) { const float v = bf2f(xr[i]); ss += v * v; }
  ss = warp_sum(ss);
  const float inv = rsqrtf(ss / (float)C + eps);
  for (int i = lane; i < C; i += 32) y[(size_t)row * C + i] = f2bf(rbf(bf2f(xr[i]) * inv) * bf2f(w[i]));
}

// ConvNeXt front: depthwise causal conv k=7 + LayerNorm(eps 1e-6) (…v2.py:230-232); one block per (b,t)
// (x_bs_rows / hist: the streaming decoder keeps 6 rows of history in front of every row's T new rows)
__global__ void dwconv_ln_kernel(const bf16* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                 const float* __restrict__ lnw, const float* __restrict__ lnb, bf16* __restrict__ y, int B, int T,
                                 int C, int x_bs_rows, int hist) {
  extern __shared__ float sh[];  // [C] conv outputs + 64 scratch
  const int bt = blockIdx.x;
  const int t = bt % T;
  const size_t xrow = (size_t)(bt / T) * x_bs_rows + hist + t;  // row of x that holds time step t of this batch row
  float s1 = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = bias[c];
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      const int tt = t - 6 + j;
      if (tt >= -hist) acc += w[c * 7 + j] * bf2f(x[(xrow - 6 + j) * C + c]);
    }
    acc = rbf(acc);
    sh[c] = acc;
    s1 += acc;
  }
  // two-pass variance, as F.layer_norm: a one-pass q / C - mean^2 loses about log2((mean / std)^2) bits of it
  float* red = sh + C;
  const int nw = blockDim.x >> 5;
  s1 = warp_sum(s1);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s1;
  __syncthreads();
  float a = 0.f;
  for (int i = 0; i < nw; ++i) a += red[i];
  const float mean = a / C;
  float s2 = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { const float d = sh[c] - mean; s2 += d * d; }
  s2 = warp_sum(s2);
  if ((threadIdx.x & 31) == 0) red[32 + (threadIdx.x >> 5)] = s2;
  __syncthreads();
  float q = 0.f;
  for (int i = 0; i < nw; ++i) q += red[32 + i];
  const float var = q / C;
  const float inv = rsqrtf(var + 1e-6f);
  for (int c = threadIdx.x; c < C; c += blockDim.x) y[(size_t)bt * C + c] = f2bf((sh[c] - mean) * inv * lnw[c] + lnb[c]);
}

// RoPE in place on q,k of qkv [B][n][3*nh*hd] at positions rp[b] + t (…v2.py:329, apply_rotary_pos_emb).  With a K/V
// window buffer kv [B][hist + n_cap][2*nh*hd] (the streaming decoder's) the rotated k and the v heads are also appended
// at rows [hist, hist+n); kv == nullptr rotates only and does not visit the v heads.  Frames past the row's count are
// skipped, so a row parked at the end of the RoPE table never indexes past it.
__global__ void rope_append_kernel(bf16* __restrict__ qkv, const bf16* __restrict__ cosT, const bf16* __restrict__ sinT,
                                   bf16* __restrict__ kv, int B, int n, int nh, int hd, const int* __restrict__ rp, int hist,
                                   int kv_bs_rows) {
  const int half = hd / 2;
  const int heads = kv ? 3 * nh : 2 * nh;  // q heads, k heads[, v heads]
  const size_t total = (size_t)B * n * heads * half;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int f = (int)(i % half);
    const int h = (int)((i / half) % heads);
    const size_t bt = i / ((size_t)half * heads);
    const int t = (int)(bt % n), b = (int)(bt / n);
    if (t >= row_count(rp, B, b, n)) continue;
    const int pos = row_pos(rp, b) + t;
    bf16* v = qkv + bt * (size_t)(3 * nh * hd) + (size_t)h * hd;
    float y1 = bf2f(v[f]), y2 = bf2f(v[f + half]);
    if (h < 2 * nh) {
      const float c = bf2f(cosT[(size_t)pos * half + f]), sn = bf2f(sinT[(size_t)pos * half + f]);
      const float x1 = y1, x2 = y2;
      y1 = rbf(x1 * c) + rbf(-x2 * sn);
      y2 = rbf(x2 * c) + rbf(x1 * sn);
      v[f] = f2bf(y1);
      v[f + half] = f2bf(y2);
      y1 = bf2f(v[f]); y2 = bf2f(v[f + half]);
    }
    if (kv && h >= nh) {  // k (rotated) and v rows go to the window buffer: [K heads | V heads]
      bf16* d = kv + ((size_t)b * kv_bs_rows + hist + t) * (size_t)(2 * nh * hd) + (size_t)(h - nh) * hd;
      d[f] = f2bf(y1);
      d[f + half] = f2bf(y2);
    }
  }
}

// causal sliding-window attention of the n queries of qkv [B][n][3*nh*hd], one warp per (b, head, t) (…v2.py:321-354;
// key k visible iff 0 <= t-k < window).  Keys and values come from a K/V view: row r of batch row b starts at
// kv + (b*kv_bs_rows + r)*ld with the K heads, then (nh*hd further) the V heads, of absolute position rp[b] - hist + r
// (rows of negative position are not valid yet); query t is row hist + t.  The one-shot forward passes qkv itself
// (kv = qkv + nh*hd, ld = 3*nh*hd, kv_bs_rows = n, hist = 0, rp = nullptr), the stream its layer's window buffer.
// Queries past the row's count are skipped (their output rows are left as they are).
__global__ void swa_stream_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ kv, int ld, int kv_bs_rows, int hist,
                                  bf16* __restrict__ out, int B, int n, int nh, int hd, int window, const int* __restrict__ rp) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= B * n * nh) return;
  const int lane = threadIdx.x & 31;
  const int h = wid % nh, t = (wid / nh) % n, b = wid / (nh * n);
  if (t >= row_count(rp, B, b, n)) return;
  const int pos0 = row_pos(rp, b);
  const bf16* q = qkv + ((size_t)b * n + t) * (size_t)(3 * nh * hd) + (size_t)h * hd;
  const int r1 = hist + t;                              // the query's own row
  const int r0 = max(max(r1 - window + 1, hist - pos0), 0);  // oldest visible row
  const int nk = r1 - r0 + 1;
  const bf16* base = kv + (size_t)b * kv_bs_rows * ld;
  const float scale = rsqrtf((float)hd);
  // scores: lane handles keys lane, lane+32, lane+64 (window <= 96)
  float sc[3];
  float mx = -INFINITY;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int kk = lane + 32 * r;
    sc[r] = -INFINITY;
    if (kk < nk) {
      const bf16* kp = base + (size_t)(r0 + kk) * ld + (size_t)h * hd;
      float d = 0.f;
      for (int i = 0; i < hd; i += 2) {
        const uint32_t qa = *reinterpret_cast<const uint32_t*>(q + i), ka = *reinterpret_cast<const uint32_t*>(kp + i);
        d += bf16lo(qa) * bf16lo(ka) + bf16hi(qa) * bf16hi(ka);
      }
      sc[r] = rbf(rbf(d) * scale);  // bf16 matmul output, then * scaling in bf16 (eager path)
      mx = fmaxf(mx, sc[r]);
    }
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int r = 0; r < 3; ++r) { sc[r] = (sc[r] == -INFINITY) ? 0.f : __expf(sc[r] - mx); sum += sc[r]; }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
  // output: lanes over dims (hd <= 64 -> 2 per lane), loop over keys with shuffles
  float o0 = 0.f, o1 = 0.f;
  for (int kk = 0; kk < nk; ++kk) {
    const float p = rbf(__shfl_sync(0xffffffffu, sc[kk >> 5], kk & 31) * inv);  // softmax cast to bf16
    const bf16* vp = base + (size_t)(r0 + kk) * ld + (size_t)(nh + h) * hd;
    if (lane * 2 < hd) {
      const uint32_t va = *reinterpret_cast<const uint32_t*>(vp + lane * 2);
      o0 += p * bf16lo(va);
      o1 += p * bf16hi(va);
    }
  }
  if (lane * 2 < hd)
    *reinterpret_cast<uint32_t*>(out + ((size_t)b * n + t) * (size_t)(nh * hd) + (size_t)h * hd + lane * 2) = pack_bf16(o0, o1);
}

// after a packet: every history buffer keeps, per batch row b, its last `hist` rows ([hist + T] rows were valid, T =
// factor * rp[B + b]: the row's count times the buffer's rows per frame) at the front.  One launch for all buffers;
// block = (entry, batch row); rows ascend so an overlapping move (T < hist) is safe.  A row with count 0 stays.
struct RollEntry { bf16* p; int hist, factor, C, bs_rows; };
constexpr int kRollMax = 48;
struct RollTable { int n; RollEntry e[kRollMax]; };
__global__ void roll_history_kernel(RollTable tb, const int* __restrict__ rp, int B) {
  const RollEntry E = tb.e[blockIdx.x / B];
  const int b = blockIdx.x % B;
  const int T = E.factor * rp[B + b];
  if (T == 0) return;
  bf16* base = E.p + (size_t)b * E.bs_rows * E.C;
  const int cv = E.C / 8;  // C % 16 == 0
  for (int r = 0; r < E.hist; ++r) {
    const uint4* src = reinterpret_cast<const uint4*>(base + (size_t)(T + r) * E.C);
    uint4* dst = reinterpret_cast<uint4*>(base + (size_t)r * E.C);
    for (int c = threadIdx.x; c < cv; c += blockDim.x) dst[c] = src[c];
    __syncthreads();  // row r complete before row r+1 may overwrite what a later source row aliases
  }
}

// zero the history rows of every buffer of the table for the batch rows b with rp[B + b] != 0 (a fresh utterance:
// zero history is the causal left padding); block = (entry, batch row)
__global__ void reset_history_kernel(RollTable tb, const int* __restrict__ rp, int B) {
  const RollEntry E = tb.e[blockIdx.x / B];
  const int b = blockIdx.x % B;
  if (rp[B + b] == 0) return;
  uint4* base = reinterpret_cast<uint4*>(E.p + (size_t)b * E.bs_rows * E.C);
  const int nv = E.hist * E.C / 8;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) base[i] = make_uint4(0u, 0u, 0u, 0u);
}

// copy the history rows of listed batch rows from one stream's buffers to another's (same codec, so the entries of
// both tables correspond one to one; B and the capacity, hence bs_rows, may differ).  rows[i] is the source row and
// rows[ld + i] the destination row of pair i; block = (entry, pair).  Destination rows are distinct, so no two blocks
// write the same bytes.
struct CopyEntry { bf16* dst; const bf16* src; int hist, C, dst_bs_rows, src_bs_rows; };
struct CopyTable { int n; CopyEntry e[kRollMax]; };
static_assert(sizeof(CopyTable) + 2 * sizeof(void*) + 2 * sizeof(int) <= 4096, "copy_rows_kernel parameters exceed 4 KB");
__global__ void copy_rows_kernel(CopyTable tb, const int* __restrict__ rows, int ld, int n) {
  const CopyEntry E = tb.e[blockIdx.x / n];
  const int i = blockIdx.x % n;
  const uint4* src = reinterpret_cast<const uint4*>(E.src + (size_t)rows[i] * E.src_bs_rows * E.C);
  uint4* dst = reinterpret_cast<uint4*>(E.dst + (size_t)rows[ld + i] * E.dst_bs_rows * E.C);
  const int nv = E.hist * E.C / 8;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) dst[v] = src[v];
}

// final causal conv k=7, C -> 1, + clamp(-1,1) (…v2.py:863,884); one thread per output sample.  The T samples of a row
// are `up` per frame; the samples of frames past the row's count are written as zeros.
__global__ void final_conv_kernel(const bf16* __restrict__ x, const float* __restrict__ w /*[7][C]*/, const float* __restrict__ bias_p,
                                  float* __restrict__ wav, int B, int T, int C, int x_bs_rows, int hist, const int* __restrict__ rp,
                                  int up) {
  const size_t total = (size_t)B * T;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T);
    const int b = (int)(i / T);
    if (rp && t >= rp[B + b] * up) { wav[i] = 0.f; continue; }
    const size_t xrow = (size_t)b * x_bs_rows + hist + t;
    float acc = __ldg(bias_p);
    for (int j = 0; j < 7; ++j) {
      const int tt = t - 6 + j;
      if (tt < -hist) continue;
      const bf16* xr = x + (xrow - 6 + j) * (size_t)C;
      for (int c = 0; c < C; c += 8) {
        const uint4 v = *reinterpret_cast<const uint4*>(xr + c);
        const float* wr = w + j * C + c;
        acc += bf16lo(v.x) * wr[0] + bf16hi(v.x) * wr[1] + bf16lo(v.y) * wr[2] + bf16hi(v.y) * wr[3] +
               bf16lo(v.z) * wr[4] + bf16hi(v.z) * wr[5] + bf16lo(v.w) * wr[6] + bf16hi(v.w) * wr[7];
      }
    }
    acc = rbf(acc);
    wav[i] = fminf(1.f, fmaxf(-1.f, acc));
  }
}

}  // namespace
