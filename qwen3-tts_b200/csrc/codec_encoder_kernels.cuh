// Per-column kernels of the codec encoder (LayerNorm, RoPE, sliding-window attention, split RVQ encode) and its
// streaming helpers (waveform load, replicate seed, code mask, history roll / reset).  Part of the codec_encoder.cu
// translation unit; tests/csrc/encoder_shim.cu includes it too, to run these kernels on inputs a test chooses.
#pragma once
#include "common.cuh"

namespace {

// LayerNorm over channels of x [B][C][ldx] -> y [B][C][ldy], T columns (nn.LayerNorm(hidden), modeling_mimi.py:933-934).
// Block = 32 time steps x 8 channel groups: loads stay coalesced along t, each thread reduces C/8 channels, groups
// combine through shared memory.
__global__ void __launch_bounds__(256) layernorm_ct_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ w,
                                                           const float* __restrict__ bb, float* __restrict__ y, int ldy, int C,
                                                           int T, float eps) {
  __shared__ float red[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int t = blockIdx.x * 32 + tx, b = blockIdx.y;
  const bool ok = t < T;
  const float* xp = x + (size_t)b * C * ldx + (ok ? t : 0);
  float s = 0.f;
  if (ok) {
#pragma unroll 8
    for (int c = ty; c < C; c += 8) s += xp[(size_t)c * ldx];
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
    for (int c = ty; c < C; c += 8) { const float d = xp[(size_t)c * ldx] - mean; v = fmaf(d, d, v); }
  }
  red[ty][tx] = v;
  __syncthreads();
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) var += red[i][tx];
  const float rstd = rsqrtf(var / (float)C + eps);
  if (!ok) return;
  float* yp = y + (size_t)b * C * ldy + t;
#pragma unroll 8
  for (int c = ty; c < C; c += 8) yp[(size_t)c * ldy] = (xp[(size_t)c * ldx] - mean) * rstd * w[c] + bb[c];
}

// Row b's 25 Hz frames of a segment: the first is at position rp[b], the first rp[B + b] are the row's own (the rest are
// padding of a ragged packet and never reach the state or the codes).  rp == nullptr: position 0, all T.
__device__ __forceinline__ int seg_pos(const int* rp, int b) { return rp ? rp[b] : 0; }
__device__ __forceinline__ int seg_valid(const int* rp, int B, int b, int T) { return rp ? rp[B + b] : T; }

// RoPE on the q and k thirds of qkv [B][3C][T] (apply_rotary_pos_emb, modeling_mimi.py:589-611; rotate_half pairs
// (i, i + hd/2)) at positions seg_pos + t; cos/sin: [Tmax][hd/2] fp32 tables computed by the host exactly as
// MimiRotaryEmbedding does.  kv == nullptr (one-shot): in place.  Otherwise the rotated keys and the values go to the
// layer's window buffer kv (k channels [0, C), v channels [C, 2C); batch stride kv_bs, column step kv_ld, kv pointing at
// the segment's first column) and grid.y covers the v third too.
__global__ void rope_ct_kernel(float* __restrict__ qkv, const float* __restrict__ cosT, const float* __restrict__ sinT, int C,
                               int T, int nh, int hd, const int* __restrict__ rp, int B, float* __restrict__ kv, long long kv_bs,
                               int kv_ld) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.z;
  if (t >= seg_valid(rp, B, b, T)) return;
  const int half = hd >> 1;
  const int pr = blockIdx.y;          // (which in {q,k,v}) x head x i
  const int i = pr % half, h = (pr / half) % nh, which = pr / (half * nh);
  float* base = qkv + ((size_t)b * 3 * C + (size_t)which * C + h * hd) * T;
  const float x1 = base[(size_t)i * T + t], x2 = base[(size_t)(i + half) * T + t];
  float* dst = base;
  size_t ld = T;
  if (kv && which > 0) { dst = kv + (size_t)b * kv_bs + ((size_t)(which - 1) * C + h * hd) * kv_ld; ld = kv_ld; }
  if (which == 2) { dst[(size_t)i * ld + t] = x1; dst[(size_t)(i + half) * ld + t] = x2; return; }
  const int p = seg_pos(rp, b) + t;
  const float c = cosT[(size_t)p * half + i], s = sinT[(size_t)p * half + i];
  dst[(size_t)i * ld + t] = x1 * c - x2 * s;
  dst[(size_t)(i + half) * ld + t] = x2 * c + x1 * s;
}

// causal sliding-window attention (eager path, modeling_mimi.py:683-738; mask = create_sliding_window_causal_mask:
// key j visible to query t iff j <= t and t - j < window).  One thread per (b, head, t); fp32 online softmax.  Queries
// come from qkv [B][3C][T]; keys and values from kv (k channels [0, C), v [C, 2C), batch stride kv_bs, column step kv_ld),
// whose column kv_hist is the segment's first: a stream's window buffer holds kv_hist = window - 1 earlier columns, the
// one-shot's view of qkv none.  Keys are walked in ascending absolute position from max(P - window + 1, 0) to P,
// P = seg_pos + t, so a streamed query sees exactly the keys, in the order, of the one-shot.  Query columns past the
// row's own frames attend over stale window columns: finite values that never reach the row's state or codes.
template <int HD>
__global__ void __launch_bounds__(128) swa_ct_kernel(const float* __restrict__ qkv, const float* __restrict__ kv, long long kv_bs,
                                                     int kv_ld, int kv_hist, float* __restrict__ out, int C, int T, int hd,
                                                     int window, float scale, const int* __restrict__ rp) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, h = blockIdx.y, b = blockIdx.z;
  if (t >= T) return;
  const float* q = qkv + ((size_t)b * 3 * C + h * hd) * T;
  const float* k = kv + (size_t)b * kv_bs + (size_t)h * hd * kv_ld;
  const float* v = k + (size_t)C * kv_ld;
  float qr[HD], acc[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) { qr[d] = d < hd ? q[(size_t)d * T + t] : 0.f; acc[d] = 0.f; }
  int off[HD];  // column-0 offsets of the key / value rows: 32-bit and hoisted, as the loop needs them every key
#pragma unroll
  for (int d = 0; d < HD; ++d) off[d] = d * kv_ld;
  float m = -INFINITY, l = 0.f;
  const int tc = t + kv_hist;   // the query's column in kv
  const int j0 = tc - min(seg_pos(rp, b) + t, window - 1);  // no key before the row's reset, none out of the window
  for (int j = j0; j <= tc; ++j) {
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < HD; ++d) if (d < hd) s = fmaf(qr[d], k[off[d] + j], s);
    s *= scale;
    const float mn = fmaxf(m, s);
    const float corr = __expf(m - mn), p = __expf(s - mn);
    l = l * corr + p;
#pragma unroll
    for (int d = 0; d < HD; ++d) if (d < hd) acc[d] = acc[d] * corr + p * v[off[d] + j];
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

// ---- streaming state (q3_codec_enc_stream_*).  A tensor that a layer reads back in time lives in a history-prefixed
// buffer [B][C][hist + cap]: time contiguous, `hist` columns of history before the segment's new columns.

// the segment's waveform into the history-prefixed input buffer: row b's first valid = factor * rp[B + b] samples of
// src [B][src_ld], zeros after them up to n (samples past a row's count are never read)
__global__ void load_wav_kernel(const float* __restrict__ src, int src_ld, float* __restrict__ dst, int dst_ld, int n,
                                const int* __restrict__ rp, int B, int factor) {
  const int b = blockIdx.y;
  const int valid = factor * rp[B + b];
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x)
    dst[(size_t)b * dst_ld + t] = t < valid ? src[(size_t)b * src_ld + t] : 0.f;
}

// the downsample's replicate padding: a row at position 0 with frames in this segment gets `hist` copies of its first
// 25 Hz column as history (the one-shot clamps negative indices to column 0, modeling_mimi.py:1420-1430)
__global__ void seed_replicate_kernel(float* __restrict__ h, int C, int hist, int ld, const int* __restrict__ rp, int B) {
  const int b = blockIdx.y;
  if (rp[b] != 0 || rp[B + b] == 0) return;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    float* row = h + ((size_t)b * C + c) * ld;
    const float v = row[hist];
    for (int r = 0; r < hist; ++r) row[r] = v;
  }
}

// codes [B][nq][T]: -1 past each row's frames (ceil(rp[B + b] / 2): the segment's 12.5 Hz frames of the row)
__global__ void mask_codes_kernel(int* __restrict__ codes, int nq, int T, const int* __restrict__ rp, int B, int ds) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * nq * T) return;
  const int t = i % T, b = i / (nq * T);
  if (t >= (rp[B + b] + ds - 1) / ds) codes[i] = -1;
}

// After a packet every history buffer keeps, per batch row b, its last `hist` columns: [hist + T) columns were valid,
// T = factor * rp[B + b] (the row's 25 Hz frames times the buffer's columns per 25 Hz frame).  Block = (entry, batch
// row) x channel slice; a warp moves one channel 32 columns at a time, reading each chunk before writing it, so an
// overlapping move (T < hist) reads every column before it is overwritten.  A row without frames stays.
struct EncRollEntry { float* p; int hist, factor, C, ld; };
constexpr int kEncRollMax = 48;
struct EncRollTable { int n; EncRollEntry e[kEncRollMax]; };
__global__ void __launch_bounds__(256) enc_roll_kernel(EncRollTable tb, const int* __restrict__ rp, int B) {
  const EncRollEntry E = tb.e[blockIdx.x / B];
  const int b = blockIdx.x % B;
  const int T = E.factor * rp[B + b];
  if (T == 0) return;
  const int lane = threadIdx.x & 31;
  for (int c = blockIdx.y * 8 + (threadIdx.x >> 5); c < E.C; c += gridDim.y * 8) {
    float* row = E.p + ((size_t)b * E.C + c) * E.ld;
    for (int r0 = 0; r0 < E.hist; r0 += 32) {
      const int r = r0 + lane;
      const float v = r < E.hist ? row[T + r] : 0.f;
      __syncwarp();
      if (r < E.hist) row[r] = v;
      __syncwarp();
    }
  }
}

// zero the history of the rows b with rp[B + b] != 0 (a new clip: zero history is the causal left padding)
__global__ void __launch_bounds__(256) enc_reset_kernel(EncRollTable tb, const int* __restrict__ rp, int B) {
  const EncRollEntry E = tb.e[blockIdx.x / B];
  const int b = blockIdx.x % B;
  if (rp[B + b] == 0) return;
  for (int c = blockIdx.y * 8 + (threadIdx.x >> 5); c < E.C; c += gridDim.y * 8) {
    float* row = E.p + ((size_t)b * E.C + c) * E.ld;
    for (int r = threadIdx.x & 31; r < E.hist; r += 32) row[r] = 0.f;
  }
}

}  // namespace
