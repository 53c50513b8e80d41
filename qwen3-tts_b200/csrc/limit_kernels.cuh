// Kernels of the streaming look-ahead limiter (csrc/limit.cu; tests/csrc/limit_shim.cu launches them directly).
#pragma once
#include "common.cuh"
#include "../../include/qwen3tts_b200.h"

constexpr int kLimL = 120;                         // look-ahead (5 ms at 24 kHz)
constexpr int kLimW = 1200;                        // release (50 ms)
constexpr int kLimHist = Q3_LIMIT_HIST;            // inputs a row keeps
constexpr int kLimReach = kLimW + 2 * kLimL - 2;   // inputs the first pending output reads back: 1438
constexpr int kLimTile = 256;                      // outputs per CTA, one per thread
constexpr int kLimThreads = kLimTile;
constexpr int kLimHistTiles = kLimHist / kLimThreads;
static_assert(kLimReach <= kLimHist && kLimHist % kLimThreads == 0, "limiter history");
// fp32(10^(-1/20)), fp32(1/1200), fp32(1/120): the ceiling, the release slope and the look-ahead mean's scale
constexpr float kLimCeil = 0x1.c8520ap-1f;
constexpr float kLimDelta = 0x1.b4e81cp-11f;
constexpr float kLimInv = 0x1.111112p-7f;

// staged per output tile: u and a over [n0 - 1319, n0 + 256 + 119), b over its first 256 + 1319, s over n0 - 1200 ..
constexpr int kLimA = kLimTile + kLimReach;        // 1694
constexpr int kLimB = kLimTile + kLimW + kLimL - 1;  // 1575
constexpr int kLimS = kLimTile + kLimW;            // 1456

// one row of one launch (or of a save / load)
struct LimitJob {
  long long n_in;   // inputs before this launch
  long long out0;   // outputs emitted before this launch
  int count;        // new inputs (this launch)
  int nout;         // outputs this launch
  int end;          // the clip ends with this launch
  int cur;          // current history half
  float gain;
  int unused;
};

// the saved image of one row (Q3_LIMIT_ROW_BYTES)
struct LimitRecord {
  float gain;
  int32_t unused;
  long long n_in;
  float hist[kLimHist];
};
static_assert(sizeof(LimitRecord) == Q3_LIMIT_ROW_BYTES, "limiter row record size");

// x[p] of a row in this launch: zero before the clip and past its inputs, else its history or its new inputs
__device__ __forceinline__ float lim_x(const LimitJob& jb, const float* h_old, const float* xr, long long p) {
  if (p < 0 || p >= jb.n_in + jb.count) return 0.f;
  return p >= jb.n_in ? xr[p - jb.n_in] : h_old[kLimHist - (jb.n_in - p)];
}

// grid (blocks, rows), kLimThreads threads.  Block x < ceil(nout/256) of row r computes outputs [out0 + 256x, +256):
//   u = g*x, a = 1 if |u| <= c else c/|u|, b[m] = min a[m .. m+119], s[m] = min(a[m], (b[m] + b[m-1] + ... +
//   b[m-119]) * inv) summed from b[m] down, G[n] = min over m in [max(0, n-1200), n] of s[m] + (n-m)*delta,
//   y = u*G, every operation fp32 round-to-nearest in that order (no contraction).
// The next kLimHistTiles blocks of a row that took inputs and did not end write its next history half.
__global__ void __launch_bounds__(kLimThreads) limit_kernel(const LimitJob* __restrict__ jobs, const float* __restrict__ x,
                                                            long long ld, float* __restrict__ hist, int rows,
                                                            float* __restrict__ out, long long cap) {
  __shared__ float su[kLimA], sa[kLimA], sb[kLimB], ss[kLimS], ramp[kLimW + 1];
  const int r = blockIdx.y, t = threadIdx.x;
  const LimitJob jb = jobs[r];
  const float* xr = x + (size_t)r * ld;
  const float* h_old = hist + ((size_t)jb.cur * rows + r) * kLimHist;
  const int tiles = (jb.nout + kLimTile - 1) / kLimTile;
  if ((int)blockIdx.x >= tiles) {
    const int k = ((int)blockIdx.x - tiles) * kLimThreads + t;
    if (k < kLimHist && jb.count > 0 && !jb.end)
      hist[((size_t)(jb.cur ^ 1) * rows + r) * kLimHist + k] = lim_x(jb, h_old, xr, jb.n_in + jb.count - kLimHist + k);
    return;
  }
  const long long n0 = jb.out0 + (long long)blockIdx.x * kLimTile;
  const long long a0 = n0 - (kLimW + kLimL - 1);   // position of su[0], sa[0], sb[0]
  for (int i = t; i < kLimA; i += kLimThreads) {
    const float u = __fmul_rn(jb.gain, lim_x(jb, h_old, xr, a0 + i));
    const float m = fabsf(u);
    su[i] = u;
    sa[i] = m <= kLimCeil ? 1.f : __fdiv_rn(kLimCeil, m);
  }
  for (int d = t; d <= kLimW; d += kLimThreads) ramp[d] = __fmul_rn((float)d, kLimDelta);
  __syncthreads();
  for (int j = t; j < kLimB; j += kLimThreads) {
    float v = sa[j];
    for (int q = 1; q < kLimL; ++q) v = fminf(v, sa[j + q]);
    sb[j] = v;
  }
  __syncthreads();
  for (int k = t; k < kLimS; k += kLimThreads) {   // s of position n0 - 1200 + k, b index k + 119
    float acc = sb[k + kLimL - 1];
    for (int q = kLimL - 2; q >= 0; --q) acc = __fadd_rn(acc, sb[k + q]);
    const float v = fminf(sa[k + kLimL - 1], __fmul_rn(acc, kLimInv));
    ss[k] = n0 - kLimW + k < 0 ? __int_as_float(0x7f800000) : v;   // m < 0 is outside the window
  }
  __syncthreads();
  if (n0 + t < jb.out0 + jb.nout) {
    float g = ss[t + kLimW];
#pragma unroll 8
    for (int d = 1; d <= kLimW; ++d) g = fminf(g, __fadd_rn(ss[t + kLimW - d], ramp[d]));
    out[(size_t)r * cap + (n0 - jb.out0) + t] = __fmul_rn(su[t + kLimW + kLimL - 1], g);
  }
}

// save (dir = 0): the listed rows' current history halves and headers -> records; load (dir = 1): records -> the
// rows' current halves.  grid (n), kLimThreads threads; jobs[i] carries row i's header and current half, rows_dev its
// row.
__global__ void __launch_bounds__(kLimThreads) limit_move_kernel(const LimitJob* __restrict__ jobs,
                                                                 const int* __restrict__ rows_dev, float* hist, int rows,
                                                                 LimitRecord* rec, int dir) {
  const int i = blockIdx.x, t = threadIdx.x;
  const LimitJob jb = jobs[i];
  float* h = hist + ((size_t)jb.cur * rows + rows_dev[i]) * kLimHist;
  if (dir == 0) {
    for (int k = t; k < kLimHist; k += kLimThreads) rec[i].hist[k] = h[k];
    if (t == 0) { rec[i].gain = jb.gain; rec[i].unused = 0; rec[i].n_in = jb.n_in; }
  } else {
    for (int k = t; k < kLimHist; k += kLimThreads) h[k] = rec[i].hist[k];
  }
}
