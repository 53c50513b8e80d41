// Kernels of the streaming WSOLA time-stretch (csrc/stretch.cu; tests/csrc/stretch_shim.cu launches them directly).
#pragma once
#include "common.cuh"
#include "../../include/qwen3tts_b200.h"

constexpr int kStHist = Q3_STRETCH_HIST;  // inputs a row keeps: its next frame reads at most 1920 back
constexpr int kStN = 960;                 // frame length
constexpr int kStHs = 480;                // synthesis hop
constexpr int kStDelta = 240;             // search tolerance
constexpr int kStCand = 2 * kStDelta + 1;  // candidate offsets, one per thread
constexpr int kStThreads = 512;
constexpr int kStPad = 1200;   // zeros staged past an ended clip: a frame k < ceil(M/480) reads below n + 1199
constexpr int kStMaxIn = 32768;

// one row of one launch (or of a save / load)
struct StretchJob {
  long long n_in;  // inputs before this launch
  long long f0;    // frames done before this launch (outputs emitted: 480 * f0)
  int row;
  int count;       // new inputs (this launch)
  int nf;          // frames this launch
  int nout;        // outputs this launch
  int end;         // the clip ends with this launch
  int ha;          // analysis hop
};

// the saved image of one row (Q3_STRETCH_ROW_BYTES)
struct StretchRecord {
  int32_t ha, unused;
  long long n_in, frames, p_last;
  float tail[kStHs];
  float hist[kStHist];
};
static_assert(sizeof(StretchRecord) == Q3_STRETCH_ROW_BYTES, "stretch row record size");

// the argmax key of candidate d with correlation c: larger c first, then smaller |d|, then negative d.  A total order
// on the candidates, so any reduction order picks the same one.  +0 and -0 compare equal, as the floats do.
__device__ __forceinline__ unsigned long long wsola_key(float c, int d) {
  uint32_t b = __float_as_uint(c == 0.f ? 0.f : c);
  b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  const int ad = d < 0 ? -d : d;
  return ((unsigned long long)b << 32) | (unsigned long long)((kStDelta - ad) << 1) | (unsigned long long)(d < 0);
}
__device__ __forceinline__ int wsola_key_delta(unsigned long long key) {
  const int ad = kStDelta - (int)((key >> 1) & 0xFF);
  return (key & 1) ? -ad : ad;
}
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
    v = u > v ? u : v;
  }
  return v;
}

// grid (rows with work), kStThreads threads, (kStHist + max count + kStPad) * 4 bytes of dynamic shared memory.
// The CTA stages s[j] = x[n_in - kStHist + j]: the row's history, its new inputs, and zeros past an ended clip.  Per
// frame k >= 1, thread j < 481 sums C(j - 240) alone; a block-wide max of the keys picks d_k; threads i < 480 then
// write output k*480 + i and keep the frame's windowed second half (the tail) in a register for the next frame.
// Finally the row's last kStHist inputs, its tail and p of its last frame go back (unless the clip ended).
__global__ void __launch_bounds__(kStThreads) wsola_kernel(const StretchJob* __restrict__ jobs,
                                                         const float* __restrict__ window, const float* __restrict__ x,
                                                         long long ld, float* __restrict__ hist,
                                                         float* __restrict__ tail, long long* __restrict__ plast,
                                                         float* __restrict__ out, long long cap) {
  extern __shared__ float s[];
  __shared__ unsigned long long red[kStThreads / 32];
  __shared__ long long p_sh;
  const StretchJob jb = jobs[blockIdx.x];
  const int r = jb.row, t = threadIdx.x;
  float* hr = hist + (size_t)r * kStHist;
  const float* xr = x + (size_t)r * ld;
  const int len = kStHist + jb.count;
  const int span = len + (jb.end ? kStPad : 0);
  for (int j = t; j < span; j += kStThreads) s[j] = j < kStHist ? hr[j] : (j < len ? xr[j - kStHist] : 0.f);
  const float wlo = t < kStHs ? window[t] : 0.f, whi = t < kStHs ? window[t + kStHs] : 0.f;
  float tl = (t < kStHs && jb.f0 > 0) ? tail[(size_t)r * kStHs + t] : 0.f;
  long long p_prev = jb.f0 > 0 ? plast[r] : 0;
  const long long base = jb.n_in - kStHist;
  float* orow = out + (size_t)r * cap;
  __syncthreads();
  for (int f = 0; f < jb.nf; ++f) {
    const long long k = jb.f0 + f;
    long long pk = 0;
    if (k > 0) {
      const long long ak = k * jb.ha;
      unsigned long long key = 0;
      if (t < kStCand) {
        const float* ref = s + (p_prev + kStHs - base);
        const float* cand = s + (ak - kStDelta - base) + t;
        float c = 0.f;
#pragma unroll 8
        for (int n = 0; n < kStHs; ++n) c = __fmaf_rn(ref[n], cand[n], c);
        key = wsola_key(c, t - kStDelta);
      }
      key = warp_max_u64(key);
      if ((t & 31) == 0) red[t >> 5] = key;
      __syncthreads();
      if (t < 32) {
        key = warp_max_u64(t < kStThreads / 32 ? red[t] : 0ull);
        if (t == 0) p_sh = ak + wsola_key_delta(key);
      }
      __syncthreads();
      pk = p_sh;
    }
    if (t < kStHs) {
      const float* xf = s + (pk - base);
      const float y = k == 0 ? xf[t] : __fadd_rn(__fmul_rn(wlo, xf[t]), tl);
      tl = __fmul_rn(whi, xf[t + kStHs]);
      const long long o = (k - jb.f0) * kStHs + t;
      if (o < jb.nout) orow[o] = y;
    }
    p_prev = pk;
  }
  if (jb.end) return;   // the row starts a new clip: it reads none of its state
  for (int j = t; j < kStHist; j += kStThreads) hr[j] = s[jb.count + j];
  if (jb.nf > 0) {
    if (t < kStHs) tail[(size_t)r * kStHs + t] = tl;
    if (t == 0) plast[r] = p_prev;
  }
}

// save (dir = 0): the listed rows' state -> records; load (dir = 1): records -> the rows.  grid (n), kStThreads
// threads; jobs[i] carries row i's index and host header (ha, n_in, f0).
__global__ void __launch_bounds__(kStThreads) stretch_move_kernel(const StretchJob* __restrict__ jobs, float* hist,
                                                                float* tail, long long* plast, StretchRecord* rec,
                                                                int dir) {
  const int i = blockIdx.x, t = threadIdx.x;
  const StretchJob jb = jobs[i];
  float* h = hist + (size_t)jb.row * kStHist;
  float* tl = tail + (size_t)jb.row * kStHs;
  StretchRecord& R = rec[i];
  if (dir == 0) {
    for (int j = t; j < kStHist; j += kStThreads) R.hist[j] = h[j];
    if (t < kStHs) R.tail[t] = tl[t];
    if (t == 0) {
      R.ha = jb.ha; R.unused = 0; R.n_in = jb.n_in; R.frames = jb.f0;
      R.p_last = jb.f0 > 0 ? plast[jb.row] : 0;
    }
  } else {
    for (int j = t; j < kStHist; j += kStThreads) h[j] = R.hist[j];
    if (t < kStHs) tl[t] = R.tail[t];
    if (t == 0) plast[jb.row] = R.p_last;
  }
}
