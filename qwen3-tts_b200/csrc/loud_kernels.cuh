// Kernels of the streaming loudness normaliser (csrc/loud.cu; tests/csrc/loud_shim.cu launches them directly).
#pragma once
#include "common.cuh"
#include "../../include/qwen3tts_b200.h"

constexpr int kLdSeg = 2400;                         // samples per segment (100 ms at 24 kHz)
constexpr int kLdChunk = 32;                         // samples per chunk of the filter scan
constexpr int kLdChunks = kLdSeg / kLdChunk;         // 75
constexpr int kLdThreads = 256;
constexpr int kLdMaxBlocks = Q3_LOUD_MAX_BLOCKS;     // segments (and blocks) of one clip
constexpr int kLdMaxIn = 32768;                      // inputs per row per launch
constexpr int kLdMaxSegs = (kLdMaxIn + kLdSeg - 1) / kLdSeg + 1;   // segments one launch can complete, with room
static_assert(kLdChunks * kLdChunk == kLdSeg && kLdChunks <= kLdThreads, "loudness segment geometry");

// the K-weighting cascade: shelf b0 b1 b2 a1 a2, then high-pass b0 b1 b2 a1 a2 (a0 = 1), and the state transition over
// one chunk, M^32, row-major over the state (s1, s2, t1, t2).  Passed by value to the kernel.
struct LoudFilter {
  float c[10];
  float m32[16];
};

// the filter of fp32 sos[12] (rows b0 b1 b2 a0 a1 a2, a0 = 1): its coefficients, and M^32 in fp64 from them, rounded
inline LoudFilter loud_filter(const float* sos) {
  LoudFilter f{};
  const int idx[10] = {0, 1, 2, 4, 5, 6, 7, 8, 10, 11};
  for (int i = 0; i < 10; ++i) f.c[i] = sos[idx[i]];
  // the zero-input transition of the state (s1, s2, t1, t2) over one sample
  const double a1 = f.c[3], a2 = f.c[4], c0 = f.c[5], c1 = f.c[6], c2 = f.c[7], d1 = f.c[8], d2 = f.c[9];
  const double m[16] = {-a1, 1, 0, 0, -a2, 0, 0, 0, c1 - d1 * c0, 0, -d1, 1, c2 - d2 * c0, 0, -d2, 0};
  double p[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  for (int n = 0; n < kLdChunk; ++n) {
    double q[16];
    for (int r = 0; r < 4; ++r)
      for (int k = 0; k < 4; ++k) {
        double v = 0;
        for (int j = 0; j < 4; ++j) v += m[4 * r + j] * p[4 * j + k];
        q[4 * r + k] = v;
      }
    for (int i = 0; i < 16; ++i) p[i] = q[i];
  }
  for (int i = 0; i < 16; ++i) f.m32[i] = (float)p[i];
  return f;
}

// one row of one launch (or of a save / load)
struct LoudJob {
  long long n_in;   // inputs of the clip before this launch
  double target;    // LUFS
  int row;
  int count;        // new inputs (this launch)
};

// a row's state on the device, which is also its saved image (Q3_LOUD_ROW_BYTES).  The header is target .. z; target and
// n_in are kept on the host and written here only by a save.  A row with n_in = 0 reads nothing of it.
struct LoudRecord {
  double target;
  long long n_in;
  float a1, a2;                 // A_{k-1}, A_{k-2}: the gains of the last two completed segments (k = n_in / 2400)
  float zf[4];                  // the filter state after the last completed segment
  double z[3];                  // z_{k-3}, z_{k-2}, z_{k-1} (0 before the clip)
  float part[kLdSeg];           // inputs of the partial segment k
  double ms[kLdMaxBlocks];      // ms_j of blocks 0 .. k-1
};
static_assert(sizeof(LoudRecord) == Q3_LOUD_ROW_BYTES && offsetof(LoudRecord, part) == Q3_LOUD_HEADER_BYTES,
              "loudness row record size");
static_assert(sizeof(LoudRecord) % 16 == 0, "records move as 16-byte words");

// one step of the K-weighting cascade in transposed direct form II: x -> y, state (s1, s2, t1, t2)
__device__ __forceinline__ float loud_step(const LoudFilter& f, float* s, float x) {
  const float y1 = f.c[0] * x + s[0];
  s[0] = f.c[1] * x - f.c[3] * y1 + s[1];
  s[1] = f.c[2] * x - f.c[4] * y1;
  const float y2 = f.c[5] * y1 + s[2];
  s[2] = f.c[6] * y1 - f.c[8] * y2 + s[3];
  s[3] = f.c[7] * y1 - f.c[9] * y2;
  return y2;
}

// block loudness -0.691 + 10*log10(ms)
__device__ __forceinline__ double loud_l(double ms) { return -0.691 + 10.0 * log10(ms); }

// the sum over threads of (v, k) into (*v, *k), in a fixed tree; every thread gets the result
__device__ __forceinline__ void loud_reduce(double* rs, int* rk, double& v, int& k) {
  const int t = threadIdx.x;
  rs[t] = v;
  rk[t] = k;
  __syncthreads();
  for (int w = kLdThreads / 2; w > 0; w >>= 1) {
    if (t < w) { rs[t] += rs[t + w]; rk[t] += rk[t + w]; }
    __syncthreads();
  }
  v = rs[0];
  k = rk[0];
  __syncthreads();
}

// grid (jobs), kLdThreads threads: CTA i serves jobs[i], a row with inputs.  It measures each segment its inputs
// complete, in order: the segment's 75 chunks are filtered from zero state, a scan of the 4-float state carries
// M^32 * S + e from chunk to chunk, each chunk is filtered again from its true state and sums y^2 in fp64, and z_s (the
// chunks' sums in order), ms_s and the gain A_s follow (DESIGN §4.9).  Then every new input n = 2400k + i becomes
//   y[n] = x[n] * (A_{k-2} + (A_{k-1} - A_{k-2}) * fp32((i+1)/2400)),   fp32 round-to-nearest without contraction,
// and the row's header and partial segment are written back.
__global__ void __launch_bounds__(kLdThreads) loud_kernel(const LoudJob* __restrict__ jobs, LoudFilter f,
                                                          const float* __restrict__ x, long long ld,
                                                          LoudRecord* st, float* __restrict__ out,
                                                          long long cap) {
  __shared__ float seg[kLdChunks * (kLdChunk + 1)];   // a segment, chunk c at c*33 (no bank conflicts across chunks)
  __shared__ float e[kLdChunks][4], sc[kLdChunks + 1][4];
  __shared__ double zc[kLdChunks], rs[kLdThreads];
  __shared__ int rk[kLdThreads];
  __shared__ float A[kLdMaxSegs + 2];                  // A[i] = A_{S0-2+i}
  __shared__ double zh[3];
  const int t = threadIdx.x;
  const LoudJob jb = jobs[blockIdx.x];
  LoudRecord& R = st[jb.row];
  const float* xr = x + (size_t)jb.row * ld;
  const long long n0 = jb.n_in, n1 = n0 + jb.count;
  const long long S0 = n0 / kLdSeg, S1 = n1 / kLdSeg;
  if (t == 0) {
    const bool fresh = n0 == 0;
    A[0] = fresh ? 1.f : R.a2;
    A[1] = fresh ? 1.f : R.a1;
    for (int q = 0; q < 4; ++q) sc[0][q] = fresh ? 0.f : R.zf[q];
    for (int q = 0; q < 3; ++q) zh[q] = fresh ? 0.0 : R.z[q];
  }
  __syncthreads();
  for (long long s = S0; s < S1; ++s) {
    for (int i = t; i < kLdSeg; i += kLdThreads) {
      const long long p = s * kLdSeg + i;
      seg[(i / kLdChunk) * (kLdChunk + 1) + i % kLdChunk] = p < n0 ? R.part[i] : xr[p - n0];
    }
    __syncthreads();
    if (t < kLdChunks) {                               // zero-state response of chunk t
      float q[4] = {0.f, 0.f, 0.f, 0.f};
      const float* xs = seg + t * (kLdChunk + 1);
      for (int i = 0; i < kLdChunk; ++i) loud_step(f, q, xs[i]);
      for (int k = 0; k < 4; ++k) e[t][k] = q[k];
    }
    __syncthreads();
    if (t == 0) {                                      // the carry: S_{c+1} = M^32 S_c + e_c
      for (int c = 0; c < kLdChunks; ++c)
        for (int r = 0; r < 4; ++r) {
          float v = e[c][r];
          for (int k = 0; k < 4; ++k) v += f.m32[4 * r + k] * sc[c][k];
          sc[c + 1][r] = v;
        }
    }
    __syncthreads();
    if (t < kLdChunks) {                               // chunk t from its true state: sum of y^2
      float q[4] = {sc[t][0], sc[t][1], sc[t][2], sc[t][3]};
      const float* xs = seg + t * (kLdChunk + 1);
      double acc = 0.0;
      for (int i = 0; i < kLdChunk; ++i) {
        const double y = loud_step(f, q, xs[i]);
        acc += y * y;
      }
      zc[t] = acc;
    }
    __syncthreads();
    if (t == 0) {
      double z = 0.0;
      for (int c = 0; c < kLdChunks; ++c) z += zc[c];
      const double sum = ((zh[0] + zh[1]) + zh[2]) + z;
      R.ms[s] = sum / (double)(kLdSeg * (s < 3 ? s + 1 : 4));
      zh[0] = zh[1]; zh[1] = zh[2]; zh[2] = z;
      for (int k = 0; k < 4; ++k) sc[0][k] = sc[kLdChunks][k];
    }
    __syncthreads();
    // the gate over blocks 0 .. s: each thread sums blocks t, t + 256, ... in order, then a fixed tree
    double v = 0.0;
    int k = 0;
    for (long long j = t; j <= s; j += kLdThreads) {
      const double m = R.ms[j];
      if (loud_l(m) > -70.0) { v += m; ++k; }
    }
    loud_reduce(rs, rk, v, k);
    const int ia = (int)(s - S0) + 2;
    if (k == 0) {
      if (t == 0) A[ia] = A[ia - 1];
    } else {
      const double gr = loud_l(v / k) - 10.0;
      double v2 = 0.0;
      int k2 = 0;
      for (long long j = t; j <= s; j += kLdThreads) {
        const double m = R.ms[j], l = loud_l(m);
        if (l > -70.0 && l > gr) { v2 += m; ++k2; }
      }
      loud_reduce(rs, rk, v2, k2);
      if (t == 0) {
        const double d = fmin(fmax(jb.target - loud_l(v2 / k2), -30.0), 30.0);
        A[ia] = (float)exp10(d / 20.0);
      }
    }
    __syncthreads();
  }
  float* yr = out + (size_t)jb.row * cap;
  for (int q = t; q < jb.count; q += kLdThreads) {
    const long long n = n0 + q;
    const long long k = n / kLdSeg;
    const int i = (int)(n - k * kLdSeg);
    const float aa = A[k - S0 + 1], ab = A[k - S0];
    const float r = __fdiv_rn((float)(i + 1), (float)kLdSeg);
    const float g = __fadd_rn(ab, __fmul_rn(__fsub_rn(aa, ab), r));
    yr[q] = __fmul_rn(xr[q], g);
  }
  // the partial segment S1: inputs before n0 are already there when S1 = S0
  for (long long p = (S1 * kLdSeg > n0 ? S1 * kLdSeg : n0) + t; p < n1; p += kLdThreads)
    R.part[p - S1 * kLdSeg] = xr[p - n0];
  if (t == 0) {
    R.a1 = A[S1 - S0 + 1];
    R.a2 = A[S1 - S0];
    for (int q = 0; q < 4; ++q) R.zf[q] = sc[0][q];
    for (int q = 0; q < 3; ++q) R.z[q] = zh[q];
  }
}

// save (dir = 0): the listed rows' states -> records, with each job's target and n_in in the header; load (dir = 1):
// records -> the rows' states.  grid (n), kLdThreads threads.
__global__ void __launch_bounds__(kLdThreads) loud_move_kernel(const LoudJob* __restrict__ jobs, LoudRecord* st,
                                                               LoudRecord* rec, int dir) {
  const int i = blockIdx.x, t = threadIdx.x;
  const LoudJob jb = jobs[i];
  const int4* src = reinterpret_cast<const int4*>(dir == 0 ? &st[jb.row] : &rec[i]);
  int4* dst = reinterpret_cast<int4*>(dir == 0 ? &rec[i] : &st[jb.row]);
  for (int k = t; k < (int)(sizeof(LoudRecord) / 16); k += kLdThreads) dst[k] = src[k];
  if (dir == 0) {
    __syncthreads();
    if (t == 0) { rec[i].target = jb.target; rec[i].n_in = jb.n_in; }
  }
}
