// Kernels of the streaming resampler (csrc/resample.cu; tests/csrc/resample_shim.cu launches them directly).
#pragma once
#include "common.cuh"
#include "../../include/qwen3tts_b200.h"

constexpr int kHist = Q3_RESAMPLE_HIST;
constexpr int kMaxFilters = 64;   // the FilterTable is a by-value kernel parameter (1.5 KB)
constexpr int kThreads = 256;

struct Filter {
  const float* taps;
  int up, down, hl;
};
struct FilterTable {
  Filter f[kMaxFilters];
};
static_assert(sizeof(FilterTable) <= 2048, "the filter table must stay well under the 4 KB kernel parameter limit");

// one row of one launch (or of a save / load)
struct RowJob {
  long long n_in;   // inputs before this launch
  long long out0;   // outputs emitted before this launch
  int count;        // new inputs (this launch)
  int nout;         // outputs this launch
  int end;          // the clip ends with this launch
  int fid, enc, cur;  // filter, encoding, current history half
};

// the saved image of one row (Q3_RESAMPLE_ROW_BYTES)
struct RowRecord {
  int32_t fid, enc;
  long long n_in;
  float hist[kHist];
};
static_assert(sizeof(RowRecord) == Q3_RESAMPLE_ROW_BYTES, "row record size");

// G.711 mu-law of a 16-bit sample, as audioop.lin2ulaw(..., 2) computes it: the 14-bit value (sample >> 2), its
// magnitude clipped at 8159, biased by 33, then segment and mantissa, all bits inverted
__device__ __forceinline__ uint8_t ulaw_of(int s16) {
  int v = s16 >> 2;
  int mask = 0xFF;
  if (v < 0) { v = -v; mask = 0x7F; }
  if (v > 8159) v = 8159;
  v += 0x84 >> 2;
  int seg = 0;
  while (seg < 8 && v > (0x40 << seg) - 1) ++seg;  // seg_uend = 0x3F, 0x7F, ..., 0x1FFF
  if (seg >= 8) return (uint8_t)(0x7F ^ mask);
  return (uint8_t)(((seg << 4) | ((v >> (seg + 1)) & 0xF)) ^ mask);
}

// grid (blocks over max(nout + kHist), rows).  Thread t < nout of row r computes output out0 + t; threads
// [nout, nout + kHist) write the row's next history half (zeros when the clip ends) for rows that moved.
__global__ void __launch_bounds__(kThreads) resample_poly_kernel(FilterTable ft, const RowJob* __restrict__ jobs,
                                                            const float* __restrict__ x, long long ld,
                                                            float* __restrict__ hist, int rows,
                                                            uint8_t* __restrict__ out, long long cap) {
  const int r = blockIdx.y;
  const RowJob jb = jobs[r];
  const int t = blockIdx.x * kThreads + threadIdx.x;
  const float* xr = x + (size_t)r * ld;
  const float* h_old = hist + ((size_t)jb.cur * rows + r) * kHist;
  const long long n_tot = jb.n_in + jb.count;
  if (t < jb.nout) {
    const Filter f = ft.f[jb.fid];
    const long long j = jb.out0 + t;
    const long long c = (long long)f.hl + j * f.down;  // tap index of input m is c - m*up
    long long m0 = c - 2LL * f.hl;
    m0 = m0 <= 0 ? 0 : (m0 + f.up - 1) / f.up;
    long long m1 = c / f.up;
    if (m1 > n_tot - 1) m1 = n_tot - 1;
    float acc = 0.f;
    for (long long m = m0; m <= m1; ++m) {
      const float xv = m >= jb.n_in ? __ldg(xr + (m - jb.n_in)) : h_old[kHist - (jb.n_in - m)];
      const float hv = __ldg(f.taps + (c - m * f.up));
      acc = m == m0 ? __fmul_rn(xv, hv) : __fmaf_rn(xv, hv, acc);
    }
    uint8_t* o = out + (size_t)r * cap;
    if (jb.enc == Q3_RESAMPLE_F32) {
      reinterpret_cast<float*>(o)[t] = acc;
    } else {
      const float q = fminf(fmaxf(rintf(acc * 32768.f), -32768.f), 32767.f);
      if (jb.enc == Q3_RESAMPLE_S16) reinterpret_cast<int16_t*>(o)[t] = (int16_t)q;
      else o[t] = ulaw_of((int)q);
    }
  } else if (t < jb.nout + kHist && (jb.count > 0 || jb.end)) {
    const int k = t - jb.nout;
    const long long m = n_tot - kHist + k;
    float v = 0.f;
    if (!jb.end && m >= 0) v = m >= jb.n_in ? xr[m - jb.n_in] : h_old[kHist - (jb.n_in - m)];
    hist[((size_t)(jb.cur ^ 1) * rows + r) * kHist + k] = v;
  }
}

// save (dir = 0): the listed rows' current history halves and headers -> records; load (dir = 1): records -> the
// rows' current halves.  grid (n), kHist threads; jobs[i] carries row i's header and current half, rows_dev its row.
__global__ void resample_move_kernel(const RowJob* __restrict__ jobs, const int* __restrict__ rows_dev, float* hist,
                                     int rows, RowRecord* rec, int dir) {
  const int i = blockIdx.x, k = threadIdx.x;
  const RowJob jb = jobs[i];
  float* h = hist + ((size_t)jb.cur * rows + rows_dev[i]) * kHist;
  if (dir == 0) {
    rec[i].hist[k] = h[k];
    if (k == 0) { rec[i].fid = jb.fid; rec[i].enc = jb.enc; rec[i].n_in = jb.n_in; }
  } else {
    h[k] = rec[i].hist[k];
  }
}

