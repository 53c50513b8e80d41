// Small kernels of the speaker encoder (log-mel front end, SE mean / gate, channel copy, attentive statistics
// pooling).  Part of the speaker_encoder.cu translation unit; tests/csrc/encoder_shim.cu includes it too, to run
// these kernels on inputs a test chooses.
#pragma once
#include "common.cuh"
#include "conv_f32.cuh"

namespace {

// log-mel front end (:396-448): one block per (frame, batch row).  Reflect-pad (n_fft - hop)/2 both sides, Hann window,
// |DFT| = sqrt(re^2 + im^2 + 1e-9) for bins 0..n_fft/2, mel projection with the librosa-style filterbank (host-computed,
// transposed [bins][mels]), log(clamp(., 1e-5)).  twc/tws: cos/sin(2*pi*j/n_fft), j < n_fft: index (k*n) mod n_fft is exact.
__global__ void __launch_bounds__(256) melspec_kernel(const float* __restrict__ wav, int T, const float* __restrict__ window,
                                                      const float* __restrict__ twc, const float* __restrict__ tws,
                                                      const float* __restrict__ fbT, float* __restrict__ out, int n_fft,
                                                      int hop, int n_mels, int n_frames) {
  extern __shared__ float sm[];
  float* xw = sm;                  // [n_fft] windowed samples
  float* c = xw + n_fft;           // [n_fft]
  float* s = c + n_fft;            // [n_fft]
  float* mag = s + n_fft;          // [n_fft/2 + 1]
  const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int pad = (n_fft - hop) / 2;
  const float* y = wav + (size_t)b * T;
  for (int n = tid; n < n_fft; n += 256) {
    xw[n] = y[reflect_idx(f * hop + n - pad, T)] * window[n];
    c[n] = twc[n];
    s[n] = tws[n];
  }
  __syncthreads();
  const int nb = n_fft / 2 + 1, mask = n_fft - 1;
  for (int k = tid; k < nb; k += 256) {
    float re = 0.f, im = 0.f;
    int idx = 0;
    for (int n = 0; n < n_fft; ++n) {
      re = fmaf(xw[n], c[idx], re);
      im = fmaf(-xw[n], s[idx], im);
      idx = (idx + k) & mask;
    }
    mag[k] = sqrtf(re * re + im * im + 1e-9f);
  }
  __syncthreads();
  for (int m = tid; m < n_mels; m += 256) {
    float v = 0.f;
    for (int k = 0; k < nb; ++k) v = fmaf(fbT[(size_t)k * n_mels + m], mag[k], v);
    out[((size_t)b * n_mels + m) * n_frames + f] = logf(fmaxf(v, 1e-5f));
  }
}

// mean over time of channels [c_off, c_off + C) of x [B][xC][T] -> m [B][C]  (SqueezeExcitationBlock :151)
__global__ void mean_t_kernel(const float* __restrict__ x, int xC, int c_off, int C, int T, float* __restrict__ m) {
  const int c = blockIdx.x, b = blockIdx.y, lane = threadIdx.x;
  const float* xp = x + ((size_t)b * xC + c_off + c) * T;
  float s = 0.f;
  for (int t = lane; t < T; t += 32) s += xp[t];
  s = warp_sum(s);
  if (lane == 0) m[(size_t)b * C + c] = s / (float)T;
}

// y[b][y_off + c][t] = h[b][c][t] * gate[b][c] + res[b][r_off + c][t]   (SE gate + the block's residual, :157, :296-297)
__global__ void se_apply_kernel(const float* __restrict__ h, const float* __restrict__ gate, const float* __restrict__ res,
                                int rC, int r_off, float* __restrict__ y, int yC, int y_off, int C, int T) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
  if (t >= T) return;
  y[((size_t)b * yC + y_off + c) * T + t] =
      h[((size_t)b * C + c) * T + t] * gate[(size_t)b * C + c] + res[((size_t)b * rC + r_off + c) * T + t];
}

// copy channels: y[b][y_off + c][t] = x[b][x_off + c][t]   (Res2Net chunk 0 passes through, :119-120)
__global__ void copy_ch_kernel(const float* __restrict__ x, int xC, int x_off, float* __restrict__ y, int yC, int y_off, int T) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
  if (t >= T) return;
  y[((size_t)b * yC + y_off + c) * T + t] = x[((size_t)b * xC + x_off + c) * T + t];
}

// AttentiveStatisticsPooling, first half (:203-215): uniform-weight mean / std over time, then the concatenation
// [x ; mean ; std] broadcast along time.  One warp per (b, c).
__global__ void asp_cat_kernel(const float* __restrict__ x, float* __restrict__ cat, int C, int T, float eps) {
  const int c = blockIdx.x, b = blockIdx.y, lane = threadIdx.x;
  const float* xp = x + ((size_t)b * C + c) * T;
  const float w = 1.f / (float)T;
  float s = 0.f;
  for (int t = lane; t < T; t += 32) s += w * xp[t];
  const float mean = warp_sum(s);
  float v = 0.f;
  for (int t = lane; t < T; t += 32) { const float d = xp[t] - mean; v += w * d * d; }
  const float sd = sqrtf(fmaxf(warp_sum(v), eps));
  float* o0 = cat + ((size_t)b * 3 * C + c) * T;
  float* o1 = cat + ((size_t)b * 3 * C + C + c) * T;
  float* o2 = cat + ((size_t)b * 3 * C + 2 * C + c) * T;
  for (int t = lane; t < T; t += 32) { o0[t] = xp[t]; o1[t] = mean; o2[t] = sd; }
}

// second half (:217-226): softmax over time of the attention logits per channel, attention-weighted mean / std,
// pooled = [mean ; std]  ([B][2C]).  One warp per (b, c).
__global__ void asp_pool_kernel(const float* __restrict__ x, const float* __restrict__ att, float* __restrict__ pooled, int C, int T,
                                float eps) {
  const int c = blockIdx.x, b = blockIdx.y, lane = threadIdx.x;
  const float* xp = x + ((size_t)b * C + c) * T;
  const float* ap = att + ((size_t)b * C + c) * T;
  float mx = -INFINITY;
  for (int t = lane; t < T; t += 32) mx = fmaxf(mx, ap[t]);
  mx = warp_max(mx);
  float z = 0.f;
  for (int t = lane; t < T; t += 32) z += expf(ap[t] - mx);
  z = warp_sum(z);
  float s = 0.f;
  for (int t = lane; t < T; t += 32) s += expf(ap[t] - mx) / z * xp[t];
  const float mean = warp_sum(s);
  float v = 0.f;
  for (int t = lane; t < T; t += 32) { const float d = xp[t] - mean; v += expf(ap[t] - mx) / z * d * d; }
  const float sd = sqrtf(fmaxf(warp_sum(v), eps));
  if (lane == 0) { pooled[(size_t)b * 2 * C + c] = mean; pooled[(size_t)b * 2 * C + C + c] = sd; }
}

}  // namespace
