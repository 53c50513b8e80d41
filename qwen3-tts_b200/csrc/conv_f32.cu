// fp32 direct 1-D convolution (conv_f32.cuh): one launch per Conv1d / Linear of the codec encoder and the speaker encoder.
#include "conv_f32.cuh"

namespace {

constexpr int CT = 64;   // output channels per block
constexpr int TT = 64;   // output time steps per block
constexpr int CI = 8;    // input channels staged per iteration
constexpr size_t kMaxSmem = 96 * 1024;

__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v : expm1f(v); }
__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f)); }

// block = 256 threads = 16 (channel groups of 4) x 16 (time lanes; each owns t = lane + 16*i, i < 4)
__global__ void __launch_bounds__(256) conv_f32_kernel(const ConvF32Args a, const int xT, const int yT) {
  extern __shared__ float sm[];
  const int XW = (TT - 1) * a.stride + (a.k - 1) * a.dil + 1;
  float* xs = sm;                 // [CI][XW]
  float* ws = sm + CI * XW;       // [CT][CI][k]
  const int b = blockIdx.z, co0 = blockIdx.y * CT, t0 = blockIdx.x * TT;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int in0 = t0 * a.stride - a.pad_left;  // input index of xs[.][0]
  const float* xb = a.x + ((size_t)b * a.xC + a.x_off) * xT;
  const float* x2b = a.x2 ? a.x2 + ((size_t)b * a.x2C + a.x2_off) * xT : nullptr;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int c0 = 0; c0 < a.Cin; c0 += CI) {
    __syncthreads();
#pragma unroll 4
    for (int e = tid; e < CI * XW; e += 256) {
      const int ci = e / XW, p = e - ci * XW;
      float v = 0.f;
      if (c0 + ci < a.Cin) {
        int ti = in0 + p;
        if (a.pad == PAD_REPLICATE) ti = min(max(ti, 0), a.Tin - 1);
        else if (a.pad == PAD_REFLECT) ti = reflect_idx(ti, a.Tin);
        if (ti >= 0 && ti < a.Tin) {
          v = xb[(size_t)(c0 + ci) * xT + ti];
          if (x2b) v += x2b[(size_t)(c0 + ci) * xT + ti];
          if (a.act_in == IN_ELU) v = elu1(v);
          else if (a.act_in == IN_TANH) v = tanhf(v);
        }
      }
      xs[e] = v;
    }
    const int wk = CI * a.k;
#pragma unroll 4
    for (int e = tid; e < CT * wk; e += 256) {
      const int co = e / wk, r = e - co * wk, ci = r / a.k, j = r - ci * a.k;
      float v = 0.f;
      if (co0 + co < a.Cout && c0 + ci < a.Cin) v = a.w[((size_t)(co0 + co) * a.Cin + c0 + ci) * a.k + j];
      ws[e] = v;
    }
    __syncthreads();
    for (int ci = 0; ci < CI; ++ci) {
      const float* xr = xs + ci * XW;
      for (int j = 0; j < a.k; ++j) {
        float wv[4], xv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) wv[i] = ws[((ty * 4 + i) * CI + ci) * a.k + j];
#pragma unroll
        for (int i = 0; i < 4; ++i) xv[i] = xr[(tx + 16 * i) * a.stride + j * a.dil];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[i][q] = fmaf(wv[i], xv[q], acc[i][q]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + ty * 4 + i;
    if (co >= a.Cout) continue;
    const float bv = a.bias ? a.bias[co] : 0.f;
    const float sc = a.scale ? a.scale[co] : 1.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int t = t0 + tx + 16 * q;
      if (t >= a.Tout) continue;
      float v = acc[i][q] + bv;
      if (a.act_out == OUT_GELU) v = gelu_erf(v);
      else if (a.act_out == OUT_RELU) v = fmaxf(v, 0.f);
      else if (a.act_out == OUT_SIGMOID) v = 1.f / (1.f + expf(-v));
      const size_t o = ((size_t)b * a.yC + a.y_off + co) * yT + t;
      if (a.scale) v = sc * v;
      if (a.res) v = a.res[o] + v;
      a.y[o] = v;
    }
  }
}

}  // namespace

int conv_f32_init() {
  Q3_CUDA(cudaFuncSetAttribute(conv_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
  return 0;
}

int conv_f32_launch(const ConvF32Args& a, int B, cudaStream_t stream, int xT, int yT) {
  const int XW = (TT - 1) * a.stride + (a.k - 1) * a.dil + 1;
  const size_t smem = (size_t)(CI * XW + CT * CI * a.k) * sizeof(float);
  Q3_REQUIRE(smem <= kMaxSmem, "conv tile needs %zu B of shared memory", smem);
  dim3 grid((a.Tout + TT - 1) / TT, (a.Cout + CT - 1) / CT, B);
  conv_f32_kernel<<<grid, 256, smem, stream>>>(a, xT ? xT : a.Tin, yT ? yT : a.Tout);
  return 0;
}
