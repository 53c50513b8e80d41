// fp32 register-tiled direct 1-D convolution, the one Conv1d / Linear kernel of the codec encoder and the speaker
// encoder.  Activations are [B][C][T] fp32, time contiguous.
//   y[b][y_off + co][t] = epi( bias[co] + sum_{ci,j} w[co][ci][j] * X[b][ci][t*stride + j*dil - pad_left] )
//   X = act_in(x[b][x_off + ci] (+ x2[b][x2_off + ci])), out-of-range time indices padded by `pad`
//   epi(v) = res + scale * act_out(v)   (scale and res optional; res is read in y's view)
// x (and x2) step xT floats per channel and y (and res) yT; 0 means Tin and Tout.  A larger step views the columns of a
// wider buffer, e.g. a streaming encoder's history-prefixed activations.  The steps are kernel arguments of their own
// rather than fields: a larger parameter struct costs the kernel its register allocation (48 instead of 64, ~4 % slower).
#pragma once
#include "common.cuh"

enum ConvPad { PAD_ZERO = 0, PAD_REPLICATE = 1, PAD_REFLECT = 2 };
enum ConvActIn { IN_NONE = 0, IN_ELU = 1, IN_TANH = 2 };
enum ConvActOut { OUT_NONE = 0, OUT_GELU = 1, OUT_RELU = 2, OUT_SIGMOID = 3 };

struct ConvF32Args {
  const float* x;      // [B][xC][Tin]  (channels [x_off, x_off + Cin) are read)
  const float* x2;     // optional second input added to x on load, [B][x2C][Tin] at channel offset x2_off
  const float* w;      // [Cout][Cin][k]
  const float* bias;   // [Cout] or null
  const float* scale;  // [Cout] or null (LayerScale)
  const float* res;    // [B][yC][Tout] or null, same view as y
  float* y;            // [B][yC][Tout] (channels [y_off, y_off + Cout) are written)
  int xC, x_off, x2C, x2_off, yC, y_off;
  int Cin, Cout, Tin, Tout, k, stride, dil, pad_left;
  int pad;             // ConvPad
  int act_in;          // ConvActIn
  int act_out;         // ConvActOut
};

#ifdef __CUDACC__
__device__ __forceinline__ int reflect_idx(int i, int T) {
  // torch "reflect" padding (no edge repetition); valid while the pad is < T
  if (i < 0) i = -i;
  if (i >= T) i = 2 * (T - 1) - i;
  return min(max(i, 0), T - 1);
}
#endif

int conv_f32_init();  // sets the kernel's 96 KB dynamic shared-memory limit on the current device
int conv_f32_launch(const ConvF32Args& a, int B, cudaStream_t stream, int xT = 0, int yT = 0);
