// Shared launcher of the Hopper tensor-core convolution (conv_f16.cu): an implicit GEMM on SPLIT operand pairs,
// wgmma from shared memory, fp32 accumulators in registers. Used by the split-fp16 path (conv_f16.cu) and by the
// 3xTF32 path (conv_tc.cu).
#pragma once
#include <cuda_runtime.h>

constexpr int WG_MAX_TAP2D = 16;

// One convolution (or one output-parity class of a transposed one). Operands:
//   activations  x_hi / x_lo  channels-last [N][Din][Hin][Win][Cs_in], Cin_pad (% 32) channels used
//   weights      w_hi / w_lo  K-major [tap][Cout_pad][Cin_pad], consecutive taps w_tap_stride elements apart
// tf32 = 0: fp16 halves, x = hi + lo * 2^-11;  tf32 = 1: fp32 words holding TF32 values, x = hi + lo.
// Product: a_hi b_hi + (a_hi b_lo + a_lo b_hi) * scale, accumulated in fp32.
struct WgConv {
  int tf32;
  const void *x_hi, *x_lo;
  int N, Din, Hin, Win, Cin_pad, Cs_in;
  const void *w_hi, *w_lo;
  long long w_tap_stride;
  int n_wslices, Cout_pad;
  const float* bias;
  double* stats;                         // [2][Cout] (sum, sum of squares) of the stored values, or null
  float* y;                              // fp32 output [N][Dout][Hout][Wout][Cs_out] at channel offset c_off ...
  void *y_hi, *y_lo;                     // ... or (when non-null) the fp16 operand pair of the next convolution
  int Cout, Dout, Hout, Wout, Cs_out, c_off, out_stride, out_off_y, out_off_x, leaky;
  int Hy, Wx, in_stride;                 // output positions per plane (before the parity interleave), conv stride
  int n_kz, n_tap;                       // depth taps, in-plane taps
  signed char dz[3], dy[WG_MAX_TAP2D], dx[WG_MAX_TAP2D];
  unsigned char wsel[3 * WG_MAX_TAP2D];  // weight slice of (kz, tap)
};

int conv_wgmma(const WgConv& c, cudaStream_t st);
