// Shared launcher of the Hopper tensor-core convolution (conv_f16.cu): an implicit GEMM on SPLIT operand pairs,
// wgmma from shared memory, fp32 accumulators in registers. Used by the split-fp16 path (conv_f16.cu) and by the
// 3xTF32 path (conv_tc.cu).
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"

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
  // affine epilogue (split-fp16 only; replaces bias / LeakyReLU / statistics when aff_scale is set):
  // v = acc * aff_scale[c] + aff_shift[c], + residual (fp32 `res`, or the pair res_hi + res_lo * 2^-11, laid out like the output),
  // then max(v, 0) when relu
  const float *aff_scale, *aff_shift, *res;
  const void *res_hi, *res_lo;
  int relu;
  int Hy, Wx, in_stride;                 // output positions per plane (before the parity interleave), conv stride
  int n_kz, n_tap;                       // depth taps, in-plane taps
  signed char dz[3], dy[WG_MAX_TAP2D], dx[WG_MAX_TAP2D];
  unsigned char wsel[3 * WG_MAX_TAP2D];  // weight slice of (kz, tap)
};

int conv_wgmma(const WgConv& c, cudaStream_t st);

// The geometry both operand forms share. The callers set the operands, the weight layout and the epilogue.

// Filters conv_wgmma takes (kd <= 3 depth taps, kh * kw <= WG_MAX_TAP2D in-plane taps, stride <= 8), and the output extent
// of nn.Conv2d for this input, kernel, stride, padding and dilation.
inline int wg_check_conv_shape(int Hin, int Win, int kd, int kh, int kw, int stride, int pad, int dilation, int Hout, int Wout) {
  NRGBD_REQUIRE(kd >= 1 && kd <= 3 && kh * kw <= WG_MAX_TAP2D && stride >= 1 && stride <= 8, "unsupported filter");
  NRGBD_REQUIRE(Hout == (Hin + 2 * pad - dilation * (kh - 1) - 1) / stride + 1 &&
                    Wout == (Win + 2 * pad - dilation * (kw - 1) - 1) / stride + 1, "output extent mismatch");
  return NRGBD_OK;
}

// Output extents, stride and tap table of a kd x kh x kw convolution (depth: stride 1, padding kd / 2): tap t reads
// weight slice t. c.Din must be set.
inline void wg_conv_taps(WgConv& c, int kd, int kh, int kw, int stride, int pad, int dilation, int Hout, int Wout) {
  c.n_wslices = kd * kh * kw;
  c.Dout = c.Din; c.Hout = Hout; c.Wout = Wout; c.out_stride = 1; c.out_off_y = 0; c.out_off_x = 0;
  c.Hy = Hout; c.Wx = Wout; c.in_stride = stride; c.n_kz = kd; c.n_tap = kh * kw;
  for (int a = 0; a < kd; ++a) c.dz[a] = (signed char)(a - kd / 2);
  int t = 0;
  for (int b = 0; b < kh; ++b)
    for (int e = 0; e < kw; ++e) { c.dy[t] = (signed char)(b * dilation - pad); c.dx[t] = (signed char)(e * dilation - pad); ++t; }
  for (int a = 0; a < kd * kh * kw; ++a) c.wsel[a] = (unsigned char)a;
}

// Output-parity class (py, px) of nn.ConvTranspose2d(kernel 4, stride 2, padding 1) on a 2-D Hin x Win input (c.Hin,
// c.Win): a stride-1 convolution of 2 x 2 taps of the 16-slice weight, written to every second output row and column.
inline void wg_transpose_k4s2_class(WgConv& c, int py, int px) {
  const int kys[2][2] = {{1, 3}, {0, 2}};
  const int dys[2][2] = {{0, -1}, {1, 0}};
  c.n_wslices = 16;
  c.Din = 1; c.Dout = 1; c.Hout = 2 * c.Hin; c.Wout = 2 * c.Win; c.out_stride = 2; c.out_off_y = py; c.out_off_x = px;
  c.Hy = c.Hin; c.Wx = c.Win; c.in_stride = 1; c.n_kz = 1; c.n_tap = 4;
  int t = 0;
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      c.dy[t] = (signed char)dys[py][a]; c.dx[t] = (signed char)dys[px][b];
      c.wsel[t] = (unsigned char)(kys[py][a] * 4 + kys[px][b]); ++t;
    }
}
