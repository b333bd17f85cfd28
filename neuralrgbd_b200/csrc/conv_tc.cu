// Tensor-core convolution with error-compensated 3xTF32 products (SURVEY §8 a5, a8, a10; DESIGN.md §4.2):
// the `conv_math = 'tf32x3'` path. The GEMM is the wgmma kernel of conv_f16.cu (conv_wgmma) on TF32 operand pairs.
//
// Why 3xTF32: the reference's results must be matched to 1e-4 on the DPV through 61 (2-D) / 12 (3-D)
// convolutions separated by batch-statistics BatchNorm; single-pass TF32 operands give 1e-2-level
// DPV errors (SURVEY §7). Each fp32 operand is split a = a_hi + a_lo with a_hi = RN_tf32(a),
// a_lo = RN_tf32(a - a_hi) and the product is accumulated as a_hi*b_hi + a_lo*b_hi + a_hi*b_lo in
// fp32 (dropped term <= 2^-22 |a b|).
//
// The activations reach the GEMM as TF32 pairs written by nrgbd_split_tf32, which can also apply the producing
// convolution's training-mode BatchNorm + ReLU: one pass (4 B read + 8 B written per element) then replaces the separate
// BatchNorm pass (4 B read + 4 B written) in front of the split.
#include <cuda.h>

#include "common.cuh"
#include "conv_wgmma.cuh"
#include "../../include/nrgbd.h"

namespace {

__device__ __forceinline__ float rn_tf32(float a) {
  uint32_t b;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(b) : "f"(a));
  return __uint_as_float(b);
}

// channels-last x [pos][Cs] -> TF32 pair [pos][Cin_pad] of [relu](x * scale + shift) (scale == null: x itself); channels
// >= C are zero. Four channels per thread (Cin_pad % 4 == 0, Cs % 4 == 0).
__global__ void __launch_bounds__(256)
split_tf32_kernel(const float* __restrict__ x, long long n4, int Cs, int Cin_pad, int C, const float* __restrict__ scale,
                  const float* __restrict__ shift, int relu, float4* __restrict__ hi, float4* __restrict__ lo) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const unsigned q = (unsigned)Cin_pad / 4;
  // the 32-bit division where the index fits: the 64-bit one costs several times its instructions in this memory-bound pass
  const long long pos = i <= 0xFFFFFFFFll ? (long long)((unsigned)i / q) : i / q;
  const int c0 = (int)(i - pos * q) * 4;
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  if (c0 < C) {
    const float4 a = *reinterpret_cast<const float4*>(x + pos * Cs + c0);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (c0 + k >= C) v[k] = 0.f;
      else if (scale) {
        v[k] = fmaf(v[k], scale[c0 + k], shift[c0 + k]);
        if (relu) v[k] = fmaxf(v[k], 0.f);
      }
    }
  }
  float h[4], l[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    h[k] = rn_tf32(v[k]);
    l[k] = rn_tf32(v[k] - h[k]);
  }
  hi[i] = make_float4(h[0], h[1], h[2], h[3]);
  lo[i] = make_float4(l[0], l[1], l[2], l[3]);
}

// PyTorch weight -> K-major packed hi / lo [tap][Cout_pad][Cin_pad]
__global__ void pack_weight_tc_kernel(const float* __restrict__ w, int kind, int Cout, int Cin, int taps, int Cin_pad,
                                      int Cout_pad, float* __restrict__ hi, float* __restrict__ lo) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n = (long long)taps * Cin_pad * Cout_pad;
  if (i >= n) return;
  int ci = (int)(i % Cin_pad);
  int co = (int)((i / Cin_pad) % Cout_pad);
  int t = (int)(i / ((long long)Cout_pad * Cin_pad));
  float v = 0.f;
  if (co < Cout && ci < Cin) v = kind == 0 ? w[((long long)co * Cin + ci) * taps + t] : w[((long long)ci * Cout + co) * taps + t];
  const float h = rn_tf32(v);
  hi[i] = h; lo[i] = rn_tf32(v - h);
}

// The TF32 operands of a convolution; the caller adds the geometry (wg_conv_taps / wg_transpose_k4s2_class)
WgConv tf32_conv(const float* x_hi, const float* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                 const float* w_lo, const float* bias, int Cout, int Cout_pad, float* y, int Cs_out, int c_off, int leaky,
                 double* stats) {
  WgConv c{};
  c.tf32 = 1;
  c.x_hi = x_hi; c.x_lo = x_lo; c.N = N; c.Din = Din; c.Hin = Hin; c.Win = Win; c.Cin_pad = Cin_pad; c.Cs_in = Cs_in;
  c.w_hi = w_hi; c.w_lo = w_lo; c.w_tap_stride = (long long)Cout_pad * Cin_pad; c.Cout_pad = Cout_pad;
  c.bias = bias; c.stats = stats; c.y = y;
  c.Cout = Cout; c.Cs_out = Cs_out; c.c_off = c_off; c.leaky = leaky;
  return c;
}

}  // namespace

extern "C" {

// Whether the tensor-core path can run a convolution with these channel counts.
int nrgbd_conv_tc_supported(int Cin_pad, int Cout_pad) {
  return (Cin_pad % 32 == 0 && Cin_pad >= 32 && Cout_pad % 16 == 0 && Cout_pad >= 16 && Cout_pad <= 256) ? 1 : 0;
}

// channels-last x [n_pos][Cs_in] -> TF32 pair hi / lo [n_pos][Cin_pad]: channels below C hold x, or [relu](x * scale + shift)
// when scale is set; channels from C up to Cin_pad hold zero.
int nrgbd_split_tf32(const float* x, long long n_pos, int Cs_in, int Cin_pad, int C, const float* scale, const float* shift,
                     int relu, float* hi, float* lo, cudaStream_t st) {
  NRGBD_REQUIRE(x && hi && lo && n_pos > 0, "bad arguments");
  NRGBD_REQUIRE(Cin_pad % 32 == 0 && Cs_in % 4 == 0 && C >= 1 && C <= Cin_pad && Cin_pad <= Cs_in, "bad channel counts");
  NRGBD_REQUIRE((((uintptr_t)x | (uintptr_t)hi | (uintptr_t)lo) & 15) == 0, "x, hi and lo must be 16-byte aligned");
  NRGBD_REQUIRE((scale == nullptr) == (shift == nullptr), "scale and shift must both be set or both be null");
  const long long n4 = n_pos * (Cin_pad / 4);
  split_tf32_kernel<<<ceil_div(n4, 256), 256, 0, st>>>(x, n4, Cs_in, Cin_pad, C, scale, shift, relu, reinterpret_cast<float4*>(hi),
                                                       reinterpret_cast<float4*>(lo));
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// PyTorch weight [Cout][Cin][taps] (transposed=0) or [Cin][Cout][taps] (1) -> hi / lo, each
// [taps][Cout_pad][Cin_pad] (K-major), TF32-split.
int nrgbd_pack_conv_weight_tc(const float* w, int transposed, int Cout, int Cin, int taps, int Cin_pad, int Cout_pad,
                              float* hi, float* lo, cudaStream_t st) {
  NRGBD_REQUIRE(w && hi && lo && Cout > 0 && Cin > 0 && taps > 0 && Cin_pad >= Cin && Cout_pad >= Cout, "bad arguments");
  long long n = (long long)taps * Cin_pad * Cout_pad;
  pack_weight_tc_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w, transposed ? 1 : 0, Cout, Cin, taps, Cin_pad, Cout_pad, hi, lo);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Tensor-core counterpart of nrgbd_conv_nhwc: same semantics, inputs given as the TF32 hi / lo split
// of the activations and of the (K-major packed) weights. Requires nrgbd_conv_tc_supported().
int nrgbd_conv_nhwc_tc(const float* x_hi, const float* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in,
                       const float* w_hi, const float* w_lo, const float* bias, int Cout, int Cout_pad, int kd, int kh, int kw,
                       int stride, int pad, int dilation, float* y, int Hout, int Wout, int Cs_out, int c_off, int leaky,
                       double* stats, cudaStream_t st) {
  NRGBD_REQUIRE(x_hi && x_lo && w_hi && w_lo && y, "null pointer");
  NRGBD_REQUIRE(nrgbd_conv_tc_supported(Cin_pad, Cout_pad) && Cin_pad <= Cs_in && Cs_in % 4 == 0 && Cout <= Cout_pad,
                "channel counts not supported by the tensor-core path");
  int rc = wg_check_conv_shape(Hin, Win, kd, kh, kw, stride, pad, dilation, Hout, Wout);
  if (rc != NRGBD_OK) return rc;
  WgConv c = tf32_conv(x_hi, x_lo, N, Din, Hin, Win, Cin_pad, Cs_in, w_hi, w_lo, bias, Cout, Cout_pad, y, Cs_out, c_off, leaky, stats);
  wg_conv_taps(c, kd, kh, kw, stride, pad, dilation, Hout, Wout);
  rc = conv_wgmma(c, st);
  if (rc != NRGBD_OK) return rc;
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Tensor-core counterpart of nrgbd_conv_transpose2d_k4s2_nhwc (four parity-class launches).
int nrgbd_conv_transpose2d_k4s2_nhwc_tc(const float* x_hi, const float* x_lo, int N, int Hin, int Win, int Cin_pad, int Cs_in,
                                        const float* w_hi, const float* w_lo, const float* bias, int Cout, int Cout_pad, float* y,
                                        int Cs_out, int c_off, int leaky, cudaStream_t st) {
  NRGBD_REQUIRE(x_hi && x_lo && w_hi && w_lo && y, "null pointer");
  NRGBD_REQUIRE(nrgbd_conv_tc_supported(Cin_pad, Cout_pad) && Cin_pad <= Cs_in && Cs_in % 4 == 0 && Cout <= Cout_pad,
                "channel counts not supported by the tensor-core path");
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      WgConv c = tf32_conv(x_hi, x_lo, N, 1, Hin, Win, Cin_pad, Cs_in, w_hi, w_lo, bias, Cout, Cout_pad, y, Cs_out, c_off, leaky, nullptr);
      wg_transpose_k4s2_class(c, py, px);
      int rc = conv_wgmma(c, st);
      if (rc != NRGBD_OK) return rc;
    }
  NRGBD_COUNT(4);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
