// Tensor-core convolution with error-compensated 3xTF32 products (SURVEY §8 a5, a8, a10; DESIGN.md §4.2):
// the `conv_math = 'tf32x3'` path. The GEMM is the wgmma kernel of conv_f16.cu (conv_wgmma) on TF32 operand pairs.
//
// Why 3xTF32: the reference's results must be matched to 1e-4 on the DPV through 61 (2-D) / 12 (3-D)
// convolutions separated by batch-statistics BatchNorm; single-pass TF32 operands give 1e-2-level
// DPV errors (SURVEY §7). Each fp32 operand is split a = a_hi + a_lo with a_hi = RN_tf32(a),
// a_lo = RN_tf32(a - a_hi) and the product is accumulated as a_hi*b_hi + a_lo*b_hi + a_hi*b_lo in
// fp32 (dropped term <= 2^-22 |a b|).
//
// Two forms of the entry points:
//   nrgbd_conv_nhwc_tc*   the activations arrive pre-split (nrgbd_split_tf32);
//   nrgbd_conv_nhwc_tc2*  raw fp32 activations (optionally the RAW output of the producing convolution, normalised here
//                         with its batch statistics: *_bn_in); the split (and the BatchNorm + ReLU) runs as one pass into
//                         stream-ordered scratch memory right before the GEMM: 4 B read + 8 B written per element, the
//                         same traffic as nrgbd_split_tf32. The *_bn_in form is what saves a pass: it replaces the separate
//                         BatchNorm pass (4 B read + 4 B written) in front of that split.
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

// x -> hi = RN_tf32(x), lo = RN_tf32(x - hi)
__global__ void __launch_bounds__(256)
split_tf32_kernel(const float4* __restrict__ x, long long n4, float4* __restrict__ hi, float4* __restrict__ lo) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 v = x[i];
  float a[4] = {v.x, v.y, v.z, v.w}, h[4], l[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    h[k] = rn_tf32(a[k]);
    l[k] = rn_tf32(a[k] - h[k]);
  }
  hi[i] = make_float4(h[0], h[1], h[2], h[3]);
  lo[i] = make_float4(l[0], l[1], l[2], l[3]);
}

// channels-last x [pos][Cs] -> TF32 pair [pos][Cin_pad] of [relu](x * scale + shift) (scale == null: x itself); channels
// >= C are zero
__global__ void __launch_bounds__(256)
split_tf32_bn_kernel(const float* __restrict__ x, long long n_pos, int Cs, int Cin_pad, int C, const float* __restrict__ scale,
                     const float* __restrict__ shift, int relu, float* __restrict__ hi, float* __restrict__ lo) {
  const long long n = n_pos * Cin_pad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long pos = i / Cin_pad;
    const int c = (int)(i - pos * Cin_pad);
    float v = 0.f;
    if (c < C) {
      v = x[pos * Cs + c];
      if (scale) {
        v = fmaf(v, scale[c], shift[c]);
        if (relu) v = fmaxf(v, 0.f);
      }
    }
    const float h = rn_tf32(v);
    hi[i] = h;
    lo[i] = rn_tf32(v - h);
  }
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

WgConv tf32_conv(const float* x_hi, const float* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                 const float* w_lo, int n_wslices, const float* bias, int Cout, int Cout_pad, float* y, int Cs_out, int c_off, int leaky,
                 double* stats) {
  WgConv c{};
  c.tf32 = 1;
  c.x_hi = x_hi; c.x_lo = x_lo; c.N = N; c.Din = Din; c.Hin = Hin; c.Win = Win; c.Cin_pad = Cin_pad; c.Cs_in = Cs_in;
  c.w_hi = w_hi; c.w_lo = w_lo; c.w_tap_stride = (long long)Cout_pad * Cin_pad; c.n_wslices = n_wslices; c.Cout_pad = Cout_pad;
  c.bias = bias; c.stats = stats; c.y = y;
  c.Cout = Cout; c.Cs_out = Cs_out; c.c_off = c_off; c.leaky = leaky;
  return c;
}

int conv_tc_impl(const float* x_hi, const float* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                 const float* w_lo, const float* bias, int Cout, int Cout_pad, int kd, int kh, int kw, int stride, int pad, int dilation,
                 float* y, int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats, cudaStream_t st) {
  WgConv c = tf32_conv(x_hi, x_lo, N, Din, Hin, Win, Cin_pad, Cs_in, w_hi, w_lo, kd * kh * kw, bias, Cout, Cout_pad, y, Cs_out, c_off, leaky, stats);
  c.Dout = Din; c.Hout = Hout; c.Wout = Wout; c.out_stride = 1;
  c.Hy = Hout; c.Wx = Wout; c.in_stride = stride; c.n_kz = kd; c.n_tap = kh * kw;
  for (int a = 0; a < kd; ++a) c.dz[a] = (signed char)(a - kd / 2);
  int t = 0;
  for (int b = 0; b < kh; ++b)
    for (int e = 0; e < kw; ++e) { c.dy[t] = (signed char)(b * dilation - pad); c.dx[t] = (signed char)(e * dilation - pad); ++t; }
  for (int a = 0; a < kd * kh * kw; ++a) c.wsel[a] = (unsigned char)a;
  return conv_wgmma(c, st);
}

// nn.ConvTranspose2d(kernel 4, stride 2, padding 1) as four output-parity classes of 2x2-tap convolutions
int conv_transpose_tc_impl(const float* x_hi, const float* x_lo, int N, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                           const float* w_lo, const float* bias, int Cout, int Cout_pad, float* y, int Cs_out, int c_off, int leaky,
                           cudaStream_t st) {
  const int kys[2][2] = {{1, 3}, {0, 2}};
  const int dys[2][2] = {{0, -1}, {1, 0}};
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      WgConv c = tf32_conv(x_hi, x_lo, N, 1, Hin, Win, Cin_pad, Cs_in, w_hi, w_lo, 16, bias, Cout, Cout_pad, y, Cs_out, c_off, leaky, nullptr);
      c.Dout = 1; c.Hout = 2 * Hin; c.Wout = 2 * Win; c.out_stride = 2; c.out_off_y = py; c.out_off_x = px;
      c.Hy = Hin; c.Wx = Win; c.in_stride = 1; c.n_kz = 1; c.n_tap = 4;
      int t = 0;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          c.dy[t] = (signed char)dys[py][a]; c.dx[t] = (signed char)dys[px][b];
          c.wsel[t] = (unsigned char)(kys[py][a] * 4 + kys[px][b]); ++t;
        }
      int rc = conv_wgmma(c, st);
      if (rc != NRGBD_OK) return rc;
    }
  return NRGBD_OK;
}

// Stream-ordered scratch for the split of raw activations: TF32 pair [n_pos][Cin_pad] (+ scale / shift of a fused input
// BatchNorm), freed on the same stream after the GEMM.
struct SplitScratch {
  float *hi = nullptr, *lo = nullptr, *scale = nullptr, *shift = nullptr;
  void* mem = nullptr;
};

int split_raw(const float* x, long long n_pos, int Cs_in, int Cin_pad, const nrgbd_bn_input* in_bn, SplitScratch& s, cudaStream_t st) {
  const long long n = n_pos * Cin_pad;
  const size_t bytes = (size_t)n * 8 + (in_bn ? (size_t)Cin_pad * 8 : 0);
  NRGBD_CUDA_CHECK(cudaMallocAsync(&s.mem, bytes, st));
  s.hi = reinterpret_cast<float*>(s.mem); s.lo = s.hi + n;
  int C = Cin_pad, relu = 0;
  if (in_bn) {
    s.scale = s.lo + n; s.shift = s.scale + Cin_pad;
    C = in_bn->C; relu = in_bn->relu;
    const bool run = in_bn->running_mean && in_bn->running_var;
    int rc = nrgbd_bn_finalize(in_bn->stats, C, in_bn->count, in_bn->gamma, in_bn->beta, in_bn->eps, s.scale, s.shift,
                               run ? in_bn->running_mean : nullptr, run ? in_bn->running_var : nullptr, in_bn->momentum, st);
    if (rc != NRGBD_OK) return rc;
  }
  long long blocks = (n + 255) / 256;
  if (blocks > nrgbd_sm_count() * 16ll) blocks = nrgbd_sm_count() * 16ll;
  split_tf32_bn_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, n_pos, Cs_in, Cin_pad, C, s.scale, s.shift, relu, s.hi, s.lo);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // namespace

extern "C" {

// Whether the tensor-core path can run a convolution with these channel counts.
int nrgbd_conv_tc_supported(int Cin_pad, int Cout_pad) {
  return (Cin_pad % 32 == 0 && Cin_pad >= 32 && Cout_pad % 16 == 0 && Cout_pad >= 16 && Cout_pad <= 256) ? 1 : 0;
}

int nrgbd_split_tf32(const float* x, long long n, float* hi, float* lo, cudaStream_t st) {
  NRGBD_REQUIRE(x && hi && lo && n > 0 && n % 4 == 0, "bad arguments");
  split_tf32_kernel<<<ceil_div(n / 4, 256), 256, 0, st>>>(reinterpret_cast<const float4*>(x), n / 4, reinterpret_cast<float4*>(hi),
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
  NRGBD_REQUIRE(kd >= 1 && kd <= 3 && kh * kw <= WG_MAX_TAP2D && stride >= 1 && stride <= 8, "unsupported filter");
  NRGBD_REQUIRE(Hout == (Hin + 2 * pad - dilation * (kh - 1) - 1) / stride + 1 &&
                    Wout == (Win + 2 * pad - dilation * (kw - 1) - 1) / stride + 1, "output extent mismatch");
  int rc = conv_tc_impl(x_hi, x_lo, N, Din, Hin, Win, Cin_pad, Cs_in, w_hi, w_lo, bias, Cout, Cout_pad, kd, kh, kw, stride, pad, dilation, y,
                        Hout, Wout, Cs_out, c_off, leaky, stats, st);
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
  int rc = conv_transpose_tc_impl(x_hi, x_lo, N, Hin, Win, Cin_pad, Cs_in, w_hi, w_lo, bias, Cout, Cout_pad, y, Cs_out, c_off, leaky, st);
  if (rc != NRGBD_OK) return rc;
  NRGBD_COUNT(4);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Raw fp32 activations, TF32-split K-major weights. Cout_pad <= 128.
int nrgbd_conv_tc2_supported(int Cin_pad, int Cout_pad) {
  return (Cin_pad % 32 == 0 && Cin_pad >= 32 && Cout_pad % 16 == 0 && Cout_pad >= 16 && Cout_pad <= 128) ? 1 : 0;
}

static int conv_nhwc_tc2_impl(const float* x, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                              const float* w_lo, const float* bias, int Cout, int Cout_pad, int kd, int kh, int kw, int stride, int pad,
                              int dilation, float* y, int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats,
                              const nrgbd_bn_input* in_bn, cudaStream_t st) {
  NRGBD_REQUIRE(x && w_hi && w_lo && y, "null pointer");
  NRGBD_REQUIRE(nrgbd_conv_tc2_supported(Cin_pad, Cout_pad) && Cin_pad <= Cs_in && Cs_in % 4 == 0 && Cout <= Cout_pad,
                "channel counts not supported by the tensor-core path");
  NRGBD_REQUIRE(kd >= 1 && kd <= 3 && kh * kw <= WG_MAX_TAP2D && stride >= 1 && stride <= 8, "unsupported filter");
  NRGBD_REQUIRE(Hout == (Hin + 2 * pad - dilation * (kh - 1) - 1) / stride + 1 &&
                    Wout == (Win + 2 * pad - dilation * (kw - 1) - 1) / stride + 1, "output extent mismatch");
  if (in_bn) {
    NRGBD_REQUIRE(in_bn->stats && in_bn->gamma && in_bn->beta && in_bn->C >= 1 && in_bn->C <= Cin_pad && in_bn->count >= 1 &&
                      in_bn->stats != stats, "bad input BatchNorm descriptor");
  }
  SplitScratch s;
  int rc = split_raw(x, (long long)N * Din * Hin * Win, Cs_in, Cin_pad, in_bn, s, st);
  if (rc == NRGBD_OK)
    rc = conv_tc_impl(s.hi, s.lo, N, Din, Hin, Win, Cin_pad, Cin_pad, w_hi, w_lo, bias, Cout, Cout_pad, kd, kh, kw, stride, pad, dilation, y, Hout,
                      Wout, Cs_out, c_off, leaky, stats, st);
  if (s.mem) NRGBD_CUDA_CHECK(cudaFreeAsync(s.mem, st));
  if (rc != NRGBD_OK) return rc;
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_conv_nhwc_tc2(const float* x, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                        const float* w_lo, const float* bias, int Cout, int Cout_pad, int kd, int kh, int kw, int stride, int pad,
                        int dilation, float* y, int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats, cudaStream_t st) {
  return conv_nhwc_tc2_impl(x, N, Din, Hin, Win, Cin_pad, Cs_in, w_hi, w_lo, bias, Cout, Cout_pad, kd, kh, kw, stride, pad, dilation, y,
                            Hout, Wout, Cs_out, c_off, leaky, stats, nullptr, st);
}

// Same convolution of [relu](BatchNorm_train(x)) where x is the RAW output of the producing conv and in_bn carries its
// per-channel sums: the normalisation is applied in the operand split (no separate pass over x).
int nrgbd_conv_nhwc_tc2_bn_in(const float* x, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                              const float* w_lo, const float* bias, int Cout, int Cout_pad, int kd, int kh, int kw, int stride, int pad,
                              int dilation, float* y, int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats,
                              const nrgbd_bn_input* in_bn, cudaStream_t st) {
  NRGBD_REQUIRE(in_bn, "null input BatchNorm descriptor");
  return conv_nhwc_tc2_impl(x, N, Din, Hin, Win, Cin_pad, Cs_in, w_hi, w_lo, bias, Cout, Cout_pad, kd, kh, kw, stride, pad, dilation, y,
                            Hout, Wout, Cs_out, c_off, leaky, stats, in_bn, st);
}

int nrgbd_conv_transpose2d_k4s2_nhwc_tc2(const float* x, int N, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                                         const float* w_lo, const float* bias, int Cout, int Cout_pad, float* y, int Cs_out,
                                         int c_off, int leaky, cudaStream_t st) {
  NRGBD_REQUIRE(x && w_hi && w_lo && y, "null pointer");
  NRGBD_REQUIRE(nrgbd_conv_tc2_supported(Cin_pad, Cout_pad) && Cin_pad <= Cs_in && Cs_in % 4 == 0 && Cout <= Cout_pad,
                "channel counts not supported by the tensor-core path");
  SplitScratch s;
  int rc = split_raw(x, (long long)N * Hin * Win, Cs_in, Cin_pad, nullptr, s, st);
  if (rc == NRGBD_OK)
    rc = conv_transpose_tc_impl(s.hi, s.lo, N, Hin, Win, Cin_pad, Cin_pad, w_hi, w_lo, bias, Cout, Cout_pad, y, Cs_out, c_off, leaky, st);
  if (s.mem) NRGBD_CUDA_CHECK(cudaFreeAsync(s.mem, st));
  if (rc != NRGBD_OK) return rc;
  NRGBD_COUNT(4);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
