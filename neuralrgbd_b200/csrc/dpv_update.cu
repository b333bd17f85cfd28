// Per-pixel reductions over the D depth planes (SURVEY §8 a4 tail, a9, a11):
//   log_softmax(+-x)                         models/basic.py:299-300, Refine.py:105
//   DPV = log_softmax(gain + prior)          models/KVNET.py:172-173   (Bayesian update)
//   depth = sum_d exp(BV_d) * d, conf = max  mutils/misc.py:532-548, test_utils/export_res.py:37-62
// One warp owns one pixel when the D values are contiguous (pixel-major engine layout); one
// thread owns one pixel when planes are strided (reference [D][h][w] layout, coalesced over x).
#include "common.cuh"

namespace {

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, s));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
  return v;
}

// y = log_softmax(sign * (a + b)) over D; optional expected depth / confidence.
// Strided variant: thread per pixel.
__global__ void __launch_bounds__(256)
dpv_rows_strided_kernel(const float* __restrict__ a, const float* __restrict__ b, float sign, int n_pix, int D,
                        long long sd, long long sp, long long bsd, long long bsp, float* __restrict__ y,
                        long long ysd, long long ysp,
                        const float* __restrict__ dpl, float* __restrict__ depth, float* __restrict__ conf) {
  int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= n_pix) return;
  const float* pa = a + (long long)pix * sp;
  const float* pb = b ? b + (long long)pix * bsp : nullptr;
  float m = -INFINITY;
  for (int d = 0; d < D; ++d) {
    float v = pa[d * sd]; if (pb) v = __fadd_rn(v, pb[d * bsd]); v *= sign;
    m = fmaxf(m, v);
  }
  float s = 0.f;
  for (int d = 0; d < D; ++d) {
    float v = pa[d * sd]; if (pb) v = __fadd_rn(v, pb[d * bsd]); v *= sign;
    s += expf(v - m);
  }
  const float ls = logf(s);
  float dep = 0.f, cf = 0.f;
  for (int d = 0; d < D; ++d) {
    float v = pa[d * sd]; if (pb) v = __fadd_rn(v, pb[d * bsd]); v *= sign;
    float o = (v - m) - ls;
    if (y) y[(long long)d * ysd + (long long)pix * ysp] = o;
    if (dpl) { float p = expf(o); dep = __fadd_rn(dep, __fmul_rn(p, dpl[d])); cf = fmaxf(cf, p); }
  }
  if (depth) depth[pix] = dep;
  if (conf) conf[pix] = cf;
}

// Contiguous variant: warp per pixel, D values consecutive in memory; each lane keeps its D/32 values
// in registers (one read of the row, one write).
template <int PER>      // values per lane: D <= 32 * PER
__global__ void __launch_bounds__(256)
dpv_rows_contig_kernel(const float* __restrict__ a, const float* __restrict__ b, float sign, int n_pix, int D,
                       float* __restrict__ y, long long ysd, long long ysp, const float* __restrict__ dpl,
                       float* __restrict__ depth, float* __restrict__ conf) {
  const int lane = threadIdx.x & 31;
  const int pix = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (pix >= n_pix) return;
  const float* pa = a + (long long)pix * D;
  const float* pb = b ? b + (long long)pix * D : nullptr;
  float v[PER];
  float m = -INFINITY;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int d = lane + 32 * k;
    float t = -INFINITY;
    if (d < D) { t = pa[d]; if (pb) t = __fadd_rn(t, pb[d]); t *= sign; }
    v[k] = t;
    m = fmaxf(m, t);
  }
  m = warp_max(m);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < PER; ++k) if (lane + 32 * k < D) s += expf(v[k] - m);
  s = warp_sum(s);
  const float ls = logf(s);
  float dep = 0.f, cf = 0.f;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int d = lane + 32 * k;
    if (d < D) {
      float o = (v[k] - m) - ls;
      if (y) y[(long long)d * ysd + (long long)pix * ysp] = o;
      if (dpl) { float p = expf(o); dep += p * dpl[d]; cf = fmaxf(cf, p); }
    }
  }
  if (dpl) {
    dep = warp_sum(dep); cf = warp_max(cf);
    if (lane == 0) { if (depth) depth[pix] = dep; if (conf) conf[pix] = cf; }
  }
}

// depth[pix] = sum_d (bv_log ? exp(bv) : bv) * d, sequential over d like the reference's
// Python loop (mutils/misc.py:541-546); conf[pix] = max_d of the same probability.
__global__ void __launch_bounds__(256)
depth_regression_kernel(const float* __restrict__ bv, int n_pix, int D, long long sd, long long sp,
                        const float* __restrict__ dpl, int bv_log, float* __restrict__ depth,
                        float* __restrict__ conf) {
  int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= n_pix) return;
  const float* p = bv + (long long)pix * sp;
  float dep = 0.f, cf = -INFINITY;
  for (int d = 0; d < D; ++d) {
    float v = p[d * sd];
    float pr = bv_log ? expf(v) : v;
    dep = __fadd_rn(dep, __fmul_rn(pr, dpl[d]));
    cf = fmaxf(cf, pr);
  }
  if (depth) depth[pix] = dep;
  if (conf) conf[pix] = cf;
}

// Backward of depth_regression_kernel's depth for one slice: autograd through the reference's
// depth + exp(BV[0, d]) * d (mutils/misc.py:541-546) gives g_bv(d, pix) = (g[pix] * d) * exp(bv), or g[pix] * d without
// the exp. Thread per (plane, pixel) with pixels fastest for the [D][hw] layout, planes fastest for the pixel-major one.
__global__ void __launch_bounds__(256)
depth_regression_backward_kernel(const float* __restrict__ g, const float* __restrict__ bv, int n_pix, int D, long long sd,
                                 long long sp, const float* __restrict__ dpl, int bv_log, int pixel_major,
                                 float* __restrict__ g_bv) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n_pix * D) return;
  int pix, d;
  if (pixel_major) { d = (int)(idx % D); pix = (int)(idx / D); }
  else { pix = (int)(idx % n_pix); d = (int)(idx / n_pix); }
  const long long o = (long long)d * sd + (long long)pix * sp;
  const float gd = __fmul_rn(__ldg(g + pix), __ldg(dpl + d));
  g_bv[o] = bv_log ? __fmul_rn(gd, expf(__ldg(bv + o))) : gd;
}

__global__ void exp_kernel(const float* __restrict__ x, long long n, float* __restrict__ y) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = expf(x[i]);
}

}  // namespace

extern "C" {

// out(d,pix) = log_softmax_d( sign * (a(d,pix) + b(d,pix)) ); b may be null.
// a element (d,pix) at d*in_sd + pix*in_sp; b at d*b_sd + pix*b_sp; out at d*out_sd + pix*out_sp. When d_planes is
// given also writes depth[pix] = sum_d exp(out)*d_planes[d] and conf[pix] = max_d exp(out)
// (either may be null). out may be null when only depth/conf are wanted.
int nrgbd_dpv_normalize(const float* a, long long in_sd, long long in_sp, const float* b, long long b_sd,
                        long long b_sp, float sign, int n_pix, int D, float* out, long long out_sd, long long out_sp,
                        const float* d_planes, float* depth, float* conf, cudaStream_t st) {
  NRGBD_REQUIRE(a && n_pix > 0 && D > 0, "bad arguments");
  NRGBD_REQUIRE(out || (d_planes && (depth || conf)), "nothing to compute");
  if (in_sd == 1 && in_sp == D && (!b || (b_sd == 1 && b_sp == D)) && D <= 256) {
    const unsigned grid = (unsigned)ceil_div((long long)n_pix * 32, 256);
    if (D <= 64) dpv_rows_contig_kernel<2><<<grid, 256, 0, st>>>(a, b, sign, n_pix, D, out, out_sd, out_sp, d_planes, depth, conf);
    else if (D <= 128) dpv_rows_contig_kernel<4><<<grid, 256, 0, st>>>(a, b, sign, n_pix, D, out, out_sd, out_sp, d_planes, depth, conf);
    else dpv_rows_contig_kernel<8><<<grid, 256, 0, st>>>(a, b, sign, n_pix, D, out, out_sd, out_sp, d_planes, depth, conf);
  } else {
    dpv_rows_strided_kernel<<<ceil_div(n_pix, 256), 256, 0, st>>>(a, b, sign, n_pix, D, in_sd, in_sp, b_sd, b_sp, out,
                                                                  out_sd, out_sp, d_planes, depth, conf);
  }
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_depth_regression(const float* bv, int n_pix, int D, long long in_sd, long long in_sp,
                           const float* d_planes, int bv_log, float* depth, float* conf, cudaStream_t st) {
  NRGBD_REQUIRE(bv && d_planes && (depth || conf) && n_pix > 0 && D > 0, "bad arguments");
  depth_regression_kernel<<<ceil_div(n_pix, 256), 256, 0, st>>>(bv, n_pix, D, in_sd, in_sp, d_planes, bv_log, depth,
                                                                conf);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_depth_regression_backward(const float* grad_depth, const float* bv, int n_pix, int D, long long in_sd,
                                    long long in_sp, const float* d_planes, int bv_log, float* g_bv, cudaStream_t st) {
  NRGBD_REQUIRE(grad_depth && d_planes && g_bv && (bv || !bv_log) && n_pix > 0 && D > 0, "bad arguments");
  const long long n = (long long)n_pix * D;
  depth_regression_backward_kernel<<<ceil_div(n, 256), 256, 0, st>>>(grad_depth, bv, n_pix, D, in_sd, in_sp, d_planes,
                                                                     bv_log, in_sd == 1 ? 1 : 0, g_bv);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_exp(const float* x, long long n, float* y, cudaStream_t st) {
  NRGBD_REQUIRE(x && y && n > 0, "bad arguments");
  exp_kernel<<<ceil_div(n, 256), 256, 0, st>>>(x, n, y);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
