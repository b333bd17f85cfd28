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

// Depth variance of one slice, sequential over d like the reference's loop (mutils/misc.py:566-572):
//   acc = acc + ((p_d * d - mean)^2) / div,  var = acc / D,  p_d = exp(bv) or bv.
// `div` is 2*d_sigma^2 rounded to fp32, as ATen rounds a Python scalar; every operation is rounded on its own (no FMA),
// and the final scaling is a division by D (`depth_var * 1. / D`), not a multiplication by 1/D.
__global__ void __launch_bounds__(256)
depth_var_kernel(const float* __restrict__ bv, int n_pix, int D, long long sd, long long sp,
                 const float* __restrict__ dpl, int bv_log, const float* __restrict__ mean, float div,
                 float* __restrict__ var) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= n_pix) return;
  const float* p = bv + (long long)pix * sp;
  const float mu = mean[pix];
  float acc = 0.f;
  for (int d = 0; d < D; ++d) {
    const float v = p[d * sd];
    const float x = __fsub_rn(__fmul_rn(bv_log ? expf(v) : v, dpl[d]), mu);
    acc = __fadd_rn(acc, __fdiv_rn(__fmul_rn(x, x), div));
  }
  var[pix] = __fdiv_rn(acc, (float)D);
}

// Backward of depth_var_kernel in autograd's order through misc.py:566-572: g_sq = (g / D) / div; per plane
// g_x = g_sq * (2x) (pow), g_bv = (g_x * d) * exp(bv) (mul by the scalar d, then exp times its result), and
// g_mean = -sum_d g_x summed from the last plane to the first, the order in which autograd's engine delivers the D
// contributions. Thread per pixel, no atomics; either output may be null.
__global__ void __launch_bounds__(256)
depth_var_backward_kernel(const float* __restrict__ g, const float* __restrict__ bv, int n_pix, int D, long long sd,
                          long long sp, const float* __restrict__ dpl, int bv_log, const float* __restrict__ mean,
                          float div, float* __restrict__ g_bv, float* __restrict__ g_mean) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= n_pix) return;
  const long long o = (long long)pix * sp;
  const float mu = mean[pix];
  const float gsq = __fdiv_rn(__fdiv_rn(g[pix], (float)D), div);
  float gm = 0.f;
  for (int d = D - 1; d >= 0; --d) {
    const float v = bv[o + d * sd];
    const float pr = bv_log ? expf(v) : v;
    const float x = __fsub_rn(__fmul_rn(pr, dpl[d]), mu);
    const float gx = __fmul_rn(gsq, __fmul_rn(2.f, x));
    gm = __fsub_rn(gm, gx);
    if (g_bv) {
      const float gp = __fmul_rn(gx, dpl[d]);
      g_bv[o + d * sd] = bv_log ? __fmul_rn(gp, pr) : gp;
    }
  }
  if (g_mean) g_mean[pix] = gm;
}

// Max (or min) over d of p_d = exp(bv) or bv, for every (slice, pixel), with the index ATen's CPU max.dim / min.dim
// return: ties keep the first plane, and the first NaN wins.
__global__ void __launch_bounds__(256)
dpv_extreme_kernel(const float* __restrict__ bv, int n_pix, int n_slices, int D, long long sn, long long sd,
                   long long sp, int bv_log, int is_min, float* __restrict__ value, int* __restrict__ index) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n_pix * n_slices) return;
  const int n = (int)(t / n_pix), pix = (int)(t % n_pix);
  const float* p = bv + n * sn + (long long)pix * sp;
  float best = bv_log ? expf(p[0]) : p[0];
  int arg = 0;
  for (int d = 0; d < D; ++d) {
    const float v = bv_log ? expf(p[d * sd]) : p[d * sd];
    if (is_min ? !(v >= best) : !(v <= best)) {
      best = v; arg = d;
      if (v != v) break;
    }
  }
  value[t] = best;
  if (index) index[t] = arg;
}

// Backward of dpv_extreme_kernel's value: g * exp(bv) (g without bv_log) at the stored plane, zero at every other one.
// Thread per (slice, plane, pixel), pixels fastest.
__global__ void __launch_bounds__(256)
dpv_extreme_backward_kernel(const float* __restrict__ g, const float* __restrict__ bv, const int* __restrict__ index,
                            int n_pix, int n_slices, int D, long long sn, long long sd, long long sp, int bv_log,
                            float* __restrict__ g_bv) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n_pix * D * n_slices) return;
  const int pix = (int)(t % n_pix);
  const long long r = t / n_pix;
  const int d = (int)(r % D), n = (int)(r / D);
  const long long o = n * sn + (long long)d * sd + (long long)pix * sp;
  const long long q = (long long)n * n_pix + pix;
  float out = 0.f;
  if (__ldg(index + q) == d) {
    const float gv = __ldg(g + q);
    out = bv_log ? __fmul_rn(gv, expf(__ldg(bv + o))) : gv;
  }
  g_bv[o] = out;
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

int nrgbd_depth_var(const float* bv, int n_pix, int D, long long in_sd, long long in_sp, const float* d_planes,
                    int bv_log, const float* mean, float var_div, float* var, cudaStream_t st) {
  NRGBD_REQUIRE(bv && d_planes && mean && var && n_pix > 0 && D > 0, "bad arguments");
  depth_var_kernel<<<ceil_div(n_pix, 256), 256, 0, st>>>(bv, n_pix, D, in_sd, in_sp, d_planes, bv_log, mean, var_div, var);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_depth_var_backward(const float* grad_var, const float* bv, int n_pix, int D, long long in_sd, long long in_sp,
                             const float* d_planes, int bv_log, const float* mean, float var_div, float* g_bv,
                             float* g_mean, cudaStream_t st) {
  NRGBD_REQUIRE(grad_var && bv && d_planes && mean && (g_bv || g_mean) && n_pix > 0 && D > 0, "bad arguments");
  depth_var_backward_kernel<<<ceil_div(n_pix, 256), 256, 0, st>>>(grad_var, bv, n_pix, D, in_sd, in_sp, d_planes, bv_log,
                                                                  mean, var_div, g_bv, g_mean);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_dpv_extreme(const float* bv, int n_pix, int n_slices, int D, long long in_sn, long long in_sd, long long in_sp,
                      int bv_log, int is_min, float* value, int* index, cudaStream_t st) {
  NRGBD_REQUIRE(bv && value && n_pix > 0 && n_slices > 0 && D > 0, "bad arguments");
  dpv_extreme_kernel<<<ceil_div((long long)n_pix * n_slices, 256), 256, 0, st>>>(bv, n_pix, n_slices, D, in_sn, in_sd,
                                                                                 in_sp, bv_log, is_min, value, index);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_dpv_extreme_backward(const float* grad_value, const float* bv, const int* index, int n_pix, int n_slices, int D,
                               long long in_sn, long long in_sd, long long in_sp, int bv_log, float* g_bv,
                               cudaStream_t st) {
  NRGBD_REQUIRE(grad_value && index && g_bv && (bv || !bv_log) && n_pix > 0 && n_slices > 0 && D > 0, "bad arguments");
  const long long n = (long long)n_pix * D * n_slices;
  dpv_extreme_backward_kernel<<<ceil_div(n, 256), 256, 0, st>>>(grad_value, bv, index, n_pix, n_slices, D, in_sn, in_sd,
                                                               in_sp, bv_log, g_bv);
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
