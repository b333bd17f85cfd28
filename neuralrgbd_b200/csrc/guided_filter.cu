// Guided filter: GuidedFilter(r, eps) (models/GF/guided_filter.py) and its BoxFilter (models/GF/box_filter.py) on
// N x C x H x W planes, forward and backward (the autograd mirrors in neuralrgbd_b200/models/GF), and the depth refinement
// of KVNET(refineNet_name='DGF'), RefineNet_DGF.forward (models/Refine.py:620-641), which runs the same forward on one plane:
//
//   y = F.upsample(dmap, scale_factor=H/h, mode='bilinear', align_corners=True)
//   x = Conv2d(64 -> 1, 1x1)(ReLU(Conv2d(3 -> 64, 1x1)(img)))
//   A = cov_xy / (var_x + eps), b = mean_y - A * mean_x; out = box(A)/N * x + box(b)/N
//
// The box filter is the reference's cumulative-sum form, cumsum(H) -> diff_x -> cumsum(W) -> diff_y, not a window sum:
// ATen's float32 cumsum accumulates in double and rounds every prefix to fp32, and the differences of those rounded prefixes
// (which reach 1e3-1e4 for x*y) are what the reference filters with. A = cov / (var + 1e-8) amplifies any change to them
// wherever the guide is locally flat, so a more accurate window sum would not reproduce the reference. Every other step is
// one IEEE-rounded fp32 operation in the reference's order (no contraction), the bilinear taps and the 1x1 convolutions
// in the FMA order of ATen's CPU kernels. No atomics: the output is identical from run to run.
//
// Parallel scans. A column pass (lines along H) gives a block 32 adjacent columns of one plane and cuts each column into
// GF_COL_SEG segments, one per threadIdx.y: loads stay coalesced across the 32 columns. A row pass (lines along W) gives
// each row a warp and each lane a contiguous segment. Every thread sums its segment in double, the segment totals are
// scanned in double (shared memory across threadIdx.y, shuffles across lanes), and the thread re-walks its segment from
// that offset, rounding each prefix to fp32. Only the double sums are reassociated; the fp32 prefixes are those of the
// sequential double accumulation unless a reassociated double lands on the other side of an fp32 rounding boundary.
//
// Forward pass (ADJ = false): prefix sums cs (ATen's cumsum), then box_diff into dst. dst may be the source plane.
// Adjoint pass (ADJ = true), autograd's order through box_filter.py: first the adjoint of box_diff (the slice / cat
// backward: d cs[i] = g[i - r] - g[i + r + 1], and at i = n-1 the broadcast `right` slice's sum g[n-r..n-1] added to
// g[n-1-r]), then cumsum's backward, a reverse prefix sum in double rounded per position. dst must not be the source.
#include "../../include/nrgbd.h"
#include "common.cuh"

namespace {

constexpr int GF_HID = 64;      // RefineNet_DGF.feature_ext: Conv2d(3, 64, 1) -> ReLU -> Conv2d(64, 1, 1)

// planes [x | y], each [H][W]: the 1x1 MLP of the guide image and the upsampled depth
__global__ void __launch_bounds__(256)
gf_prep_kernel(const float* __restrict__ dmap, int h, int w, const float* __restrict__ img, long long img_sc, long long img_sp,
               int H, int W, float sy, float sx, const float* __restrict__ w0, const float* __restrict__ b0,
               const float* __restrict__ w1, const float* __restrict__ b1, float* __restrict__ planes) {
  __shared__ float s_w0[GF_HID * 3], s_b0[GF_HID], s_w1[GF_HID];
  for (int i = threadIdx.x; i < GF_HID * 3; i += blockDim.x) s_w0[i] = w0[i];
  for (int i = threadIdx.x; i < GF_HID; i += blockDim.x) { s_b0[i] = b0[i]; s_w1[i] = w1[i]; }
  __syncthreads();
  const long long HW = (long long)H * W;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const int oy = (int)(p / W), ox = (int)(p % W);
  // ATen upsample_bilinear2d, align_corners=True: source index scale * dst in fp32, lambda clamped to [0, 1]
  const float fy = __fmul_rn(sy, (float)oy), fx = __fmul_rn(sx, (float)ox);
  const int y0 = min((int)floorf(fy), h - 1), x0 = min((int)floorf(fx), w - 1);
  const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
  const float ly = fminf(fmaxf(__fsub_rn(fy, (float)y0), 0.f), 1.f), lx = fminf(fmaxf(__fsub_rn(fx, (float)x0), 0.f), 1.f);
  const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  const float v00 = dmap[y0 * w + x0], v01 = dmap[y0 * w + x1], v10 = dmap[y1 * w + x0], v11 = dmap[y1 * w + x1];
  const float t0 = __fmaf_rn(hx, v00, __fmul_rn(lx, v01));
  const float t1 = __fmaf_rn(hx, v10, __fmul_rn(lx, v11));
  const float yv = __fmaf_rn(hy, t0, __fmul_rn(ly, t1));
  // 1x1 convolutions: accumulator starts at the bias, one FMA per input channel in channel order
  const float r = img[p * img_sp], g = img[p * img_sp + img_sc], bl = img[p * img_sp + 2 * img_sc];
  float xv = b1[0];
#pragma unroll 8
  for (int k = 0; k < GF_HID; ++k) {
    float a = __fmaf_rn(s_w0[3 * k], r, s_b0[k]);
    a = __fmaf_rn(s_w0[3 * k + 1], g, a);
    a = __fmaf_rn(s_w0[3 * k + 2], bl, a);
    xv = __fmaf_rn(s_w1[k], fmaxf(a, 0.f), xv);
  }
  planes[p] = xv;
  planes[HW + p] = yv;
}

// box_filter.py's diff_x / diff_y of the rounded prefix sums cs of one line of length n (element i at cs[i * step]):
// cat(left, middle, right) is out[i] = cs[min(i + r, n - 1)] - (i > r ? cs[i - r - 1] : 0), for n >= 2r + 1.
__device__ __forceinline__ float box_diff(const float* cs, long long step, int i, int n, int r) {
  const float hi = cs[min(i + r, n - 1) * step];
  return i > r ? __fsub_rn(hi, cs[(i - r - 1) * step]) : hi;
}

// N of guided_filter.py: the box filter of ones, i.e. the number of pixels of the (2r+1)^2 window inside the image
__device__ __forceinline__ float box_count(int i, int j, int H, int W, int r) {
  return (float)((min(i + r, H - 1) - max(i - r, 0) + 1) * (min(j + r, W - 1) - max(j - r, 0) + 1));
}

// guided_filter.py:79-91 at one pixel, from the box sums of x, y, x*y, x*x and the window count N:
// mean_x, mean_y, cov_xy, var_x (+ eps), A, b, each one fp32 operation in the reference's order
struct GfCoef {
  float mx, my, cov, ve, A, b;
  __device__ __forceinline__ GfCoef(float bx, float by, float bxy, float bxx, float N, float eps) {
    mx = __fdiv_rn(bx, N);
    my = __fdiv_rn(by, N);
    cov = __fsub_rn(__fdiv_rn(bxy, N), __fmul_rn(mx, my));
    ve = __fadd_rn(__fsub_rn(__fdiv_rn(bxx, N), __fmul_rn(mx, mx)), eps);
    A = __fdiv_rn(cov, ve);
    b = __fsub_rn(my, __fmul_rn(A, mx));
  }
};

// guided_filter.py:94-97: mean_A * x + mean_b
__device__ __forceinline__ float gf_out(float bA, float bb, float x, float N) {
  return __fadd_rn(__fmul_rn(__fdiv_rn(bA, N), x), __fdiv_rn(bb, N));
}

constexpr int GF_COL_SEG = 16;   // column pass: 32 columns x 16 segments per block
constexpr int GF_ROW_WARPS = 4;  // row pass: one warp per row, 4 rows per block

// Sources: bind(q) gives the functor line(p, i, j) with the value of plane q at pixel p = i * W + j.
struct PlainSrc {  // a stack of planes
  const float* a;
  long long HW;
  struct Line {
    const float* a;
    __device__ __forceinline__ float operator()(long long p, int, int) const { return a[p]; }
  };
  __device__ __forceinline__ Line bind(int q) const { return Line{a + q * HW}; }
};

struct GfInSrc {  // the four box-filter inputs of guided_filter.py:80-86, planes [x: N*Cx | y: N*Cy | x*y: N*Cy | x*x: N*Cx]
  const float *x, *y;
  int N, Cx, Cy;
  long long HW;
  struct Line {
    const float *a, *b;
    __device__ __forceinline__ float operator()(long long p, int, int) const { return b ? __fmul_rn(a[p], b[p]) : a[p]; }
  };
  __device__ __forceinline__ Line bind(int q) const {
    const int nx = N * Cx, ny = N * Cy;
    if (q < nx) return Line{x + q * HW, nullptr};
    if ((q -= nx) < ny) return Line{y + q * HW, nullptr};
    if ((q -= ny) < ny) return Line{x + (long long)(q / Cy * Cx + (Cx == 1 ? 0 : q % Cy)) * HW, y + q * HW};
    q -= ny;
    return Line{x + q * HW, x + q * HW};
  }
};

// the box-sum planes [x | y | xy | xx] of GfInSrc's layout
struct GfBox {
  const float *bx, *by, *bxy, *bxx;
  __device__ __forceinline__ GfBox(const float* box, int N, int Cx, int Cy, long long HW)
      : bx(box), by(box + (long long)N * Cx * HW), bxy(by + (long long)N * Cy * HW), bxx(bxy + (long long)N * Cy * HW) {}
};

struct GfCoefSrc {  // A and b of guided_filter.py:89-91 from the box sums, planes [A: N*Cy | b: N*Cy]
  const float* box;
  int N, Cx, Cy, H, W, r;
  float eps;
  long long HW;
  struct Line {
    const float *bx, *by, *bxy, *bxx;
    int H, W, r;
    float eps;
    bool want_b;
    __device__ __forceinline__ float operator()(long long p, int i, int j) const {
      const GfCoef k(bx[p], by[p], bxy[p], bxx[p], box_count(i, j, H, W, r), eps);
      return want_b ? k.b : k.A;
    }
  };
  __device__ __forceinline__ Line bind(int q) const {
    const int ny = N * Cy;
    const bool want_b = q >= ny;
    if (want_b) q -= ny;
    const long long qx = (long long)(q / Cy * Cx + (Cx == 1 ? 0 : q % Cy)) * HW;
    const GfBox s(box, N, Cx, Cy, HW);
    return Line{s.bx + qx, s.by + q * HW, s.bxy + q * HW, s.bxx + qx, H, W, r, eps, want_b};
  }
};

struct GfGradOutSrc {  // autograd through guided_filter.py:94-97: d box(A) = g * x / N, d box(b) = g / N, planes [A | b]
  const float *g, *x;
  int N, Cx, Cy, H, W, r;
  long long HW;
  struct Line {
    const float *g, *x;
    int H, W, r;
    __device__ __forceinline__ float operator()(long long p, int i, int j) const {
      const float N = box_count(i, j, H, W, r);
      return __fdiv_rn(x ? __fmul_rn(g[p], x[p]) : g[p], N);
    }
  };
  __device__ __forceinline__ Line bind(int q) const {
    const int ny = N * Cy;
    if (q >= ny) return Line{g + (q - ny) * HW, nullptr, H, W, r};
    return Line{g + q * HW, x + (long long)(q / Cy * Cx + (Cx == 1 ? 0 : q % Cy)) * HW, H, W, r};
  }
};

// the adjoint of box_diff at position i of a line of length n, from the line's upstream gradient val(.)
template <class F>
__device__ __forceinline__ float box_diff_adjoint(const F& val, int i, int n, int r) {
  if (i == n - 1) {
    float t = 0.f;
    for (int k = n - r; k < n; ++k) t = __fadd_rn(t, val(k));
    return __fadd_rn(val(n - 1 - r), t);
  }
  const float a = i >= r ? val(i - r) : 0.f;
  return i + r + 1 < n ? __fsub_rn(a, val(i + r + 1)) : a;
}

template <bool ADJ, class Src>
__global__ void __launch_bounds__(32 * GF_COL_SEG)
gf_col_scan_kernel(Src src, float* __restrict__ cs, float* dst, int H, int W, int r, int tiles) {
  __shared__ double tot[GF_COL_SEG][32];
  const int q = blockIdx.x / tiles;
  const int j = (blockIdx.x % tiles) * 32 + threadIdx.x;
  const int ty = threadIdx.y;
  const long long HW = (long long)H * W;
  const int L = (H + GF_COL_SEG - 1) / GF_COL_SEG;
  const int s0 = min(ty * L, H), s1 = min(s0 + L, H);
  const bool on = j < W;
  const auto line = src.bind(q);
  const auto val = [&](int i) { return line((long long)i * W + j, i, j); };
  const auto elem = [&](int i) { return ADJ ? box_diff_adjoint(val, i, H, r) : val(i); };
  double t = 0.0;
  if (on)
    for (int i = s0; i < s1; ++i) t += (double)elem(i);
  tot[ty][threadIdx.x] = t;
  __syncthreads();
  double s = 0.0;
  if (ADJ) {
    for (int k = GF_COL_SEG - 1; k > ty; --k) s += tot[k][threadIdx.x];
  } else {
    for (int k = 0; k < ty; ++k) s += tot[k][threadIdx.x];
  }
  float* dq = dst + q * HW;
  if (ADJ) {
    if (on)
      for (int i = s1 - 1; i >= s0; --i) {
        s += (double)elem(i);
        dq[(long long)i * W + j] = (float)s;
      }
  } else {
    float* cq = cs + q * HW;
    if (on)
      for (int i = s0; i < s1; ++i) {
        s += (double)elem(i);
        cq[(long long)i * W + j] = (float)s;
      }
    __syncthreads();
    if (on)
      for (int i = s0; i < s1; ++i) dq[(long long)i * W + j] = box_diff(cq + j, W, i, H, r);
  }
}

template <bool ADJ, class Src>
__global__ void __launch_bounds__(32 * GF_ROW_WARPS)
gf_row_scan_kernel(Src src, float* __restrict__ cs, float* dst, int planes, int H, int W, int r) {
  const int row = blockIdx.x * GF_ROW_WARPS + threadIdx.y;  // uniform across the warp
  if (row >= planes * H) return;
  const int q = row / H, i = row % H, lane = threadIdx.x;
  const long long HW = (long long)H * W, rb = (long long)i * W;
  const int L = (W + 31) / 32;
  const int s0 = min(lane * L, W), s1 = min(s0 + L, W);
  const auto line = src.bind(q);
  const auto val = [&](int j) { return line(rb + j, i, j); };
  const auto elem = [&](int j) { return ADJ ? box_diff_adjoint(val, j, W, r) : val(j); };
  double t = 0.0;
  for (int j = s0; j < s1; ++j) t += (double)elem(j);
  // inclusive scan of the lane totals (towards the last lane, or towards the first for the adjoint), then exclusive
  double inc = t;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double v = ADJ ? __shfl_down_sync(0xffffffffu, inc, o) : __shfl_up_sync(0xffffffffu, inc, o);
    if (ADJ ? lane + o < 32 : lane >= o) inc += v;
  }
  const double ex = ADJ ? __shfl_down_sync(0xffffffffu, inc, 1) : __shfl_up_sync(0xffffffffu, inc, 1);
  double s = (ADJ ? lane < 31 : lane > 0) ? ex : 0.0;
  float* dr = dst + q * HW + rb;
  if (ADJ) {
    for (int j = s1 - 1; j >= s0; --j) {
      s += (double)elem(j);
      dr[j] = (float)s;
    }
  } else {
    float* cr = cs + q * HW + rb;
    for (int j = s0; j < s1; ++j) {
      s += (double)elem(j);
      cr[j] = (float)s;
    }
    __syncwarp();
    for (int j = s0; j < s1; ++j) dr[j] = box_diff(cr, 1, j, W, r);
  }
}

// box filter of `planes` planes: cumsum(H) -> diff_x, then cumsum(W) -> diff_y (ADJ: the adjoint, rows first)
template <bool ADJ, class Src>
void col_pass(const Src& src, float* cs, float* dst, int planes, int H, int W, int r, cudaStream_t st) {
  const int tiles = ceil_div(W, 32);
  gf_col_scan_kernel<ADJ><<<planes * tiles, dim3(32, GF_COL_SEG), 0, st>>>(src, cs, dst, H, W, r, tiles);
}

template <bool ADJ, class Src>
void row_pass(const Src& src, float* cs, float* dst, int planes, int H, int W, int r, cudaStream_t st) {
  gf_row_scan_kernel<ADJ><<<ceil_div((long long)planes * H, GF_ROW_WARPS), dim3(32, GF_ROW_WARPS), 0, st>>>(
      src, cs, dst, planes, H, W, r);
}

// out[n, c] = mean_A * x[n, cx] + mean_b, from box(A), box(b) ([A | b] planes)
__global__ void __launch_bounds__(256)
gf_apply_kernel(const float* __restrict__ bab, const float* __restrict__ x, int N, int Cx, int Cy, int H, int W, int r,
                float* __restrict__ out) {
  const long long HW = (long long)H * W, n_out = (long long)N * Cy * HW;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_out) return;
  const long long p = t % HW;
  const int q = (int)(t / HW);
  const long long qx = (long long)(q / Cy * Cx + (Cx == 1 ? 0 : q % Cy)) * HW;
  out[t] = gf_out(bab[t], bab[n_out + t], x[qx + p], box_count((int)(p / W), (int)(p % W), H, W, r));
}

// Autograd through guided_filter.py:79-91, one thread per (n, channel of x, pixel): from d A (box(A)'s adjoint plus
// -d b * mean_x) and d b, the gradients of the four box sums, in GfBox's layout. With C_x = 1 the gradients reaching
// mean_x and var_x are summed over y's channels, each broadcast term on its own, as autograd's sum_to_size does.
__global__ void __launch_bounds__(256)
gf_coef_backward_kernel(const float* __restrict__ box, const float* __restrict__ gab, int N, int Cx, int Cy, int H, int W,
                        int r, float eps, float* __restrict__ gbox) {
  const long long HW = (long long)H * W;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * Cx * HW) return;
  const long long p = t % HW;
  const int qx = (int)(t / HW), n = qx / Cx;
  const float Nw = box_count((int)(p / W), (int)(p % W), H, W, r);
  const GfBox s(box, N, Cx, Cy, HW);
  float* g_bx = gbox;
  float* g_by = gbox + (long long)N * Cx * HW;
  float* g_bxy = g_by + (long long)N * Cy * HW;
  float* g_bxx = g_bxy + (long long)N * Cy * HW;
  const float* gA = gab;
  const float* gb = gab + (long long)N * Cy * HW;
  const int c0 = Cx == 1 ? 0 : qx % Cx, c1 = Cx == 1 ? Cy : c0 + 1;
  float s_mx_b = 0.f, s_mx_cov = 0.f, s_var = 0.f;
  for (int c = c0; c < c1; ++c) {
    const long long e = (long long)(n * Cy + c) * HW + p;
    const GfCoef k(s.bx[t], s.by[e], s.bxy[e], s.bxx[t], Nw, eps);
    const float gbv = gb[e], ngb = -gbv;
    const float gAt = __fadd_rn(gA[e], __fmul_rn(ngb, k.mx));            // b = mean_y - A * mean_x
    const float g_cov = __fdiv_rn(gAt, k.ve);                              // A = cov / (var + eps)
    const float g_var = __fdiv_rn(__fmul_rn(-gAt, k.cov), __fmul_rn(k.ve, k.ve));
    const float ngc = -g_cov;                                              // cov = box(xy) / N - mean_x * mean_y
    g_bxy[e] = __fdiv_rn(g_cov, Nw);
    g_by[e] = __fdiv_rn(__fadd_rn(gbv, __fmul_rn(ngc, k.mx)), Nw);
    s_mx_b = c == c0 ? __fmul_rn(ngb, k.A) : __fadd_rn(s_mx_b, __fmul_rn(ngb, k.A));
    s_mx_cov = c == c0 ? __fmul_rn(ngc, k.my) : __fadd_rn(s_mx_cov, __fmul_rn(ngc, k.my));
    s_var = c == c0 ? g_var : __fadd_rn(s_var, g_var);
  }
  // var = box(xx) / N - mean_x * mean_x; mean_x = box(x) / N
  const float mx = __fdiv_rn(s.bx[t], Nw);
  const float m = __fmul_rn(-s_var, mx);
  g_bxx[t] = __fdiv_rn(s_var, Nw);
  g_bx[t] = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(s_mx_b, s_mx_cov), m), m), Nw);
}

// d x and d y from the adjoint box sums G (GfBox layout), box(A) and the upstream gradient g: x feeds box(x), x*y, x*x
// and mean_A * x; y feeds box(y) and x*y. One thread per (n, channel of x, pixel); with C_x = 1 it sums over y's channels.
__global__ void __launch_bounds__(256)
gf_input_backward_kernel(const float* __restrict__ G, const float* __restrict__ bab, const float* __restrict__ g,
                         const float* __restrict__ x, const float* __restrict__ y, int N, int Cx, int Cy, int H, int W,
                         int r, float* __restrict__ gx, float* __restrict__ gy) {
  const long long HW = (long long)H * W;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * Cx * HW) return;
  const long long p = t % HW;
  const int qx = (int)(t / HW), n = qx / Cx;
  const float Nw = box_count((int)(p / W), (int)(p % W), H, W, r);
  const GfBox s(G, N, Cx, Cy, HW);
  const float xv = x[t];
  const int c0 = Cx == 1 ? 0 : qx % Cx, c1 = Cx == 1 ? Cy : c0 + 1;
  float s_out = 0.f, s_xy = 0.f;
  for (int c = c0; c < c1; ++c) {
    const long long e = (long long)(n * Cy + c) * HW + p;
    const float o = __fmul_rn(g[e], __fdiv_rn(bab[e], Nw));   // out = mean_A * x + mean_b
    const float v = __fmul_rn(s.bxy[e], y[e]);                 // x * y
    s_out = c == c0 ? o : __fadd_rn(s_out, o);
    s_xy = c == c0 ? v : __fadd_rn(s_xy, v);
    if (gy) gy[e] = __fadd_rn(s.by[e], __fmul_rn(s.bxy[e], xv));
  }
  const float xx = __fmul_rn(s.bxx[t], xv);                   // x * x
  if (gx) gx[t] = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s.bx[t], s_out), s_xy), xx), xx);
}

int check_gf_dims(int N, int Cx, int Cy, int H, int W, int r) {
  NRGBD_REQUIRE(N > 0 && Cy > 0 && (Cx == 1 || Cx == Cy), "x must have one channel or as many as y (guided_filter.py:72)");
  NRGBD_REQUIRE(r >= 0 && H > 2 * r + 1 && W > 2 * r + 1, "image smaller than the box (guided_filter.py:74)");
  return NRGBD_OK;
}

}  // namespace

extern "C" {

// workspace [x | y | the GuidedFilter forward's workspace for one plane]
long long nrgbd_guided_filter_workspace_floats(int H, int W) {
  return 2LL * H * W + nrgbd_gf_workspace_floats(1, 1, 1, H, W, 0);
}

// gf_prep_kernel writes the guide x and the upsampled depth y, then nrgbd_guided_filter filters y guided by x
int nrgbd_guided_filter_refine(const float* dmap, int h, int w, const float* img, long long img_sc, long long img_sp, int H,
                               int W, const float* w0, const float* b0, const float* w1, const float* b1, int r, float eps,
                               float* ws, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(dmap && img && w0 && b0 && w1 && b1 && ws && out, "null pointer");
  NRGBD_REQUIRE(h > 0 && w > 0 && H % h == 0 && W % w == 0 && H / h == W / w && H / h > 1,
                "the guide must be an integer multiple > 1 of the depth map's size, the same in both axes (Refine.py:633-637)");
  if (int rc = check_gf_dims(1, 1, 1, H, W, r)) return rc;
  const long long HW = (long long)H * W;
  const float sy = h > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = w > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  gf_prep_kernel<<<ceil_div(HW, 256), 256, 0, st>>>(dmap, h, w, img, img_sc, img_sp, H, W, sy, sx, w0, b0, w1, b1, ws);
  NRGBD_COUNT(1);
  return nrgbd_guided_filter(ws, ws + HW, 1, 1, 1, H, W, r, eps, ws + 2 * HW, out, st);
}

long long nrgbd_box_filter_workspace_floats(int N, int C, int H, int W) { return (long long)N * C * H * W; }

int nrgbd_box_filter(const float* x, int N, int C, int H, int W, int r, float* ws, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(x && ws && out, "null pointer");
  NRGBD_REQUIRE(N > 0 && C > 0 && r >= 0 && H >= 2 * r + 1 && W >= 2 * r + 1,
                "image smaller than the box: box_filter.py's diff changes the shape below 2r + 1");
  const long long HW = (long long)H * W;
  col_pass<false>(PlainSrc{x, HW}, ws, out, N * C, H, W, r, st);
  row_pass<false>(PlainSrc{out, HW}, ws, out, N * C, H, W, r, st);
  NRGBD_COUNT(2);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_box_filter_backward(const float* grad_out, int N, int C, int H, int W, int r, float* ws, float* grad_x,
                              cudaStream_t st) {
  NRGBD_REQUIRE(grad_out && ws && grad_x, "null pointer");
  NRGBD_REQUIRE(N > 0 && C > 0 && r >= 0 && H >= 2 * r + 1 && W >= 2 * r + 1,
                "image smaller than the box: box_filter.py's diff changes the shape below 2r + 1");
  NRGBD_REQUIRE(ws != grad_out && grad_x != ws, "the workspace must not alias the gradients");
  const long long HW = (long long)H * W;
  row_pass<true>(PlainSrc{grad_out, HW}, nullptr, ws, N * C, H, W, r, st);
  col_pass<true>(PlainSrc{ws, HW}, nullptr, grad_x, N * C, H, W, r, st);
  NRGBD_COUNT(2);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

long long nrgbd_gf_workspace_floats(int N, int Cx, int Cy, int H, int W, int backward) {
  const long long HW = (long long)H * W, p4 = 2LL * N * (Cx + Cy), pab = 2LL * N * Cy;
  return (backward ? 3 * p4 + 2 * pab : 2 * p4 + pab) * HW;
}

// forward: box sums of [x | y | xy | xx] (the products formed while scanning), box sums of [A | b] (A and b formed while
// scanning), then mean_A * x + mean_b. Workspace [box4 | prefix scratch | box(A), box(b)].
static int gf_forward_planes(const float* x, const float* y, int N, int Cx, int Cy, int H, int W, int r, float eps,
                             float* ws, cudaStream_t st) {
  const long long HW = (long long)H * W;
  const int p4 = 2 * N * (Cx + Cy), pab = 2 * N * Cy;
  float* box4 = ws;
  float* cs = box4 + p4 * HW;
  float* bab = cs + p4 * HW;
  col_pass<false>(GfInSrc{x, y, N, Cx, Cy, HW}, cs, box4, p4, H, W, r, st);
  row_pass<false>(PlainSrc{box4, HW}, cs, box4, p4, H, W, r, st);
  col_pass<false>(GfCoefSrc{box4, N, Cx, Cy, H, W, r, eps, HW}, cs, bab, pab, H, W, r, st);
  row_pass<false>(PlainSrc{bab, HW}, cs, bab, pab, H, W, r, st);
  return 4;
}

int nrgbd_guided_filter(const float* x, const float* y, int N, int Cx, int Cy, int H, int W, int r, float eps, float* ws,
                        float* out, cudaStream_t st) {
  NRGBD_REQUIRE(x && y && ws && out, "null pointer");
  if (int rc = check_gf_dims(N, Cx, Cy, H, W, r)) return rc;
  const long long HW = (long long)H * W;
  const int n = gf_forward_planes(x, y, N, Cx, Cy, H, W, r, eps, ws, st);
  const float* bab = ws + 4LL * N * (Cx + Cy) * HW;
  gf_apply_kernel<<<ceil_div((long long)N * Cy * HW, 256), 256, 0, st>>>(bab, x, N, Cx, Cy, H, W, r, out);
  NRGBD_COUNT(n + 1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// backward: recompute the forward's box sums (only x and y are kept between the passes), then the adjoint of
// guided_filter.py:76-97 in autograd's order. Workspace [box4 | scratch (P4) | box(A), box(b) | d A, d b | adjoint (P4)].
int nrgbd_guided_filter_backward(const float* grad_out, const float* x, const float* y, int N, int Cx, int Cy, int H,
                                 int W, int r, float eps, float* ws, float* grad_x, float* grad_y, cudaStream_t st) {
  NRGBD_REQUIRE(grad_out && x && y && ws, "null pointer");
  if (int rc = check_gf_dims(N, Cx, Cy, H, W, r)) return rc;
  const long long HW = (long long)H * W;
  const int p4 = 2 * N * (Cx + Cy), pab = 2 * N * Cy;
  float* box4 = ws;
  float* cs = box4 + p4 * HW;
  float* bab = cs + p4 * HW;
  float* gab = bab + pab * HW;
  float* adj = gab + pab * HW;
  const int n = gf_forward_planes(x, y, N, Cx, Cy, H, W, r, eps, ws, st);
  // d box(A), d box(b) -> d A, d b (their box filters' adjoints: rows, then columns)
  row_pass<true>(GfGradOutSrc{grad_out, x, N, Cx, Cy, H, W, r, HW}, nullptr, cs, pab, H, W, r, st);
  col_pass<true>(PlainSrc{cs, HW}, nullptr, gab, pab, H, W, r, st);
  const unsigned grid = (unsigned)ceil_div((long long)N * Cx * HW, 256);
  gf_coef_backward_kernel<<<grid, 256, 0, st>>>(box4, gab, N, Cx, Cy, H, W, r, eps, cs);
  // d box4 -> d [x | y | xy | xx]
  row_pass<true>(PlainSrc{cs, HW}, nullptr, adj, p4, H, W, r, st);
  col_pass<true>(PlainSrc{adj, HW}, nullptr, cs, p4, H, W, r, st);
  gf_input_backward_kernel<<<grid, 256, 0, st>>>(cs, bab, grad_out, x, y, N, Cx, Cy, H, W, r, grad_x, grad_y);
  NRGBD_COUNT(n + 6);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
