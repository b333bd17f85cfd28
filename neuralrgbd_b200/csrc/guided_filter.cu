// Guided-filter depth refinement: RefineNet_DGF.forward (models/Refine.py:620-641) with GuidedFilter(r, eps)
// (models/GF/guided_filter.py) and its BoxFilter (models/GF/box_filter.py), for KVNET(refineNet_name='DGF').
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
#include "common.cuh"

namespace {

constexpr int GF_HID = 64;      // RefineNet_DGF.feature_ext: Conv2d(3, 64, 1) -> ReLU -> Conv2d(64, 1, 1)

// planes [x | y | x*y | x*x], each [H][W]: the upsampled depth, the 1x1 MLP of the guide image and the two products
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
  planes[2 * HW + p] = __fmul_rn(xv, yv);
  planes[3 * HW + p] = __fmul_rn(xv, xv);
}

// One thread per (plane, line): prefix sums along the line in double, each rounded to fp32 (ATen's float cumsum),
// then box_filter.py's diff: out[i] = cs[min(i + r, n - 1)] - (i > r ? cs[i - r - 1] : 0).
// Lines run along H (columns, `step` = W, consecutive threads on consecutive columns) or along W (rows, `step` = 1).
// src may equal dst (each thread reads its whole line before writing it).
__global__ void __launch_bounds__(128)
gf_scan_diff_kernel(const float* src, float* __restrict__ cs, float* dst, int planes, int lines,
                    long long line_stride, int n, long long step, int r, long long plane_stride) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= planes * lines) return;
  const long long base = (long long)(t / lines) * plane_stride + (long long)(t % lines) * line_stride;
  double s = 0.0;
  for (int i = 0; i < n; ++i) {
    s += (double)src[base + i * step];
    cs[base + i * step] = (float)s;
  }
  for (int i = 0; i < n; ++i) {
    const float hi = cs[base + min(i + r, n - 1) * step];
    dst[base + i * step] = i > r ? __fsub_rn(hi, cs[base + (i - r - 1) * step]) : hi;
  }
}

__device__ __forceinline__ float box_count(int i, int j, int H, int W, int r) {
  return (float)((min(i + r, H - 1) - max(i - r, 0) + 1) * (min(j + r, W - 1) - max(j - r, 0) + 1));
}

// box sums of [x | y | xy | xx] -> A, b (guided_filter.py: N, mean_x, mean_y, cov_xy, var_x, A, b)
__global__ void __launch_bounds__(256)
gf_coef_kernel(const float* __restrict__ box, int H, int W, int r, float eps, float* __restrict__ A, float* __restrict__ b) {
  const long long HW = (long long)H * W;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const float N = box_count((int)(p / W), (int)(p % W), H, W, r);
  const float mx = __fdiv_rn(box[p], N), my = __fdiv_rn(box[HW + p], N);
  const float cov = __fsub_rn(__fdiv_rn(box[2 * HW + p], N), __fmul_rn(mx, my));
  const float var = __fsub_rn(__fdiv_rn(box[3 * HW + p], N), __fmul_rn(mx, mx));
  const float a = __fdiv_rn(cov, __fadd_rn(var, eps));
  A[p] = a;
  b[p] = __fsub_rn(my, __fmul_rn(a, mx));
}

// out = box(A)/N * x + box(b)/N
__global__ void __launch_bounds__(256)
gf_out_kernel(const float* __restrict__ box_ab, const float* __restrict__ x, int H, int W, int r, float* __restrict__ out) {
  const long long HW = (long long)H * W;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const float N = box_count((int)(p / W), (int)(p % W), H, W, r);
  out[p] = __fadd_rn(__fmul_rn(__fdiv_rn(box_ab[p], N), x[p]), __fdiv_rn(box_ab[HW + p], N));
}

// box filter of `np` planes of src (plane stride HW) into dst, cs as scratch: column pass src -> dst, row pass dst -> dst
void box_filter(const float* src, float* cs, float* dst, int np, int H, int W, int r, cudaStream_t st) {
  const long long HW = (long long)H * W;
  gf_scan_diff_kernel<<<ceil_div((long long)np * W, 128), 128, 0, st>>>(src, cs, dst, np, W, 1, H, W, r, HW);
  gf_scan_diff_kernel<<<ceil_div((long long)np * H, 128), 128, 0, st>>>(dst, cs, dst, np, H, W, W, 1, r, HW);
}

}  // namespace

extern "C" {

long long nrgbd_guided_filter_workspace_floats(int H, int W) { return 12LL * H * W; }

int nrgbd_guided_filter_refine(const float* dmap, int h, int w, const float* img, long long img_sc, long long img_sp, int H,
                               int W, const float* w0, const float* b0, const float* w1, const float* b1, int r, float eps,
                               float* ws, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(dmap && img && w0 && b0 && w1 && b1 && ws && out, "null pointer");
  NRGBD_REQUIRE(h > 0 && w > 0 && H % h == 0 && W % w == 0 && H / h == W / w && H / h > 1,
                "the guide must be an integer multiple > 1 of the depth map's size, the same in both axes (Refine.py:633-637)");
  NRGBD_REQUIRE(r >= 0 && H > 2 * r + 1 && W > 2 * r + 1, "guide smaller than the box (guided_filter.py:73)");
  const long long HW = (long long)H * W;
  float* planes = ws;             // [x | y | xy | xx], then [x | A | b]
  float* cs = ws + 4 * HW;        // prefix sums
  float* box = ws + 8 * HW;       // box sums
  const unsigned grid = (unsigned)ceil_div(HW, 256);
  const float sy = h > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = w > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  gf_prep_kernel<<<grid, 256, 0, st>>>(dmap, h, w, img, img_sc, img_sp, H, W, sy, sx, w0, b0, w1, b1, planes);
  box_filter(planes, cs, box, 4, H, W, r, st);
  gf_coef_kernel<<<grid, 256, 0, st>>>(box, H, W, r, eps, planes + HW, planes + 2 * HW);
  box_filter(planes + HW, cs, box, 2, H, W, r, st);
  gf_out_kernel<<<grid, 256, 0, st>>>(box, planes, H, W, r, out);
  NRGBD_COUNT(7);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
