// Shared helpers for the nrgbd sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#define NRGBD_OK 0
#define NRGBD_ERR_BAD_ARG (-1)
#define NRGBD_ERR_CUDA (-2)
#define NRGBD_ERR_UNSUPPORTED (-3)
#define NRGBD_ERR_NOMEM (-4)

void nrgbd_set_error(const char* fmt, ...);

#define NRGBD_REQUIRE(cond, msg)                                   \
  do {                                                             \
    if (!(cond)) {                                                 \
      nrgbd_set_error("%s: %s", __func__, msg);                    \
      return NRGBD_ERR_BAD_ARG;                                    \
    }                                                              \
  } while (0)

#define NRGBD_CUDA_CHECK(expr)                                                    \
  do {                                                                            \
    cudaError_t _e = (expr);                                                      \
    if (_e != cudaSuccess) {                                                      \
      nrgbd_set_error("%s: CUDA error %s at %s:%d", __func__, cudaGetErrorString(_e), \
                      __FILE__, __LINE__);                                        \
      return NRGBD_ERR_CUDA;                                                      \
    }                                                                             \
  } while (0)

#define NRGBD_LAUNCH_CHECK() NRGBD_CUDA_CHECK(cudaGetLastError())

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// SMs of the current device (queried once per translation unit): grid caps of the grid-stride kernels
static inline int nrgbd_sm_count() {
  static int n = 0;
  if (n < 1) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = 1;
  }
  return n;
}

// launch counter (bench.py reports it as gpu_launches)
extern "C" void nrgbd_count_launch(int n);
#define NRGBD_COUNT(n) nrgbd_count_launch(n)

// ---------------------------------------------------------------------------
// Coordinate arithmetic with a pinned rounding order (see DESIGN.md).
// torch eager executes every op separately (no contraction across ops), and its
// small matmuls are sgemm FMA chains over k. These helpers keep nvcc from fusing.
// ---------------------------------------------------------------------------
__device__ __forceinline__ float dot3_chain(float a0, float a1, float a2, float b0, float b1, float b2) {
  float acc = __fmul_rn(a0, b0);
  acc = __fmaf_rn(a1, b1, acc);
  acc = __fmaf_rn(a2, b2, acc);
  return acc;
}

// ATen grid_sampler_unnormalize, align_corners=False: ((g + 1) * size - 1) / 2
__device__ __forceinline__ float unnormalize(float g, float size) {
  return __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(g, 1.f), size), 1.f), 2.f);
}

struct Tap2D {
  // clamped element offsets (y*W + x) of the 4 corners and their weights (0 when out of range)
  int o_nw, o_ne, o_sw, o_se;
  float w_nw, w_ne, w_sw, w_se;
};

// Bilinear corner set for F.grid_sample(mode='bilinear', padding_mode='zeros',
// align_corners=False) at un-normalised location (ix, iy) in a W x H image.
__device__ __forceinline__ Tap2D make_tap2d(float ix, float iy, int W, int H) {
  Tap2D t;
  // NaN / inf / far-out coordinates: all four corners out of range -> contributes 0
  bool bad = !(fabsf(ix) < 1.0e9f) || !(fabsf(iy) < 1.0e9f);
  float fx0 = floorf(ix), fy0 = floorf(iy);
  float fx1 = __fadd_rn(fx0, 1.f), fy1 = __fadd_rn(fy0, 1.f);
  float ax = __fsub_rn(fx1, ix), bx = __fsub_rn(ix, fx0);   // (ix_se - ix), (ix - ix_nw)
  float ay = __fsub_rn(fy1, iy), by = __fsub_rn(iy, fy0);
  int x0 = bad ? -2 : (int)fx0, y0 = bad ? -2 : (int)fy0;
  int x1 = x0 + 1, y1 = y0 + 1;
  bool vx0 = (x0 >= 0) && (x0 < W), vx1 = (x1 >= 0) && (x1 < W);
  bool vy0 = (y0 >= 0) && (y0 < H), vy1 = (y1 >= 0) && (y1 < H);
  int cx0 = min(max(x0, 0), W - 1), cx1 = min(max(x1, 0), W - 1);
  int cy0 = min(max(y0, 0), H - 1), cy1 = min(max(y1, 0), H - 1);
  t.o_nw = cy0 * W + cx0; t.o_ne = cy0 * W + cx1;
  t.o_sw = cy1 * W + cx0; t.o_se = cy1 * W + cx1;
  t.w_nw = (vx0 && vy0) ? __fmul_rn(ax, ay) : 0.f;
  t.w_ne = (vx1 && vy0) ? __fmul_rn(bx, ay) : 0.f;
  t.w_sw = (vx0 && vy1) ? __fmul_rn(ax, by) : 0.f;
  t.w_se = (vx1 && vy1) ? __fmul_rn(bx, by) : 0.f;
  return t;
}

// Homography back-projection of one reference pixel onto one plane
// (warping/homography.py:434-446 + ATen un-normalisation): returns (ix, iy).
// t1 = K.t (3), t2 = (K.R).ray (3) for this pixel, d = plane depth, cx/cy from intrinsic_M.
__device__ __forceinline__ void plane_project(float t1x, float t1y, float t1z, float t2x, float t2y,
                                              float t2z, float d, float cx, float cy, float Wf, float Hf,
                                              float& ix, float& iy) {
  float px = __fadd_rn(t1x, __fmul_rn(t2x, d));
  float py = __fadd_rn(t1y, __fmul_rn(t2y, d));
  float pz = __fadd_rn(t1z, __fmul_rn(t2z, d));
  float den = __fadd_rn(pz, 1e-10f);
  px = __fdiv_rn(px, den);
  py = __fdiv_rn(py, den);
  float gx = __fdiv_rn(__fsub_rn(px, cx), cx);
  float gy = __fdiv_rn(__fsub_rn(py, cy), cy);
  ix = unnormalize(gx, Wf);
  iy = unnormalize(gy, Hf);
}


// ---------------------------------------------------------------------------
// Split-fp16 operand pair of the second-generation tensor-core convolution (csrc/conv_f16.cu):
// a = hi + lo * 2^-11 with hi = RN_f16(a), lo = RN_f16((a - hi) * 2^11); saturating at the fp16 range.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void nrgbd_split_pair(float a, __half& hi, __half& lo) {
  const float c = fminf(fmaxf(a, -65504.f), 65504.f);
  hi = __float2half_rn(c);
  const float r = (c - __half2float(hi)) * 2048.f;           // exact difference, exact power-of-two scale
  lo = __float2half_rn(fminf(fmaxf(r, -65504.f), 65504.f));
}
// value of four packed pairs: hi + lo * 2^-11 (exact in fp32 when |lo| * 2^-11 <= ulp(hi) / 2, i.e. always for pairs made by nrgbd_split_pair)
__device__ __forceinline__ void nrgbd_join_pair4(const uint2& hi, const uint2& lo, float* o) {
  const uint32_t hw[2] = {hi.x, hi.y}, lw[2] = {lo.x, lo.y};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float h = __half2float(__ushort_as_half((unsigned short)(hw[k >> 1] >> (16 * (k & 1)))));
    const float l = __half2float(__ushort_as_half((unsigned short)(lw[k >> 1] >> (16 * (k & 1)))));
    o[k] = fmaf(l, 1.f / 2048.f, h);
  }
}
__device__ __forceinline__ void nrgbd_split_pair4(const float* o, uint2& hi, uint2& lo) {
  __half h[4], l[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) nrgbd_split_pair(o[k], h[k], l[k]);
  hi.x = (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16);
  hi.y = (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16);
  lo.x = (uint32_t)__half_as_ushort(l[0]) | ((uint32_t)__half_as_ushort(l[1]) << 16);
  lo.y = (uint32_t)__half_as_ushort(l[2]) | ((uint32_t)__half_as_ushort(l[3]) << 16);
}
