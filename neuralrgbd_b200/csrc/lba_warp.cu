// Depth-map back-warp of the local bundle adjustment and its gradients (SURVEY §8 f-3).
//
// Replaces warping/homography.py:479-529 (back_warp_th_Rt_msrc) and :530-574 (back_warp_th_Rt): the reference depth map is
// back-projected with the unit-ray table (X = d * ray), moved into each source camera (R X + t), projected with K,
// normalised to [-1, 1] and the source image is sampled there with F.grid_sample (bilinear, zeros padding,
// align_corners = False under torch >= 1.3). ICP/opt_pose_numerical.py:99-160 differentiates the warped image with
// respect to R and t (60 Adam iterations x 3 scales per frame): the backward kernel is grid_sampler_2d_backward with
// respect to the grid chained through the perspective division and the two small matmuls, plus the scatter-add of the
// image gradient. One thread per (view, reference pixel); no N x H x W x 2 grid tensor, no homogeneous point matrices.
#include "lba_common.cuh"
#include "../../include/nrgbd.h"

namespace {

__global__ void __launch_bounds__(256)
lba_warp_forward_kernel(const float* __restrict__ imgs, const float* __restrict__ dmap, const float* __restrict__ Rs,
                        const float* __restrict__ ts, const float* __restrict__ K, const float* __restrict__ rays, int N, int C,
                        int H, int W, float* __restrict__ out) {
  const int hw = H * W;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= (long long)N * hw) return;
  const int n = (int)(gid / hw), p = (int)(gid - (long long)n * hw);
  const LbaGeom g = lba_project(dmap[p], rays[p], rays[hw + p], rays[2 * hw + p], Rs + n * 9, ts + n * 3, K, (float)W, (float)H);
  const Tap2D tp = make_tap2d(g.ix, g.iy, W, H);
  const float* src = imgs + (long long)n * C * hw;
  float* dst = out + (long long)n * C * hw + p;
  for (int c = 0; c < C; ++c) {
    const float* s = src + (long long)c * hw;
    // ATen grid_sampler_2d: nw * w_nw + ne * w_ne + sw * w_sw + se * w_se, accumulated in this order
    float acc = __fmul_rn(__ldg(s + tp.o_nw), tp.w_nw);
    acc = __fadd_rn(acc, __fmul_rn(__ldg(s + tp.o_ne), tp.w_ne));
    acc = __fadd_rn(acc, __fmul_rn(__ldg(s + tp.o_sw), tp.w_sw));
    acc = __fadd_rn(acc, __fmul_rn(__ldg(s + tp.o_se), tp.w_se));
    dst[(long long)c * hw] = acc;
  }
}

// g_pose[n][0..8] += dL/dR (row-major), g_pose[n][9..11] += dL/dt (double accumulators, one atomic set per block and view);
// g_imgs (optional, zeroed by the caller) gets the scatter-add of the bilinear weights.
__global__ void __launch_bounds__(256)
lba_warp_backward_kernel(const float* __restrict__ grad_out, const float* __restrict__ imgs, const float* __restrict__ dmap,
                         const float* __restrict__ Rs, const float* __restrict__ ts, const float* __restrict__ K,
                         const float* __restrict__ rays, int N, int C, int H, int W, float* __restrict__ g_imgs,
                         double* __restrict__ g_pose) {
  const int hw = H * W;
  const int n = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  float acc[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) acc[i] = 0.f;
  if (p < hw) {
    const float Wf = (float)W, Hf = (float)H;
    const LbaGeom g = lba_project(dmap[p], rays[p], rays[hw + p], rays[2 * hw + p], Rs + n * 9, ts + n * 3, K, Wf, Hf);
    const bool bad = !(fabsf(g.ix) < 1.0e9f) || !(fabsf(g.iy) < 1.0e9f);
    if (!bad) {
      const float fx0 = floorf(g.ix), fy0 = floorf(g.iy);
      const int x0 = (int)fx0, y0 = (int)fy0, x1 = x0 + 1, y1 = y0 + 1;
      const float ax = (fx0 + 1.f) - g.ix, bx = g.ix - fx0, ay = (fy0 + 1.f) - g.iy, by = g.iy - fy0;
      const bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
      const float* src = imgs + (long long)n * C * hw;
      const float* go = grad_out + (long long)n * C * hw + p;
      float* gi = g_imgs ? g_imgs + (long long)n * C * hw : nullptr;
      float gix = 0.f, giy = 0.f;
      for (int c = 0; c < C; ++c) {
        const float gv = go[(long long)c * hw];
        const float* s = src + (long long)c * hw;
        const float nw = (vx0 && vy0) ? __ldg(s + y0 * W + x0) : 0.f, ne = (vx1 && vy0) ? __ldg(s + y0 * W + x1) : 0.f;
        const float sw = (vx0 && vy1) ? __ldg(s + y1 * W + x0) : 0.f, se = (vx1 && vy1) ? __ldg(s + y1 * W + x1) : 0.f;
        lba_grid_grad(gv, nw, ne, sw, se, ax, bx, ay, by, gix, giy);
        if (gi) {
          float* d = gi + (long long)c * hw;
          if (vx0 && vy0) atomicAdd(d + y0 * W + x0, gv * ax * ay);
          if (vx1 && vy0) atomicAdd(d + y0 * W + x1, gv * bx * ay);
          if (vx0 && vy1) atomicAdd(d + y1 * W + x0, gv * ax * by);
          if (vx1 && vy1) atomicAdd(d + y1 * W + x1, gv * bx * by);
        }
      }
      lba_pose_grad(g, gix, giy, K, Wf, Hf, acc);
    }
  }
  // block reduction of the 12 pose-gradient terms (double from the warp level on)
  __shared__ double red[8][12];
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    double v = (double)acc[i];
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    if (lane == 0) red[wrp][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < 12) {
    double v = 0.0;
    for (int k = 0; k < 8; ++k) v += red[k][threadIdx.x];
    atomicAdd(g_pose + n * 12 + threadIdx.x, v);
  }
}

__global__ void lba_pose_to_float_kernel(const double* __restrict__ g_pose, int N, float* __restrict__ gR, float* __restrict__ gt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * 12) return;
  const int n = i / 12, k = i % 12;
  if (k < 9) gR[n * 9 + k] = (float)g_pose[i]; else gt[n * 3 + (k - 9)] = (float)g_pose[i];
}

}  // namespace

extern "C" {

// imgs [N][C][H][W], dmap [H][W], Rs [N][3][3], ts [N][3], K 3x3 (intrinsic_M_cuda), rays [3][H*W] -> out [N][C][H][W]
int nrgbd_lba_back_warp(const float* imgs, const float* dmap, const float* Rs, const float* ts, const float* K, const float* rays, int N,
                        int C, int H, int W, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(imgs && dmap && Rs && ts && K && rays && out && N > 0 && C > 0 && H > 0 && W > 0, "bad arguments");
  const long long n = (long long)N * H * W;
  lba_warp_forward_kernel<<<ceil_div(n, 256), 256, 0, st>>>(imgs, dmap, Rs, ts, K, rays, N, C, H, W, out);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Gradients of nrgbd_lba_back_warp for grad_out [N][C][H][W]: g_R [N][3][3], g_t [N][3] (either both or none), g_imgs
// [N][C][H][W] (optional; zeroed here, then scatter-added with atomics like ATen's grid_sampler backward).
// ws: N * 12 doubles of device scratch.
int nrgbd_lba_back_warp_backward(const float* grad_out, const float* imgs, const float* dmap, const float* Rs, const float* ts, const float* K,
                                 const float* rays, int N, int C, int H, int W, float* g_imgs, float* g_R, float* g_t, double* ws,
                                 cudaStream_t st) {
  NRGBD_REQUIRE(grad_out && imgs && dmap && Rs && ts && K && rays && ws && N > 0 && C > 0 && H > 0 && W > 0, "bad arguments");
  NRGBD_REQUIRE((g_R != nullptr) == (g_t != nullptr) && (g_R || g_imgs), "nothing to compute");
  NRGBD_CUDA_CHECK(cudaMemsetAsync(ws, 0, sizeof(double) * 12 * N, st));
  if (g_imgs) NRGBD_CUDA_CHECK(cudaMemsetAsync(g_imgs, 0, sizeof(float) * (size_t)N * C * H * W, st));
  dim3 grid(ceil_div((long long)H * W, 256), N);
  lba_warp_backward_kernel<<<grid, 256, 0, st>>>(grad_out, imgs, dmap, Rs, ts, K, rays, N, C, H, W, g_imgs, ws);
  int launches = 1;
  if (g_R) { lba_pose_to_float_kernel<<<ceil_div(N * 12, 128), 128, 0, st>>>(ws, N, g_R, g_t); ++launches; }
  NRGBD_COUNT(launches);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
