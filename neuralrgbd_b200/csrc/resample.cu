// DPV re-projection into the next camera (SURVEY §8 a12).
//
// Replaces warping/homography.py:654-723 (resample_vol_cuda) + :873-887 (_set_vol_border) +
// the clamp of test_utils/test_KVNet.py:54-59 with one trilinear-gather kernel: the point
// cloud d * ray is never built on the host nor uploaded (the reference ships 3*D*h*w floats
// per call), the six volume faces are overwritten with padding_value on the fly instead of
// cloning the volume, and the [-1000, 0] clamp is applied in the same pass.
// Bug-for-bug details kept (torch 2.11 semantics): align_corners=False un-normalisation (an
// identity pose is NOT an identity resample), z range taken from d_candi, division of all
// coordinates by (w + 1e-10), border clamping before interpolation.
#include "common.cuh"

namespace {

__device__ __forceinline__ float clip_coord(float x, float hi) { return fminf(hi, fmaxf(x, 0.f)); }

// Border-clamped sampling location (ix, iy, iz) in the source volume of output voxel (d, pix):
// the point float32(d) * float32(ray) moved by rel_extM and normalised as homography.py:679-708.
// Shared by the forward and the backward, so both see the same corners and weights bit for bit.
__device__ __forceinline__ void resample_coords(const float* __restrict__ E, const float* __restrict__ rays,
                                                const float* __restrict__ d_pts, int d, int pix, int D, int H, int W,
                                                float tan_hh, float tan_hv, float z_half, float z_radius, float& ix,
                                                float& iy, float& iz) {
  const int hw = H * W;
  // point in the reference camera: float32(d) * float32(ray)   (homography.py:679-681)
  const float dv = __ldg(d_pts + d);
  const float X = __fmul_rn(dv, rays[pix]);
  const float Y = __fmul_rn(dv, rays[hw + pix]);
  const float Z = __fmul_rn(dv, rays[2 * hw + pix]);
  float r[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {           // rel_extM . [X;Y;Z;1], sgemm FMA-chain order (:700)
    float acc = __fmul_rn(E[i * 4 + 0], X);
    acc = __fmaf_rn(E[i * 4 + 1], Y, acc);
    acc = __fmaf_rn(E[i * 4 + 2], Z, acc);
    acc = __fmaf_rn(E[i * 4 + 3], 1.f, acc);
    r[i] = acc;
  }
  const float den = __fadd_rn(r[2], 1e-10f);
  float gx = __fdiv_rn(__fdiv_rn(r[0], den), tan_hh);        // :703
  float gy = __fdiv_rn(__fdiv_rn(r[1], den), tan_hv);        // :704
  float gz = __fdiv_rn(__fsub_rn(r[2], z_half), z_radius);   // :705
  const float wden = __fadd_rn(r[3], 1e-10f);                // :708
  gx = __fdiv_rn(gx, wden); gy = __fdiv_rn(gy, wden); gz = __fdiv_rn(gz, wden);
  ix = clip_coord(unnormalize(gx, (float)W), (float)(W - 1));
  iy = clip_coord(unnormalize(gy, (float)H), (float)(H - 1));
  iz = clip_coord(unnormalize(gz, (float)D), (float)(D - 1));
}

// Visits the in-range trilinear corners of (ix, iy, iz) in ATen's order (tnw ... bse) as f(zz, yy, xx, face, weight);
// `face` marks the six faces that _set_vol_border overwrites. NaN coordinates visit no corner.
template <typename F>
__device__ __forceinline__ void for_each_corner(float ix, float iy, float iz, int D, int H, int W, F&& f) {
  if (isnan(ix) || isnan(iy) || isnan(iz)) return;
  const float x0 = floorf(ix), y0 = floorf(iy), z0 = floorf(iz);
  const float x1 = __fadd_rn(x0, 1.f), y1 = __fadd_rn(y0, 1.f), z1 = __fadd_rn(z0, 1.f);
  const float wx[2] = {__fsub_rn(x1, ix), __fsub_rn(ix, x0)};
  const float wy[2] = {__fsub_rn(y1, iy), __fsub_rn(iy, y0)};
  const float wz[2] = {__fsub_rn(z1, iz), __fsub_rn(iz, z0)};
  const int xi[2] = {(int)x0, (int)x0 + 1}, yi[2] = {(int)y0, (int)y0 + 1}, zi[2] = {(int)z0, (int)z0 + 1};
#pragma unroll
  for (int c = 0; c < 2; ++c)
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const int xx = xi[a], yy = yi[b], zz = zi[c];
        if (xx < W && yy < H && zz < D) {     // lower bounds hold after the clip
          const bool face = (xx == 0) || (xx == W - 1) || (yy == 0) || (yy == H - 1) || (zz == 0) || (zz == D - 1);
          f(zz, yy, xx, face, __fmul_rn(__fmul_rn(wx[a], wy[b]), wz[c]));
        }
      }
}

__device__ __forceinline__ float resample_value(const float* __restrict__ vol, long long in_sd, long long in_sp, float ix,
                                                float iy, float iz, int D, int H, int W, float pad) {
  float res = 0.f;
  for_each_corner(ix, iy, iz, D, H, W, [&](int zz, int yy, int xx, bool face, float wgt) {
    const float v = face ? pad : __ldg(vol + (long long)zz * in_sd + (long long)(yy * W + xx) * in_sp);
    res = __fadd_rn(res, __fmul_rn(v, wgt));
  });
  return res;
}

__global__ void __launch_bounds__(256)
resample_dpv_kernel(const float* __restrict__ vol, long long in_sd, long long in_sp, const float* __restrict__ E,
                    const float* __restrict__ rays, const float* __restrict__ d_pts, int D, int H, int W,
                    float tan_hh, float tan_hv, float z_half, float z_radius, float pad, int do_clamp,
                    float clamp_lo, float clamp_hi, float* __restrict__ out, long long out_sd, long long out_sp,
                    int pixel_major) {
  const int hw = H * W;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)hw * D) return;
  int pix, d;
  if (pixel_major) { d = (int)(idx % D); pix = (int)(idx / D); }
  else { pix = (int)(idx % hw); d = (int)(idx / hw); }
  float ix, iy, iz;
  resample_coords(E, rays, d_pts, d, pix, D, H, W, tan_hh, tan_hv, z_half, z_radius, ix, iy, iz);
  float res = resample_value(vol, in_sd, in_sp, ix, iy, iz, D, H, W, pad);
  if (do_clamp) res = fminf(clamp_hi, fmaxf(res, clamp_lo));
  out[(long long)d * out_sd + (long long)pix * out_sp] = res;
}

// Input gradient of the forward: what autograd gives through _set_vol_border + grid_sample(bilinear, border) 3-D
// (+ torch.clamp). Each in-range corner that is not on a face receives grad * weight (the faces were overwritten by
// pad_value, so their gradient is zero); with do_clamp the gradient passes only where lo <= res <= hi, as in
// torch.clamp's backward, which needs the pre-clamp value and so re-reads vol. fp32 atomics: the order is not fixed.
__global__ void __launch_bounds__(256)
resample_dpv_backward_kernel(const float* __restrict__ vol, long long in_sd, long long in_sp, const float* __restrict__ E,
                             const float* __restrict__ rays, const float* __restrict__ d_pts, int D, int H, int W,
                             float tan_hh, float tan_hv, float z_half, float z_radius, float pad, int do_clamp,
                             float clamp_lo, float clamp_hi, const float* __restrict__ grad_out, long long out_sd,
                             long long out_sp, int pixel_major, float* __restrict__ g_vol) {
  const int hw = H * W;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)hw * D) return;
  int pix, d;
  if (pixel_major) { d = (int)(idx % D); pix = (int)(idx / D); }
  else { pix = (int)(idx % hw); d = (int)(idx / hw); }
  const float g = __ldg(grad_out + (long long)d * out_sd + (long long)pix * out_sp);
  if (g == 0.f) return;
  float ix, iy, iz;
  resample_coords(E, rays, d_pts, d, pix, D, H, W, tan_hh, tan_hv, z_half, z_radius, ix, iy, iz);
  if (do_clamp) {
    const float res = resample_value(vol, in_sd, in_sp, ix, iy, iz, D, H, W, pad);
    if (!(res >= clamp_lo && res <= clamp_hi)) return;
  }
  for_each_corner(ix, iy, iz, D, H, W, [&](int zz, int yy, int xx, bool face, float wgt) {
    if (!face && wgt != 0.f) atomicAdd(g_vol + (long long)zz * in_sd + (long long)(yy * W + xx) * in_sp, g * wgt);
  });
}

}  // namespace

extern "C" {

// vol/out element (d, pix) lives at d*stride_d + pix*stride_pix: (hw, 1) for the reference's
// [D][h][w] layout, (1, D) for the engine's pixel-major layout. d_pts: the D plane depths used to
// build the point cloud (d_candi_new if given else d_candi). E: 4x4 row-major, device.
int nrgbd_resample_dpv(const float* vol, long long in_stride_d, long long in_stride_pix, const float* E,
                       const float* rays, const float* d_pts, int D, int H, int W, float tan_hh, float tan_hv,
                       float z_half, float z_radius, float pad_value, int do_clamp, float clamp_lo,
                       float clamp_hi, float* out, long long out_stride_d, long long out_stride_pix,
                       cudaStream_t st) {
  NRGBD_REQUIRE(vol && E && rays && d_pts && out, "null pointer");
  NRGBD_REQUIRE(D > 0 && H > 0 && W > 0, "empty volume");
  long long n = (long long)D * H * W;
  resample_dpv_kernel<<<ceil_div(n, 256), 256, 0, st>>>(vol, in_stride_d, in_stride_pix, E, rays, d_pts, D, H, W,
                                                        tan_hh, tan_hv, z_half, z_radius, pad_value, do_clamp,
                                                        clamp_lo, clamp_hi, out, out_stride_d, out_stride_pix,
                                                        out_stride_d == 1 ? 1 : 0);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Gradient of nrgbd_resample_dpv with respect to vol, for the same arguments. grad_out is read with the output strides,
// g_vol is written with the input strides, which must describe a dense D*H*W buffer ((hw, 1) or (1, D)); it is zeroed
// here before the scatter. vol is read only when do_clamp != 0 (it may be NULL otherwise).
int nrgbd_resample_dpv_backward(const float* vol, long long in_stride_d, long long in_stride_pix, const float* E,
                                const float* rays, const float* d_pts, int D, int H, int W, float tan_hh, float tan_hv,
                                float z_half, float z_radius, float pad_value, int do_clamp, float clamp_lo,
                                float clamp_hi, const float* grad_out, long long out_stride_d, long long out_stride_pix,
                                float* g_vol, cudaStream_t st) {
  NRGBD_REQUIRE(E && rays && d_pts && grad_out && g_vol && (vol || !do_clamp), "null pointer");
  NRGBD_REQUIRE(D > 0 && H > 0 && W > 0, "empty volume");
  const long long hw = (long long)H * W;
  NRGBD_REQUIRE((in_stride_d == hw && in_stride_pix == 1) || (in_stride_d == 1 && in_stride_pix == D),
                "the gradient volume must be dense: strides (H*W, 1) or (1, D)");
  long long n = (long long)D * hw;
  NRGBD_CUDA_CHECK(cudaMemsetAsync(g_vol, 0, sizeof(float) * (size_t)n, st));
  resample_dpv_backward_kernel<<<ceil_div(n, 256), 256, 0, st>>>(vol, in_stride_d, in_stride_pix, E, rays, d_pts, D, H, W,
                                                                 tan_hh, tan_hv, z_half, z_radius, pad_value, do_clamp,
                                                                 clamp_lo, clamp_hi, grad_out, out_stride_d, out_stride_pix,
                                                                 out_stride_d == 1 ? 1 : 0, g_vol);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
