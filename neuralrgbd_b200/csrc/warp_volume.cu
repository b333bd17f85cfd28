// Image warp to a plane-sweep volume (SURVEY §8 a7) and K-Net input assembly (a8 head).
//
// Replaces warping/homography.py:234-280 (warp_img_feats_v3) / :183-232 (_mgpu) and the
// cat/repeat/transpose assembly of models/KVNET.py:147-166. Pure write-bound gather:
// one thread per (pixel, plane) evaluates the homography per view and bilinearly samples
// a <=4-channel image stored pixel-interleaved ([hw][4], one LDG.128 per corner).
#include "common.cuh"
#include "../../include/nrgbd.h"

namespace {

__device__ __forceinline__ float4 sample4(const float4* __restrict__ img, const Tap2D& tp) {
  float4 a = __ldg(img + tp.o_nw), b = __ldg(img + tp.o_ne), c = __ldg(img + tp.o_sw), e = __ldg(img + tp.o_se);
  float4 r;
  r.x = fmaf(e.x, tp.w_se, fmaf(c.x, tp.w_sw, fmaf(b.x, tp.w_ne, a.x * tp.w_nw)));
  r.y = fmaf(e.y, tp.w_se, fmaf(c.y, tp.w_sw, fmaf(b.y, tp.w_ne, a.y * tp.w_nw)));
  r.z = fmaf(e.z, tp.w_se, fmaf(c.z, tp.w_sw, fmaf(b.z, tp.w_ne, a.z * tp.w_nw)));
  r.w = fmaf(e.w, tp.w_se, fmaf(c.w, tp.w_sw, fmaf(b.w, tp.w_ne, a.w * tp.w_nw)));
  return r;
}

// Bilinear taps of source view v for the reference pixel with ray (r0, r1, r2) on the plane at depth dval: the
// homography of warping/homography.py:434-446 in the pinned rounding order. Shared by the forward warp and its
// backward, so the backward scatters to the forward's corners with the forward's weights, bit for bit.
__device__ __forceinline__ Tap2D warp_tap(const float* __restrict__ t1, const float* __restrict__ KR, int v, float r0,
                                          float r1, float r2, float dval, float cx, float cy, int w, int h) {
  const float* kr = KR + v * 9;
  const float t2x = dot3_chain(kr[0], kr[1], kr[2], r0, r1, r2);
  const float t2y = dot3_chain(kr[3], kr[4], kr[5], r0, r1, r2);
  const float t2z = dot3_chain(kr[6], kr[7], kr[8], r0, r1, r2);
  float ix, iy;
  plane_project(t1[v * 3], t1[v * 3 + 1], t1[v * 3 + 2], t2x, t2y, t2z, dval, cx, cy, (float)w, (float)h, ix, iy);
  return make_tap2d(ix, iy, w, h);
}

// MODE 0: out[v][c_off + c][d][pix]  (reference layout: list of V tensors C x D x h x w)
// MODE 1: out[d][pix][CK] with channels [v*3+c | ref rgb | bv_cur - bv_pred]  (K-Net input, NDHWC)
template <int MODE>
__global__ void __launch_bounds__(256)
warp_volume_kernel(const float4* __restrict__ imgs, int c_cnt, int c_off, int C_total,
                   const float* __restrict__ t1, const float* __restrict__ KR,
                   const float* __restrict__ rays, const float* __restrict__ dpl, int V, int D, int w, int h,
                   float cx, float cy, float* __restrict__ out, const float4* __restrict__ ref_img,
                   const float* __restrict__ bv_cur_hwd, const float* __restrict__ bv_pred_hwd, int CK) {
  const int hw = w * h;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)hw * D) return;
  const int pix = (int)(idx % hw);
  const int d = (int)(idx / hw);
  const float r0 = rays[pix], r1 = rays[hw + pix], r2 = rays[2 * hw + pix];
  const float dval = __ldg(dpl + d);
  float* o1 = nullptr;
  if (MODE == 1) o1 = out + ((size_t)d * hw + pix) * CK;
  for (int v = 0; v < V; ++v) {
    const Tap2D tp = warp_tap(t1, KR, v, r0, r1, r2, dval, cx, cy, w, h);
    float4 s = sample4(imgs + (size_t)v * hw, tp);
    const float sv[4] = {s.x, s.y, s.z, s.w};
    if (MODE == 0) {
      for (int c = 0; c < c_cnt; ++c)
        out[(((size_t)v * C_total + c_off + c) * D + d) * hw + pix] = sv[c];
    } else {
      o1[v * 3 + 0] = s.x; o1[v * 3 + 1] = s.y; o1[v * 3 + 2] = s.z;
    }
  }
  if (MODE == 1) {
    float4 r = __ldg(ref_img + pix);
    o1[3 * V + 0] = r.x; o1[3 * V + 1] = r.y; o1[3 * V + 2] = r.z;
    o1[3 * V + 3] = bv_cur_hwd[(size_t)pix * D + d] - bv_pred_hwd[(size_t)pix * D + d];
    for (int c = 3 * V + 4; c < CK; ++c) o1[c] = 0.f;
  }
}

// K-Net input rows, vectorised: one thread builds the whole channels-last row of its (plane, pixel) voxel in registers
// ([v*3+c warped src RGB | ref RGB | BV_cur - BV_predict | zero padding], models/KVNET.py:163-166) and stores it as
// full 16-byte vectors - each thread writes one contiguous 64 / 128-byte line instead of 16-32 scalar stores at a
// 128-byte stride - as fp32 (optional) and / or as the split-fp16 operand pair of the f16-pair convolution that
// consumes it (no fp32 volume, no split pass). CK4 = CK / 4 (4 or 8).
template <int CK4>
__global__ void __launch_bounds__(256)
knet_volume_rows_kernel(const float4* __restrict__ imgs, const float* __restrict__ t1, const float* __restrict__ KR,
                        const float* __restrict__ rays, const float* __restrict__ dpl, int V, int D, int w, int h,
                        float cx, float cy, const float4* __restrict__ ref_img, const float* __restrict__ bv_cur_hwd,
                        const float* __restrict__ bv_pred_hwd, float4* __restrict__ out, uint2* __restrict__ out_hi,
                        uint2* __restrict__ out_lo) {
  constexpr int CK = 4 * CK4;
  constexpr int MAXV = (CK - 4) / 3;
  const int hw = w * h;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)hw * D) return;
  const int pix = (int)(idx % hw);
  const int d = (int)(idx / hw);
  const float Wf = (float)w, Hf = (float)h;
  const float r0 = rays[pix], r1 = rays[hw + pix], r2 = rays[2 * hw + pix];
  const float dval = __ldg(dpl + d);
  float row[CK];
#pragma unroll
  for (int c = 0; c < CK; ++c) row[c] = 0.f;
#pragma unroll
  for (int v = 0; v < MAXV; ++v) {
    if (v < V) {
      const float* kr = KR + v * 9;
      const float t2x = dot3_chain(kr[0], kr[1], kr[2], r0, r1, r2);
      const float t2y = dot3_chain(kr[3], kr[4], kr[5], r0, r1, r2);
      const float t2z = dot3_chain(kr[6], kr[7], kr[8], r0, r1, r2);
      float ix, iy;
      plane_project(t1[v * 3], t1[v * 3 + 1], t1[v * 3 + 2], t2x, t2y, t2z, dval, cx, cy, Wf, Hf, ix, iy);
      const Tap2D tp = make_tap2d(ix, iy, w, h);
      const float4 sv = sample4(imgs + (size_t)v * hw, tp);
      row[v * 3 + 0] = sv.x; row[v * 3 + 1] = sv.y; row[v * 3 + 2] = sv.z;
    }
  }
  {
    const float4 r = __ldg(ref_img + pix);
    const float diff = bv_cur_hwd[(size_t)pix * D + d] - bv_pred_hwd[(size_t)pix * D + d];
    // the tail [ref rgb | diff] starts at channel 3 V (runtime): select instead of dynamic register indexing
#pragma unroll
    for (int c = 0; c < CK; ++c) {
      const int k = c - 3 * V;
      if (k == 0) row[c] = r.x; else if (k == 1) row[c] = r.y; else if (k == 2) row[c] = r.z; else if (k == 3) row[c] = diff;
    }
  }
  const size_t vox = (size_t)d * hw + pix;
  if (out) {
#pragma unroll
    for (int g = 0; g < CK4; ++g) out[vox * CK4 + g] = make_float4(row[4 * g], row[4 * g + 1], row[4 * g + 2], row[4 * g + 3]);
  }
  if (out_hi) {
#pragma unroll
    for (int g = 0; g < CK4; ++g) {
      uint2 hq, lq;
      nrgbd_split_pair4(row + 4 * g, hq, lq);
      out_hi[vox * CK4 + g] = hq; out_lo[vox * CK4 + g] = lq;
    }
  }
}

// Backward of MODE 0 (F.grid_sample's bilinear / zeros / align_corners=False input gradient, summed over the D
// planes): g_imgs[v][c][q] += grad_out[v][c][d][pix] * w_q for the in-range corners q of (d, pix). One thread per
// (plane, pixel) as in the forward; the corners are scattered with fp32 atomics, so the summation order is not fixed.
__global__ void __launch_bounds__(256)
warp_volume_backward_kernel(const float* __restrict__ grad_out, int C, const float* __restrict__ t1,
                            const float* __restrict__ KR, const float* __restrict__ rays, const float* __restrict__ dpl,
                            int V, int D, int w, int h, float cx, float cy, float* __restrict__ g_imgs) {
  const int hw = w * h;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)hw * D) return;
  const int pix = (int)(idx % hw);
  const int d = (int)(idx / hw);
  const float r0 = rays[pix], r1 = rays[hw + pix], r2 = rays[2 * hw + pix];
  const float dval = __ldg(dpl + d);
  for (int v = 0; v < V; ++v) {
    const Tap2D tp = warp_tap(t1, KR, v, r0, r1, r2, dval, cx, cy, w, h);
    const float wt[4] = {tp.w_nw, tp.w_ne, tp.w_sw, tp.w_se};
    const int off[4] = {tp.o_nw, tp.o_ne, tp.o_sw, tp.o_se};
    if (wt[0] == 0.f && wt[1] == 0.f && wt[2] == 0.f && wt[3] == 0.f) continue;
    const float* go = grad_out + ((size_t)v * C * D + d) * hw + pix;
    float* gi = g_imgs + (size_t)v * C * hw;
    for (int c = 0; c < C; ++c) {
      const float g = __ldg(go + (size_t)c * D * hw);
      if (g == 0.f) continue;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (wt[k] != 0.f) atomicAdd(gi + (size_t)c * hw + off[k], g * wt[k]);
    }
  }
}

__global__ void warp_setup_kernel(const float* __restrict__ K, const float* __restrict__ R,
                                  const float* __restrict__ t, int V, float* __restrict__ t1,
                                  float* __restrict__ KR) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const float* Rv = R + v * 9;
  const float* tv = t + v * 3;
  for (int i = 0; i < 3; ++i) {
    t1[v * 3 + i] = dot3_chain(K[i * 3 + 0], K[i * 3 + 1], K[i * 3 + 2], tv[0], tv[1], tv[2]);
    for (int j = 0; j < 3; ++j)
      KR[v * 9 + i * 3 + j] = dot3_chain(K[i * 3 + 0], K[i * 3 + 1], K[i * 3 + 2], Rv[j], Rv[3 + j], Rv[6 + j]);
  }
}

}  // namespace

extern "C" {

// imgs_packed: [V][hw][4] (channels c_off..c_off+c_cnt of each view, zero padded to 4)
// out: [V][C_total][D][hw]; ws: V*12 floats.
int nrgbd_warp_to_volume(const float* imgs_packed, int c_cnt, int c_off, int C_total, int V, int D, int h, int w,
                         const float* K, const float* R, const float* t, const float* rays,
                         const float* d_planes, float cx, float cy, float* ws, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(imgs_packed && K && R && t && rays && d_planes && ws && out, "null pointer");
  NRGBD_REQUIRE(V > 0 && D > 0 && h > 0 && w > 0, "empty problem");
  NRGBD_REQUIRE(c_cnt >= 1 && c_cnt <= 4 && c_off >= 0 && c_off + c_cnt <= C_total, "bad channel window");
  float* t1 = ws; float* KR = ws + 3 * V;
  warp_setup_kernel<<<ceil_div(V, 32), 32, 0, st>>>(K, R, t, V, t1, KR);
  long long n = (long long)h * w * D;
  warp_volume_kernel<0><<<ceil_div(n, 256), 256, 0, st>>>(reinterpret_cast<const float4*>(imgs_packed), c_cnt,
                                                          c_off, C_total, t1, KR, rays, d_planes, V, D, w, h, cx,
                                                          cy, out, nullptr, nullptr, nullptr, 0);
  NRGBD_COUNT(2);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Gradient of nrgbd_warp_to_volume with respect to the source images, all C channels at once.
// grad_out: [V][C][D][hw]; g_imgs: [V][C][hw], zeroed here before the scatter; ws: V*12 floats.
int nrgbd_warp_to_volume_backward(const float* grad_out, int C, int V, int D, int h, int w, const float* K,
                                  const float* R, const float* t, const float* rays, const float* d_planes, float cx,
                                  float cy, float* ws, float* g_imgs, cudaStream_t st) {
  NRGBD_REQUIRE(grad_out && K && R && t && rays && d_planes && ws && g_imgs, "null pointer");
  NRGBD_REQUIRE(C > 0 && V > 0 && D > 0 && h > 0 && w > 0, "empty problem");
  float* t1 = ws; float* KR = ws + 3 * V;
  warp_setup_kernel<<<ceil_div(V, 32), 32, 0, st>>>(K, R, t, V, t1, KR);
  NRGBD_CUDA_CHECK(cudaMemsetAsync(g_imgs, 0, sizeof(float) * (size_t)V * C * h * w, st));
  long long n = (long long)h * w * D;
  warp_volume_backward_kernel<<<ceil_div(n, 256), 256, 0, st>>>(grad_out, C, t1, KR, rays, d_planes, V, D, w, h, cx, cy,
                                                                g_imgs);
  NRGBD_COUNT(2);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// K-Net input volume [D][hw][CK], CK >= 3V+4 (models/KVNET.py:163-166), from the
// quarter-resolution RGB of the V sources ([V][hw][4]) and the reference ([hw][4]) and the two
// pixel-major log-DPVs.
int nrgbd_knet_input_volume(const float* src_rgb_packed, const float* ref_rgb_packed, const float* bv_cur_hwd,
                            const float* bv_pred_hwd, int V, int D, int h, int w, int CK, const float* K,
                            const float* R, const float* t, const float* rays, const float* d_planes, float cx,
                            float cy, float* ws, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(src_rgb_packed && ref_rgb_packed && bv_cur_hwd && bv_pred_hwd && K && R && t && rays &&
                    d_planes && ws && out, "null pointer");
  NRGBD_REQUIRE(V > 0 && D > 0 && h > 0 && w > 0 && CK >= 3 * V + 4, "bad shape");
  return nrgbd_knet_input_volume_pair(src_rgb_packed, ref_rgb_packed, bv_cur_hwd, bv_pred_hwd, V, D, h, w, CK, K, R, t, rays, d_planes, cx, cy,
                                     ws, out, nullptr, nullptr, st);
}

// Same volume, optionally (also / only) as the split-fp16 operand pair (out_hi, out_lo: half [D][hw][CK]) of the f16-pair
// convolution that consumes it; out may be NULL when the pair is requested.
int nrgbd_knet_input_volume_pair(const float* src_rgb_packed, const float* ref_rgb_packed, const float* bv_cur_hwd,
                                 const float* bv_pred_hwd, int V, int D, int h, int w, int CK, const float* K,
                                 const float* R, const float* t, const float* rays, const float* d_planes, float cx,
                                 float cy, float* ws, float* out, void* out_hi, void* out_lo, cudaStream_t st) {
  NRGBD_REQUIRE(src_rgb_packed && ref_rgb_packed && bv_cur_hwd && bv_pred_hwd && K && R && t && rays &&
                    d_planes && ws && (out || (out_hi && out_lo)), "null pointer");
  NRGBD_REQUIRE(V > 0 && D > 0 && h > 0 && w > 0 && CK >= 3 * V + 4 && (out_hi == nullptr) == (out_lo == nullptr), "bad shape");
  float* t1 = ws; float* KR = ws + 3 * V;
  warp_setup_kernel<<<ceil_div(V, 32), 32, 0, st>>>(K, R, t, V, t1, KR);
  long long n = (long long)h * w * D;
  const float4* si = reinterpret_cast<const float4*>(src_rgb_packed);
  const float4* ri = reinterpret_cast<const float4*>(ref_rgb_packed);
  if (CK == 16 || CK == 32) {
    if (CK == 16) knet_volume_rows_kernel<4><<<ceil_div(n, 256), 256, 0, st>>>(si, t1, KR, rays, d_planes, V, D, w, h, cx, cy, ri, bv_cur_hwd, bv_pred_hwd,
                                                                             reinterpret_cast<float4*>(out), reinterpret_cast<uint2*>(out_hi), reinterpret_cast<uint2*>(out_lo));
    else knet_volume_rows_kernel<8><<<ceil_div(n, 256), 256, 0, st>>>(si, t1, KR, rays, d_planes, V, D, w, h, cx, cy, ri, bv_cur_hwd, bv_pred_hwd,
                                                                    reinterpret_cast<float4*>(out), reinterpret_cast<uint2*>(out_hi), reinterpret_cast<uint2*>(out_lo));
  } else {
    NRGBD_REQUIRE(out && !out_hi, "the operand-pair output needs a channel stride of 16 or 32");
    warp_volume_kernel<1><<<ceil_div(n, 256), 256, 0, st>>>(si, 3, 0, 3, t1, KR, rays, d_planes, V, D, w, h, cx, cy, out, ri, bv_cur_hwd, bv_pred_hwd, CK);
  }
  NRGBD_COUNT(2);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
