// Geometry of the local bundle adjustment's depth-map back-warp, shared by the warp kernels (lba_warp.cu) and the fused
// pose optimiser (lba_opt.cu): the projection of a reference pixel into a source view and the chain from the sampling
// location's gradient (gix, giy) back to the pose (dL/dR, dL/dt).
#pragma once
#include "common.cuh"

struct LbaGeom {
  float ix, iy;        // un-normalised sampling location
  float X0, X1, X2;    // back-projected point
  float Px, Py, Pz;    // K (R X + t)
};

// Coordinate chain in the reference's op order (warping/homography.py:546-567): elementwise d * ray, 4x4 matmuls as sgemm
// FMA chains over k (the homogeneous 1 contributes fma(t, 1, acc) = acc + t; the zero last column of the 4x4 intrinsic
// matrix nothing), division by P_z WITHOUT an epsilon, (u - cx) / cx, ATen's un-normalisation.
__device__ __forceinline__ LbaGeom lba_project(float d, float r0, float r1, float r2, const float* __restrict__ R, const float* __restrict__ t,
                                               const float* __restrict__ K, float Wf, float Hf) {
  LbaGeom g;
  g.X0 = __fmul_rn(d, r0); g.X1 = __fmul_rn(d, r1); g.X2 = __fmul_rn(d, r2);
  const float c0 = __fadd_rn(dot3_chain(R[0], R[1], R[2], g.X0, g.X1, g.X2), t[0]);
  const float c1 = __fadd_rn(dot3_chain(R[3], R[4], R[5], g.X0, g.X1, g.X2), t[1]);
  const float c2 = __fadd_rn(dot3_chain(R[6], R[7], R[8], g.X0, g.X1, g.X2), t[2]);
  g.Px = dot3_chain(K[0], K[1], K[2], c0, c1, c2);
  g.Py = dot3_chain(K[3], K[4], K[5], c0, c1, c2);
  g.Pz = dot3_chain(K[6], K[7], K[8], c0, c1, c2);
  const float u = __fdiv_rn(g.Px, g.Pz), v = __fdiv_rn(g.Py, g.Pz);
  const float cx = K[2], cy = K[5];
  g.ix = unnormalize(__fdiv_rn(__fsub_rn(u, cx), cx), Wf);
  g.iy = unnormalize(__fdiv_rn(__fsub_rn(v, cy), cy), Hf);
  return g;
}

// ATen grid_sampler_2d_backward (bilinear, zeros): one channel's d out / d ix, d out / d iy for the output gradient gv, the
// four corner values (0 outside the image) and the corner distances ax = x1 - ix, bx = ix - x0, ay, by.
__device__ __forceinline__ void lba_grid_grad(float gv, float nw, float ne, float sw, float se, float ax, float bx, float ay, float by,
                                              float& gix, float& giy) {
  gix += gv * (-nw * ay + ne * ay - sw * by + se * by);
  giy += gv * (-nw * ax - ne * bx + sw * ax + se * bx);
}

// (gix, giy) -> acc[0..8] = dL/dR (row-major) and acc[9..11] = dL/dt of one pixel.
// ix = ((u - cx) / cx + 1) W / 2 - 1 / 2  ->  d ix / d u = W / (2 cx); u = Px / Pz; g_Xc = K^T g_P.
__device__ __forceinline__ void lba_pose_grad(const LbaGeom& g, float gix, float giy, const float* __restrict__ K, float Wf, float Hf,
                                              float* acc) {
  const float cx = K[2], cy = K[5];
  const float gu = gix * (Wf * 0.5f) / cx, gvv = giy * (Hf * 0.5f) / cy;
  const float iz = 1.f / g.Pz;
  const float gPx = gu * iz, gPy = gvv * iz, gPz = -(gu * g.Px + gvv * g.Py) * iz * iz;
  const float gc0 = K[0] * gPx + K[3] * gPy + K[6] * gPz;
  const float gc1 = K[1] * gPx + K[4] * gPy + K[7] * gPz;
  const float gc2 = K[2] * gPx + K[5] * gPy + K[8] * gPz;
  acc[0] = gc0 * g.X0; acc[1] = gc0 * g.X1; acc[2] = gc0 * g.X2;
  acc[3] = gc1 * g.X0; acc[4] = gc1 * g.X1; acc[5] = gc1 * g.X2;
  acc[6] = gc2 * g.X0; acc[7] = gc2 * g.X1; acc[8] = gc2 * g.X2;
  acc[9] = gc0; acc[10] = gc1; acc[11] = gc2;
}
