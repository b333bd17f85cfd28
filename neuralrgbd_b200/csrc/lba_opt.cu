// The local bundle adjustment's pose optimiser on the device (ICP/opt_pose_numerical.py:28-304, local_BA_direct(_parallel)).
//
// One launch is one Adam iteration over all views and pixels of one pyramid level. Every thread takes one (view, reference
// pixel): back-warp of the three source channels (lba_common.cuh), mask = (warped != 0), the confidence-weighted L1 residual
// and its sign, grid_sampler_2d_backward with respect to the sampling location, and the chain to dL/dR, dL/dt. Each block
// writes its 12 gradient partials and its |residual| sum (double) to its own workspace slot; the last block to finish (ticket
// counter) reduces the slots of every view in a fixed order, so the result is the same from run to run. That block then
// takes dL/dR through quaternion2Rotation and unitQ_to_quat to the unit-quaternion parameter u, applies torch.optim.Adam
// (the op order of torch 2.11's CPU step) to u and / or t, writes the rotation the next launch warps with, records the
// iteration's loss and re-arms the ticket. The iterations of a level are enqueued back to back; nothing returns to the host.
#include "lba_common.cuh"
#include "../../include/nrgbd.h"

#include <math.h>

namespace {

constexpr int kThreads = 256;
constexpr int kTerms = 13;                 // dL/dR (9), dL/dt (3), sum |residual|
constexpr int kMaxViews = 64;
constexpr size_t kTicketBytes = 256;       // workspace header: the ticket counter, then the block partials

// unitQ_to_quat then quaternion2Rotation (mutils/misc.py:459-471, :295-336), each torch op rounded in fp32 as the reference
// evaluates it: x**2 is x*x, 1/n is a reciprocal, 2*s*(...) is (2s)(...).
__device__ inline void unitq_to_rotation(const float* u, float* R) {
  const float x = u[0], y = u[1], z = u[2];
  const float a2 = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
  const float den = __fadd_rn(a2, 1.f);
  const float qw = __fdiv_rn(__fmul_rn(x, 2.f), den), qx = __fdiv_rn(__fmul_rn(y, 2.f), den);
  const float qy = __fdiv_rn(__fmul_rn(z, 2.f), den), qz = __fdiv_rn(__fsub_rn(1.f, a2), den);
  const float n = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(qw, qw), __fmul_rn(qx, qx)), __fmul_rn(qy, qy)), __fmul_rn(qz, qz));
  const float s2 = __fmul_rn(__fdiv_rn(1.f, n), 2.f);
  const float xx = __fmul_rn(qx, qx), yy = __fmul_rn(qy, qy), zz = __fmul_rn(qz, qz);
  R[0] = __fsub_rn(1.f, __fmul_rn(s2, __fadd_rn(yy, zz)));
  R[4] = __fsub_rn(1.f, __fmul_rn(s2, __fadd_rn(xx, zz)));
  R[8] = __fsub_rn(1.f, __fmul_rn(s2, __fadd_rn(xx, yy)));
  R[1] = __fmul_rn(__fsub_rn(__fmul_rn(qx, qy), __fmul_rn(qw, qz)), 2.f);
  R[3] = __fmul_rn(__fadd_rn(__fmul_rn(qx, qy), __fmul_rn(qw, qz)), 2.f);
  R[2] = __fmul_rn(__fadd_rn(__fmul_rn(qx, qz), __fmul_rn(qw, qy)), 2.f);
  R[6] = __fmul_rn(__fsub_rn(__fmul_rn(qx, qz), __fmul_rn(qw, qy)), 2.f);
  R[5] = __fmul_rn(__fsub_rn(__fmul_rn(qy, qz), __fmul_rn(qw, qx)), 2.f);
  R[7] = __fmul_rn(__fadd_rn(__fmul_rn(qy, qz), __fmul_rn(qw, qx)), 2.f);
}

// dL/du from dL/dR: quaternion2Rotation differentiated as written (s = 1 / |q|^2 included), then unitQ_to_quat.
__device__ inline void rotation_grad_to_unitq(const float* u, const double* G, double* gu) {
  const double x = u[0], y = u[1], z = u[2];
  const double a2 = x * x + y * y + z * z, D = 1.0 + a2;
  const double qw = 2.0 * x / D, qx = 2.0 * y / D, qy = 2.0 * z / D, qz = (1.0 - a2) / D;
  const double n = qw * qw + qx * qx + qy * qy + qz * qz, s = 1.0 / n;
  // diagonal: R_ii = 1 - 2 s B_i; A = sum_i G_ii B_i
  const double A = G[0] * (qy * qy + qz * qz) + G[4] * (qx * qx + qz * qz) + G[8] * (qx * qx + qy * qy);
  const double dA_x = 2.0 * qx * (G[4] + G[8]), dA_y = 2.0 * qy * (G[0] + G[8]), dA_z = 2.0 * qz * (G[0] + G[4]);
  // d(-2 s A)/dq_i = -2 (ds/dq_i A + s dA/dq_i), ds/dq_i = -2 q_i s^2
  const double ss = 2.0 * s * s;
  double gqx = -2.0 * (-qx * ss * A + s * dA_x), gqy = -2.0 * (-qy * ss * A + s * dA_y);
  double gqz = -2.0 * (-qz * ss * A + s * dA_z), gqw = -2.0 * (-qw * ss * A);
  // off-diagonal terms 2 (q_a q_b -+ q_w q_c)
  const double S01 = G[1] + G[3], D10 = G[3] - G[1], S02 = G[2] + G[6], D02 = G[2] - G[6], S12 = G[5] + G[7], D21 = G[7] - G[5];
  gqx += 2.0 * (qy * S01 + qz * S02 + qw * D21);
  gqy += 2.0 * (qx * S01 + qz * S12 + qw * D02);
  gqz += 2.0 * (qx * S02 + qy * S12 + qw * D10);
  gqw += 2.0 * (qz * D10 + qy * D02 + qx * D21);
  // (qw, qx, qy) = 2 (x, y, z) / D, qz = (1 - a2) / D
  const double P = gqw * x + gqx * y + gqy * z, c = 4.0 * (P + gqz) / (D * D);
  gu[0] = 2.0 * gqw / D - x * c;
  gu[1] = 2.0 * gqx / D - y * c;
  gu[2] = 2.0 * gqy / D - z * c;
}

// torch.optim.Adam (betas .9 / .999, eps 1e-8, no weight decay), one element, in the fp32 op order of torch 2.11's CPU step:
// exp_avg.lerp_(g, 1 - b1) = fma(w, g - m, m); exp_avg_sq.mul_(b2).addcmul_(g, g, 1 - b2) = fma((1 - b2) g, g, b2 v);
// denom = sqrt(v) / sqrt(bc2) + eps; p.addcdiv_(m, denom, -lr / bc1) = p + (-step m) / denom.
__device__ inline void adam_step(float* p, float* m, float* v, const float* g, int n, float neg_step, float bc2_sqrt) {
  const float w1 = (float)(1.0 - 0.9), b2 = (float)0.999, w2 = (float)(1.0 - 0.999), eps = (float)1e-8;
  for (int i = 0; i < n; ++i) {
    m[i] = __fmaf_rn(w1, __fsub_rn(g[i], m[i]), m[i]);
    v[i] = __fmaf_rn(__fmul_rn(w2, g[i]), g[i], __fmul_rn(v[i], b2));
    const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(v[i]), bc2_sqrt), eps);
    p[i] = __fadd_rn(p[i], __fdiv_rn(__fmul_rn(neg_step, m[i]), den));
  }
}

__global__ void __launch_bounds__(kThreads)
lba_opt_iter_kernel(const float* __restrict__ ref, const float* __restrict__ conf, const float* __restrict__ dmap,
                    const float* __restrict__ srcs, const float* __restrict__ K, const float* __restrict__ rays, int V, int H, int W,
                    int mode, double loss_scale, float neg_step, float bc2_sqrt, float* __restrict__ state,
                    double* __restrict__ losses, double* __restrict__ part, unsigned int* __restrict__ ticket) {
  const int hw = H * W, nblk = gridDim.x, n = blockIdx.y;
  const int p = blockIdx.x * kThreads + threadIdx.x;
  const float* S = state + n * NRGBD_LBA_STATE_FLOATS;
  float acc[kTerms];
#pragma unroll
  for (int i = 0; i < kTerms; ++i) acc[i] = 0.f;
  if (p < hw) {
    const float Wf = (float)W, Hf = (float)H;
    const LbaGeom g = lba_project(dmap[p], rays[p], rays[hw + p], rays[2 * hw + p], S + NRGBD_LBA_R, S + NRGBD_LBA_T, K, Wf, Hf);
    const bool bad = !(fabsf(g.ix) < 1.0e9f) || !(fabsf(g.iy) < 1.0e9f);
    const float cf = conf[p];
    if (!bad) {
      const float fx0 = floorf(g.ix), fy0 = floorf(g.iy);
      const int x0 = (int)fx0, y0 = (int)fy0, x1 = x0 + 1, y1 = y0 + 1;
      const float ax = __fsub_rn(__fadd_rn(fx0, 1.f), g.ix), bx = __fsub_rn(g.ix, fx0);
      const float ay = __fsub_rn(__fadd_rn(fy0, 1.f), g.iy), by = __fsub_rn(g.iy, fy0);
      const bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
      // ATen grid_sampler_2d forward weights (zero outside the image), summed nw, ne, sw, se as the warp kernel does
      const float w_nw = (vx0 && vy0) ? __fmul_rn(ax, ay) : 0.f, w_ne = (vx1 && vy0) ? __fmul_rn(bx, ay) : 0.f;
      const float w_sw = (vx0 && vy1) ? __fmul_rn(ax, by) : 0.f, w_se = (vx1 && vy1) ? __fmul_rn(bx, by) : 0.f;
      const float* src = srcs + (long long)n * 3 * hw;
      float gix = 0.f, giy = 0.f, l1 = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* s = src + (long long)c * hw;
        const float nw = (vx0 && vy0) ? __ldg(s + y0 * W + x0) : 0.f, ne = (vx1 && vy0) ? __ldg(s + y0 * W + x1) : 0.f;
        const float sw = (vx0 && vy1) ? __ldg(s + y1 * W + x0) : 0.f, se = (vx1 && vy1) ? __ldg(s + y1 * W + x1) : 0.f;
        float w = __fmul_rn(nw, w_nw);
        w = __fadd_rn(w, __fmul_rn(ne, w_ne));
        w = __fadd_rn(w, __fmul_rn(sw, w_sw));
        w = __fadd_rn(w, __fmul_rn(se, w_se));
        if (w != 0.f) {
          // |w * mask * conf - ref * mask * conf| with mask = 1; its gradient with respect to w is sign(residual) * conf
          const float r = __fsub_rn(__fmul_rn(w, cf), __fmul_rn(ref[(long long)c * hw + p], cf));
          l1 += fabsf(r);
          const float gv = r > 0.f ? cf : (r < 0.f ? -cf : 0.f);
          lba_grid_grad(gv, nw, ne, sw, se, ax, bx, ay, by, gix, giy);
        }
      }
      lba_pose_grad(g, gix, giy, K, Wf, Hf, acc);
      acc[12] = l1;
    }
  }
  // block partials of the 13 terms (double from the warp level on), one slot per (view, block): no atomics on the sums
  __shared__ double red[kThreads / 32][kTerms];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < kTerms; ++i) {
    double v = (double)acc[i];
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    if (lane == 0) red[wrp][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < kTerms) {
    double v = 0.0;
    for (int k = 0; k < kThreads / 32; ++k) v += red[k][threadIdx.x];
    part[((long long)n * nblk + blockIdx.x) * kTerms + threadIdx.x] = v;
    __threadfence();
  }
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == (unsigned)(nblk * V - 1);
  __syncthreads();
  if (!last) return;
  __threadfence();

  // ---- epilogue (last block): fixed-order reduction, chain rule, Adam ----
  __shared__ double sums[kMaxViews][kTerms];
  for (int j = wrp; j < V * kTerms; j += kThreads / 32) {
    const int vn = j / kTerms, i = j - vn * kTerms;
    double v = 0.0;
    for (int b = lane; b < nblk; b += 32) v += __ldcg(part + ((long long)vn * nblk + b) * kTerms + i);
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    if (lane == 0) sums[vn][i] = v;
  }
  __syncthreads();
  if (threadIdx.x < V) {
    const int vn = threadIdx.x;
    float* St = state + vn * NRGBD_LBA_STATE_FLOATS;
    double G[9], gu[3];
    for (int i = 0; i < 9; ++i) G[i] = sums[vn][i] * loss_scale;
    rotation_grad_to_unitq(St + NRGBD_LBA_U, G, gu);
    for (int i = 0; i < 3; ++i) {
      St[NRGBD_LBA_G_U + i] = (float)gu[i];
      St[NRGBD_LBA_G_T + i] = (float)(sums[vn][9 + i] * loss_scale);
    }
    if (mode & NRGBD_LBA_OPT_R) {
      adam_step(St + NRGBD_LBA_U, St + NRGBD_LBA_M_U, St + NRGBD_LBA_V_U, St + NRGBD_LBA_G_U, 3, neg_step, bc2_sqrt);
      unitq_to_rotation(St + NRGBD_LBA_U, St + NRGBD_LBA_R);
    }
    if (mode & NRGBD_LBA_OPT_T)
      adam_step(St + NRGBD_LBA_T, St + NRGBD_LBA_M_T, St + NRGBD_LBA_V_T, St + NRGBD_LBA_G_T, 3, neg_step, bc2_sqrt);
    losses[vn] = sums[vn][12];
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// F.avg_pool2d(x, k) (stride k, no padding, floor): fp32 sum over the window rows then columns, divided by k * k, as ATen does.
__global__ void lba_avgpool_kernel(const float* __restrict__ x, int N, int H, int W, int k, float* __restrict__ out) {
  const int h = H / k, w = W / k;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * h * w) return;
  const int ox = (int)(i % w), oy = (int)((i / w) % h);
  const long long nn = i / ((long long)w * h);
  const float* s = x + nn * H * W + (long long)oy * k * W + ox * k;
  float acc = 0.f;
  for (int dy = 0; dy < k; ++dy)
    for (int dx = 0; dx < k; ++dx) acc = __fadd_rn(acc, s[dy * W + dx]);
  out[i] = __fdiv_rn(acc, (float)(k * k));
}

long long partial_bytes(int V, int H, int W) { return (long long)V * ceil_div((long long)H * W, kThreads) * kTerms * sizeof(double); }

}  // namespace

extern "C" {

int nrgbd_lba_avgpool(const float* x, int N, int H, int W, int k, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(x && out && N > 0 && k > 0 && H >= k && W >= k, "bad arguments");
  const long long n = (long long)N * (H / k) * (W / k);
  lba_avgpool_kernel<<<ceil_div(n, 256), 256, 0, st>>>(x, N, H, W, k, out);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

long long nrgbd_lba_pose_opt_workspace_bytes(int V, int H, int W) {
  if (V <= 0 || H <= 0 || W <= 0) return -1;
  return (long long)kTicketBytes + partial_bytes(V, H, W);
}

int nrgbd_lba_pose_opt_scale(const float* ref, const float* conf, const float* dmap, const float* srcs, const float* K, const float* rays,
                             int V, int H, int W, int mode, double loss_scale, double lr, int first_step, int n_iter, float* state,
                             double* losses, void* ws, cudaStream_t st) {
  NRGBD_REQUIRE(ref && conf && dmap && srcs && K && rays && state && losses && ws, "null pointer");
  NRGBD_REQUIRE(V > 0 && V <= kMaxViews && H > 0 && W > 0 && first_step >= 0 && n_iter >= 0, "bad sizes");
  NRGBD_REQUIRE(mode >= 1 && mode <= 3, "mode must be NRGBD_LBA_OPT_R, NRGBD_LBA_OPT_T or both");
  unsigned int* ticket = (unsigned int*)ws;
  double* part = (double*)((char*)ws + kTicketBytes);
  if (n_iter == 0) return NRGBD_OK;
  NRGBD_CUDA_CHECK(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st));
  const dim3 grid(ceil_div((long long)H * W, kThreads), V);
  for (int it = 0; it < n_iter; ++it) {
    // Adam's bias corrections as Python doubles (torch 2.11 _single_tensor_adam), with the host's pow as Python uses it
    const double step = (double)(first_step + it + 1);
    const double bc1 = 1.0 - pow(0.9, step), bc2 = 1.0 - pow(0.999, step);
    const float neg_step = (float)(-(lr / bc1)), bc2_sqrt = (float)pow(bc2, 0.5);
    lba_opt_iter_kernel<<<grid, kThreads, 0, st>>>(ref, conf, dmap, srcs, K, rays, V, H, W, mode, loss_scale, neg_step, bc2_sqrt, state,
                                                   losses + (long long)it * V, part, ticket);
  }
  NRGBD_COUNT(n_iter);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
