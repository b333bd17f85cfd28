// Fused plane-sweep cost volume (SURVEY §8 a1-a3).
//
// Replaces warping/homography.py:293-331 (est_swp_volume_v4) + :421-448
// (_back_warp_homo_parallel) + :81-87 (img_dis_L2_pard / img_dis_L1_pard): for every
// reference pixel, depth plane and source view the homography is evaluated in
// registers, the four bilinear corners are gathered from a channel-last copy of the
// source features (one tap = one contiguous vector), the feature distance to the
// reference pixel is reduced across the lanes of a lane-group and accumulated over the
// views. No `repeat`, no grid tensor, no warped tensor: the D x C x h x w intermediates
// of the reference (329 MB per view at 640x480) never exist.
//
// Data layout (device, fp32):
//   wide  features  [hw][Cw]      Cw = 4 * G channels, one float4 per lane per pass
//   narrow features [hw][4]       the C % 4 remainder channels (RGB intensity for C=67)
//   cost            [hw][D]       pixel-major ("HWD"), so softmax over D is contiguous
// Work mapping: a lane-group of LANES threads owns one reference pixel and walks the
// planes in batches of LANES: lane l evaluates the homography of plane d0+l once and
// publishes the corner record through shared memory; all lanes then cooperate on each
// plane with 4 coalesced LDG.128 per tap set; a transposing shuffle-reduction leaves
// lane l with the total for plane d0+l. The narrow channels are handled plane-per-lane.
#include "common.cuh"
#include "../../include/nrgbd.h"

namespace {

struct __align__(16) TapRec {
  int o[4];
  float w[4];
};

template <bool L1>
__device__ __forceinline__ float dist4(float4 a, float4 r, float acc) {
  float dx = a.x - r.x, dy = a.y - r.y, dz = a.z - r.z, dw = a.w - r.w;
  if (L1) {
    acc += fabsf(dx); acc += fabsf(dy); acc += fabsf(dz); acc += fabsf(dw);
  } else {
    acc = fmaf(dx, dx, acc); acc = fmaf(dy, dy, acc); acc = fmaf(dz, dz, acc); acc = fmaf(dw, dw, acc);
  }
  return acc;
}

__device__ __forceinline__ float4 bilerp4(float4 a, float4 b, float4 c, float4 d, const float* w) {
  float4 r;
  r.x = fmaf(d.x, w[3], fmaf(c.x, w[2], fmaf(b.x, w[1], a.x * w[0])));
  r.y = fmaf(d.y, w[3], fmaf(c.y, w[2], fmaf(b.y, w[1], a.y * w[0])));
  r.z = fmaf(d.z, w[3], fmaf(c.z, w[2], fmaf(b.z, w[1], a.z * w[0])));
  r.w = fmaf(d.w, w[3], fmaf(c.w, w[2], fmaf(b.w, w[1], a.w * w[0])));
  return r;
}

// term1 = K.t, KR = K.R for every view (homography.py:315-317), sgemm FMA-chain order.
__global__ void sweep_setup_kernel(const float* __restrict__ K, const float* __restrict__ R,
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

template <int LANES, int PASSES, bool L1>
__global__ void __launch_bounds__(256)
plane_sweep_kernel(const float4* __restrict__ ref_w, const float4* __restrict__ src_w, int G,
                   const float4* __restrict__ ref_n, const float4* __restrict__ src_n,
                   const float* __restrict__ t1, const float* __restrict__ KR,
                   const float* __restrict__ rays, const float* __restrict__ dpl, int V, int D, int w,
                   int h, float cx, float cy, float sigma, float* __restrict__ cost) {
  constexpr int GROUPS_PER_BLOCK = 256 / LANES;
  __shared__ TapRec recs[LANES > 1 ? 256 : 1];
  const int hw = w * h;
  const int lane = threadIdx.x % LANES;
  const int grp = threadIdx.x / LANES;
  int pix = blockIdx.x * GROUPS_PER_BLOCK + grp;
  const bool live = pix < hw;
  if (!live) pix = hw - 1;                       // keep the group converged; results discarded
  const float Wf = (float)w, Hf = (float)h;
  const float r0 = rays[pix], r1 = rays[hw + pix], r2 = rays[2 * hw + pix];

  float4 refw[PASSES > 0 ? PASSES : 1];
#pragma unroll
  for (int p = 0; p < PASSES; ++p) {
    int g = lane + p * LANES;
    refw[p] = (g < G) ? __ldg(ref_w + (size_t)pix * G + g) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float4 refn = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ref_n) refn = __ldg(ref_n + pix);
  TapRec* myrecs = recs + grp * LANES;

  for (int d0 = 0; d0 < D; d0 += LANES) {
    const int dmine = min(d0 + lane, D - 1);
    const float dval = __ldg(dpl + dmine);
    float cost_l = 0.f;
    for (int v = 0; v < V; ++v) {
      const float* kr = KR + v * 9;
      const float t2x = dot3_chain(kr[0], kr[1], kr[2], r0, r1, r2);
      const float t2y = dot3_chain(kr[3], kr[4], kr[5], r0, r1, r2);
      const float t2z = dot3_chain(kr[6], kr[7], kr[8], r0, r1, r2);
      float ix, iy;
      plane_project(t1[v * 3], t1[v * 3 + 1], t1[v * 3 + 2], t2x, t2y, t2z, dval, cx, cy, Wf, Hf, ix, iy);
      Tap2D tp = make_tap2d(ix, iy, w, h);
      float wt[4] = {tp.w_nw, tp.w_ne, tp.w_sw, tp.w_se};
      // narrow channels: this lane's own plane
      float dn = 0.f;
      if (src_n) {
        const float4* sn = src_n + (size_t)v * hw;
        float4 a = __ldg(sn + tp.o_nw), b = __ldg(sn + tp.o_ne), c = __ldg(sn + tp.o_sw), e = __ldg(sn + tp.o_se);
        dn = dist4<L1>(bilerp4(a, b, c, e, wt), refn, 0.f);
      }
      float dist = dn;
      if (PASSES > 0) {
        const float4* sw = src_w + (size_t)v * hw * G;
        if (LANES == 1) {
          float acc = 0.f;
#pragma unroll
          for (int p = 0; p < PASSES; ++p) {
            if (p < G) {
              float4 a = __ldg(sw + (size_t)tp.o_nw * G + p), b = __ldg(sw + (size_t)tp.o_ne * G + p);
              float4 c = __ldg(sw + (size_t)tp.o_sw * G + p), e = __ldg(sw + (size_t)tp.o_se * G + p);
              acc = dist4<L1>(bilerp4(a, b, c, e, wt), refw[p], acc);
            }
          }
          dist += acc;
        } else {
          __syncwarp();
          myrecs[lane].o[0] = tp.o_nw; myrecs[lane].o[1] = tp.o_ne;
          myrecs[lane].o[2] = tp.o_sw; myrecs[lane].o[3] = tp.o_se;
          myrecs[lane].w[0] = wt[0]; myrecs[lane].w[1] = wt[1];
          myrecs[lane].w[2] = wt[2]; myrecs[lane].w[3] = wt[3];
          __syncwarp();
          float part[LANES];
#pragma unroll
          for (int j = 0; j < LANES; ++j) {
            const int4 o = *reinterpret_cast<const int4*>(myrecs[j].o);
            const float4 wq = *reinterpret_cast<const float4*>(myrecs[j].w);
            const float wj[4] = {wq.x, wq.y, wq.z, wq.w};
            float acc = 0.f;
#pragma unroll
            for (int p = 0; p < PASSES; ++p) {
              int g = lane + p * LANES;
              if (g < G) {
                float4 a = __ldg(sw + (size_t)o.x * G + g), b = __ldg(sw + (size_t)o.y * G + g);
                float4 c = __ldg(sw + (size_t)o.z * G + g), e = __ldg(sw + (size_t)o.w * G + g);
                acc = dist4<L1>(bilerp4(a, b, c, e, wj), refw[p], acc);
              }
            }
            part[j] = acc;
          }
          // transposing reduction: afterwards lane l holds sum over lanes of part[l]
#pragma unroll
          for (int s = LANES / 2; s >= 1; s >>= 1) {
            const bool upper = (lane & s) != 0;
#pragma unroll
            for (int j = 0; j < s; ++j) {
              float keep = upper ? part[j + s] : part[j];
              float send = upper ? part[j] : part[j + s];
              part[j] = keep + __shfl_xor_sync(0xffffffffu, send, s, 32);
            }
          }
          dist += part[0];
        }
      }
      cost_l = __fadd_rn(cost_l, __fdiv_rn(dist, sigma));   // costV += dist / sigma  (homography.py:325)
    }
    if (live && d0 + lane < D) cost[(size_t)pix * D + d0 + lane] = cost_l;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Second-generation kernel (C >= 64 wide channels, D <= 256): corner vectors are kept in REGISTERS across planes.
//
// The kernel above re-fetches, for every (pixel, plane, view), its four 268-byte corner vectors - an L1 traffic of many GB
// for 30.9 MB of algorithmic bytes at 640x480x64x4 - although, along
// the epipolar line of one pixel, consecutive planes mostly hit the SAME corners (uniform depth planes: beyond the first
// ~20 of 64 planes the total disparity change is about one texel) or the neighbouring column. Here the view loop is the
// outer one and each lane keeps the four corner float4s of its channel slice from plane to plane: a plane whose (clamped)
// corner offsets equal the previous plane's loads nothing, a one-texel step along x loads two corners instead of four.
// The interpolation / distance / reduction arithmetic and its order are unchanged, so costs are bit-identical to the
// kernel above. The per-plane totals stay in registers (lane l of the 16-lane group owns planes l, 16 + l, ...), and the
// epilogue either stores the raw cost (est_swp_volume_v4 mirror) or finishes the D-Net head in place:
// BV = log_softmax(-cost) (models/basic.py:299-300), expected depth sum exp(BV) d and confidence max exp(BV).
// ---------------------------------------------------------------------------------------------------------------
// LANES threads per reference pixel (each PASSES float4 channel slices), NB = ceil(D / LANES) plane batches. With 8 lanes
// and two slices per lane (64 channels) the per-plane overhead - corner record, reuse test, reduction, loop - is spread over
// twice the arithmetic of the 16-lane form.
template <int LANES, int PASSES, bool L1, int NB, int BT, int MINB>
__global__ void __launch_bounds__(BT, MINB)
plane_sweep2_kernel(const float4* __restrict__ ref_w, const float4* __restrict__ src_w, int G,
                    const float4* __restrict__ ref_n, const float4* __restrict__ src_n,
                    const float* __restrict__ t1, const float* __restrict__ KR,
                    const float* __restrict__ rays, const float* __restrict__ dpl, int V, int D, int w,
                    int h, float cx, float cy, float sigma, float* __restrict__ cost, float* __restrict__ bv,
                    float* __restrict__ depth, float* __restrict__ conf) {
  constexpr int GROUPS_PER_BLOCK = BT / LANES;
  __shared__ TapRec recs[BT];
  // per-plane totals: thread t owns s_tot[b][t] (plane LANES b + lane of its pixel). Kept in shared memory so that the batch
  // loop can stay ROLLED: fully unrolled over the NB batches the kernel was instruction-fetch bound (ncu: 2.5 "no
  // instruction" stall cycles per issue with ~80 KB of code)
  __shared__ float s_tot[NB][BT];
  const int hw = w * h;
  const int lane = threadIdx.x % LANES;
  const int grp = threadIdx.x / LANES;
  int pix = blockIdx.x * GROUPS_PER_BLOCK + grp;
  const bool live = pix < hw;
  if (!live) pix = hw - 1;                       // keep the group converged; results discarded
  const float Wf = (float)w, Hf = (float)h;
  const float r0 = rays[pix], r1 = rays[hw + pix], r2 = rays[2 * hw + pix];
  float4 refw[PASSES];
#pragma unroll
  for (int p = 0; p < PASSES; ++p) {
    int g = lane + p * LANES;
    refw[p] = (g < G) ? __ldg(ref_w + (size_t)pix * G + g) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float4 refn = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ref_n) refn = __ldg(ref_n + pix);
  TapRec* myrecs = recs + grp * LANES;
#pragma unroll
  for (int b = 0; b < NB; ++b) s_tot[b][threadIdx.x] = 0.f;

  for (int v = 0; v < V; ++v) {
    const float* kr = KR + v * 9;
    const float t2x = dot3_chain(kr[0], kr[1], kr[2], r0, r1, r2);
    const float t2y = dot3_chain(kr[3], kr[4], kr[5], r0, r1, r2);
    const float t2z = dot3_chain(kr[6], kr[7], kr[8], r0, r1, r2);
    const float t1x = t1[v * 3], t1y = t1[v * 3 + 1], t1z = t1[v * 3 + 2];
    const float4* sw = src_w + (size_t)v * hw * G;
    const float4* sn = src_n ? src_n + (size_t)v * hw : nullptr;
    // corner vectors of the previous plane (this lane's channel slice of every pass) and their offsets
    float4 ca[PASSES], cb[PASSES], cc[PASSES], ce[PASSES];
    int4 po = make_int4(-1, -1, -1, -1);
#pragma unroll 1
    for (int b = 0; b < NB; ++b) {
      const int d0 = b * LANES;
      if (d0 < D) {
        const int dmine = min(d0 + lane, D - 1);
        const float dval = __ldg(dpl + dmine);
        float ix, iy;
        plane_project(t1x, t1y, t1z, t2x, t2y, t2z, dval, cx, cy, Wf, Hf, ix, iy);
        Tap2D tp = make_tap2d(ix, iy, w, h);
        float wt[4] = {tp.w_nw, tp.w_ne, tp.w_sw, tp.w_se};
        float dn = 0.f;                                     // narrow channels: this lane's own plane
        if (sn) {
          float4 a = __ldg(sn + tp.o_nw), bq = __ldg(sn + tp.o_ne), c = __ldg(sn + tp.o_sw), e = __ldg(sn + tp.o_se);
          dn = dist4<L1>(bilerp4(a, bq, c, e, wt), refn, 0.f);
        }
        __syncwarp();
        myrecs[lane].o[0] = tp.o_nw; myrecs[lane].o[1] = tp.o_ne; myrecs[lane].o[2] = tp.o_sw; myrecs[lane].o[3] = tp.o_se;
        myrecs[lane].w[0] = wt[0]; myrecs[lane].w[1] = wt[1]; myrecs[lane].w[2] = wt[2]; myrecs[lane].w[3] = wt[3];
        __syncwarp();
        float part[LANES];
#pragma unroll
        for (int j = 0; j < LANES; ++j) {
          const int4 o = *reinterpret_cast<const int4*>(myrecs[j].o);
          const float4 wq = *reinterpret_cast<const float4*>(myrecs[j].w);
          const float wj[4] = {wq.x, wq.y, wq.z, wq.w};
          // group-uniform decisions (every lane reads the same record)
          const bool same = o.x == po.x && o.y == po.y && o.z == po.z && o.w == po.w;
          if (!same) {
            const bool step_x = o.x == po.y && o.z == po.w;          // one texel to the right: west corners = old east corners
#pragma unroll
            for (int p = 0; p < PASSES; ++p) {
              const int g = lane + p * LANES;
              if (g < G) {
                if (step_x) { ca[p] = cb[p]; cc[p] = ce[p]; }
                else { ca[p] = __ldg(sw + (size_t)o.x * G + g); cc[p] = __ldg(sw + (size_t)o.z * G + g); }
                cb[p] = __ldg(sw + (size_t)o.y * G + g); ce[p] = __ldg(sw + (size_t)o.w * G + g);
              }
            }
            po = o;
          }
          float acc = 0.f;
#pragma unroll
          for (int p = 0; p < PASSES; ++p) {
            const int g = lane + p * LANES;
            if (g < G) acc = dist4<L1>(bilerp4(ca[p], cb[p], cc[p], ce[p], wj), refw[p], acc);
          }
          part[j] = acc;
        }
        // transposing reduction: afterwards lane l holds the sum over lanes of part[l]
#pragma unroll
        for (int s = LANES / 2; s >= 1; s >>= 1) {
          const bool upper = (lane & s) != 0;
#pragma unroll
          for (int j = 0; j < s; ++j) {
            float keep = upper ? part[j + s] : part[j];
            float send = upper ? part[j] : part[j + s];
            part[j] = keep + __shfl_xor_sync(0xffffffffu, send, s, 32);
          }
        }
        const float dist = dn + part[0];
        s_tot[b][threadIdx.x] = __fadd_rn(s_tot[b][threadIdx.x], __fdiv_rn(dist, sigma));   // costV += dist / sigma  (homography.py:325)
      }
    }
  }
  // ---- epilogue ----
  float tot[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) tot[b] = s_tot[b][threadIdx.x];
  if (cost) {
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const int d = b * LANES + lane;
      if (live && d < D) cost[(size_t)pix * D + d] = tot[b];
    }
  }
  if (bv || depth || conf) {
    // BV = log_softmax(-cost) over the D planes of this pixel: max / sum over the 16-lane group
    float m = -INFINITY;
#pragma unroll
    for (int b = 0; b < NB; ++b) if (b * LANES + lane < D) m = fmaxf(m, -tot[b]);
#pragma unroll
    for (int s = LANES / 2; s >= 1; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s, 32));
    float se = 0.f;
#pragma unroll
    for (int b = 0; b < NB; ++b) if (b * LANES + lane < D) se += expf(-tot[b] - m);
#pragma unroll
    for (int s = LANES / 2; s >= 1; s >>= 1) se += __shfl_xor_sync(0xffffffffu, se, s, 32);
    const float ls = logf(se);
    float dep = 0.f, cf = 0.f;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const int d = b * LANES + lane;
      if (d < D) {
        const float o = (-tot[b] - m) - ls;
        if (bv && live) bv[(size_t)pix * D + d] = o;
        const float pr = expf(o);
        dep += pr * __ldg(dpl + d); cf = fmaxf(cf, pr);
      }
    }
#pragma unroll
    for (int s = LANES / 2; s >= 1; s >>= 1) { dep += __shfl_xor_sync(0xffffffffu, dep, s, 32); cf = fmaxf(cf, __shfl_xor_sync(0xffffffffu, cf, s, 32)); }
    if (live && lane == 0) { if (depth) depth[pix] = dep; if (conf) conf[pix] = cf; }
  }
}

template <bool L1>
int launch_sweep2(int G, int D, int hw, cudaStream_t st, const float4* ref_w, const float4* src_w, const float4* ref_n,
                  const float4* src_n, const float* t1, const float* KR, const float* rays, const float* dpl, int V, int w, int h, float cx,
                  float cy, float sigma, float* cost, float* bv, float* depth, float* conf) {
#define NRGBD_SWEEP2_V(LN, P, NBV, BTV, MB)                                                                                          \
  plane_sweep2_kernel<LN, P, L1, NBV, BTV, MB><<<ceil_div((long long)hw * LN, BTV), BTV, 0, st>>>(ref_w, src_w, G, ref_n, src_n, t1, KR, \
                                                                                        rays, dpl, V, D, w, h, cx, cy, sigma, cost, bv, depth, conf)
// 128-thread blocks with a 6-resident-block register target (80 registers, no spills); without the target ptxas takes 144
// registers for this kernel and a block of it fills an SM on its own
#define NRGBD_SWEEP2(LN, P, NBV) NRGBD_SWEEP2_V(LN, P, NBV, 128, 6)
  if (G == 16 && (long long)hw * D >= (8ll << 20)) {      // 64 wide channels, large volumes: 8 lanes x 2 slices (half the per-pixel set-up per
                                                           // plane; at small volumes the lower occupancy costs more than that saves)
    const int nb = (D + 7) / 8;
    if (nb <= 4) NRGBD_SWEEP2(8, 2, 4); else if (nb <= 8) NRGBD_SWEEP2(8, 2, 8); else if (nb <= 16) NRGBD_SWEEP2(8, 2, 16); else NRGBD_SWEEP2(8, 2, 32);
    return NRGBD_OK;
  }
  const int passes = ceil_div(G, 16);  // 16 lanes
  const int nb = (D + 15) / 16;
  if (passes == 1) {
    if (nb <= 2) NRGBD_SWEEP2(16, 1, 2); else if (nb <= 4) NRGBD_SWEEP2(16, 1, 4); else if (nb <= 8) NRGBD_SWEEP2(16, 1, 8); else NRGBD_SWEEP2(16, 1, 16);
  } else if (passes == 2) {
    if (nb <= 2) NRGBD_SWEEP2(16, 2, 2); else if (nb <= 4) NRGBD_SWEEP2(16, 2, 4); else if (nb <= 8) NRGBD_SWEEP2(16, 2, 8); else NRGBD_SWEEP2(16, 2, 16);
  } else {
    return NRGBD_ERR_UNSUPPORTED;
  }
#undef NRGBD_SWEEP2
#undef NRGBD_SWEEP2_V
  return NRGBD_OK;
}

// [C][hw] (NCHW plane-major) -> wide [hw][Cw] (+ zero pad) and narrow [hw][4]
__global__ void pack_features_kernel(const float* __restrict__ in, int C, int hw, int Cw_src, int Cw,
                                     float* __restrict__ wide, float* __restrict__ narrow) {
  // tile transpose through shared memory: 32 pixels x 32 channels
  __shared__ float tile[32][33];
  int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  int Ct = Cw + 4;   // virtual channel space: [0,Cw) wide, [Cw, Cw+4) narrow
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    float v = 0.f;
    if (p < hw && c < Ct) {
      int csrc = (c < Cw) ? (c < Cw_src ? c : -1) : (Cw_src + (c - Cw) < C ? Cw_src + (c - Cw) : -1);
      if (csrc >= 0) v = in[(size_t)csrc * hw + p];
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    if (p < hw && c < Ct) {
      float v = tile[threadIdx.x][i];
      if (c < Cw) { if (wide) wide[(size_t)p * Cw + c] = v; }
      else if (narrow) narrow[(size_t)p * 4 + (c - Cw)] = v;
    }
  }
}

// out[b][a] = in[a][b]  (rows A, cols B)
__global__ void transpose2d_kernel(const float* __restrict__ in, int A, int B, float* __restrict__ out) {
  __shared__ float tile[32][33];
  int a0 = blockIdx.y * 32, b0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int a = a0 + i, b = b0 + threadIdx.x;
    if (a < A && b < B) tile[i][threadIdx.x] = in[(size_t)a * B + b];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int b = b0 + i, a = a0 + threadIdx.x;
    if (a < A && b < B) out[(size_t)b * A + a] = tile[threadIdx.x][i];
  }
}

template <int LANES, bool L1>
int launch_sweep_p(int passes, dim3 grid, cudaStream_t st, const float4* ref_w, const float4* src_w, int G,
                   const float4* ref_n, const float4* src_n, const float* t1, const float* KR,
                   const float* rays, const float* dpl, int V, int D, int w, int h, float cx, float cy,
                   float sigma, float* cost) {
#define NRGBD_SWEEP_CASE(P)                                                                           \
  case P:                                                                                             \
    plane_sweep_kernel<LANES, P, L1><<<grid, 256, 0, st>>>(ref_w, src_w, G, ref_n, src_n, t1, KR,     \
                                                           rays, dpl, V, D, w, h, cx, cy, sigma, cost); \
    break;
  switch (passes) {
    NRGBD_SWEEP_CASE(0)
    NRGBD_SWEEP_CASE(1)
    NRGBD_SWEEP_CASE(2)
    NRGBD_SWEEP_CASE(4)
    default: return NRGBD_ERR_UNSUPPORTED;
  }
#undef NRGBD_SWEEP_CASE
  return NRGBD_OK;
}

}  // namespace

extern "C" {

int nrgbd_sweep_workspace_floats(int V) { return V * 12; }

// Channel split used by the sweep: C = Cw + Cn with Cw % 4 == 0 and Cn = C % 4.
void nrgbd_sweep_channel_split(int C, int* Cw, int* Cn) {
  *Cn = C % 4;
  *Cw = C - *Cn;
}

int nrgbd_pack_features(const float* nchw, int C, int hw, int n_img, float* wide, float* narrow,
                        cudaStream_t st) {
  NRGBD_REQUIRE(nchw && C > 0 && hw > 0 && n_img > 0, "bad arguments");
  int Cw, Cn;
  nrgbd_sweep_channel_split(C, &Cw, &Cn);
  NRGBD_REQUIRE((Cw == 0 || wide) && (Cn == 0 || narrow), "missing output buffer");
  dim3 blk(32, 8), grid(ceil_div(hw, 32), ceil_div(Cw + 4, 32));
  for (int n = 0; n < n_img; ++n) {
    pack_features_kernel<<<grid, blk, 0, st>>>(nchw + (size_t)n * C * hw, C, hw, Cw, Cw,
                                               Cw ? wide + (size_t)n * hw * Cw : nullptr,
                                               Cn ? narrow + (size_t)n * hw * 4 : nullptr);
  }
  NRGBD_COUNT(n_img);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_transpose2d(const float* in, int A, int B, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(in && out && A > 0 && B > 0, "bad arguments");
  dim3 blk(32, 8), grid(ceil_div(B, 32), ceil_div(A, 32));
  transpose2d_kernel<<<grid, blk, 0, st>>>(in, A, B, out);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

static int sweep_impl(const float* ref_wide, const float* ref_narrow, const float* src_wide, const float* src_narrow, int Cw, int Cn,
                      int V, int D, int h, int w, const float* K, const float* R, const float* t, const float* rays,
                      const float* d_planes, float cx, float cy, float sigma, int metric, float* ws, float* cost_hwd, float* bv_hwd,
                      float* depth, float* conf, cudaStream_t st) {
  NRGBD_REQUIRE(V > 0 && D > 0 && h > 0 && w > 0, "empty problem");
  NRGBD_REQUIRE(Cw % 4 == 0 && Cn >= 0 && Cn <= 4 && Cw + Cn > 0, "bad channel split");
  NRGBD_REQUIRE((Cw == 0 || (ref_wide && src_wide)) && (Cn == 0 || (ref_narrow && src_narrow)), "null features");
  NRGBD_REQUIRE(K && R && t && rays && d_planes && ws && (cost_hwd || bv_hwd || depth || conf), "null pointer");
  if (metric != 0 && metric != 1) {
    nrgbd_set_error("undefined metric for feature distance ...");   // homography.py:329
    return NRGBD_ERR_BAD_ARG;
  }
  float* t1 = ws;
  float* KR = ws + 3 * V;
  sweep_setup_kernel<<<ceil_div(V, 32), 32, 0, st>>>(K, R, t, V, t1, KR);
  const int G = Cw / 4;
  const int hw = h * w;
  const float4* rw = reinterpret_cast<const float4*>(ref_wide);
  const float4* sw = reinterpret_cast<const float4*>(src_wide);
  const float4* rn = Cn ? reinterpret_cast<const float4*>(ref_narrow) : nullptr;
  const float4* sn = Cn ? reinterpret_cast<const float4*>(src_narrow) : nullptr;
  const bool fused_head = bv_hwd || depth || conf;
  if (G >= 16 && G <= 32 && D <= 256) {
    // register-cached corners (plane_sweep2_kernel), optional fused D-Net head
    int rc = metric == 0 ? launch_sweep2<false>(G, D, hw, st, rw, sw, rn, sn, t1, KR, rays, d_planes, V, w, h, cx, cy, sigma, cost_hwd, bv_hwd, depth, conf)
                         : launch_sweep2<true>(G, D, hw, st, rw, sw, rn, sn, t1, KR, rays, d_planes, V, w, h, cx, cy, sigma, cost_hwd, bv_hwd, depth, conf);
    if (rc == NRGBD_OK) { NRGBD_COUNT(2); NRGBD_LAUNCH_CHECK(); return NRGBD_OK; }
  }
  NRGBD_REQUIRE(cost_hwd || !fused_head, "this channel configuration needs a cost buffer (the fused head runs as a second pass)");
  // lane-group width: the widest power of two (<=16) that keeps every lane busy in pass 0
  int lanes = 1;
  if (G >= 16) lanes = 16; else if (G >= 4) lanes = 4;
  int passes = G == 0 ? 0 : ceil_div(G, lanes);
  if (passes == 3) passes = 4;
  if (passes > 4) { nrgbd_set_error("plane sweep supports at most 256 wide channels per call"); return NRGBD_ERR_UNSUPPORTED; }
  dim3 grid(ceil_div((long long)hw * lanes, 256));
  int rc;
#define NRGBD_SWEEP_LANES(L)                                                                               \
  rc = metric == 0 ? launch_sweep_p<L, false>(passes, grid, st, rw, sw, G, rn, sn, t1, KR, rays, d_planes, V, \
                                              D, w, h, cx, cy, sigma, cost_hwd)                            \
                   : launch_sweep_p<L, true>(passes, grid, st, rw, sw, G, rn, sn, t1, KR, rays, d_planes, V,  \
                                             D, w, h, cx, cy, sigma, cost_hwd);
  if (lanes == 16) { NRGBD_SWEEP_LANES(16) } else if (lanes == 4) { NRGBD_SWEEP_LANES(4) } else { NRGBD_SWEEP_LANES(1) }
#undef NRGBD_SWEEP_LANES
  if (rc != NRGBD_OK) { nrgbd_set_error("plane sweep: unsupported channel configuration"); return rc; }
  NRGBD_COUNT(2);
  NRGBD_LAUNCH_CHECK();
  if (fused_head) return nrgbd_dpv_normalize(cost_hwd, 1, D, nullptr, 0, 0, -1.f, hw, D, bv_hwd, 1, D, d_planes, depth, conf, (nrgbd_stream_t)st);
  return NRGBD_OK;
}

// Cost volume from packed (channel-last) features. cost is [h*w][D].
// ws: V*12 floats of device scratch (term1, K.R).
int nrgbd_plane_sweep_cost_packed(const float* ref_wide, const float* ref_narrow, const float* src_wide,
                                  const float* src_narrow, int Cw, int Cn, int V, int D, int h, int w,
                                  const float* K, const float* R, const float* t, const float* rays,
                                  const float* d_planes, float cx, float cy, float sigma, int metric,
                                  float* ws, float* cost_hwd, cudaStream_t st) {
  NRGBD_REQUIRE(cost_hwd, "null pointer");
  return sweep_impl(ref_wide, ref_narrow, src_wide, src_narrow, Cw, Cn, V, D, h, w, K, R, t, rays, d_planes, cx, cy, sigma, metric, ws,
                    cost_hwd, nullptr, nullptr, nullptr, st);
}

// The whole D-Net head after the feature CNN in one kernel (models/basic.py:270-300): plane-sweep cost, then
// BV = log_softmax(-cost) [h*w][D] (pixel-major), expected depth sum exp(BV) d and confidence max exp(BV) (any of the three
// may be NULL); the cost volume itself is written only when cost_hwd is given.
int nrgbd_plane_sweep_dpv_packed(const float* ref_wide, const float* ref_narrow, const float* src_wide,
                                 const float* src_narrow, int Cw, int Cn, int V, int D, int h, int w,
                                 const float* K, const float* R, const float* t, const float* rays,
                                 const float* d_planes, float cx, float cy, float sigma, int metric,
                                 float* ws, float* cost_hwd, float* bv_hwd, float* depth, float* conf, cudaStream_t st) {
  return sweep_impl(ref_wide, ref_narrow, src_wide, src_narrow, Cw, Cn, V, D, h, w, K, R, t, rays, d_planes, cx, cy, sigma, metric, ws,
                    cost_hwd, bv_hwd, depth, conf, st);
}

}  // extern "C"
