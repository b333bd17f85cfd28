// Tensor-core convolution: wgmma implicit GEMM on SPLIT operand pairs with a shared-memory HALO tile
// (SURVEY §8 a5, a8, a10; DESIGN.md §4.4). Hopper (sm_90a): TMA + mbarrier pipeline, wgmma from shared memory,
// fp32 accumulators in registers.
//
// Arithmetic. Every fp32 operand is carried as two parts. Split-fp16 pairs (the default path, this file's entry points):
// a = hi + lo * 2^-11 with hi = RN_f16(a) and lo = RN_f16((a - hi) * 2^11) (a - hi is exact in fp32; the 2^11 scale keeps
// the residual out of the fp16 subnormal range). 3xTF32 pairs (conv_tc.cu): a = hi + lo, both TF32. A product is
// accumulated as
//     main  += a_hi * b_hi                       cross += a_hi * b_lo + a_lo * b_hi          out = main + scale * cross
// (dropped term ~2^-22 |a b|). Activations are produced in pair form by the previous pass (nrgbd_split_f16_pair or the
// fused BatchNorm pass), so both operands go TMA -> shared memory -> tensor core.
//
// Halo tile. One (TH + 2p) x (TW + 2p) pixel halo box per (depth tap, 32-channel chunk) is staged once and all in-plane
// taps read it through shifted wgmma descriptors: the output tile is TH x TW = 16 x 8 or 8 x 16 pixels, and each
// warpgroup's 64 GEMM rows are 8 core-matrix groups of 8 pixels that are each a piece of one tile row (16 x 8: rows
// [8 cw, 8 cw + 8); 8 x 16: columns [8 cw, 8 cw + 8) of all 8 rows, a start offset of 8 pixels). A tap (dy, dx) is a
// start-address offset of (dy * pitch + dx) pixel rows and the stride-byte-offset between groups is the halo pitch
// (pitch * row bytes, not a multiple of the swizzle atom: the swizzle is a function of the absolute shared-memory
// address, as is TMA's, so any 16-byte-aligned row offset stays consistent). A 3x3 convolution reads its input tile 1.4x
// instead of 9x. Strided convolutions use one box per tap ("tap mode"). The launch takes the orientation that pads fewer
// output positions: 8 x 16 divides the 120-row planes of the 1/4-resolution layers, 16 x 8 leaves a 1/16 ragged row.
//
// Roles (persistent CTAs over 128-pixel x BN-channel tiles, grid.y = Cout chunks of BN <= 128 channels):
//   warps 0-7   two consumer warpgroups, 64 pixels each: per K step and tap, wgmma a_hi x b_hi -> main, a_hi x b_lo and
//               a_lo x b_hi -> cross; the ring slots of step s are released once step s + 1 is issued and step s has
//               retired (wgmma.wait_group 1), the last step's at the end of the tile; then the epilogue straight from the
//               registers: main + scale * cross, bias / LeakyReLU, fp32 or fp16-pair stores, BatchNorm column sums
//               (summed per CTA over its tiles, then one pair of fp64 atomics per column and CTA). The affine form (AFF,
//               eval-mode BatchNorm with fixed coefficients) applies per-channel scale / shift, an optional residual and
//               ReLU instead, and accumulates nothing: no atomics, the same output on every run.
//               (a_hi x [b_hi | b_lo] as one wgmma of N = 2 BN would read a_hi once, but its accumulators overlap those of
//               a_lo x b_hi in part, and ptxas then serialises every wgmma (C7511): 8-15 % slower on H100.)
//   warp 8      TMA producer: halo / tap box of the hi and the lo activation planes into the A ring, G taps of the hi and
//               lo K-major weight tiles into the B ring; expect-tx mbarriers. It runs on into the next tile's stages, so
//               that tile's first loads overlap this tile's last steps and epilogue.
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "conv_wgmma.cuh"
#include "wgmma.cuh"
#include "../../include/nrgbd_dev.h"

namespace {

constexpr int WG_THREADS = 288;        // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int BKC = 32;                // input channels per K chunk

struct WgParams {
  float* y; const float* bias; double* stats;
  __half *y_hi, *y_lo;
  const float *aff_scale, *aff_shift, *res;   // affine epilogue (AFF instantiations only)
  const __half *res_hi, *res_lo;
  int relu;
  int N, Dz, Hy, Wx, tiles_x, tiles_y, n_tiles, wide;   // wide: 8 x 16 output tile (else 16 x 8)
  int cin_chunks, n_kz, n_tap, halo, in_stride, org_y, org_x;
  int Cout, c_first;                     // logical output channels; first channel of this launch's chunk 0
  int Dout, Hout, Wout, Cs_out, c_off, out_stride, out_off_y, out_off_x, leaky;
  int stages_a, stages_b, box_w, box_h;  // ring depths; activation box in pixels (halo pitch x halo rows, or the tile)
  uint32_t a_tile_bytes, a_stage_bytes, a_tx_bytes, b_stage_bytes, wg_row16;   // wg_row16: second warpgroup's A offset, 16-byte units
  uint32_t a_desc_hi, b_desc_hi;         // high words of the shared-memory descriptors (SBO, swizzle mode)
  signed char dz[3];
  signed char dy[WG_MAX_TAP2D], dx[WG_MAX_TAP2D];
  unsigned short a_off16[WG_MAX_TAP2D];  // halo mode: offset of the tap inside the halo tile, 16-byte units
  unsigned char wsel[3 * WG_MAX_TAP2D];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Bounded spin: a protocol bug becomes a trap (an error the caller sees) instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
#pragma unroll 1
  for (uint32_t it = 0; it < (1u << 27); ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return;
  }
  __trap();
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"((uint64_t)tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"((uint64_t)tm), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// K-major shared-memory matrix descriptor: start address >> 4 [0,14), LBO >> 4 [16,30) (unused when swizzled: 1),
// SBO >> 4 [32,46), swizzle mode [62,64) (1: 128 B, 2: 64 B); the high word is precomputed on the host.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t hi) {
  return ((uint64_t)hi << 32) | (uint64_t)(((saddr & 0x3FFFFu) >> 4) | (1u << 16));
}

template <int BN, bool TF32>
__device__ __forceinline__ void wg_mma(float* d, uint64_t a, uint64_t b) {
  if constexpr (TF32) Wgmma<BN>::tf32(d, a, b); else Wgmma<BN>::f16(d, a, b);
}

// BN: output channels per CTA (16..128). TF32: operand kind. G: in-plane taps per pipeline step (one weight box and one
// barrier round trip per G taps). AFF: affine epilogue (see WgConv).
template <int BN, bool TF32, int G, bool AFF>
__global__ void __launch_bounds__(WG_THREADS, BN <= 64 ? 2 : 1)
conv_wg_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
               const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo, const WgParams p) {
  constexpr int RB = TF32 ? 128 : 64;                 // bytes of one 32-channel pixel row
  constexpr int KS = TF32 ? 4 : 2;                    // MMA K slices per 32-channel chunk (32 bytes each)
  constexpr float SCALE = TF32 ? 1.f : 1.f / 2048.f;
  constexpr uint32_t B_HALF = (uint32_t)(G * BN * RB);
  constexpr int NJ = BN / 8;                          // 8-column accumulator blocks
  // shared memory: [A ring: stages_a x (hi | lo)][B ring: stages_b x (hi G taps | lo G taps)][column sums 8 x 2 x BN floats]
  //                [CTA column sums 2 x BN doubles][barriers]
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = smem_u32(smem_raw);
  if (base & 1023u) __trap();
  const uint32_t b_ring = base + (uint32_t)p.stages_a * p.a_stage_bytes;
  const uint32_t sums_off = (uint32_t)p.stages_a * p.a_stage_bytes + (uint32_t)p.stages_b * p.b_stage_bytes;
  float* part = reinterpret_cast<float*>(smem_raw + sums_off);
  double* cta_sums = reinterpret_cast<double*>(smem_raw + sums_off + 8u * 2u * BN * 4u);
  const uint32_t bars = base + sums_off + 8u * 2u * BN * 4u + 2u * BN * 8u;
  const uint32_t bar_afull = bars, bar_aempty = bars + 64, bar_bfull = bars + 128, bar_bempty = bars + 192;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages_a; ++s) { mbar_init(bar_afull + 8 * s, 1); mbar_init(bar_aempty + 8 * s, 8); }
    for (int s = 0; s < p.stages_b; ++s) { mbar_init(bar_bfull + 8 * s, 1); mbar_init(bar_bempty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < 2 * BN) cta_sums[threadIdx.x] = 0.0;
  if constexpr (AFF) {
    // the affine form keeps no column sums: the partial-sum area holds this CTA's scale [BN] | shift [BN] instead
    const int c0 = p.c_first + (int)blockIdx.y * BN, t = threadIdx.x % BN;
    if (threadIdx.x < 2 * BN) part[threadIdx.x] = c0 + t < p.Cout ? __ldg((threadIdx.x < BN ? p.aff_scale : p.aff_shift) + c0 + t) : 0.f;
  }
  __syncthreads();

  // Persistent CTAs: tiles blockIdx.x, blockIdx.x + gridDim.x, ... The rings and their phases run on across tiles, so
  // the producer loads the next tile's first stages while the consumers run this tile's epilogue.
  const int th = p.wide ? 8 : 16, tw = p.wide ? 16 : 8;
  const int cbase = p.c_first + (int)blockIdx.y * BN;
  const int n_steps = p.n_kz * p.cin_chunks * (p.n_tap / G);

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      int sa = 0, sb = 0;
      uint32_t pha = 0, phb = 0;
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        int t = tile;
        const int ox0 = (t % p.tiles_x) * tw; t /= p.tiles_x;
        const int oy0 = (t % p.tiles_y) * th; t /= p.tiles_y;
        const int z0 = t % p.Dz, n0 = t / p.Dz;
        for (int kz = 0; kz < p.n_kz; ++kz) {
          const int cz = z0 + p.dz[kz];
          for (int cc = 0; cc < p.cin_chunks; ++cc) {
            for (int tap = 0; tap < p.n_tap; tap += G) {
              if (!p.halo || tap == 0) {
                const int cx = ox0 * p.in_stride + (p.halo ? p.org_x : (int)p.dx[tap]);
                const int cy = oy0 * p.in_stride + (p.halo ? p.org_y : (int)p.dy[tap]);
                mbar_wait(bar_aempty + 8 * sa, pha ^ 1u);
                mbar_expect_tx(bar_afull + 8 * sa, p.a_tx_bytes);
                const uint32_t dst = base + (uint32_t)sa * p.a_stage_bytes;
                tma_load_5d(dst, &tm_a_hi, bar_afull + 8 * sa, cc * BKC, cx, cy, cz, n0);
                tma_load_5d(dst + p.a_tile_bytes, &tm_a_lo, bar_afull + 8 * sa, cc * BKC, cx, cy, cz, n0);
                if (++sa == p.stages_a) { sa = 0; pha ^= 1u; }
              }
              mbar_wait(bar_bempty + 8 * sb, phb ^ 1u);
              mbar_expect_tx(bar_bfull + 8 * sb, 2 * B_HALF);
              const uint32_t dst = b_ring + (uint32_t)sb * p.b_stage_bytes;
              const int ws = p.wsel[kz * p.n_tap + tap];
              tma_load_3d(dst, &tm_b_hi, bar_bfull + 8 * sb, cc * BKC, cbase, ws);
              tma_load_3d(dst + B_HALF, &tm_b_lo, bar_bfull + 8 * sb, cc * BKC, cbase, ws);
              if (++sb == p.stages_b) { sb = 0; phb ^= 1u; }
            }
          }
        }
      }
    }
    return;
  }

  // ===== consumers: 64 GEMM rows per warpgroup; 16x8 tile: cw owns tile rows [8 cw, 8 cw + 8), 8x16 tile: columns
  // [8 cw, 8 cw + 8) of all 8 rows. Either way core-matrix group g is one tile row, one halo pitch down. =====
  const int cw = warp >> 2, w4 = warp & 3;
  float acc_m[BN / 2], acc_c[BN / 2];
  const uint32_t wg_off = (uint32_t)cw * p.wg_row16 * 16u;
  int sa = 0, sb = 0, sa_cur = 0, tap = 0;
  uint32_t pha = 0, phb = 0;
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
#pragma unroll
    for (int k = 0; k < BN / 2; ++k) { acc_m[k] = 0.f; acc_c[k] = 0.f; }
    int rel_a = -1, rel_b = -1;                       // slots of the previous step, released once it has retired
    for (int step = 0; step < n_steps; ++step) {
      const bool new_a = !p.halo || tap == 0;
      if (new_a) {
        mbar_wait(bar_afull + 8 * sa, pha);
        sa_cur = sa;
        if (++sa == p.stages_a) { sa = 0; pha ^= 1u; }
      }
      mbar_wait(bar_bfull + 8 * sb, phb);
      const uint32_t a_hi = base + (uint32_t)sa_cur * p.a_stage_bytes + wg_off;
      const uint32_t b_hi = b_ring + (uint32_t)sb * p.b_stage_bytes;
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const uint32_t ao = a_hi + (p.halo ? (uint32_t)p.a_off16[tap + g] * 16u : 0u);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          const uint32_t ah = ao + 32u * ks, al = ah + p.a_tile_bytes;
          const uint32_t bh = b_hi + (uint32_t)(g * BN * RB) + 32u * ks, bl = bh + B_HALF;
          wg_mma<BN, TF32>(acc_m, wg_desc(ah, p.a_desc_hi), wg_desc(bh, p.b_desc_hi));
          wg_mma<BN, TF32>(acc_c, wg_desc(ah, p.a_desc_hi), wg_desc(bl, p.b_desc_hi));
          wg_mma<BN, TF32>(acc_c, wg_desc(al, p.a_desc_hi), wg_desc(bh, p.b_desc_hi));
        }
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
      if (lane == 0) {
        if (rel_b >= 0) mbar_arrive(bar_bempty + 8 * rel_b);
        if (rel_a >= 0) mbar_arrive(bar_aempty + 8 * rel_a);
      }
      tap += G;
      const bool last_of_a = !p.halo || tap == p.n_tap;
      if (tap == p.n_tap) tap = 0;
      rel_b = sb; rel_a = last_of_a ? sa_cur : -1;
      if (++sb == p.stages_b) { sb = 0; phb ^= 1u; }
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    // the last step's slots: the producer may already be waiting on them for the next tile
    if (lane == 0) {
      mbar_arrive(bar_bempty + 8 * rel_b);
      mbar_arrive(bar_aempty + 8 * rel_a);
    }

    // ===== epilogue from the accumulator registers (its indices are computed here, not held through the K loop) =====
    int t = tile;
    const int ox0 = (t % p.tiles_x) * tw; t /= p.tiles_x;
    const int oy0 = (t % p.tiles_y) * th; t /= p.tiles_y;
    const int z0 = t % p.Dz, n0 = t / p.Dz;
    const int n_here = min(BN, p.Cout - cbase);
    const bool pair = p.y_hi != nullptr;
    const bool vec2 = ((p.Cs_out | (p.c_off + cbase)) & 1) == 0;
    float* dst_row[2] = {nullptr, nullptr};
    long long pix[2] = {0, 0};
    bool valid[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 16 * w4 + (lane >> 2) + 8 * i;    // GEMM row within the warpgroup: tile row r / 8, column r % 8
      const int iy = oy0 + (r >> 3) + (p.wide ? 0 : 8 * cw), ix = ox0 + (r & 7) + (p.wide ? 8 * cw : 0);
      valid[i] = iy < p.Hy && ix < p.Wx;
      const int oy = iy * p.out_stride + p.out_off_y, ox = ix * p.out_stride + p.out_off_x;
      pix[i] = (((long long)n0 * p.Dout + z0) * p.Hout + oy) * p.Wout + ox;
      if (!pair) dst_row[i] = p.y + pix[i] * (long long)p.Cs_out + p.c_off + cbase;
    }
    if constexpr (AFF) {
      // main + scale * cross for every column first: the cross accumulators die here, which leaves registers for the
      // residual loads of the store loop (no spills at BN = 64)
#pragma unroll
      for (int k = 0; k < BN / 2; ++k) acc_m[k] = fmaf(acc_c[k], SCALE, acc_m[k]);
    }
    constexpr int NJ_PAIR = ((BN + 31) / 32) * 4;     // pair output: pad channels up to the next 32 are stored as zeros
    const int nj_store = pair ? NJ_PAIR : NJ;
#pragma unroll
    for (int j = 0; j < NJ_PAIR; ++j) {
      if (j >= nj_store) break;
      const int c = 8 * j + 2 * (lane & 3);
      float v[2][2];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float f = 0.f;
          if (j < NJ && c + e < n_here && valid[i]) {
            if constexpr (AFF) {
              f = fmaf(acc_m[4 * j + 2 * i + e], part[c + e], part[BN + c + e]);      // residual and ReLU: in the store loop below
            } else {
              f = fmaf(acc_c[4 * j + 2 * i + e], SCALE, acc_m[4 * j + 2 * i + e]);
              if (p.bias) f += __ldg(p.bias + cbase + c + e);
              if (p.leaky) f = f >= 0.f ? f : f * 0.01f;
            }
          }
          v[i][e] = f;
        }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!valid[i]) continue;
        if constexpr (AFF) {
          // residual (the output's layout: the pair output has c_off 0, so o is also the store offset), then ReLU
          const long long o = pix[i] * (long long)p.Cs_out + p.c_off + cbase + c;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (j < NJ && c + e < n_here) {
              if (p.res) v[i][e] += __ldg(p.res + o + e);
              else if (p.res_hi) v[i][e] += fmaf(__half2float(p.res_lo[o + e]), 1.f / 2048.f, __half2float(p.res_hi[o + e]));
              if (p.relu) v[i][e] = fmaxf(v[i][e], 0.f);
            }
          }
        }
        if (pair) {
          __half h0, l0, h1, l1;
          nrgbd_split_pair(v[i][0], h0, l0); nrgbd_split_pair(v[i][1], h1, l1);
          const long long o = pix[i] * (long long)p.Cs_out + cbase + c;
          *reinterpret_cast<__half2*>(p.y_hi + o) = __halves2half2(h0, h1);
          *reinterpret_cast<__half2*>(p.y_lo + o) = __halves2half2(l0, l1);
        } else if (vec2 && c + 1 < n_here) {
          *reinterpret_cast<float2*>(dst_row[i] + c) = make_float2(v[i][0], v[i][1]);
        } else {
          if (c < n_here) dst_row[i][c] = v[i][0];
          if (c + 1 < n_here) dst_row[i][c + 1] = v[i][1];
        }
      }
      if (!AFF && p.stats && j < NJ) {
        // column sums over this warp's 16 rows: the thread's two rows, then across the 8 lane quads
        float s1[2], s2[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          s1[e] = v[0][e] + v[1][e];
          s2[e] = fmaf(v[0][e], v[0][e], v[1][e] * v[1][e]);
#pragma unroll
          for (int m = 4; m < 32; m <<= 1) {
            s1[e] += __shfl_xor_sync(0xffffffffu, s1[e], m);
            s2[e] += __shfl_xor_sync(0xffffffffu, s2[e], m);
          }
        }
        if (lane < 4) {
#pragma unroll
          for (int e = 0; e < 2; ++e) { part[(warp * 2) * BN + c + e] = s1[e]; part[(warp * 2 + 1) * BN + c + e] = s2[e]; }
        }
      }
    }
    if (!AFF && p.stats) {
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const int c = threadIdx.x;
      if (c < n_here) {
        double a1 = 0.0, a2 = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { a1 += (double)part[(w * 2) * BN + c]; a2 += (double)part[(w * 2 + 1) * BN + c]; }
        cta_sums[c] += a1; cta_sums[BN + c] += a2;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");   // the next tile overwrites the partial sums
    }
  }
  const int c = threadIdx.x;
  if (!AFF && p.stats && c < min(BN, p.Cout - cbase) && (int)blockIdx.x < p.n_tiles) {
    atomicAdd(p.stats + cbase + c, cta_sums[c]);
    atomicAdd(p.stats + p.Cout + cbase + c, cta_sums[BN + c]);
  }
}

int g_h2_smem_cap_kb = 0;   // development: cap on the dynamic shared memory per CTA (0 = chosen by the plan below)
int g_h2_flags = 0;         // development knobs (nrgbd_dev_conv_h2_set_flags), all off in production:
                            //   4 one box per tap (no halo tile)   8 always the 16 x 8 output tile
                            //   32 one tile per CTA (no persistent CTAs)   128 one tap per pipeline step

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// Encoded maps are memoised per thread (the engine's pool hands out the same blocks every frame).
struct MapKey { const void* p; long long a; int b, c, d, e, f, g, h, i; };
struct MapEnt { MapKey k; CUtensorMap m; };
inline bool same_key(const MapKey& x, const MapKey& y) {
  return x.p == y.p && x.a == y.a && x.b == y.b && x.c == y.c && x.d == y.d && x.e == y.e && x.f == y.f && x.g == y.g && x.h == y.h && x.i == y.i;
}
thread_local MapEnt g_maps[1024];
inline unsigned key_slot(const MapKey& k) {
  unsigned long long h = (unsigned long long)k.p * 0x9E3779B97F4A7C15ull;
  h ^= (unsigned long long)(k.a * 73856093ll) ^ (unsigned long long)(k.b * 19349663u) ^ (unsigned long long)(k.c * 83492791u) ^
       (unsigned long long)(k.d * 2654435761u) ^ (unsigned long long)(k.e * 40503u) ^ (unsigned long long)(k.f * 2246822519u) ^
       (unsigned long long)(k.g * 3266489917u) ^ (unsigned long long)(k.h * 668265263u) ^ (unsigned long long)(k.i * 374761393u);
  return (unsigned)(h >> 40) & 1023u;
}

// 5-D map over a channels-last tensor [N][D][H][W][Cs] of `esize`-byte elements; box [32][box_w (after stride)][box_h]
int encode_act_map(CUtensorMap* tm, const void* x, int esize, int N, int D, int H, int W, int C, int Cs, int box_w, int box_h, int stride) {
  MapKey k{x, (long long)N * 8 + esize, D, H, W, C, Cs, box_w, box_h, stride};
  MapEnt& e = g_maps[key_slot(k)];
  if (same_key(e.k, k) && e.k.p) { *tm = e.m; return NRGBD_OK; }
  EncodeTiledFn enc = get_encode();
  if (!enc) { nrgbd_set_error("cuTensorMapEncodeTiled unavailable"); return NRGBD_ERR_CUDA; }
  cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)D, (cuuint64_t)N};
  cuuint64_t strides[4] = {(cuuint64_t)Cs * esize, (cuuint64_t)W * Cs * esize, (cuuint64_t)H * W * Cs * esize, (cuuint64_t)D * H * W * Cs * esize};
  cuuint32_t box[5] = {(cuuint32_t)BKC, (cuuint32_t)(box_w * stride), (cuuint32_t)(box_h * stride), 1, 1};
  cuuint32_t estr[5] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1, 1};
  CUresult r = enc(tm, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<void*>(x), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, esize == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { nrgbd_set_error("cuTensorMapEncodeTiled(activation, esize %d) failed: %d", esize, (int)r); return NRGBD_ERR_CUDA; }
  e.k = k; e.m = *tm;
  return NRGBD_OK;
}

// 3-D map over one half of the packed weights: [taps (tap_stride elements apart)][Cout_pad][Cin_pad]; box [32][BN][G]
int encode_w_map(CUtensorMap* tm, const void* w, int esize, long long tap_stride, int taps, int Cout_pad, int Cin_pad, int BN, int G) {
  MapKey k{w, tap_stride * 8 + esize, taps, Cout_pad, Cin_pad, BN, G, -7, -7, -7};
  MapEnt& e = g_maps[key_slot(k)];
  if (same_key(e.k, k) && e.k.p) { *tm = e.m; return NRGBD_OK; }
  EncodeTiledFn enc = get_encode();
  if (!enc) { nrgbd_set_error("cuTensorMapEncodeTiled unavailable"); return NRGBD_ERR_CUDA; }
  cuuint64_t dims[3] = {(cuuint64_t)Cin_pad, (cuuint64_t)Cout_pad, (cuuint64_t)taps};
  cuuint64_t strides[2] = {(cuuint64_t)Cin_pad * esize, (cuuint64_t)tap_stride * esize};
  cuuint32_t box[3] = {(cuuint32_t)BKC, (cuuint32_t)BN, (cuuint32_t)G};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(w), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, esize == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { nrgbd_set_error("cuTensorMapEncodeTiled(weights, esize %d) failed: %d", esize, (int)r); return NRGBD_ERR_CUDA; }
  e.k = k; e.m = *tm;
  return NRGBD_OK;
}

inline uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }

typedef void (*WgKernel)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const WgParams);

template <bool TF32, int G, bool AFF = false>
WgKernel pick_kernel(int BN) {
  switch (BN) {
    case 16: return conv_wg_kernel<16, TF32, G, AFF>;
    case 32: return conv_wg_kernel<32, TF32, G, AFF>;
    case 48: return conv_wg_kernel<48, TF32, G, AFF>;
    case 64: return conv_wg_kernel<64, TF32, G, AFF>;
    case 80: return conv_wg_kernel<80, TF32, G, AFF>;
    case 96: return conv_wg_kernel<96, TF32, G, AFF>;
    case 112: return conv_wg_kernel<112, TF32, G, AFF>;
    case 128: return conv_wg_kernel<128, TF32, G, AFF>;
  }
  return nullptr;
}

// One launch: output channels [c_first, c_first + n_chunks * BN) in chunks of BN.
int launch_chunks(const WgConv& c, WgParams p, int BN, int n_chunks, int c_first, cudaStream_t st) {
  const bool tf32 = c.tf32 != 0;
  const int esize = tf32 ? 4 : 2, RB = BKC * esize;
  p.c_first = c_first;
  // taps per pipeline step: a whole kernel row when the weight slices of the taps are consecutive (plain convolutions)
  int G = 1;
  if (p.halo && p.n_tap % 3 == 0 && !(g_h2_flags & 128)) {
    bool consecutive = true;
    for (int t = 1; t < p.n_kz * p.n_tap; ++t) consecutive = consecutive && c.wsel[t] == c.wsel[t - 1] + 1;
    if (consecutive) G = 3;
  }
  // shared memory: two CTAs per SM when BN <= 64 and two A + two B stages fit half of the SM's 228 KB
  const size_t extra = (size_t)8 * 2 * BN * 4 + (size_t)2 * BN * 8 + 256;
  auto plan = [&](size_t cap, int g, int& sa, int& sb) {
    const size_t b_stage = (size_t)2 * g * BN * RB;
    sa = 2;
    if (cap < extra + 2 * (size_t)p.a_stage_bytes + 2 * b_stage) return false;
    sb = (int)((cap - extra - 2 * (size_t)p.a_stage_bytes) / b_stage);
    if (sb > 8) sb = 8;
    if (sb >= 6 && cap >= extra + 3 * (size_t)p.a_stage_bytes + 4 * b_stage) { sa = 3; sb = (int)((cap - extra - 3 * (size_t)p.a_stage_bytes) / b_stage); if (sb > 8) sb = 8; }
    return true;
  };
  size_t cap = g_h2_smem_cap_kb > 0 ? (size_t)g_h2_smem_cap_kb * 1024 : (BN <= 64 ? 115712 - 1024 : 232448);
  int sa = 0, sb = 0;
  bool ok = plan(cap, G, sa, sb);
  if (!ok && G == 3) { G = 1; ok = plan(cap, G, sa, sb); }
  if (!ok) { cap = 232448; ok = plan(cap, G, sa, sb); }
  if (!ok) { nrgbd_set_error("conv_wgmma: tile does not fit the shared-memory pipeline"); return NRGBD_ERR_UNSUPPORTED; }
  p.stages_a = sa; p.stages_b = sb;
  p.b_stage_bytes = (uint32_t)(2 * G * BN * RB);
  const size_t smem = (size_t)sa * p.a_stage_bytes + (size_t)sb * p.b_stage_bytes + extra;
  CUtensorMap tb_hi, tb_lo;
  int rc = encode_w_map(&tb_hi, c.w_hi, esize, c.w_tap_stride, c.n_wslices, c.Cout_pad, c.Cin_pad, BN, G);
  if (rc == NRGBD_OK) rc = encode_w_map(&tb_lo, c.w_lo, esize, c.w_tap_stride, c.n_wslices, c.Cout_pad, c.Cin_pad, BN, G);
  if (rc != NRGBD_OK) return rc;
  CUtensorMap ta_hi, ta_lo;
  rc = encode_act_map(&ta_hi, c.x_hi, esize, c.N, c.Din, c.Hin, c.Win, c.Cin_pad, c.Cs_in, p.box_w, p.box_h, p.in_stride);
  if (rc == NRGBD_OK) rc = encode_act_map(&ta_lo, c.x_lo, esize, c.N, c.Din, c.Hin, c.Win, c.Cin_pad, c.Cs_in, p.box_w, p.box_h, p.in_stride);
  if (rc != NRGBD_OK) return rc;
  const bool aff = p.aff_scale != nullptr;
  if (aff && tf32) { nrgbd_set_error("conv_wgmma: the affine epilogue is built for split-fp16 operands only"); return NRGBD_ERR_UNSUPPORTED; }
  WgKernel fn = aff ? (G == 3 ? pick_kernel<false, 3, true>(BN) : pick_kernel<false, 1, true>(BN))
                    : tf32 ? (G == 3 ? pick_kernel<true, 3>(BN) : pick_kernel<true, 1>(BN))
                           : (G == 3 ? pick_kernel<false, 3>(BN) : pick_kernel<false, 1>(BN));
  if (!fn) { nrgbd_set_error("conv_wgmma: unsupported chunk width %d", BN); return NRGBD_ERR_UNSUPPORTED; }
  static size_t configured[2][2][2][8] = {};
  size_t& conf = configured[aff][tf32][G == 3][BN / 16 - 1];
  if (smem > conf) {
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { nrgbd_set_error("conv_wgmma: cannot opt in to %zu bytes of shared memory: %s", smem, cudaGetErrorString(e)); return NRGBD_ERR_CUDA; }
    conf = smem;
  }
  // persistent CTAs: one per resident slot (the smem plan and __launch_bounds__ give the CTAs per SM), shared out
  // among the Cout chunks
  int grid_x = p.n_tiles;
  if (!(g_h2_flags & 32)) {
    const int per_sm = (int)std::min<size_t>(BN <= 64 ? 2 : 1, 233472 / (smem + 1024));
    grid_x = std::min(grid_x, ceil_div(nrgbd_sm_count() * per_sm, n_chunks));
  }
  fn<<<dim3((unsigned)grid_x, (unsigned)n_chunks), WG_THREADS, smem, st>>>(ta_hi, ta_lo, tb_hi, tb_lo, p);
  return NRGBD_OK;
}

}  // namespace

int conv_wgmma(const WgConv& c, cudaStream_t st) {
  NRGBD_REQUIRE(c.n_tap >= 1 && c.n_tap <= WG_MAX_TAP2D && c.n_kz >= 1 && c.n_kz <= 3 && c.Cin_pad % BKC == 0 && c.Cout_pad % 16 == 0,
                "unsupported convolution shape");
  const int esize = c.tf32 ? 4 : 2, RB = BKC * esize;
  WgParams p{};
  p.y = c.y; p.bias = c.bias; p.stats = c.stats;
  p.y_hi = reinterpret_cast<__half*>(c.y_hi); p.y_lo = reinterpret_cast<__half*>(c.y_lo);
  p.aff_scale = c.aff_scale; p.aff_shift = c.aff_shift; p.res = c.res; p.relu = c.relu;
  p.res_hi = reinterpret_cast<const __half*>(c.res_hi); p.res_lo = reinterpret_cast<const __half*>(c.res_lo);
  p.N = c.N; p.Dz = c.Din; p.Hy = c.Hy; p.Wx = c.Wx;
  // output tile 8 x 16 when it pads fewer positions than 16 x 8 (120-row planes), else 16 x 8
  const long long pad_tall = (long long)ceil_div(c.Hy, 16) * ceil_div(c.Wx, 8), pad_wide = (long long)ceil_div(c.Hy, 8) * ceil_div(c.Wx, 16);
  p.wide = (pad_wide < pad_tall && !(g_h2_flags & 8)) ? 1 : 0;
  const int TH = p.wide ? 8 : 16, TW = p.wide ? 16 : 8;
  p.tiles_x = ceil_div(c.Wx, TW); p.tiles_y = ceil_div(c.Hy, TH);
  NRGBD_REQUIRE((long long)p.N * p.Dz * p.tiles_x * p.tiles_y < (1ll << 31), "too many output tiles");
  p.n_tiles = p.N * p.Dz * p.tiles_x * p.tiles_y;
  p.cin_chunks = c.Cin_pad / BKC; p.n_kz = c.n_kz; p.n_tap = c.n_tap; p.in_stride = c.in_stride;
  p.Cout = c.Cout; p.Dout = c.Dout; p.Hout = c.Hout; p.Wout = c.Wout; p.Cs_out = c.Cs_out; p.c_off = c.c_off;
  p.out_stride = c.out_stride; p.out_off_y = c.out_off_y; p.out_off_x = c.out_off_x; p.leaky = c.leaky;
  for (int a = 0; a < 3; ++a) p.dz[a] = c.dz[a];
  for (int t = 0; t < WG_MAX_TAP2D; ++t) { p.dy[t] = c.dy[t]; p.dx[t] = c.dx[t]; }
  for (int t = 0; t < 3 * WG_MAX_TAP2D; ++t) p.wsel[t] = c.wsel[t];
  // halo: stride-1 filters with more than one in-plane tap
  p.halo = (c.in_stride == 1 && c.n_tap > 1 && !(g_h2_flags & 4)) ? 1 : 0;
  int pitch = TW, halo_rows = TH;
  if (p.halo) {
    int min_dy = 127, max_dy = -127, min_dx = 127, max_dx = -127;
    for (int t = 0; t < c.n_tap; ++t) {
      min_dy = c.dy[t] < min_dy ? c.dy[t] : min_dy; max_dy = c.dy[t] > max_dy ? c.dy[t] : max_dy;
      min_dx = c.dx[t] < min_dx ? c.dx[t] : min_dx; max_dx = c.dx[t] > max_dx ? c.dx[t] : max_dx;
    }
    pitch = TW + (max_dx - min_dx); halo_rows = TH + (max_dy - min_dy);
    if (pitch > TW + 16 || halo_rows > TH + 16) { p.halo = 0; pitch = TW; halo_rows = TH; }
    else {
      p.org_y = min_dy; p.org_x = min_dx;
      for (int t = 0; t < c.n_tap; ++t) p.a_off16[t] = (unsigned short)((((c.dy[t] - min_dy) * pitch + (c.dx[t] - min_dx)) * RB) >> 4);
    }
  }
  const uint32_t swz_mode = c.tf32 ? 1u : 2u;                    // 128-byte / 64-byte swizzle = one pixel row
  p.a_desc_hi = (uint32_t)((pitch * RB) >> 4) | (swz_mode << 30);  // SBO = one row of the (halo) tile
  p.b_desc_hi = (uint32_t)((8 * RB) >> 4) | (swz_mode << 30);
  p.wg_row16 = (uint32_t)((8 * (p.wide ? 1 : pitch) * RB) >> 4);   // 8 pixels right / 8 (halo) rows down
  p.box_w = pitch; p.box_h = halo_rows;
  p.a_tx_bytes = 2u * (uint32_t)(halo_rows * pitch * RB);
  p.a_tile_bytes = round_up((uint32_t)(halo_rows * pitch * RB), 1024);
  p.a_stage_bytes = 2 * p.a_tile_bytes;
  // Cout in chunks of 128 channels, the last one narrower (320 = 128 + 128 + 64): one launch per chunk width
  const int n_chunks = (c.Cout_pad + 127) / 128;
  const int BN = c.Cout_pad < 128 ? c.Cout_pad : 128;
  const int BN_last = c.Cout_pad - (n_chunks - 1) * BN;
  const int n_full = BN_last == BN ? n_chunks : n_chunks - 1;
  int rc = launch_chunks(c, p, BN, n_full, 0, st);
  if (rc == NRGBD_OK && n_full < n_chunks) rc = launch_chunks(c, p, BN_last, 1, n_full * BN, st);
  return rc;
}

namespace {
// ---- operand preparation -------------------------------------------------------------------------------------------
__device__ __forceinline__ void split_pair(float a, __half& hi, __half& lo) { nrgbd_split_pair(a, hi, lo); }

// fp32 [n] -> hi / lo halves [n]
__global__ void __launch_bounds__(256)
split_f16_pair_kernel(const float4* __restrict__ x, long long n4, uint2* __restrict__ hi, uint2* __restrict__ lo) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = x[i];
    __half h[4], l[4];
    split_pair(v.x, h[0], l[0]); split_pair(v.y, h[1], l[1]); split_pair(v.z, h[2], l[2]); split_pair(v.w, h[3], l[3]);
    uint2 ho, lo2;
    ho.x = (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16);
    ho.y = (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16);
    lo2.x = (uint32_t)__half_as_ushort(l[0]) | ((uint32_t)__half_as_ushort(l[1]) << 16);
    lo2.y = (uint32_t)__half_as_ushort(l[2]) | ((uint32_t)__half_as_ushort(l[3]) << 16);
    hi[i] = ho; lo[i] = lo2;
  }
}

// PyTorch weight -> K-major pair tiles [tap][2 (hi | lo)][Cout_pad][Cin_pad] halves
__global__ void pack_weight_h2_kernel(const float* __restrict__ w, int kind, int Cout, int Cin, int taps, int Cin_pad, int Cout_pad,
                                      __half* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n = (long long)taps * Cin_pad * Cout_pad;
  if (i >= n) return;
  int ci = (int)(i % Cin_pad);
  int co = (int)((i / Cin_pad) % Cout_pad);
  int t = (int)(i / ((long long)Cout_pad * Cin_pad));
  float v = 0.f;
  if (co < Cout && ci < Cin) v = kind == 0 ? w[((long long)co * Cin + ci) * taps + t] : w[((long long)ci * Cout + co) * taps + t];
  __half h, l;
  split_pair(v, h, l);
  const long long tile = (long long)Cout_pad * Cin_pad;
  out[(long long)t * 2 * tile + (long long)co * Cin_pad + ci] = h;
  out[(long long)t * 2 * tile + tile + (long long)co * Cin_pad + ci] = l;
}

}  // namespace

extern "C" {

void nrgbd_dev_conv_h2_set_flags(int flags) { g_h2_flags = flags; }
void nrgbd_dev_conv_h2_set_smem_cap_kb(int kb) { g_h2_smem_cap_kb = kb; }

// Channel plan of the f16-pair path: Cin padded to 32; Cout padded to 16 and cut into chunks of BN = min(128, Cout_pad)
// channels per CTA (grid.y), the last chunk taking the remainder (128 + 128 + 64 for 320, 128 + 16 for 131).
int nrgbd_conv_h2_plan(int Cin, int Cout, int* Cin_pad, int* Cout_pad, int* BN) {
  if (Cin < 1 || Cout < 1) return 0;
  const int c16 = (Cout + 15) / 16 * 16;
  if (Cin_pad) *Cin_pad = (Cin + 31) / 32 * 32;
  if (Cout_pad) *Cout_pad = c16;
  if (BN) *BN = c16 < 128 ? c16 : 128;
  return 1;
}

int nrgbd_split_f16_pair(const float* x, long long n, void* hi, void* lo, cudaStream_t st) {
  NRGBD_REQUIRE(x && hi && lo && n > 0 && n % 4 == 0, "bad arguments");
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > nrgbd_sm_count() * 16ll) blocks = nrgbd_sm_count() * 16ll;
  split_f16_pair_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(x), n / 4, reinterpret_cast<uint2*>(hi),
                                                         reinterpret_cast<uint2*>(lo));
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

int nrgbd_pack_conv_weight_h2(const float* w, int transposed, int Cout, int Cin, int taps, int Cin_pad, int Cout_pad, void* out,
                              cudaStream_t st) {
  NRGBD_REQUIRE(w && out && Cout > 0 && Cin > 0 && taps > 0 && Cin_pad >= Cin && Cout_pad >= Cout, "bad arguments");
  long long n = (long long)taps * Cin_pad * Cout_pad;
  pack_weight_h2_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w, transposed ? 1 : 0, Cout, Cin, taps, Cin_pad, Cout_pad, reinterpret_cast<__half*>(out));
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

static int conv_nhwc_h2_impl(const void* x_hi, const void* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const void* w,
                             const float* bias, int Cout, int Cout_pad, int BN, int kd, int kh, int kw, int stride, int pad, int dilation, float* y,
                             void* y_hi, void* y_lo, int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats, cudaStream_t st,
                             const WgConv* aff = nullptr);

int nrgbd_conv_nhwc_h2(const void* x_hi, const void* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const void* w,
                       const float* bias, int Cout, int Cout_pad, int BN, int kd, int kh, int kw, int stride, int pad, int dilation, float* y,
                       int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats, cudaStream_t st) {
  NRGBD_REQUIRE(y, "null pointer");
  return conv_nhwc_h2_impl(x_hi, x_lo, N, Din, Hin, Win, Cin_pad, Cs_in, w, bias, Cout, Cout_pad, BN, kd, kh, kw, stride, pad, dilation, y, nullptr,
                           nullptr, Hout, Wout, Cs_out, c_off, leaky, stats, st);
}

// Same convolution, the result (after bias / LeakyReLU) written ONLY as the split-fp16 operand pair of the convolution that
// consumes it: y_hi / y_lo are half tensors [N][D][Hout][Wout][Cs_out], Cs_out % 32 == 0, every channel stored (pad channels
// as zeros). Saves the separate split pass (one fp32 read + one pair write per element) for conv -> conv chains without a
// BatchNorm in between (R-Net, models/Refine.py:79-107).
int nrgbd_conv_nhwc_h2_pair(const void* x_hi, const void* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const void* w,
                            const float* bias, int Cout, int Cout_pad, int BN, int kd, int kh, int kw, int stride, int pad, int dilation,
                            void* y_hi, void* y_lo, int Hout, int Wout, int Cs_out, int leaky, cudaStream_t st) {
  NRGBD_REQUIRE(y_hi && y_lo, "null pointer");
  return conv_nhwc_h2_impl(x_hi, x_lo, N, Din, Hin, Win, Cin_pad, Cs_in, w, bias, Cout, Cout_pad, BN, kd, kh, kw, stride, pad, dilation, nullptr, y_hi,
                           y_lo, Hout, Wout, Cs_out, 0, leaky, nullptr, st);
}

static int conv_nhwc_h2_impl(const void* x_hi, const void* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const void* w,
                             const float* bias, int Cout, int Cout_pad, int BN, int kd, int kh, int kw, int stride, int pad, int dilation, float* y,
                             void* y_hi, void* y_lo, int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats, cudaStream_t st,
                             const WgConv* aff) {
  NRGBD_REQUIRE(x_hi && x_lo && w, "null pointer");
  NRGBD_REQUIRE(Cin_pad % 32 == 0 && Cin_pad >= 32 && Cin_pad <= Cs_in && Cs_in % 8 == 0 && Cout_pad % 16 == 0 && Cout <= Cout_pad && Cout > Cout_pad - 16 &&
                    BN == (Cout_pad < 128 ? Cout_pad : 128), "channel counts not supported by the f16-pair tensor-core path");
  NRGBD_REQUIRE(kd >= 1 && kd <= 3 && kh * kw <= WG_MAX_TAP2D && stride >= 1 && stride <= 8, "unsupported filter");
  NRGBD_REQUIRE(Hout == (Hin + 2 * pad - dilation * (kh - 1) - 1) / stride + 1 &&
                    Wout == (Win + 2 * pad - dilation * (kw - 1) - 1) / stride + 1, "output extent mismatch");
  if (y_hi) {
    // the output as the operand pair of the next convolution: every Cs_out channel stored, pad channels as zeros
    NRGBD_REQUIRE(Cs_out % 32 == 0 && Cs_out >= Cout_pad && c_off == 0 && stats == nullptr && (((uintptr_t)y_hi | (uintptr_t)y_lo) & 15) == 0 && y_lo,
                  "pair output needs Cs_out % 32 == 0, c_off == 0 and no statistics");
  }
  WgConv c{};
  c.tf32 = 0;
  c.x_hi = x_hi; c.x_lo = x_lo; c.N = N; c.Din = Din; c.Hin = Hin; c.Win = Win; c.Cin_pad = Cin_pad; c.Cs_in = Cs_in;
  c.w_hi = w; c.w_lo = reinterpret_cast<const __half*>(w) + (long long)Cout_pad * Cin_pad; c.w_tap_stride = 2ll * Cout_pad * Cin_pad;
  c.n_wslices = kd * kh * kw; c.Cout_pad = Cout_pad;
  c.bias = bias; c.stats = stats; c.y = y; c.y_hi = y_hi; c.y_lo = y_lo;
  c.Cout = Cout; c.Dout = Din; c.Hout = Hout; c.Wout = Wout; c.Cs_out = Cs_out; c.c_off = c_off;
  c.out_stride = 1; c.out_off_y = 0; c.out_off_x = 0; c.leaky = leaky;
  if (aff) { c.aff_scale = aff->aff_scale; c.aff_shift = aff->aff_shift; c.res = aff->res; c.res_hi = aff->res_hi; c.res_lo = aff->res_lo; c.relu = aff->relu; }
  c.Hy = Hout; c.Wx = Wout; c.in_stride = stride; c.n_kz = kd; c.n_tap = kh * kw;
  for (int a = 0; a < kd; ++a) c.dz[a] = (signed char)(a - kd / 2);
  int t = 0;
  for (int b = 0; b < kh; ++b)
    for (int e = 0; e < kw; ++e) { c.dy[t] = (signed char)(b * dilation - pad); c.dx[t] = (signed char)(e * dilation - pad); ++t; }
  for (int a = 0; a < kd * kh * kw; ++a) c.wsel[a] = (unsigned char)a;
  int rc = conv_wgmma(c, st);
  if (rc != NRGBD_OK) return rc;
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Eval-mode convbn in one pass: the convolution, then per output channel v = acc * scale + shift (+ residual) (ReLU), written
// either as fp32 (y, channel offset c_off) or as the operand pair of the next convolution (y_hi / y_lo, as
// nrgbd_conv_nhwc_h2_pair). No bias, no statistics.
int nrgbd_conv_nhwc_h2_affine(const void* x_hi, const void* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const void* w,
                              int Cout, int Cout_pad, int BN, int kd, int kh, int kw, int stride, int pad, int dilation,
                              const float* scale, const float* shift, const float* res, const void* res_hi, const void* res_lo, int relu,
                              float* y, void* y_hi, void* y_lo, int Hout, int Wout, int Cs_out, int c_off, cudaStream_t st) {
  NRGBD_REQUIRE(scale && shift, "null scale / shift");
  NRGBD_REQUIRE((y != nullptr) != (y_hi != nullptr) && (y_hi == nullptr) == (y_lo == nullptr), "the output is either fp32 (y) or a pair (y_hi, y_lo)");
  NRGBD_REQUIRE((res_hi == nullptr) == (res_lo == nullptr) && !(res && res_hi), "the residual is either an fp32 tensor or an operand pair");
  WgConv aff{};
  aff.aff_scale = scale; aff.aff_shift = shift; aff.res = res; aff.res_hi = res_hi; aff.res_lo = res_lo; aff.relu = relu ? 1 : 0;
  return conv_nhwc_h2_impl(x_hi, x_lo, N, Din, Hin, Win, Cin_pad, Cs_in, w, nullptr, Cout, Cout_pad, BN, kd, kh, kw, stride, pad, dilation, y,
                           y_hi, y_lo, Hout, Wout, Cs_out, c_off, 0, nullptr, st, &aff);
}

// nn.ConvTranspose2d(kernel 4, stride 2, padding 1) as four output-parity classes of 2x2-tap convolutions
int nrgbd_conv_transpose2d_k4s2_nhwc_h2(const void* x_hi, const void* x_lo, int N, int Hin, int Win, int Cin_pad, int Cs_in, const void* w,
                                        const float* bias, int Cout, int Cout_pad, int BN, float* y, int Cs_out, int c_off, int leaky,
                                        cudaStream_t st) {
  NRGBD_REQUIRE(x_hi && x_lo && w && y, "null pointer");
  NRGBD_REQUIRE(Cin_pad % 32 == 0 && Cin_pad >= 32 && Cin_pad <= Cs_in && Cs_in % 8 == 0 && Cout_pad % 16 == 0 && Cout <= Cout_pad && Cout > Cout_pad - 16 &&
                    BN == (Cout_pad < 128 ? Cout_pad : 128), "channel counts not supported by the f16-pair tensor-core path");
  const int kys[2][2] = {{1, 3}, {0, 2}};
  const int dys[2][2] = {{0, -1}, {1, 0}};
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      WgConv c{};
      c.tf32 = 0;
      c.x_hi = x_hi; c.x_lo = x_lo; c.N = N; c.Din = 1; c.Hin = Hin; c.Win = Win; c.Cin_pad = Cin_pad; c.Cs_in = Cs_in;
      c.w_hi = w; c.w_lo = reinterpret_cast<const __half*>(w) + (long long)Cout_pad * Cin_pad; c.w_tap_stride = 2ll * Cout_pad * Cin_pad;
      c.n_wslices = 16; c.Cout_pad = Cout_pad;
      c.bias = bias; c.stats = nullptr; c.y = y;
      c.Cout = Cout; c.Dout = 1; c.Hout = 2 * Hin; c.Wout = 2 * Win; c.Cs_out = Cs_out; c.c_off = c_off;
      c.out_stride = 2; c.out_off_y = py; c.out_off_x = px; c.leaky = leaky;
      c.Hy = Hin; c.Wx = Win; c.in_stride = 1; c.n_kz = 1; c.n_tap = 4;
      int t = 0;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          c.dy[t] = (signed char)dys[py][a]; c.dx[t] = (signed char)dys[px][b];
          c.wsel[t] = (unsigned char)(kys[py][a] * 4 + kys[px][b]); ++t;
        }
      int rc = conv_wgmma(c, st);
      if (rc != NRGBD_OK) return rc;
    }
  NRGBD_COUNT(4);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
