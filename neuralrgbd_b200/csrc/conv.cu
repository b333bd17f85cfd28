// fp32 implicit-GEMM convolution for the KVNET conv stacks (SURVEY §8 a5, a8, a10).
//
// Replaces nn.Conv2d / nn.Conv3d / nn.ConvTranspose2d (+ bias, LeakyReLU) and the statistics
// half of nn.BatchNorm2d/3d in training mode (models/psm_submodule.py:10-23, models/basic.py:71-94,
// models/Refine.py:47-77, models/m_submodule.py:18-43).
//
// Layout: activations are channels-last [N][D][H][W][Cs] fp32 with a channel stride Cs that is a
// multiple of 4 (pad channels hold zeros), so one K-chunk of the implicit GEMM is a contiguous
// 16-byte vector and a whole tap is a contiguous run. Weights are packed [tap][Cin_pad][Cout_pad].
// GEMM view: M = N*Dz*Hy*Wx output positions, N = Cout, K = taps * Cin_pad.
// One kernel covers conv2d (any stride / dilation / padding), conv3d 3x3x3 and the four parity
// classes of ConvTranspose2d(k=4, s=2, p=1) through a per-launch tap table.
//
// This is the exact-fp32 (CUDA-core FFMA) path: it is the parity anchor for the conv stacks.
// DESIGN.md explains why single-pass TF32/BF16 tensor-core operands cannot meet the 1e-4 DPV
// tolerance (SURVEY §7 'hard parts') and what the wgmma 3xTF32 variant must do.
#include "common.cuh"

namespace {

constexpr int MAX_TAPS = 27;

struct ConvParams {
  const float* x;     // input activations
  const float* w;     // packed weights [n_wslices][Cin_pad][Cout_pad]
  const float* bias;  // [Cout] or null
  float* y;           // output activations
  double* stats;      // [2][Cout] running sum / sum of squares (atomicAdd) or null
  int N, Dz, Hy, Wx;  // iteration space (output positions before out_stride/out_off)
  int Din, Hin, Win;  // input extents
  int Cin_pad, Cs_in; // K per tap, input channel stride
  int Cout, Cout_pad; // logical / packed output channels
  int Dout, Hout, Wout, Cs_out, c_off;   // output tensor extents, channel stride, channel offset
  int in_stride;                          // input coord = out coord * in_stride + tap offset
  int out_stride, out_off_y, out_off_x;   // output coord = iter coord * out_stride + off
  int n_taps;
  int leaky;                              // apply LeakyReLU(0.01) after bias
  signed char dz[MAX_TAPS], dy[MAX_TAPS], dx[MAX_TAPS];
  unsigned char wsel[MAX_TAPS];
};

// BM x BN output tile per CTA, BK-deep K steps, 256 threads as 16 (n) x 16 (m), TM x TN per thread.
template <int BM, int BN>
__global__ void __launch_bounds__(256)
conv_igemm_kernel(const ConvParams p) {
  constexpr int BK = 16;
  constexpr int TM = BM / 16, TN = BN / 16;
  constexpr int AS = BM + 4;     // smem row stride of the transposed A tile (16 B aligned rows)
  __shared__ __align__(16) float As[2][BK][AS];
  __shared__ __align__(16) float Bs[2][BK][BN];
  __shared__ float red[2][16][BN];

  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;
  const long long M = (long long)p.N * p.Dz * p.Hy * p.Wx;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- A-load assignment: thread -> (row m_l, k4 slot j); BM*4 float4 per K step -------------
  constexpr int A_ITERS = (BM * 4) / 256;
  int a_m[A_ITERS], a_j[A_ITERS];
  int a_n[A_ITERS], a_z[A_ITERS], a_y[A_ITERS], a_x[A_ITERS];
  bool a_ok[A_ITERS];
#pragma unroll
  for (int i = 0; i < A_ITERS; ++i) {
    int idx = tid + i * 256;
    a_j[i] = idx % 4;
    a_m[i] = idx / 4;
    long long m = m0 + a_m[i];
    a_ok[i] = m < M;
    long long r = a_ok[i] ? m : 0;
    a_x[i] = (int)(r % p.Wx); r /= p.Wx;
    a_y[i] = (int)(r % p.Hy); r /= p.Hy;
    a_z[i] = (int)(r % p.Dz); r /= p.Dz;
    a_n[i] = (int)r;
  }
  // ---- B-load assignment: BK * BN / 4 float4 per K step ---------------------------------------
  constexpr int B_F4 = BK * BN / 4;
  constexpr int B_ITERS = (B_F4 + 255) / 256;

  const int K = p.n_taps * p.Cin_pad;
  const int nk = (K + BK - 1) / BK;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float4 a_reg[A_ITERS];
  float4 b_reg[B_ITERS];

  auto load_tiles = [&](int ks) {
    const int k0 = ks * BK;
#pragma unroll
    for (int i = 0; i < A_ITERS; ++i) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      int kk = k0 + 4 * a_j[i];
      if (a_ok[i] && kk < K) {
        int tap = kk / p.Cin_pad;
        int ci = kk - tap * p.Cin_pad;
        int iz = a_z[i] + p.dz[tap];
        int iy = a_y[i] * p.in_stride + p.dy[tap];
        int ix = a_x[i] * p.in_stride + p.dx[tap];
        if (iz >= 0 && iz < p.Din && iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win) {
          const float* src = p.x + ((((long long)a_n[i] * p.Din + iz) * p.Hin + iy) * p.Win + ix) * p.Cs_in + ci;
          v = __ldg(reinterpret_cast<const float4*>(src));
        }
      }
      a_reg[i] = v;
    }
#pragma unroll
    for (int i = 0; i < B_ITERS; ++i) {
      int idx = tid + i * 256;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < B_F4) {
        int kr = idx / (BN / 4), nc = (idx % (BN / 4)) * 4;
        int kk = k0 + kr;
        if (kk < K && n0 + nc < p.Cout_pad) {
          int tap = kk / p.Cin_pad;
          int ci = kk - tap * p.Cin_pad;
          const float* src = p.w + ((long long)p.wsel[tap] * p.Cin_pad + ci) * p.Cout_pad + n0 + nc;
          v = __ldg(reinterpret_cast<const float4*>(src));
        }
      }
      b_reg[i] = v;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_ITERS; ++i) {
      int kb = 4 * a_j[i];
      As[buf][kb + 0][a_m[i]] = a_reg[i].x;
      As[buf][kb + 1][a_m[i]] = a_reg[i].y;
      As[buf][kb + 2][a_m[i]] = a_reg[i].z;
      As[buf][kb + 3][a_m[i]] = a_reg[i].w;
    }
#pragma unroll
    for (int i = 0; i < B_ITERS; ++i) {
      int idx = tid + i * 256;
      if (idx < B_F4) {
        int kr = idx / (BN / 4), nc = (idx % (BN / 4)) * 4;
        *reinterpret_cast<float4*>(&Bs[buf][kr][nc]) = b_reg[i];
      }
    }
  };

  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int ks = 0; ks < nk; ++ks) {
    const int buf = ks & 1;
    if (ks + 1 < nk) load_tiles(ks + 1);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        float4 v = *reinterpret_cast<const float4*>(&As[buf][kk][ty * TM + i]);
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
      }
      if (TN >= 4) {
#pragma unroll
        for (int j = 0; j < TN; j += 4) {
          float4 v = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * TN + j]);
          b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
        }
      } else {
        float2 v = *reinterpret_cast<const float2*>(&Bs[buf][kk][tx * TN]);
        b[0] = v.x; b[1] = v.y;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (ks + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- epilogue: bias, LeakyReLU, store, BN statistics ------------------------------------------
  float s1[TN], s2[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) { s1[j] = 0.f; s2[j] = 0.f; }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    long long m = m0 + ty * TM + i;
    if (m < M) {
      long long r = m;
      int x = (int)(r % p.Wx); r /= p.Wx;
      int y = (int)(r % p.Hy); r /= p.Hy;
      int z = (int)(r % p.Dz); r /= p.Dz;
      int n = (int)r;
      int oy = y * p.out_stride + p.out_off_y, ox = x * p.out_stride + p.out_off_x;
      float* dst = p.y + ((((long long)n * p.Dout + z) * p.Hout + oy) * p.Wout + ox) * p.Cs_out + p.c_off;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        int co = n0 + tx * TN + j;
        if (co < p.Cout) {
          float v = acc[i][j];
          if (p.bias) v += __ldg(p.bias + co);
          if (p.leaky) v = v >= 0.f ? v : v * 0.01f;
          dst[co] = v;
          s1[j] += v; s2[j] = fmaf(v, v, s2[j]);
        }
      }
    }
  }
  if (p.stats) {
#pragma unroll
    for (int j = 0; j < TN; ++j) { red[0][ty][tx * TN + j] = s1[j]; red[1][ty][tx * TN + j] = s2[j]; }
    __syncthreads();
    if (tid < BN) {
      int co = n0 + tid;
      if (co < p.Cout) {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int r = 0; r < 16; ++r) { a += red[0][r][tid]; b += red[1][r][tid]; }
        atomicAdd(p.stats + co, (double)a);
        atomicAdd(p.stats + p.Cout + co, (double)b);
      }
    }
  }
}

// w_out[slice][ci][co] (zero padded) from PyTorch layouts.
//  kind 0: Conv2d/Conv3d weight [Cout][Cin][taps]   kind 1: ConvTranspose2d weight [Cin][Cout][taps]
__global__ void pack_weight_kernel(const float* __restrict__ w, int kind, int Cout, int Cin, int taps, int Cin_pad,
                                   int Cout_pad, float* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n = (long long)taps * Cin_pad * Cout_pad;
  if (i >= n) return;
  int co = (int)(i % Cout_pad);
  int ci = (int)((i / Cout_pad) % Cin_pad);
  int t = (int)(i / ((long long)Cout_pad * Cin_pad));
  float v = 0.f;
  if (co < Cout && ci < Cin)
    v = kind == 0 ? w[((long long)co * Cin + ci) * taps + t] : w[((long long)ci * Cout + co) * taps + t];
  out[i] = v;
}

// scale/shift from accumulated statistics; optional running-stat update (momentum 0.1, unbiased var)
__global__ void bn_finalize_kernel(const double* __restrict__ stats, int C, double count, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float* __restrict__ scale,
                                   float* __restrict__ shift, float* __restrict__ run_mean, float* __restrict__ run_var,
                                   float momentum) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double mean = stats[c] / count;
  double var = stats[C + c] / count - mean * mean;
  if (var < 0) var = 0;
  float invstd = (float)(1.0 / sqrt(var + (double)eps));
  float sc = gamma[c] * invstd;
  scale[c] = sc;
  shift[c] = beta[c] - (float)mean * sc;
  if (run_mean) {
    double unb = count > 1 ? var * count / (count - 1) : var;
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * (float)mean;
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)unb;
  }
}

// Eval-mode coefficients (ATen's CPU order: invstd = 1 / sqrt(var + eps), scale = invstd * gamma, shift = beta - mean * scale),
// one block per layer
__global__ void bn_eval_coeffs_kernel(const BnEvalTable t) {
  const int l = blockIdx.x;
  for (int c = threadIdx.x; c < t.C[l]; c += blockDim.x) {
    const float invstd = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(t.var[l][c], t.eps)));
    const float sc = __fmul_rn(invstd, t.gamma[l][c]);
    t.scale[l][c] = sc;
    t.shift[l][c] = __fsub_rn(t.beta[l][c], __fmul_rn(t.mean[l][c], sc));
  }
}

// y = act(x * scale[c] + shift[c]) (+ res), channels-last with stride Cs; pad channels stay 0.
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ shift,
                const float* __restrict__ res, int relu, long long n4, int Cs, int C, float* __restrict__ y) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  int c = (int)((i * 4) % Cs);
  float4 v = reinterpret_cast<const float4*>(x)[i];
  float o[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (c + k < C) {
      float t = fmaf(o[k], scale[c + k], shift[c + k]);
      if (relu) t = fmaxf(t, 0.f);
      o[k] = t;
    } else {
      o[k] = 0.f;
    }
  }
  if (res) {
    float4 r = reinterpret_cast<const float4*>(res)[i];
    o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
  }
  reinterpret_cast<float4*>(y)[i] = make_float4(o[0], o[1], o[2], o[3]);
}

// BatchNorm finalize + apply in one kernel: every block derives scale/shift for all C channels from
// the accumulated statistics into shared memory (C <= 512), then streams its slice of the activation.
// Block 0 also performs the training-mode running-statistics update.
template <int U>
__global__ void __launch_bounds__(256)
bn_apply_stats_kernel(const float* __restrict__ x, const double* __restrict__ stats, double count,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                      float* __restrict__ run_mean, float* __restrict__ run_var, float momentum,
                      const float* __restrict__ res, const uint2* __restrict__ res_hi, const uint2* __restrict__ res_lo, int relu,
                      long long n4, int Cs, int C, float* __restrict__ y,
                      uint2* __restrict__ y_hi, uint2* __restrict__ y_lo, double* __restrict__ stats_to_zero,
                      unsigned int* __restrict__ done_counter) {
  __shared__ float s_scale[512], s_shift[512];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double mean = stats[c] / count;
    double var = stats[C + c] / count - mean * mean;
    if (var < 0) var = 0;
    float invstd = (float)(1.0 / sqrt(var + (double)eps));
    float sc = gamma[c] * invstd;
    s_scale[c] = sc;
    s_shift[c] = beta[c] - (float)mean * sc;
    if (run_mean && blockIdx.x == 0) {
      double unb = count > 1 ? var * count / (count - 1) : var;
      run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * (float)mean;
      run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)unb;
    }
  }
  __syncthreads();
  if (stats_to_zero && threadIdx.x == 0) {
    // every block has now copied the statistics into its shared memory: the LAST block to get here re-zeroes them, so the next
    // convolution accumulates into a clean buffer without a memset node in between (~70 memsets per frame otherwise)
    __threadfence();
    const unsigned int prev = atomicAdd(done_counter, 1u);
    if (prev == gridDim.x - 1) {
      for (int c = 0; c < 2 * C; ++c) stats_to_zero[c] = 0.0;
      __threadfence();
      *done_counter = 0u;
    }
  }
  // four 16-byte vectors per thread and iteration, all loads issued before the first use: 64 (128 with a residual) bytes in
  // flight per thread instead of 16 - this pass is pure streaming and was latency-bound with one vector per iteration
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < n4; i0 += stride * U) {
    float4 v[U], rr[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * stride;
      if (i < n4) {
        v[u] = reinterpret_cast<const float4*>(x)[i];
        if (res) rr[u] = reinterpret_cast<const float4*>(res)[i];
        else if (res_hi) {               // the residual as the operand pair its producer emitted (no fp32 copy of it exists)
          float q[4];
          nrgbd_join_pair4(res_hi[i], res_lo[i], q);
          rr[u] = make_float4(q[0], q[1], q[2], q[3]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * stride;
      if (i >= n4) continue;
      const int c = (int)((i * 4) % Cs);
      float o[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (c + k < C) {
          float t = fmaf(o[k], s_scale[c + k], s_shift[c + k]);
          if (relu) t = fmaxf(t, 0.f);
          o[k] = t;
        } else {
          o[k] = 0.f;
        }
      }
      if (res || res_hi) { o[0] += rr[u].x; o[1] += rr[u].y; o[2] += rr[u].z; o[3] += rr[u].w; }
      if (y) reinterpret_cast<float4*>(y)[i] = make_float4(o[0], o[1], o[2], o[3]);
      if (y_hi) {                      // the consumer is an f16-pair convolution: emit its operand planes in the same pass
        uint2 h, l;
        nrgbd_split_pair4(o, h, l);
        y_hi[i] = h;
        if (y_lo) y_lo[i] = l;         // no y_lo: hi only, the plain fp16 operand of a single-product convolution
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Single-output-channel 3x3x3 convolution as (1x1x1 conv to one channel PER TAP) + (shifted sum of the taps).
// K-Net's last layer (models/basic.py:136-137, Conv3d(64 -> 1, k3)) has Cout = 1: as an implicit GEMM its N is 1 (padded to
// 16), i.e. 27 x 4 x 3 tiny MMAs per 128 positions - issue-bound at 8 TFLOP/s. Re-associated,
//   out[p] = sum_t sum_c x[p + off_t][c] w[t][c] = sum_t Q[p + off_t][t],   Q[q][t] = sum_c x[q][c] w[t][c],
// Q is ONE pointwise convolution with 27 output channels (a single N = 32 GEMM on the tensor cores, 27x fewer MMAs) and the
// rest is this gather: every Q element is used exactly once.
// Q: [N][D][H][W][Cs] fp32 (Cs >= kd*k*k), out: [N][D][H][W] fp32, zero padding `pad` in all three axes.
// ---------------------------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(256)
tap_gather_sum_kernel(const float* __restrict__ Q, int D, int H, int W, int Cs, int kd, float bias, float* __restrict__ out) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int nd = blockIdx.z;                       // n * D + d
  const int d = nd % D;
  if (x >= W || y >= H) return;
  const int pd = kd / 2, p = K / 2;
  float acc = bias;
  for (int tz = 0; tz < kd; ++tz) {
    const int dz = d + tz - pd;
    if (dz < 0 || dz >= D) continue;
    const float* plane = Q + (size_t)(nd + tz - pd) * H * W * Cs;
#pragma unroll
    for (int ty = 0; ty < K; ++ty) {
      const int yy = y + ty - p;
      if (yy < 0 || yy >= H) continue;
#pragma unroll
      for (int tx = 0; tx < K; ++tx) {
        const int xx = x + tx - p;
        if (xx < 0 || xx >= W) continue;
        acc += __ldg(plane + ((size_t)yy * W + xx) * Cs + (tz * K + ty) * K + tx);
      }
    }
  }
  out[((size_t)nd * H + y) * W + x] = acc;
}

// BatchNorm pass shape, measured over a K-Net volume (1248x376 / 4, D = 128, 64 channels; tools/bench_kernels.py bnsweep) on an H100
// SXM (400 W power limit): TWO vectors in flight and 32 blocks per SM 700 us (2.75 TB/s of algorithmic traffic, 82 % of the 3.35 TB/s
// data-sheet HBM bandwidth) / 1030 us with a pair residual; 1 or 4 vectors and 16 / 32 blocks per SM within 2 % of that; 8 blocks
// per SM 13-15 % slower whatever the vector count. The same ordering holds at 120x160, D = 64 (245 MB) and at 5x240x320 (98 MB: 95 us
// against 108 us for the light shape). At 5x120x160 (24.6 MB, mostly L2-resident on the H100's 50 MB) the light shape - one vector,
// 8 blocks per SM, 41 us - is as fast as any, the streaming one 49 us: the switch sits at 64 MB.
int g_bn_unroll = 0;           // development override of the vectors in flight per thread (0 = by size; nrgbd_dev_set_bn_unroll)
int g_bn_blocks_per_sm = 0;    // development override of the grid cap in blocks per SM (0 = by size; nrgbd_dev_set_bn_blocks_per_sm)

}  // namespace

int bn_eval_coeffs(const BnEvalTable& t, cudaStream_t st) {
  NRGBD_REQUIRE(t.n >= 1 && t.n <= NRGBD_BN_EVAL_MAX, "bad layer count");
  bn_eval_coeffs_kernel<<<t.n, 128, 0, st>>>(t);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

extern "C" {

void nrgbd_dev_set_bn_unroll(int u) { g_bn_unroll = u; }
void nrgbd_dev_set_bn_blocks_per_sm(int b) { g_bn_blocks_per_sm = b; }

int nrgbd_pack_conv_weight(const float* w, int transposed, int Cout, int Cin, int taps, int Cin_pad, int Cout_pad,
                           float* out, cudaStream_t st) {
  NRGBD_REQUIRE(w && out && Cout > 0 && Cin > 0 && taps > 0 && Cin_pad >= Cin && Cout_pad >= Cout &&
                    Cin_pad % 4 == 0 && Cout_pad % 4 == 0, "bad arguments");
  long long n = (long long)taps * Cin_pad * Cout_pad;
  pack_weight_kernel<<<ceil_div(n, 256), 256, 0, st>>>(w, transposed ? 1 : 0, Cout, Cin, taps, Cin_pad, Cout_pad, out);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Generic channels-last convolution. kd x kh x kw taps (kd = 1 for 2-D), stride/pad/dilation on H,W
// (depth: stride 1, pad kd/2). x [N][Din][Hin][Win][Cs_in]; y [N][Din][Hout][Wout][Cs_out] written at
// channels [c_off, c_off+Cout). w packed [kd*kh*kw][Cin_pad][Cout_pad]. stats: [2][Cout] doubles,
// accumulated (caller zeroes) or null. leaky: LeakyReLU(0.01) after bias.
int nrgbd_conv_nhwc(const float* x, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const float* w,
                    const float* bias, int Cout, int Cout_pad, int kd, int kh, int kw, int stride, int pad,
                    int dilation, float* y, int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats,
                    cudaStream_t st) {
  NRGBD_REQUIRE(x && w && y, "null pointer");
  NRGBD_REQUIRE(Cin_pad % 4 == 0 && Cs_in % 4 == 0 && Cin_pad <= Cs_in && Cout_pad % 4 == 0 && Cout <= Cout_pad,
                "channel padding must be a multiple of 4");
  NRGBD_REQUIRE(kd * kh * kw <= MAX_TAPS && kd >= 1 && kh >= 1 && kw >= 1, "too many taps");
  NRGBD_REQUIRE(Hout == (Hin + 2 * pad - dilation * (kh - 1) - 1) / stride + 1 &&
                    Wout == (Win + 2 * pad - dilation * (kw - 1) - 1) / stride + 1, "output extent mismatch");
  ConvParams p;
  p.x = x; p.w = w; p.bias = bias; p.y = y; p.stats = stats;
  p.N = N; p.Dz = Din; p.Hy = Hout; p.Wx = Wout;
  p.Din = Din; p.Hin = Hin; p.Win = Win; p.Cin_pad = Cin_pad; p.Cs_in = Cs_in;
  p.Cout = Cout; p.Cout_pad = Cout_pad;
  p.Dout = Din; p.Hout = Hout; p.Wout = Wout; p.Cs_out = Cs_out; p.c_off = c_off;
  p.in_stride = stride; p.out_stride = 1; p.out_off_y = 0; p.out_off_x = 0;
  p.leaky = leaky;
  int t = 0;
  for (int a = 0; a < kd; ++a)
    for (int b = 0; b < kh; ++b)
      for (int c = 0; c < kw; ++c) {
        p.dz[t] = (signed char)(a - kd / 2);
        p.dy[t] = (signed char)(b * dilation - pad);
        p.dx[t] = (signed char)(c * dilation - pad);
        p.wsel[t] = (unsigned char)t;
        ++t;
      }
  p.n_taps = t;
  long long M = (long long)N * p.Dz * p.Hy * p.Wx;
  if (Cout_pad <= 32) {
    dim3 grid(ceil_div(M, 128), ceil_div(Cout_pad, 32));
    conv_igemm_kernel<128, 32><<<grid, 256, 0, st>>>(p);
  } else {
    dim3 grid(ceil_div(M, 128), ceil_div(Cout_pad, 64));
    conv_igemm_kernel<128, 64><<<grid, 256, 0, st>>>(p);
  }
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// ConvTranspose2d(kernel 4, stride 2, padding 1) as four parity-class 2x2 convolutions.
// x [N][Hin][Win][Cs_in]; y [N][2Hin][2Win][Cs_out] at channel offset c_off. w packed [16][Cin_pad][Cout_pad]
// (tap index ky*4+kx of the PyTorch [Cin][Cout][4][4] weight).
int nrgbd_conv_transpose2d_k4s2_nhwc(const float* x, int N, int Hin, int Win, int Cin_pad, int Cs_in, const float* w,
                                     const float* bias, int Cout, int Cout_pad, float* y, int Cs_out, int c_off,
                                     int leaky, cudaStream_t st) {
  NRGBD_REQUIRE(x && w && y, "null pointer");
  NRGBD_REQUIRE(Cin_pad % 4 == 0 && Cs_in % 4 == 0 && Cin_pad <= Cs_in && Cout_pad % 4 == 0 && Cout <= Cout_pad,
                "channel padding must be a multiple of 4");
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      ConvParams p;
      p.x = x; p.w = w; p.bias = bias; p.y = y; p.stats = nullptr;
      p.N = N; p.Dz = 1; p.Hy = Hin; p.Wx = Win;
      p.Din = 1; p.Hin = Hin; p.Win = Win; p.Cin_pad = Cin_pad; p.Cs_in = Cs_in;
      p.Cout = Cout; p.Cout_pad = Cout_pad;
      p.Dout = 1; p.Hout = 2 * Hin; p.Wout = 2 * Win; p.Cs_out = Cs_out; p.c_off = c_off;
      p.in_stride = 1; p.out_stride = 2; p.out_off_y = py; p.out_off_x = px;
      p.leaky = leaky;
      // oy = 2*iy - 1 + ky: even rows use ky in {1 (iy=y), 3 (iy=y-1)}, odd rows ky in {0 (iy=y+1), 2 (iy=y)}
      const int kys[2][2] = {{1, 3}, {0, 2}};
      const int dys[2][2] = {{0, -1}, {1, 0}};
      int t = 0;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          p.dz[t] = 0; p.dy[t] = (signed char)dys[py][a]; p.dx[t] = (signed char)dys[px][b];
          p.wsel[t] = (unsigned char)(kys[py][a] * 4 + kys[px][b]);
          ++t;
        }
      p.n_taps = 4;
      long long M = (long long)N * Hin * Win;
      if (Cout_pad <= 32) {
        dim3 grid(ceil_div(M, 128), ceil_div(Cout_pad, 32));
        conv_igemm_kernel<128, 32><<<grid, 256, 0, st>>>(p);
      } else {
        dim3 grid(ceil_div(M, 128), ceil_div(Cout_pad, 64));
        conv_igemm_kernel<128, 64><<<grid, 256, 0, st>>>(p);
      }
    }
  NRGBD_COUNT(4);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// BatchNorm (batch statistics) second half: scale/shift from stats accumulated by nrgbd_conv_nhwc.
int nrgbd_bn_finalize(const double* stats, int C, double count, const float* gamma, const float* beta, float eps,
                      float* scale, float* shift, float* run_mean, float* run_var, float momentum, cudaStream_t st) {
  NRGBD_REQUIRE(stats && gamma && beta && scale && shift && C > 0 && count > 0, "bad arguments");
  bn_finalize_kernel<<<ceil_div(C, 128), 128, 0, st>>>(stats, C, count, gamma, beta, eps, scale, shift, run_mean,
                                                       run_var, momentum);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Training-mode BatchNorm in one pass: finalize (scale/shift from the accumulated statistics, optional
// running-stat update) + y = [relu](x*scale + shift) [+ res]. C <= 512.
int nrgbd_bn_apply_stats(const float* x, const double* stats, double count, const float* gamma, const float* beta, float eps,
                         float* run_mean, float* run_var, float momentum, const float* res, int relu, long long n_pos, int Cs,
                         int C, float* y, cudaStream_t st) {
  NRGBD_REQUIRE(x && stats && gamma && beta && y && Cs % 4 == 0 && C <= Cs && C <= 512 && n_pos > 0 && count > 0, "bad arguments");
  long long n4 = n_pos * Cs / 4;
  long long blocks = (n4 + 255) / 256;
  if (blocks > nrgbd_sm_count() * 8ll) blocks = nrgbd_sm_count() * 8ll;
  bn_apply_stats_kernel<1><<<(unsigned)blocks, 256, 0, st>>>(x, stats, count, gamma, beta, eps, run_mean, run_var, momentum, res, nullptr,
                                                            nullptr, relu, n4, Cs, C, y, nullptr, nullptr, nullptr, nullptr);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// Same pass, additionally (or only: y may be NULL) writing the result as the split-fp16 operand pair of the f16-pair
// convolution that consumes it (nrgbd_conv_nhwc_h2): y_hi / y_lo are half tensors with x's layout (both may be NULL).
// y_hi set and y_lo NULL: only hi = RN_f16(result) is written (the operand of the single-product convolution).
// rezero_counter (optional): a zero-initialised device word; when given, the last block to have read `stats` sets them back
// to zero (and the word back to 0), so the next convolution can accumulate into `stats` without a memset in between.
int nrgbd_bn_apply_stats_pair(const float* x, double* stats, double count, const float* gamma, const float* beta, float eps,
                              float* run_mean, float* run_var, float momentum, const float* res, const void* res_hi, const void* res_lo,
                              int relu, long long n_pos, int Cs, int C, float* y, void* y_hi, void* y_lo, unsigned int* rezero_counter,
                              cudaStream_t st) {
  NRGBD_REQUIRE(x && stats && gamma && beta && (y || y_hi) && !(y_lo && !y_hi) && Cs % 4 == 0 && C <= Cs &&
                    C <= 512 && n_pos > 0 && count > 0, "bad arguments");
  NRGBD_REQUIRE((res_hi == nullptr) == (res_lo == nullptr) && !(res && res_hi), "the residual is either an fp32 tensor or an operand pair");
  const uint2* rh = reinterpret_cast<const uint2*>(res_hi);
  const uint2* rl = reinterpret_cast<const uint2*>(res_lo);
  long long n4 = n_pos * Cs / 4;
  long long blocks = (n4 + 255) / 256;
  // streaming shape (two vectors in flight, 32 blocks per SM) for tensors that do not fit L2 anyway (>= 64 MB of fp32: K-Net volumes,
  // the larger feature maps); the small 2-D passes of a 640x480 frame are launch / L2-latency bound and keep the light shape
  const bool big = n4 >= (4ll << 20);
  const int unroll = g_bn_unroll > 0 ? g_bn_unroll : (big ? 2 : 1);
  const long long cap = (long long)nrgbd_sm_count() * (g_bn_blocks_per_sm > 0 ? g_bn_blocks_per_sm : (big ? 32 : 8));
  if (blocks > cap) blocks = cap;
  if (unroll == 4)
    bn_apply_stats_kernel<4><<<(unsigned)blocks, 256, 0, st>>>(x, stats, count, gamma, beta, eps, run_mean, run_var, momentum, res, rh, rl,
                                                              relu, n4, Cs, C, y, reinterpret_cast<uint2*>(y_hi), reinterpret_cast<uint2*>(y_lo),
                                                              rezero_counter ? stats : nullptr, rezero_counter);
  else if (unroll == 2)
    bn_apply_stats_kernel<2><<<(unsigned)blocks, 256, 0, st>>>(x, stats, count, gamma, beta, eps, run_mean, run_var, momentum, res, rh, rl,
                                                              relu, n4, Cs, C, y, reinterpret_cast<uint2*>(y_hi), reinterpret_cast<uint2*>(y_lo),
                                                              rezero_counter ? stats : nullptr, rezero_counter);
  else
    bn_apply_stats_kernel<1><<<(unsigned)blocks, 256, 0, st>>>(x, stats, count, gamma, beta, eps, run_mean, run_var, momentum, res, rh, rl,
                                                              relu, n4, Cs, C, y, reinterpret_cast<uint2*>(y_hi), reinterpret_cast<uint2*>(y_lo),
                                                              rezero_counter ? stats : nullptr, rezero_counter);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// out[n][d][h][w] = bias + sum over the kd x k x k taps t of Q[n][d + tz - kd/2][h + ty - k/2][w + tx - k/2][t] (zero outside):
// the second half of a single-output-channel convolution whose first half is the pointwise convolution Q = x * w[t][:]
// (see tap_gather_sum_kernel). k = 3, kd in {1, 3}.
int nrgbd_tap_gather_sum(const float* Q, int N, int D, int H, int W, int Cs, int kd, int k, float bias, float* out, cudaStream_t st) {
  NRGBD_REQUIRE(Q && out && N > 0 && D > 0 && H > 0 && W > 0 && k == 3 && (kd == 1 || kd == 3) && Cs >= kd * k * k, "bad arguments");
  NRGBD_REQUIRE((long long)N * D <= 65535, "too many planes for one launch");
  dim3 grid(ceil_div(W, 32), ceil_div(H, 8), N * D);
  tap_gather_sum_kernel<3><<<grid, 256, 0, st>>>(Q, D, H, W, Cs, kd, bias, out);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

// y = [relu](x*scale + shift) [+ res]; n_pos positions of Cs channels (C logical). In place allowed.
int nrgbd_bn_eval_coeffs(const float* gamma, const float* beta, const float* running_mean, const float* running_var, float eps, int C,
                         float* scale, float* shift, cudaStream_t st) {
  NRGBD_REQUIRE(gamma && beta && running_mean && running_var && scale && shift && C > 0, "bad arguments");
  BnEvalTable t{};
  t.gamma[0] = gamma; t.beta[0] = beta; t.mean[0] = running_mean; t.var[0] = running_var;
  t.scale[0] = scale; t.shift[0] = shift; t.C[0] = C; t.n = 1; t.eps = eps;
  return bn_eval_coeffs(t, st);
}

int nrgbd_bn_apply(const float* x, const float* scale, const float* shift, const float* res, int relu,
                   long long n_pos, int Cs, int C, float* y, cudaStream_t st) {
  NRGBD_REQUIRE(x && scale && shift && y && Cs % 4 == 0 && C <= Cs && n_pos > 0, "bad arguments");
  long long n4 = n_pos * Cs / 4;
  bn_apply_kernel<<<ceil_div(n4, 256), 256, 0, st>>>(x, scale, shift, res, relu, n4, Cs, C, y);
  NRGBD_COUNT(1);
  NRGBD_LAUNCH_CHECK();
  return NRGBD_OK;
}

}  // extern "C"
