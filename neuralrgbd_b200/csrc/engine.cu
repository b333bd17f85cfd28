// KVNET inference engine: the native runtime behind models.KVNET.KVNET.forward (SURVEY §8 a4-a10).
//
// One engine object owns the layer plan of the reference network (models/KVNET.py:93-185,
// models/basic.py:223-323 D-Net, :113-139 K-Net, models/psm_submodule.py:141-167 feature CNN,
// models/Refine.py:79-107 R-Net), a stream-ordered device buffer pool, the packed conv weights and
// the camera tables, and runs a whole depth frame as a fixed sequence of nrgbd kernels on one
// stream: no Python between layers, no allocation after warm-up, activations channels-last.
// Parameters are registered by their reference state_dict names (borrowed device pointers or
// engine-owned copies of host arrays), so kvnet_*.tar checkpoints map one to one.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "../../include/nrgbd.h"

namespace {

struct Act {            // channels-last activation [N][D][H][W][Cs]
  float* p = nullptr;
  int N = 0, D = 1, H = 0, W = 0, C = 0, Cs = 0;
  bool pair_only = false;   // f16-pair mode: the BatchNorm pass wrote only the operand pair; p holds the RAW conv output (and keys the pair)
  long long pos() const { return (long long)N * D * H * W; }
  long long floats() const { return pos() * Cs; }
};

struct Block { float* p; size_t bytes; bool busy; };

struct Pool {           // stream-ordered reuse of cudaMalloc'd blocks (single stream => safe)
  std::vector<Block> blocks;
  size_t total = 0;
  float* acquire(size_t bytes) {
    int best = -1;
    for (int i = 0; i < (int)blocks.size(); ++i)
      if (!blocks[i].busy && blocks[i].bytes >= bytes && (best < 0 || blocks[i].bytes < blocks[best].bytes)) best = i;
    if (best >= 0 && blocks[best].bytes <= bytes * 2 + (1 << 20)) { blocks[best].busy = true; return blocks[best].p; }
    void* q = nullptr;
    if (cudaMalloc(&q, bytes) != cudaSuccess) return nullptr;
    blocks.push_back({(float*)q, bytes, true});
    total += bytes;
    return (float*)q;
  }
  void release(float* p) {
    for (auto& b : blocks) if (b.p == p) { b.busy = false; return; }
  }
  void destroy() { for (auto& b : blocks) cudaFree(b.p); blocks.clear(); total = 0; }
};

struct ParamRef { float* p; long long n; bool owned; };
// One packing of a conv weight: fp32 (PK_F32), TF32 hi planes in w and lo planes in lo (PK_TC), or f16-pair tiles
// [taps][2][Cout_pad][Cin_pad] halves in w with the kernel's N tile BN (PK_H2, PK_H2_TAPS). w null: not packed yet.
struct Packed { float* w = nullptr; float* lo = nullptr; int Cin_pad = 0, Cout_pad = 0, BN = 0; };
enum Packing { PK_F32, PK_TC, PK_H2, PK_H2_TAPS, PK_COUNT };
typedef std::array<Packed, PK_COUNT> PackedSet;                    // every packing of one parameter
struct PairBuf { float* hi = nullptr; float* lo = nullptr; };      // split-fp16 planes of an activation (pool blocks); lo null: fp16 only

struct Camera {
  bool set = false;
  float* K = nullptr;      // 3x3
  float* rays = nullptr;   // 3 x hw
  float cx = 0, cy = 0, tan_hh = 0, tan_hv = 0;
};

inline int pad4(int c) { return (c + 3) / 4 * 4; }
inline int pad16(int c) { return (c + 15) / 16 * 16; }
inline int pad32(int c) { return (c + 31) / 32 * 32; }

}  // namespace

struct nrgbd_kvnet {
  int H, W, D, V, F, KF;
  int h, w;
  float sigma;
  int metric = 0;
  int bn_update_running = 1;
  int bn_eval = 0;                  // the module is in .eval(): BatchNorm layers with running statistics normalise with them
  float* eval_coef = nullptr;       // [NRGBD_BN_EVAL_MAX][scale 512 | shift 512] of those layers, recomputed by every forward
  std::unordered_map<std::string, int> eval_slot;   // BatchNorm prefix -> row of eval_coef (empty in train mode)
  std::unordered_map<std::string, ParamRef> params;
  std::unordered_map<std::string, PackedSet> packed;   // by parameter name: set_param drops all packings of a re-set weight
  // activations that currently have a split-fp16 copy (conv_math 2 and 3). In conv_math 3 only the tensors read as residuals
  // keep a lo half; the rest are plain fp16 (lo null), since a convolution reads hi only.
  std::unordered_map<const float*, PairBuf> pairs;
  // 0: exact fp32 FFMA implicit GEMM; 1: wgmma 3xTF32; 2: wgmma split-fp16 pairs (conv_f16.cu); 3: single fp16 products on the
  // same paths as 2 (convolutions launched with x_lo = NULL)
  int conv_math = 0;
  int refine = 0;                   // refinement of KVNET(...): 0 the DPV R-Net, 1 the guided filter ('DGF'), 2 none (if_refined=False)
  int refine_up = 0;                // DPV R-Net with if_upsample_d: widths D0 = 2D, D1 = 4D (Refine.py:44-48)
  Camera cam[2];
  float* d_planes = nullptr;
  std::vector<float> d_host;
  Pool pool;
  double* stats = nullptr;          // [2][512] per-channel sums of the conv in flight
  double* stats_b = nullptr;        // second set: a conv that consumes one BatchNorm (fused) while producing the next
  unsigned int* bn_counter = nullptr;   // f16-pair mode: the BatchNorm pass re-zeroes the statistics it consumed (no memset nodes)
  float* ws_sweep = nullptr;        // V*12
  cudaStream_t st = nullptr;
  int rc = 0;                       // first error of the current forward
  // persistent per-frame products (valid after forward)
  float* bv_cur_hwd = nullptr;      // [hw][D]
  float* dpv_hwd = nullptr;         // [hw][D]
  float* prior_hwd = nullptr;       // [hw][D]
  float* depth = nullptr;           // [hw] expected depth of the low-res DPV
  float* conf = nullptr;
  // optional per-kernel event profiling (bench.py roofline): category 0 = conv (work = flops),
  // 1 = plane sweep (work = algorithmic bytes)
  // CUDA-graph replay of a whole frame: after one eager (warm-up) forward every buffer the frame needs is in
  // the pool and every weight is packed, so the launch sequence is static; it is captured once per distinct
  // tuple of caller pointers and replayed (≈330 launches + ≈90 memsets become one cudaGraphLaunch).
  int use_graph = 1;
  bool warm = false;            // eager first-window forward done
  bool warm_steady = false;     // eager K-Net (steady-state) forward done
  struct GraphEnt { int variant; cudaStream_t stream; cudaGraphExec_t exec; long long launches; };
  float* x0_buf = nullptr;          // [V+1][H][W][4] input frames, channels-last
  float* rt_buf = nullptr;          // [V][3][3] rotations then [V][3] translations
  float* ref_cur_hwd = nullptr;     // [HW][refined_planes()] refined output of the measurement (log-DPV, or guided-filter depth)
  float* ref_kv_hwd = nullptr;      // [HW][refined_planes()] refined output of the filtered DPV (steady state)
  long long ref_floats = 0;         // floats allocated for each of the two
  // planes of a refined output: the DPV R-Net's D (4D with if_upsample_d), 1 for the guided filter, 0 without refinement
  int refined_planes() const { return refine == 0 ? (refine_up ? 4 * D : D) : (refine == 1 ? 1 : 0); }
  std::vector<GraphEnt> graphs;
  unsigned long long graph_clock = 0;
  int profile = 0;
  struct ProfRec { cudaEvent_t a, b; int cat; double work; char tag[56]; };
  std::vector<ProfRec> prof;
  std::vector<cudaEvent_t> ev_free;
};

namespace {

typedef nrgbd_kvnet Eng;

#define ENG_CALL(e, expr)                 \
  do {                                    \
    if ((e)->rc == 0) {                   \
      int _r = (expr);                    \
      if (_r != 0) (e)->rc = _r;          \
    }                                     \
  } while (0)

cudaEvent_t prof_event(Eng* e) {
  if (!e->ev_free.empty()) { cudaEvent_t ev = e->ev_free.back(); e->ev_free.pop_back(); return ev; }
  cudaEvent_t ev; cudaEventCreate(&ev); return ev;
}
struct ProfScope {
  Eng* e; bool on; nrgbd_kvnet::ProfRec r;
  ProfScope(Eng* e_, int cat, double work, const char* tag = "") : e(e_), on(e_->profile && e_->rc == 0 && e_->prof.size() < 200000) {
    if (on) {
      r.a = prof_event(e); r.b = prof_event(e); r.cat = cat; r.work = work;
      snprintf(r.tag, sizeof(r.tag), "%s", tag);
      cudaEventRecord(r.a, e->st);
    }
  }
  ~ProfScope() { if (on) { cudaEventRecord(r.b, e->st); e->prof.push_back(r); } }
};

Act acquire(Eng* e, int N, int D, int H, int W, int C, int Cs = -1) {
  Act a; a.N = N; a.D = D; a.H = H; a.W = W; a.C = C;
  a.Cs = Cs >= 0 ? Cs : ((e->conv_math >= 1 && C >= 16) ? pad32(C) : pad4(C));   // tensor-core K-steps are 32 channels
  if (e->rc) return a;
  a.p = e->pool.acquire((size_t)a.floats() * sizeof(float));
  if (!a.p) { nrgbd_set_error("engine: out of device memory (%lld floats)", a.floats()); e->rc = NRGBD_ERR_NOMEM; return a; }
  if (a.Cs != a.C) cudaMemsetAsync(a.p, 0, (size_t)a.floats() * sizeof(float), e->st);   // pad channels must be 0
  return a;
}
void release(Eng* e, Act& a) {
  if (a.p) {
    auto it = e->pairs.find(a.p);
    if (it != e->pairs.end()) { e->pool.release(it->second.hi); e->pool.release(it->second.lo); e->pairs.erase(it); }
    e->pool.release(a.p);
  }
  a.p = nullptr;
}

// conv_math 2 and 3 take the f16-pair paths; 3 differs only in what the pairs hold and how convolutions are launched
inline bool pair_mode(const Eng* e) { return e->conv_math == 2 || e->conv_math == 3; }
// Whether a pair written now needs its lo half: always in conv_math 2; in conv_math 3 only when a residual add reads it
// (a residual keeps its 22-bit value; convolutions read hi only)
inline bool keep_lo(const Eng* e, bool res_read) { return e->conv_math == 2 || res_read; }
// x_lo of a convolution launch: NULL runs the single-product kernel (conv_math 3) even when the pair has a lo for a residual
inline const void* conv_lo(const Eng* e, const PairBuf* pb) { return e->conv_math == 3 ? nullptr : pb->lo; }

// Pool blocks of a split-fp16 pair of `floats` elements: hi, then lo when `lo` is set (see keep_lo)
bool acquire_pair(Eng* e, long long floats, bool lo, PairBuf& pb) {
  if (e->rc) return false;
  pb.hi = e->pool.acquire((size_t)floats * 2);
  pb.lo = lo ? e->pool.acquire((size_t)floats * 2) : nullptr;
  if (pb.hi && (pb.lo || !lo)) return true;
  nrgbd_set_error("engine: out of device memory"); e->rc = NRGBD_ERR_NOMEM;
  return false;
}

// An activation written only as the operand pair of the convolutions that read it (f16-pair mode): y.p is a 16-byte pool
// block that keys the pair in e->pairs, not an fp32 tensor. res_read: a residual add reads it too, so its lo half is kept.
Act pair_act(Eng* e, int N, int D, int H, int W, int C, bool res_read, PairBuf& pb) {
  Act y; y.N = N; y.D = D; y.H = H; y.W = W; y.C = C; y.Cs = pad32(C); y.pair_only = true;
  if (e->rc) return y;
  y.p = e->pool.acquire(16);
  if (!acquire_pair(e, y.floats(), keep_lo(e, res_read), pb)) return y;
  if (!y.p) { nrgbd_set_error("engine: out of device memory"); e->rc = NRGBD_ERR_NOMEM; return y; }
  e->pairs[y.p] = pb;
  return y;
}

// Split-fp16 operand planes of an activation (x = hi + lo * 2^-11), created on first use by a convolution and kept
// until the activation is released: several convolutions may consume the same tensor (BasicBlock input: conv1 +
// downsample). Activations are never written again after their first conv consumer has run. conv_math 3: hi only.
const PairBuf* pair_of(Eng* e, const Act& x) {
  auto it = e->pairs.find(x.p);
  if (it != e->pairs.end()) return &it->second;
  PairBuf pb;
  if (!acquire_pair(e, x.floats(), keep_lo(e, false), pb)) return nullptr;
  ENG_CALL(e, nrgbd_split_f16_pair(x.p, x.floats(), pb.hi, pb.lo, (nrgbd_stream_t)e->st));
  return &(e->pairs[x.p] = pb);
}

// Residual operand of a BatchNorm epilogue: the fp32 tensor, or the (hi, lo) pair of a residual that exists only as a pair
struct Residual { const float* f = nullptr; const void* hi = nullptr; const void* lo = nullptr; };
Residual residual_of(Eng* e, const Act* res) {
  Residual r;
  if (!res) return r;
  if (!res->pair_only) { r.f = res->p; return r; }
  auto it = e->pairs.find(res->p);
  if (it == e->pairs.end() || !it->second.lo) {
    nrgbd_set_error("engine: residual has neither an fp32 copy nor a full operand pair"); e->rc = NRGBD_ERR_BAD_ARG; return r;
  }
  r.hi = it->second.hi; r.lo = it->second.lo;
  return r;
}

float* param(Eng* e, const std::string& name) {
  auto it = e->params.find(name);
  if (it == e->params.end()) {
    if (e->rc == 0) { nrgbd_set_error("engine: parameter '%s' was never set", name.c_str()); e->rc = NRGBD_ERR_BAD_ARG; }
    return nullptr;
  }
  return it->second.p;
}
float* param_opt(Eng* e, const std::string& name) {
  auto it = e->params.find(name);
  return it == e->params.end() ? nullptr : it->second.p;
}

// Training-mode BatchNorm `pre`: its affine parameters, and the running buffers the pass updates (both, or neither: option
// bn_update_running off, or a layer without running statistics)
struct BnParams { float* gamma; float* beta; float* rm; float* rv; };
BnParams bn_params(Eng* e, const std::string& pre) {
  BnParams p;
  p.gamma = param(e, pre + ".weight"); p.beta = param(e, pre + ".bias");
  float* rm = e->bn_update_running ? param_opt(e, pre + ".running_mean") : nullptr;
  float* rv = e->bn_update_running ? param_opt(e, pre + ".running_var") : nullptr;
  p.rm = rm && rv ? rm : nullptr; p.rv = rm && rv ? rv : nullptr;
  return p;
}

void free_packed(PackedSet& s) { for (auto& pk : s) { cudaFree(pk.w); cudaFree(pk.lo); } }

// Conv weight `name` [Cout][Cin][taps] (transposed: [Cin][Cout][taps]) in the packing `kind`, made on first use.
// PK_H2_TAPS is the weight of a single-output-channel conv [1][Cin][taps] packed as the POINTWISE conv [taps][Cin] (one
// output channel per tap) for the tap-gather form of K-Net's last layer (nrgbd_tap_gather_sum): the transposed-kind f16-pair
// packing, requested with Cout = taps and 1 tap.
const Packed* packw(Eng* e, const std::string& name, Packing kind, int Cout, int Cin, int taps, bool transposed) {
  auto it = e->packed.find(name);
  if (it != e->packed.end() && it->second[kind].w) return &it->second[kind];
  float* src = param(e, name);
  if (!src || e->rc) return nullptr;
  const long long n = e->params[name].n;
  if (n != (long long)Cout * Cin * taps) {
    nrgbd_set_error("engine: parameter '%s' has %lld elements, expected %lld", name.c_str(), n, (long long)Cout * Cin * taps);
    e->rc = NRGBD_ERR_BAD_ARG;
    return nullptr;
  }
  const bool h2 = kind == PK_H2 || kind == PK_H2_TAPS;
  Packed pk;
  if (h2) nrgbd_conv_h2_plan(Cin, Cout, &pk.Cin_pad, &pk.Cout_pad, &pk.BN);
  else if (kind == PK_TC) { pk.Cin_pad = pad32(Cin); pk.Cout_pad = pad16(Cout); }
  else { pk.Cin_pad = pad4(Cin); pk.Cout_pad = pad4(Cout); }
  const size_t bytes = (size_t)taps * pk.Cin_pad * pk.Cout_pad * (h2 ? 2 * 2 : sizeof(float));    // f16 pairs: two halves
  if (cudaMalloc((void**)&pk.w, bytes) != cudaSuccess || (kind == PK_TC && cudaMalloc((void**)&pk.lo, bytes) != cudaSuccess)) {
    cudaFree(pk.w); e->rc = NRGBD_ERR_NOMEM; nrgbd_set_error("engine: cudaMalloc failed for packed weight"); return nullptr;
  }
  const int tr = transposed ? 1 : 0;
  nrgbd_stream_t st = (nrgbd_stream_t)e->st;
  if (h2) ENG_CALL(e, nrgbd_pack_conv_weight_h2(src, tr, Cout, Cin, taps, pk.Cin_pad, pk.Cout_pad, pk.w, st));
  else if (kind == PK_TC) ENG_CALL(e, nrgbd_pack_conv_weight_tc(src, tr, Cout, Cin, taps, pk.Cin_pad, pk.Cout_pad, pk.w, pk.lo, st));
  else ENG_CALL(e, nrgbd_pack_conv_weight(src, tr, Cout, Cin, taps, pk.Cin_pad, pk.Cout_pad, pk.w, st));
  return &(e->packed[name][kind] = pk);
}

// f16-pair tensor path: any conv whose activation carries its channels padded to the packed weight's Cin_pad = pad32(C).
// Channels [C, Cs) are zero in every activation (acquire() clears them, pair outputs and the K-Net volume rows store
// zeros there) and the packed weight's rows [C, Cin_pad) are zero, so the padding adds exact zeros to every sum. This
// is also the one condition under which an activation may exist only as its operand pair (the K-Net input volume).
bool use_h2(Eng* e, const Act& x) {
  return pair_mode(e) && pad32(x.C) <= x.Cs && x.Cs % 8 == 0;
}

bool use_tc(Eng* e, const Act& x, int Cout) {
  return e->conv_math == 1 && nrgbd_conv_tc_supported(pad32(x.C), pad16(Cout)) && pad32(x.C) <= x.Cs;
}

// TF32 hi / lo split of an activation into two pool buffers
void split_act(Eng* e, const Act& x, Act& hi, Act& lo) {
  hi = x; lo = x; hi.p = lo.p = nullptr;
  if (e->rc) return;
  hi.p = e->pool.acquire((size_t)x.floats() * sizeof(float));
  lo.p = e->pool.acquire((size_t)x.floats() * sizeof(float));
  if (!hi.p || !lo.p) { nrgbd_set_error("engine: out of device memory"); e->rc = NRGBD_ERR_NOMEM; return; }
  ENG_CALL(e, nrgbd_split_tf32(x.p, x.floats(), hi.p, lo.p, (nrgbd_stream_t)e->st));
}

// Output extent, algorithmic FLOPs and profile tag of a convolution; bench.py's roofline and --layer-table read the tags.
// transposed: a ConvTranspose2d, whose every output reads 1 / stride^2 of the taps.
struct ConvGeom { int Ho, Wo; double flops; char tag[56]; };
ConvGeom conv_geom(const Act& x, int Cout, int kd, int k, int stride, int pad, int dil, bool transposed = false) {
  ConvGeom g;
  const int span = dil * (k - 1) + 1;
  g.Ho = transposed ? (x.H - 1) * stride - 2 * pad + span : (x.H + 2 * pad - span) / stride + 1;
  g.Wo = transposed ? (x.W - 1) * stride - 2 * pad + span : (x.W + 2 * pad - span) / stride + 1;
  g.flops = 2.0 * x.N * x.D * g.Ho * g.Wo * Cout * x.C * kd * k * k / (transposed ? stride * stride : 1);
  if (transposed) snprintf(g.tag, sizeof(g.tag), "convT k%d s%d %d->%d %dx%dx%d", k, stride, x.C, Cout, x.N, g.Ho, g.Wo);
  else snprintf(g.tag, sizeof(g.tag), "conv%dd k%d s%d d%d %d->%d %dx%dx%dx%d", kd > 1 ? 3 : 2, k, stride, dil, x.C, Cout, x.N, x.D, g.Ho, g.Wo);
  return g;
}

// Where conv() writes. Default: a fresh activation with acquire()'s channel stride, per-channel sums into e->stats.
struct ConvOut {
  Act* dst = nullptr;                       // write into this activation instead
  int Cs = -1;                              // channel stride of the fresh activation
  double* stats = nullptr;                  // per-channel sums into this buffer instead
  const nrgbd_bn_input* in_bn = nullptr;    // 3xTF32: x is the RAW output of a conv, normalised while its operands are split
  // f16-pair mode, no BatchNorm after the conv: the result is written only as the operand pair of the convolution that
  // consumes it (y.p is a 16-byte key of the pair, y.pair_only) - no fp32 tensor, no split pass
  bool pair_only = false;
};

// conv (2-D when x.D == 1 and kd == 1)
Act conv(Eng* e, const Act& x, const std::string& wname, int Cout, int kd, int k, int stride, int pad, int dil,
         const char* bias_name, bool leaky, bool want_stats, const ConvOut& out = ConvOut()) {
  double* stats = want_stats ? (out.stats ? out.stats : e->stats) : nullptr;
  nrgbd_stream_t st = (nrgbd_stream_t)e->st;
  if (x.pair_only && !use_h2(e, x)) {          // x.p is no fp32 tensor: only the f16-pair path can read x
    if (!e->rc) { nrgbd_set_error("engine: '%s' reads an activation that exists only as an operand pair", wname.c_str()); e->rc = NRGBD_ERR_BAD_ARG; }
    return Act();
  }
  const ConvGeom g = conv_geom(x, Cout, kd, k, stride, pad, dil);
  const int taps = kd * k * k;
  float* b = bias_name ? param(e, bias_name) : nullptr;
  if (out.pair_only && use_h2(e, x) && Cout >= 16 && !out.dst && !want_stats && out.Cs < 0 && stride == 1) {
    const Packed* ph = packw(e, wname, PK_H2, Cout, x.C, taps, false);
    const PairBuf* pin = pair_of(e, x);
    PairBuf pb;
    Act y = pair_act(e, x.N, x.D, g.Ho, g.Wo, Cout, false, pb);      // R-Net: no residuals
    if (e->rc) return y;
    ProfScope ps(e, 0, g.flops, g.tag);
    ENG_CALL(e, nrgbd_conv_nhwc_h2_pair(pin->hi, conv_lo(e, pin), x.N, x.D, x.H, x.W, ph->Cin_pad, x.Cs, ph->w, b, Cout, ph->Cout_pad, ph->BN, kd, k, k,
                                        stride, pad, dil, pb.hi, pb.lo, g.Ho, g.Wo, y.Cs, leaky ? 1 : 0, st));
    return y;
  }
  Act y = out.dst ? *out.dst : acquire(e, x.N, x.D, g.Ho, g.Wo, Cout, out.Cs);
  if (e->rc) return y;
  if (stats && !pair_mode(e)) cudaMemsetAsync(stats, 0, sizeof(double) * 2 * Cout, e->st);   // f16-pair mode: kept zero by the BN pass
  if (use_h2(e, x)) {
    const Packed* ph = packw(e, wname, PK_H2, Cout, x.C, taps, false);
    const PairBuf* pb = pair_of(e, x);
    if (e->rc) return y;
    ProfScope ps(e, 0, g.flops, g.tag);
    ENG_CALL(e, nrgbd_conv_nhwc_h2(pb->hi, conv_lo(e, pb), x.N, x.D, x.H, x.W, ph->Cin_pad, x.Cs, ph->w, b, Cout, ph->Cout_pad, ph->BN, kd, k, k, stride,
                                   pad, dil, y.p, g.Ho, g.Wo, y.Cs, 0, leaky ? 1 : 0, stats, st));
    return y;
  }
  if (use_tc(e, x, Cout)) {
    const Packed* pt = packw(e, wname, PK_TC, Cout, x.C, taps, false);
    if (!e->rc && out.in_bn) {
      // x is the RAW output of the producing conv: BatchNorm + ReLU are applied in the pass that splits the operands
      // (4 B read + 8 B written per element, against 4 + 4 for a separate BatchNorm pass and 4 + 8 for the split after it)
      ProfScope ps(e, 0, g.flops, g.tag);
      ENG_CALL(e, nrgbd_conv_nhwc_tc2_bn_in(x.p, x.N, x.D, x.H, x.W, pt->Cin_pad, x.Cs, pt->w, pt->lo, b, Cout, pt->Cout_pad, kd, k, k,
                                            stride, pad, dil, y.p, g.Ho, g.Wo, y.Cs, 0, leaky ? 1 : 0, stats, out.in_bn, st));
      return y;
    }
    Act xh, xl;
    split_act(e, x, xh, xl);
    if (!e->rc) {
      ProfScope ps(e, 0, g.flops, g.tag);
      ENG_CALL(e, nrgbd_conv_nhwc_tc(xh.p, xl.p, x.N, x.D, x.H, x.W, pt->Cin_pad, x.Cs, pt->w, pt->lo, b, Cout, pt->Cout_pad, kd, k, k,
                                     stride, pad, dil, y.p, g.Ho, g.Wo, y.Cs, 0, leaky ? 1 : 0, stats, st));
    }
    release(e, xh); release(e, xl);
    return y;
  }
  const Packed* pk = packw(e, wname, PK_F32, Cout, x.C, taps, false);
  if (e->rc) return y;
  ProfScope ps(e, 0, g.flops, g.tag);
  ENG_CALL(e, nrgbd_conv_nhwc(x.p, x.N, x.D, x.H, x.W, pk->Cin_pad, x.Cs, pk->w, b, Cout, pk->Cout_pad, kd, k, k, stride,
                              pad, dil, y.p, g.Ho, g.Wo, y.Cs, 0, leaky ? 1 : 0, stats, st));
  return y;
}

// Eval mode: scale / shift of every BatchNorm that tracks running statistics (its running_mean is registered), computed on
// the device by one launch at the start of each forward. The launch is part of the captured graph, so a replay reads the
// running statistics as they are then (a train-mode forward in between may have updated them in place).
void eval_coeffs(Eng* e) {
  e->eval_slot.clear();
  if (!e->bn_eval || e->rc) return;
  const std::string suf = ".running_mean";
  std::vector<std::string> pres;
  for (auto& kv : e->params) {
    const std::string& k = kv.first;
    if (k.size() > suf.size() && k.compare(k.size() - suf.size(), suf.size(), suf) == 0) pres.push_back(k.substr(0, k.size() - suf.size()));
  }
  if (pres.empty()) return;
  if ((int)pres.size() > NRGBD_BN_EVAL_MAX) {
    nrgbd_set_error("engine: %d BatchNorm layers with running statistics, at most %d supported", (int)pres.size(), NRGBD_BN_EVAL_MAX);
    e->rc = NRGBD_ERR_UNSUPPORTED; return;
  }
  std::sort(pres.begin(), pres.end());
  BnEvalTable t{};
  t.n = (int)pres.size(); t.eps = 1e-5f;
  for (int i = 0; i < t.n; ++i) {
    const std::string& pre = pres[i];
    t.gamma[i] = param(e, pre + ".weight"); t.beta[i] = param(e, pre + ".bias");
    t.mean[i] = param(e, pre + ".running_mean"); t.var[i] = param(e, pre + ".running_var");
    if (e->rc) return;
    t.C[i] = (int)e->params[pre + ".weight"].n;
    if (t.C[i] > 512 || e->params[pre + ".running_mean"].n != t.C[i] || e->params[pre + ".running_var"].n != t.C[i]) {
      nrgbd_set_error("engine: BatchNorm '%s' has inconsistent or more than 512 channels", pre.c_str());
      e->rc = NRGBD_ERR_BAD_ARG; return;
    }
    t.scale[i] = e->eval_coef + (size_t)i * 1024; t.shift[i] = t.scale[i] + 512;
    e->eval_slot[pre] = i;
  }
  ENG_CALL(e, bn_eval_coeffs(t, e->st));
}

// eval-mode scale of BatchNorm `pre` (its shift is 512 floats further), or null: train mode, or a layer without running
// statistics (it keeps batch statistics in eval mode too)
const float* eval_coef(Eng* e, const std::string& pre) {
  auto it = e->eval_slot.find(pre);
  return it == e->eval_slot.end() ? nullptr : e->eval_coef + (size_t)it->second * 1024;
}

// Eval-mode Conv (no bias) + BatchNorm(running statistics) [+ residual] [+ ReLU] of a tracked layer. f16-pair mode: ONE
// convolution with the affine epilogue, written as the operand pair of the next convolution when only convolutions read it
// (out_use 2), else as fp32. Other modes: the convolution without statistics, then nrgbd_bn_apply. No statistic is read or
// written, no running buffer updated. res_read: a later residual add reads the pair (see convbn).
Act convbn_eval(Eng* e, const Act& x, const std::string& wname, int Cout, int kd, int k, int stride, int pad, int dil, bool relu,
                const Act* res, int out_use, const float* scale, bool res_read = false) {
  const float* shift = scale + 512;
  if (use_h2(e, x)) {
    const ConvGeom g = conv_geom(x, Cout, kd, k, stride, pad, dil);
    const Packed* ph = packw(e, wname, PK_H2, Cout, x.C, kd * k * k, false);
    const PairBuf* pin = pair_of(e, x);
    if (e->rc) return Act();
    PairBuf pb;
    Act y = out_use == 2 ? pair_act(e, x.N, x.D, g.Ho, g.Wo, Cout, res_read, pb) : acquire(e, x.N, x.D, g.Ho, g.Wo, Cout);
    if (e->rc) return y;
    if (res && (res->Cs != y.Cs || res->pos() != y.pos())) { nrgbd_set_error("engine: residual layout differs from the output's"); e->rc = NRGBD_ERR_BAD_ARG; return y; }
    const Residual r = residual_of(e, res);
    if (e->rc) return y;
    ProfScope ps(e, 0, g.flops, g.tag);
    ENG_CALL(e, nrgbd_conv_nhwc_h2_affine(pin->hi, conv_lo(e, pin), x.N, x.D, x.H, x.W, ph->Cin_pad, x.Cs, ph->w, Cout, ph->Cout_pad, ph->BN, kd, k, k,
                                          stride, pad, dil, scale, shift, r.f, r.hi, r.lo, relu ? 1 : 0, out_use == 2 ? nullptr : y.p,
                                          pb.hi, pb.lo, g.Ho, g.Wo, y.Cs, 0, (nrgbd_stream_t)e->st));
    return y;
  }
  if (res && res->pair_only) { nrgbd_set_error("engine: residual exists only as an operand pair"); e->rc = NRGBD_ERR_BAD_ARG; return Act(); }
  Act y = conv(e, x, wname, Cout, kd, k, stride, pad, dil, nullptr, false, false);
  if (!e->rc)
    ENG_CALL(e, nrgbd_bn_apply(y.p, scale, shift, res ? res->p : nullptr, relu ? 1 : 0, y.pos(), y.Cs, y.C, y.p, (nrgbd_stream_t)e->st));
  return y;
}

// Training-mode BatchNorm `pre` [+ residual] [+ ReLU] in place on the RAW conv output y, from that conv's sums `stats`
void bn_train(Eng* e, Act& y, const std::string& pre, const double* stats, const float* res, bool relu) {
  const BnParams bn = bn_params(e, pre);
  ENG_CALL(e, nrgbd_bn_apply_stats(y.p, stats, (double)y.pos(), bn.gamma, bn.beta, 1e-5f, bn.rm, bn.rv, 0.1f, res, relu ? 1 : 0,
                                   y.pos(), y.Cs, y.C, y.p, (nrgbd_stream_t)e->st));
}

// 3xTF32 descriptor of training-mode BatchNorm `pre` + ReLU on t, the RAW output of the conv whose sums are in `stats`:
// applied by the convolution that reads t while it splits its operands (nrgbd_conv_nhwc_tc2_bn_in)
nrgbd_bn_input bn_input(Eng* e, const std::string& pre, const double* stats, const Act& t) {
  const BnParams p = bn_params(e, pre);
  nrgbd_bn_input bn;
  bn.stats = stats; bn.count = (double)t.pos();
  bn.gamma = p.gamma; bn.beta = p.beta; bn.running_mean = p.rm; bn.running_var = p.rv;
  bn.eps = 1e-5f; bn.momentum = 0.1f; bn.relu = 1; bn.C = t.C;
  return bn;
}

// Conv (no bias) + BatchNorm(batch statistics) [+ ReLU] [+ residual]; BN applied in place.
// `pre` is the Sequential(Conv, BN) prefix: weights pre.0.weight, pre.1.{weight,bias,running_*}.
// out_use (f16-pair mode only): 0 = the result is read as fp32 only; 1 = also by a convolution (the BatchNorm pass emits the
// split-fp16 operand planes together with the fp32 tensor); 2 = ONLY by a convolution (no fp32 copy is written: y.p keeps
// the raw conv output and must not be read as an activation). A residual `res` that itself exists only as a pair (out_use 2
// of an earlier layer) is read from that pair. res_read (out_use 2): a later residual add reads the result, so its pair keeps
// the lo half in conv_math 3 too (elsewhere conv_math 3 writes hi only).
Act convbn(Eng* e, const Act& x, const std::string& pre, int Cout, int kd, int k, int stride, int pad, int dil,
           bool relu, const Act* res, int out_use = 0, bool res_read = false) {
  int p = (kd == 1 && dil > 1) ? dil : pad;          // psm_submodule.convbn :13
  if (const float* sc = eval_coef(e, pre + ".1"))
    return convbn_eval(e, x, pre + ".0.weight", Cout, kd, k, stride, p, dil, relu, res, out_use, sc, res_read);
  Act y = conv(e, x, pre + ".0.weight", Cout, kd, k, stride, p, dil, nullptr, false, true);
  if (!pair_mode(e)) { bn_train(e, y, pre + ".1", e->stats, res ? res->p : nullptr, relu); return y; }
  const BnParams bn = bn_params(e, pre + ".1");
  if (e->rc) return y;
  const bool pair = out_use && use_h2(e, y);
  PairBuf pb;
  // out_use 1: a residual add reads the fp32 copy
  if (pair && !acquire_pair(e, y.floats(), keep_lo(e, res_read && out_use == 2), pb)) return y;
  const Residual r = residual_of(e, res);
  if (e->rc) return y;
  ENG_CALL(e, nrgbd_bn_apply_stats_pair(y.p, e->stats, (double)y.pos(), bn.gamma, bn.beta, 1e-5f, bn.rm, bn.rv, 0.1f, r.f, r.hi, r.lo,
                                        relu ? 1 : 0, y.pos(), y.Cs, y.C, (pair && out_use == 2) ? nullptr : y.p, pb.hi, pb.lo,
                                        e->bn_counter, (nrgbd_stream_t)e->st));
  y.pair_only = pair && out_use == 2;
  if (pair) e->pairs[y.p] = pb;
  return y;
}

// Whether conv `Cin -> Cout` at this activation takes the 3xTF32 path that can fold an input BN into its operand split
bool takes_tc2(Eng* e, const Act& x, int Cout) {
  return use_tc(e, x, Cout) && nrgbd_conv_tc2_supported(pad32(x.C), pad16(Cout));
}

// psm_submodule.BasicBlock :31-49
// fp32_out: the block's output is read as an fp32 tensor by something other than a convolution / residual add (f16-pair mode:
// otherwise only its operand pair is written)
Act basic_block(Eng* e, Act& x, const std::string& pre, int planes, int stride, int dil, bool down, bool fp32_out = true) {
  const int p1 = dil > 1 ? dil : 1;                  // psm_submodule.convbn :13
  // Fused form (3xTF32 path): conv1 leaves its RAW output and per-channel sums; BN1 + ReLU are applied by conv2 while it
  // splits its operands (nrgbd_conv_nhwc_tc2_bn_in) - one read + one write of the activation less per block.
  Act probe = x; probe.C = planes; probe.Cs = pad32(planes);
  const bool fused = takes_tc2(e, x, planes) && takes_tc2(e, probe, planes);
  Act t;
  if (fused) {
    ConvOut raw; raw.stats = e->stats_b;
    t = conv(e, x, pre + ".conv1.0.0.weight", planes, 1, 3, stride, p1, dil, nullptr, false, true, raw);
  } else {
    t = convbn(e, x, pre + ".conv1.0", planes, 1, 3, stride, 1, dil, true, nullptr, 2);
  }
  Act sc; const Act* res = &x;
  if (down) {      // downsample = Sequential(Conv2d 1x1 stride, BatchNorm2d) :125-131
    sc = convbn(e, x, pre + ".downsample", planes, 1, 1, stride, 0, 1, false, nullptr);
    res = &sc;
  }
  Act o;
  if (fused) {
    const nrgbd_bn_input bn = bn_input(e, pre + ".conv1.0.1", e->stats_b, t);
    ConvOut bn_in; bn_in.in_bn = &bn;
    o = conv(e, t, pre + ".conv2.0.weight", planes, 1, 3, 1, p1, dil, nullptr, false, true, bn_in);
    bn_train(e, o, pre + ".conv2.1", e->stats, res->p, false);
  } else {
    // a block output that exists only as a pair is the residual of the next block (layer1-3 inner blocks, layer3 -> layer4.0)
    o = convbn(e, t, pre + ".conv2", planes, 1, 3, 1, 1, dil, false, res, fp32_out ? 1 : 2, true);
  }
  release(e, t);
  if (down) release(e, sc);
  return o;
}

Act make_layer(Eng* e, Act x, bool own_x, const std::string& pre, int planes, int blocks, int stride, int dil, bool down,
               bool fp32_out = true) {
  Act cur = x;
  for (int i = 0; i < blocks; ++i) {
    Act o = basic_block(e, cur, pre + "." + std::to_string(i), planes, i == 0 ? stride : 1, dil, down && i == 0,
                        i == blocks - 1 ? fp32_out : false);
    if (i > 0 || own_x) release(e, cur);
    cur = o;
  }
  return cur;
}

// psm_submodule.feature_extraction.forward :141-167 -> (layer1 output @1/2, features @1/4)
void feature_cnn(Eng* e, const Act& x0, Act& l1_out, Act& feat_out) {
  const std::string P = "feature_extractor.feature_extraction";
  // firstconv = convbn+ReLU x3 (psm_submodule.py:90-92). 3xTF32 path: the first two BatchNorm+ReLU are folded into the
  // operand split of the conv that consumes them (the raw 5x240x320x32 tensors are read once instead of read+written+read).
  Act c;
  Act probe32 = x0; probe32.C = 32; probe32.Cs = pad32(32); probe32.H = (x0.H + 2 - 3) / 2 + 1; probe32.W = (x0.W + 2 - 3) / 2 + 1;
  if (takes_tc2(e, probe32, 32)) {
    ConvOut oa; oa.Cs = pad32(32); oa.stats = e->stats_b;
    Act a = conv(e, x0, P + ".firstconv.0.0.weight", 32, 1, 3, 2, 1, 1, nullptr, false, true, oa);
    const nrgbd_bn_input bn_a = bn_input(e, P + ".firstconv.0.1", e->stats_b, a);
    ConvOut ob; ob.in_bn = &bn_a;
    Act b = conv(e, a, P + ".firstconv.2.0.weight", 32, 1, 3, 1, 1, 1, nullptr, false, true, ob);
    release(e, a);
    const nrgbd_bn_input bn_b = bn_input(e, P + ".firstconv.2.1", e->stats, b);
    ConvOut oc; oc.stats = e->stats_b; oc.in_bn = &bn_b;
    c = conv(e, b, P + ".firstconv.4.0.weight", 32, 1, 3, 1, 1, 1, nullptr, false, true, oc);
    release(e, b);
    bn_train(e, c, P + ".firstconv.4.1", e->stats_b, nullptr, true);
  } else {
    Act a = convbn(e, x0, P + ".firstconv.0", 32, 1, 3, 2, 1, 1, true, nullptr, 2);
    Act b = convbn(e, a, P + ".firstconv.2", 32, 1, 3, 1, 1, 1, true, nullptr, 2); release(e, a);
    c = convbn(e, b, P + ".firstconv.4", 32, 1, 3, 1, 1, 1, true, nullptr, 2, true); release(e, b);     // layer1.0 reads it as conv input and as residual: pair only
  }
  Act l1 = make_layer(e, c, true, P + ".layer1", 32, 3, 1, 1, false);
  Act raw = make_layer(e, l1, false, P + ".layer2", 64, 16, 2, 1, true);
  Act l3 = make_layer(e, raw, false, P + ".layer3", 128, 3, 1, 1, true, false);     // feeds layer4 only (conv input + residual)
  Act skip = make_layer(e, l3, true, P + ".layer4", 128, 3, 1, 2, false);
  Act cat = acquire(e, skip.N, 1, skip.H, skip.W, 320);
  if (!e->rc) {
    ENG_CALL(e, nrgbd_copy_channels(raw.p, raw.pos(), raw.Cs, 0, 64, 0, cat.p, cat.Cs, 0, (nrgbd_stream_t)e->st));
    ENG_CALL(e, nrgbd_copy_channels(skip.p, skip.pos(), skip.Cs, 0, 128, 0, cat.p, cat.Cs, 64, (nrgbd_stream_t)e->st));
  }
  // cat order (:161): raw, skip, branch4, branch3, branch2, branch1.
  // SPP pooling (AvgPool2d 64/32/16/8, psm_submodule.py:103-117) is built hierarchically: the 8x8 means
  // once from the feature map, then 16/32/64 as 2x2 means of the previous level (window origins are
  // aligned multiples, so the result is the same mean; a 64x64 window pooled directly would run on
  // N*1*2 blocks only).
  const int ks[4] = {64, 32, 16, 8};
  const int offs[4] = {288, 256, 224, 192};
  Act pools[4];
  for (int bi = 3; bi >= 0 && !e->rc; --bi) {
    const int k = ks[bi];
    if (skip.H / k < 1 || skip.W / k < 1) {
      nrgbd_set_error("engine: frame too small for the SPP AvgPool2d(%d) branch (need H/4, W/4 >= 64)", k);
      e->rc = NRGBD_ERR_BAD_ARG; break;
    }
    pools[bi] = acquire(e, skip.N, 1, skip.H / k, skip.W / k, 128);
    if (bi == 3) {
      ENG_CALL(e, nrgbd_avgpool_nhwc(skip.p, skip.N, skip.H, skip.W, skip.Cs, 128, 8, pools[bi].p, pools[bi].Cs, 0, (nrgbd_stream_t)e->st));
    } else {
      const Act& f = pools[bi + 1];
      ENG_CALL(e, nrgbd_avgpool_nhwc(f.p, f.N, f.H, f.W, f.Cs, 128, 2, pools[bi].p, pools[bi].Cs, 0, (nrgbd_stream_t)e->st));
    }
  }
  for (int bi = 0; bi < 4 && !e->rc; ++bi) {
    Act& pl = pools[bi];
    Act br = convbn(e, pl, P + ".branch" + std::to_string(bi + 1) + ".1", 32, 1, 1, 1, 0, 1, true, nullptr);
    ENG_CALL(e, nrgbd_upsample_bilinear_ac_nhwc(br.p, br.N, br.H, br.W, br.Cs, 32, cat.p, cat.H, cat.W, cat.Cs, offs[bi],
                                                (nrgbd_stream_t)e->st));
    release(e, br);
  }
  for (int bi = 0; bi < 4; ++bi) release(e, pools[bi]);
  release(e, raw); release(e, skip);
  Act lc = convbn(e, cat, P + ".lastconv.0", 128, 1, 3, 1, 1, 1, true, nullptr, 2);
  release(e, cat);
  ConvOut dense; dense.Cs = pad4(e->F);                              // the sweep's wide layout
  feat_out = conv(e, lc, P + ".lastconv.2.weight", e->F, 1, 1, 1, 0, 1, nullptr, false, false, dense);
  release(e, lc);
  l1_out = l1;
}

// ConvTranspose2d(k4, s2, p1) + bias + LeakyReLU into channels [0, Cout) of dst
void conv_transpose(Eng* e, const Act& x, const std::string& wname, const char* bias_name, int Cout, Act& dst) {
  float* tb = param(e, bias_name);
  if (e->rc) return;
  nrgbd_stream_t st = (nrgbd_stream_t)e->st;
  const ConvGeom g = conv_geom(x, Cout, 1, 4, 2, 1, 1, true);
  if (use_h2(e, x)) {
    const Packed* ph = packw(e, wname, PK_H2, Cout, x.C, 16, true);
    const PairBuf* pb = pair_of(e, x);
    if (e->rc) return;
    ProfScope ps(e, 0, g.flops, g.tag);
    ENG_CALL(e, nrgbd_conv_transpose2d_k4s2_nhwc_h2(pb->hi, conv_lo(e, pb), x.N, x.H, x.W, ph->Cin_pad, x.Cs, ph->w, tb, Cout, ph->Cout_pad, ph->BN,
                                                    dst.p, dst.Cs, 0, 1, st));
    return;
  }
  if (use_tc(e, x, Cout)) {
    const Packed* pt = packw(e, wname, PK_TC, Cout, x.C, 16, true);
    if (!e->rc && nrgbd_conv_tc2_supported(pt->Cin_pad, pt->Cout_pad)) {
      ProfScope ps(e, 0, g.flops, g.tag);
      ENG_CALL(e, nrgbd_conv_transpose2d_k4s2_nhwc_tc2(x.p, x.N, x.H, x.W, pt->Cin_pad, x.Cs, pt->w, pt->lo, tb, Cout, pt->Cout_pad,
                                                       dst.p, dst.Cs, 0, 1, st));
      return;
    }
    Act xh, xl;
    split_act(e, x, xh, xl);
    if (!e->rc) {
      ProfScope ps(e, 0, g.flops, g.tag);
      ENG_CALL(e, nrgbd_conv_transpose2d_k4s2_nhwc_tc(xh.p, xl.p, x.N, x.H, x.W, pt->Cin_pad, x.Cs, pt->w, pt->lo, tb, Cout, pt->Cout_pad,
                                                      dst.p, dst.Cs, 0, 1, st));
    }
    release(e, xh); release(e, xl);
    return;
  }
  const Packed* pk = packw(e, wname, PK_F32, Cout, x.C, 16, true);
  if (e->rc) return;
  ProfScope ps(e, 0, g.flops, g.tag);
  ENG_CALL(e, nrgbd_conv_transpose2d_k4s2_nhwc(x.p, x.N, x.H, x.W, pk->Cin_pad, x.Cs, pk->w, tb, Cout, pk->Cout_pad, dst.p, dst.Cs, 0, 1, st));
}

// models/Refine.py:79-107. prob source: log-DPV pixel-major [hw][D]; returns log-DPV [H*W][D1]. The transposed convolutions
// widen the DPV to D0 and D1 planes: D0 = D1 = D, or with if_upsample_d D0 = 2D, D1 = 4D (Refine.py:44-48).
void r_net(Eng* e, const float* bv_hwd, const float* feat_ref, int feat_Cs, const float* l1_ref, int l1_Cs, const Act& frame_ref, Act& out) {
  const int D = e->D, h = e->h, w = e->w, H = e->H, W = e->W, F = e->F;
  const int D0 = e->refine_up ? 2 * D : D, D1 = e->refine_up ? 4 * D : D;
  const long long hw = (long long)h * w;
  nrgbd_stream_t st = (nrgbd_stream_t)e->st;
  Act in0 = acquire(e, 1, 1, h, w, D + F);
  if (!e->rc) {
    ENG_CALL(e, nrgbd_copy_channels(bv_hwd, hw, D, 0, D, 1, in0.p, in0.Cs, 0, st));           // torch.exp(BV)
    ENG_CALL(e, nrgbd_copy_channels(feat_ref, hw, feat_Cs, 0, F, 0, in0.p, in0.Cs, D, st));
  }
  ConvOut pair; pair.pair_only = true;          // conv0 ... conv2_1: each one's only reader is the next convolution
  Act a = conv(e, in0, "r_net.conv0.0.weight", D + F, 1, 3, 1, 1, 1, "r_net.conv0.0.bias", true, false, pair); release(e, in0);
  Act b = conv(e, a, "r_net.conv0_1.0.weight", D + F, 1, 3, 1, 1, 1, "r_net.conv0_1.0.bias", true, false, pair); release(e, a);
  Act t0 = acquire(e, 1, 1, 2 * h, 2 * w, D0 + F / 2);
  conv_transpose(e, b, "r_net.trans_conv0.0.weight", "r_net.trans_conv0.0.bias", D0, t0);
  if (!e->rc) ENG_CALL(e, nrgbd_copy_channels(l1_ref, 4 * hw, l1_Cs, 0, F / 2, 0, t0.p, t0.Cs, D0, st));
  release(e, b);
  Act c = conv(e, t0, "r_net.conv1.0.weight", D0 + F / 2, 1, 3, 1, 1, 1, "r_net.conv1.0.bias", true, false, pair); release(e, t0);
  Act d = conv(e, c, "r_net.conv1_1.0.weight", D0 + F / 2, 1, 3, 1, 1, 1, "r_net.conv1_1.0.bias", true, false, pair); release(e, c);
  Act t1 = acquire(e, 1, 1, H, W, D1 + 3);
  conv_transpose(e, d, "r_net.trans_conv1.0.weight", "r_net.trans_conv1.0.bias", D1, t1);
  if (!e->rc) ENG_CALL(e, nrgbd_copy_channels(frame_ref.p, (long long)H * W, frame_ref.Cs, 0, 3, 0, t1.p, t1.Cs, D1, st));
  release(e, d);
  Act f = conv(e, t1, "r_net.conv2.0.weight", D1 + 3, 1, 3, 1, 1, 1, "r_net.conv2.0.bias", true, false, pair); release(e, t1);
  Act g = conv(e, f, "r_net.conv2_1.0.weight", D1, 1, 3, 1, 1, 1, "r_net.conv2_1.0.bias", true, false, pair); release(e, f);
  ConvOut into_out; into_out.dst = &out;
  conv(e, g, "r_net.conv2_2.weight", D1, 1, 3, 1, 1, 1, "r_net.conv2_2.bias", false, false, into_out); release(e, g);
  // F.log_softmax(conv2_2_out, dim=1): channels are contiguous per pixel (Cs == D1); above 256 planes dpv_normalize takes
  // its thread-per-pixel path
  if (!e->rc)
    ENG_CALL(e, nrgbd_dpv_normalize(out.p, 1, D1, nullptr, 0, 0, 1.f, H * W, D1, out.p, 1, D1, nullptr, nullptr, nullptr, st));
}

// models/KVNET.py:129-132,176-178 with refineNet_name='DGF': expected depth of the low-resolution log-DPV in
// depth_val_regression's sequential order (mutils/misc.py:541-546; dpv_normalize's warp-reduced depth is not that order),
// then RefineNet_DGF (Refine.py:620-641) guided by the reference frame; out [H][W] depth.
void dgf_refine(Eng* e, const float* bv_hwd, const Act& frame_ref, float* out) {
  const int D = e->D, h = e->h, w = e->w, H = e->H, W = e->W;
  const long long hw = (long long)h * w;
  nrgbd_stream_t st = (nrgbd_stream_t)e->st;
  const float* w0 = param(e, "r_net.feature_ext.0.weight");
  const float* b0 = param(e, "r_net.feature_ext.0.bias");
  const float* w1 = param(e, "r_net.feature_ext.2.weight");
  const float* b1 = param(e, "r_net.feature_ext.2.bias");
  if (e->rc) return;
  float* dmap = e->pool.acquire((size_t)hw * sizeof(float));
  float* ws = e->pool.acquire((size_t)nrgbd_guided_filter_workspace_floats(H, W) * sizeof(float));
  if (!dmap || !ws) { nrgbd_set_error("engine: out of device memory (guided filter)"); e->rc = NRGBD_ERR_NOMEM; }
  ENG_CALL(e, nrgbd_depth_regression(bv_hwd, (int)hw, D, 1, D, e->d_planes, 1, dmap, nullptr, st));
  ENG_CALL(e, nrgbd_guided_filter_refine(dmap, h, w, frame_ref.p, 1, frame_ref.Cs, H, W, w0, b0, w1, b1, 1, 1e-8f, ws, out, st));
  if (dmap) e->pool.release(dmap);
  if (ws) e->pool.release(ws);
}

// models/basic.py:113-139 on a channels-last volume [D][h][w][CK] -> gain [D][hw] (DHW, Cs = 1)
Act kv_net(Eng* e, const Act& vol) {
  const int f = e->KF;
  auto cb = [&](const Act& x, const std::string& name, bool relu, const Act* res, int out_use, bool res_read) {
    return convbn(e, x, name, f, 3, 3, 1, 1, 1, relu, res, out_use, res_read);
  };
  Act a = cb(vol, "kv_net.dres0.0", true, nullptr, 2, false);
  // in f16-pair mode no K-Net activation has an fp32 copy: convolutions read the operand pairs, and so do the residual adds
  Act c = cb(a, "kv_net.dres0.2", true, nullptr, 2, true); release(e, a);      // also the residual of dres1
  for (int i = 1; i <= 4; ++i) {
    std::string p = "kv_net.dres" + std::to_string(i);
    Act r = cb(c, p + ".0", true, nullptr, 2, false);
    Act o = cb(r, p + ".2", false, &c, 2, i < 4);                              // the residual of dres(i + 1)
    release(e, r); release(e, c);
    c = o;
  }
  Act o = cb(c, "kv_net.classify.0", true, nullptr, 2, false); release(e, c);
  Act gain;
  if (use_h2(e, o)) {
    // Conv3d(f -> 1, k3) (models/basic.py:136-137) as a pointwise conv to 27 per-tap channels on the tensor cores + the shifted
    // sum of the taps: as a direct implicit GEMM its N is 1 (27 x 12 sixteen-column MMAs per 128 positions, issue-bound)
    const Packed* ph = packw(e, "kv_net.classify.2.weight", PK_H2_TAPS, 27, o.C, 1, true);
    const PairBuf* pb = pair_of(e, o);
    Act q; q.N = o.N; q.D = o.D; q.H = o.H; q.W = o.W; q.C = 27; q.Cs = 28; q.p = nullptr;
    gain = acquire(e, o.N, o.D, o.H, o.W, 1, 1);
    if (!e->rc) {
      q.p = e->pool.acquire((size_t)q.floats() * sizeof(float));      // pad channel 27 is never read: no memset
      if (!q.p) { nrgbd_set_error("engine: out of device memory (%lld floats)", q.floats()); e->rc = NRGBD_ERR_NOMEM; }
    }
    if (!e->rc) {
      char tag[56];
      snprintf(tag, sizeof(tag), "conv3d k3 s1 d1 %d->1 %dx%dx%dx%d", o.C, o.N, o.D, o.H, o.W);
      ProfScope ps(e, 0, 2.0 * (double)o.pos() * o.C * 27, tag);
      ENG_CALL(e, nrgbd_conv_nhwc_h2(pb->hi, conv_lo(e, pb), o.N, o.D, o.H, o.W, ph->Cin_pad, o.Cs, ph->w, nullptr, 27, ph->Cout_pad, ph->BN, 1, 1, 1, 1,
                                     0, 1, q.p, o.H, o.W, q.Cs, 0, 0, nullptr, (nrgbd_stream_t)e->st));
      ENG_CALL(e, nrgbd_tap_gather_sum(q.p, o.N, o.D, o.H, o.W, q.Cs, 3, 3, 0.f, gain.p, (nrgbd_stream_t)e->st));
    }
    if (q.p) e->pool.release(q.p);
  } else {
    ConvOut dense; dense.Cs = 1;
    gain = conv(e, o, "kv_net.classify.2.weight", 1, 3, 3, 1, 1, 1, nullptr, false, false, dense);
  }
  release(e, o);
  return gain;
}

// rt[v*9 + i*3 + j] = pose_v[i][j]; rt[9V + v*3 + i] = pose_v[i][3]
__global__ void gather_rt_kernel(const float* __restrict__ poses, int V, float* __restrict__ rt) {
  int i = threadIdx.x;
  if (i < 9 * V) { int v = i / 9, r = (i % 9) / 3, c = i % 3; rt[i] = poses[v * 16 + r * 4 + c]; }
  else if (i < 12 * V) { int k = i - 9 * V, v = k / 3, r = k % 3; rt[i] = poses[v * 16 + r * 4 + 3]; }
}

void drop_graphs(Eng* e) {
  for (auto& g : e->graphs) cudaGraphExecDestroy(g.exec);
  e->graphs.clear();
  e->warm = false; e->warm_steady = false;
}

int upload(float** dst, const float* host, size_t n) {
  if (*dst) { cudaFree(*dst); *dst = nullptr; }
  if (cudaMalloc((void**)dst, n * sizeof(float)) != cudaSuccess) return NRGBD_ERR_NOMEM;
  if (cudaMemcpy(*dst, host, n * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return NRGBD_ERR_CUDA;
  return NRGBD_OK;
}

}  // namespace

extern "C" {

int nrgbd_kvnet_create(int H, int W, int D, int V, int feature_dim, int kv_feature_dim, float sigma, int metric,
                       nrgbd_kvnet** out) {
  NRGBD_REQUIRE(out, "null handle pointer");
  NRGBD_REQUIRE(H > 0 && W > 0 && H % 4 == 0 && W % 4 == 0, "H and W must be positive multiples of 4");
  NRGBD_REQUIRE(H / 4 >= 64 && W / 4 >= 64, "H/4 and W/4 must be >= 64 (SPP AvgPool2d(64), psm_submodule.py:103)");
  NRGBD_REQUIRE(D > 0 && V > 0 && feature_dim > 0 && feature_dim % 8 == 0 && kv_feature_dim > 0 && kv_feature_dim % 4 == 0,
                "bad network dimensions");
  NRGBD_REQUIRE(metric == 0 || metric == 1, "undefined metric for feature distance ...");
  nrgbd_kvnet* e = new nrgbd_kvnet();
  e->H = H; e->W = W; e->D = D; e->V = V; e->F = feature_dim; e->KF = kv_feature_dim;
  e->h = H / 4; e->w = W / 4; e->sigma = sigma; e->metric = metric;
  const size_t hw = (size_t)e->h * e->w;
  bool ok = cudaMalloc((void**)&e->stats, sizeof(double) * 2 * 512) == cudaSuccess &&
            cudaMalloc((void**)&e->stats_b, sizeof(double) * 2 * 512) == cudaSuccess &&
            cudaMalloc((void**)&e->bn_counter, sizeof(unsigned int)) == cudaSuccess &&
            cudaMalloc((void**)&e->eval_coef, sizeof(float) * 1024 * NRGBD_BN_EVAL_MAX) == cudaSuccess &&
            cudaMalloc((void**)&e->ws_sweep, sizeof(float) * 12 * V) == cudaSuccess &&
            cudaMalloc((void**)&e->bv_cur_hwd, sizeof(float) * hw * D) == cudaSuccess &&
            cudaMalloc((void**)&e->dpv_hwd, sizeof(float) * hw * D) == cudaSuccess &&
            cudaMalloc((void**)&e->prior_hwd, sizeof(float) * hw * D) == cudaSuccess &&
            cudaMalloc((void**)&e->depth, sizeof(float) * hw) == cudaSuccess &&
            cudaMalloc((void**)&e->conf, sizeof(float) * hw) == cudaSuccess;
  if (!ok) { nrgbd_set_error("nrgbd_kvnet_create: cudaMalloc failed"); delete e; return NRGBD_ERR_NOMEM; }
  cudaMemset(e->stats, 0, sizeof(double) * 2 * 512); cudaMemset(e->stats_b, 0, sizeof(double) * 2 * 512); cudaMemset(e->bn_counter, 0, sizeof(unsigned int));
  *out = e;
  return NRGBD_OK;
}

int nrgbd_kvnet_destroy(nrgbd_kvnet* e) {
  if (!e) return NRGBD_OK;
  for (auto& kv : e->params) if (kv.second.owned) cudaFree(kv.second.p);
  for (auto& kv : e->packed) free_packed(kv.second);
  for (int i = 0; i < 2; ++i) { cudaFree(e->cam[i].K); cudaFree(e->cam[i].rays); }
  cudaFree(e->d_planes); cudaFree(e->stats); cudaFree(e->stats_b); cudaFree(e->bn_counter); cudaFree(e->eval_coef); cudaFree(e->ws_sweep);
  cudaFree(e->bv_cur_hwd); cudaFree(e->dpv_hwd); cudaFree(e->prior_hwd); cudaFree(e->depth); cudaFree(e->conf);
  cudaFree(e->x0_buf); cudaFree(e->rt_buf); cudaFree(e->ref_cur_hwd); cudaFree(e->ref_kv_hwd);
  drop_graphs(e);
  e->pool.destroy();
  for (auto& r : e->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (auto ev : e->ev_free) cudaEventDestroy(ev);
  delete e;
  return NRGBD_OK;
}

// Register a parameter under its reference state_dict name. is_device != 0: `data` is a device
// pointer the engine borrows (must outlive the engine or be re-set); else a host array that is copied.
// Setting a conv weight again drops every packed copy of it.
int nrgbd_kvnet_set_param(nrgbd_kvnet* e, const char* name, const float* data, long long n, int is_device) {
  NRGBD_REQUIRE(e && name && data && n > 0, "bad arguments");
  drop_graphs(e);
  std::string key(name);
  if (key.rfind("module.", 0) == 0) key = key.substr(7);                         // DataParallel prefix
  const std::string alias = "d_net.feature_extraction.";                          // same tensors, second name (KVNET.py:63-67)
  if (key.rfind(alias, 0) == 0) key = "feature_extractor." + key.substr(alias.size());
  auto it = e->params.find(key);
  if (it != e->params.end()) {
    if (it->second.owned) cudaFree(it->second.p);
    e->params.erase(it);
  }
  auto pk = e->packed.find(key);
  if (pk != e->packed.end()) { free_packed(pk->second); e->packed.erase(pk); }
  ParamRef r; r.n = n; r.owned = !is_device;
  if (is_device) {
    r.p = const_cast<float*>(data);
  } else {
    void* q = nullptr;
    NRGBD_CUDA_CHECK(cudaMalloc(&q, n * sizeof(float)));
    NRGBD_CUDA_CHECK(cudaMemcpy(q, data, n * sizeof(float), cudaMemcpyHostToDevice));
    r.p = (float*)q;
  }
  e->params[key] = r;
  return NRGBD_OK;
}

// slot 0: the intrinsics captured at construction (D-Net sweep, KVNET.py:64-67 / basic.py:270-278)
// slot 1: the per-call intrinsics (K-Net image warp KVNET.py:160-161 and DPV propagation)
// K_host 3x3 (intrinsic_M_cuda), rays_host 3 x (h*w) (unit_ray_array_2D), cx/cy from intrinsic_M,
// hfov/vfov in degrees.
int nrgbd_kvnet_set_camera(nrgbd_kvnet* e, int slot, const float* K_host, const float* rays_host, float cx, float cy,
                           double hfov_deg, double vfov_deg) {
  NRGBD_REQUIRE(e && (slot == 0 || slot == 1) && K_host && rays_host, "bad arguments");
  drop_graphs(e);
  Camera& c = e->cam[slot];
  int rc = upload(&c.K, K_host, 9);
  if (rc == NRGBD_OK) rc = upload(&c.rays, rays_host, (size_t)3 * e->h * e->w);
  if (rc != NRGBD_OK) { nrgbd_set_error("nrgbd_kvnet_set_camera: upload failed"); return rc; }
  c.cx = cx; c.cy = cy;
  c.tan_hh = (float)std::tan(hfov_deg * M_PI / 180.0 * .5);
  c.tan_hv = (float)std::tan(vfov_deg * M_PI / 180.0 * .5);
  c.set = true;
  return NRGBD_OK;
}

int nrgbd_kvnet_set_planes(nrgbd_kvnet* e, const float* d_host, int D) {
  NRGBD_REQUIRE(e && d_host && D == e->D, "d_candi length must equal the engine's D");
  drop_graphs(e);
  e->d_host.assign(d_host, d_host + D);
  int rc = upload(&e->d_planes, d_host, D);
  if (rc != NRGBD_OK) nrgbd_set_error("nrgbd_kvnet_set_planes: upload failed");
  return rc;
}

int nrgbd_kvnet_set_option(nrgbd_kvnet* e, const char* key, int value) {
  NRGBD_REQUIRE(e && key, "bad arguments");
  std::string k(key);
  if (k == "bn_update_running") { drop_graphs(e); e->bn_update_running = value; return NRGBD_OK; }
  if (k == "profile") { e->profile = value; return NRGBD_OK; }
  if (k == "bn_eval") { drop_graphs(e); e->bn_eval = value ? 1 : 0; return NRGBD_OK; }
  if (k == "use_graph") { drop_graphs(e); e->use_graph = value; return NRGBD_OK; }
  if (k == "refine") {               // 0: DPV R-Net (default); 1: guided filter (DGF); 2: none
    if (value < 0 || value > 2) { nrgbd_set_error("refine must be 0 (DPV), 1 (DGF) or 2 (none)"); return NRGBD_ERR_BAD_ARG; }
    if (e->refine != value) drop_graphs(e);
    e->refine = value;
    return NRGBD_OK;
  }
  if (k == "refine_upsample_d") {    // DPV R-Net with if_upsample_d: refined outputs of 4D planes
    if (e->refine_up != (value ? 1 : 0)) drop_graphs(e);
    e->refine_up = value ? 1 : 0;
    return NRGBD_OK;
  }
  if (k == "conv_math") {            // 0: exact fp32 (CUDA cores); 1: wgmma 3xTF32; 2: wgmma split-fp16 pairs; 3: single fp16 products
    if (value < 0 || value > 3) { nrgbd_set_error("conv_math must be 0 (fp32), 1 (tf32x3), 2 (f16x3) or 3 (f16)"); return NRGBD_ERR_BAD_ARG; }
    drop_graphs(e); e->conv_math = value;
    // f16-pair mode keeps the statistics buffers zero between uses (the BatchNorm pass re-zeroes what it consumed)
    cudaMemset(e->stats, 0, sizeof(double) * 2 * 512); cudaMemset(e->stats_b, 0, sizeof(double) * 2 * 512); cudaMemset(e->bn_counter, 0, sizeof(unsigned int));
    return NRGBD_OK;
  }
  nrgbd_set_error("nrgbd_kvnet_set_option: unknown option '%s'", key);
  return NRGBD_ERR_BAD_ARG;
}

long long nrgbd_kvnet_workspace_bytes(nrgbd_kvnet* e) { return e ? (long long)e->pool.total : 0; }

// Sum of the event-timed durations (ms), work units and launch count of one profiled kernel
// category since the last read (category 0: conv kernels, work = algorithmic flops; 1: plane sweep,
// work = algorithmic bytes). Synchronises on the recorded events and clears the records.
int nrgbd_kvnet_profile_read(nrgbd_kvnet* e, int category, double* ms, double* work, long long* launches) {
  NRGBD_REQUIRE(e && ms && work && launches, "bad arguments");
  *ms = 0; *work = 0; *launches = 0;
  std::vector<nrgbd_kvnet::ProfRec> keep;
  for (auto& r : e->prof) {
    if (r.cat != category) { keep.push_back(r); continue; }
    float t = 0.f;
    NRGBD_CUDA_CHECK(cudaEventSynchronize(r.b));
    NRGBD_CUDA_CHECK(cudaEventElapsedTime(&t, r.a, r.b));
    *ms += t; *work += r.work; *launches += 1;
    e->ev_free.push_back(r.a); e->ev_free.push_back(r.b);
  }
  e->prof.swap(keep);
  return NRGBD_OK;
}

// Per-shape table of the profiled launches of one category (development / DESIGN.md tables): text lines
// "tag;launches;total_ms;work" aggregated by tag, written to buf (NUL-terminated, truncated to cap).
// Does not clear the records.
int nrgbd_kvnet_profile_table(nrgbd_kvnet* e, int category, char* buf, long long cap) {
  NRGBD_REQUIRE(e && buf && cap > 0, "bad arguments");
  std::map<std::string, std::array<double, 3>> agg;
  for (auto& r : e->prof) {
    if (r.cat != category) continue;
    float t = 0.f;
    NRGBD_CUDA_CHECK(cudaEventSynchronize(r.b));
    NRGBD_CUDA_CHECK(cudaEventElapsedTime(&t, r.a, r.b));
    auto& a = agg[r.tag];
    a[0] += 1; a[1] += t; a[2] += r.work;
  }
  std::string out;
  char line[160];
  for (auto& kv : agg) {
    snprintf(line, sizeof(line), "%s;%d;%.6f;%.6e\n", kv.first.c_str(), (int)kv.second[0], kv.second[1], kv.second[2]);
    out += line;
  }
  snprintf(buf, (size_t)cap, "%s", out.c_str());
  return NRGBD_OK;
}

// One depth frame (models/KVNET.py:93-185, if_refined=True, refineNet_name='DPV').
//  frames  [V+1][3][H][W]  source views then the reference frame (basic.py:245 cat order), device
//  poses   [V][4][4]       relative poses E_src.E_ref^-1, device
//  bv_predict [D][h][w] or NULL: NULL -> first-window branch (:138-140). (The NaN-sentinel test of
//  :142 reads one element on the host and is done by the caller.)
//  outputs (device, any may be NULL): dmap_cur_refined [D][H][W], dmap_refined [D][H][W] (option "refine" 1: [H][W] depth;
//  2: both must be NULL),
//  bv_cur [D][h][w], dpv [D][h][w]; depth_lowres/conf_lowres [h][w] = expected depth / max prob of dpv.
// ---- one depth frame = eager head -> core (CUDA graph) -> eager tail --------------------------------
// head: caller inputs -> engine-owned buffers (frames to channels-last, R|t gather, prior to pixel-major)
// core: D-Net, R-Net, [K-Net, R-Net] entirely on engine-owned memory (graph-captured per branch/need-set)
// tail: engine results -> caller tensors in the reference layouts ([D][H][W] / [D][h][w])
// The refined-output buffers are sized by the refinement option; a change of option drops the graphs that captured them.
static int ensure_io_buffers(nrgbd_kvnet* e) {
  const size_t HW = (size_t)e->H * e->W;
  if (!e->x0_buf) {
    bool ok = cudaMalloc((void**)&e->x0_buf, sizeof(float) * (e->V + 1) * HW * 4) == cudaSuccess &&
              cudaMalloc((void**)&e->rt_buf, sizeof(float) * 12 * e->V) == cudaSuccess;
    if (!ok) { nrgbd_set_error("engine: cudaMalloc failed for the I/O staging buffers"); return NRGBD_ERR_NOMEM; }
    cudaMemset(e->x0_buf, 0, sizeof(float) * (e->V + 1) * HW * 4);      // pad channel stays 0
  }
  const long long need = (long long)HW * e->refined_planes();
  if (need != e->ref_floats) {
    cudaFree(e->ref_cur_hwd); cudaFree(e->ref_kv_hwd);
    e->ref_cur_hwd = e->ref_kv_hwd = nullptr; e->ref_floats = 0;
    if (need > 0) {
      bool ok = cudaMalloc((void**)&e->ref_cur_hwd, sizeof(float) * need) == cudaSuccess &&
                cudaMalloc((void**)&e->ref_kv_hwd, sizeof(float) * need) == cudaSuccess;
      if (!ok) { nrgbd_set_error("engine: cudaMalloc failed for the refined outputs"); return NRGBD_ERR_NOMEM; }
      e->ref_floats = need;
    }
  }
  return NRGBD_OK;
}

static int forward_head(nrgbd_kvnet* e, const float* frames, const float* poses, const float* bv_predict, nrgbd_stream_t st) {
  const int V = e->V, N = V + 1;
  const long long HW = (long long)e->H * e->W, hw = (long long)e->h * e->w;
  int rc = nrgbd_nchw_to_nhwc(frames, N, 3, HW, e->x0_buf, 4, 0, st);
  if (rc) return rc;
  // Rs / ts (basic.py:266-267): gather 3x3 and 3 from the V 4x4 poses
  gather_rt_kernel<<<1, 32 * ((12 * V + 31) / 32), 0, (cudaStream_t)st>>>(poses, V, e->rt_buf);
  nrgbd_count_launch(1);
  if (bv_predict) { rc = nrgbd_transpose2d(bv_predict, e->D, (int)hw, e->prior_hwd, st); if (rc) return rc; }
  return NRGBD_OK;
}

static int forward_core(nrgbd_kvnet* e, bool steady, bool need_cur_refined, bool need_kv_refined, nrgbd_stream_t stream);

static int forward_tail(nrgbd_kvnet* e, bool steady, float* dmap_cur_refined, float* dmap_refined, float* bv_cur, float* dpv,
                        float* depth_lowres, float* conf_lowres, nrgbd_stream_t st) {
  const int D = e->D;
  const long long HW = (long long)e->H * e->W, hw = (long long)e->h * e->w;
  int rc = NRGBD_OK;
  if (bv_cur && !rc) rc = nrgbd_transpose2d(e->bv_cur_hwd, (int)hw, D, bv_cur, st);
  if (dpv && !rc) rc = nrgbd_transpose2d(e->dpv_hwd, (int)hw, D, dpv, st);
  if (e->refine == 1) {              // guided filter: [H][W] depth maps, already in the caller's layout
    if (dmap_cur_refined) NRGBD_CUDA_CHECK(cudaMemcpyAsync(dmap_cur_refined, e->ref_cur_hwd, sizeof(float) * HW, cudaMemcpyDeviceToDevice, (cudaStream_t)st));
    if (dmap_refined)
      NRGBD_CUDA_CHECK(cudaMemcpyAsync(dmap_refined, steady ? e->ref_kv_hwd : e->ref_cur_hwd, sizeof(float) * HW, cudaMemcpyDeviceToDevice,
                                       (cudaStream_t)st));
  } else {
    const int Dr = e->refined_planes();
    if (dmap_cur_refined && !rc) rc = nrgbd_transpose2d(e->ref_cur_hwd, (int)HW, Dr, dmap_cur_refined, st);
    if (dmap_refined && !rc) rc = nrgbd_transpose2d(steady ? e->ref_kv_hwd : e->ref_cur_hwd, (int)HW, Dr, dmap_refined, st);
  }
  if (rc) return rc;
  if (depth_lowres) NRGBD_CUDA_CHECK(cudaMemcpyAsync(depth_lowres, e->depth, sizeof(float) * hw, cudaMemcpyDeviceToDevice, (cudaStream_t)st));
  if (conf_lowres) NRGBD_CUDA_CHECK(cudaMemcpyAsync(conf_lowres, e->conf, sizeof(float) * hw, cudaMemcpyDeviceToDevice, (cudaStream_t)st));
  return NRGBD_OK;
}

int nrgbd_kvnet_forward(nrgbd_kvnet* e, const float* frames, const float* poses, const float* bv_predict,
                        float* dmap_cur_refined, float* dmap_refined, float* bv_cur, float* dpv, float* depth_lowres,
                        float* conf_lowres, nrgbd_stream_t stream) {
  NRGBD_REQUIRE(e && frames && poses, "null input");
  NRGBD_REQUIRE(e->cam[0].set && e->d_planes, "camera / depth planes not set");
  NRGBD_REQUIRE(!bv_predict || e->cam[1].set, "per-call camera (slot 1) not set");
  NRGBD_REQUIRE(e->refine != 2 || (!dmap_cur_refined && !dmap_refined), "refine option 2 (none) has no refined outputs: pass NULL");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ensure_io_buffers(e);
  if (rc) return rc;
  const bool steady = bv_predict != nullptr;
  const bool need_cur = dmap_cur_refined != nullptr || (!steady && dmap_refined != nullptr);
  const bool need_kv = steady && dmap_refined != nullptr;
  rc = forward_head(e, frames, poses, bv_predict, stream);
  if (rc) return rc;

  const int variant = (steady ? 4 : 0) | (need_cur ? 2 : 0) | (need_kv ? 1 : 0);
  const bool branch_warm = steady ? e->warm_steady : e->warm;
  bool done = false;
  if (e->use_graph && branch_warm && !e->profile) {
    for (auto& g : e->graphs) {
      if (g.variant == variant && g.stream == st) {
        NRGBD_CUDA_CHECK(cudaGraphLaunch(g.exec, st));
        nrgbd_count_launch((int)g.launches);
        done = true;
        break;
      }
    }
    if (!done) {
      // capture the core for this (branch, needed outputs, stream): same kernels in the same order - the buffer
      // pool is deterministic after the eager warm-up of the branch
      const long long before = nrgbd_launch_count();
      cudaGraph_t graph = nullptr;
      if (cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed) == cudaSuccess) {
        int crc = forward_core(e, steady, need_cur, need_kv, stream);
        cudaError_t ce = cudaStreamEndCapture(st, &graph);
        const long long captured = nrgbd_launch_count() - before;
        cudaGraphExec_t exec = nullptr;
        if (crc == NRGBD_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess && exec) {
          nrgbd_kvnet::GraphEnt g; g.variant = variant; g.stream = st; g.exec = exec; g.launches = captured;
          e->graphs.push_back(g);
          NRGBD_CUDA_CHECK(cudaGraphLaunch(exec, st));        // the captured work has not run yet
          done = true;
        }
        if (graph) cudaGraphDestroy(graph);
        if (crc != NRGBD_OK) return crc;
      }
      cudaGetLastError();
    }
  }
  if (!done) {
    rc = forward_core(e, steady, need_cur, need_kv, stream);
    if (rc) return rc;
    if (steady) e->warm_steady = true; else e->warm = true;
  }
  return forward_tail(e, steady, dmap_cur_refined, dmap_refined, bv_cur, dpv, depth_lowres, conf_lowres, stream);
}

// One depth frame on engine-owned memory (models/KVNET.py:93-185, if_refined=True, refineNet_name='DPV').
// Inputs: x0_buf (frames, channels-last, sources then reference), rt_buf (R|t), prior_hwd (steady only).
// Results: bv_cur_hwd, dpv_hwd, depth, conf, ref_cur_hwd / ref_kv_hwd (log-DPVs at image size, pixel-major).
static int forward_core(nrgbd_kvnet* e, bool steady, bool need_cur_refined, bool need_kv_refined, nrgbd_stream_t stream) {
  e->st = (cudaStream_t)stream; e->rc = 0;
  nrgbd_stream_t st = stream;
  eval_coeffs(e);
  const int H = e->H, W = e->W, D = e->D, V = e->V, h = e->h, w = e->w, F = e->F, N = V + 1;
  const long long hw = (long long)h * w, HW = (long long)H * W;

  // ---- D-Net: features for the V+1 frames as one batch (basic.py:244-252) ------------------------
  Act x0; x0.p = e->x0_buf; x0.N = N; x0.D = 1; x0.H = H; x0.W = W; x0.C = 3; x0.Cs = 4;
  Act l1, feat;
  feature_cnn(e, x0, l1, feat);
  // image intensity features: avg_pool2d(rgb, 4) (basic.py:254-263) -> the sweep's narrow layout [N][hw][4]
  Act rgbq = acquire(e, N, 1, h, w, 3);
  ENG_CALL(e, nrgbd_avgpool_nhwc(x0.p, N, H, W, x0.Cs, 3, 4, rgbq.p, rgbq.Cs, 0, st));
  const float* Rs = e->rt_buf; const float* ts = e->rt_buf + 9 * V;
  const size_t featS = (size_t)hw * feat.Cs;
  const Camera& c0 = e->cam[0];
  if (!e->rc) {
    {
    ProfScope ps(e, 1, ((1.0 + V) * (F + 3) + D + 3) * (double)hw * 4.0);
    // fused D-Net head: plane-sweep cost + BV = log_softmax(-costV) (basic.py:299-300) + expected depth / confidence;
    // the cost volume stays in registers (F >= 64, D <= 256), otherwise dpv_hwd serves as its scratch
    const bool in_regs = F >= 64 && F <= 128 && D <= 256;
    ENG_CALL(e, nrgbd_plane_sweep_dpv_packed(feat.p + (size_t)V * featS, rgbq.p + (size_t)V * hw * 4, feat.p, rgbq.p, F, 3, V, D,
                                             h, w, c0.K, Rs, ts, c0.rays, e->d_planes, c0.cx, c0.cy, e->sigma, e->metric,
                                             e->ws_sweep, in_regs ? nullptr : e->dpv_hwd, e->bv_cur_hwd, e->depth, e->conf, st));
    }
  }
  // ---- R-Net on the measurement (KVNET.py:134) ----------------------------------------------------
  const float* feat_ref = feat.p ? feat.p + (size_t)V * featS : nullptr;
  const float* l1_ref = l1.p ? l1.p + (size_t)V * 4 * hw * l1.Cs : nullptr;
  Act frame_ref = x0; frame_ref.N = 1; frame_ref.p = x0.p + (size_t)V * HW * x0.Cs;
  Act out_cur; out_cur.p = e->ref_cur_hwd; out_cur.N = 1; out_cur.D = 1; out_cur.H = H; out_cur.W = W;
  out_cur.C = out_cur.Cs = e->refined_planes();
  Act out_kv = out_cur; out_kv.p = e->ref_kv_hwd;
  if (need_cur_refined) {
    if (e->refine == 1) dgf_refine(e, e->bv_cur_hwd, frame_ref, out_cur.p);
    else r_net(e, e->bv_cur_hwd, feat_ref, feat.Cs, l1_ref, l1.Cs, frame_ref, out_cur);
  }
  if (!steady) {
    // first window: DPV = BV_cur (KVNET.py:138-140)
    if (!e->rc) cudaMemcpyAsync(e->dpv_hwd, e->bv_cur_hwd, sizeof(float) * hw * D, cudaMemcpyDeviceToDevice, e->st);
  } else {
    // ---- K-Net (KVNET.py:147-173) ------------------------------------------------------------------
    const Camera& c1 = e->cam[1];
    const int CK = 3 * V + 4;
    Act vol;
    vol.N = 1; vol.D = D; vol.H = h; vol.W = w; vol.C = CK; vol.Cs = pad32(CK);
    if (vol.Cs == 32 && use_h2(e, vol)) {
      // f16-pair mode: the volume is written directly as the operand pair of dres0.0 (no fp32 volume, no split pass);
      // vol.p is only the key of the pair buffers (a 16-byte block). dres0.0 decides its path by the same use_h2(vol),
      // so it reads the pair: CK = 10 (t_win_r = 1) runs at Cin_pad = 32 like CK = 16 and 28. The row kernel stores
      // 32 channels, the zeros [CK, 32) included.
      PairBuf pb;
      vol = pair_act(e, 1, D, h, w, CK, false, pb);
      ENG_CALL(e, nrgbd_knet_input_volume_pair(rgbq.p, rgbq.p + (size_t)V * hw * 4, e->bv_cur_hwd, e->prior_hwd, V, D, h, w, vol.Cs,
                                               c1.K, Rs, ts, c1.rays, e->d_planes, c1.cx, c1.cy, e->ws_sweep, nullptr, pb.hi, pb.lo, st));
    } else {
      vol = acquire(e, 1, D, h, w, CK);
      ENG_CALL(e, nrgbd_knet_input_volume(rgbq.p, rgbq.p + (size_t)V * hw * 4, e->bv_cur_hwd, e->prior_hwd, V, D, h, w, vol.Cs,
                                          c1.K, Rs, ts, c1.rays, e->d_planes, c1.cx, c1.cy, e->ws_sweep, vol.p, st));
    }
    Act gain = kv_net(e, vol);
    release(e, vol);
    // DPV = log_softmax(gain + BV_predict) (:172-173); gain is [D][hw], prior pixel-major
    ENG_CALL(e, nrgbd_dpv_normalize(gain.p, hw, 1, e->prior_hwd, 1, D, 1.f, (int)hw, D, e->dpv_hwd, 1, D, e->d_planes, e->depth,
                                    e->conf, st));
    release(e, gain);
    if (need_kv_refined) {
      if (e->refine == 1) dgf_refine(e, e->dpv_hwd, frame_ref, out_kv.p);
      else r_net(e, e->dpv_hwd, feat_ref, feat.Cs, l1_ref, l1.Cs, frame_ref, out_kv);
    }
  }
  release(e, l1); release(e, feat); release(e, rgbq);
  if (e->rc == 0) { cudaError_t ce = cudaGetLastError(); if (ce != cudaSuccess) { nrgbd_set_error("nrgbd_kvnet_forward: %s", cudaGetErrorString(ce)); e->rc = NRGBD_ERR_CUDA; } }
  return e->rc;
}

// Propagate the engine's current DPV into the next camera (test_utils/test_KVNet.py:46-59):
// BV_predict' = clamp(resample(dpv, rel_pose_inv, pad=log(1/D)), -1000, 0), written to out [D][h][w].
int nrgbd_kvnet_propagate(nrgbd_kvnet* e, const float* dpv_dhw, const float* rel_pose_inv_dev, float* out_dhw,
                          nrgbd_stream_t stream) {
  NRGBD_REQUIRE(e && rel_pose_inv_dev && out_dhw, "null pointer");
  NRGBD_REQUIRE(e->cam[1].set && e->d_planes && !e->d_host.empty(), "per-call camera / planes not set");
  const int D = e->D, h = e->h, w = e->w;
  float zmax = e->d_host[0], zmin = e->d_host[0];
  for (float d : e->d_host) { zmax = fmaxf(zmax, d); zmin = fminf(zmin, d); }
  const float z_half = (zmax + zmin) * .5f, z_radius = (zmax - zmin) * .5f;
  const Camera& c = e->cam[1];
  const float pad = (float)std::log(1.0 / (double)D);
  if (dpv_dhw)
    return nrgbd_resample_dpv(dpv_dhw, (long long)h * w, 1, rel_pose_inv_dev, c.rays, e->d_planes, D, h, w, c.tan_hh, c.tan_hv,
                              z_half, z_radius, pad, 1, -1000.f, 0.f, out_dhw, (long long)h * w, 1, stream);
  return nrgbd_resample_dpv(e->dpv_hwd, 1, D, rel_pose_inv_dev, c.rays, e->d_planes, D, h, w, c.tan_hh, c.tan_hv, z_half,
                            z_radius, pad, 1, -1000.f, 0.f, out_dhw, (long long)h * w, 1, stream);
}

}  // extern "C"
