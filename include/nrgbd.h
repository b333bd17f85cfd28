/* nrgbd.h - C ABI of the H100-native plane-sweep DPV engine (libnrgbd.so).
 *
 * The reference (NVlabs/neuralrgbd) has no FFI / plugin ABI of its own: its boundary is the
 * Python import surface `warping.homography` (free functions) and `models.KVNET.KVNET`
 * (an nn.Module). Each entry point below names the reference call it replaces (paths relative to
 * the reference's code/ directory); `neuralrgbd_b200/warping/homography.py` and
 * `neuralrgbd_b200/models/KVNET.py` bind them through ctypes with the reference's names and
 * argument conventions (see INTEGRATION.md).
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer to float32 unless the name
 *    says `host`; `stream` is a cudaStream_t (0 = legacy default stream).
 *  - return value: 0 on success, negative NRGBD_ERR_* otherwise; nothing throws across the
 *    boundary. nrgbd_last_error() returns a thread-local message for the last failure.
 *  - the caller owns every buffer; the library keeps no hidden global state besides the launch
 *    counter. All entry points are re-entrant and launch on the stream they are given.
 *  - development probes and A/B knobs are NOT part of this header: see include/nrgbd_dev.h (not bound by the
 *    product's Python layer; no environment variable changes what a product entry point runs).
 */
#ifndef NRGBD_H_
#define NRGBD_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* nrgbd_stream_t;

#define NRGBD_OK 0
#define NRGBD_ERR_BAD_ARG (-1)
#define NRGBD_ERR_CUDA (-2)
#define NRGBD_ERR_UNSUPPORTED (-3)
#define NRGBD_ERR_NOMEM (-4)
#define NRGBD_ERR_IO (-5)

#define NRGBD_METRIC_L2 0 /* img_dis_L2_pard, warping/homography.py:81-83 */
#define NRGBD_METRIC_L1 1 /* img_dis_L1_pard, warping/homography.py:85-87 */

/* ---- runtime -------------------------------------------------------------------------- */
int nrgbd_abi_version(void);
const char* nrgbd_last_error(void);
long long nrgbd_launch_count(void);      /* kernels launched by this library since the last reset */
void nrgbd_reset_launch_count(void);

/* ---- layout helpers --------------------------------------------------------------------- */
/* Channel split used by the sweep: C = Cw + Cn, Cw % 4 == 0 ("wide", [hw][Cw]), Cn = C % 4
 * ("narrow", [hw][4] zero padded). */
void nrgbd_sweep_channel_split(int C, int* Cw, int* Cn);
/* n_img images [C][hw] (NCHW planes) -> wide [n_img][hw][Cw] and narrow [n_img][hw][4]. */
int nrgbd_pack_features(const float* nchw, int C, int hw, int n_img, float* wide, float* narrow,
                        nrgbd_stream_t stream);
/* out[b][a] = in[a][b] (in has A rows of B). Used for [hw][D] <-> [D][hw]. */
int nrgbd_transpose2d(const float* in, int A, int B, float* out, nrgbd_stream_t stream);
int nrgbd_sweep_workspace_floats(int V); /* scratch floats needed by the sweep / warp entries */

/* ---- a1-a3: fused plane-sweep cost volume ------------------------------------------------
 * replaces warping/homography.py:293-331 est_swp_volume_v4 (+ :421-448 _back_warp_homo_parallel,
 * :81-87 img_dis_L{2,1}_pard).  cost_hwd[pix][d] = sum_v dist(warp_{v,d}(src_v)[pix], ref[pix]) / sigma.
 * K 3x3, R [V][3][3], t [V][3], rays [3][hw] (cam_intrinsic['unit_ray_array_2D']), d_planes [D];
 * cx, cy = cam_intrinsic['intrinsic_M'][0,2], [1,2]. ws: nrgbd_sweep_workspace_floats(V) floats.
 * metric other than L2/L1 -> NRGBD_ERR_BAD_ARG with message
 * "undefined metric for feature distance ..." (homography.py:329). */
int nrgbd_plane_sweep_cost_packed(const float* ref_wide, const float* ref_narrow, const float* src_wide,
                                  const float* src_narrow, int Cw, int Cn, int V, int D, int h, int w,
                                  const float* K, const float* R, const float* t, const float* rays,
                                  const float* d_planes, float cx, float cy, float sigma, int metric,
                                  float* ws, float* cost_hwd, nrgbd_stream_t stream);

/* The D-Net head after the feature CNN in ONE kernel (models/basic.py:270-300): the cost above, then
 * BV = log_softmax(-cost) [h*w][D], expected depth sum_d exp(BV) d (mutils/misc.py:532-548) and confidence max_d exp(BV);
 * any of cost_hwd / bv_hwd / depth / conf may be NULL (the cost volume then never reaches memory). */
int nrgbd_plane_sweep_dpv_packed(const float* ref_wide, const float* ref_narrow, const float* src_wide,
                                 const float* src_narrow, int Cw, int Cn, int V, int D, int h, int w,
                                 const float* K, const float* R, const float* t, const float* rays,
                                 const float* d_planes, float cx, float cy, float sigma, int metric,
                                 float* ws, float* cost_hwd, float* bv_hwd, float* depth, float* conf,
                                 nrgbd_stream_t stream);

/* ---- a7: image warp to volume --------------------------------------------------------------
 * replaces warping/homography.py:234-280 warp_img_feats_v3 and :183-232 warp_img_feats_mgpu.
 * imgs_packed [V][hw][4] holds channels [c_off, c_off+c_cnt) of each source view;
 * out [V][C_total][D][hw] (the reference returns V tensors C x D x h x w). */
int nrgbd_warp_to_volume(const float* imgs_packed, int c_cnt, int c_off, int C_total, int V, int D, int h,
                         int w, const float* K, const float* R, const float* t, const float* rays,
                         const float* d_planes, float cx, float cy, float* ws, float* out,
                         nrgbd_stream_t stream);
/* f-5: gradient of nrgbd_warp_to_volume with respect to the source images (autograd of warp_img_feats_v3 / _mgpu:
 * F.grid_sample bilinear / zeros / align_corners=False input gradient; R, t, K, d are constants: no gradient).
 * grad_out [V][C][D][hw] (all C channels, no chunking); g_imgs [V][C][hw] is zeroed by the call, then scatter-added
 * with fp32 atomics at the forward's corners and weights (order not deterministic, like ATen's grid_sampler backward).
 * Same camera arguments and workspace (V*12 floats) as the forward. */
int nrgbd_warp_to_volume_backward(const float* grad_out, int C, int V, int D, int h, int w, const float* K,
                                  const float* R, const float* t, const float* rays, const float* d_planes, float cx,
                                  float cy, float* ws, float* g_imgs, nrgbd_stream_t stream);
/* K-Net input volume, channels-last [D][hw][CK]: [v*3+c warped src RGB | ref RGB | BV_cur - BV_predict]
 * replaces models/KVNET.py:147-166 (avg-pooled RGB is passed in packed [.][hw][4]). */
int nrgbd_knet_input_volume(const float* src_rgb_packed, const float* ref_rgb_packed,
                            const float* bv_cur_hwd, const float* bv_pred_hwd, int V, int D, int h, int w,
                            int CK, const float* K, const float* R, const float* t, const float* rays,
                            const float* d_planes, float cx, float cy, float* ws, float* out,
                            nrgbd_stream_t stream);

/* the same volume, optionally (also / only: out may be NULL) as the split-fp16 operand pair (out_hi, out_lo: half
 * [D][hw][CK], CK = 16 or 32) of the f16-pair convolution that consumes it - see nrgbd_conv_nhwc_h2. out_lo == NULL with
 * out_hi set: only hi = RN_f16(volume) is written (the operand of the single-product convolution). */
int nrgbd_knet_input_volume_pair(const float* src_rgb_packed, const float* ref_rgb_packed,
                                 const float* bv_cur_hwd, const float* bv_pred_hwd, int V, int D, int h, int w,
                                 int CK, const float* K, const float* R, const float* t, const float* rays,
                                 const float* d_planes, float cx, float cy, float* ws, float* out, void* out_hi,
                                 void* out_lo, nrgbd_stream_t stream);

/* ---- a12: DPV re-projection -----------------------------------------------------------------
 * replaces warping/homography.py:654-723 resample_vol_cuda + :873-887 _set_vol_border (+ the
 * clamp of test_utils/test_KVNet.py:54-59 when do_clamp != 0). Element (d,pix) of vol/out lives at
 * d*stride_d + pix*stride_pix. E: 4x4 row-major rel_extM. d_pts: plane depths of the sampled
 * points (d_candi_new if given else d_candi). tan_hh/tan_hv = tan(radians(hfov)/2), tan(radians(vfov)/2);
 * z_half/z_radius as in :695-696. */
int nrgbd_resample_dpv(const float* vol, long long in_stride_d, long long in_stride_pix, const float* E,
                       const float* rays, const float* d_pts, int D, int H, int W, float tan_hh,
                       float tan_hv, float z_half, float z_radius, float pad_value, int do_clamp,
                       float clamp_lo, float clamp_hi, float* out, long long out_stride_d,
                       long long out_stride_pix, nrgbd_stream_t stream);
/* f-5: gradient of nrgbd_resample_dpv with respect to vol (autograd of _set_vol_border + grid_sample(bilinear,
 * border) 3-D, + torch.clamp when do_clamp != 0; E, d_pts and the camera are constants). Same arguments and strides
 * as the forward; grad_out is read at the out strides, g_vol is written at the in strides, which must be dense
 * ((hw, 1) or (1, D)). The six faces get zero gradient; with do_clamp the gradient passes where lo <= x <= hi (vol
 * is re-read for that, and may be NULL when do_clamp == 0). g_vol is zeroed by the call, then scatter-added with
 * fp32 atomics (order not deterministic). */
int nrgbd_resample_dpv_backward(const float* vol, long long in_stride_d, long long in_stride_pix, const float* E,
                                const float* rays, const float* d_pts, int D, int H, int W, float tan_hh,
                                float tan_hv, float z_half, float z_radius, float pad_value, int do_clamp,
                                float clamp_lo, float clamp_hi, const float* grad_out, long long out_stride_d,
                                long long out_stride_pix, float* g_vol, nrgbd_stream_t stream);

/* ---- a4 tail, a9, a11: reductions over the D planes -------------------------------------------
 * out = log_softmax_d(sign * (a + b)) (b may be NULL):
 *   sign=-1, b=NULL : BV = log_softmax(-costV)            models/basic.py:299-300
 *   sign=+1, b=prior: DPV = log_softmax(gain + BV_predict) models/KVNET.py:172-173
 * with d_planes also depth[pix] = sum_d exp(out)*d (mutils/misc.py:532-548) and
 * conf[pix] = max_d exp(out) (test_utils/export_res.py:55-62). out may be NULL.
 * Element (d,pix) of a / b / out lives at d*_sd + pix*_sp of the respective array. */
int nrgbd_dpv_normalize(const float* a, long long in_sd, long long in_sp, const float* b, long long b_sd,
                        long long b_sp, float sign, int n_pix, int D, float* out, long long out_sd,
                        long long out_sp, const float* d_planes, float* depth, float* conf,
                        nrgbd_stream_t stream);
/* depth[pix] = sum_d (bv_log ? exp(bv) : bv)(d,pix) * d_planes[d]  -- mutils/misc.py:532-548
 * depth_val_regression (no normalisation); conf[pix] = max_d of the same probability. */
int nrgbd_depth_regression(const float* bv, int n_pix, int D, long long in_sd, long long in_sp,
                           const float* d_planes, int bv_log, float* depth, float* conf,
                           nrgbd_stream_t stream);
/* f-5: gradient of the depth of nrgbd_depth_regression with respect to bv, same layout and arguments:
 * g_bv(d,pix) = (grad_depth[pix] * d_planes[d]) * exp(bv(d,pix))  (bv_log != 0; the rounding order of autograd
 * through misc.py:541-546), or grad_depth[pix] * d_planes[d] (bv_log == 0; bv may then be NULL). Every element of
 * g_bv is written; no atomics. conf has no gradient. */
int nrgbd_depth_regression_backward(const float* grad_depth, const float* bv, int n_pix, int D, long long in_sd,
                                    long long in_sp, const float* d_planes, int bv_log, float* g_bv,
                                    nrgbd_stream_t stream);
/* Depth variance of one slice (mutils/misc.py:550-572 depth_var), same bv layout as nrgbd_depth_regression; mean and var
 * are [n_pix]:
 *   var[pix] = (sum_d ((p(d,pix) * d_planes[d] - mean[pix])^2) / var_div) / D,  p = bv_log ? exp(bv) : bv,
 * summed sequentially over d, every operation rounded on its own. var_div is 2 * d_sigma^2 rounded to float. */
int nrgbd_depth_var(const float* bv, int n_pix, int D, long long in_sd, long long in_sp, const float* d_planes,
                    int bv_log, const float* mean, float var_div, float* var, nrgbd_stream_t stream);
/* Gradient of nrgbd_depth_var with respect to bv (g_bv, same layout as bv: every plane written) and mean (g_mean
 * [n_pix]), in the rounding order of autograd through misc.py:566-572. Either output may be NULL; no atomics. */
int nrgbd_depth_var_backward(const float* grad_var, const float* bv, int n_pix, int D, long long in_sd, long long in_sp,
                             const float* d_planes, int bv_log, const float* mean, float var_div, float* g_bv,
                             float* g_mean, nrgbd_stream_t stream);
/* value[n*n_pix + pix] = max_d (is_min: min_d) of p(n,d,pix), p = bv_log ? exp(bv) : bv, element (n,d,pix) of bv at
 * n*in_sn + d*in_sd + pix*in_sp (misc.py:599-604 dpv_statistics 'max' / 'min'). index (may be NULL) receives the plane as
 * ATen's max.dim / min.dim on the CPU gives it: ties keep the first plane, the first NaN wins. */
int nrgbd_dpv_extreme(const float* bv, int n_pix, int n_slices, int D, long long in_sn, long long in_sd, long long in_sp,
                      int bv_log, int is_min, float* value, int* index, nrgbd_stream_t stream);
/* Gradient of nrgbd_dpv_extreme's value: g_bv = grad_value * exp(bv) (bv_log; grad_value alone otherwise, bv may then be
 * NULL) at the plane index names, 0 at every other plane. Every element of g_bv is written; same layout as bv. */
int nrgbd_dpv_extreme_backward(const float* grad_value, const float* bv, const int* index, int n_pix, int n_slices, int D,
                               long long in_sn, long long in_sd, long long in_sp, int bv_log, float* g_bv,
                               nrgbd_stream_t stream);
int nrgbd_exp(const float* x, long long n, float* y, nrgbd_stream_t stream);

/* ---- f-1: backward of the plane sweep (autograd of warping/homography.py:293-331 as used by
 * train_utils/train_KVNet.py:149-153; R, t, K, d are constants: only the two feature gradients) ----------------
 * Same packed layout, camera terms and workspace as nrgbd_plane_sweep_cost_packed. grad_cost_hwd [h*w][D].
 * g_ref_* / g_src_* have the shapes of ref_* / src_*; g_src_* are zeroed by the call, then scatter-added with
 * vector atomics (order not deterministic, like ATen's grid_sampler backward). */
int nrgbd_plane_sweep_backward_packed(const float* ref_wide, const float* ref_narrow, const float* src_wide,
                                      const float* src_narrow, int Cw, int Cn, int V, int D, int h, int w,
                                      const float* K, const float* R, const float* t, const float* rays,
                                      const float* d_planes, float cx, float cy, float sigma, int metric, float* ws,
                                      const float* grad_cost_hwd, float* g_ref_wide, float* g_ref_narrow,
                                      float* g_src_wide, float* g_src_narrow, nrgbd_stream_t stream);
/* Inverse of nrgbd_pack_features: n_img images of wide [hw][C - C%4] (+ narrow [hw][4]) -> NCHW [C][hw]. */
int nrgbd_unpack_features(const float* wide, const float* narrow, int C, int hw, int n_img, float* nchw,
                          nrgbd_stream_t stream);

/* ---- f-3: depth-map back-warp of the local bundle adjustment and its gradients -------------------------------------
 * replaces warping/homography.py:479-529 back_warp_th_Rt_msrc and :530-574 back_warp_th_Rt (consumer:
 * ICP/opt_pose_numerical.py:99-160, which differentiates the warped image w.r.t. R and t through F.grid_sample's grid).
 * imgs [N][C][H][W], dmap [H][W] (reference depth), Rs [N][3][3], ts [N][3] (reference -> source), K 3x3
 * (cam_intrinsic['intrinsic_M_cuda']), rays [3][H*W] (cam_intrinsic['unit_ray_array_2D']) -> out [N][C][H][W]. */
int nrgbd_lba_back_warp(const float* imgs, const float* dmap, const float* Rs, const float* ts, const float* K,
                        const float* rays, int N, int C, int H, int W, float* out, nrgbd_stream_t stream);
/* grad_out [N][C][H][W] -> g_R [N][3][3] and g_t [N][3] (both or neither), g_imgs [N][C][H][W] (optional; scatter-added
 * with atomics, like ATen's grid_sampler backward). ws: N * 12 doubles of device scratch. */
int nrgbd_lba_back_warp_backward(const float* grad_out, const float* imgs, const float* dmap, const float* Rs,
                                 const float* ts, const float* K, const float* rays, int N, int C, int H, int W,
                                 float* g_imgs, float* g_R, float* g_t, double* ws, nrgbd_stream_t stream);

/* ---- the LBA pose optimiser (replaces ICP/opt_pose_numerical.py local_BA_direct(_parallel): Adam on the unit-quaternion
 * rotation u and / or the translation t of every source view, L1 photometric loss of the back-warp, 3 pyramid levels) ----
 * Per-view state: NRGBD_LBA_STATE_FLOATS floats, owned by the caller and updated in place. u (unitQ parameter, 3), t (3),
 * R = UnitQ2Rotation(u) (row-major 3x3, the rotation the warp uses), Adam's exp_avg / exp_avg_sq of u and of t, and the
 * gradients of the last iteration. */
#define NRGBD_LBA_STATE_FLOATS 40
#define NRGBD_LBA_U 0
#define NRGBD_LBA_T 3
#define NRGBD_LBA_R 6
#define NRGBD_LBA_M_U 15
#define NRGBD_LBA_V_U 18
#define NRGBD_LBA_M_T 21
#define NRGBD_LBA_V_T 24
#define NRGBD_LBA_G_U 27
#define NRGBD_LBA_G_T 30
#define NRGBD_LBA_OPT_R 1 /* mode bits: which parameters Adam updates */
#define NRGBD_LBA_OPT_T 2
/* F.avg_pool2d(x, k) of N planes [N][H][W] -> out [N][H/k][W/k] (floor), bit-exact with ATen. */
int nrgbd_lba_avgpool(const float* x, int N, int H, int W, int k, float* out, nrgbd_stream_t stream);
/* Bytes of device workspace nrgbd_lba_pose_opt_scale needs for V views of H x W (-1 for bad sizes). */
long long nrgbd_lba_pose_opt_workspace_bytes(int V, int H, int W);
/* n_iter Adam iterations at one pyramid level, enqueued on `stream` with no host synchronisation (one kernel each).
 * ref [3][H][W], conf [H][W], dmap [H][W], srcs [V][3][H][W], K 3x3, rays [3][H*W]; mode = NRGBD_LBA_OPT_R | NRGBD_LBA_OPT_T;
 * loss_scale = 1 / (number of residuals the reference's mean runs over); lr: this level's learning rate; first_step: Adam
 * steps taken before this call. state [V][NRGBD_LBA_STATE_FLOATS] is updated in place; losses [n_iter][V] (double)
 * receives each iteration's sum of |residual| per view, evaluated before the step. ws: workspace_bytes(V, H, W) bytes,
 * 8-byte aligned; one call at a time per workspace. */
int nrgbd_lba_pose_opt_scale(const float* ref, const float* conf, const float* dmap, const float* srcs, const float* K,
                             const float* rays, int V, int H, int W, int mode, double loss_scale, double lr, int first_step,
                             int n_iter, float* state, double* losses, void* ws, nrgbd_stream_t stream);

/* ---- f-4: input stage (replaces mdataloader/scanNet.py:368-369 PIL nearest resize and
 * mdataloader/m_preprocess.py:15-21 ToTensor + Normalize, both host-side per frame) ------------------------------
 * dst[c][y][x] = ((float)src[ys[y]][xs[x]][c] / 255 - mean[c]) / std[c], each op rounded in fp32 (bit-exact with
 * torchvision). src_hwc: device uint8 [Hs][Ws][3]; ys [H], xs [W]: device int32 source indices (PIL's NEAREST table,
 * neuralrgbd_b200.mdataloader.m_preprocess.nearest_index); mean3 / std3: HOST float[3]; dst_chw: device [3][H][W]. */
int nrgbd_preprocess_rgb_u8(const unsigned char* src_hwc, int Hs, int Ws, const int* ys, const int* xs, int H, int W,
                            const float* mean3, const float* std3, float* dst_chw, nrgbd_stream_t stream);

/* ---- f-2: output stage (replaces test_utils/export_res.py:37-75 export_res_img and the map part of
 * :77-100 export_res_refineNet, which move the whole D x H x W volume to the host first) -----------
 * One pass over the reference-layout log-DPV [D][HW] (plane-major, device):
 *   dmap[p] = sum_d exp(bv[d][p]) * d_candi[d]   (depth_regression :37-41; misc.depth_val_regression)
 *   conf[p] = exp(max_d bv[d][p])                (:56-59)
 *   dmap_u16 = (uint16)(dmap * depth_scale), conf_u16 = (uint16)(conf * conf_scale)   (:74-75, numpy
 *   astype(np.uint16): truncation toward zero; out-of-range values, undefined there, are clamped)
 * Any of the four outputs may be NULL. d_candi: device float[D]. */
int nrgbd_export_depth_conf(const float* log_dpv, const float* d_candi, int D, long long HW, float depth_scale,
                            float conf_scale, float* dmap, float* conf, unsigned short* dmap_u16,
                            unsigned short* conf_u16, nrgbd_stream_t stream);
/* Host-only: 16-bit binary PGM byte-identical to mio/imgIO.py:9-10 export2pgm (PIL mode 'I' -> P5,
 * maxval 65535, big-endian samples). pixels: HOST pointer, row-major [height][width].
 * Returns 0, NRGBD_ERR_BAD_ARG, or NRGBD_ERR_IO when the file cannot be written. */
int nrgbd_write_pgm16(const char* path, const unsigned short* pixels, int width, int height);

/* ---- a5, a8, a10: conv stacks (channels-last fp32, channel stride Cs % 4 == 0) ---------------
 * Replace nn.Conv2d/Conv3d/ConvTranspose2d (+bias, +LeakyReLU) and training-mode BatchNorm
 * (models/psm_submodule.py:10-23, models/basic.py:71-94, models/Refine.py:47-77,
 * models/m_submodule.py:18-43). */
/* PyTorch weight [Cout][Cin][taps] (transposed=0) or [Cin][Cout][taps] (transposed=1) ->
 * packed [taps][Cin_pad][Cout_pad], zero padded. */
int nrgbd_pack_conv_weight(const float* w, int transposed, int Cout, int Cin, int taps, int Cin_pad,
                           int Cout_pad, float* out, nrgbd_stream_t stream);
/* x [N][Din][Hin][Win][Cs_in] -> y [N][Din][Hout][Wout][Cs_out] channels [c_off, c_off+Cout);
 * kd x kh x kw taps (kd=1: 2-D; depth stride 1, pad kd/2). stats: [2][Cout] doubles accumulated
 * (sum, sum of squares of the stored outputs) for BatchNorm, or NULL. */
int nrgbd_conv_nhwc(const float* x, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in,
                    const float* w, const float* bias, int Cout, int Cout_pad, int kd, int kh, int kw,
                    int stride, int pad, int dilation, float* y, int Hout, int Wout, int Cs_out, int c_off,
                    int leaky, double* stats, nrgbd_stream_t stream);
/* nn.ConvTranspose2d(kernel 4, stride 2, padding 1); w packed [16][Cin_pad][Cout_pad]. */
int nrgbd_conv_transpose2d_k4s2_nhwc(const float* x, int N, int Hin, int Win, int Cin_pad, int Cs_in,
                                     const float* w, const float* bias, int Cout, int Cout_pad, float* y,
                                     int Cs_out, int c_off, int leaky, nrgbd_stream_t stream);
/* scale = gamma/sqrt(var+eps), shift = beta - mean*scale from accumulated stats (biased variance);
 * run_mean/run_var (may be NULL) get the training-mode momentum update. */
int nrgbd_bn_finalize(const double* stats, int C, double count, const float* gamma, const float* beta,
                      float eps, float* scale, float* shift, float* run_mean, float* run_var,
                      float momentum, nrgbd_stream_t stream);
/* finalize + apply in one pass (C <= 512): scale/shift are derived per block from `stats`. */
int nrgbd_bn_apply_stats(const float* x, const double* stats, double count, const float* gamma, const float* beta,
                         float eps, float* run_mean, float* run_var, float momentum, const float* res, int relu,
                         long long n_pos, int Cs, int C, float* y, nrgbd_stream_t stream);
/* same pass, also (or only: y may be NULL) emitting the result as the split-fp16 operand pair (y_hi, y_lo: half tensors with
 * x's layout; both may be NULL) of the f16-pair convolution that consumes it - see nrgbd_conv_nhwc_h2. The residual is either
 * the fp32 tensor `res` or the operand pair (res_hi, res_lo) of a tensor that was only ever written as a pair (its value
 * hi + lo * 2^-11 carries 22 significand bits); at most one of the two forms. y_hi set and y_lo == NULL: only
 * hi = RN_f16(result) is written (the operand of the single-product convolution). rezero_counter
 * (optional, a zero-initialised device word): the last block to have read `stats` sets them back to zero, so the next
 * convolution accumulates into a clean buffer without a memset in between. */
int nrgbd_bn_apply_stats_pair(const float* x, double* stats, double count, const float* gamma, const float* beta,
                              float eps, float* run_mean, float* run_var, float momentum, const float* res, const void* res_hi,
                              const void* res_lo, int relu, long long n_pos, int Cs, int C, float* y, void* y_hi, void* y_lo,
                              unsigned int* rezero_counter, nrgbd_stream_t stream);
/* Second half of a SINGLE-output-channel k3 convolution (models/basic.py:136-137, K-Net's Conv3d(64 -> 1)): with
 * Q[n][d][h][w][t] = sum_c x[..][c] w[0][c][t] - one pointwise convolution with kd*k*k output channels, e.g. nrgbd_conv_nhwc_h2 on
 * the weight packed with transposed = 1, Cout = kd*k*k, taps = 1 - this gathers
 * out[n][d][h][w] = bias + sum_t Q[n][d + tz - kd/2][h + ty - 1][w + tx - 1][t]  (zero outside the volume; t = (tz*3 + ty)*3 + tx).
 * Q has Cs >= kd*k*k floats per position; k = 3, kd in {1, 3}. */
int nrgbd_tap_gather_sum(const float* Q, int N, int D, int H, int W, int Cs, int kd, int k, float bias, float* out,
                         nrgbd_stream_t stream);
/* Eval-mode BatchNorm coefficients from the running statistics (only read), ATen's order of operations:
 * scale = (1 / sqrt(running_var + eps)) * gamma, shift = beta - running_mean * scale, C channels. */
int nrgbd_bn_eval_coeffs(const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                         float eps, int C, float* scale, float* shift, nrgbd_stream_t stream);
/* y = [relu](x*scale + shift) [+ res] over n_pos positions of Cs channels (C logical). */
int nrgbd_bn_apply(const float* x, const float* scale, const float* shift, const float* res, int relu,
                   long long n_pos, int Cs, int C, float* y, nrgbd_stream_t stream);
/* Tensor-core (wgmma / TMA) variants: 3xTF32 error-compensated products, fp32 accumulate.
 * Activations and K-major packed weights are passed as their TF32 hi / lo splits
 * (nrgbd_split_tf32, nrgbd_pack_conv_weight_tc -> [taps][Cout_pad][Cin_pad]). Semantics otherwise
 * identical to nrgbd_conv_nhwc / nrgbd_conv_transpose2d_k4s2_nhwc. */
int nrgbd_conv_tc_supported(int Cin_pad, int Cout_pad);   /* Cin_pad % 32 == 0, Cout_pad % 16 == 0, <= 256 */
int nrgbd_split_tf32(const float* x, long long n, float* hi, float* lo, nrgbd_stream_t stream);
int nrgbd_pack_conv_weight_tc(const float* w, int transposed, int Cout, int Cin, int taps, int Cin_pad,
                              int Cout_pad, float* hi, float* lo, nrgbd_stream_t stream);
int nrgbd_conv_nhwc_tc(const float* x_hi, const float* x_lo, int N, int Din, int Hin, int Win, int Cin_pad,
                       int Cs_in, const float* w_hi, const float* w_lo, const float* bias, int Cout,
                       int Cout_pad, int kd, int kh, int kw, int stride, int pad, int dilation, float* y,
                       int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats,
                       nrgbd_stream_t stream);
int nrgbd_conv_transpose2d_k4s2_nhwc_tc(const float* x_hi, const float* x_lo, int N, int Hin, int Win,
                                        int Cin_pad, int Cs_in, const float* w_hi, const float* w_lo,
                                        const float* bias, int Cout, int Cout_pad, float* y, int Cs_out,
                                        int c_off, int leaky, nrgbd_stream_t stream);
/* v2 entries: raw fp32 activations (split into TF32 pairs in stream-ordered scratch right before the GEMM),
 * pre-split K-major weights. Cout_pad <= 128. Same semantics as the v1 entries. */
/* Training-mode BatchNorm (+ReLU) of a conv's INPUT, folded into the operand split of the consuming tensor-core convolution: x is the RAW output
 * of the producing conv (psm_submodule.convbn :10-16 = Conv2d + BatchNorm2d, BasicBlock :31-49 conv1 -> bn -> relu -> conv2)
 * and `stats` its per-channel [sum(C) | sum of squares(C)] as written by the conv entry points. The consumer computes
 * scale = gamma / sqrt(var + eps), shift = beta - mean * scale once and applies fmaf(x, scale, shift) (+ReLU) while it
 * splits its operands - the same arithmetic as nrgbd_bn_apply_stats, without that pass over the tensor. Padding stays
 * zero. running_mean / running_var (optional) get the momentum update once. `stats` must differ from the consumer's own. */
typedef struct nrgbd_bn_input {
  const double* stats; double count;            /* [2*C] sums of the producing conv; number of positions N*D*H*W */
  const float* gamma; const float* beta;        /* BatchNorm weight / bias [C] */
  float* running_mean; float* running_var;      /* optional [C] */
  float eps, momentum;
  int relu, C;
} nrgbd_bn_input;
int nrgbd_conv_nhwc_tc2_bn_in(const float* x, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const float* w_hi,
                              const float* w_lo, const float* bias, int Cout, int Cout_pad, int kd, int kh, int kw,
                              int stride, int pad, int dilation, float* y, int Hout, int Wout, int Cs_out, int c_off,
                              int leaky, double* stats, const nrgbd_bn_input* in_bn, nrgbd_stream_t stream);
int nrgbd_conv_tc2_supported(int Cin_pad, int Cout_pad);
int nrgbd_conv_nhwc_tc2(const float* x, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in,
                        const float* w_hi, const float* w_lo, const float* bias, int Cout, int Cout_pad,
                        int kd, int kh, int kw, int stride, int pad, int dilation, float* y, int Hout,
                        int Wout, int Cs_out, int c_off, int leaky, double* stats, nrgbd_stream_t stream);
int nrgbd_conv_transpose2d_k4s2_nhwc_tc2(const float* x, int N, int Hin, int Win, int Cin_pad, int Cs_in,
                                         const float* w_hi, const float* w_lo, const float* bias, int Cout,
                                         int Cout_pad, float* y, int Cs_out, int c_off, int leaky,
                                         nrgbd_stream_t stream);
/* Second-generation tensor-core path (csrc/conv_f16.cu): wgmma on SPLIT-FP16 operand pairs, fp32 accumulate.
 * Every fp32 value a is carried as two halves, a = hi + lo * 2^-11 (hi = RN_f16(a), lo = RN_f16((a - hi) * 2^11)), and a
 * product is accumulated as hi*hi + 2^-11 (hi*lo + lo*hi): the 22-bit product of the 3xTF32 path at twice the MMA rate
 * and half the operand bytes. Activations are consumed in pair form (two half tensors with the fp32 tensor's
 * channels-last layout and channel stride) from nrgbd_split_f16_pair / the fused BatchNorm pass; weights are packed once
 * by nrgbd_pack_conv_weight_h2 -> [taps][2 (hi | lo)][Cout_pad][Cin_pad] halves. Stride-1 filters stage ONE halo tile per
 * 32-channel chunk for all in-plane taps (the tap-per-box kernels re-read the tile kh*kw times from L2).
 * Same convolution semantics, outputs (fp32) and BatchNorm statistics as nrgbd_conv_nhwc. */
/* Single product (conv_math = 'f16'): a pair whose lo is NULL is a plain fp16 tensor. Every entry below taking x_lo runs
 * the single-product kernel when x_lo == NULL: out = sum RN_f16(x) * RN_f16(w) in fp32 (RN_f16: round to nearest even,
 * saturating at +-65504), one wgmma per product, the packed weights' lo half never loaded; bias, LeakyReLU, statistics
 * and the affine epilogue unchanged. A pair output with y_lo == NULL stores only hi = RN_f16(result) (pad channels as
 * zeros). The residual of the affine epilogue keeps its pair form (res_hi and res_lo both set, or both NULL). */
int nrgbd_conv_h2_plan(int Cin, int Cout, int* Cin_pad, int* Cout_pad, int* BN);   /* channel padding: Cin to 32; Cout into equal chunks of BN <= 128 */
/* lo == NULL: only hi = RN_f16(x) is written, a plain fp32 -> fp16 conversion (saturating) */
int nrgbd_split_f16_pair(const float* x, long long n, void* hi, void* lo, nrgbd_stream_t stream);
int nrgbd_pack_conv_weight_h2(const float* w, int transposed, int Cout, int Cin, int taps, int Cin_pad, int Cout_pad, void* out,
                              nrgbd_stream_t stream);
int nrgbd_conv_nhwc_h2(const void* x_hi, const void* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in, const void* w,
                       const float* bias, int Cout, int Cout_pad, int BN, int kd, int kh, int kw, int stride, int pad, int dilation,
                       float* y, int Hout, int Wout, int Cs_out, int c_off, int leaky, double* stats, nrgbd_stream_t stream);
/* nrgbd_conv_nhwc_h2 with the result (after bias / LeakyReLU) written ONLY as the split-fp16 operand pair of the convolution
 * that consumes it: y_hi / y_lo are half tensors [N][D][Hout][Wout][Cs_out], Cs_out % 32 == 0, every channel stored (pad
 * channels as zeros). For conv -> conv chains without a BatchNorm in between (R-Net, models/Refine.py:79-107): saves the
 * separate split pass. No statistics, no channel offset. */
int nrgbd_conv_nhwc_h2_pair(const void* x_hi, const void* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in,
                            const void* w, const float* bias, int Cout, int Cout_pad, int BN, int kd, int kh, int kw, int stride,
                            int pad, int dilation, void* y_hi, void* y_lo, int Hout, int Wout, int Cs_out, int leaky,
                            nrgbd_stream_t stream);
/* Eval-mode Conv + BatchNorm (running statistics) [+ residual] [+ ReLU] in ONE pass: nrgbd_conv_nhwc_h2 without bias whose
 * epilogue computes, per output element, v = acc * scale[c] + shift[c]; v += residual (optional); v = max(v, 0) (relu != 0).
 * scale / shift [Cout]: nrgbd_bn_eval_coeffs. The residual has the output's layout ([N][D][Hout][Wout][Cs_out], channels from
 * c_off) and is either the fp32 tensor `res` or the operand pair (res_hi, res_lo: value hi + lo * 2^-11); at most one form.
 * The output is either fp32 (y, channels [c_off, c_off + Cout)) or the split-fp16 operand pair of the next convolution
 * (y_hi / y_lo as in nrgbd_conv_nhwc_h2_pair: Cs_out % 32 == 0, c_off == 0, pad channels stored as zeros). No statistics and
 * no atomics: the output is identical from run to run. (K-Net's convbn_3d layers, models/basic.py:71-94, and the feature
 * CNN's downsample shortcuts, models/psm_submodule.py:128-131, with the module in .eval().) */
int nrgbd_conv_nhwc_h2_affine(const void* x_hi, const void* x_lo, int N, int Din, int Hin, int Win, int Cin_pad, int Cs_in,
                              const void* w, int Cout, int Cout_pad, int BN, int kd, int kh, int kw, int stride, int pad,
                              int dilation, const float* scale, const float* shift, const float* res, const void* res_hi,
                              const void* res_lo, int relu, float* y, void* y_hi, void* y_lo, int Hout, int Wout, int Cs_out,
                              int c_off, nrgbd_stream_t stream);
int nrgbd_conv_transpose2d_k4s2_nhwc_h2(const void* x_hi, const void* x_lo, int N, int Hin, int Win, int Cin_pad, int Cs_in,
                                        const void* w, const float* bias, int Cout, int Cout_pad, int BN, float* y, int Cs_out,
                                        int c_off, int leaky, nrgbd_stream_t stream);
/* layout / pooling helpers (P = positions per image) */
int nrgbd_nchw_to_nhwc(const float* x, int N, int C, long long P, float* y, int Cs, int c_off,
                       nrgbd_stream_t stream);
int nrgbd_nhwc_to_nchw(const float* x, int N, int C, long long P, int Cs, int c_off, float* y,
                       nrgbd_stream_t stream);
int nrgbd_avgpool_nhwc(const float* x, int N, int H, int W, int Cs_in, int C, int k, float* y, int Cs_out,
                       int c_off, nrgbd_stream_t stream);
int nrgbd_upsample_bilinear_ac_nhwc(const float* x, int N, int Hi, int Wi, int Cs_in, int C, float* y,
                                    int Ho, int Wo, int Cs_out, int c_off, nrgbd_stream_t stream);
/* y[p][c_off_out + c] = op(x[p][c_off_in + c]), op 0 = copy, 1 = exp */
int nrgbd_copy_channels(const float* x, long long P, int Cs_in, int c_off_in, int C, int op, float* y,
                        int Cs_out, int c_off_out, nrgbd_stream_t stream);

/* ---- guided-filter depth refinement: models/Refine.py:620-641 RefineNet_DGF.forward with
 * models/GF/guided_filter.py GuidedFilter(r, eps) (KVNET(refineNet_name='DGF') uses r = 1, eps = 1e-8).
 * dmap [h][w] low-resolution depth; img: channel c (0..2) of pixel p at img[c * img_sc + p * img_sp], [H][W];
 * w0 [64][3], b0 [64], w1 [64], b1 [1] = r_net.feature_ext.{0,2}.{weight,bias}; out [H][W].
 * H / h == W / w > 1. ws: nrgbd_guided_filter_workspace_floats(H, W) floats. Box sums use the reference's
 * cumulative-sum form (double-accumulated prefixes rounded to fp32); no atomics, identical from run to run. */
long long nrgbd_guided_filter_workspace_floats(int H, int W);
int nrgbd_guided_filter_refine(const float* dmap, int h, int w, const float* img, long long img_sc, long long img_sp,
                               int H, int W, const float* w0, const float* b0, const float* w1, const float* b1,
                               int r, float eps, float* ws, float* out, nrgbd_stream_t stream);

/* ---- a4, a6: whole-frame engine -------------------------------------------------------------
 * replaces models/KVNET.py:35-185 (KVNET.__init__/forward with if_refined=True, refineNet_name='DPV')
 * + models/basic.py:223-323 (D_NET_BASIC.forward) + the DPV propagation of
 * test_utils/test_KVNet.py:46-59. The layer plan, buffer pool, packed weights and camera tables live
 * in the opaque engine; one call runs one depth frame on `stream`. */
typedef struct nrgbd_kvnet nrgbd_kvnet;
int nrgbd_kvnet_create(int H, int W, int D, int V, int feature_dim, int kv_feature_dim, float sigma,
                       int metric, nrgbd_kvnet** out);
int nrgbd_kvnet_destroy(nrgbd_kvnet* e);
/* name = reference state_dict key (a leading "module." and the d_net.feature_extraction alias are
 * folded); is_device: borrow a device pointer, else copy a host array. */
int nrgbd_kvnet_set_param(nrgbd_kvnet* e, const char* name, const float* data, long long n, int is_device);
/* slot 0: intrinsics captured at construction (D-Net); slot 1: per-call intrinsics (K-Net warp,
 * propagation). Host arrays: K 3x3, rays 3 x (H/4*W/4); fovs in degrees (cam_intrinsic dict). */
int nrgbd_kvnet_set_camera(nrgbd_kvnet* e, int slot, const float* K_host, const float* rays_host, float cx,
                           float cy, double hfov_deg, double vfov_deg);
int nrgbd_kvnet_set_planes(nrgbd_kvnet* e, const float* d_host, int D);   /* float32(d_candi) */
int nrgbd_kvnet_set_option(nrgbd_kvnet* e, const char* key, int value);   /* "bn_update_running", "profile", "conv_math" (0 fp32 FFMA, 1 wgmma 3xTF32, 2 wgmma split-fp16 pairs, 3 wgmma single fp16 products), "use_graph" (CUDA-graph replay, default 1), "bn_eval" (1: the module is in .eval(): BatchNorm layers with running statistics normalise with them and update nothing, the others keep batch statistics; default 0), "refine" (refined outputs: 0 the DPV R-Net, default; 1 the guided filter of refineNet_name='DGF', [H][W] depth maps; 2 none, if_refined=False), "refine_upsample_d" (1: the DPV R-Net of if_upsample_d=True, refined log-DPVs of 4D planes; default 0) */
/* with option "profile"=1 the engine brackets its conv (category 0, work = flops) and plane-sweep
 * (category 1, work = algorithmic bytes) launches with CUDA events; this returns and clears the sums. */
int nrgbd_kvnet_profile_read(nrgbd_kvnet* e, int category, double* ms, double* work, long long* launches);

/* Development aid: per-shape table of the profiled launches of one category, text lines
 * "tag;launches;total_ms;work" written NUL-terminated into buf (truncated to cap). Records are kept. */
int nrgbd_kvnet_profile_table(nrgbd_kvnet* e, int category, char* buf, long long cap);
long long nrgbd_kvnet_workspace_bytes(nrgbd_kvnet* e);
/* frames [V+1][3][H][W] (sources then reference), poses [V][4][4], bv_predict [D][h][w] or NULL
 * (first window). Outputs (any may be NULL): dmap_cur_refined, dmap_refined [D][H][W] log-DPV
 * (option "refine" 1: [H][W] depth; 2: both must be NULL; "refine_upsample_d" 1: [4D][H][W]);
 * bv_cur, dpv [D][h][w] log-DPV; depth_lowres, conf_lowres [h][w]. All device pointers. */
int nrgbd_kvnet_forward(nrgbd_kvnet* e, const float* frames, const float* poses, const float* bv_predict,
                        float* dmap_cur_refined, float* dmap_refined, float* bv_cur, float* dpv,
                        float* depth_lowres, float* conf_lowres, nrgbd_stream_t stream);
/* out [D][h][w] = clamp(resample(dpv, rel_pose_inv, pad = log(1/D)), -1000, 0); dpv_dhw NULL = the
 * engine's own DPV of the last forward. */
int nrgbd_kvnet_propagate(nrgbd_kvnet* e, const float* dpv_dhw, const float* rel_pose_inv_dev, float* out_dhw,
                          nrgbd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* NRGBD_H_ */
