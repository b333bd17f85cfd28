"""Drop-in mirror of the reference's `warping.homography` hot-path functions.

Same names, positional order, argument meaning (numpy float64 `d_candi`, dict intrinsics,
list-or-tensor R/t), return shapes/dtypes and error behaviour as
/root/reference/code/warping/homography.py; every function dispatches to the hand-written
sm_90a kernels in libnrgbd.so through the C ABI of include/nrgbd.h. torch is used for
device memory and the current stream only. There is no CPU path: tensors must live on a
CUDA device and the library must be built.
"""
import ctypes
import math

import numpy as np
import torch

from .. import _lib
from .._devcache import planes_tensor
from .._lib import ptr, check

_F = ctypes.c_float


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(x):
    if not x.is_cuda:
        raise _lib.NrgbdError('neuralrgbd_b200 has no CPU path: expected a CUDA tensor')
    return x.device


_cam_cache = {}


def _cam_tensors(cam_intrinsic, device):
    """K (3x3) and rays (3 x hw) of an intrinsics dict on `device`, cached per dict object."""
    key = (id(cam_intrinsic), device.index)
    hit = _cam_cache.get(key)
    if hit is not None and hit[0] is cam_intrinsic:
        return hit[1], hit[2]
    K = torch.as_tensor(cam_intrinsic['intrinsic_M_cuda'], dtype=torch.float32).to(device).contiguous()
    rays = torch.as_tensor(cam_intrinsic['unit_ray_array_2D'], dtype=torch.float32).to(device).contiguous()
    if len(_cam_cache) > 64:
        _cam_cache.clear()
    _cam_cache[key] = (cam_intrinsic, K, rays)
    return K, rays


def _planes(d_candi, device):
    # homography.py:311: torch.from_numpy(d_candi.astype(np.float32)).cuda()
    return planes_tensor(d_candi, device)


def _stack_Rt(R, t, device):
    if isinstance(R, (list, tuple)):
        R = torch.stack([torch.as_tensor(r) for r in R])
        t = torch.stack([torch.as_tensor(x).reshape(3) for x in t])
    R = R.to(device=device, dtype=torch.float32).reshape(-1, 3, 3).contiguous()
    t = t.to(device=device, dtype=torch.float32).reshape(-1, 3).contiguous()
    return R, t


def get_rel_extrinsicM(ext_ref, ext_src):
    ''' Get the extrinisc matrix from ref_view to src_view (homography.py:904-906) '''
    return ext_src.dot(np.linalg.inv(ext_ref))


def img_dis_L2_pard(img0, img1):
    """homography.py:81-83. Standalone helper kept for API completeness; inside
    est_swp_volume_v4 this reduction is fused into the sweep kernel."""
    return torch.sum((img0 - img1) ** 2, 1)


def img_dis_L1_pard(img0, img1):
    """homography.py:85-87 (see img_dis_L2_pard)."""
    return torch.sum(torch.abs(img0 - img1), 1)


def pack_features(x_nchw):
    """[N,C,h,w] -> (wide [N,hw,Cw] or None, narrow [N,hw,4] or None), the sweep's layouts."""
    L = _lib.lib()
    x = x_nchw.contiguous()
    N, C, h, w = x.shape
    Cw = C - C % 4
    Cn = C % 4
    wide = torch.empty((N, h * w, Cw), device=x.device, dtype=torch.float32) if Cw else None
    narrow = torch.empty((N, h * w, 4), device=x.device, dtype=torch.float32) if Cn else None
    check(L.nrgbd_pack_features(ptr(x), C, h * w, N, ptr(wide), ptr(narrow), _stream()))
    return wide, narrow


def unpack_features(wide, narrow, C, h, w):
    """Inverse of pack_features: (wide [N,hw,Cw], narrow [N,hw,4]) -> [N,C,h,w]."""
    L = _lib.lib()
    t0 = wide if wide is not None else narrow
    N = t0.shape[0]
    out = torch.empty((N, C, h, w), device=t0.device, dtype=torch.float32)
    check(L.nrgbd_unpack_features(ptr(wide), ptr(narrow), C, h * w, N, ptr(out), _stream()))
    return out


def _sweep_forward(ref_w, ref_n, src_w, src_n, C, V, D, H, W, K, Rs, ts, rays, dpl, cx, cy, sigma, metric):
    L = _lib.lib()
    dev = (ref_w if ref_w is not None else ref_n).device
    ws = torch.empty(L.nrgbd_sweep_workspace_floats(V), device=dev, dtype=torch.float32)
    cost_hwd = torch.empty((H * W, D), device=dev, dtype=torch.float32)
    check(L.nrgbd_plane_sweep_cost_packed(ptr(ref_w), ptr(ref_n), ptr(src_w), ptr(src_n), C - C % 4, C % 4,
                                          V, D, H, W, ptr(K), ptr(Rs), ptr(ts), ptr(rays), ptr(dpl),
                                          _F(cx), _F(cy), _F(sigma), metric, ptr(ws), ptr(cost_hwd), _stream()))
    costV = torch.empty((1, D, H, W), device=dev, dtype=torch.float32)
    check(L.nrgbd_transpose2d(ptr(cost_hwd), H * W, D, ptr(costV), _stream()))
    return costV


class _PlaneSweepCost(torch.autograd.Function):
    """est_swp_volume_v4 with the feature gradients the reference gets from autograd
    (train_utils/train_KVNet.py:149-153); poses, intrinsics and plane depths carry no gradient there either."""

    @staticmethod
    def forward(ctx, feat_img_ref, feat_img_src, K, Rs, ts, rays, dpl, cx, cy, sigma, metric):
        C, H, W = feat_img_ref.shape[1:]
        V, D = feat_img_src.shape[1], dpl.numel()
        ref_w, ref_n = pack_features(feat_img_ref.detach().float())
        src_w, src_n = pack_features(feat_img_src.detach()[0].float())
        ctx.save_for_backward(*[x if x is not None else torch.empty(0, device=K.device) for x in (ref_w, ref_n, src_w, src_n)],
                              K, Rs, ts, rays, dpl)
        ctx.meta = (C, V, D, H, W, cx, cy, sigma, metric)
        return _sweep_forward(ref_w, ref_n, src_w, src_n, C, V, D, H, W, K, Rs, ts, rays, dpl, cx, cy, sigma, metric)

    @staticmethod
    def backward(ctx, grad_cost):
        L = _lib.lib()
        ref_w, ref_n, src_w, src_n, K, Rs, ts, rays, dpl = ctx.saved_tensors
        C, V, D, H, W, cx, cy, sigma, metric = ctx.meta
        opt = lambda x: x if x.numel() else None          # noqa: E731
        ref_w, ref_n, src_w, src_n = opt(ref_w), opt(ref_n), opt(src_w), opt(src_n)
        dev = K.device
        with torch.cuda.device(dev):
            g_hwd = torch.empty((H * W, D), device=dev, dtype=torch.float32)
            check(L.nrgbd_transpose2d(ptr(grad_cost.detach().float().contiguous()), D, H * W, ptr(g_hwd), _stream()))
            like = lambda x: torch.empty_like(x) if x is not None else None      # noqa: E731
            g_rw, g_rn, g_sw, g_sn = like(ref_w), like(ref_n), like(src_w), like(src_n)
            ws = torch.empty(L.nrgbd_sweep_workspace_floats(V), device=dev, dtype=torch.float32)
            check(L.nrgbd_plane_sweep_backward_packed(ptr(ref_w), ptr(ref_n), ptr(src_w), ptr(src_n), C - C % 4, C % 4, V, D, H, W,
                                                      ptr(K), ptr(Rs), ptr(ts), ptr(rays), ptr(dpl), _F(cx), _F(cy), _F(sigma),
                                                      metric, ptr(ws), ptr(g_hwd), ptr(g_rw), ptr(g_rn), ptr(g_sw), ptr(g_sn),
                                                      _stream()))
            g_ref = unpack_features(g_rw, g_rn, C, H, W)
            g_src = unpack_features(g_sw, g_sn, C, H, W).unsqueeze(0)
        return g_ref, g_src, None, None, None, None, None, None, None, None, None


def est_swp_volume_v4(feat_img_ref, feat_img_src, d_candi, R, t, cam_intrinsic, costV_sigma,
                      feat_dist='L2', debug_ipdb=False):
    r'''
    feat_img_ref - NCHW tensor
    feat_img_src - NVCHW tensor.  V is for different views
    R, t - R[idx_view, :, :] - 3x3 rotation matrix
           t[idx_view, :] - 3x1 transition vector
    Returns costV [1, D, H, W] (homography.py:293-331). Differentiable w.r.t. the two feature tensors
    (the reference trains through it, train_utils/train_KVNet.py:149-153).
    '''
    if feat_dist not in ('L2', 'L1'):
        raise Exception('undefined metric for feature distance ...')
    dev = _dev(feat_img_ref)
    with torch.cuda.device(dev):
        K, rays = _cam_tensors(cam_intrinsic, dev)
        dpl = _planes(d_candi, dev)
        Rs, ts = _stack_Rt(R, t, dev)
        cx = float(cam_intrinsic['intrinsic_M'][0, 2]); cy = float(cam_intrinsic['intrinsic_M'][1, 2])
        metric = 0 if feat_dist == 'L2' else 1
        if torch.is_grad_enabled() and (feat_img_ref.requires_grad or feat_img_src.requires_grad):
            return _PlaneSweepCost.apply(feat_img_ref, feat_img_src, K, Rs, ts, rays, dpl, cx, cy, float(costV_sigma), metric)
        C, H, W = feat_img_ref.shape[1:]
        ref_w, ref_n = pack_features(feat_img_ref.float())
        src_w, src_n = pack_features(feat_img_src[0].float())
        return _sweep_forward(ref_w, ref_n, src_w, src_n, C, feat_img_src.shape[1], len(d_candi), H, W, K, Rs, ts, rays, dpl,
                              cx, cy, float(costV_sigma), metric)


def _warp_forward(x, D, K, Rs, ts, rays, dpl, cx, cy):
    """x [V,C,h,w] float32 contiguous -> [V,C,D,h,w], in 4-channel chunks."""
    L = _lib.lib()
    V, C, H, W = x.shape
    ws = torch.empty(L.nrgbd_sweep_workspace_floats(V), device=x.device, dtype=torch.float32)
    out = torch.empty((V, C, D, H, W), device=x.device, dtype=torch.float32)
    for c0 in range(0, C, 4):
        cc = min(4, C - c0)
        chunk = x[:, c0:c0 + cc].contiguous()
        wide, narrow = pack_features(chunk)          # cc == 4 packs as wide [V,hw,4]: same memory layout
        packed = narrow if narrow is not None else wide
        check(L.nrgbd_warp_to_volume(ptr(packed), cc, c0, C, V, D, H, W, ptr(K), ptr(Rs), ptr(ts), ptr(rays),
                                     ptr(dpl), _F(cx), _F(cy), ptr(ws), ptr(out), _stream()))
    return out


class _WarpToVolume(torch.autograd.Function):
    """warp_img_feats_v3 / _mgpu with the image-feature gradients autograd gives the reference through
    F.grid_sample (homography.py:183-280). Poses, intrinsics and plane depths get no gradient, as in the sweep.
    Inputs after the camera terms are the views as the caller passed them (V tensors 1xCxhxw, or one NxCxhxw
    tensor); each gets its own gradient."""

    @staticmethod
    def forward(ctx, K, Rs, ts, rays, dpl, cx, cy, *imgs):
        x = torch.cat([i.detach().float() for i in imgs], dim=0).contiguous()
        ctx.save_for_backward(K, Rs, ts, rays, dpl)
        ctx.meta = (cx, cy, x.shape, [(i.shape[0], i.dtype) for i in imgs])
        return _warp_forward(x, dpl.numel(), K, Rs, ts, rays, dpl, cx, cy)

    @staticmethod
    def backward(ctx, grad_out):
        L = _lib.lib()
        K, Rs, ts, rays, dpl = ctx.saved_tensors
        cx, cy, (V, C, H, W), views = ctx.meta
        dev = K.device
        with torch.cuda.device(dev):
            go = grad_out.detach().float().contiguous()
            ws = torch.empty(L.nrgbd_sweep_workspace_floats(V), device=dev, dtype=torch.float32)
            g = torch.empty((V, C, H, W), device=dev, dtype=torch.float32)
            check(L.nrgbd_warp_to_volume_backward(ptr(go), C, V, dpl.numel(), H, W, ptr(K), ptr(Rs), ptr(ts), ptr(rays),
                                                  ptr(dpl), _F(cx), _F(cy), ptr(ws), ptr(g), _stream()))
        grads, v0 = [], 0
        for n, dt in views:
            grads.append(g[v0:v0 + n].to(dt))
            v0 += n
        return (None,) * 7 + tuple(grads)


def _warp_views(feat_img_src, d_candi, R, t, K, rays, cx, cy):
    is_list = isinstance(R, (list, tuple)) and isinstance(t, (list, tuple))
    imgs = list(feat_img_src) if is_list else [feat_img_src]
    dev = _dev(imgs[0])
    with torch.cuda.device(dev):
        D = len(d_candi)
        dpl = _planes(d_candi, dev)
        Rs, ts = _stack_Rt(list(R) if is_list else [R], list(t) if is_list else [t], dev)
        if torch.is_grad_enabled() and any(i.requires_grad for i in imgs):
            out = _WarpToVolume.apply(K, Rs, ts, rays, dpl, cx, cy, *imgs)
        else:
            x = torch.cat([i.float() for i in imgs], dim=0).contiguous()       # [V,C,h,w]
            out = _warp_forward(x, D, K, Rs, ts, rays, dpl, cx, cy)
    outs = [out[v] for v in range(out.shape[0])]
    return outs if is_list else outs[0]


def warp_img_feats_v3(feat_img_src, d_candi, R, t, cam_intrinsic):
    r'''
    Warp the feat_imgs_src to the reference view for all candidate depths (homography.py:234-280)
    feat_img_src - list of source image features (each NCHW, N=1) or one NCHW tensor
    Returns a list of V tensors C x D x h x w (or one tensor). Differentiable w.r.t. the source features when
    they require grad (one gradient per list element); R, t and the intrinsics get none.
    '''
    first = feat_img_src[0] if isinstance(feat_img_src, (list, tuple)) else feat_img_src
    K, rays = _cam_tensors(cam_intrinsic, _dev(first))
    cx = float(cam_intrinsic['intrinsic_M'][0, 2]); cy = float(cam_intrinsic['intrinsic_M'][1, 2])
    return _warp_views(feat_img_src, d_candi, R, t, K, rays, cx, cy)


def warp_img_feats_mgpu(feat_img_src, d_candi, R, t, IntM_tensors, unit_ray_arrays_2D):
    r'''homography.py:183-232: intrinsics arrive as stacked tensors (1x3x3, 1x3xhw) scattered by
    DataParallel; u/v centre are IntM[0,2], IntM[1,2].'''
    first = feat_img_src[0] if isinstance(feat_img_src, (list, tuple)) else feat_img_src
    dev = _dev(first)
    K = IntM_tensors.squeeze(0).to(device=dev, dtype=torch.float32).contiguous()
    rays = unit_ray_arrays_2D.squeeze(0).to(device=dev, dtype=torch.float32).contiguous()
    Kh = K.cpu()
    return _warp_views(feat_img_src, d_candi, R, t, K, rays, float(Kh[0, 2]), float(Kh[1, 2]))


def _set_vol_border(vol, border_val):
    '''homography.py:873-887 (clone + six face fills). Standalone helper; resample_vol_cuda
    applies the same overwrite inside its kernel without materialising the copy.'''
    vol_ = vol + 0.
    vol_[:, :, 0, :, :] = border_val
    vol_[:, :, :, 0, :] = border_val
    vol_[:, :, :, :, 0] = border_val
    vol_[:, :, -1, :, :] = border_val
    vol_[:, :, :, -1, :] = border_val
    vol_[:, :, :, :, -1] = border_val
    return vol_


def resample_params(cam_intrinsic, d_candi, d_candi_new=None):
    """(d_pts float32 ndarray, tan_hh, tan_hv, z_half, z_radius) per homography.py:668-696."""
    hhfov = math.radians(cam_intrinsic['hfov']) * .5
    hvfov = math.radians(cam_intrinsic['vfov']) * .5
    d_ = d_candi_new if d_candi_new is not None else d_candi
    d_pts = np.asarray(d_).astype(np.float32)
    if d_candi_new is not None:
        z_max, z_min = np.max(d_candi), np.min(d_candi)          # float64, as numpy scalars (:687)
        z_half = np.float32((z_max + z_min) * .5)
        z_radius = np.float32((z_max - z_min) * .5)
    else:
        z_max, z_min = np.float32(d_pts.max()), np.float32(d_pts.min())   # point-cloud z = f32(d)*1 (:689-690)
        z_half = np.float32((z_max + z_min) * np.float32(.5))
        z_radius = np.float32((z_max - z_min) * np.float32(.5))
    return d_pts, np.float32(math.tan(hhfov)), np.float32(math.tan(hvfov)), z_half, z_radius


def _resample_forward(vol, E, rays, dp, D, H, W, tan_hh, tan_hv, z_half, z_radius, pad, clamp):
    L = _lib.lib()
    out = torch.empty((D, H, W), device=vol.device, dtype=torch.float32)
    lo, hi = (clamp if clamp is not None else (0., 0.))
    check(L.nrgbd_resample_dpv(ptr(vol), H * W, 1, ptr(E), ptr(rays), ptr(dp), D, H, W, _F(tan_hh), _F(tan_hv),
                               _F(z_half), _F(z_radius), _F(pad), 1 if clamp is not None else 0,
                               _F(lo), _F(hi), ptr(out), H * W, 1, _stream()))
    return out


class _ResampleDpv(torch.autograd.Function):
    """resample_vol_cuda with the volume gradient autograd gives the reference through _set_vol_border +
    grid_sample(bilinear, border) 3-D (homography.py:713-716), and through torch.clamp for the `clamp` extension.
    rel_extM, the intrinsics and the plane depths get no gradient."""

    @staticmethod
    def forward(ctx, src_vol, E, rays, dp, params, pad, clamp):
        N, D, H, W = src_vol.shape
        vol = src_vol.detach().float().contiguous()
        ctx.save_for_backward(vol, E, rays, dp)
        ctx.meta = (params, pad, clamp, src_vol.dtype)
        return _resample_forward(vol, E, rays, dp, D, H, W, *params, pad, clamp)

    @staticmethod
    def backward(ctx, grad_out):
        L = _lib.lib()
        vol, E, rays, dp = ctx.saved_tensors
        (tan_hh, tan_hv, z_half, z_radius), pad, clamp, dtype = ctx.meta
        N, D, H, W = vol.shape
        lo, hi = (clamp if clamp is not None else (0., 0.))
        with torch.cuda.device(vol.device):
            go = grad_out.detach().float().contiguous()
            g = torch.empty((D, H, W), device=vol.device, dtype=torch.float32)
            check(L.nrgbd_resample_dpv_backward(ptr(vol), H * W, 1, ptr(E), ptr(rays), ptr(dp), D, H, W, _F(tan_hh),
                                                _F(tan_hv), _F(z_half), _F(z_radius), _F(pad),
                                                1 if clamp is not None else 0, _F(lo), _F(hi), ptr(go), H * W, 1,
                                                ptr(g), _stream()))
            g = g.unsqueeze(0)
            if N > 1:          # the forward reads the first volume only
                g = torch.cat([g, torch.zeros((N - 1, D, H, W), device=vol.device, dtype=torch.float32)])
        return g.to(dtype), None, None, None, None, None, None


def resample_vol_cuda(src_vol, rel_extM, cam_intrinsic=None, d_candi=None, d_candi_new=None,
                      padding_value=0., output_tensor=False, is_debug=False,
                      PointsDs_ref_cam_coord_in=None, clamp=None):
    r'''
    homography.py:654-723. src_vol [1,D,H,W]; rel_extM 4x4 tensor; returns [D,H,W].
    if d_candi_new is not None:
    d_candi : candidate depth values for the src view;
    d_candi_new : candidate depth values for the ref view.
    `clamp=(lo, hi)` (extension) fuses the clamp of test_utils/test_KVNet.py:58-59.
    Differentiable w.r.t. src_vol when it requires grad (faces of the volume get zero gradient, as the reference
    overwrites them before sampling); rel_extM, the intrinsics and the plane depths get none.
    '''
    assert d_candi is not None, 'd_candi should be some np.array object'
    if PointsDs_ref_cam_coord_in is not None or is_debug:
        raise _lib.NrgbdError('resample_vol_cuda: PointsDs_ref_cam_coord_in / is_debug are not supported '
                              '(the point cloud is never materialised)')
    dev = _dev(src_vol)
    with torch.cuda.device(dev):
        N, D, H, W = src_vol.shape
        K, rays = _cam_tensors(cam_intrinsic, dev)
        d_pts, tan_hh, tan_hv, z_half, z_radius = resample_params(cam_intrinsic, d_candi, d_candi_new)
        dp = planes_tensor(d_pts, dev)
        E = rel_extM.detach().to(device=dev, dtype=torch.float32).contiguous()
        params = (tan_hh, tan_hv, z_half, z_radius)
        if torch.is_grad_enabled() and src_vol.requires_grad:
            return _ResampleDpv.apply(src_vol, E, rays, dp, params, float(padding_value), clamp)
        vol = src_vol.float().contiguous()
        return _resample_forward(vol, E, rays, dp, D, H, W, *params, float(padding_value), clamp)


# ---------------------------------------------------------------------------------------------------------------
# f-3: depth-map back-warp of the local bundle adjustment (warping/homography.py:479-574) with the gradients
# ICP/opt_pose_numerical.py:99-160 takes through it (w.r.t. R, t; also w.r.t. the images, as autograd would give)
# ---------------------------------------------------------------------------------------------------------------
class _LbaBackWarp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, imgs, dmap, Rs, ts, K, rays):
        L = _lib.lib()
        N, C, H, W = imgs.shape
        out = torch.empty((N, C, H, W), device=imgs.device, dtype=torch.float32)
        check(L.nrgbd_lba_back_warp(ptr(imgs), ptr(dmap), ptr(Rs), ptr(ts), ptr(K), ptr(rays), N, C, H, W, ptr(out), _stream()))
        ctx.save_for_backward(imgs, dmap, Rs, ts, K, rays)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        imgs, dmap, Rs, ts, K, rays = ctx.saved_tensors
        L = _lib.lib()
        N, C, H, W = imgs.shape
        need_img, need_pose = ctx.needs_input_grad[0], ctx.needs_input_grad[2] or ctx.needs_input_grad[3]
        if ctx.needs_input_grad[1]:
            raise NotImplementedError('back_warp_th_Rt: no gradient with respect to the depth map (the reference optimises R, t only)')
        g_img = torch.empty_like(imgs) if need_img else None
        g_R = torch.empty((N, 3, 3), device=imgs.device, dtype=torch.float32) if need_pose else None
        g_t = torch.empty((N, 3), device=imgs.device, dtype=torch.float32) if need_pose else None
        if need_img or need_pose:
            ws = torch.empty(N * 12, device=imgs.device, dtype=torch.float64)
            go = grad_out.float().contiguous()
            with torch.cuda.device(imgs.device):
                check(L.nrgbd_lba_back_warp_backward(ptr(go), ptr(imgs), ptr(dmap), ptr(Rs), ptr(ts), ptr(K), ptr(rays), N, C, H, W,
                                                     ptr(g_img), ptr(g_R), ptr(g_t), ctypes.c_void_p(ws.data_ptr()), _stream()))
        return g_img, None, g_R if ctx.needs_input_grad[2] else None, g_t if ctx.needs_input_grad[3] else None, None, None


def back_warp_th_Rt_msrc(imgs_src, dmap, Rs, ts, cam_intrinsic):
    '''
    imgs_src - NCHW multiple src frames
    Rs, ts - Rs[iview, ... ], ts[iview, ...] rotation/translation from ref to src view
    Given the depth map ( 2D torch tensor), the camera poses (R,t, as torch.tensor) warp the src. image
    (warping/homography.py:479-529; one fused kernel, differentiable w.r.t. imgs_src, Rs and ts)
    '''
    assert isinstance(imgs_src, torch.Tensor)
    dev = _dev(imgs_src)
    npts = dmap.numel()
    assert cam_intrinsic['unit_ray_array_2D'].shape[1] == npts
    K, rays = _cam_tensors(cam_intrinsic, dev)
    with torch.cuda.device(dev):
        imgs = imgs_src.float().contiguous()
        d = dmap.detach().to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        Rs_ = Rs.to(device=dev, dtype=torch.float32).reshape(-1, 3, 3).contiguous()
        ts_ = ts.to(device=dev, dtype=torch.float32).reshape(-1, 3).contiguous()
        assert Rs_.shape[0] == imgs.shape[0] and ts_.shape[0] == imgs.shape[0]
        return _LbaBackWarp.apply(imgs, d, Rs_, ts_, K, rays)


def back_warp_th_Rt(img_src, dmap, R, t, cam_intrinsic):
    '''
    img_src - NCHW
    Given the depth map ( 2D torch tensor), the camera poses (R,t, as torch.tensor) warp the src. image
    R, t - rotation/translation from ref to src view   (warping/homography.py:530-574)
    '''
    assert isinstance(R, torch.Tensor) and isinstance(t, torch.Tensor), 'R,t should be torch tensors'
    assert img_src.shape[0] == 1
    return back_warp_th_Rt_msrc(img_src, dmap, R.reshape(1, 3, 3), t.reshape(1, 3), cam_intrinsic)
