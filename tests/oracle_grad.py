"""Numpy backward of the geometry mirrors (f-5): what torch autograd computes through the reference's
warp_img_feats_v3 / _mgpu (F.grid_sample bilinear / zeros), resample_vol_cuda (_set_vol_border + grid_sample bilinear /
border 3-D, + torch.clamp) and depth_val_regression, with respect to the image features, the volume and BV_measure.

Poses, intrinsics and plane depths are constants, so each op is linear in its differentiable input given its sampling
taps (up to the clamp mask and the exp of the regression). The taps come from oracle/planesweep_oracle.py's pinned fp32
coordinate arithmetic; sums are accumulated in float64. Each op also has a float64 forward over the same taps, for
finite-difference checks of the backward.
"""
import math

import numpy as np

from oracle import planesweep_oracle as O

f32 = np.float32
f64 = np.float64


# ---- image / feature warp ----------------------------------------------------------------------------------------
def warp_taps(d_candi, R, t, cam, h, w):
    """Per view: the 4 bilinear corners [(flat index [D*hw], fp32 weight [D*hw])], weight 0 where out of range."""
    d32 = np.asarray(d_candi).astype(f32)
    K, rays = cam['intrinsic_M_cuda'], cam['unit_ray_array_2D']
    cx, cy = cam['intrinsic_M'][0, 2], cam['intrinsic_M'][1, 2]
    taps = []
    for Rv, tv in zip(R, t):
        term1, _, term2 = O.homography_terms(K, Rv, tv, rays)
        gx, gy = O.back_warp_grid(term1, term2, d32, cx, cy)
        taps.append([(i.reshape(-1), wt.reshape(-1)) for i, wt in O._corners(gx, gy, w, h)])
    return taps


def warp_forward64(imgs, taps, D):
    """imgs: per view [C, hw] -> per view [C, D, hw] in float64."""
    outs = []
    for img, tp in zip(imgs, taps):
        img = np.asarray(img, f64)
        acc = np.zeros((img.shape[0], tp[0][0].size), f64)
        for idx, wt in tp:
            acc += img[:, idx] * wt.astype(f64)[None]
        outs.append(acc.reshape(img.shape[0], D, -1))
    return outs


def warp_backward(grads, taps, hw):
    """grads: per view [C, D, hw] -> per view d loss / d image [C, hw] (float64 scatter-add of grad * weight)."""
    outs = []
    for g, tp in zip(grads, taps):
        g = np.asarray(g, f64).reshape(g.shape[0], -1)
        idx = np.concatenate([i for i, _ in tp])
        wt = np.concatenate([x for _, x in tp]).astype(f64)
        outs.append(np.stack([np.bincount(idx, weights=np.tile(gc, 4) * wt, minlength=hw) for gc in g]))
    return outs


def warp_img_feats_backward(grads, d_candi, R, t, cam, h, w):
    """grads: per view [C, D, h, w] -> per view [1, C, h, w] float32 (the list form of warp_img_feats_v3)."""
    taps = warp_taps(d_candi, R, t, cam, h, w)
    return [g.reshape(1, -1, h, w).astype(f32) for g in warp_backward(grads, taps, h * w)]


# ---- DPV resample ------------------------------------------------------------------------------------------------
def resample_taps(rel_extM, cam, d_candi, d_candi_new, D, H, W):
    """The 8 trilinear corners of every output voxel, in ATen's order:
    [(flat index [D*hw], fp32 weight, in range, on a face)] (homography.py:654-716 with oracle.resample_vol_cuda's
    coordinate arithmetic)."""
    d_ = d_candi_new if d_candi_new is not None else d_candi
    rays = np.asarray(cam['unit_ray_array']).astype(f32)
    pts = np.stack([f32(d) * rays for d in d_]).astype(f32)
    if d_candi_new is not None:
        z_half = f32((np.max(d_candi) + np.min(d_candi)) * .5)
        z_radius = f32((np.max(d_candi) - np.min(d_candi)) * .5)
    else:
        z_max = pts[..., 2].max(); z_min = pts[..., 2].min()
        z_half = (z_max + z_min) * f32(.5)
        z_radius = (z_max - z_min) * f32(.5)
    E = np.asarray(rel_extM, f32)
    X = pts[..., 0].reshape(-1); Y = pts[..., 1].reshape(-1); Z = pts[..., 2].reshape(-1)

    def row(i):
        acc = (E[i, 0] * X).astype(f32)
        acc = O._fma(E[i, 1], Y, acc)
        acc = O._fma(E[i, 2], Z, acc)
        return O._fma(E[i, 3], f32(1), acc)
    xs, ys, zs, ws = row(0), row(1), row(2), row(3)
    den = zs + f32(1e-10)
    gx = xs / den / f32(math.tan(math.radians(cam['hfov']) * .5))
    gy = ys / den / f32(math.tan(math.radians(cam['vfov']) * .5))
    gz = (zs - z_half) / z_radius
    wden = ws + f32(1e-10)
    gx = (gx / wden).astype(f32); gy = (gy / wden).astype(f32); gz = (gz / wden).astype(f32)
    ix = O._clip(O._unnormalize(gx, W), W - 1)
    iy = O._clip(O._unnormalize(gy, H), H - 1)
    iz = O._clip(O._unnormalize(gz, D), D - 1)
    bad = np.isnan(ix) | np.isnan(iy) | np.isnan(iz)
    ix = np.where(bad, f32(0), ix); iy = np.where(bad, f32(0), iy); iz = np.where(bad, f32(0), iz)
    x0 = np.floor(ix); y0 = np.floor(iy); z0 = np.floor(iz)
    x1 = x0 + f32(1); y1 = y0 + f32(1); z1 = z0 + f32(1)
    taps = []
    for (zz, wz) in ((z0, z1 - iz), (z1, iz - z0)):
        for (yy, wy) in ((y0, y1 - iy), (y1, iy - y0)):
            for (xx, wx) in ((x0, x1 - ix), (x1, ix - x0)):
                wgt = ((wx * wy) * wz).astype(f32)
                xi = xx.astype(np.int64); yi = yy.astype(np.int64); zi = zz.astype(np.int64)
                ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H) & (zi >= 0) & (zi < D) & ~bad
                face = (xi == 0) | (xi == W - 1) | (yi == 0) | (yi == H - 1) | (zi == 0) | (zi == D - 1)
                taps.append((np.where(ok, (zi * H + yi) * W + xi, 0), wgt, ok, face))
    return taps


def resample_forward64(vol, taps, pad, clamp=None):
    """vol [D*hw] -> out [D*hw] in float64 over the same taps (faces read as pad)."""
    vol = np.asarray(vol, f64).reshape(-1)
    out = np.zeros(taps[0][0].size, f64)
    for idx, wgt, ok, face in taps:
        v = np.where(face, float(pad), vol[idx])
        out += np.where(ok, v * wgt.astype(f64), 0.0)
    return np.clip(out, clamp[0], clamp[1]) if clamp is not None else out


def resample_backward(grad, taps, n, res=None, clamp=None):
    """grad [D*hw] -> d loss / d vol [D*hw] (float64). With `clamp`, the gradient passes where lo <= res <= hi
    (torch.clamp's backward), res being the forward value before the clamp."""
    g = np.asarray(grad, f64).reshape(-1)
    if clamp is not None:
        r = np.asarray(res).reshape(-1)
        g = np.where((r >= clamp[0]) & (r <= clamp[1]), g, 0.0)
    out = np.zeros(n, f64)
    for idx, wgt, ok, face in taps:
        keep = ok & ~face
        out += np.bincount(idx[keep], weights=g[keep] * wgt[keep].astype(f64), minlength=n)
    return out


def resample_vol_cuda_backward(grad, src_vol, rel_extM, cam, d_candi, d_candi_new=None, padding_value=0., clamp=None):
    """grad [D,h,w] -> d loss / d src_vol [1,D,h,w] float32. The clamp mask uses the pinned fp32 forward."""
    _, D, H, W = np.asarray(src_vol).shape
    taps = resample_taps(rel_extM, cam, d_candi, d_candi_new, D, H, W)
    res = O.resample_vol_cuda(src_vol, rel_extM, cam, d_candi, d_candi_new, padding_value) if clamp is not None else None
    return resample_backward(grad, taps, D * H * W, res, clamp).reshape(1, D, H, W).astype(f32)


# ---- depth regression --------------------------------------------------------------------------------------------
def depth_val_regression64(BV, d_candi, BV_log=True):
    BV = np.asarray(BV, f64)
    p = np.exp(BV[0]) if BV_log else BV[0]
    return np.tensordot(np.asarray(d_candi, f32).astype(f64), p, axes=(0, 0))[None]


def depth_val_regression_backward(grad, BV, d_candi, BV_log=True):
    """grad [1,h,w] -> d loss / d BV [N,D,h,w] float32: slice 0 gets (g * f32(d)) * exp(BV) (autograd's order through
    misc.py:541-546), or g * f32(d) without the exp; the other slices get zero."""
    BV = np.asarray(BV, f32)
    g = np.asarray(grad, f32).reshape(1, *BV.shape[2:])
    d = np.asarray(d_candi).astype(f32).reshape(-1, 1, 1)
    gd = (g * d).astype(f32)
    out = np.zeros(BV.shape, f32)
    out[0] = (gd * np.exp(BV[0])).astype(f32) if BV_log else gd
    return out
