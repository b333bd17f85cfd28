"""CPU oracle, network half: the conv/BN stacks and KVNET.forward orchestration.

TEST INFRASTRUCTURE ONLY (see planesweep_oracle.py header for the rules).

numpy float32 restatement (im2col + BLAS sgemm) of:
  models/psm_submodule.py:10-16,31-49,76-167   feature CNN (batch-statistics BN; running statistics in .eval())
  models/basic.py:53-139                        K-Net (conv3d + BN3d residual stack)
  models/basic.py:223-323                       D-Net forward
  models/Refine.py:24-107                       R-Net (RefineNet_DPV_upsample)
  models/KVNET.py:93-185                        KVNET.forward (both branches)
Parameters are a dict {state_dict name: ndarray} using the reference's names
(KVNET.state_dict(), with or without the DataParallel 'module.' prefix).
"""
from __future__ import annotations

import math
import numpy as np

from . import planesweep_oracle as G

f32 = np.float32
BN_EPS = 1e-5           # nn.BatchNorm2d/3d default eps
LEAKY = 0.01            # nn.LeakyReLU default negative_slope


# --------------------------------------------------------------------------
# primitive layers (NCHW / NCDHW, float32)
# --------------------------------------------------------------------------
def conv2d(x, w, b=None, stride=1, pad=0, dilation=1):
    """nn.Conv2d forward: cross-correlation, zero padding."""
    x = np.asarray(x, f32); w = np.asarray(w, f32)
    N, C, H, W = x.shape
    O, Ci, kh, kw = w.shape
    assert Ci == C
    Ho = (H + 2 * pad - dilation * (kh - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dilation * (kw - 1) - 1) // stride + 1
    xp = np.pad(x, ((0, 0), (0, 0), (pad, pad), (pad, pad))) if pad else x
    out = np.empty((N, O, Ho, Wo), f32)
    wm = w.reshape(O, C * kh * kw)
    for n in range(N):
        cols = np.empty((C, kh, kw, Ho, Wo), f32)
        for i in range(kh):
            for j in range(kw):
                cols[:, i, j] = xp[n, :, i * dilation:i * dilation + (Ho - 1) * stride + 1:stride,
                                   j * dilation:j * dilation + (Wo - 1) * stride + 1:stride]
        o = wm @ cols.reshape(C * kh * kw, Ho * Wo)
        out[n] = o.reshape(O, Ho, Wo)
    if b is not None:
        out += np.asarray(b, f32).reshape(1, O, 1, 1)
    return out


def conv_transpose2d(x, w, b=None, stride=2, pad=1):
    """nn.ConvTranspose2d forward (w is [Cin, Cout, kh, kw]), output_padding 0."""
    x = np.asarray(x, f32); w = np.asarray(w, f32)
    N, C, H, W = x.shape
    Ci, O, kh, kw = w.shape
    assert Ci == C
    Ho = (H - 1) * stride - 2 * pad + kh
    Wo = (W - 1) * stride - 2 * pad + kw
    full = np.zeros((N, O, (H - 1) * stride + kh, (W - 1) * stride + kw), f32)
    wm = w.reshape(C, O * kh * kw)
    for n in range(N):
        contrib = (wm.T @ x[n].reshape(C, H * W)).reshape(O, kh, kw, H, W)
        for i in range(kh):
            for j in range(kw):
                full[n, :, i:i + (H - 1) * stride + 1:stride, j:j + (W - 1) * stride + 1:stride] += contrib[:, i, j]
    out = full[:, :, pad:pad + Ho, pad:pad + Wo]
    if b is not None:
        out = out + np.asarray(b, f32).reshape(1, O, 1, 1)
    return np.ascontiguousarray(out, f32)


def conv3d(x, w, pad=1):
    """nn.Conv3d forward, stride 1, 3x3x3, zero padding, no bias. x [1,C,D,H,W]."""
    x = np.asarray(x, f32); w = np.asarray(w, f32)
    N, C, D, H, W = x.shape
    O, Ci, kd, kh, kw = w.shape
    assert N == 1 and Ci == C
    xp = np.pad(x[0], ((0, 0), (pad, pad), (pad, pad), (pad, pad)))
    out = np.zeros((O, D * H * W), f32)
    # accumulate per kd slab to bound the im2col buffer
    for a in range(kd):
        cols = np.empty((C, kh, kw, D, H, W), f32)
        for i in range(kh):
            for j in range(kw):
                cols[:, i, j] = xp[:, a:a + D, i:i + H, j:j + W]
        out += w[:, :, a].reshape(O, C * kh * kw) @ cols.reshape(C * kh * kw, D * H * W)
    return out.reshape(1, O, D, H, W)


def batch_norm(x, gamma, beta, eps=BN_EPS):
    """BatchNorm in training mode (batch statistics; the reference never calls
    .eval(), and psm_submodule.convbn builds BN2d with track_running_stats=False):
    y = (x - mean) / sqrt(var_biased + eps) * gamma + beta over all dims but C.
    Statistics accumulated in float64, applied in float32 as
    y = x * scale + shift with scale = gamma * rsqrt(var+eps), shift = beta - mean*scale."""
    x = np.asarray(x, f32)
    axes = tuple(i for i in range(x.ndim) if i != 1)
    mean = x.mean(axis=axes, dtype=np.float64)
    var = np.square(x.astype(np.float64) - mean.reshape((1, -1) + (1,) * (x.ndim - 2))).mean(axis=axes)
    inv = 1.0 / np.sqrt(var + eps)
    shp = (1, -1) + (1,) * (x.ndim - 2)
    y = (x.astype(np.float64) - mean.reshape(shp)) * inv.reshape(shp) * np.asarray(gamma, np.float64).reshape(shp) \
        + np.asarray(beta, np.float64).reshape(shp)
    return y.astype(f32)


def relu(x):
    return np.maximum(x, f32(0))


def leaky_relu(x):
    return np.where(x >= 0, x, x * f32(LEAKY)).astype(f32)


def avg_pool2d(x, k):
    """F.avg_pool2d(x, k) (stride k, floor)."""
    x = np.asarray(x, f32)
    N, C, H, W = x.shape
    Ho, Wo = H // k, W // k
    v = x[:, :, :Ho * k, :Wo * k].reshape(N, C, Ho, k, Wo, k)
    return (v.sum(axis=(3, 5), dtype=np.float64) / (k * k)).astype(f32)


def upsample_bilinear_ac(x, size):
    """F.upsample(mode='bilinear', align_corners=True)."""
    x = np.asarray(x, f32)
    N, C, H, W = x.shape
    Ho, Wo = size

    def axis_coords(n_in, n_out):
        if n_out == 1 or n_in == 1:
            src = np.zeros(n_out, np.float64)
        else:
            src = np.arange(n_out, dtype=np.float64) * ((n_in - 1) / (n_out - 1))
        src = src.astype(f32)
        i0 = np.floor(src).astype(np.int64)
        i0 = np.minimum(i0, n_in - 1)
        i1 = np.minimum(i0 + 1, n_in - 1)
        l1 = (src - i0.astype(f32)).astype(f32)
        return i0, i1, (f32(1) - l1), l1
    y0, y1, hy0, hy1 = axis_coords(H, Ho)
    x0, x1, wx0, wx1 = axis_coords(W, Wo)
    r0 = x[:, :, y0, :]; r1 = x[:, :, y1, :]
    top = r0[:, :, :, x0] * wx0 + r0[:, :, :, x1] * wx1
    bot = r1[:, :, :, x0] * wx0 + r1[:, :, :, x1] * wx1
    return (top * hy0[None, None, :, None] + bot * hy1[None, None, :, None]).astype(f32)


# --------------------------------------------------------------------------
# parameter access
# --------------------------------------------------------------------------
class Params:
    def __init__(self, sd):
        self.sd = {(k[7:] if k.startswith('module.') else k): np.asarray(v) for k, v in sd.items()}

    def __call__(self, name):
        return self.sd[name]


def batch_norm_eval(x, gamma, beta, running_mean, running_var, eps=BN_EPS):
    """nn.BatchNorm{2,3}d.forward in eval mode (ATen's CPU transform, batch_norm_cpu_collect_linear_and_constant_terms),
    per channel in float32:
        alpha = (1 / sqrt(running_var + eps)) * gamma,   beta' = beta - running_mean * alpha,   y = x * alpha + beta'
    The running buffers are only read."""
    x = np.asarray(x, f32)
    invstd = f32(1) / np.sqrt(np.asarray(running_var, f32) + f32(eps))
    alpha = (invstd * np.asarray(gamma, f32)).astype(f32)
    beta2 = (np.asarray(beta, f32) - np.asarray(running_mean, f32) * alpha).astype(f32)
    shp = (1, -1) + (1,) * (x.ndim - 2)
    return (x * alpha.reshape(shp) + beta2.reshape(shp)).astype(f32)


def tracked(P, pre):
    """Whether BatchNorm `pre` tracks running statistics: the state_dict holds its running_mean, as in the reference's
    module tree. Tracked: the 11 BatchNorm3d of K-Net (psm_submodule.convbn_3d :19-23, used by basic.py:71-94) and the
    downsample BatchNorm2d of the feature CNN's layer2.0 and layer3.0 (psm_submodule.py:128-131). Every other layer
    comes from psm_submodule.convbn (:10-16) with bn_running_avg=False."""
    return (pre + '.running_mean') in P.sd


def bn(P, pre, x, training=True):
    """BatchNorm `pre` (pre.weight, pre.bias): running statistics in eval mode for a tracked layer, batch statistics
    otherwise (also in eval mode: nn.BatchNorm with track_running_stats=False)."""
    if not training and tracked(P, pre):
        return batch_norm_eval(x, P(pre + '.weight'), P(pre + '.bias'), P(pre + '.running_mean'), P(pre + '.running_var'))
    return batch_norm(x, P(pre + '.weight'), P(pre + '.bias'))


def _convbn(P, pre, x, stride, pad, dilation, training=True):
    """psm_submodule.convbn :10-16 -> Sequential(Conv2d(bias=False), BatchNorm2d)."""
    w = P(pre + '.0.weight')
    p = dilation if dilation > 1 else pad
    y = conv2d(x, w, None, stride, p, dilation)
    return bn(P, pre + '.1', y, training)


def _basic_block(P, pre, x, stride, pad, dilation, has_down, training=True):
    """psm_submodule.BasicBlock :31-49 (no ReLU after the residual add)."""
    out = relu(_convbn(P, pre + '.conv1.0', x, stride, pad, dilation, training))
    out = _convbn(P, pre + '.conv2', out, 1, pad, dilation, training)
    if has_down:
        sc = conv2d(x, P(pre + '.downsample.0.weight'), None, stride, 0, 1)
        x = bn(P, pre + '.downsample.1', sc, training)
    return out + x


def _layer(P, pre, x, blocks, stride, dilation, has_down, training=True):
    for i in range(blocks):
        x = _basic_block(P, '%s.%d' % (pre, i), x, stride if i == 0 else 1, 1, dilation,
                         has_down and i == 0, training)
    return x


def feature_extraction(P, pre, x, training=True):
    """psm_submodule.feature_extraction.forward :141-167 (multi_scale=True).
    pre = 'feature_extractor.feature_extraction'. Returns (layer1 out @1/2, feat @1/4)."""
    o = relu(_convbn(P, pre + '.firstconv.0', x, 2, 1, 1, training))
    o = relu(_convbn(P, pre + '.firstconv.2', o, 1, 1, 1, training))
    o = relu(_convbn(P, pre + '.firstconv.4', o, 1, 1, 1, training))
    l1 = _layer(P, pre + '.layer1', o, 3, 1, 1, False, training)
    raw = _layer(P, pre + '.layer2', l1, 16, 2, 1, True, training)
    o = _layer(P, pre + '.layer3', raw, 3, 1, 1, True, training)
    skip = _layer(P, pre + '.layer4', o, 3, 1, 2, False, training)
    hw = skip.shape[2:]
    branches = []
    for name, k in (('branch1', 64), ('branch2', 32), ('branch3', 16), ('branch4', 8)):
        b = avg_pool2d(skip, k)
        b = relu(_convbn(P, '%s.%s.1' % (pre, name), b, 1, 0, 1, training))
        branches.append(upsample_bilinear_ac(b, hw))
    b1, b2, b3, b4 = branches
    cat = np.concatenate((raw, skip, b4, b3, b2, b1), axis=1)
    o = relu(_convbn(P, pre + '.lastconv.0', cat, 1, 1, 1, training))
    feat = conv2d(o, P(pre + '.lastconv.2.weight'), None, 1, 0, 1)
    return l1, feat


def d_net(P, ref_frame, src_frames, src_cam_poses, cam_intrinsics, d_candi, sigma, feat_dist='L2', training=True):
    """models/basic.py:223-323 with use_img_intensity=True, BV_log=True,
    output_features=True, BV_predict=None."""
    assert src_frames.shape[0] == 1
    l1, feats = feature_extraction(P, 'feature_extractor.feature_extraction',
                                   np.concatenate((src_frames[0], ref_frame), axis=0), training)
    feat_ref_l1 = l1[-1:]
    feat_src = feats[:-1][None]
    feat_ref = feats[-1:]
    dw = int(ref_frame.shape[3] / feat_ref.shape[3])
    feat_ref = np.concatenate((feat_ref, avg_pool2d(ref_frame, dw)), axis=1)
    feat_src = np.concatenate((feat_src, avg_pool2d(src_frames[0], dw)[None]), axis=2)
    Rs = src_cam_poses[0, :, :3, :3]
    ts = src_cam_poses[0, :, :3, 3]
    costV = G.est_swp_volume_v4(feat_ref, feat_src, d_candi, Rs, ts, cam_intrinsics, sigma, feat_dist)
    BV = G.log_softmax(-costV, axis=1)
    return BV, [feat_ref[:, :-3], feat_ref_l1]


def kv_net(P, vol, pre='kv_net', training=True):
    """models/basic.py:113-139 (if_normalize=False, up_sample_ratio=None)."""
    def cb(name, x):
        return bn(P, name + '.1', conv3d(x, P(name + '.0.weight')), training)
    c0 = relu(cb(pre + '.dres0.0', vol))
    c0 = relu(cb(pre + '.dres0.2', c0))
    c = c0
    for i in (1, 2, 3, 4):
        r = relu(cb('%s.dres%d.0' % (pre, i), c))
        r = cb('%s.dres%d.2' % (pre, i), r)
        c = r + c
    o = relu(cb(pre + '.classify.0', c))
    return conv3d(o, P(pre + '.classify.2.weight'))


def r_net(P, dpv_raw, img_features, pre='r_net'):
    """models/Refine.py:79-107."""
    def cl(name, x):
        return leaky_relu(conv2d(x, P(name + '.0.weight'), P(name + '.0.bias'), 1, 1, 1))

    def tl(name, x):
        return leaky_relu(conv_transpose2d(x, P(name + '.0.weight'), P(name + '.0.bias'), 2, 1))
    o = cl(pre + '.conv0', np.concatenate([dpv_raw, img_features[0]], axis=1))
    o = cl(pre + '.conv0_1', o)
    o = tl(pre + '.trans_conv0', o)
    o = cl(pre + '.conv1', np.concatenate([o, img_features[1]], axis=1))
    o = cl(pre + '.conv1_1', o)
    o = tl(pre + '.trans_conv1', o)
    o = cl(pre + '.conv2', np.concatenate([o, img_features[2]], axis=1))
    o = cl(pre + '.conv2_1', o)
    o = conv2d(o, P(pre + '.conv2_2.weight'), P(pre + '.conv2_2.bias'), 1, 1, 1)
    return G.log_softmax(o, axis=1)


def kvnet_forward(sd, ref_frame, src_frames, src_cam_poses, cam_intrinsics, d_candi, sigma,
                  BV_predict=None, t_win_r=2, cam_intrinsics_call=None, training=True):
    """models/KVNET.py:93-185 (if_refined=True, refineNet_name='DPV').
    cam_intrinsics: the dict captured at construction (used by D-Net, KVNET.py:64-67);
    cam_intrinsics_call: the per-call dict used by the K-Net image warp (:160-161),
    defaults to the same. training=False is the module in .eval(): the BatchNorm layers that track running
    statistics use them (tracked), every other layer keeps batch statistics.
    Returns (dmap_cur_refined, dmap_refined, BV_cur, DPV)."""
    P = sd if isinstance(sd, Params) else Params(sd)
    BV_cur, feats = d_net(P, ref_frame, src_frames, src_cam_poses, cam_intrinsics, d_candi, sigma, training=training)
    feats.append(ref_frame)
    dmap_cur_refined = r_net(P, np.exp(BV_cur), feats)
    if BV_predict is None or not G.valid_dpv(BV_predict):
        return dmap_cur_refined, dmap_cur_refined, BV_cur, BV_cur
    assert BV_predict.shape[0] == 1
    rate = int(ref_frame.shape[3] / BV_cur.shape[3])
    ref_dw = avg_pool2d(ref_frame, rate)
    src_dw = [avg_pool2d(s[None], rate) for s in src_frames[0]]
    Rs = [p[:3, :3] for p in src_cam_poses[0]]
    ts = [p[:3, 3] for p in src_cam_poses[0]]
    cam = cam_intrinsics_call if cam_intrinsics_call is not None else cam_intrinsics
    warped = G.warp_img_feats_v3(src_dw, d_candi, Rs, ts, cam)
    D = len(d_candi)
    ref_rep = np.repeat(ref_dw[0][:, None], D, axis=1)
    vol = np.concatenate((np.concatenate(warped, axis=0), ref_rep, BV_cur - BV_predict), axis=0)[None]
    gain = kv_net(P, vol, training=training)
    DPV = G.log_softmax(gain[:, 0] + BV_predict, axis=1)
    dmap_refined = r_net(P, np.exp(DPV), feats)
    return dmap_cur_refined, dmap_refined, BV_cur, DPV
