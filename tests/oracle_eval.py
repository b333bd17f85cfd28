"""CPU oracle of KVNET.forward with the module in .eval(): the BatchNorm layers that track running statistics use
them, every other layer keeps batch statistics (numpy float32, TEST INFRASTRUCTURE ONLY).

Layers built with track_running_stats=True in the reference:
  - the 11 BatchNorm3d of K-Net: psm_submodule.convbn_3d (models/psm_submodule.py:19-23), used by
    models/basic.py:71-94 (dres0.0, dres0.2, dres1..4.{0,2}, classify.0);
  - the downsample BatchNorm2d of the feature CNN's layer2.0 and layer3.0 (models/psm_submodule.py:128-131).
All others come from psm_submodule.convbn (:10-16) with bn_running_avg=False (batch statistics in either mode).
A layer counts as tracked when the state_dict holds its running_mean, exactly as in the reference module tree.

The primitives (convolutions, batch-statistics BatchNorm, pooling, plane sweep, R-Net) are those of
oracle/kvnet_oracle.py; the orchestration below restates models/KVNET.py:93-185 with a `training` switch.
"""
import numpy as np

from oracle import kvnet_oracle as N
from oracle import planesweep_oracle as G

f32 = np.float32


def batch_norm_eval(x, gamma, beta, running_mean, running_var, eps=N.BN_EPS):
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
    return (pre + '.running_mean') in P.sd


def bn(P, pre, x, training):
    """BatchNorm `pre` (pre.weight, pre.bias): running statistics in eval mode for a tracked layer, batch statistics
    otherwise (also in eval mode: nn.BatchNorm with track_running_stats=False)."""
    if not training and tracked(P, pre):
        return batch_norm_eval(x, P(pre + '.weight'), P(pre + '.bias'), P(pre + '.running_mean'), P(pre + '.running_var'))
    return N.batch_norm(x, P(pre + '.weight'), P(pre + '.bias'))


def _convbn(P, pre, x, stride, pad, dilation, training):
    p = dilation if dilation > 1 else pad
    return bn(P, pre + '.1', N.conv2d(x, P(pre + '.0.weight'), None, stride, p, dilation), training)


def _basic_block(P, pre, x, stride, dilation, has_down, training):
    out = N.relu(_convbn(P, pre + '.conv1.0', x, stride, 1, dilation, training))
    out = _convbn(P, pre + '.conv2', out, 1, 1, dilation, training)
    if has_down:
        x = bn(P, pre + '.downsample.1', N.conv2d(x, P(pre + '.downsample.0.weight'), None, stride, 0, 1), training)
    return out + x


def _layer(P, pre, x, blocks, stride, dilation, has_down, training):
    for i in range(blocks):
        x = _basic_block(P, '%s.%d' % (pre, i), x, stride if i == 0 else 1, dilation, has_down and i == 0, training)
    return x


def feature_extraction(P, x, training):
    """psm_submodule.feature_extraction.forward :141-167 -> (layer1 out @1/2, feat @1/4)."""
    pre = 'feature_extractor.feature_extraction'
    o = N.relu(_convbn(P, pre + '.firstconv.0', x, 2, 1, 1, training))
    o = N.relu(_convbn(P, pre + '.firstconv.2', o, 1, 1, 1, training))
    o = N.relu(_convbn(P, pre + '.firstconv.4', o, 1, 1, 1, training))
    l1 = _layer(P, pre + '.layer1', o, 3, 1, 1, False, training)
    raw = _layer(P, pre + '.layer2', l1, 16, 2, 1, True, training)
    o = _layer(P, pre + '.layer3', raw, 3, 1, 1, True, training)
    skip = _layer(P, pre + '.layer4', o, 3, 1, 2, False, training)
    hw = skip.shape[2:]
    branches = []
    for name, k in (('branch1', 64), ('branch2', 32), ('branch3', 16), ('branch4', 8)):
        b = N.relu(_convbn(P, '%s.%s.1' % (pre, name), N.avg_pool2d(skip, k), 1, 0, 1, training))
        branches.append(N.upsample_bilinear_ac(b, hw))
    b1, b2, b3, b4 = branches
    o = N.relu(_convbn(P, pre + '.lastconv.0', np.concatenate((raw, skip, b4, b3, b2, b1), axis=1), 1, 1, 1, training))
    return l1, N.conv2d(o, P(pre + '.lastconv.2.weight'), None, 1, 0, 1)


def d_net(P, ref_frame, src_frames, src_cam_poses, cam, d_candi, sigma, training):
    """models/basic.py:223-323 (as kvnet_oracle.d_net)."""
    l1, feats = feature_extraction(P, np.concatenate((src_frames[0], ref_frame), axis=0), training)
    feat_src = feats[:-1][None]
    feat_ref = feats[-1:]
    dw = int(ref_frame.shape[3] / feat_ref.shape[3])
    feat_ref = np.concatenate((feat_ref, N.avg_pool2d(ref_frame, dw)), axis=1)
    feat_src = np.concatenate((feat_src, N.avg_pool2d(src_frames[0], dw)[None]), axis=2)
    costV = G.est_swp_volume_v4(feat_ref, feat_src, d_candi, src_cam_poses[0, :, :3, :3], src_cam_poses[0, :, :3, 3], cam,
                                sigma, 'L2')
    return G.log_softmax(-costV, axis=1), [feat_ref[:, :-3], l1[-1:]]


def kv_net(P, vol, training):
    """models/basic.py:113-139."""
    def cb(name, x):
        return bn(P, name + '.1', N.conv3d(x, P(name + '.0.weight')), training)
    c = N.relu(cb('kv_net.dres0.2', N.relu(cb('kv_net.dres0.0', vol))))
    for i in (1, 2, 3, 4):
        c = cb('kv_net.dres%d.2' % i, N.relu(cb('kv_net.dres%d.0' % i, c))) + c
    return N.conv3d(N.relu(cb('kv_net.classify.0', c)), P('kv_net.classify.2.weight'))


def kvnet_forward(sd, ref_frame, src_frames, src_cam_poses, cam, d_candi, sigma, BV_predict=None, training=False):
    """models/KVNET.py:93-185 -> (dmap_cur_refined, dmap_refined, BV_cur, DPV); training=True equals
    oracle.kvnet_oracle.kvnet_forward."""
    P = sd if isinstance(sd, N.Params) else N.Params(sd)
    BV_cur, feats = d_net(P, ref_frame, src_frames, src_cam_poses, cam, d_candi, sigma, training)
    feats.append(ref_frame)
    dmap_cur_refined = N.r_net(P, np.exp(BV_cur), feats)
    if BV_predict is None or not G.valid_dpv(BV_predict):
        return dmap_cur_refined, dmap_cur_refined, BV_cur, BV_cur
    rate = int(ref_frame.shape[3] / BV_cur.shape[3])
    ref_dw = N.avg_pool2d(ref_frame, rate)
    src_dw = [N.avg_pool2d(s[None], rate) for s in src_frames[0]]
    warped = G.warp_img_feats_v3(src_dw, d_candi, [p[:3, :3] for p in src_cam_poses[0]], [p[:3, 3] for p in src_cam_poses[0]],
                                 cam)
    D = len(d_candi)
    vol = np.concatenate((np.concatenate(warped, axis=0), np.repeat(ref_dw[0][:, None], D, axis=1), BV_cur - BV_predict),
                         axis=0)[None]
    DPV = G.log_softmax(kv_net(P, vol, training)[:, 0] + BV_predict, axis=1)
    return dmap_cur_refined, N.r_net(P, np.exp(DPV), feats), BV_cur, DPV
