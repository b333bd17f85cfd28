"""Seeded cases for the gradients of the geometry mirrors (numpy only): the image / feature warp
(warp_img_feats_v3 / _mgpu), the DPV resample (resample_vol_cuda) and the depth regression (depth_val_regression).

Shared by tests/golden/make_golden.py grad (which runs torch autograd through the unmodified reference on them) and the
tests. Every input and every upstream gradient is regenerated from its seed; the fixtures hold gradients only.
"""
import math

import numpy as np

from neuralrgbd_b200 import synth
from tests import cases

# warp: V = 4 views (the list form of models/KVNET.py:153-159), except the tensor-form case (one N = 1 tensor)
WARP_CFG = {
    'warp_v4_c3_37x53_d7': dict(seed=81, h=37, w=53, D=7, C=3, V=4),
    'warp_v4_c67_37x53_d7': dict(seed=82, h=37, w=53, D=7, C=67, V=4),
    # the K-Net warp of the 640x480 workload: quarter resolution, 64 planes
    'warp_v4_c3_120x160_d64': dict(seed=83, h=120, w=160, D=64, C=3, V=4),
    'warp_v4_c67_120x160_d64': dict(seed=84, h=120, w=160, D=64, C=67, V=4),
    'warp_tensor_c5_37x53_d7': dict(seed=85, h=37, w=53, D=7, C=5, V=1, tensor=True),
}
WARP_CASES = list(WARP_CFG)

# resample: quarter (120x160) and image (480x640) resolution of the 640x480 workload, 64 planes
RESAMPLE_CFG = {
    'rs_identity_q_d64': dict(seed=91, h=120, w=160, D=64, identity=True),
    'rs_pose_q_d64': dict(seed=92, h=120, w=160, D=64),
    'rs_identity_dnew_q_d64': dict(seed=93, h=120, w=160, D=64, identity=True, d_new=True),
    'rs_pose_dnew_q_d64': dict(seed=94, h=120, w=160, D=64, d_new=True),
    # a clamp range that cuts through the volume's values, so the clamp mask matters
    'rs_pose_clamp_q_d64': dict(seed=95, h=120, w=160, D=64, clamp=(-5.0, -3.0)),
    'rs_pose_img_d64': dict(seed=96, h=480, w=640, D=64),
    'rs_pose_dnew_img_d64': dict(seed=97, h=480, w=640, D=64, d_new=True, clamp=(-1000.0, 0.0)),
}
RESAMPLE_CASES = list(RESAMPLE_CFG)

REGRESSION_CFG = {
    'reg_log_120x160_d64': dict(seed=101, h=120, w=160, D=64, N=1, log=True),
    'reg_lin_120x160_d64': dict(seed=102, h=120, w=160, D=64, N=1, log=False),
    'reg_log_n2_37x53_d16': dict(seed=103, h=37, w=53, D=16, N=2, log=True),
}
REGRESSION_CASES = list(REGRESSION_CFG)


def upstream(seed, shape, zero_block=True):
    """Seeded float32 upstream gradient, with a block of exact zeros (skipped work in the kernels)."""
    g = np.random.default_rng(seed).standard_normal(size=shape, dtype=np.float32)
    if zero_block:
        g.reshape(-1)[: g.size // 8] = 0.0
    return g


def _log_dpv(rng, N, D, h, w):
    logits = 3.0 * np.stack([synth.smooth_image(rng, D, h, w) for _ in range(N)])
    m = logits.max(axis=1, keepdims=True)
    return (logits - m - np.log(np.exp(logits - m).sum(axis=1, keepdims=True))).astype(np.float32)


def warp_case(name):
    """-> dict(imgs [V x (1,C,h,w)] (or one (1,C,h,w) for the tensor form), d, R, t (lists / arrays), w, h, grads)."""
    cfg = WARP_CFG[name]
    rng = np.random.RandomState(cfg['seed'])
    C, h, w, V, D = cfg['C'], cfg['h'], cfg['w'], cfg['V'], cfg['D']
    imgs = [synth.smooth_image(rng, C, h, w)[None].astype(np.float32) for _ in range(V)]
    poses = cases._poses(rng, max(V, 2))[:V]
    d = synth.d_candidates(D)
    R = [np.ascontiguousarray(p[:3, :3]) for p in poses]
    t = [np.ascontiguousarray(p[:3, 3]) for p in poses]
    grads = [upstream(cfg['seed'] * 10 + v, (C, D, h, w)) for v in range(V)]
    c = dict(imgs=imgs, d=d, R=R, t=t, w=w, h=h, C=C, V=V, D=D, grads=grads, tensor=cfg.get('tensor', False))
    if c['tensor']:
        c.update(imgs=imgs[0], R=R[0], t=t[0], grads=grads[0])
    return c


def resample_case(name):
    """-> dict(vol [1,D,h,w] log-DPV, rel 4x4, d, d_new or None, pad, clamp or None, w, h, grad [D,h,w])."""
    cfg = RESAMPLE_CFG[name]
    rng = np.random.RandomState(cfg['seed'])
    D, h, w = cfg['D'], cfg['h'], cfg['w']
    vol = _log_dpv(rng, 1, D, h, w)
    exts = synth.camera_track(rng, 2, 0.05)
    rel = np.linalg.inv(exts[1].dot(np.linalg.inv(exts[0]))).astype(np.float32)
    if cfg.get('identity'):
        rel = np.eye(4, dtype=np.float32)
    d = synth.d_candidates(D)
    d_new = synth.d_candidates(D, 0.3, 4.0) if cfg.get('d_new') else None
    return dict(vol=vol, rel=rel, d=d, d_new=d_new, w=w, h=h, D=D, pad=math.log(1.0 / D), clamp=cfg.get('clamp'),
                grad=upstream(cfg['seed'] * 10, (D, h, w)))


def regression_case(name):
    """-> dict(bv [N,D,h,w] (log-DPV, or its probabilities when log=False), d, log, grad [1,h,w])."""
    cfg = REGRESSION_CFG[name]
    rng = np.random.RandomState(cfg['seed'])
    bv = _log_dpv(rng, cfg['N'], cfg['D'], cfg['h'], cfg['w'])
    if not cfg['log']:
        bv = np.exp(bv).astype(np.float32)
    return dict(bv=bv, d=synth.d_candidates(cfg['D']), log=cfg['log'], grad=upstream(cfg['seed'] * 10, (1, cfg['h'], cfg['w'])))


SUB_LIMIT = 8000        # values per stored gradient array (strided, cases.subsample_to)


def sub(a):
    return cases.subsample_to(a, SUB_LIMIT)
