"""Seeded scenes for the LBA pose optimiser (ICP/opt_pose_numerical.py local_BA_direct(_parallel)), numpy only.

Shared by tests/golden/make_golden.py lba_opt (which runs the live reference on them and commits its outputs), the tests and
tools/bench_lba.py. Every input is regenerated from its seed, so the fixtures hold reference outputs only.
"""
import math

import numpy as np

from tests.cases import cam_for


def _axis_angle(rng, deg):
    a = rng.standard_normal(3); a /= np.linalg.norm(a)
    th = math.radians(deg)
    Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(th) * Kx + (1 - math.cos(th)) * Kx.dot(Kx)


def lba_scene(seed, H, W, V, perturb_R=True, perturb_t=True):
    """A textured plane n.X = d0 (reference camera coordinates) seen by the reference camera and V source cameras.
    Every image is rendered analytically, so the true relative poses (reference -> source, what back_warp_th_Rt takes)
    explain the reference image up to bilinear sampling; the initial poses perturb R and / or t of the true ones.
    -> dict(ref [1,3,H,W], srcs [V] x [1,3,H,W], dmap [1,1,H,W], conf [1,1,H,W], poses_true / poses_init [V,4,4] float32)."""
    from oracle.planesweep_oracle import make_cam_intrinsics
    rng = np.random.RandomState(seed)
    n = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), 1.0]); n /= np.linalg.norm(n)
    d0 = rng.uniform(1.6, 2.4)
    # channel x term x xyz wave vectors (rad / m): wavelengths from about 1.5 m down to 0.3 m, so that every level has texture
    ks = rng.standard_normal((3, 3, 3))
    ks *= (np.array([4.0, 10.0, 20.0])[None, :, None] / np.linalg.norm(ks, axis=2, keepdims=True))
    ph = rng.uniform(0, 2 * math.pi, (3, 3))
    amp = np.array([0.15, 0.12, 0.1])
    rays = cam_for(make_cam_intrinsics, W, H)['unit_ray_array']          # [H, W, 3], z = 1

    def texture(X):                                           # X [H, W, 3] on the plane -> [3, H, W]
        return np.stack([0.5 + sum(amp[j] * np.sin(X.dot(ks[c, j]) + ph[c, j]) for j in range(3)) for c in range(3)])

    def render(R, t):
        Rt_r = rays.dot(R)                                     # R^T r per pixel (row vectors)
        lam = (d0 + n.dot(R.T.dot(t))) / Rt_r.dot(n)
        X = lam[..., None] * Rt_r - R.T.dot(t)[None, None]
        return texture(X)[None].astype(np.float32)

    dmap = (d0 / rays.dot(n))[None, None].astype(np.float32)
    yy, xx = np.mgrid[0:H, 0:W]
    # confidence: smooth, falling to 0 towards the image border (as a DPV's confidence does where views stop overlapping)
    ramp = lambda a, n: np.clip(np.minimum(a + 0.5, n - 0.5 - a) / (0.15 * n), 0, 1)      # noqa: E731
    conf = ((0.65 + 0.3 * np.sin(xx * (2 * math.pi / W) + rng.uniform(0, 6)) * np.cos(yy * (math.pi / H))) * ramp(xx, W) * ramp(yy, H))
    conf = conf[None, None].astype(np.float32)
    poses_true, poses_init, srcs = [], [], []
    for _ in range(V):
        R = _axis_angle(rng, rng.uniform(0.5, 2.0))           # neighbouring frames of a window: the views overlap
        t = rng.uniform(-0.05, 0.05, 3)
        srcs.append(render(R, t))
        Ri = _axis_angle(rng, rng.uniform(0.6, 1.2)).dot(R) if perturb_R else R
        ti = t + (rng.uniform(0.015, 0.03) * rng.standard_normal(3) / math.sqrt(3) if perturb_t else 0.0)
        for lst, (RR, tt) in ((poses_true, (R, t)), (poses_init, (Ri, ti))):
            P = np.eye(4); P[:3, :3] = RR; P[:3, 3] = tt
            lst.append(P.astype(np.float32))
    return dict(ref=render(np.eye(3), np.zeros(3)), srcs=srcs, dmap=dmap, conf=conf, poses_true=np.stack(poses_true),
                poses_init=np.stack(poses_init))


LBA_OPT_MODES = {'m01': [0, 1], 'm11': [1, 1], 'm10': [1, 0]}


def lba_opt_case(name):
    """-> the scene of lba_scene plus entry ('parallel' | 'serial'), opt_vars, dw_scales, max_iter, step, H, W and the cams of
    the pyramid levels (numpy dicts, cams[s] for dw_scales[s])."""
    from oracle.planesweep_oracle import make_cam_intrinsics
    cfg = {'lbaopt_par_m01_v3_64x48': dict(entry='parallel', mode='m01', V=3, H=48, W=64, seed=61, max_iter=8),
           'lbaopt_par_m11_v2_48x80': dict(entry='parallel', mode='m11', V=2, H=48, W=80, seed=62, max_iter=8),
           'lbaopt_par_m10_v3_64x64': dict(entry='parallel', mode='m10', V=3, H=64, W=64, seed=63, max_iter=8),
           'lbaopt_seq_m01_v2_32x64': dict(entry='serial', mode='m01', V=2, H=32, W=64, seed=64, max_iter=8),
           'lbaopt_seq_m11_v2_48x64': dict(entry='serial', mode='m11', V=2, H=48, W=64, seed=65, max_iter=8),
           'lbaopt_seq_m10_v1_48x48': dict(entry='serial', mode='m10', V=1, H=48, W=48, seed=66, max_iter=8),
           # the docs/LBA.md setting: 384 x 256, four source views, 20 iterations per level, step 0.01, translation only
           'lbaopt_par_m01_v4_256x384': dict(entry='parallel', mode='m01', V=4, H=256, W=384, seed=67, max_iter=20)}[name]
    ov = LBA_OPT_MODES[cfg['mode']]
    c = lba_scene(cfg['seed'], cfg['H'], cfg['W'], cfg['V'], perturb_R=ov[0] == 1, perturb_t=ov[0] != 1 or ov[1] == 1)
    dw = [4, 2, 1]
    c.update(entry=cfg['entry'], opt_vars=ov, dw_scales=dw, max_iter=cfg['max_iter'], step=0.01, H=cfg['H'], W=cfg['W'],
             cams=[cam_for(make_cam_intrinsics, cfg['W'] // d, cfg['H'] // d) for d in dw])
    return c


LBA_OPT_CASES = ['lbaopt_par_m01_v3_64x48', 'lbaopt_par_m11_v2_48x80', 'lbaopt_par_m10_v3_64x64', 'lbaopt_seq_m01_v2_32x64',
                 'lbaopt_seq_m11_v2_48x64', 'lbaopt_seq_m10_v1_48x48', 'lbaopt_par_m01_v4_256x384']


