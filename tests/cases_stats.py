"""Seeded cases for the DPV statistics mirrors (numpy only): mutils.misc.depth_var and mutils.misc.dpv_statistics.

Shared by tests/golden/make_golden.py stats (which runs the unmodified reference and torch autograd through it on them)
and the tests. Every input and every upstream gradient is regenerated from its seed; the fixtures hold outputs and
gradients only.
"""
import math

import numpy as np

from neuralrgbd_b200 import synth
from tests import cases
from tests.cases_grad import upstream

# the four statistics train_utils/train_KVNet.py:_loss_RNet_UNet2D asks for (:229)
ALL_STATS = ['E_mean', 'variance', 'max', 'min']

STATS_CFG = {
    # a sharp D-Net-like log-DPV at the 640x480 workload's quarter resolution (softmax of sigma-10 costs)
    'sharp_120x160_d64': dict(seed=111, h=120, w=160, D=64, N=1, sharp=12.0),
    # a propagated prior: the six faces of the volume set to log(1/D) as resample_vol_cuda's _set_vol_border does, so
    # every border pixel has D exactly equal planes (ties for max and min)
    'prior_pad_120x160_d64': dict(seed=112, h=120, w=160, D=64, N=1, sharp=3.0, pad=True),
    # probabilities, not log-probabilities (BV_log=False; 'min' then gives the max, misc.py:603)
    'lin_120x160_d64': dict(seed=113, h=120, w=160, D=64, N=1, sharp=3.0, log=False),
    # 1/D not exact in binary
    'd100_60x80': dict(seed=114, h=60, w=80, D=100, N=1, sharp=4.0),
    # d_sigma other than 1 (2 sigma^2 = 0.98 is rounded to fp32)
    'sigma07_120x160_d64': dict(seed=115, h=120, w=160, D=64, N=1, sharp=3.0, sigma=0.7),
    # N = 2: depth_var reads slice 0 only; 'max' / 'min' reduce every slice
    'n2_37x53_d16': dict(seed=116, h=37, w=53, D=16, N=2, sharp=3.0, stats=['max', 'min']),
    # depth_mean given as H x W instead of depth_val_regression's 1 x H x W
    'mean_hw_120x160_d64': dict(seed=117, h=120, w=160, D=64, N=1, sharp=3.0, mean_hw=True),
}
CASES = list(STATS_CFG)


def _log_dpv(rng, N, D, h, w, sharp):
    logits = sharp * np.stack([synth.smooth_image(rng, D, h, w) for _ in range(N)])
    m = logits.max(axis=1, keepdims=True)
    return (logits - m - np.log(np.exp(logits - m).sum(axis=1, keepdims=True))).astype(np.float32)


def case(name):
    """-> dict(bv [N,D,h,w], d, log, sigma, mean (1 x h x w, or h x w when mean_hw), stats, g_var (the shape of depth_var's output), g_stats
    (the shape of dpv_statistics' output), ...)."""
    cfg = STATS_CFG[name]
    rng = np.random.RandomState(cfg['seed'])
    N, D, h, w = cfg['N'], cfg['D'], cfg['h'], cfg['w']
    bv = _log_dpv(rng, N, D, h, w, cfg['sharp'])
    if cfg.get('pad'):
        pad = np.float32(math.log(1.0 / D))
        bv[:, 0] = bv[:, -1] = pad
        bv[:, :, 0] = bv[:, :, -1] = pad
        bv[:, :, :, 0] = bv[:, :, :, -1] = pad
    log = cfg.get('log', True)
    if not log:
        bv = np.exp(bv).astype(np.float32)
    stats = cfg.get('stats', ALL_STATS)
    mean_hw = cfg.get('mean_hw', False)
    # depth_mean: the expected depth of slice 0 (fp32, sequential over d, as depth_val_regression computes it)
    mean = np.zeros((1, h, w), np.float32)
    for i, dv in enumerate(synth.d_candidates(D).astype(np.float32)):
        mean = mean + (np.exp(bv[0, i]) if log else bv[0, i]) * dv
    n_out = N if all(s in ('max', 'min') for s in stats) else 1       # E_mean / variance have one slice
    return dict(bv=bv, d=synth.d_candidates(D), log=log, sigma=cfg.get('sigma', 1.0), mean_hw=mean_hw, stats=stats,
                mean=mean[0] if mean_hw else mean,
                N=N, D=D, h=h, w=w,
                g_var=upstream(cfg['seed'] * 10, (h, w) if mean_hw else (1, h, w)),
                g_stats=upstream(cfg['seed'] * 10 + 1, (n_out, len(stats), h, w)))


SUB_LIMIT = 2500        # values per stored array (strided, cases.subsample_to)


def sub(a):
    return cases.subsample_to(a, SUB_LIMIT)
