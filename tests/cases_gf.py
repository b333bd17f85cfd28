"""Seeded cases for the models.GF mirrors (numpy only): GuidedFilter(r, eps) and BoxFilter(r) of the reference's
models/GF, as RefineNet_DGF (models/Refine.py:587-641) uses them and beyond: ragged sizes, the KVNET-DGF 480x640 shape,
flat guides, wider boxes, N = 2, three channels with and without a broadcast guide, and a larger eps.

Shared by tests/golden/make_golden.py gf (which runs the unmodified reference and torch autograd through it on them) and
the tests. Every input and every upstream gradient is regenerated from its seed; the fixtures hold outputs and gradients.
"""
import numpy as np

from neuralrgbd_b200 import synth
from tests import cases
from tests.cases_grad import upstream

GF_CFG = {
    'ragged_13x17': dict(seed=201, H=13, W=17),
    'ragged_37x53': dict(seed=202, H=37, W=53),
    # the KVNET(refineNet_name='DGF') shape: one-channel guide and depth at 480x640
    'textured_480x640': dict(seed=203, H=480, W=640),
    # a guide flat over whole regions (var_x = 0 there: A = cov / eps), a textured band and sharp edges between
    'flat_120x160': dict(seed=204, H=120, W=160, flat=True),
    'r2_60x80': dict(seed=205, H=60, W=80, r=2),
    'r4_60x80': dict(seed=206, H=60, W=80, r=4),
    'n2_48x64': dict(seed=207, H=48, W=64, N=2),
    # C_x = 1 broadcast over three channels of y, and C_x = C_y = 3
    'cx1_cy3_60x80': dict(seed=208, H=60, W=80, Cy=3),
    'c3_60x80': dict(seed=209, H=60, W=80, Cx=3, Cy=3),
    'eps1e-2_60x80': dict(seed=210, H=60, W=80, eps=1e-2),
}
CASES = list(GF_CFG)


def case(name):
    """-> dict(x [N,Cx,H,W], y [N,Cy,H,W], r, eps, g [N,Cy,H,W] (upstream gradient of the output), g_box (of BoxFilter(r)
    applied to y), ...) in float32."""
    cfg = GF_CFG[name]
    rng = np.random.RandomState(cfg['seed'])
    N, Cx, Cy, H, W = cfg.get('N', 1), cfg.get('Cx', 1), cfg.get('Cy', 1), cfg['H'], cfg['W']
    # the guide: RefineNet_DGF's 1x1-MLP features of the image, O(1) with texture; y: an upsampled depth map around 2.5
    x = np.stack([synth.smooth_image(rng, Cx, H, W) for _ in range(N)]).astype(np.float32)
    y = np.stack([2.5 + synth.smooth_image(rng, Cy, H, W, n_waves=6) for _ in range(N)]).astype(np.float32)
    if cfg.get('flat'):
        x[:] = 0
        x[:, :, :H // 2, :W // 3] = np.float32(0.3)
        x[:, :, :H // 2, W // 3:] = np.float32(-0.7)
        x[:, :, H // 2:, :] = np.float32(1.1)
        x[:, :, H // 2 + 8:H // 2 + 16, :] += (0.5 * rng.standard_normal((N, Cx, 8, W))).astype(np.float32)
    return dict(x=x, y=y, r=cfg.get('r', 1), eps=cfg.get('eps', 1e-8), N=N, Cx=Cx, Cy=Cy, H=H, W=W,
                g=upstream(cfg['seed'] * 10, (N, Cy, H, W)), g_box=upstream(cfg['seed'] * 10 + 1, (N, Cy, H, W)))


SUB_LIMIT = 2500        # values per stored array (strided, cases.subsample_to)


def sub(a):
    return cases.subsample_to(a, SUB_LIMIT)
