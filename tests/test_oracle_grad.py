"""CPU checks of tests/oracle_grad.py, the numpy backward of the geometry mirrors (f-5):
 * against torch autograd through the unmodified reference (tests/golden/make_golden.py grad), at the pinned floor;
 * torch.autograd.gradcheck (float64 central differences) of each oracle backward against its float64 forward over the
   same taps, and the taps against the pinned fp32 forward of oracle/planesweep_oracle.py;
 * the properties the kernels rely on: the six faces of a resampled volume get zero gradient, the clamp mask is the one
   of torch.clamp's backward, and the regression's extra slices get zero."""
import numpy as np
import pytest
import torch

from oracle import planesweep_oracle as O
from tests import cases, cases_grad as CG, oracle_grad as OG, harness


gold = harness.golden_fixture('grad_outputs.npz')
pin = harness.pinning_fixture('PINNING_grad.json')


def _cam(w, h):
    return cases.cam_for(O.make_cam_intrinsics, w, h)


def _check(gold, pin, key, mine):
    p = pin[key]
    assert list(mine.shape) == p['shape']
    # the oracle is deterministic: it reproduces the deviation it was pinned at (float64 sums vs the reference's fp32)
    assert np.abs(CG.sub(mine).astype(np.float64) - gold[key + '/g']).max() <= p['maxabs_oracle']
    s, want = cases.summary(mine), gold[key + '/stats']
    assert s[2] == want[2] and abs(s[3] - want[3]) <= p['maxabs_oracle']
    assert abs(s[1] - want[1]) <= 1e-5 * want[1]
    assert abs(s[0] - want[0]) <= p['maxabs_oracle'] * want[2]


@pytest.mark.parametrize('name', [n for n in CG.WARP_CASES if '120x160' not in n or 'c3' in n])
def test_warp_backward_vs_reference(gold, pin, name):
    c = CG.warp_case(name)
    cam = _cam(c['w'], c['h'])
    if c['tensor']:
        g = OG.warp_img_feats_backward([c['grads']], c['d'], [c['R']], [c['t']], cam, c['h'], c['w'])[0]
    else:
        g = np.concatenate(OG.warp_img_feats_backward(c['grads'], c['d'], c['R'], c['t'], cam, c['h'], c['w']))
    _check(gold, pin, 'warp/' + name, g)


@pytest.mark.parametrize('name', [n for n in CG.RESAMPLE_CASES if 'img' not in n])
def test_resample_backward_vs_reference(gold, pin, name):
    c = CG.resample_case(name)
    g = OG.resample_vol_cuda_backward(c['grad'], c['vol'], c['rel'], _cam(c['w'], c['h']), c['d'], c['d_new'], c['pad'],
                                      c['clamp'])
    _check(gold, pin, 'resample/' + name, g)
    D, h, w = c['D'], c['h'], c['w']
    for face in (g[0, 0], g[0, -1], g[0, :, 0], g[0, :, -1], g[0, :, :, 0], g[0, :, :, -1]):
        assert not face.any()


@pytest.mark.parametrize('name', CG.REGRESSION_CASES)
def test_regression_backward_vs_reference(gold, pin, name):
    c = CG.regression_case(name)
    g = OG.depth_val_regression_backward(c['grad'], c['bv'], c['d'], c['log'])
    _check(gold, pin, 'regression/' + name, g)
    assert not g[1:].any()


def test_clamp_mask_is_exercised():
    """The clamp case cuts through the volume's values: a good share of voxels is masked and a good share passes."""
    c = CG.resample_case('rs_pose_clamp_q_d64')
    res = O.resample_vol_cuda(c['vol'], c['rel'], _cam(c['w'], c['h']), c['d'], c['d_new'], c['pad'])
    inside = ((res >= c['clamp'][0]) & (res <= c['clamp'][1])).mean()
    assert 0.2 < inside < 0.8, inside


# ---- gradcheck of the oracle backward (float64), small problems --------------------------------------------------
class _Op(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fwd, bwd):
        ctx.bwd, ctx.x = bwd, x.detach().numpy()
        return torch.from_numpy(np.asarray(fwd(ctx.x), np.float64))

    @staticmethod
    def backward(ctx, g):
        return torch.from_numpy(np.asarray(ctx.bwd(g.detach().numpy(), ctx.x), np.float64)), None, None


def _gradcheck(x0, fwd, bwd):
    x = torch.from_numpy(np.asarray(x0, np.float64)).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda t: _Op.apply(t, fwd, bwd), (x,), eps=1e-6, atol=1e-8, rtol=1e-6)


def test_gradcheck_warp():
    h, w, D, C, V = 6, 7, 3, 2, 2
    rng = np.random.RandomState(3)
    cam = _cam(w, h)
    poses = cases._poses(rng, V)
    R, t, d = poses[:, :3, :3], poses[:, :3, 3], np.linspace(0.5, 3.0, D)
    taps = OG.warp_taps(d, R, t, cam, h, w)
    imgs = rng.standard_normal((V, C, h * w))
    fwd = lambda x: np.stack(OG.warp_forward64(list(x), taps, D))                     # noqa: E731
    bwd = lambda g, x: np.stack(OG.warp_backward(list(g.reshape(V, C, D, -1)), taps, h * w))   # noqa: E731
    _gradcheck(imgs, fwd, bwd)
    # the taps are the pinned fp32 forward's
    want = O.warp_img_feats_v3([i.reshape(1, C, h, w).astype(np.float32) for i in imgs], d, R, t, cam)
    assert np.abs(np.stack(want).reshape(V, C, D, -1) - fwd(imgs)).max() <= 1e-5


@pytest.mark.parametrize('clamp', [None, (-2.5, -1.5)])
@pytest.mark.parametrize('d_new', [False, True])
def test_gradcheck_resample(clamp, d_new):
    h, w, D = 6, 7, 5
    rng = np.random.RandomState(4)
    cam = _cam(w, h)
    exts = cases.synth.camera_track(rng, 2, 0.05)
    rel = np.linalg.inv(exts[1].dot(np.linalg.inv(exts[0]))).astype(np.float32)
    d = np.linspace(0.5, 3.0, D)
    dn = np.linspace(0.6, 2.5, D) if d_new else None
    taps = OG.resample_taps(rel, cam, d, dn, D, h, w)
    pad = np.log(1.0 / D)
    vol = rng.uniform(-3.0, -1.0, D * h * w)
    res0 = OG.resample_forward64(vol, taps, pad)
    if clamp is not None:        # keep every voxel away from the clamp's kinks, where the finite difference is undefined
        near = (np.abs(res0 - clamp[0]) < 1e-3) | (np.abs(res0 - clamp[1]) < 1e-3)
        assert near.mean() < 0.05
        res0 = np.where(near, np.nan, res0)
    fwd = lambda x: OG.resample_forward64(x, taps, pad, clamp)                        # noqa: E731
    bwd = lambda g, x: OG.resample_backward(g, taps, D * h * w, OG.resample_forward64(x, taps, pad), clamp)   # noqa: E731
    if clamp is not None:
        keep = ~np.isnan(res0)
        fwd = (lambda f: lambda x: np.where(keep, f(x), 0.0))(fwd)
        bwd = (lambda b: lambda g, x: b(np.where(keep, g, 0.0), x))(bwd)
    _gradcheck(vol, fwd, bwd)
    want = O.resample_vol_cuda(vol.reshape(1, D, h, w).astype(np.float32), rel, cam, d, dn, pad).reshape(-1)
    assert np.abs(want - OG.resample_forward64(vol.astype(np.float32), taps, pad)).max() <= 1e-5


@pytest.mark.parametrize('log', [True, False])
def test_gradcheck_regression(log):
    rng = np.random.RandomState(5)
    D, h, w = 4, 3, 5
    bv = rng.uniform(-3.0, -0.5, (2, D, h, w))
    d = np.linspace(0.5, 3.0, D)
    fwd = lambda x: OG.depth_val_regression64(x, d, log)                              # noqa: E731
    bwd = lambda g, x: OG.depth_val_regression_backward(g, x, d, log).astype(np.float64)   # noqa: E731
    # the backward rounds to fp32 (as autograd through the reference does): compare at fp32 precision
    x = torch.from_numpy(bv).requires_grad_(True)
    y = _Op.apply(x, fwd, bwd)
    gy = torch.from_numpy(rng.standard_normal(y.shape))
    (ga,) = torch.autograd.grad(y, x, gy)
    num = np.zeros_like(bv)
    eps = 1e-6
    for i in range(bv.size):
        e = np.zeros(bv.size); e[i] = eps
        e = e.reshape(bv.shape)
        num.reshape(-1)[i] = ((fwd(bv + e) - fwd(bv - e)) * gy.numpy()).sum() / (2 * eps)
    assert np.abs(ga.numpy() - num).max() <= 1e-6 * np.abs(num).max()
