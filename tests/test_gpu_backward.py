"""f-1 on the device: autograd through the est_swp_volume_v4 mirror against torch autograd through the reference
(golden), the oracle, and directional-derivative / linearity properties at the BASELINE sweep shape."""
import numpy as np
import pytest
import torch

from oracle import planesweep_oracle as O
from tests import cases, harness

pytestmark = pytest.mark.gpu
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731


gold = harness.golden_fixture('sweep_backward.npz')


def _cam(w, h):
    from neuralrgbd_b200 import camera
    return cases.cam_for(camera.make_cam_intrinsics, w, h)


@pytest.mark.parametrize('name', cases.SWEEP_BACKWARD_CASES)
def test_sweep_backward_vs_reference_autograd(gold, name):
    from neuralrgbd_b200.warping import homography as H
    c = cases.sweep_case(name)
    cam = _cam(c['w'], c['h'])
    ref = T(c['ref']).requires_grad_(True)
    src = T(c['src']).requires_grad_(True)
    cost = H.est_swp_volume_v4(ref, src, c['d'], T(c['R']), T(c['t']), cam, c['sigma'], feat_dist=c['feat_dist'])
    g = cases.sweep_grad(name, tuple(cost.shape))
    cost.backward(T(g))
    for mine, key in ((ref.grad, '/g_ref'), (src.grad, '/g_src')):
        want = gold[name + key]
        assert tuple(mine.shape) == want.shape
        # fp32 scatter-add in hardware order vs autograd's: rounding of sums of up to D*V (*4 corners) terms
        assert np.abs(mine.cpu().numpy() - want).max() <= 2e-5 * np.abs(want).max()
    # the forward value is unchanged by the autograd path
    with torch.no_grad():
        plain = H.est_swp_volume_v4(ref.detach(), src.detach(), c['d'], T(c['R']), T(c['t']), cam, c['sigma'], feat_dist=c['feat_dist'])
    assert torch.equal(plain, cost.detach())
    # oracle (float64 accumulation)
    o_ref, o_src = O.est_swp_volume_v4_backward(g, c['ref'], c['src'], c['d'], c['R'], c['t'],
                                                cases.cam_for(O.make_cam_intrinsics, c['w'], c['h']), c['sigma'], c['feat_dist'])
    assert np.abs(ref.grad.cpu().numpy() - o_ref).max() <= 2e-5 * np.abs(o_ref).max()
    assert np.abs(src.grad.cpu().numpy() - o_src).max() <= 2e-5 * np.abs(o_src).max()


def test_sweep_backward_properties_at_metric_shape():
    """120x160, D=64, V=4, C=67 (the in-network sweep of the 640x480 workload): the L2 cost is quadratic in the features,
    so a central difference along a random direction equals <grad, direction> up to rounding; the backward is linear in
    the upstream gradient; zero upstream gradient gives exactly zero."""
    from neuralrgbd_b200.warping import homography as H
    h, w, D, V, C = 120, 160, 64, 4, 67
    cam = _cam(w, h)
    rng = np.random.RandomState(5)
    ref0, src0 = cases._feat_pair(rng, C, h, w, V)
    poses = cases._poses(rng, V)
    R, t = T(poses[:, :3, :3]), T(poses[:, :3, 3])
    d = np.linspace(0.1, 5.0, D)
    gen = torch.Generator(device='cuda').manual_seed(9)
    g1 = torch.randn((1, D, h, w), device='cuda', generator=gen)
    g2 = torch.randn((1, D, h, w), device='cuda', generator=gen)

    def grads(g):
        ref = T(ref0).requires_grad_(True); src = T(src0).requires_grad_(True)
        H.est_swp_volume_v4(ref, src, d, R, t, cam, 10.0).backward(g)
        return ref.grad, src.grad

    gr1, gs1 = grads(g1)
    gr2, gs2 = grads(g2)
    gr3, gs3 = grads(0.5 * g1 + g2)
    for a, b in ((gr3, 0.5 * gr1 + gr2), (gs3, 0.5 * gs1 + gs2)):
        assert float((a - b).abs().max()) <= 2e-5 * float(b.abs().max())
    z_ref, z_src = grads(torch.zeros_like(g1))
    assert float(z_ref.abs().max()) == 0.0 and float(z_src.abs().max()) == 0.0
    # directional derivative (float64 reduction of the fp32 costs)
    dr = torch.randn(ref0.shape, device='cuda', generator=gen)
    ds = torch.randn(src0.shape, device='cuda', generator=gen)
    eps = 0.25
    with torch.no_grad():
        cp = H.est_swp_volume_v4(T(ref0) + eps * dr, T(src0) + eps * ds, d, R, t, cam, 10.0)
        cm = H.est_swp_volume_v4(T(ref0) - eps * dr, T(src0) - eps * ds, d, R, t, cam, 10.0)
    fd = float(((cp.double() - cm.double()) * g1.double()).sum() / (2 * eps))
    an = float((gr1.double() * dr.double()).sum() + (gs1.double() * ds.double()).sum())
    assert abs(fd - an) <= 2e-4 * max(abs(an), 1.0), (fd, an)
