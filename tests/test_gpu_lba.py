"""GPU parity of the LBA depth-map back-warp and its gradients (SURVEY 8 f-3): warping.homography.back_warp_th_Rt(_msrc)
mirrors against (i) the outputs of the unmodified reference and of torch autograd through it (tests/golden/lba_outputs.npz,
tests/golden/make_golden_lba.py) and (ii) the numpy oracle; plus the optimiser-facing behaviour: autograd through the mirror
gives the pose gradients ICP/opt_pose_numerical.py:99-160 steps on, and a few Adam steps reduce a photometric loss."""
import numpy as np
import pytest
import torch

from oracle import planesweep_oracle as O
from tests import cases, harness
from tests.conftest import maxabs

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731


gold = harness.golden_fixture('lba_outputs.npz')


@pytest.mark.parametrize('name', cases.LBA_CASES)
def test_back_warp_forward_vs_reference_and_oracle(gold, name):
    import neuralrgbd_b200.warping.homography as H
    c = cases.lba_case(name)
    cam_np = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    cam = harness.cam_tensors(cam_np)
    out = H.back_warp_th_Rt_msrc(T(c['imgs']), T(c['dmap']), T(c['Rs']), T(c['ts']), cam).cpu().numpy()
    assert out.shape == gold[name + '/warp_msrc'].shape
    assert maxabs(out, gold[name + '/warp_msrc']) <= 2e-5                      # the live reference
    assert maxabs(out, O.back_warp_th_Rt_msrc(c['imgs'], c['dmap'], c['Rs'], c['ts'], cam_np)) <= 2e-5
    one = H.back_warp_th_Rt(T(c['imgs'][:1]), T(c['dmap']), T(c['Rs'][0]), T(c['ts'][0]), cam).cpu().numpy()
    assert maxabs(one, out[:1]) == 0.0                                         # single-view entry = view 0 of the multi-view one


@pytest.mark.parametrize('name', cases.LBA_CASES)
def test_back_warp_gradients_vs_reference_autograd(gold, name):
    import neuralrgbd_b200.warping.homography as H
    c = cases.lba_case(name)
    cam = harness.cam_tensors(cases.cam_for(O.make_cam_intrinsics, c['w'], c['h']))
    img = T(c['imgs'][:1]).requires_grad_(True)
    R = T(c['Rs'][0]).requires_grad_(True)
    t = T(c['ts'][0]).requires_grad_(True)
    out = H.back_warp_th_Rt(img, T(c['dmap']), R, t, cam)
    out.backward(T(gold[name + '/grad_out']))
    gR, gt, gi = R.grad.cpu().numpy(), t.grad.cpu().numpy(), img.grad.cpu().numpy()
    # fixtures: torch autograd through the unmodified reference (float32 sums there, double block sums here)
    assert maxabs(gR, gold[name + '/g_R']) <= 2e-4 * np.abs(gold[name + '/g_R']).max()
    assert maxabs(gt, gold[name + '/g_t']) <= 2e-4 * np.abs(gold[name + '/g_t']).max()
    assert maxabs(gi, gold[name + '/g_img']) <= 2e-5


def test_pose_refinement_step_reduces_the_photometric_loss():
    """A miniature of ICP/opt_pose_numerical.py:99-160: Adam on (R via a small-angle update, t) through the mirror."""
    import neuralrgbd_b200.warping.homography as H
    c = cases.lba_case('lba_v3_c3_48x64')
    cam_np = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    cam = harness.cam_tensors(cam_np)
    rng = np.random.RandomState(3)
    from neuralrgbd_b200 import synth
    src = synth.smooth_image(rng, 3, c['h'], c['w'])[None]
    R_true, t_true = c['Rs'][0], c['ts'][0]
    target = T(O.back_warp_th_Rt(src, c['dmap'], R_true, t_true, cam_np))          # what the true pose sees
    t = (T(t_true) + torch.tensor([0.02, -0.015, 0.01], device=dev)).requires_grad_(True)
    R = T(R_true).clone().requires_grad_(True)
    opt = torch.optim.Adam([t, R], lr=2e-3)
    losses = []
    for _ in range(40):
        opt.zero_grad()
        warped = H.back_warp_th_Rt(T(src), T(c['dmap']), R, t, cam)
        mask = (warped != 0).float()
        loss = torch.nn.functional.l1_loss(warped * mask, target * mask)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < 0.6 * losses[0], losses[::8]
