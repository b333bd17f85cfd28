"""f-3, oracle first: the numpy restatement of the LBA depth-map back-warp and of its pose / image gradients against the
unmodified reference (forward) and torch autograd through it (backward): tests/golden/lba_outputs.npz. The device
kernels for this row are not built yet (DESIGN.md 7); this pins the checker they will be tested against."""
import numpy as np
import pytest

from oracle import planesweep_oracle as O
from tests import cases, harness


gold = harness.golden_fixture('lba_outputs.npz')


@pytest.mark.parametrize('name', cases.LBA_CASES)
def test_lba_warp_and_gradients(gold, name):
    c = cases.lba_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    warped = O.back_warp_th_Rt_msrc(c['imgs'], c['dmap'], c['Rs'], c['ts'], cam)
    assert warped.shape == gold[name + '/warp_msrc'].shape
    assert np.abs(warped - gold[name + '/warp_msrc']).max() <= 2e-5
    gR, gt, gi = O.back_warp_th_Rt_backward(gold[name + '/grad_out'], c['imgs'][:1], c['dmap'], c['Rs'][0], c['ts'][0], cam)
    assert np.abs(gR - gold[name + '/g_R']).max() <= 5e-6 * np.abs(gold[name + '/g_R']).max()
    assert np.abs(gt - gold[name + '/g_t']).max() <= 5e-6 * np.abs(gold[name + '/g_t']).max()
    assert np.abs(gi - gold[name + '/g_img']).max() <= 2e-5


def test_lba_identity_pose_is_identity_warp():
    c = cases.lba_case('lba_v1_c5_37x53')
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    out = O.back_warp_th_Rt(c['imgs'][:1], c['dmap'], np.eye(3, dtype=np.float32), np.zeros(3, np.float32), cam)
    # rays are at pixel centres (+0.5) and grid_sample(align_corners=False) samples centres: the warp reproduces the image
    assert np.abs(out - c['imgs'][:1]).max() <= 2e-4
