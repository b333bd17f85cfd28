"""GPU parity of the geometry kernels (SURVEY §8 a1-a3, a7, a9, a11, a12) through the
reference-named Python surface -> C ABI -> sm_90a kernels, against (i) the numpy oracle on the
same seeded inputs and (ii) the committed outputs of the live reference.

Tolerances (float32 path; see DESIGN.md 'tolerance domain'):
  cost / log-DPV of the sweep vs oracle   1e-4   (coordinates are bit-identical by construction,
                                                   the residual is channel-summation order)
  image warp vs oracle                     2e-5
  resample vs oracle                       1e-5   (same arithmetic order -> expected exact)
  everything vs the reference fixtures     same bounds as the oracle-vs-reference record
"""
import math

import numpy as np
import pytest
import torch

from oracle import planesweep_oracle as O
from tests import cases
from tests.conftest import maxabs

pytestmark = pytest.mark.gpu

dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731


def cam_torch(cam):
    c = dict(cam)
    c['unit_ray_array_2D'] = torch.from_numpy(cam['unit_ray_array_2D'])
    c['intrinsic_M_cuda'] = torch.from_numpy(cam['intrinsic_M_cuda'])
    return c


@pytest.fixture(scope='module')
def H():
    import neuralrgbd_b200.warping.homography as h
    return h


@pytest.mark.parametrize('name', cases.SWEEP_CASES)
def test_sweep_vs_oracle_and_reference(H, golden, name):
    c = cases.sweep_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    got = H.est_swp_volume_v4(T(c['ref']), T(c['src']), c['d'], T(c['R']), T(c['t']), cam_torch(cam), c['sigma'],
                              feat_dist=c['feat_dist'])
    assert got.shape == (1, len(c['d']), c['h'], c['w']) and got.dtype == torch.float32 and got.is_cuda
    got = got.cpu().numpy()
    ref = golden['sweep/%s/cost' % name]
    assert maxabs(cases.subsample(got), ref) <= 1e-4
    if c['h'] * c['w'] <= 80 * 64:        # oracle finishes in seconds
        orc = O.est_swp_volume_v4(c['ref'], c['src'], c['d'], c['R'], c['t'], cam, c['sigma'], c['feat_dist'])
        assert maxabs(got, orc) <= 1e-4
        assert maxabs(O.d_net_dpv_from_cost(got), O.d_net_dpv_from_cost(orc)) <= 1e-4
    st = cases.stats(got); rs = golden['sweep/%s/cost_stats' % name]
    assert st[2] == rs[2] and abs(st[0] - rs[0]) <= 1e-6 * max(1.0, abs(rs[0]))


def test_sweep_bad_metric_raises(H):
    c = cases.sweep_case('ragged_v3_d7_c5')
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    with pytest.raises(Exception, match='undefined metric'):
        H.est_swp_volume_v4(T(c['ref']), T(c['src']), c['d'], T(c['R']), T(c['t']), cam_torch(cam), 10., 'L3')


def test_sweep_inputs_not_mutated_and_noncontiguous_poses(H):
    c = cases.sweep_case('small_v4_d32_c67_L2')
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    poses = np.tile(np.eye(4, dtype=np.float32), (4, 1, 1)); poses[:, :3, :3] = c['R']; poses[:, :3, 3] = c['t']
    P = T(poses[None])
    ref, src = T(c['ref']), T(c['src'])
    ref0, src0 = ref.clone(), src.clone()
    a = H.est_swp_volume_v4(ref, src, c['d'], P[0, :, :3, :3], P[0, :, :3, 3], cam_torch(cam), c['sigma'])
    b = H.est_swp_volume_v4(ref, src, c['d'], T(c['R']), T(c['t']), cam_torch(cam), c['sigma'])
    assert torch.equal(a, b) and torch.equal(ref, ref0) and torch.equal(src, src0)


def test_sweep_full_size_properties(H):
    """BASELINE metric shape (quarter-res 160x120, C=67, V=4, D=64): size-independent properties.
    identity pose + src==ref => cost ~ 0 (SURVEY §8c pin i); probabilities sum to 1; a pure x
    translation moves the minimum-cost plane monotonically with depth (pin ii)."""
    h, w, C, V, D = 120, 160, 67, 4, 64
    rng = np.random.RandomState(5)
    cam = cases.cam_for(O.make_cam_intrinsics, w, h)
    from neuralrgbd_b200 import synth, dpv
    ref = synth.smooth_image(rng, C, h, w)[None]
    src = np.repeat(ref[:, None], V, axis=1)
    d = synth.d_candidates(D)
    R = np.tile(np.eye(3, dtype=np.float32), (V, 1, 1)); t = np.zeros((V, 3), np.float32)
    c0 = H.est_swp_volume_v4(T(ref), T(src), d, T(R), T(t), cam_torch(cam), 10.)
    assert float(c0.max()) <= 1e-8
    # translated views of a fronto-parallel plane at depth d[k]: src_v(u) = ref(u - fx*tx_v/d_k)
    k = 20
    fx = cam['intrinsic_M'][0, 0]
    txs = np.array([-0.06, -0.03, 0.03, 0.06], np.float32)
    t2 = np.zeros((V, 3), np.float32); t2[:, 0] = txs
    big = synth.smooth_image(rng, C, h, w + 64)
    ref2 = big[:, :, 32:32 + w][None]
    srcs = []
    for tx in txs:
        shift = fx * tx / d[k]                       # u_src = u_ref + fx*tx/d
        x = np.arange(w) + 32 - shift                # src(u) = ref(u - shift)
        x0 = np.floor(x).astype(int); fr = (x - x0).astype(np.float32)
        srcs.append(big[:, :, x0] * (1 - fr) + big[:, :, x0 + 1] * fr)
    src2 = np.stack(srcs)[None].astype(np.float32)
    c2 = H.est_swp_volume_v4(T(ref2), T(src2), d, T(R), T(t2), cam_torch(cam), 10.)
    bv = dpv.log_softmax_planes(c2, sign=-1.0)
    p = bv.exp()
    assert float((p.sum(1) - 1).abs().max()) <= 1e-5
    inner = bv[0, :, 8:-8, 24:-24].argmax(0)
    assert float((inner == k).float().mean()) > 0.95


@pytest.mark.parametrize('name', cases.WARP_CASES)
def test_warp_vs_oracle_and_reference(H, golden, name):
    c = cases.warp_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    got = H.warp_img_feats_v3([T(i) for i in c['imgs']], c['d'], [T(r) for r in c['R']], [T(t) for t in c['t']],
                              cam_torch(cam))
    assert isinstance(got, list) and len(got) == len(c['imgs'])
    assert got[0].shape == (3, len(c['d']), c['h'], c['w'])
    got = np.stack([g.cpu().numpy() for g in got])
    orc = np.stack(O.warp_img_feats_v3(c['imgs'], c['d'], c['R'], c['t'], cam))
    assert maxabs(got, orc) <= 2e-5
    assert maxabs(cases.subsample(got), golden['warp/%s/vol' % name]) <= 2e-5
    mg = H.warp_img_feats_mgpu([T(i) for i in c['imgs']], c['d'], [T(r) for r in c['R']], [T(t) for t in c['t']],
                               T(cam['intrinsic_M_cuda'])[None], T(cam['unit_ray_array_2D'])[None])
    assert maxabs(np.stack([g.cpu().numpy() for g in mg]), got) == 0.0


def test_warp_tensor_branch_and_wide_channels(H):
    """Non-list branch (homography.py:264-278) and C > 4 (chunked)."""
    c = cases.warp_case('warp_v2_d5_ragged')
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    rng = np.random.RandomState(9)
    from neuralrgbd_b200 import synth
    img = synth.smooth_image(rng, 6, c['h'], c['w'])[None]
    got = H.warp_img_feats_v3(T(img), c['d'], T(c['R'][0]), T(c['t'][0]), cam_torch(cam))
    assert got.shape == (6, len(c['d']), c['h'], c['w'])
    orc = O.warp_img_feats_v3([img], c['d'], [c['R'][0]], [c['t'][0]], cam)[0]
    assert maxabs(got.cpu().numpy(), orc) <= 2e-5


@pytest.mark.parametrize('name', cases.RESAMPLE_CASES)
def test_resample_vs_oracle_and_reference(H, golden, name):
    c = cases.resample_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    got = H.resample_vol_cuda(T(c['vol']), T(c['rel']), cam_torch(cam), c['d'], d_candi_new=c['d_new'],
                              padding_value=c['pad'])
    assert got.shape == c['vol'].shape[1:]
    got = got.cpu().numpy()
    orc = O.resample_vol_cuda(c['vol'], c['rel'], cam, c['d'], d_candi_new=c['d_new'], padding_value=c['pad'])
    assert maxabs(got, orc) <= 1e-5
    assert maxabs(cases.subsample(got), golden['resample/%s/vol' % name]) <= 1e-5
    clamped = H.resample_vol_cuda(T(c['vol']), T(c['rel']), cam_torch(cam), c['d'], d_candi_new=c['d_new'],
                                  padding_value=c['pad'], clamp=(-1000., 0.)).cpu().numpy()
    assert maxabs(clamped, np.clip(got, -1000., 0.)) == 0.0


def test_depth_regression_and_sentinel(golden):
    from neuralrgbd_b200.mutils import misc
    c = cases.resample_case('resample_pose_d32')
    dep, conf = misc.depth_val_regression(T(c['vol']), c['d'], BV_log=True, return_conf=True)
    assert dep.shape == (1, c['h'], c['w'])
    assert maxabs(dep.cpu().numpy(), golden['regress/resample_pose_d32/depth']) <= 1e-5
    assert maxabs(dep.cpu().numpy(), O.depth_val_regression(c['vol'], c['d'])) <= 2e-6
    assert maxabs(conf.cpu().numpy()[0], np.exp(c['vol'][0]).max(0)) <= 1e-6
    assert misc.valid_dpv(T(c['vol'])) and not misc.valid_dpv(None)
    bad = T(c['vol']).clone(); bad[0, 0, 0, 0] = float('nan')
    assert not misc.valid_dpv(bad)


def test_bayes_update_vs_oracle():
    from neuralrgbd_b200 import dpv
    c = cases.resample_case('resample_pose_d32')
    rng = np.random.RandomState(3)
    gain = (2.0 * rng.standard_normal((1, 1) + c['vol'].shape[1:])).astype(np.float32)
    got, dep, conf = dpv.log_softmax_planes(T(gain[:, 0]), sign=1.0, add=T(c['vol']), d_candi=c['d'])
    orc = O.bayes_update(gain, c['vol'])
    assert maxabs(got.cpu().numpy(), orc) <= 2e-6
    assert maxabs(dep.cpu().numpy(), O.depth_val_regression(orc, c['d'])) <= 5e-6
    assert float((got.exp().sum(1) - 1).abs().max()) <= 1e-5
