"""Pin the oracle against the committed reference outputs (CPU only, no GPU).

tests/golden/reference_outputs.npz was produced by the UNMODIFIED reference
(tests/golden/make_golden.py). Tolerances: geometry ops 1e-4 on costs/log-DPV (the
measured deviation is <=5e-5, tests/golden/PINNING.json), resample bit-exact,
pipeline outputs on PROBABILITIES (see DESIGN.md 'tolerance domain').
"""
import math

import numpy as np
import pytest

from oracle import planesweep_oracle as O
from oracle import kvnet_oracle as N
from tests import cases, harness
from tests.conftest import maxabs


@pytest.mark.parametrize('name', cases.SWEEP_CASES)
def test_sweep_cost_matches_reference(golden, name):
    c = cases.sweep_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    cost = O.est_swp_volume_v4(c['ref'], c['src'], c['d'], c['R'], c['t'], cam, c['sigma'], c['feat_dist'])
    ref = golden['sweep/%s/cost' % name]
    assert maxabs(cases.subsample(cost), ref) <= 1e-4
    st = cases.stats(cost); rs = golden['sweep/%s/cost_stats' % name]
    assert st[2] == rs[2] and abs(st[0] - rs[0]) <= 1e-6 * max(1.0, abs(rs[0]))
    bv = O.d_net_dpv_from_cost(cases.subsample(cost)); bvr = O.d_net_dpv_from_cost(ref)
    assert maxabs(bv, bvr) <= 1e-4


def test_sweep_identity_is_zero_cost():
    c = cases.sweep_case('identity_v1_d8_c16')
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    cost = O.est_swp_volume_v4(c['ref'], c['src'], c['d'], c['R'], c['t'], cam, c['sigma'])
    assert cost.max() <= 1e-9          # SURVEY §8(c) pin (i): identity pose => cost ~ 0


def test_sweep_bad_metric_raises():
    c = cases.sweep_case('ragged_v3_d7_c5')
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    with pytest.raises(Exception, match='undefined metric'):
        O.est_swp_volume_v4(c['ref'], c['src'], c['d'], c['R'], c['t'], cam, c['sigma'], 'L3')


@pytest.mark.parametrize('name', cases.WARP_CASES)
def test_warp_matches_reference(golden, name):
    c = cases.warp_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    vol = np.stack(O.warp_img_feats_v3(c['imgs'], c['d'], c['R'], c['t'], cam))
    assert maxabs(cases.subsample(vol), golden['warp/%s/vol' % name]) <= 2e-5
    mg = np.stack(O.warp_img_feats_mgpu(c['imgs'], c['d'], c['R'], c['t'], cam['intrinsic_M_cuda'][None],
                                        cam['unit_ray_array_2D'][None]))
    assert maxabs(mg, vol) == 0.0


@pytest.mark.parametrize('name', cases.RESAMPLE_CASES)
def test_resample_matches_reference(golden, name):
    c = cases.resample_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['w'], c['h'])
    out = O.resample_vol_cuda(c['vol'], c['rel'], cam, c['d'], d_candi_new=c['d_new'], padding_value=c['pad'])
    assert maxabs(cases.subsample(out), golden['resample/%s/vol' % name]) <= 1e-5
    if name == 'resample_identity_d16':
        # SURVEY §8(c) pin (vi): identity pose is NOT identity under align_corners=False
        assert maxabs(out, c['vol'][0]) > 1.0


def test_depth_regression_matches_reference(golden):
    c = cases.resample_case('resample_pose_d32')
    dep = O.depth_val_regression(c['vol'], c['d'])
    assert maxabs(dep, golden['regress/resample_pose_d32/depth']) <= 1e-5


def test_valid_dpv_sentinel():
    assert not O.valid_dpv(None)
    a = np.zeros((1, 4, 3, 3), np.float32)
    assert O.valid_dpv(a)
    a[0, 0, 0, 0] = np.nan
    assert not O.valid_dpv(a)


def test_kvnet_first_window_matches_reference(golden):
    """Full KVNET.forward, first-window branch (D-Net + R-Net), smallest legal frame.
    The streaming / K-Net steps are pinned by make_golden.py (PINNING.json) and
    re-run against the CUDA path in the gpu tests; running them here too would push
    the CPU suite past a few minutes."""
    name = 'kvnet_256x320_d8'
    c = cases.kvnet_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    ref_f, src_f, poses = cases.window(c, 2)
    o = N.kvnet_forward(c['sd'], ref_f, src_f, poses, cam, c['d'], c['sigma'])
    key = 'kvnet/%s/step0' % name
    for nm, a in zip(['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV'], o):
        r = golden['%s/%s' % (key, nm)]
        assert maxabs(np.exp(cases.subsample(a)), np.exp(r)) <= 1e-4, nm
    dep = O.depth_val_regression(o[3], c['d'])
    assert np.isfinite(dep).all()


def test_pinning_record_within_bounds():
    """The deviations measured when the fixtures were generated stay inside the
    documented envelope (DESIGN.md)."""
    pin = harness.pinning('PINNING.json')
    for k, v in pin.items():
        if k.startswith('sweep/'):
            assert v['logdpv_maxabs'] <= 1e-4 and v['prob_maxabs'] <= 1e-5
        elif k.startswith('warp/'):
            assert v['maxabs'] <= 2e-5 and v['mgpu_vs_v3'] == 0.0
        elif k.startswith('resample/'):
            assert v['maxabs'] <= 1e-5
        elif k.startswith('kvnet/') and isinstance(v, dict):
            assert v['BV_cur_prob'] <= 1e-4 and v['dmap_cur_refined_prob'] <= 1e-4
            assert v['DPV_prob'] <= 5e-4 and v['depth_mm'] <= 1.0


def test_torch_port_reproduces_reference(golden):
    """oracle/torch_port.py (the timed CPU arm of bench.py) uses the same ATen ops as the
    reference: its first-window outputs must equal the recorded reference outputs exactly."""
    from oracle import torch_port as TP
    name = 'kvnet_256x320_d8'
    c = cases.kvnet_case(name)
    cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    ref_f, src_f, poses = cases.window(c, 2)
    r, bv, dep = TP.kvnet_first_window(c['sd'], ref_f, src_f, poses, cam, c['d'], c['sigma'])
    assert maxabs(cases.subsample(bv), golden['kvnet/%s/step0/BV_cur' % name]) <= 1e-6
    assert maxabs(cases.subsample(r), golden['kvnet/%s/step0/dmap_cur_refined' % name]) <= 1e-6
