"""CPU checks at temporal window radii other than 2: the numpy oracle against the fixtures of the unmodified reference
(tests/golden/make_golden.py twin) at r = 1 and 3, and KVNET(t_win_r=r)'s state_dict against the reference's for r = 1..4."""
import contextlib
import io
import json

import numpy as np
import pytest
import torch

from oracle import kvnet_oracle as N
from oracle import planesweep_oracle as O
from tests import cases, harness
from tests import cases_twin as CT
from tests.conftest import maxabs

NAMES4 = ['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV']


@pytest.mark.parametrize('r,cin', [(1, 10), (2, 16), (3, 22), (4, 28)])
def test_state_dict_matches_reference(r, cin):
    from neuralrgbd_b200.models.KVNET import KVNET
    gold = harness.golden('twin_outputs.npz')
    c = CT.twin_case('r1_256_d16')
    cam = CT.twin_cam(O.make_cam_intrinsics, c)
    with contextlib.redirect_stdout(io.StringIO()):
        m = KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=10.0, KVNet_feature_dim=64,
                  d_upsample_ratio_KV_net=None, t_win_r=r)
    sd = m.state_dict()
    assert list(sd.keys()) == list(gold['twin/sd/r%d/keys' % r])
    assert [list(v.shape) for v in sd.values()] == json.loads(str(gold['twin/sd/r%d/shapes' % r]))
    assert tuple(sd['kv_net.dres0.0.0.weight'].shape) == (64, cin, 3, 3, 3)
    assert sd['kv_net.dres0.0.0.weight'].dtype == torch.float32


@pytest.mark.parametrize('mode', ['train', 'eval'])
@pytest.mark.parametrize('step', [0, 1])
@pytest.mark.parametrize('name', ['r1_256_d16', 'r3_256_d16'])
def test_oracle_vs_reference_fixture(name, step, mode):
    gold = harness.golden('twin_outputs.npz')
    pin = harness.pinning('PINNING_twin.json')
    c = CT.twin_case(name)
    cam = CT.twin_cam(O.make_cam_intrinsics, c)
    sd = {k: np.asarray(v) for k, v in c['sd'].items()}
    if mode == 'eval':
        pre = 'twin/eval/%s/rs/' % name
        sd.update({k[len(pre):]: np.asarray(gold[k]) for k in gold.files if k.startswith(pre)})
    ref_f, src_f, poses = cases.window(c, c['t_win_r'] + step)
    assert src_f.shape[1] == 2 * c['t_win_r']
    o = N.kvnet_forward(sd, ref_f, src_f, poses, cam, c['d'], c['sigma'], BV_predict=CT.prior(name, step) if step else None,
                        training=mode == 'train')
    key = 'twin/%s/%s/step%d' % (mode, name, step)
    checked = 0
    for nm, a in zip(NAMES4, o):
        if '%s/%s' % (key, nm) not in gold.files:          # first window: the filtered outputs equal the stored ones
            continue
        e = maxabs(np.exp(cases.subsample_to(a, 8000)), np.exp(gold['%s/%s' % (key, nm)]))
        floor = pin[key]['oracle_%s_prob_sub' % nm]
        assert e <= 2.0 * floor + 1e-6, (nm, e, floor)
        checked += 1
    assert checked == 2
