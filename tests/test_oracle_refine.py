"""KVNET's refinement configurations on the host: the guided-filter oracle (tests/oracle_refine.py) against the unmodified
reference's RefineNet_DGF (tests/golden/make_golden_refine.py), and the mirror's constructor surface - module tree,
state_dict keys / shapes / order, strict checkpoint loading and printed lines - for refineNet_name='DGF', if_refined=False
and the depth-upsampled DPV R-Net (if_upsample_d=True) against the reference's own lists."""
import contextlib
import io
import json

import numpy as np
import pytest
import torch

from neuralrgbd_b200 import arch
from tests import oracle_refine as R, harness

CONFIGS = {'DPV': dict(if_refined=True, refineNet_name='DPV'), 'DGF': dict(if_refined=True, refineNet_name='DGF'),
           'none': dict(if_refined=False), 'none_DGF': dict(if_refined=False, refineNet_name='DGF'),
           'DPV_upsample_d': dict(if_refined=True, refineNet_name='DPV', if_upsample_d=True)}
REFINE = {'DPV': 'DPV', 'DGF': 'DGF', 'none': None, 'none_DGF': None, 'DPV_upsample_d': 'DPV'}
UPSAMPLE = {'DPV_upsample_d': True}


def _model(D=16, **cfg):
    from neuralrgbd_b200.models.KVNET import KVNET
    from oracle import planesweep_oracle as O
    from tests import cases
    cam = cases.cam_for(O.make_cam_intrinsics, 64, 64)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        m = KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=np.linspace(0.1, 5.0, D), sigma_soft_max=10.0, KVNet_feature_dim=64,
                  d_upsample_ratio_KV_net=cfg.pop('d_upsample_ratio_KV_net', None), t_win_r=2, **cfg)
    return m, buf.getvalue().splitlines()


@pytest.mark.parametrize('name', R.GF_CASES)
def test_guided_filter_oracle_vs_reference(name):
    """RefineNet_DGF alone on seeded inputs; bit-exact wherever the fixture recorded it so."""
    g = R.gf_case(name)
    ref = harness.golden('refine_outputs.npz')['refine/gf/%s/out' % name]
    pin = harness.pinning('PINNING_refine.json')['gf/%s' % name]
    o = R.dgf_refine(g['dmap'], g['img'], g['sd'])
    if pin['oracle_bitexact']:
        assert np.array_equal(o, ref)
    else:
        assert np.abs(o.astype(np.float64) - ref).max() <= pin['oracle_m']


def test_box_filter_counts_are_the_analytic_window_sizes():
    H, W, r = 9, 7, 1
    N = R.box_filter(np.ones((H, W), np.float32), r)
    i, j = np.mgrid[0:H, 0:W]
    want = (np.minimum(i + r, H - 1) - np.maximum(i - r, 0) + 1) * (np.minimum(j + r, W - 1) - np.maximum(j - r, 0) + 1)
    assert np.array_equal(N, want.astype(np.float32))


@pytest.mark.parametrize('cfg', list(CONFIGS))
def test_state_dict_matches_reference(cfg):
    gold = harness.golden('refine_outputs.npz')
    m, printed = _model(**CONFIGS[cfg])
    sd = m.state_dict()
    assert list(sd.keys()) == list(gold['refine/sd/%s/keys' % cfg])
    assert [list(v.shape) for v in sd.values()] == json.loads(str(gold['refine/sd/%s/shapes' % cfg]))
    assert printed == list(gold['refine/sd/%s/printed' % cfg])
    assert [n for n, _, _ in arch.kvnet_param_specs(64, 16, 2, 64, REFINE[cfg], UPSAMPLE.get(cfg, False))] == list(sd.keys())


@pytest.mark.parametrize('cfg', ['DGF', 'none', 'DPV_upsample_d'])
@pytest.mark.parametrize('prefix', ['', 'module.'])
def test_reference_checkpoint_loads_strictly(cfg, prefix):
    sd = arch.synth_state_dict(3, 64, 16, 2, 64, refine=REFINE[cfg], upsample_d=UPSAMPLE.get(cfg, False))
    ckpt = {prefix + k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
    m, _ = _model(**CONFIGS[cfg])
    target = torch.nn.DataParallel(m) if prefix else m
    target.load_state_dict(ckpt, strict=True)
    for k, v in sd.items():
        assert np.array_equal(m.state_dict()[k].numpy(), np.asarray(v)), k
    # a checkpoint of another configuration does not load strictly
    other = arch.synth_state_dict(3, 64, 16, 2, 64, refine='DPV')
    with pytest.raises(RuntimeError):
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in other.items()}, strict=True)


def test_upsample_ratio_raises_and_upsample_d_only_widens_dpv():
    with pytest.raises(NotImplementedError, match='KVNET.py:172'):
        _model(d_upsample_ratio_KV_net=2)
    # if_upsample_d is ignored unless the configuration is DPV, as in the reference
    m, _ = _model(if_refined=True, refineNet_name='DGF', if_upsample_d=True)
    assert list(m.state_dict().keys()) == list(harness.golden('refine_outputs.npz')['refine/sd/DGF/keys'])
    m, _ = _model(if_refined=False, if_upsample_d=True)
    assert list(m.state_dict().keys()) == list(harness.golden('refine_outputs.npz')['refine/sd/none/keys'])
