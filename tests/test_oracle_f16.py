"""conv_math='f16' fixtures and oracle on the CPU (tests/golden/make_golden.py f16, tests/oracle_f16.py).

 * The convolutions whose operands the fixtures round are exactly the ones the engine runs on tensor cores: every
   convolution of the architecture except the 3-input-channel first layer (from arch.kvnet_param_specs).
 * The f16 oracle reproduces its pinned deviation from the f16-emulated reference on the stored samples of the 256x256
   first windows (train, .eval() and t_win_r = 1).
 * The pinned deviations are consistent: the TF32- and f16-emulated references both differ from fp32 by more than the
   f16 oracle does from its reference on first-window probabilities.
"""
import numpy as np
import pytest

from neuralrgbd_b200 import arch
from oracle import planesweep_oracle as O
from tests import cases, harness
from tests import cases_f16 as CF
from tests import oracle_f16 as OF
from tests.conftest import maxabs


def test_hooked_layers_are_the_engine_tensor_core_layers():
    specs = arch.kvnet_param_specs(64, 16, 2, 64, 'DPV', False)
    hooked = sorted(harness.golden('f16_outputs.npz')['f16/hooked_layers'].tolist())
    tc = CF.tc_layers(specs)
    assert hooked == tc
    convs = [n for n, s, _ in specs if len(s) >= 4 and n.endswith('.weight') and not n.startswith('d_net.')]
    assert sorted(set(convs) - set(tc)) == ['feature_extractor.feature_extraction.firstconv.0.0.weight']


def test_round_tf32():
    x = np.array([1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, -3.0 + 2 ** -12, 0.0, 65504.0], np.float32)
    r = CF.round_tf32(x)
    assert r.tolist() == [1.0, 1.0 + 2 ** -10, 1.0, 1.0 + 2 ** -9, -3.0, 0.0, 65504.0]


@pytest.mark.parametrize('name', ['stream_256_d16', 'eval_256_d16', 'r1_256_d16'])
def test_oracle_f16_first_window_matches_fixture(name):
    gold, pin = harness.golden('f16_outputs.npz'), harness.pinning('PINNING_f16.json')
    c = CF.f16_case(name)
    cam = CF.cam(O.make_cam_intrinsics, c)
    ref_f, src_f, poses = cases.window(c, c['t_win_r'])
    o = OF.kvnet_forward(CF.state_dict(c), ref_f, src_f, poses, cam, c['d'], c['sigma'], training=CF.MODE[name] == 'train')
    kk = 'f16/%s/step0' % name
    for nm in CF.STORED[True]:
        a = np.exp(cases.subsample_to(o[CF.NAMES4.index(nm)], CF.SUB_LIMIT))
        d = maxabs(a, np.exp(gold['%s/f16/%s' % (kk, nm)]))
        assert d <= pin[kk]['oracle_vs_f16'][nm]['prob'] + 1e-7, (nm, d)


def test_pinned_deviations_are_consistent():
    pin = harness.pinning('PINNING_f16.json')
    for name in CF.F16_CASES:
        p = pin['f16/%s/step0' % name]
        for nm in ('BV_cur', 'dmap_cur_refined'):
            assert p['oracle_vs_f16'][nm]['prob'] < p['f16_vs_fp32'][nm]['prob'], (name, nm)
            assert p['oracle_vs_f16'][nm]['prob'] < p['tf32_vs_fp32'][nm]['prob'], (name, nm)
