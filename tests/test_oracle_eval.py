"""CPU checks of the eval-mode oracle (oracle/kvnet_oracle.py, training=False) against the eval fixtures of the unmodified
reference (tests/golden/make_golden.py eval), and of which layers eval mode touches."""
import numpy as np
import pytest

from oracle import kvnet_oracle as N
from oracle import planesweep_oracle as O
from tests import cases, harness
from tests.conftest import maxabs

NAME = 'kvnet_256_d16'
NAMES4 = ['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV']


def _sd(c, gold):
    sd = {k: np.asarray(v) for k, v in c['sd'].items()}
    pre = 'eval/%s/rs/' % NAME
    sd.update({k[len(pre):]: np.asarray(gold[k]) for k in gold.files if k.startswith(pre)})
    return sd


def test_fixture_holds_warmed_running_statistics():
    gold = harness.golden('eval_outputs.npz')
    rs = [k for k in gold.files if k.startswith('eval/%s/rs/' % NAME) and '/rs/d_net.' not in k]   # d_net.*: the same tensors
    assert len(rs) == 3 * 13
    for k in rs:
        if k.endswith('running_var'):
            v = gold[k]
            assert np.all(v > 0) and not np.allclose(v, 1.0), k          # produced by the reference, not He-init ones
        if k.endswith('num_batches_tracked'):
            assert int(gold[k]) > 0, k


@pytest.mark.parametrize('step', [0, 1])
def test_eval_oracle_vs_reference_fixture(step):
    gold = harness.golden('eval_outputs.npz')
    pin = harness.pinning('PINNING_eval.json')
    c = cases.kvnet_case(NAME)
    cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    ref_f, src_f, poses = cases.window(c, 2 + step)
    ref_gold = harness.golden('reference_outputs.npz')
    prior = ref_gold['kvnet/%s/step%d/BV_predict_next_full' % (NAME, step - 1)] if step else None      # as recorded
    o = N.kvnet_forward(_sd(c, gold), ref_f, src_f, poses, cam, c['d'], c['sigma'], BV_predict=prior, training=False)
    key = 'eval/%s/step%d' % (NAME, step)
    for nm, a in zip(NAMES4, o):
        if '%s/%s' % (key, nm) not in gold.files:          # first window: the filtered outputs equal the stored ones
            continue
        e = maxabs(np.exp(cases.subsample_to(a, 8000)), np.exp(gold['%s/%s' % (key, nm)]))
        floor = pin[key]['oracle_%s_prob_sub' % nm]
        assert e <= 2.0 * floor + 1e-6, (nm, e, floor)


def test_untracked_layers_keep_batch_statistics_in_eval_mode():
    """Only layers whose running_mean is in the state_dict change in eval mode: the feature CNN up to layer1 (no tracked
    layer) is bit-identical to train mode, layer2 (tracked downsample) is not; K-Net (all tracked) is not."""
    gold = harness.golden('eval_outputs.npz')
    c = cases.kvnet_case(NAME)
    P = N.Params(_sd(c, gold))
    pre = 'feature_extractor.feature_extraction'
    x = c['frames'][2][None].astype(np.float32)
    a = N._convbn(P, pre + '.firstconv.0', x, 2, 1, 1, True)
    b = N._convbn(P, pre + '.firstconv.0', x, 2, 1, 1, False)
    assert np.array_equal(a, b)
    l1_t = N._layer(P, pre + '.layer1', N.relu(a), 3, 1, 1, False, True)
    l1_e = N._layer(P, pre + '.layer1', N.relu(b), 3, 1, 1, False, False)
    assert np.array_equal(l1_t, l1_e)
    blk_t = N._basic_block(P, pre + '.layer2.1', l1_t[:, :, ::2, ::2].repeat(2, axis=1), 1, 1, 1, False, True)
    blk_e = N._basic_block(P, pre + '.layer2.1', l1_t[:, :, ::2, ::2].repeat(2, axis=1), 1, 1, 1, False, False)
    assert np.array_equal(blk_t, blk_e)                    # a block without a downsample: nothing tracked
    d_t = N._basic_block(P, pre + '.layer2.0', l1_t, 2, 1, 1, True, True)
    d_e = N._basic_block(P, pre + '.layer2.0', l1_t, 2, 1, 1, True, False)
    assert not np.array_equal(d_t, d_e)
    assert N.tracked(P, pre + '.layer2.0.downsample.1') and not N.tracked(P, pre + '.layer2.0.conv1.0.1')
    n_tracked = sum(1 for k in P.sd if k.endswith('.running_mean') and not k.startswith('d_net.'))
    assert n_tracked == 13
    # K-Net: eval mode reads the running buffers; without them every layer falls back to batch statistics
    rng = np.random.RandomState(0)
    vol = rng.standard_normal((1, 16, 4, 8, 8)).astype(np.float32)
    untracked = N.Params({k: v for k, v in P.sd.items() if '.running_' not in k})
    assert np.array_equal(N.kv_net(untracked, vol, training=False), N.kv_net(untracked, vol, training=True))
    assert not np.array_equal(N.kv_net(P, vol, training=False), N.kv_net(P, vol, training=True))
