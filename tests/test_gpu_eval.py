"""Eval-mode KVNET on the GPU: running-statistics BatchNorm in the tensor-core convolution's epilogue.

 * Op level: nrgbd_conv_nhwc_h2_affine against the fp32 numpy oracle at the 6e-6 convolution gate of test_gpu_conv_h2.py
   (3-D k3 64 -> 64 with / without a pair residual and ReLU, pair output, both tile orientations; 2-D 1x1 stride 2 with
   fp32 output), bit-identical from run to run and under the schedule switches 8 / 32 (test_gpu_conv_sched.py).
 * Engine against the eval fixtures of tests/golden/make_golden_eval.py (unmodified reference, warmed running statistics),
   in all three conv_math modes: first window at 1e-4 on probabilities and 1 mm on depth; a steady K-Net step re-seeded with
   the reference's train-mode prior at train mode's gate for that step (C3: 1.5e-4 in f16x3, 5e-4 otherwise), and at twice
   the measured fp32-vs-fp32 floor of PINNING_eval.json at the 16-plane shape; every full array through the relative
   deviation of its sum of squared probabilities.
 * No buffer moves in eval mode; eval -> train -> eval on one engine; the reference's own test() on an .eval() model; and
   in f16x3 a steady eval step launches exactly 13 fewer BatchNorm-pass kernels than a steady train step.
Measured deviations are written to $NRGBD_PARITY_DIR/parity_eval.json when that variable is set.
"""
import json
import math

import numpy as np
import pytest
import torch

from oracle import kvnet_oracle as N
from oracle import planesweep_oracle as O
from tests import cases, harness
from tests import oracle_eval as E
from tests.conftest import maxabs
from tests.harness import NAMES4, T, rel_err

pytestmark = pytest.mark.gpu
SUB_LIMIT = 8000          # the fixture's strided samples (make_golden_eval.py)
TOL_SUMSQ_REL = 1e-4      # full-array check: relative deviation of the sum of squared probabilities
TOL_FIRST = 1e-4
TOL_DEPTH_MM = 1.0
TOL_KNET_F16 = 1.5e-4
TOL_KNET = 5e-4
MODES = ['f16x3', 'tf32x3', 'fp32']


def set_flags(flags):
    from neuralrgbd_b200 import _lib
    _lib.dev_lib().nrgbd_dev_conv_h2_set_flags(flags)


# ---- op level ----------------------------------------------------------------------------------------------------------
def _coeffs(rng, C):
    g = (1 + 0.5 * rng.standard_normal(C)).astype(np.float32)
    b = (0.5 * rng.standard_normal(C)).astype(np.float32)
    rm = (0.3 * rng.standard_normal(C)).astype(np.float32)
    rv = (0.5 + rng.rand(C)).astype(np.float32)
    return g, b, rm, rv


def _affine_ref(y, g, b, rm, rv, res, relu):
    out = E.batch_norm_eval(y, g, b, rm, rv)
    if res is not None:
        out = out + res
    return N.relu(out) if relu else out


@pytest.mark.parametrize('hw', [(40, 48), (48, 40)])         # 8 x 16 tiles pad fewer / 16 x 8 tiles pad fewer
@pytest.mark.parametrize('res,relu', [(False, True), (True, False), (True, True), (False, False)])
def test_affine_conv3d_pair_out_vs_oracle(hw, res, relu):
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(11 + 2 * res + relu)
    x = rng.standard_normal((1, 64, 5) + hw).astype(np.float32)
    w = (rng.standard_normal((64, 64, 3, 3, 3)) / math.sqrt(64 * 27)).astype(np.float32)
    g, b, rm, rv = _coeffs(rng, 64)
    r = rng.standard_normal((1, 64, 5) + hw).astype(np.float32) if res else None
    sc, sh = convops.bn_eval_coeffs(T(g), T(b), T(rm), T(rv))
    invstd = np.float32(1) / np.sqrt(rv + np.float32(1e-5))
    assert np.array_equal(sc.cpu().numpy(), (invstd * g).astype(np.float32))
    ref = _affine_ref(N.conv3d(x, w), g, b, rm, rv, r, relu)
    run = lambda: convops.conv_h2_affine(T(x), T(w), sc, sh, 1, 1, 1, res=None if r is None else T(r), res_pair=True,   # noqa: E731
                                         relu=relu, pair_out=True)
    y, yh, yl = run()
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
    assert not torch.isnan(yh).any() and not torch.isnan(yl).any()            # pad channels written (zeros)
    assert (yh[..., 64:] == 0).all() if yh.shape[-1] > 64 else True
    _, yh2, yl2 = run()
    assert torch.equal(yh2, yh) and torch.equal(yl2, yl), 'not bit-identical from run to run'
    try:
        for flags in (8, 32, 40):
            set_flags(flags)
            _, yh3, yl3 = run()
            assert torch.equal(yh3, yh) and torch.equal(yl3, yl), 'flags %d change the output' % flags
    finally:
        set_flags(0)


@pytest.mark.parametrize('res,relu', [(False, False), (True, True)])
def test_affine_conv2d_1x1_stride2_fp32_out_vs_oracle(res, relu):
    """The downsample shortcut's form (psm_submodule.py:128-131): Conv2d 1x1 stride 2 + BatchNorm2d, fp32 output."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(21 + res)
    x = rng.standard_normal((2, 32, 240, 320)).astype(np.float32)
    w = (rng.standard_normal((64, 32, 1, 1)) / math.sqrt(32)).astype(np.float32)
    g, b, rm, rv = _coeffs(rng, 64)
    r = rng.standard_normal((2, 64, 120, 160)).astype(np.float32) if res else None
    sc, sh = convops.bn_eval_coeffs(T(g), T(b), T(rm), T(rv))
    ref = _affine_ref(N.conv2d(x, w, None, 2, 0, 1), g, b, rm, rv, r, relu)
    run = lambda: convops.conv_h2_affine(T(x), T(w), sc, sh, 2, 0, 1, res=None if r is None else T(r), relu=relu)   # noqa: E731
    y = run()
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
    assert torch.equal(run(), y)
    try:
        for flags in (8, 32, 40):
            set_flags(flags)
            assert torch.equal(run(), y), 'flags %d change the output' % flags
    finally:
        set_flags(0)


# ---- engine ------------------------------------------------------------------------------------------------------------
def _case(name):
    if name in cases.KVNET_CASES:
        c = cases.kvnet_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    else:
        c = cases.big_case(name)
        cam = cases.big_cam(O.make_cam_intrinsics, c)
    return c, cam


def _eval_sd(c, gold, name):
    """The case's weights with the running statistics the reference produced (make_golden_eval.py)."""
    sd = {k: np.asarray(v) for k, v in c['sd'].items()}
    pre = 'eval/%s/rs/' % name
    sd.update({k[len(pre):]: np.asarray(gold[k]) for k in gold.files if k.startswith(pre)})
    return sd


def _knet_gate(pin, name, key, conv_math):
    """Probability gate of a re-seeded K-Net step. C2/C3: train mode's gate for the same step and arithmetic
    (test_gpu_configs.py: 1.5e-4 in f16x3, 5e-4 otherwise). kvnet_256_d16 (16 planes): twice the measured oracle-vs-reference
    floor of this step (full arrays, PINNING_eval.json), the fp32-vs-fp32 noise at that shape."""
    if name in cases.KVNET_CASES:
        p = pin[key]
        return 2.0 * max(p['oracle_DPV_prob'], p['oracle_dmap_refined_prob'])
    return TOL_KNET_F16 if conv_math == 'f16x3' else TOL_KNET


# the steady steps, each re-seeded with the reference's train-mode prior of the step before (as the fixture was recorded)
RESEEDED = [('kvnet_256_d16', 1), ('kvnet_256_d16', 2), ('c23_640x480_d64_v4_stream30', 1)]


@pytest.mark.parametrize('conv_math', MODES)
@pytest.mark.parametrize('name', ['kvnet_256_d16', 'c23_640x480_d64_v4_stream30'])
def test_engine_eval_vs_reference(name, conv_math):
    gold, pin = harness.golden('eval_outputs.npz'), harness.pinning('PINNING_eval.json')
    c, cam = _case(name)
    cam_t = harness.cam_tensors(cam)
    m = harness.engine_kvnet(c, cam_t, _eval_sd(c, gold, name), conv_math).eval()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    rows = {}
    full = harness.engine_forward(m, c, cam_t, 0, None)[1]
    rows['step0'] = r0 = harness.compare_outputs(gold, 'eval/%s/step0' % name, full, c['d'])
    for nm, s in RESEEDED:
        if nm != name:
            continue
        key = 'eval/%s/step%d' % (name, s)
        full = harness.engine_forward(m, c, cam_t, s, harness.reference_prior(name, s))[1]
        rows['step%d' % s] = r = harness.compare_outputs(gold, key, full, c['d'])
        r['gate'] = _knet_gate(pin, name, key, conv_math)
    harness.parity_dump('eval', '%s/%s' % (name, conv_math), rows)
    msg = json.dumps(rows)
    assert max(r0[nm] for nm in NAMES4) <= TOL_FIRST and r0['depth_mm'] <= TOL_DEPTH_MM, msg
    for k, r in rows.items():
        if k == 'step0':
            continue
        assert r['DPV'] <= r['gate'] and r['dmap_refined'] <= r['gate'], msg       # depth: recorded, gated on first windows
    assert max(v for r in rows.values() for k, v in r.items() if k.endswith('_sumsq_rel')) <= TOL_SUMSQ_REL, msg
    # no buffer moves in eval mode: running statistics, num_batches_tracked, the whole state_dict
    after = m.state_dict()
    assert before.keys() == after.keys()
    changed = [k for k in before if not torch.equal(before[k].cpu(), after[k].cpu())]
    assert not changed, changed


def test_engine_eval_train_eval_on_one_engine():
    """eval -> train -> eval: the train forward matches the train-mode fixture and updates the running statistics; the
    second eval forward normalises with the updated statistics (checked against the eval oracle fed those buffers)."""
    name = 'kvnet_256_d16'
    gold = harness.golden('eval_outputs.npz')
    ref_gold = harness.golden('reference_outputs.npz')
    c, cam = _case(name)
    cam_t = harness.cam_tensors(cam)
    m = harness.engine_kvnet(c, cam_t, {k: np.asarray(v) for k, v in c['sd'].items()}, 'f16x3')
    prior_eval = harness.reference_prior(name, 1)
    m.eval()
    e1 = harness.engine_forward(m, c, cam_t, 1, prior_eval)[1]
    # train mode, the steady step of the train fixture (its own prior): K-Net's BatchNorm3d and the downsample layers update
    m.train()
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    t = harness.engine_forward(m, c, cam_t, 1, prior_eval)[1]
    for nm, a in zip(NAMES4, t):
        e = maxabs(np.exp(cases.subsample(a.cpu().numpy())), np.exp(ref_gold['kvnet/%s/step1/%s' % (name, nm)]))
        assert e <= (1e-4 if nm in ('BV_cur', 'dmap_cur_refined') else 5e-4), (nm, e)
    sd1 = {k: v.clone() for k, v in m.state_dict().items()}
    moved = [k for k in sd0 if k.endswith('running_mean') and not k.startswith('d_net.') and not torch.equal(sd0[k], sd1[k])]
    assert len(moved) == 13, moved
    m.eval()
    e2 = harness.engine_forward(m, c, cam_t, 1, prior_eval)[1]
    assert not torch.equal(e1[3], e2[3])                        # the updated statistics are used
    sd2 = m.state_dict()
    assert all(torch.equal(sd1[k].cpu(), sd2[k].cpu()) for k in sd1)
    ref_f, src_f, poses = cases.window(c, c['t_win_r'] + 1)
    o = E.kvnet_forward({k: v.cpu().numpy() for k, v in sd1.items()}, ref_f, src_f, poses, cam, c['d'], c['sigma'],
                        BV_predict=prior_eval, training=False)
    sub = lambda a: cases.subsample_to(a, SUB_LIMIT)     # noqa: E731  (sampled as every other comparison here)
    row = {nm: maxabs(np.exp(sub(a.cpu().numpy())), np.exp(sub(b))) for nm, a, b in zip(NAMES4, e2, o)}
    harness.parity_dump('eval', '%s/eval_train_eval' % name, row)
    assert row['BV_cur'] <= TOL_FIRST and row['dmap_cur_refined'] <= TOL_FIRST, row
    assert row['DPV'] <= 5e-4 and row['dmap_refined'] <= 5e-4, row


def test_reference_test_runs_eval_model_unmodified():
    out = harness.run_reference_driver('step', 'eval', timeout=900)
    harness.parity_dump('eval', 'dropin', out)
    assert out['class'] == 'neuralrgbd_b200.models.KVNET' and out['training'] is False
    pin = harness.pinning('PINNING_eval.json')
    assert out['steps'][0]['DPV'] <= TOL_FIRST, out
    for s, st in enumerate(out['steps'][1:], 1):                     # re-seeded K-Net steps: the gate of the engine test
        assert st['DPV'] <= _knet_gate(pin, 'kvnet_256_d16', 'eval/kvnet_256_d16/step%d' % s, 'f16x3'), out


def test_eval_step_has_13_fewer_bn_passes():
    """f16x3: K-Net's 11 BatchNorm3d and the 2 downsample BatchNorm2d run in the convolution epilogue in eval mode."""
    from torch.profiler import profile, ProfilerActivity
    from neuralrgbd_b200 import _lib
    name = 'kvnet_256_d16'
    gold = harness.golden('eval_outputs.npz')
    c, cam = _case(name)
    cam_t = harness.cam_tensors(cam)
    m = harness.engine_kvnet(c, cam_t, _eval_sd(c, gold, name), 'f16x3')
    prior = harness.reference_prior(name, 1)

    def count(training):
        m.train(training)
        harness.engine_forward(m, c, cam_t, 1, prior)                       # warm (eager) step of this mode
        ent = next(iter(m._engines.values()))
        _lib.lib().nrgbd_kvnet_set_option(ent['h'], b'use_graph', 0)     # kernels by name, outside a graph
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            harness.engine_forward(m, c, cam_t, 1, prior)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        _lib.lib().nrgbd_kvnet_set_option(ent['h'], b'use_graph', 1)
        return sum('bn_apply' in n for n in names), sum('conv_wg_kernel' in n for n in names)
    bn_train, conv_train = count(True)
    bn_eval, conv_eval = count(False)
    harness.parity_dump('eval', 'bn_launches', {'train': bn_train, 'eval': bn_eval, 'conv_train': conv_train, 'conv_eval': conv_eval})
    assert bn_train - bn_eval == 13, (bn_train, bn_eval)
    assert conv_train == conv_eval, (conv_train, conv_eval)
