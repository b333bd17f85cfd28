"""KVNET at temporal window radii 1 and 3 (V = 2 and 6 source views; K-Net input volumes of 10 and 22 channels) on the GPU.

 * Engine against tests/golden/make_golden_twin.py (unmodified reference, re-seeded steady steps) in all three conv_math
   modes, train mode and .eval(): first windows at 1e-4 on probabilities and 1 mm on depth; a steady step at 640x480 D64 at
   train mode's K-Net gate for that arithmetic (test_gpu_configs.py: 1.5e-4 in f16x3, 5e-4 otherwise); the 16-plane steady
   steps at twice the pinned oracle-vs-reference floor (PINNING_twin.json, the largest of the case's steady steps); every
   full array through the relative deviation of its sum of squared probabilities.
 * r = 1 with refineNet_name='DGF' and with if_refined=False; two f16x3 eval-mode steady steps at r = 1 bit for bit; the
   reference's unmodified test() at r = 1 and 3; FrameWindow's window order; and, in f16x3 at r = 1, K-Net's first layer on
   the same tensor-core pair path as at r = 2 (no fp32-path convolution, no split pass for the volume).
Measured deviations are written to $NRGBD_PARITY_DIR/parity_twin.json when that variable is set.
"""
import contextlib
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from neuralrgbd_b200 import arch
from oracle import planesweep_oracle as O
from tests import cases
from tests import cases_twin as CT
from tests import oracle_refine as R
from tests.conftest import ROOT, maxabs

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
NAMES4 = ['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV']
SUB_LIMIT = 8000          # the fixture's strided samples (make_golden_twin.py)
DEPTH_LIMIT = 2000
TOL_SUMSQ_REL = 1e-4
TOL_FIRST = 1e-4
TOL_DEPTH_MM = 1.0
TOL_KNET_F16 = 1.5e-4
TOL_KNET = 5e-4
TOL_SELF_M = 1e-5         # engine DGF vs the oracle's filter on the engine's own low-resolution DPV (test_gpu_refine.py)
MODES = ['f16x3', 'tf32x3', 'fp32']


def _dump(key, row):
    d = os.environ.get('NRGBD_PARITY_DIR')
    if not d:
        return
    try:
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, 'parity_twin.json')
        cur = json.load(open(path)) if os.path.exists(path) else {}
        cur[key] = row
        with open(path, 'w') as f:
            json.dump(cur, f, indent=1, sort_keys=True)
    except OSError:
        pass


def _gold():
    return np.load(os.path.join(ROOT, 'tests', 'golden', 'twin_outputs.npz'))


def _pin():
    return json.load(open(os.path.join(ROOT, 'tests', 'golden', 'PINNING_twin.json')))['cases']


def _case(name):
    c = CT.twin_case(name)
    cam = CT.twin_cam(O.make_cam_intrinsics, c)
    return c, cam, dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']),
                        intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))


def _sd(c, gold=None, name=None, refine='DPV'):
    """The case's weights; with `gold`, the running statistics the reference warmed (eval fixtures); refine='DGF' / None swaps
    in that configuration's R-Net weights."""
    sd = {k: np.asarray(v) for k, v in c['sd'].items()}
    if gold is not None:
        pre = 'twin/eval/%s/rs/' % name
        sd.update({k[len(pre):]: np.asarray(gold[k]) for k in gold.files if k.startswith(pre)})
    if refine != 'DPV':
        sd = {k: v for k, v in sd.items() if not k.startswith('r_net.')}
        if refine == 'DGF':
            rn = arch.synth_state_dict(c['wseed'], 64, c['D'], c['t_win_r'], 64, refine='DGF')
            sd.update({k: v for k, v in rn.items() if k.startswith('r_net.')})
    return sd


def _model(c, cam_t, sd, conv_math, **kw):
    from neuralrgbd_b200.models.KVNET import KVNET
    with contextlib.redirect_stdout(io.StringIO()):
        m = KVNET(feature_dim=64, cam_intrinsics=cam_t, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                  d_upsample_ratio_KV_net=None, t_win_r=c['t_win_r'], **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    m = m.to(dev)
    m.conv_math = conv_math
    return m


def _forward(m, c, cam_t, step, prior):
    ref_f, src_f, poses = cases.window(c, c['t_win_r'] + step)
    assert src_f.shape[1] == 2 * c['t_win_r']
    with torch.no_grad():
        out = m(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam_t], BV_predict=None if prior is None else T(prior))
    return ref_f, out


def _compare(gold, key, full, d):
    """As test_gpu_eval.py: max-abs probability deviation on the stored samples, the sum of squared probabilities of every
    full array, the expected depth in mm."""
    row = {}
    aliases = {'DPV': 'BV_cur', 'dmap_refined': 'dmap_cur_refined'} if key.endswith('/step0') else {}
    for nm, a in zip(NAMES4, full):
        a = a.cpu().numpy()
        assert np.isfinite(a).all(), (key, nm)
        k = '%s/%s' % (key, aliases.get(nm, nm))
        if k in gold.files:
            row[nm] = maxabs(np.exp(cases.subsample_to(a, SUB_LIMIT)), np.exp(gold[k]))
        st, gs = cases.stats(np.exp(a.astype(np.float64))), gold['%s/%s_stats' % (key, nm)]
        row[nm + '_sumsq_rel'] = abs(st[1] - gs[1]) / gs[1]
    from neuralrgbd_b200.mutils import misc
    dep = misc.depth_val_regression(full[3], d).cpu().numpy()
    row['depth_mm'] = 1000.0 * maxabs(cases.subsample_to(dep, DEPTH_LIMIT), gold[key + '/depth'])
    return row


def _knet_gate(pin, c, key, conv_math):
    """Probability gate of a re-seeded K-Net step: train mode's gate for the arithmetic at 640x480 D64; at 16 planes twice
    the pinned oracle-vs-reference floor (full arrays), the fp32-vs-fp32 noise at that shape. The floor is the largest of
    the case's steady steps, train and eval: one step's floor is one sample of that noise (r = 1, step 2: 8.4e-5 in train
    mode, 1.5e-4 in eval mode, same frames and prior)."""
    if c['D'] == 16:
        case = key.split('/')[2]
        return 2.0 * max(max(p['oracle_DPV_prob'], p['oracle_dmap_refined_prob']) for k, p in pin.items()
                         if k.split('/')[2] == case and not k.endswith('/step0'))
    return TOL_KNET_F16 if conv_math == 'f16x3' else TOL_KNET


RUNS = [(n, 'train') for n in CT.TWIN_CASES] + [(n, 'eval') for n in CT.EVAL_CASES]


@pytest.mark.parametrize('conv_math', MODES)
@pytest.mark.parametrize('name,mode', RUNS)
def test_engine_twin_vs_reference(name, mode, conv_math):
    gold, pin = _gold(), _pin()
    c, cam, cam_t = _case(name)
    m = _model(c, cam_t, _sd(c, gold if mode == 'eval' else None, name), conv_math)
    m.train(mode == 'train')
    rows = {}
    for k in range(c['n_steps']):
        key = 'twin/%s/%s/step%d' % (mode, name, k)
        _, full = _forward(m, c, cam_t, k, CT.prior(name, k) if k else None)
        rows['step%d' % k] = r = _compare(gold, key, full, c['d'])
        if k:
            r['gate'] = _knet_gate(pin, c, key, conv_math)
    _dump('%s/%s/%s' % (mode, name, conv_math), rows)
    msg = json.dumps(rows)
    r0 = rows['step0']
    assert max(r0[nm] for nm in NAMES4) <= TOL_FIRST and r0['depth_mm'] <= TOL_DEPTH_MM, msg
    for k, r in rows.items():
        if k != 'step0':
            assert r['DPV'] <= r['gate'] and r['dmap_refined'] <= r['gate'], msg       # depth: recorded, gated on first windows
    assert max(v for r in rows.values() for k, v in r.items() if k.endswith('_sumsq_rel')) <= TOL_SUMSQ_REL, msg


def _self_check(out_refined, lowres, ref_f, d, sd):
    """The engine's DGF map against the oracle's filter fed the engine's own low-resolution DPV (test_gpu_refine.py)."""
    from neuralrgbd_b200.mutils import misc
    dm = misc.depth_val_regression(lowres, d).cpu().numpy()[0]
    return maxabs(out_refined.cpu().numpy()[0, 0], R.dgf_refine(dm, ref_f[0], sd))


@pytest.mark.parametrize('conv_math', MODES)
@pytest.mark.parametrize('cfg', ['DGF', 'none'])
def test_refine_configurations_at_r1(cfg, conv_math):
    """refineNet_name='DGF' and if_refined=False at r = 1, first window + one steady step. The low-resolution DPV does not
    depend on the refinement: it meets the train-mode fixture's gates. The DGF maps equal the oracle's guided filter fed the
    engine's own DPV."""
    name = 'r1_256_d16'
    gold, pin = _gold(), _pin()
    c, cam, cam_t = _case(name)
    sd = _sd(c, refine='DGF' if cfg == 'DGF' else None)
    m = _model(c, cam_t, sd, conv_math, **({'refineNet_name': 'DGF'} if cfg == 'DGF' else {'if_refined': False}))
    rows = {}
    for k in range(2):
        ref_f, out = _forward(m, c, cam_t, k, CT.prior(name, k) if k else None)
        key = 'twin/train/%s/step%d' % (name, k)
        lowres = out[2] if k == 0 else out[3]
        r = {'prob': maxabs(np.exp(cases.subsample_to(lowres.cpu().numpy(), SUB_LIMIT)), np.exp(gold[key + ('/BV_cur' if k == 0 else '/DPV')])),
             'gate': TOL_FIRST if k == 0 else _knet_gate(pin, c, key, conv_math)}
        if cfg == 'none':
            assert out[0] == -1 and out[1] == -1
        else:
            assert out[0].shape == (1, 1, c['H'], c['W']) and out[1].shape == (1, 1, c['H'], c['W'])
            r['self_m'] = _self_check(out[0] if k == 0 else out[1], lowres, ref_f, c['d'], sd)
            if k:
                r['self_cur_m'] = _self_check(out[0], out[2], ref_f, c['d'], sd)
        rows['step%d' % k] = r
    _dump('%s/%s/%s' % (cfg, name, conv_math), rows)
    for r in rows.values():
        assert r['prob'] <= r['gate'], rows
        assert r.get('self_m', 0) <= TOL_SELF_M and r.get('self_cur_m', 0) <= TOL_SELF_M, rows


def test_f16_eval_steady_step_bit_identical_at_r1():
    """Eval mode in f16x3 uses no atomics, so repeated steady steps at r = 1 (eager, graph capture, graph replay) give the
    same bits: no uninitialised or out-of-range data reaches the outputs."""
    name = 'r1_256_d16'
    gold = _gold()
    c, cam, cam_t = _case(name)
    m = _model(c, cam_t, _sd(c, gold, name), 'f16x3').eval()
    prior = CT.prior(name, 1)
    _forward(m, c, cam_t, 0, None)
    runs = [[t.clone() for t in _forward(m, c, cam_t, 1, prior)[1]] for _ in range(3)]
    for run in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], run))


@pytest.mark.parametrize('name', ['r1_256_d16', 'r3_256_d16'])
def test_reference_test_runs_unmodified(name):
    from oracle import fetch_reference
    ref_code = fetch_reference.code_dir()
    assert ref_code, 'no copy of the reference: oracle/_ref is made by __graft_entry__.build() (oracle/fetch_reference.py)'
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'dropin_twin_driver.py'), ref_code, name],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    out = json.loads(r.stdout.strip().splitlines()[-1])
    _dump('dropin/%s' % name, out)
    c = CT.twin_case(name)
    pin = _pin()
    assert out['class'] == 'neuralrgbd_b200.models.KVNET' and out['t_win_r'] == c['t_win_r']
    assert len(out['steps']) == 3 and all(s['V'] == 2 * c['t_win_r'] and s['prior_finite'] for s in out['steps']), out
    assert out['steps'][0]['DPV'] <= TOL_FIRST, out
    for k, s in enumerate(out['steps'][1:], 1):
        assert s['DPV'] <= _knet_gate(pin, c, 'twin/train/%s/step%d' % (name, k), 'f16x3'), out


@pytest.mark.parametrize('r', [1, 3])
def test_frame_window_order(r):
    """FrameWindow(t_win_r=r) hands out the reference's split (split_frame_list, misc.py:509-517): reference = the middle
    frame, sources = the others in window order, as the fixtures' windows (synth.window_rel_poses)."""
    from neuralrgbd_b200.mdataloader import m_preprocess as M
    from neuralrgbd_b200.mutils import misc
    from neuralrgbd_b200 import synth
    n = 2 * r + 1
    frames = [np.full((16, 16, 3), 10 * i, np.uint8) for i in range(n + 2)]
    win = M.FrameWindow(t_win_r=r, img_size=(16, 16))
    full = [win.push(f, extM=i) for i, f in enumerate(frames)]
    assert full == [False] * (n - 1) + [True] * 3
    ref, src = win.window()                                    # frames 2 .. n + 1
    assert tuple(src.shape) == (1, 2 * r, 3, 16, 16)
    ref_d, src_d = misc.split_frame_list(win.frame_dicts(), r)
    assert ref_d['extM'] == r + 2 and torch.equal(ref_d['img'], ref)
    assert [d['extM'] for d in src_d] == [i for i in range(2, n + 2) if i != r + 2]
    for k, d in enumerate(src_d):
        assert torch.equal(d['img'][0], src[0, k])
    exts = synth.camera_track(np.random.RandomState(0), n + 2)
    _, idx = synth.window_rel_poses(exts, r + 2, r)
    assert list(idx) == [d['extM'] for d in src_d]


def test_r1_knet_first_layer_on_the_pair_path():
    """f16x3, steady step at r = 1: the 10-channel K-Net volume is written as the operand pair of dres0.0 and read by the
    tensor-core convolution at Cin_pad = 32, as the 16-channel volume at r = 2 is. Both radii launch the same number of
    tensor-core convolutions, fp32-path convolutions (the feature CNN's 3-channel first layer only, as in a first window)
    and split passes."""
    from torch.profiler import profile, ProfilerActivity
    from neuralrgbd_b200 import _lib

    def count(c, cam_t, prior, step):
        m = _model(c, cam_t, _sd(c), 'f16x3')
        _forward(m, c, cam_t, 0, None)
        _forward(m, c, cam_t, 1, prior)                        # warm (eager) steady step
        ent = next(iter(m._engines.values()))
        _lib.lib().nrgbd_kvnet_set_option(ent['h'], b'use_graph', 0)     # kernels by name, outside a graph
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _forward(m, c, cam_t, step, prior if step else None)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        return {k: sum(k in n for n in names) for k in ('conv_igemm_kernel', 'conv_wg_kernel', 'split_f16_pair_kernel')}

    c1, _, cam1 = _case('r1_256_d16')
    c2 = cases.kvnet_case('kvnet_256_d16')
    cam2 = cases.cam_for(O.make_cam_intrinsics, c2['W'] // 4, c2['H'] // 4)
    cam2 = dict(cam2, unit_ray_array_2D=torch.from_numpy(cam2['unit_ray_array_2D']), intrinsic_M_cuda=torch.from_numpy(cam2['intrinsic_M_cuda']))
    prior = CT.prior('r1_256_d16', 1)
    r1_first, r1 = count(c1, cam1, prior, 0), count(c1, cam1, prior, 1)
    r2 = count(c2, cam2, prior, 1)
    _dump('launches', {'r1_first': r1_first, 'r1_steady': r1, 'r2_steady': r2})
    assert r1 == r2, (r1, r2)
    assert r1['conv_igemm_kernel'] == r1_first['conv_igemm_kernel'], (r1, r1_first)
    assert r1['conv_wg_kernel'] > r1_first['conv_wg_kernel'], (r1, r1_first)
