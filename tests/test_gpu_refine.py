"""KVNET's other refinement configurations on the GPU: refineNet_name='DGF' (guided-filter depth maps) and if_refined=False.

 * Op level: nrgbd_guided_filter_refine against tests/oracle_refine.py, bit for bit, on ragged sizes, a textured guide and a
   guide that is flat over whole regions (var_x = 0 there: A = cov / 1e-8), against the reference's RefineNet_DGF within its
   pinned floor, and bit-identical from run to run; bit for bit against the oracle at the engine's 256x256 and 480x640.
 * Engine against tests/golden/make_golden.py refine (unmodified reference, re-seeded steady steps) in all three conv_math
   modes. if_refined=False: -1 for both refined outputs, probabilities at 1e-4 on first windows and the train-mode K-Net gate
   on steady steps. DGF: depth maps in metres at GATE_MULT times the larger pinned oracle-vs-reference deviation of the step
   (the fp32-vs-fp32 floor of the ill-conditioned filter), and bit-close to the oracle's filter fed the engine's own DPV.
 * Eval mode with each configuration, the reference's unmodified test(), and no R-Net kernel for if_refined=False.
Measured deviations are written to $NRGBD_PARITY_DIR/parity_refine.json when that variable is set.
"""
import json

import numpy as np
import pytest
import torch

from neuralrgbd_b200 import arch
from oracle import planesweep_oracle as O
from tests import cases, harness
from tests import oracle_refine as R
from tests.conftest import maxabs
from tests.harness import DEV as dev, T

pytestmark = pytest.mark.gpu
SUB_LIMIT = 8000
TOL_FIRST = 1e-4
TOL_KNET_F16 = 1.5e-4
TOL_KNET = 5e-4
GATE_MULT = 2.0
TOL_DEPTH_MM = 1.0
TOL_SELF_M = 1e-5          # engine DGF vs the oracle's filter on the engine's own low-resolution DPV
MODES = ['f16x3', 'tf32x3', 'fp32']
STEPS = {'kvnet_256_d16': 3, 'c23_640x480_d64_v4_stream30': 2}


# ---- op level ----------------------------------------------------------------------------------------------------------
def _gf_refine(g):
    from neuralrgbd_b200 import convops
    sd = {k: T(v) for k, v in g['sd'].items()}
    return convops.guided_filter_refine(T(g['dmap']), T(g['img']), sd['r_net.feature_ext.0.weight'], sd['r_net.feature_ext.0.bias'],
                                        sd['r_net.feature_ext.2.weight'], sd['r_net.feature_ext.2.bias'])


@pytest.mark.parametrize('name', R.GF_CASES)
def test_guided_filter_kernel_vs_oracle(name):
    g = R.gf_case(name)
    y = _gf_refine(g)
    got = y.cpu().numpy()
    want = R.dgf_refine(g['dmap'], g['img'], g['sd'])
    ref = harness.golden('refine_outputs.npz')['refine/gf/%s/out' % name]
    row = {'oracle_m': maxabs(got, want), 'reference_m': maxabs(got, ref), 'bitexact_oracle': bool(np.array_equal(got, want))}
    harness.parity_dump('refine', 'gf/%s' % name, row)
    assert np.array_equal(got, want), row
    assert row['reference_m'] <= harness.pinning('PINNING_refine.json')['gf/%s' % name]['oracle_m'], row
    assert torch.equal(_gf_refine(g), y), 'not bit-identical from run to run'


@pytest.mark.parametrize('name', R.GF_ENGINE_CASES)
def test_guided_filter_kernel_vs_oracle_at_engine_sizes(name):
    """256x256 (kvnet_256_d16) and 480x640 (c23), where the column pass's segments and the row pass's lane segments are
    long: bit for bit against the oracle."""
    g = R.gf_case(name)
    got, want = _gf_refine(g).cpu().numpy(), R.dgf_refine(g['dmap'], g['img'], g['sd'])
    assert np.array_equal(got, want), {'oracle_m': maxabs(got, want), 'differing': int((got != want).sum()),
                                       'first': np.argwhere(got != want)[:4].tolist()}


# ---- engine ------------------------------------------------------------------------------------------------------------
def _case(name):
    if name in cases.KVNET_CASES:
        c = cases.kvnet_case(name)
        cam = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
        wseed = 5
    else:
        c = cases.big_case(name)
        cam = cases.big_cam(O.make_cam_intrinsics, c)
        wseed = cases.BIG_CFG[name]['wseed']
    return c, cam, wseed


KW = {'DGF': dict(if_refined=True, refineNet_name='DGF'), 'none': dict(if_refined=False),
      'DPV_up': dict(if_refined=True, refineNet_name='DPV', if_upsample_d=True)}


def _sd(c, wseed, cfg):
    sd = {k: np.asarray(v) for k, v in c['sd'].items() if not k.startswith('r_net.')}
    if cfg != 'none':
        rn = arch.synth_state_dict(wseed, 64, c['D'], c['t_win_r'], 64, refine='DGF' if cfg == 'DGF' else 'DPV',
                                   upsample_d=cfg == 'DPV_up')
        sd.update({k: v for k, v in rn.items() if k.startswith('r_net.')})
    return sd


def _self_check(out_refined, lowres, ref_f, d, sd):
    """The engine's DGF map against the oracle's filter fed the engine's own low-resolution DPV and expected depth (same
    depth_val_regression kernel): the filter and its plumbing without the DPV's fp32 deviation."""
    from neuralrgbd_b200.mutils import misc
    dm = misc.depth_val_regression(lowres, d).cpu().numpy()[0]
    return maxabs(out_refined.cpu().numpy()[0, 0], R.dgf_refine(dm, ref_f[0], sd))


@pytest.mark.parametrize('conv_math', MODES)
@pytest.mark.parametrize('name', ['kvnet_256_d16', 'c23_640x480_d64_v4_stream30'])
@pytest.mark.parametrize('cfg', ['DGF', 'none'])
def test_engine_refine_vs_reference(cfg, name, conv_math):
    gold, pin = harness.golden('refine_outputs.npz'), harness.pinning('PINNING_refine.json')
    c, cam, wseed = _case(name)
    cam_t = harness.cam_tensors(cam)
    sd = _sd(c, wseed, cfg)
    m = harness.engine_kvnet(c, cam_t, sd, conv_math, **KW[cfg])
    rows = {}
    for k in range(STEPS[name]):
        prior = harness.reference_prior(name, k) if k else None
        ref_f, out = harness.engine_forward(m, c, cam_t, k, prior)
        key = 'refine/%s/%s/step%d' % (cfg, name, k)
        lowres = out[2] if k == 0 else out[3]
        a = lowres.cpu().numpy()
        assert np.isfinite(a).all()
        # the low-resolution DPV does not depend on the refinement: the fixture stores it once, under 'none'
        r = {'prob': maxabs(np.exp(cases.subsample_to(a, SUB_LIMIT)), np.exp(gold['refine/none/%s/step%d/DPV' % (name, k)]))}
        r['prob_gate'] = TOL_FIRST if k == 0 else (TOL_KNET_F16 if conv_math == 'f16x3' and name not in cases.KVNET_CASES else TOL_KNET)
        if cfg == 'none':
            assert out[0] == -1 and out[1] == -1
        else:
            assert out[0].shape == (1, 1, c['H'], c['W']) and out[1].shape == (1, 1, c['H'], c['W'])
            if k == 0:
                assert torch.equal(out[0], out[1])
            dm = out[0] if k == 0 else out[1]
            assert torch.isfinite(dm).all()
            p = pin[key]
            r['dmap_m'] = maxabs(cases.subsample_to(dm.cpu().numpy()[0, 0], SUB_LIMIT), gold[key + '/dmap'])
            r['dmap_gate_m'] = GATE_MULT * max(p['oracle_dgf_m'], p['oracle_fwd_dgf_m'])
            st, gs = cases.stats(dm.cpu().numpy()[0, 0]), gold[key + '/dmap_stats']
            r['dmap_mean_rel'] = abs(st[0] - gs[0]) / abs(gs[0])
            r['self_m'] = _self_check(dm, lowres, ref_f, c['d'], sd)
            if k:
                r['dmap_cur_m'] = maxabs(cases.subsample_to(out[0].cpu().numpy()[0, 0], SUB_LIMIT), gold[key + '/dmap_cur'])
                r['self_cur_m'] = _self_check(out[0], out[2], ref_f, c['d'], sd)
        rows['step%d' % k] = r
    harness.parity_dump('refine', '%s/%s/%s' % (cfg, name, conv_math), rows)
    msg = json.dumps(rows)
    for r in rows.values():
        assert r['prob'] <= r['prob_gate'], msg
        if cfg == 'DGF':
            assert r['dmap_m'] <= r['dmap_gate_m'] and r.get('dmap_cur_m', 0) <= r['dmap_gate_m'], msg
            assert r['dmap_mean_rel'] <= 1e-4, msg
            assert r['self_m'] <= TOL_SELF_M and r.get('self_cur_m', 0) <= TOL_SELF_M, msg


def _dup4(d):
    """The loaders' 4D candidates (mdataloader/scanNet.py:327, dl_7scenes.py:250)."""
    return np.linspace(d.min(), d.max(), 4 * len(d))


@pytest.mark.parametrize('conv_math', MODES)
@pytest.mark.parametrize('name', ['kvnet_256_d16', 'c23_640x480_d64_v4_stream30'])
def test_engine_upsample_d_vs_reference(name, conv_math):
    """if_upsample_d=True: refined log-DPVs of 4D planes. Probabilities at 1e-4 on first windows and at the train-mode K-Net
    gate on re-seeded steady steps; the expected depth over the loaders' dup4_candi through the depth_val_regression and export
    mirrors at 1 mm on first windows (twice the oracle's floor, at least 1 mm, on steady steps), and both mirrors against the
    numpy regression of the same array."""
    from neuralrgbd_b200.mutils import misc
    from neuralrgbd_b200.test_utils import export_res
    gold, pin = harness.golden('refine_outputs.npz'), harness.pinning('PINNING_refine.json')
    c, cam, wseed = _case(name)
    cam_t = harness.cam_tensors(cam)
    m = harness.engine_kvnet(c, cam_t, _sd(c, wseed, 'DPV_up'), conv_math, **KW['DPV_up'])
    dup4 = _dup4(c['d'])
    rows = {}
    for k in range(STEPS[name]):
        prior = harness.reference_prior(name, k) if k else None
        _, out = harness.engine_forward(m, c, cam_t, k, prior)
        key = 'refine/DPV_up/%s/step%d' % (name, k)
        ref = out[0] if k == 0 else out[1]
        assert ref.shape == (1, 4 * c['D'], c['H'], c['W']) and out[2].shape == (1, c['D'], c['H'] // 4, c['W'] // 4)
        if k == 0:
            assert torch.equal(out[0], out[1])
        a = ref.cpu().numpy()
        assert np.isfinite(a).all()
        r = {'prob': maxabs(np.exp(cases.subsample_to(a[0], SUB_LIMIT)), np.exp(gold[key + '/dpv_up']))}
        r['prob_gate'] = TOL_FIRST if k == 0 else (TOL_KNET_F16 if conv_math == 'f16x3' and name not in cases.KVNET_CASES else TOL_KNET)
        st, gs = cases.stats(np.exp(a.astype(np.float64))), gold[key + '/dpv_up_stats']
        r['sumsq_rel'] = abs(st[1] - gs[1]) / gs[1]
        dep = misc.depth_val_regression(ref, dup4).cpu().numpy()[0]
        r['depth_mm'] = 1000 * maxabs(cases.subsample_to(dep, SUB_LIMIT), gold[key + '/depth_dup4'])
        r['depth_gate_mm'] = TOL_DEPTH_MM if k == 0 else max(TOL_DEPTH_MM, 2 * pin[key]['oracle_up_depth_mm'])
        exp_dep = export_res.depth_conf_maps(ref, dup4, want_u16=False)['dmap'].cpu().numpy()
        num = O.depth_val_regression(a, dup4)[0]
        r['mirrors_vs_numpy_m'] = max(maxabs(dep, num), maxabs(exp_dep, num))
        rows['step%d' % k] = r
    harness.parity_dump('refine', 'DPV_up/%s/%s' % (name, conv_math), rows)
    msg = json.dumps(rows)
    for r in rows.values():
        assert r['prob'] <= r['prob_gate'] and r['sumsq_rel'] <= 1e-4, msg
        assert r['depth_mm'] <= r['depth_gate_mm'], msg
        assert r['mirrors_vs_numpy_m'] <= 1e-5, msg


def test_log_softmax_over_1024_contiguous_planes():
    """nrgbd_dpv_normalize's thread-per-pixel path, which the upsampled R-Net takes above 256 planes (D = 256 -> 1024)."""
    import ctypes
    from neuralrgbd_b200 import _lib
    from neuralrgbd_b200._lib import ptr
    rng = np.random.RandomState(3)
    D, n = 1024, 3000
    x = (4 * rng.standard_normal((n, D))).astype(np.float32)
    xt = T(x)
    y = torch.empty_like(xt)
    _lib.check(_lib.lib().nrgbd_dpv_normalize(ptr(xt), 1, D, None, 0, 0, ctypes.c_float(1.0), n, D, ptr(y), 1, D, None, None, None,
                                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    x64 = x.astype(np.float64)
    want = x64 - x64.max(1, keepdims=True) - np.log(np.exp(x64 - x64.max(1, keepdims=True)).sum(1, keepdims=True))
    assert maxabs(y.cpu().numpy(), want) <= 2e-5


@pytest.mark.parametrize('cfg', ['DGF', 'none', 'DPV_up'])
def test_eval_mode_each_configuration(cfg):
    """.eval() with each configuration: the running-statistics BatchNorm path with the new refinements; nothing moves."""
    name = 'kvnet_256_d16'
    c, cam, wseed = _case(name)
    cam_t = harness.cam_tensors(cam)
    sd = _sd(c, wseed, cfg)
    m = harness.engine_kvnet(c, cam_t, sd, 'f16x3', **KW[cfg]).eval()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    for k in range(2):
        ref_f, out = harness.engine_forward(m, c, cam_t, k, harness.reference_prior(name, k) if k else None)
        lowres = out[2] if k == 0 else out[3]
        assert torch.isfinite(lowres).all()
        if cfg == 'none':
            assert out[0] == -1 and out[1] == -1
        elif cfg == 'DPV_up':
            assert out[1].shape[1] == 4 * c['D'] and torch.isfinite(out[1]).all()
            assert torch.allclose(out[1].exp().sum(1), torch.ones(1, device=dev), atol=1e-4)
        else:
            assert _self_check(out[1], lowres, ref_f, c['d'], sd) <= TOL_SELF_M
    after = m.state_dict()
    assert all(torch.equal(before[k], after[k]) for k in before)


@pytest.mark.parametrize('cfg', ['DGF', 'none', 'DPV_up'])
def test_reference_test_runs_unmodified(cfg):
    pin = harness.pinning('PINNING_refine.json')
    for mode in ('train', 'eval'):
        out = harness.run_reference_driver('step', 'refine', cfg, mode, timeout=900)
        harness.parity_dump('refine', 'dropin/%s/%s' % (cfg, mode), out)
        assert out['class'] == 'neuralrgbd_b200.models.KVNET'
        assert all(s['finite'] for s in out['steps'])
        if mode == 'eval':
            continue                         # the fixtures are train-mode outputs
        for k, s in enumerate(out['steps']):
            if cfg == 'DGF':
                assert s['shape'] == [1, 1, 256, 256]
                p = pin['refine/DGF/kvnet_256_d16/step%d' % k]
                assert s['dmap_m'] <= GATE_MULT * max(p['oracle_dgf_m'], p['oracle_fwd_dgf_m']), out
            elif cfg == 'DPV_up':
                assert s['shape'] == [1, 64, 256, 256]
                assert s['DPV'] <= (TOL_FIRST if k == 0 else TOL_KNET), out
            else:
                assert s['shape'] == [1, 16, 64, 64]
                assert s['DPV'] <= (TOL_FIRST if k == 0 else TOL_KNET), out


def test_no_rnet_launches_when_unrefined():
    """if_refined=False: a steady frame launches exactly the kernels of the default engine asked for no refined output -
    no R-Net kernel - and fewer than the default configuration."""
    import ctypes
    from neuralrgbd_b200 import _lib
    from neuralrgbd_b200._lib import ptr
    L = _lib.lib()
    name = 'kvnet_256_d16'
    c, cam, wseed = _case(name)
    cam_t = harness.cam_tensors(cam)
    prior = harness.reference_prior(name, 1)

    def steady_launches(m, call):
        for _ in range(3):                   # eager warm-up, capture, replay
            L.nrgbd_reset_launch_count()
            call(m)
            torch.cuda.synchronize()
        return L.nrgbd_launch_count()

    fwd = lambda m: harness.engine_forward(m, c, cam_t, 1, prior)      # noqa: E731
    n_none = steady_launches(harness.engine_kvnet(c, cam_t, _sd(c, wseed, 'none'), 'f16x3', **KW['none']), fwd)
    m_dpv = harness.engine_kvnet(c, cam_t, c['sd'], 'f16x3')
    n_dpv = steady_launches(m_dpv, fwd)

    def null_refined(m):
        # the default engine, both refined outputs NULL: D-Net, K-Net and the low-resolution outputs only
        ent = next(iter(m._engines.values()))
        ref_f, src_f, poses = cases.window(c, c['t_win_r'] + 1)
        frames = torch.cat((T(src_f)[0], T(ref_f)), 0).contiguous()
        bv_cur = torch.empty((1, c['D'], c['H'] // 4, c['W'] // 4), device=dev)
        dpv = torch.empty_like(bv_cur)
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(L.nrgbd_kvnet_forward(ent['h'], ptr(frames), ptr(T(poses)[0].contiguous()), ptr(T(prior)[0].contiguous()), None,
                                         None, ptr(bv_cur), ptr(dpv), None, None, st))
    n_null = steady_launches(m_dpv, null_refined)
    harness.parity_dump('refine', 'launches', {'none': n_none, 'dpv': n_dpv, 'dpv_null_refined': n_null})
    assert n_none == n_null < n_dpv, (n_none, n_null, n_dpv)
