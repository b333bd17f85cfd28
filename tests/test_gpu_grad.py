"""f-5 on the device: autograd through the warp_img_feats_v3 / _mgpu, resample_vol_cuda and depth_val_regression mirrors.

 * Each backward kernel against tests/oracle_grad.py (float64 sums) and against torch autograd through the unmodified
   reference (tests/golden/make_golden.py grad), gated from the oracle-vs-reference floor pinned in PINNING_grad.json.
 * The no-grad path: the same launches and bit-identical outputs whether or not the inputs require grad, under
   torch.no_grad() or not; the autograd path's forward value is the no-grad one, bit for bit.
 * The reference's own models.KVNET.KVNET (refineNet_name='DGF') trained for one step with the mirrors patched into
   warping.homography / mutils.misc against the unpatched reference (tests/reference_driver.py grad geometry).
Measured deviations are written to $NRGBD_PARITY_DIR/parity_grad.json when that variable is set.
"""
import numpy as np
import pytest
import torch

from oracle import planesweep_oracle as O
from tests import cases, cases_grad as CG, oracle_grad as OG, harness

pytestmark = pytest.mark.gpu
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731

# Gates, relative to the largest reference gradient of the case, on top of the pinned oracle-vs-reference floor:
#  * warp: every source pixel sums grad * weight over up to 4 corners x D planes x the reference pixels that land near
#    it, with fp32 atomics in hardware order; the reference sums the same terms in fp32 in another order (its floor is 2e-6
#    .. 5e-6 of the maximum). 2e-5, as the plane-sweep backward.
#  * resample: a source voxel receives the 8-corner weights of the few output voxels around it (fp32 atomics, 2e-6).
#  * regression: no atomics; the only difference from the oracle is expf against numpy's exp (a few ulp, 1e-6).
REL = {'warp': 2e-5, 'resample': 2e-6, 'regression': 1e-6}


gold = harness.golden_fixture('grad_outputs.npz')
pin = harness.pinning_fixture('PINNING_grad.json')


def _cam(w, h):
    from neuralrgbd_b200 import camera
    return cases.cam_for(camera.make_cam_intrinsics, w, h)


def _ocam(w, h):
    return cases.cam_for(O.make_cam_intrinsics, w, h)


def _gate(gold, pin, key, mine, orc):
    """mine / orc: full gradients (numpy). Against the oracle at REL; against the reference's sample and statistics at
    the pinned floor plus the same allowance."""
    op = key.split('/')[0]
    p = pin[key]
    allow = REL[op] * p['max_ref']
    e_orc = float(np.abs(mine.astype(np.float64) - orc).max())
    e_ref = float(np.abs(CG.sub(mine).astype(np.float64) - gold[key + '/g']).max())
    s, want = cases.summary(mine), gold[key + '/stats']
    harness.parity_dump('grad', key, {'vs_oracle': e_orc, 'vs_reference_sample': e_ref, 'floor': p['maxabs_oracle'], 'max_ref': p['max_ref'],
                'gate': allow})
    assert list(mine.shape) == p['shape']
    assert e_orc <= allow, (key, e_orc, allow)
    assert e_ref <= p['maxabs_oracle'] + allow, (key, e_ref, p['maxabs_oracle'] + allow)
    assert s[2] == want[2]
    assert abs(s[3] - want[3]) <= p['maxabs_oracle'] + allow
    assert abs(s[1] - want[1]) <= 1e-5 * want[1]
    assert abs(s[0] - want[0]) <= (p['maxabs_oracle'] + allow) * want[2]


# ---- warp -----------------------------------------------------------------------------------------------------------
def _warp_grad(c, mgpu=False):
    from neuralrgbd_b200.warping import homography as H
    cam = _cam(c['w'], c['h'])
    if c['tensor']:
        img = T(c['imgs']).requires_grad_(True)
        out = H.warp_img_feats_v3(img, c['d'], T(c['R']), T(c['t']), cam)
        out.backward(T(c['grads']))
        return img.grad.cpu().numpy()
    imgs = [T(i).requires_grad_(True) for i in c['imgs']]
    R, t = [T(r) for r in c['R']], [T(x) for x in c['t']]
    if mgpu:
        out = H.warp_img_feats_mgpu(imgs, c['d'], R, t, T(cam['intrinsic_M_cuda'])[None], T(cam['unit_ray_array_2D'])[None])
    else:
        out = H.warp_img_feats_v3(imgs, c['d'], R, t, cam)
    torch.autograd.backward(out, [T(g) for g in c['grads']])
    for i in imgs:
        assert i.grad is not None and tuple(i.grad.shape) == tuple(i.shape)
    return np.concatenate([i.grad.cpu().numpy() for i in imgs])


@pytest.mark.parametrize('name', CG.WARP_CASES)
def test_warp_backward(gold, pin, name):
    c = CG.warp_case(name)
    mine = _warp_grad(c)
    grads = [c['grads']] if c['tensor'] else c['grads']
    R, t = ([c['R']], [c['t']]) if c['tensor'] else (c['R'], c['t'])
    orc = np.stack(OG.warp_backward([g.reshape(c['C'], c['D'], -1) for g in grads],
                                    OG.warp_taps(c['d'], R, t, _ocam(c['w'], c['h']), c['h'], c['w']), c['h'] * c['w']))
    _gate(gold, pin, 'warp/' + name, mine, orc.reshape(mine.shape))


def test_warp_backward_mgpu_equals_v3():
    """warp_img_feats_mgpu (intrinsics as stacked tensors) has the same gradient as warp_img_feats_v3, up to the atomics'
    order."""
    c = CG.warp_case('warp_v4_c67_37x53_d7')
    a, b = _warp_grad(c), _warp_grad(c, mgpu=True)
    assert np.abs(a - b).max() <= REL['warp'] * np.abs(a).max()


def test_warp_backward_linear_and_dtype():
    """Linear in the upstream gradient; zero upstream gradient gives exactly zero; float64 features get a float64
    gradient."""
    from neuralrgbd_b200.warping import homography as H
    c = CG.warp_case('warp_v4_c3_37x53_d7')
    cam = _cam(c['w'], c['h'])
    R, t = [T(r) for r in c['R']], [T(x) for x in c['t']]

    def grads(gs, dtype=torch.float32):
        imgs = [T(i).to(dtype).requires_grad_(True) for i in c['imgs']]
        torch.autograd.backward(H.warp_img_feats_v3(imgs, c['d'], R, t, cam), gs)
        return torch.cat([i.grad for i in imgs])
    g1 = [T(g) for g in c['grads']]
    g2 = [torch.roll(g, 1, -1) for g in g1]
    a, b, ab = grads(g1), grads(g2), grads([0.5 * x + y for x, y in zip(g1, g2)])
    assert float((ab - (0.5 * a + b)).abs().max()) <= REL['warp'] * float(ab.abs().max())
    assert float(grads([torch.zeros_like(g) for g in g1]).abs().max()) == 0.0
    assert grads(g1, torch.float64).dtype == torch.float64


# ---- resample -------------------------------------------------------------------------------------------------------
def _resample_grad(c):
    from neuralrgbd_b200.warping import homography as H
    vol = T(c['vol']).requires_grad_(True)
    clamp = tuple(c['clamp']) if c['clamp'] is not None else None
    out = H.resample_vol_cuda(vol, T(c['rel']), _cam(c['w'], c['h']), c['d'], c['d_new'], padding_value=c['pad'], clamp=clamp)
    out.backward(T(c['grad']))
    return vol.grad.cpu().numpy()


@pytest.mark.parametrize('name', CG.RESAMPLE_CASES)
def test_resample_backward(gold, pin, name):
    c = CG.resample_case(name)
    mine = _resample_grad(c)
    orc = OG.resample_vol_cuda_backward(c['grad'], c['vol'], c['rel'], _ocam(c['w'], c['h']), c['d'], c['d_new'], c['pad'],
                                        c['clamp'])
    _gate(gold, pin, 'resample/' + name, mine, orc)
    for face in (mine[0, 0], mine[0, -1], mine[0, :, 0], mine[0, :, -1], mine[0, :, :, 0], mine[0, :, :, -1]):
        assert not face.any()


def test_resample_clamp_mask_matches_torch_clamp():
    """The fused clamp's gradient equals resample (no clamp) followed by torch.clamp, differentiated by autograd."""
    from neuralrgbd_b200.warping import homography as H
    c = CG.resample_case('rs_pose_clamp_q_d64')
    cam = _cam(c['w'], c['h'])
    lo, hi = c['clamp']
    a = T(c['vol']).requires_grad_(True)
    H.resample_vol_cuda(a, T(c['rel']), cam, c['d'], padding_value=c['pad'], clamp=(lo, hi)).backward(T(c['grad']))
    b = T(c['vol']).requires_grad_(True)
    H.resample_vol_cuda(b, T(c['rel']), cam, c['d'], padding_value=c['pad']).clamp(min=lo, max=hi).backward(T(c['grad']))
    assert float((a.grad - b.grad).abs().max()) <= REL['resample'] * float(b.grad.abs().max())


# ---- regression -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', CG.REGRESSION_CASES)
def test_regression_backward(gold, pin, name):
    from neuralrgbd_b200.mutils import misc as M
    c = CG.regression_case(name)
    bv = T(c['bv']).requires_grad_(True)
    M.depth_val_regression(bv, c['d'], BV_log=c['log']).backward(T(c['grad']))
    mine = bv.grad.cpu().numpy()
    assert not mine[1:].any()
    _gate(gold, pin, 'regression/' + name, mine, OG.depth_val_regression_backward(c['grad'], c['bv'], c['d'], c['log']))


def test_regression_conf_has_no_gradient():
    from neuralrgbd_b200.mutils import misc as M
    c = CG.regression_case('reg_log_n2_37x53_d16')
    bv = T(c['bv']).requires_grad_(True)
    depth, conf = M.depth_val_regression(bv, c['d'], return_conf=True)
    depth.sum().backward(retain_graph=True)            # depth alone: fine
    assert bv.grad is not None
    with pytest.raises(NotImplementedError):
        (depth.sum() + conf.sum()).backward()


# ---- the no-grad path -----------------------------------------------------------------------------------------------
def _calls():
    from neuralrgbd_b200.warping import homography as H
    from neuralrgbd_b200.mutils import misc as M
    w = CG.warp_case('warp_v4_c67_37x53_d7')
    r = CG.resample_case('rs_pose_clamp_q_d64')
    g = CG.regression_case('reg_log_n2_37x53_d16')
    camw, camr = _cam(w['w'], w['h']), _cam(r['w'], r['h'])
    Rw, tw = [T(x) for x in w['R']], [T(x) for x in w['t']]
    C, V = w['C'], w['V']
    return [
        # pack_features (V launches) + setup + warp per 4-channel chunk
        ('warp', lambda rg: H.warp_img_feats_v3([T(i).requires_grad_(rg) for i in w['imgs']], w['d'], Rw, tw, camw),
         -(-C // 4) * (V + 2)),
        ('resample', lambda rg: H.resample_vol_cuda(T(r['vol']).requires_grad_(rg), T(r['rel']), camr, r['d'],
                                                    padding_value=r['pad'], clamp=tuple(r['clamp'])), 1),
        ('regression', lambda rg: M.depth_val_regression(T(g['bv']).requires_grad_(rg), g['d'], return_conf=True), 1),
    ]


@pytest.mark.parametrize('op', ['warp', 'resample', 'regression'])
def test_no_grad_path_unchanged(op):
    name, fn, want = [x for x in _calls() if x[0] == op][0]
    n0, plain = harness.launch_count(lambda: fn(False))
    with torch.no_grad():
        n1, nog = harness.launch_count(lambda: fn(True))
    n2, withgrad = harness.launch_count(lambda: fn(True))
    flat = lambda o: [x.detach() for x in (o if isinstance(o, (list, tuple)) else [o])]   # noqa: E731
    assert n0 == n1 == n2 == want, (n0, n1, n2, want)
    for a, b, c in zip(flat(plain), flat(nog), flat(withgrad)):
        assert a.grad_fn is None and b.grad_fn is None
        assert torch.equal(a, b) and torch.equal(a, c)
    assert all(x.requires_grad for x in (withgrad if isinstance(withgrad, (list, tuple)) else [withgrad]))


# ---- end to end on the reference's own module ---------------------------------------------------------------------
def test_reference_kvnet_dgf_gradients_with_mirrors():
    """One training step of the reference's KVNET(refineNet_name='DGF'): the D-Net / K-Net parameters get their loss
    gradient only through depth_val_regression (models/KVNET.py:129,176) and the propagated prior (resample_vol_cuda).
    With the mirrors patched in, every parameter gets a gradient, and it matches the unpatched reference."""
    res = harness.run_reference_driver('grad', 'geometry', timeout=1200)
    harness.parity_dump('grad', 'kvnet_dgf', res)
    assert not res['missing'], res['missing']
    assert res['restored'] is True                  # the reference's own functions are back after the patched run
    params = res['params']
    assert len(params) > 200
    la, lb, lp = res['loss']
    assert abs(lb - la) <= 1e-6 * abs(la) and abs(lp - la) <= 1e-5 * abs(la)
    # Without the regression backward (the mirror before f-5) only R-Net gets a gradient: the silent loss this guards.
    assert res['with_grad_without_f5'] and all(n.startswith('r_net.') for n in res['with_grad_without_f5'])
    # Gate. Two unpatched runs differ by cuDNN's run-to-run floor only (2.5e-6 of the largest gradient on an H100): their
    # forwards are bit-identical. The mirrors' forwards are not bit-identical to the reference's GPU ops: the sweep, for one,
    # sums in another order (DESIGN 4.1). Those rounding differences pass through train-mode BatchNorm and the whole
    # backward: measured 2.4e-3 of the largest gradient, 4.9e-3 of a parameter's own largest, on every parameter alike.
    # A missing gradient term changes the affected parameters by O(1) (the check above). Gate: 2e-2 of each parameter's
    # largest gradient, and for parameters whose true gradient is zero up to rounding (the guided filter does not change
    # when a constant is added to the guide, so r_net.feature_ext.2.bias has none) 2e-5 of the largest gradient overall.
    gmax = max(p['max'] for p in params.values())
    rel_floor = max(p['floor'] for p in params.values()) / gmax
    assert rel_floor <= 1e-4, rel_floor
    for n, p in params.items():
        if p['max'] >= 1e-4 * gmax:
            assert p['dev'] <= 2e-2 * p['max'], (n, p)
        else:
            assert p['dev'] <= 2e-5 * gmax, (n, p, gmax)
