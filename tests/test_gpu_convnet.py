"""GPU parity of the conv-stack kernels and of the whole-frame engine (SURVEY §8 a4-a10).

Op level: each kernel against the numpy oracle (im2col + sgemm) on seeded inputs.
Engine level: KVNET.forward (both branches) and the streaming test() loop against (i) the
committed outputs of the live reference and (ii) the oracle. Tolerances on PROBABILITIES for
pipeline outputs (DESIGN.md 'tolerance domain'): D-Net / R-Net DPVs 1e-4, K-Net DPV 5e-4 (the
measured fp32 noise floor between the reference and an independent fp32 implementation is
1.6e-4, tests/golden/PINNING.json), expected depth 1 mm.
"""
import io
import contextlib
import math

import numpy as np
import pytest
import torch

from oracle import planesweep_oracle as O
from oracle import kvnet_oracle as N
from tests import cases, harness
from tests.conftest import maxabs
from tests.harness import rel_err

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731


@pytest.mark.parametrize('cfg', [
    dict(N=2, Cin=3, Cout=32, H=40, W=56, k=3, s=2, p=1, d=1),      # firstconv.0
    dict(N=2, Cin=32, Cout=32, H=33, W=47, k=3, s=1, p=1, d=1),     # ragged tile edges
    dict(N=1, Cin=64, Cout=128, H=24, W=40, k=1, s=1, p=0, d=1),    # layer3 downsample
    dict(N=2, Cin=32, Cout=64, H=32, W=48, k=1, s=2, p=0, d=1),     # layer2 downsample (stride 2, 1x1)
    dict(N=1, Cin=128, Cout=128, H=20, W=28, k=3, s=1, p=2, d=2),   # layer4 dilation 2
    dict(N=1, Cin=67, Cout=67, H=24, W=36, k=3, s=1, p=1, d=1),     # R-Net conv2 (odd channels)
    dict(N=1, Cin=320, Cout=128, H=16, W=24, k=3, s=1, p=1, d=1),   # lastconv.0
    dict(N=3, Cin=128, Cout=32, H=1, W=2, k=1, s=1, p=0, d=1),      # SPP branch conv on a 1x2 map
])
def test_conv2d_vs_oracle(cfg):
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(1)
    x = rng.standard_normal((cfg['N'], cfg['Cin'], cfg['H'], cfg['W'])).astype(np.float32)
    w = (rng.standard_normal((cfg['Cout'], cfg['Cin'], cfg['k'], cfg['k'])) / math.sqrt(cfg['Cin'] * cfg['k'] ** 2)).astype(np.float32)
    b = rng.standard_normal(cfg['Cout']).astype(np.float32)
    y, st = convops.conv(T(x), T(w), T(b), cfg['s'], cfg['p'], cfg['d'], leaky=True, want_stats=True)
    ref = N.leaky_relu(N.conv2d(x, w, b, cfg['s'], cfg['p'], cfg['d']))
    assert y.shape == ref.shape
    assert rel_err(y.cpu().numpy(), ref) <= 2e-6
    st = st.cpu().numpy()
    assert np.allclose(st[0], ref.sum(axis=(0, 2, 3), dtype=np.float64), rtol=1e-5, atol=1e-4)
    assert np.allclose(st[1], np.square(ref.astype(np.float64)).sum(axis=(0, 2, 3)), rtol=1e-5, atol=1e-4)


def test_conv3d_vs_oracle():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(2)
    for cin, cout in ((16, 64), (64, 64), (64, 1)):
        x = rng.standard_normal((1, cin, 9, 14, 18)).astype(np.float32)
        w = (rng.standard_normal((cout, cin, 3, 3, 3)) / math.sqrt(cin * 27)).astype(np.float32)
        y = convops.conv(T(x), T(w), None, 1, 1, 1)
        ref = N.conv3d(x, w)
        assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 2e-6


def test_conv_transpose2d_vs_oracle():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(3)
    for cin, cout, h, w_ in ((128, 64, 9, 13), (96, 64, 16, 20), (8, 5, 5, 7)):
        x = rng.standard_normal((1, cin, h, w_)).astype(np.float32)
        w = (rng.standard_normal((cin, cout, 4, 4)) / math.sqrt(cin * 4)).astype(np.float32)
        b = rng.standard_normal(cout).astype(np.float32)
        y = convops.conv_transpose2d(T(x), T(w), T(b), leaky=True)
        ref = N.leaky_relu(N.conv_transpose2d(x, w, b, 2, 1))
        assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 2e-6


def test_batchnorm_relu_residual_vs_oracle():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(4)
    x = (3.0 + 2.0 * rng.standard_normal((5, 32, 12, 20))).astype(np.float32)   # non-zero mean: E[x^2]-m^2 path
    w = np.zeros((32, 32, 1, 1), np.float32); w[np.arange(32), np.arange(32)] = 1.0   # identity conv to get stats
    g = rng.uniform(.5, 1.5, 32).astype(np.float32); b = rng.standard_normal(32).astype(np.float32)
    res = rng.standard_normal(x.shape).astype(np.float32)
    y, st = convops.conv(T(x), T(w), None, 1, 0, 1, want_stats=True)
    assert maxabs(y.cpu().numpy(), x) == 0.0
    out = convops.batch_norm(y, st, T(g), T(b), relu=True, residual=T(res))
    ref = N.relu(N.batch_norm(x, g, b)) + res
    assert maxabs(out.cpu().numpy(), ref) <= 5e-6
    # degenerate batch: 10 values per channel (SPP branch1 at 640x480: N=5, 1x2 map)
    x2 = rng.standard_normal((5, 32, 1, 2)).astype(np.float32)
    y2, st2 = convops.conv(T(x2), T(w), None, 1, 0, 1, want_stats=True)
    out2 = convops.batch_norm(y2, st2, T(g), T(b), relu=False)
    assert maxabs(out2.cpu().numpy(), N.batch_norm(x2, g, b)) <= 5e-6


def test_pool_and_upsample_vs_oracle():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(5)
    x = rng.standard_normal((2, 128, 64, 96)).astype(np.float32)
    for k in (64, 32, 16, 8, 4):
        assert maxabs(convops.avg_pool2d(T(x), k).cpu().numpy(), N.avg_pool2d(x, k)) <= 2e-6
    x3 = rng.standard_normal((2, 3, 37, 53)).astype(np.float32)       # floor semantics
    assert maxabs(convops.avg_pool2d(T(x3), 4).cpu().numpy(), N.avg_pool2d(x3, 4)) <= 2e-6
    for (hi, wi) in ((1, 2), (2, 3), (8, 12)):
        s = rng.standard_normal((2, 32, hi, wi)).astype(np.float32)
        assert maxabs(convops.upsample_bilinear_ac(T(s), (64, 96)).cpu().numpy(), N.upsample_bilinear_ac(s, (64, 96))) <= 5e-6


def build_model(c, cam):
    from neuralrgbd_b200.models.KVNET import KVNET
    with contextlib.redirect_stdout(io.StringIO()):
        m = KVNET(feature_dim=64, cam_intrinsics=cam, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                  d_upsample_ratio_KV_net=None, t_win_r=2, if_refined=True)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in c['sd'].items()})
    return m.to(dev)


@pytest.mark.parametrize('conv_math', ['fp32', 'tf32x3', 'f16x3'])
@pytest.mark.parametrize('name', cases.KVNET_CASES)
def test_kvnet_forward_streaming_vs_reference(golden, name, conv_math):
    """KVNET.forward first-window + steady branches and the streaming test() loop against the
    live-reference fixtures; each step is fed the REFERENCE's prior so deviations do not compound."""
    from neuralrgbd_b200.test_utils.test_KVNet import test as kv_test
    c = cases.kvnet_case(name)
    cam = harness.cam_tensors(cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4))
    base = build_model(c, cam)
    base.conv_math = conv_math        # exact fp32 CUDA-core path / wgmma 3xTF32 tensor-core path: same gates
    model = torch.nn.DataParallel(base, device_ids=[0])      # as test_KVNet.py:163
    n_steps = len(c['frames']) - 4
    bv_pred = None
    for step in range(n_steps):
        ref_f, src_f, poses = cases.window(c, 2 + step)
        key = 'kvnet/%s/step%d' % (name, step)
        with torch.no_grad():
            full = model(ref_frame=T(ref_f), src_frames=T(src_f), src_cam_poses=T(poses), BatchIdx=torch.zeros(1),
                         cam_intrinsics=[cam], BV_predict=bv_pred)
        tol = {'dmap_cur_refined': 1e-4, 'dmap_refined': 1e-4 if bv_pred is None else 5e-4, 'BV_cur': 1e-4,
               'DPV': 1e-4 if bv_pred is None else 5e-4}
        for nm, a in zip(['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV'], full):
            a = a.cpu().numpy()
            r = golden['%s/%s' % (key, nm)]
            assert maxabs(np.exp(cases.subsample(a)), np.exp(r)) <= tol[nm], (key, nm)
            st = cases.stats(np.exp(a)); rs = cases.stats(np.exp(r))
            assert np.isfinite(a).all()
        if bv_pred is None:
            assert full[0] is full[1] and full[2] is full[3]          # KVNET.py:138-140 returns the same tensors
        # expected depth within 1 mm of the reference's (both from the sub-sampled DPV grid)
        dep = O.depth_val_regression(cases.subsample(full[3].cpu().numpy()), c['d'])
        dep_ref = O.depth_val_regression(golden[key + '/DPV'], c['d'])
        assert maxabs(dep, dep_ref) * 1000.0 <= 1.0
        from neuralrgbd_b200.mutils import misc
        dep_dev = misc.depth_val_regression(full[3], c['d']).cpu().numpy()
        assert maxabs(dep_dev, O.depth_val_regression(full[3].cpu().numpy(), c['d'])) * 1000.0 <= 0.01
        # the reference's inference step: forward + propagation
        Ref_Dats = [{'img': T(ref_f)}]
        Src_Dats = [[{'img': T(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]]
        kv_dpv, bv_next = kv_test(model, c['d'], [cam], 2, Ref_Dats, Src_Dats, T(poses), bv_pred, R_net=False)
        assert maxabs(kv_dpv.cpu().numpy(), full[3].cpu().numpy()) == 0.0      # deterministic
        r_next = golden[key + '/BV_predict_next']
        got_next = cases.subsample(bv_next.cpu().numpy())
        # log-space values down to -1000: compare probabilities, and logs where the reference is > -20
        assert maxabs(np.exp(got_next), np.exp(r_next)) <= 5e-4
        if step < n_steps - 1:
            bv_pred = T(golden[key + '/BV_predict_next_full'])
    # NaN prior takes the first-window branch (KVNET.py:142)
    ref_f, src_f, poses = cases.window(c, 2)
    nanp = torch.full((1, c['D'], c['H'] // 4, c['W'] // 4), float('nan'), device=dev)
    with torch.no_grad():
        a = model(ref_frame=T(ref_f), src_frames=T(src_f), src_cam_poses=T(poses), BatchIdx=torch.zeros(1),
                  cam_intrinsics=[cam], BV_predict=nanp)
        b = model(ref_frame=T(ref_f), src_frames=T(src_f), src_cam_poses=T(poses), BatchIdx=torch.zeros(1),
                  cam_intrinsics=[cam], BV_predict=None)
    assert torch.equal(a[3], b[3]) and torch.equal(a[0], b[0])


@pytest.mark.parametrize('conv_math', ['fp32', 'tf32x3', 'f16x3'])
def test_kvnet_vs_oracle_first_window(conv_math):
    """Engine vs the numpy oracle on a fresh seed (not in the fixtures)."""
    c = cases.kvnet_case('kvnet_256x320_d8')
    cam_np = cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4)
    model = build_model(c, harness.cam_tensors(cam_np))
    model.conv_math = conv_math
    ref_f, src_f, poses = cases.window(c, 3)
    with torch.no_grad():
        got = model(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[harness.cam_tensors(cam_np)], BV_predict=None)
    orc = N.kvnet_forward(c['sd'], ref_f, src_f, poses, cam_np, c['d'], c['sigma'])
    assert maxabs(np.exp(got[2].cpu().numpy()), np.exp(orc[2])) <= 1e-4
    assert maxabs(np.exp(got[0].cpu().numpy()), np.exp(orc[0])) <= 1e-4


@pytest.mark.parametrize('conv_math', ['fp32', 'tf32x3', 'f16x3', 'f16'])
def test_kvnet_load_state_dict_after_forward(conv_math):
    """New weights loaded into a module whose engine has run reach every packed copy of them: the next K-Net step
    matches a fresh module built with those weights (the f16 modes keep K-Net's last layer in a second, per-tap packing)."""
    c = cases.kvnet_case('kvnet_256_d16')
    cam = harness.cam_tensors(cases.cam_for(O.make_cam_intrinsics, c['W'] // 4, c['H'] // 4))
    rng = np.random.RandomState(11)
    sd_b = {k: (v * (1 + 0.1 * rng.standard_normal(v.shape))).astype(v.dtype) if v.dtype.kind == 'f' else v
            for k, v in ((k, np.asarray(v)) for k, v in c['sd'].items())}
    ref_f, src_f, poses = cases.window(c, 2)

    def dpv(m, prior):
        with torch.no_grad():
            return m(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam], BV_predict=prior)[3]
    model = build_model(c, cam)
    model.conv_math = conv_math
    prior = dpv(model, None).clone()                 # first window with state dict A
    before = dpv(model, prior).cpu().numpy()         # K-Net step with A
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd_b.items()})
    got = dpv(model, prior).cpu().numpy()
    fresh = build_model(dict(c, sd=sd_b), cam)
    fresh.conv_math = conv_math
    want = dpv(fresh, prior).cpu().numpy()
    # two identical modules agree to the rounding of the BatchNorm sums' double-precision atomics, far below the K-Net gate
    # (5e-4); the change of weights moves the DPV by far more
    assert maxabs(np.exp(got), np.exp(want)) <= 1e-5
    assert maxabs(np.exp(before), np.exp(want)) > 1e-3


def test_engine_rejects_bad_shapes():
    from neuralrgbd_b200 import _lib
    import ctypes
    L = _lib.lib()
    h = ctypes.c_void_p()
    assert L.nrgbd_kvnet_create(250, 256, 16, 4, 64, 64, ctypes.c_float(10.), 0, ctypes.byref(h)) != 0   # not /4
    assert L.nrgbd_kvnet_create(128, 256, 16, 4, 64, 64, ctypes.c_float(10.), 0, ctypes.byref(h)) != 0   # H/4 < 64
    assert b'64' in L.nrgbd_last_error()
