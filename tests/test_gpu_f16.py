"""conv_math='f16' (single fp16 products, fp32 accumulation) on the GPU.

 * Kernel: every convolution shape the engine runs, with x_lo = NULL, against a float64 convolution of the RN_f16-rounded
   operands. The operands are identical, so only the fp32 summation order differs: the 6e-6 gate of test_gpu_conv_h2.py
   (relative to the output scale). Also the BatchNorm sums, a pair output with y_lo = NULL (hi = RN_f16 of the fp32
   result, pad channels zero), the affine epilogue with a 22-bit pair residual, and the K-Net volume, the BatchNorm pass and
   the split pass with a NULL lo.
 * Engine against the reference with its convolutions' operands rounded to fp16 (tests/golden/make_golden_f16.py): first
   windows and re-seeded steps within max(f16x3's gate, 2 F), free-running stream steps within max(f16x3's gate, 4 F), F the
   pinned deviation of the f16 oracle (tests/oracle_f16.py) from that reference, on probabilities and expected depth (for a
   steady step the largest of the case's steady steps). Against
   the plain fp32 reference: at most twice the emulated reference's own deviation plus that gate.
 * f16x3 -> f16 -> f16x3 on one module gives bit-identical f16x3 outputs; a steady frame launches the same kernels as in
   f16x3 and the pool is smaller; the reference's unmodified test() runs with conv_math='f16'.
Measured deviations are written to $NRGBD_PARITY_DIR/parity_f16.json when that variable is set.
"""
import contextlib
import ctypes
import io
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from oracle import planesweep_oracle as O
from tests import cases
from tests import cases_f16 as CF
from tests.conftest import ROOT, maxabs

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
TOL_REL = 6e-6
G16X3_FIRST = 1e-4        # f16x3's gates: first windows (probability), test_gpu_twin.py / test_gpu_eval.py
G16X3_STEADY = 3e-4       # the largest of f16x3's steady-step gates at these shapes (twice the pinned fp32 floor)
G16X3_DEPTH_MM = 1.0


def _dump(key, row):
    d = os.environ.get('NRGBD_PARITY_DIR')
    if not d:
        return
    try:
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, 'parity_f16.json')
        cur = json.load(open(path)) if os.path.exists(path) else {}
        cur[key] = row
        with open(path, 'w') as f:
            json.dump(cur, f, indent=1, sort_keys=True)
    except OSError:
        pass


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def r16(a):
    return torch.from_numpy(np.asarray(a, np.float32)).half().double()


# ---- kernel ------------------------------------------------------------------------------------------------------------
CONV_SHAPES = {
    # name: (N, Cin, Cout, D or None, H, W, k, stride, pad, dilation)
    'halo_3x3_32': (2, 32, 32, None, 30, 41, 3, 1, 1, 1),
    'halo_3x3_64_120rows': (1, 64, 64, None, 120, 40, 3, 1, 1, 1),
    'halo_3x3_128': (1, 128, 128, None, 24, 40, 3, 1, 1, 1),
    'lastconv_320_128': (1, 320, 128, None, 20, 36, 3, 1, 1, 1),
    'dilated_d2_128': (1, 128, 128, None, 22, 30, 3, 1, 2, 2),
    'strided_s2_32_64': (2, 32, 64, None, 33, 47, 3, 2, 1, 1),
    'pointwise_s2_64_128': (1, 64, 128, None, 40, 52, 1, 2, 0, 1),
    'rnet_80_80': (1, 80, 80, None, 26, 34, 3, 1, 1, 1),
    'cout_131': (1, 35, 131, None, 17, 29, 3, 1, 1, 1),
    'conv3d_64_64': (1, 64, 64, 9, 14, 18, 3, 1, 1, 1),
    'conv3d_cin10_pad32': (1, 10, 64, 8, 12, 20, 3, 1, 1, 1),
}


@pytest.mark.parametrize('name', list(CONV_SHAPES))
def test_single_product_conv_shapes(name):
    from neuralrgbd_b200 import convops
    N, Cin, Cout, D, H, W, k, s, p, dl = CONV_SHAPES[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    shp = (N, Cin) + ((D,) if D else ()) + (H, W)
    x = rng.standard_normal(shp).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin) + ((3,) if D else ()) + (k, k)) / math.sqrt(Cin * k * k)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32) if not D else None
    y, st = convops.conv_h2(T(x), T(w), None if b is None else T(b), s, p, dl, want_stats=True, single=True)
    if D:
        ref = Fn.conv3d(r16(x), r16(w), None, 1, 1)
    else:
        ref = Fn.conv2d(r16(x), r16(w), torch.from_numpy(b).double(), s, p, dl)
    ref = ref.numpy()
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= TOL_REL, rel_err(y.cpu().numpy(), ref)
    # BatchNorm sums of the stored fp32 values (as test_gpu_conv_h2.py)
    yv = y.cpu().numpy().astype(np.float64)
    red = (0,) + tuple(range(2, yv.ndim))
    st = st.cpu().numpy()
    assert np.abs(st[0] - yv.sum(axis=red)).max() <= 1e-6 * np.abs(yv).max() * yv[:, 0].size + 1e-5
    assert np.allclose(st[1], np.square(yv).sum(axis=red), rtol=2e-5, atol=1e-3)
    # and the f16x3 kernel on the same inputs is the 22-bit product: the two modes differ by the operand rounding only
    y3 = convops.conv_h2(T(x), T(w), None if b is None else T(b), s, p, dl).cpu().numpy()
    assert rel_err(yv, y3) > 1e-5


def test_single_product_transposed_k4s2():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(3)
    for Cin, Cout, H, W in ((80, 16, 30, 40), (48, 64, 17, 23)):
        x = rng.standard_normal((1, Cin, H, W)).astype(np.float32)
        w = (rng.standard_normal((Cin, Cout, 4, 4)) / math.sqrt(Cin * 4)).astype(np.float32)
        b = rng.standard_normal(Cout).astype(np.float32)
        y = convops.conv_transpose2d_h2(T(x), T(w), T(b), leaky=True, single=True).cpu().numpy()
        ref = Fn.leaky_relu(Fn.conv_transpose2d(r16(x), r16(w), torch.from_numpy(b).double(), 2, 1), 0.01).numpy()
        assert y.shape == ref.shape and rel_err(y, ref) <= TOL_REL


def test_single_product_tap_gather():
    """The 27-output pointwise convolution in front of nrgbd_tap_gather_sum (K-Net's last layer)."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(4)
    x = rng.standard_normal((1, 64, 10, 12, 20)).astype(np.float32)
    w = (rng.standard_normal((1, 64, 3, 3, 3)) / math.sqrt(64 * 27)).astype(np.float32)
    y = convops.conv_cout1_h2(T(x), T(w), single=True).cpu().numpy()
    ref = Fn.conv3d(r16(x), r16(w), None, 1, 1).numpy()
    assert y.shape == ref.shape and rel_err(y, ref) <= TOL_REL


def test_single_product_pair_output_hi_only():
    """y_lo = NULL: hi is RN_f16 of the fp32 result of the same kernel, every channel written, pad channels zero."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(5)
    x = rng.standard_normal((1, 80, 26, 34)).astype(np.float32)
    w = (rng.standard_normal((72, 80, 3, 3)) / math.sqrt(720)).astype(np.float32)
    b = rng.standard_normal(72).astype(np.float32)
    val, yh, yl = convops.conv_h2_pair_out(T(x), T(w), T(b), 1, 1, 1, leaky=True, single=True)
    assert yl is None and yh.shape[-1] == 96
    y = convops.conv_h2(T(x), T(w), T(b), 1, 1, 1, leaky=True, single=True)
    assert torch.equal(val, y.half().float())
    assert torch.isfinite(yh.float()).all() and (yh[..., 72:] == 0).all()
    ref = Fn.leaky_relu(Fn.conv2d(r16(x), r16(w), torch.from_numpy(b).double(), 1, 1), 0.01).numpy()
    assert rel_err(val.cpu().numpy(), ref) <= 2.0 ** -11 + TOL_REL


@pytest.mark.parametrize('pair_out', [False, True])
def test_single_product_affine_with_pair_residual(pair_out):
    """Eval-mode convbn in one pass: single products, the 22-bit pair residual, ReLU; fp32 or hi-only output."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(6)
    x = rng.standard_normal((1, 64, 8, 14, 20)).astype(np.float32)
    w = (rng.standard_normal((64, 64, 3, 3, 3)) / math.sqrt(64 * 27)).astype(np.float32)
    res = rng.standard_normal((1, 64, 8, 14, 20)).astype(np.float32)
    sc = (rng.rand(64) + 0.5).astype(np.float32); sh = rng.standard_normal(64).astype(np.float32)
    out = convops.conv_h2_affine(T(x), T(w), T(sc), T(sh), 1, 1, 1, res=T(res), res_pair=True, relu=True, pair_out=pair_out, single=True)
    conv = Fn.conv3d(r16(x), r16(w), None, 1, 1).numpy()
    ref = np.maximum(conv * sc.reshape(1, -1, 1, 1, 1) + sh.reshape(1, -1, 1, 1, 1) + res, 0)
    if pair_out:
        val, yh, yl = out
        assert yl is None and torch.isfinite(yh.float()).all()
        assert rel_err(val.cpu().numpy(), ref) <= 2.0 ** -11 + TOL_REL
    else:
        assert rel_err(out.cpu().numpy(), ref) <= TOL_REL


def test_split_bn_and_volume_with_null_lo():
    """nrgbd_split_f16_pair, nrgbd_bn_apply_stats_pair and nrgbd_knet_input_volume_pair with lo = NULL write the hi of the
    pair they write with a lo (bit for bit) and nothing else."""
    from neuralrgbd_b200 import _lib, convops, synth
    from neuralrgbd_b200._lib import ptr, check
    L = _lib.lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    F = ctypes.c_float
    x = torch.randn(4096, device=dev) * 3
    x[:4] = torch.tensor([70000.0, -1e6, 1e-7, 65519.0])
    h1, l1 = convops.split_f16_pair(x)
    h0, l0 = convops.split_f16_pair(x, single=True)
    assert l0 is None and torch.equal(h0, h1) and torch.equal(h0, x.clamp(-65504, 65504).half())
    # BatchNorm pass with a pair residual, hi-only output
    n, C = 3000, 64
    xk = torch.randn(n, C, device=dev)
    s64 = torch.stack([xk.double().sum(0), (xk.double() ** 2).sum(0)]).contiguous()
    g = torch.rand(C, device=dev) + 0.5; bb = torch.randn(C, device=dev)
    rh, rl = convops.split_f16_pair(torch.randn(n, C, device=dev))
    outs = []
    for single in (False, True):
        yh = torch.full((n, C), float('nan'), device=dev, dtype=torch.float16)
        yl = None if single else torch.full((n, C), float('nan'), device=dev, dtype=torch.float16)
        check(L.nrgbd_bn_apply_stats_pair(ptr(xk), ctypes.c_void_p(s64.data_ptr()), float(n), ptr(g), ptr(bb), F(1e-5), None, None, F(0.1),
                                          None, ptr(rh), ptr(rl), 1, n, C, C, None, ptr(yh), ptr(yl), None, st))
        outs.append(yh)
    assert torch.equal(outs[0], outs[1])
    # K-Net input volume rows (CK = 32, V = 2: 10 channels, the rest zero)
    V, D, h, w = 2, 8, 24, 32
    hw = h * w
    rng = np.random.RandomState(7)
    rgb = torch.randn(V, hw, 4, device=dev); refq = torch.randn(hw, 4, device=dev)
    bv = torch.log_softmax(torch.randn(hw, D, device=dev), 1).contiguous(); prior = torch.log_softmax(torch.randn(hw, D, device=dev), 1).contiguous()
    exts = synth.camera_track(rng, V + 1)
    poses, _ = synth.window_rel_poses(exts, 1, 1)
    R = T(np.ascontiguousarray(poses[:, :3, :3])); t = T(np.ascontiguousarray(poses[:, :3, 3]))
    K = torch.tensor([[w / 2 / (320 / 585.), 0, w / 2], [0, h / 2 / (240 / 585.), h / 2], [0, 0, 1]], dtype=torch.float32, device=dev)
    xs = (np.arange(w) + .5) / w * 2 - 1; ys = (np.arange(h) + .5) / h * 2 - 1
    rays = T(np.stack([np.tile(320 / 585. * xs[None], (h, 1)), np.tile(240 / 585. * ys[:, None], (1, w)), np.ones((h, w))]).reshape(3, -1).astype(np.float32))
    dpl = T(synth.d_candidates(D).astype(np.float32)); ws = torch.empty(V * 12, device=dev)
    vols = []
    for single in (False, True):
        vh = torch.full((D, hw, 32), float('nan'), device=dev, dtype=torch.float16)
        vl = None if single else torch.full((D, hw, 32), float('nan'), device=dev, dtype=torch.float16)
        check(L.nrgbd_knet_input_volume_pair(ptr(rgb), ptr(refq), ptr(bv), ptr(prior), V, D, h, w, 32, ptr(K), ptr(R), ptr(t), ptr(rays),
                                             ptr(dpl), F(w / 2), F(h / 2), ptr(ws), None, ptr(vh), ptr(vl), st))
        vols.append(vh)
    assert torch.equal(vols[0], vols[1]) and (vols[1][..., 10:] == 0).all()


# ---- engine ------------------------------------------------------------------------------------------------------------
def _gold():
    return np.load(os.path.join(ROOT, 'tests', 'golden', 'f16_outputs.npz'))


def _pin():
    return json.load(open(os.path.join(ROOT, 'tests', 'golden', 'PINNING_f16.json')))['cases']


def _cam_t(cam):
    return dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']), intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']))


def _model(c, cam_t, conv_math):
    from neuralrgbd_b200.models.KVNET import KVNET
    with contextlib.redirect_stdout(io.StringIO()):
        m = KVNET(feature_dim=64, cam_intrinsics=cam_t, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                  d_upsample_ratio_KV_net=None, t_win_r=c['t_win_r'])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in CF.state_dict(c).items()}, strict=True)
    m = m.to(dev)
    m.conv_math = conv_math
    m.train(CF.MODE[c['name']] == 'train')
    return m


class _Recorder(torch.nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model
        self.last = None

    def forward(self, **kw):
        self.last = self.model(**kw)
        return self.last


def _run(c, cam_t, conv_math):
    """The case's steps through the package's test() (re-seeded or free-running as the fixture) -> list of 4 outputs."""
    from neuralrgbd_b200.test_utils import test_KVNet
    rec = _Recorder(_model(c, cam_t, conv_math))
    outs, prior = [], None
    for k in range(c['n_steps']):
        if k and c['name'] not in CF.FREE_RUNNING:
            prior = T(CF.reseed_prior(c['name'], k))
        ref_f, src_f, poses = cases.window(c, c['t_win_r'] + k)
        _, nxt = test_KVNet.test(rec, c['d'], [cam_t], c['t_win_r'], [{'img': T(ref_f)}],
                                 [[{'img': T(src_f[0, v:v + 1])} for v in range(src_f.shape[1])]], T(poses), prior if k else None,
                                 R_net=False)
        outs.append([a.cpu().numpy() for a in rec.last])
        prior = nxt
    return outs


def _floor(pin, name, k, nm, key):
    """F of step k: the first window's own; for a steady step the largest of the case's steady steps (as test_gpu_twin.py: one
    step's floor is one sample of that noise, and a free-running step carries the drift of the steps before it)."""
    ks = [k] if k == 0 else [j for j in range(1, 64) if 'f16/%s/step%d' % (name, j) in pin]
    return max(pin['f16/%s/step%d' % (name, j)]['oracle_vs_f16'][nm][key] for j in ks)


def _depth(a, d):
    p = np.exp(a.astype(np.float64))
    return (p * np.asarray(d, np.float64).reshape(1, -1, 1, 1)).sum(1)


@pytest.mark.parametrize('name', CF.F16_CASES)
def test_engine_f16_vs_emulated_reference(name):
    gold, pin = _gold(), _pin()
    c = CF.f16_case(name)
    cam_t = _cam_t(CF.cam(O.make_cam_intrinsics, c))
    outs = _run(c, cam_t, 'f16')
    rows = {}
    for k, full in enumerate(outs):
        kk = 'f16/%s/step%d' % (name, k)
        p = pin[kk]
        mult = 4.0 if (name in CF.FREE_RUNNING and k) else 2.0
        row = {}
        for nm, a in zip(CF.NAMES4, full):
            assert np.isfinite(a).all(), (kk, nm)
            if nm not in CF.STORED[k == 0]:
                continue
            s = np.exp(cases.subsample_to(a, CF.SUB_LIMIT))
            row[nm] = maxabs(s, np.exp(gold['%s/f16/%s' % (kk, nm)]))
            row[nm + '_gate'] = max(G16X3_FIRST if k == 0 else G16X3_STEADY, mult * _floor(pin, name, k, nm, 'prob'))
            row[nm + '_fp32'] = maxabs(s, np.exp(gold['%s/fp32/%s' % (kk, nm)]))
            row[nm + '_fp32_gate'] = 2.0 * p['f16_vs_fp32'][nm]['prob'] + row[nm + '_gate']
            row[nm + '_ref_f16_vs_fp32'] = p['f16_vs_fp32'][nm]['prob']
            row[nm + '_ref_tf32_vs_fp32'] = p['tf32_vs_fp32'][nm]['prob']
        dep = cases.subsample_to(_depth(full[3], c['d']), CF.DEPTH_LIMIT)
        row['depth_mm'] = 1000.0 * maxabs(dep, gold[kk + '/f16/depth'])
        row['depth_gate_mm'] = max(G16X3_DEPTH_MM, mult * _floor(pin, name, k, 'DPV', 'depth_mm'))
        row['depth_fp32_mm'] = 1000.0 * maxabs(dep, gold[kk + '/fp32/depth'])
        row['depth_fp32_gate_mm'] = 2.0 * p['f16_vs_fp32']['DPV']['depth_mm'] + row['depth_gate_mm']
        row['depth_ref_tf32_vs_fp32_mm'] = p['tf32_vs_fp32']['DPV']['depth_mm']
        rows['step%d' % k] = row
    _dump('engine/%s' % name, rows)
    print(json.dumps(rows, indent=1))
    msg = json.dumps(rows)
    for r in rows.values():
        for nm in CF.NAMES4:
            if nm in r:
                assert r[nm] <= r[nm + '_gate'], msg
                assert r[nm + '_fp32'] <= r[nm + '_fp32_gate'], msg
        assert r['depth_mm'] <= r['depth_gate_mm'] and r['depth_fp32_mm'] <= r['depth_fp32_gate_mm'], msg


def _forward(m, c, cam_t, step, prior):
    ref_f, src_f, poses = cases.window(c, c['t_win_r'] + step)
    with torch.no_grad():
        return [t.clone() for t in m(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam_t],
                                     BV_predict=None if prior is None else T(prior))]


def test_f16x3_unchanged_after_f16():
    """One module in .eval() (no atomics: deterministic): f16x3, then f16, then f16x3 again - the f16x3 outputs of a first
    window and a steady step are bit-identical to the first run's, and f16 differs from them."""
    c = CF.f16_case('eval_256_d16')
    cam_t = _cam_t(CF.cam(O.make_cam_intrinsics, c))
    prior = CF.reseed_prior('eval_256_d16', 1)
    m = _model(c, cam_t, 'f16x3')
    runs = {}
    for i, mode in enumerate(['f16x3', 'f16', 'f16x3']):
        m.conv_math = mode
        runs[i] = _forward(m, c, cam_t, 0, None) + _forward(m, c, cam_t, 1, prior)
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[2]))
    assert not torch.equal(runs[0][3], runs[1][3]) and not torch.equal(runs[0][7], runs[1][7])


def _launches(c, cam_t, conv_math, prior):
    from torch.profiler import profile, ProfilerActivity
    from neuralrgbd_b200 import _lib
    m = _model(c, cam_t, conv_math)
    _forward(m, c, cam_t, 0, None)
    _forward(m, c, cam_t, 1, prior)
    ent = next(iter(m._engines.values()))
    _lib.lib().nrgbd_kvnet_set_option(ent['h'], b'use_graph', 0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _forward(m, c, cam_t, 1, prior)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    counts = {k: sum(k in n for n in names) for k in ('conv_igemm_kernel', 'conv_wg_kernel', 'split_f16_pair_kernel', 'bn_apply_stats_kernel')}
    counts['kernels'] = len([n for n in names if 'Memset' not in n and 'Memcpy' not in n])
    return counts


def test_f16_takes_the_f16x3_path():
    """A steady 256x256 frame launches the same kernels in f16 as in f16x3: the same tensor-core convolutions, fp32-path
    convolutions, split passes and BatchNorm passes."""
    c = CF.f16_case('eval_256_d16')
    cam_t = _cam_t(CF.cam(O.make_cam_intrinsics, c))
    prior = CF.reseed_prior('eval_256_d16', 1)
    a, b = _launches(c, cam_t, 'f16x3', prior), _launches(c, cam_t, 'f16', prior)
    _dump('launches', {'f16x3': a, 'f16': b})
    assert a == b, (a, b)
    assert a['conv_wg_kernel'] > 0 and a['conv_igemm_kernel'] == 1


def test_f16_workspace_smaller_at_c2_c3():
    """The pool after a first window and a steady step at 640x480, D = 64, V = 4 holds no lo half for tensors only
    convolutions read: strictly smaller in f16 than in f16x3."""
    from neuralrgbd_b200 import _lib
    c = CF.f16_case('c2_640x480_d64')
    cam_t = _cam_t(CF.cam(O.make_cam_intrinsics, c))
    prior = CF.reseed_prior('c2_640x480_d64', 1)
    ws = {}
    for mode in ('f16x3', 'f16'):
        m = _model(c, cam_t, mode)
        _forward(m, c, cam_t, 0, None)
        _forward(m, c, cam_t, 1, prior)
        ent = next(iter(m._engines.values()))
        ws[mode] = _lib.lib().nrgbd_kvnet_workspace_bytes(ent['h'])
        del m
        torch.cuda.empty_cache()
    _dump('workspace_bytes', ws)
    assert 0 < ws['f16'] < ws['f16x3'], ws


def test_bad_conv_math_lists_all_modes():
    c = CF.f16_case('r1_256_d16')
    cam_t = _cam_t(CF.cam(O.make_cam_intrinsics, c))
    m = _model(c, cam_t, 'f8')
    with pytest.raises(ValueError, match="'fp32', 'tf32x3', 'f16x3' or 'f16'"):
        _forward(m, c, cam_t, 0, None)


def test_reference_test_runs_unmodified_in_f16():
    from oracle import fetch_reference
    ref_code = fetch_reference.code_dir()
    assert ref_code, 'no copy of the reference: oracle/_ref is made by __graft_entry__.build() (oracle/fetch_reference.py)'
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'dropin_f16_driver.py'), ref_code],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    out = json.loads(r.stdout.strip().splitlines()[-1])
    _dump('dropin', out)
    pin = _pin()
    assert out['class'] == 'neuralrgbd_b200.models.KVNET' and out['conv_math'] == 'f16'
    assert len(out['steps']) == 2 and all(s['prior_finite'] for s in out['steps']), out
    for k, s in enumerate(out['steps']):
        F = pin['f16/r1_256_d16/step%d' % k]['oracle_vs_f16']['DPV' if k else 'BV_cur']['prob']
        assert s['DPV'] <= max(G16X3_FIRST if k == 0 else G16X3_STEADY, 2.0 * F), out
