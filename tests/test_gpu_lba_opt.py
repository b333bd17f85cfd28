"""GPU: the device LBA pose optimiser (csrc/lba_opt.cu behind neuralrgbd_b200.ICP.opt_pose_numerical) against the unmodified
reference's local_BA_direct(_parallel) (tests/golden/lba_opt_outputs.npz) and the numpy oracle's pinned deviations
(PINNING_lba_opt.json): one iteration from every recorded reference state, full free-running runs, run-to-run
reproducibility, convergence at the docs/LBA.md size, launches per call and the drop-in on an unmodified checkout."""
import contextlib
import ctypes
import io
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cases
from tests import cases_lba_opt as LC
from tests.conftest import ROOT

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
GOLD = os.path.join(ROOT, 'tests', 'golden')


@pytest.fixture(scope='module')
def gold():
    return np.load(os.path.join(GOLD, 'lba_opt_outputs.npz'))


@pytest.fixture(scope='module')
def pin():
    return json.load(open(os.path.join(GOLD, 'PINNING_lba_opt.json')))['cases']


def cam_torch(cam):
    c = dict(cam)
    c['unit_ray_array_2D'] = torch.from_numpy(cam['unit_ray_array_2D'])
    c['intrinsic_M_cuda'] = torch.from_numpy(cam['intrinsic_M_cuda'])
    return c


def run(c, on_gpu=True, fn=None):
    from neuralrgbd_b200.ICP import opt_pose_numerical as M
    T = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)) if on_gpu else torch.from_numpy      # noqa: E731
    fn = fn or (M.local_BA_direct_parallel if c['entry'] == 'parallel' else M.local_BA_direct)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        poses = fn(T(c['ref']), [T(s) for s in c['srcs']], T(c['dmap']), T(c['conf']), [cam_torch(k) for k in c['cams']], c['dw_scales'],
                   list(c['poses_init']), c['max_iter'], c['step'], c['opt_vars'])
    return np.stack([p.numpy() for p in poses]), buf.getvalue().splitlines()


LINE = re.compile(r'^opt_pose\(\): scale=(\d), iter (\d+)/(\d+), d_loss = (-?\d+\.\d{6})$')


@pytest.mark.parametrize('name', LC.LBA_OPT_CASES)
def test_one_iteration_from_every_reference_state(gold, pin, name):
    """(a) the state the reference held before each Adam step, one device iteration: gradients within max(2e-4, 4 x the
    oracle's) of the largest reference gradient, parameters within max(1e-6, 4 x the oracle's) of the reference's step."""
    from neuralrgbd_b200 import _lib
    from neuralrgbd_b200.ICP import opt_pose_numerical as M
    from neuralrgbd_b200.warping.homography import _cam_tensors
    from oracle import lba_opt_oracle as LO
    L = _lib.lib()
    c = LC.lba_opt_case(name)
    p = pin[name]
    V, S = len(c['srcs']), 3 * c['max_iter']
    names = [nm for nm in ('t', 'u') if name + '/g/' + nm in gold]
    mode = M._mode(c['opt_vars'])
    init = M.initial_state(c['poses_init'])
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    levels = LO.pyramid(c['ref'], c['srcs'], c['dmap'], c['conf'], c['dw_scales'])
    slot = {'t': (M._T, 21, 24, 30), 'u': (M._U, 15, 18, 27)}                        # param, m, v, gradient offsets
    g_err = {nm: 0.0 for nm in names}
    p_err = {nm: 0.0 for nm in names}
    for k in range(S):
        s = k // c['max_iter']
        ref, srcs, dm, cf = levels[s]
        h, w = dm.shape
        planes = torch.from_numpy(np.concatenate([ref.reshape(3, h, w), cf[None], dm[None]] + [x.reshape(3, h, w) for x in srcs])).to(dev)
        st = init.copy()
        for nm in names:
            off, mo, vo, _ = slot[nm]
            st[:, off:off + 3] = gold[name + '/p/' + nm][k]
            st[:, mo:mo + 3] = gold[name + '/m/' + nm][k]
            st[:, vo:vo + 3] = gold[name + '/v/' + nm][k]
        for v in range(V):
            st[v, M._R:M._R + 9] = M._unitq_to_rotation(st[v, M._U:M._U + 3]).reshape(9)
        state = torch.from_numpy(st).to(dev)
        losses = torch.empty(V, device=dev, dtype=torch.float64)
        ws = torch.empty(L.nrgbd_lba_pose_opt_workspace_bytes(V, h, w), device=dev, dtype=torch.uint8)
        K, rays = _cam_tensors(c['cams'][s], torch.device(dev))
        _lib.check(L.nrgbd_lba_pose_opt_scale(_lib.ptr(planes[0:3]), _lib.ptr(planes[3]), _lib.ptr(planes[4]), _lib.ptr(planes[5:]), _lib.ptr(K),
                                              _lib.ptr(rays), V, h, w, mode, 1.0 / ((V if c['entry'] == 'parallel' else 1) * 3 * h * w),
                                              c['step'] / 2 ** s, k, 1, _lib.ptr(state), ctypes.c_void_p(losses.data_ptr()),
                                              ctypes.c_void_p(ws.data_ptr()), stream))
        out = state.cpu().numpy()
        for nm in names:
            off, _, _, go = slot[nm]
            g_ref = gold[name + '/g/' + nm][k]
            g_err[nm] = max(g_err[nm], float(np.abs(out[:, go:go + 3] - g_ref).max() / np.abs(g_ref).max()))
            p_err[nm] = max(p_err[nm], float(np.abs(out[:, off:off + 3] - gold[name + '/p1/' + nm][k]).max()))
    for nm in names:
        assert g_err[nm] <= max(2e-4, 4 * p['grad_%s_rel' % nm]), (nm, g_err[nm])
        assert p_err[nm] <= max(1e-6, 4 * p['step_%s_maxabs' % nm]), (nm, p_err[nm])


@pytest.mark.parametrize('name', LC.LBA_OPT_CASES)
def test_full_run_matches_the_reference(gold, pin, name):
    """(b) free-running: final poses within max(2e-5, 4 x the oracle's deviation); the printed lines as the reference's."""
    c = LC.lba_opt_case(name)
    poses, lines = run(c)
    tol = max(2e-5, 4 * pin[name]['final_pose_maxabs'])
    assert np.abs(poses - gold[name + '/poses']).max() <= tol
    ref_lines = list(gold[name + '/printed'])
    assert len(lines) == len(ref_lines)
    for a, b in zip(lines, ref_lines):
        ma, mb = LINE.match(a), LINE.match(b)
        assert ma and mb, (a, b)
        assert ma.groups()[:3] == mb.groups()[:3]
        assert abs(float(ma.group(4)) - float(mb.group(4))) <= 5e-3 + 0.02 * abs(float(mb.group(4))), (a, b)


def test_two_calls_are_bit_identical():
    """(c) fixed-order reductions: the same inputs give the same poses, run after run."""
    c = LC.lba_opt_case('lbaopt_par_m11_v2_48x80')
    a, la = run(c)
    b, lb = run(c)
    assert np.array_equal(a, b) and la == lb


@pytest.mark.parametrize('mode', ['m01', 'm11', 'm10'])
def test_converges_at_the_driver_size(mode):
    """(d) 384 x 256, four views, 20 iterations per level, step 0.01: at most half the initial pose error remains."""
    from oracle.planesweep_oracle import make_cam_intrinsics
    ov = LC.LBA_OPT_MODES[mode]
    c = LC.lba_scene(71, 256, 384, 4, perturb_R=ov[0] == 1, perturb_t=ov[0] != 1 or ov[1] == 1)
    c.update(entry='parallel', opt_vars=ov, dw_scales=[4, 2, 1], max_iter=20, step=0.01,
             cams=[cases.cam_for(make_cam_intrinsics, 384 // d, 256 // d) for d in (4, 2, 1)])
    poses, _ = run(c)
    e0 = np.abs(c['poses_init'] - c['poses_true']).max()
    e1 = np.abs(poses - c['poses_true']).max()
    assert e1 <= 0.5 * e0, (e0, e1)


@pytest.mark.parametrize('name', ['lbaopt_par_m01_v4_256x384', 'lbaopt_seq_m11_v2_48x64'])
def test_launches_per_call(name):
    """(e) one kernel per iteration plus the pyramid."""
    from neuralrgbd_b200 import _lib
    L = _lib.lib()
    c = LC.lba_opt_case(name)
    run(c)
    torch.cuda.synchronize()
    L.nrgbd_reset_launch_count()
    run(c)
    assert L.nrgbd_launch_count() <= 3 * c['max_iter'] + 4


DROPIN_PROBE = r'''
import contextlib, io, json, sys
sys.path.insert(0, %(root)r)
import numpy as np, torch
from tests import cases_lba_opt as LC
sys.path.insert(0, %(ref)r)
import ICP.opt_pose_numerical as opn                   # the unmodified reference
c = LC.lba_opt_case(%(name)r)
def cam(k):
    d = dict(k); d['unit_ray_array_2D'] = torch.from_numpy(k['unit_ray_array_2D']); d['intrinsic_M_cuda'] = torch.from_numpy(k['intrinsic_M_cuda'])
    return d
def call():
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    with contextlib.redirect_stdout(io.StringIO()):
        P = opn.local_BA_direct_parallel(T(c['ref']), [T(s) for s in c['srcs']], T(c['dmap']), T(c['conf']), [cam(k) for k in c['cams']],
                                         c['dw_scales'], list(c['poses_init']), c['max_iter'], c['step'], c['opt_vars'])
    return np.stack([p.numpy() for p in P])
ref = call()
import neuralrgbd_b200
ns = neuralrgbd_b200.install_as_reference_modules(%(ref)r)
mine = call()
print(json.dumps({'module': opn.local_BA_direct_parallel.__module__, 'diff': float(np.abs(mine - ref).max())}))
'''


def test_dropin_routes_the_reference_optimiser():
    """(f) with the reference copy in oracle/_ref: its own ICP.opt_pose_numerical, patched, against the same module unpatched
    (eager ATen on this GPU)."""
    from oracle import fetch_reference
    ref = fetch_reference.code_dir()
    if not ref or not os.path.isdir(os.path.join(ref, 'ICP')):
        pytest.skip('no reference checkout with ICP/ (oracle/_ref is made by build())')
    name = 'lbaopt_par_m11_v2_48x80'
    r = subprocess.run([sys.executable, '-c', DROPIN_PROBE % dict(root=ROOT, ref=ref, name=name)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out['module'] == 'neuralrgbd_b200.ICP.opt_pose_numerical'
    p = json.load(open(os.path.join(GOLD, 'PINNING_lba_opt.json')))['cases'][name]
    assert out['diff'] <= max(1e-4, 4 * p['final_pose_maxabs']), out
