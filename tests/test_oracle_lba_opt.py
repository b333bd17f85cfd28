"""The LBA pose optimiser, oracle first (CPU): oracle/lba_opt_oracle.py against the unmodified reference's
ICP/opt_pose_numerical.py local_BA_direct(_parallel) (tests/golden/lba_opt_outputs.npz, make_golden.py lba_opt), its
Adam against torch.optim.Adam, the initial-pose conversion, and the drop-in patch of ICP.opt_pose_numerical."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import lba_opt_oracle as LO
from tests import cases_lba_opt as LC, harness
from tests.conftest import ROOT


gold = harness.golden_fixture('lba_opt_outputs.npz')
pin = harness.pinning_fixture('PINNING_lba_opt.json')


@pytest.mark.parametrize('name', LC.LBA_OPT_CASES)
def test_oracle_matches_the_reference_within_its_pinned_deviation(gold, pin, name):
    c = LC.lba_opt_case(name)
    poses = np.stack(LO.local_ba(c['ref'], c['srcs'], c['dmap'], c['conf'], c['cams'], c['dw_scales'], c['poses_init'], c['max_iter'],
                                 c['step'], c['opt_vars'], c['entry'] == 'parallel'))
    assert np.abs(poses - gold[name + '/poses']).max() <= 1.5 * pin[name]['final_pose_maxabs'] + 1e-7
    assert len(gold[name + '/printed']) == 3 * (1 if c['entry'] == 'parallel' else len(c['srcs']))


@pytest.mark.parametrize('name', LC.LBA_OPT_CASES)
def test_initial_pose_round_trip_is_bit_identical(gold, name):
    from neuralrgbd_b200.ICP import opt_pose_numerical as M
    c = LC.lba_opt_case(name)
    for v, P in enumerate(c['poses_init']):
        u = LO.rotation_to_unitq(P[:3, :3])
        assert np.array_equal(u, gold[name + '/init_u'][v])
        assert np.array_equal(LO.unitq_to_rotation(u), gold[name + '/init_R'][v])
        st = M.initial_state([P])[0]                                      # the mirror's host conversion
        assert np.array_equal(st[M._U:M._U + 3], u) and np.array_equal(st[M._R:M._R + 9].reshape(3, 3), gold[name + '/init_R'][v])


def test_oracle_adam_is_bit_identical_to_torch():
    rng = np.random.RandomState(5)
    for shape in [(3,), (4, 3)]:
        p0 = rng.standard_normal(shape).astype(np.float32)
        P = torch.tensor(p0.copy(), requires_grad=True)
        opt = torch.optim.Adam([P], lr=0.01, betas=(.9, .999))
        p, m, v = p0.copy(), np.zeros_like(p0), np.zeros_like(p0)
        for s in range(3):
            for g_ in opt.param_groups:
                g_['lr'] = 0.01 / 2 ** s
            for it in range(20):
                g = (rng.standard_normal(shape) * 10 ** rng.uniform(-5, 0)).astype(np.float32)
                P.grad = torch.from_numpy(g.copy())
                opt.step()
                p, m, v = LO.adam_step(p, g, m, v, s * 20 + it + 1, 0.01 / 2 ** s)
                assert np.array_equal(P.detach().numpy(), p)
                assert np.array_equal(opt.state[P]['exp_avg'].numpy(), m) and np.array_equal(opt.state[P]['exp_avg_sq'].numpy(), v)


def test_oracle_rotation_gradient_matches_autograd():
    """dL/du through quaternion2Rotation as written and unitQ_to_quat, against torch autograd of the same formulas."""
    rng = np.random.RandomState(8)
    for _ in range(5):
        u = (np.array([1.0, 0, 0]) + 0.1 * rng.standard_normal(3)).astype(np.float32)
        G = rng.standard_normal((3, 3))
        ut = torch.tensor(u.astype(np.float64), requires_grad=True)
        x, y, z = ut[0], ut[1], ut[2]
        a2 = x ** 2 + y ** 2 + z ** 2
        qw, qx, qy, qz = 2 * x / (a2 + 1), 2 * y / (a2 + 1), 2 * z / (a2 + 1), (1 - a2) / (1 + a2)
        s = 1 / (qw ** 2 + qx ** 2 + qy ** 2 + qz ** 2)
        R = torch.stack([torch.stack([1 - 2 * s * (qy ** 2 + qz ** 2), 2 * (qx * qy - qw * qz), 2 * (qx * qz + qw * qy)]),
                         torch.stack([2 * (qx * qy + qw * qz), 1 - 2 * s * (qx ** 2 + qz ** 2), 2 * (qy * qz - qw * qx)]),
                         torch.stack([2 * (qx * qz - qw * qy), 2 * (qy * qz + qw * qx), 1 - 2 * s * (qx ** 2 + qy ** 2)])])
        (R * torch.from_numpy(G)).sum().backward()
        assert np.allclose(LO.unitq_grad(u, G), ut.grad.numpy(), rtol=1e-10, atol=1e-12)


def test_avg_pool_is_bit_identical_to_torch():
    x = np.random.RandomState(2).rand(2, 3, 24, 36).astype(np.float32)
    for k in (2, 4):
        assert np.array_equal(LO.avg_pool(x, k), torch.nn.functional.avg_pool2d(torch.from_numpy(x), k).numpy())


STANDIN_PROBE = r'''
import json, sys
sys.path.insert(0, %(root)r)
import neuralrgbd_b200
ns = neuralrgbd_b200.install_as_reference_modules(%(ref)r)
import ICP.opt_pose_numerical as opn
out = {'file': opn.__file__, 'patched': [opn.local_BA_direct.__module__, opn.local_BA_direct_parallel.__module__],
       'ns': ns.opt_pose_numerical is opn, 'listed': sorted(ns.patched.get('ICP.opt_pose_numerical', []))}
neuralrgbd_b200.uninstall_reference_patches()
out['restored'] = [opn.local_BA_direct.__module__, opn.local_BA_direct_parallel.__module__]
print(json.dumps(out))
'''


def test_install_patches_and_restores_icp_opt_pose_numerical(tmp_path):
    """A stand-in checkout with the reference's package layout, ICP/opt_pose_numerical.py included."""
    from tests.test_dropin_host import STANDIN
    root = tmp_path / 'code'
    files = dict(STANDIN)
    files['ICP/__init__.py'] = ''
    files['ICP/opt_pose_numerical.py'] = ('import warping.homography as warp_homo\nimport mutils.misc as m_misc\n\n\n'
                                          'def local_BA_direct(*a, **k):\n    raise NotImplementedError\n\n\n'
                                          'def local_BA_direct_parallel(*a, **k):\n    raise NotImplementedError\n')
    for rel, src in files.items():
        (root / os.path.dirname(rel)).mkdir(parents=True, exist_ok=True)
        (root / rel).write_text(src)
    r = subprocess.run([sys.executable, '-c', STANDIN_PROBE % dict(root=ROOT, ref=str(root))], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out['file'].startswith(str(root)) and out['ns']
    assert out['patched'] == ['neuralrgbd_b200.ICP.opt_pose_numerical'] * 2
    assert out['listed'] == ['local_BA_direct', 'local_BA_direct_parallel']
    assert out['restored'] == ['ICP.opt_pose_numerical'] * 2


def test_install_without_a_checkout_registers_the_optimiser():
    code = ('import sys; sys.path.insert(0, %r); import neuralrgbd_b200 as n; ns = n.install_as_reference_modules(); '
            'import ICP.opt_pose_numerical as o; print(o.__name__, ns.opt_pose_numerical is o)' % ROOT)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=600, cwd='/tmp')
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ['neuralrgbd_b200.ICP.opt_pose_numerical', 'True']


def test_undefined_optimisation_option_raises_like_the_reference():
    from neuralrgbd_b200.ICP import opt_pose_numerical as M
    with pytest.raises(Exception, match='undefined optmization variable option'):
        M._mode([1, 2])
    assert M._mode([0, 1]) == M._mode([0, 0]) == M._mode([0, 7]) == M.OPT_T
    assert M._mode([1, 0]) == M.OPT_R and M._mode([1, 1]) == M.OPT_R | M.OPT_T
