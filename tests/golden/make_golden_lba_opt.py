"""Golden vectors for the LBA pose optimiser (ICP/opt_pose_numerical.py local_BA_direct / local_BA_direct_parallel).

Run in the build container only (needs the reference checkout):
    python tests/golden/make_golden_lba_opt.py [reference code/ directory]
Runs the UNMODIFIED reference on CPU (the 4-line .cuda() shim) on the scenes of tests/cases_lba_opt.py:lba_opt_case and records,
per case: the returned poses, the printed lines, Rotation2UnitQ / UnitQ2Rotation of the initial poses and, for every Adam
step (torch.optim.Adam.step is wrapped here, and only here), the parameters, gradients and Adam state before and after it and
the L1 loss the iteration evaluated (nn.L1Loss.forward is wrapped too). Writes tests/golden/lba_opt_outputs.npz and the
oracle's deviations from the reference to PINNING_lba_opt.json.
"""
import contextlib
import io
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = sys.argv[1] if len(sys.argv) > 1 else '/root/reference/code'
sys.path.insert(0, REF)
warnings.filterwarnings('ignore')

torch.Tensor.cuda = lambda s, *a, **k: s
torch.nn.Module.cuda = lambda s, *a, **k: s
torch.cuda.current_device = lambda: 0
torch.Tensor.get_device = lambda s: 0

import ICP.opt_pose_numerical as ref_opt             # noqa: E402  (reference)
import mutils.misc as ref_misc                       # noqa: E402  (reference)

from oracle import lba_opt_oracle as LO               # noqa: E402
from tests import cases_lba_opt as LC                 # noqa: E402

T = torch.from_numpy
_steps, _losses = [], []
_adam_step = torch.optim.Adam.step
_l1_forward = torch.nn.L1Loss.forward


def _snap(self, *a, **k):
    ps = [p for g in self.param_groups for p in g['params']]
    st = [self.state.get(p, {}) for p in ps]
    rec = {'p': [p.detach().clone().numpy() for p in ps], 'g': [p.grad.clone().numpy() for p in ps],
           'm': [s['exp_avg'].clone().numpy() if 'exp_avg' in s else np.zeros(tuple(p.shape), np.float32) for p, s in zip(ps, st)],
           'v': [s['exp_avg_sq'].clone().numpy() if 'exp_avg_sq' in s else np.zeros(tuple(p.shape), np.float32) for p, s in zip(ps, st)],
           'lr': self.param_groups[0]['lr']}
    out = _adam_step(self, *a, **k)
    rec['p1'] = [p.detach().clone().numpy() for p in ps]
    rec['m1'] = [self.state[p]['exp_avg'].clone().numpy() for p in ps]
    rec['v1'] = [self.state[p]['exp_avg_sq'].clone().numpy() for p in ps]
    _steps.append(rec)
    return out


def _loss(self, a, b):
    out = _l1_forward(self, a, b)
    _losses.append(float(out.detach()))
    return out


def _cam_t(cam):
    c = dict(cam)
    c['unit_ray_array_2D'] = T(cam['unit_ray_array_2D']); c['intrinsic_M_cuda'] = T(cam['intrinsic_M_cuda'])
    return c


def run_reference(c):
    del _steps[:], _losses[:]
    fn = ref_opt.local_BA_direct_parallel if c['entry'] == 'parallel' else ref_opt.local_BA_direct
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        poses = fn(T(c['ref']), [T(s) for s in c['srcs']], T(c['dmap']), T(c['conf']), [_cam_t(k) for k in c['cams']], c['dw_scales'],
                   list(c['poses_init']), c['max_iter'], c['step'], c['opt_vars'])
    return np.stack([p.numpy() for p in poses]), buf.getvalue().splitlines()


def per_step(c):
    """Steps as arrays [S, V, 3] for 't' / 'u' (whichever Adam updates), loss [S, V] (serial) or [S, 1] (parallel)."""
    V, S = len(c['srcs']), 3 * c['max_iter']
    ov = c['opt_vars']
    names = {(0, 1): ['t'], (0, 0): ['t'], (1, 1): ['t', 'u'], (1, 0): ['u']}[tuple(ov)]
    out = {}
    serial = c['entry'] == 'serial'
    for j, nm in enumerate(names):
        for key in ('p', 'g', 'm', 'v', 'p1', 'm1', 'v1'):
            a = np.stack([np.asarray(r[key][j], np.float32).reshape(-1, 3) for r in _steps])       # [V*S or S, 1 or V, 3]
            out['%s/%s' % (key, nm)] = a.reshape(V, S, 3).transpose(1, 0, 2) if serial else a
    out['lr'] = np.array([r['lr'] for r in _steps][:S])
    la = np.asarray(_losses, np.float32)
    out['loss'] = la.reshape(V, S).T if serial else la.reshape(S, 1)
    return out


def one_step_deviation(c, steps):
    """The oracle's iteration started from every recorded reference state: its gradients (relative to the largest reference
    gradient) and the parameters after its Adam step, against the reference's."""
    levels = LO.pyramid(c['ref'], c['srcs'], c['dmap'], c['conf'], c['dw_scales'])
    init = [LO.init_state(p) for p in c['poses_init']]
    names = [nm for nm in ('t', 'u') if 'g/' + nm in steps]
    S = steps['g/' + names[0]].shape[0]
    d = {}
    for nm in names:
        d['grad_%s_rel' % nm] = 0.0
        d['step_%s_maxabs' % nm] = 0.0
    for k in range(S):
        states = []
        for v, x0 in enumerate(init):
            x = dict(x0)
            for nm in names:
                x[nm] = steps['p/' + nm][k][v]
            x['R'] = LO.unitq_to_rotation(x['u'])
            states.append(x)
        _, g_u, g_t = LO.gradients(levels[k // c['max_iter']], states, c['cams'][k // c['max_iter']], c['entry'] == 'parallel')
        for nm, g in (('t', g_t), ('u', g_u)):
            if nm not in names:
                continue
            g_ref = steps['g/' + nm][k]
            d['grad_%s_rel' % nm] = max(d['grad_%s_rel' % nm], float(np.abs(g - g_ref).max() / np.abs(g_ref).max()))
            p1, _, _ = LO.adam_step(steps['p/' + nm][k], g, steps['m/' + nm][k], steps['v/' + nm][k], k + 1, c['step'] / 2 ** (k // c['max_iter']))
            d['step_%s_maxabs' % nm] = max(d['step_%s_maxabs' % nm], float(np.abs(p1 - steps['p1/' + nm][k]).max()))
    return d


def main():
    torch.optim.Adam.step = _snap
    torch.nn.L1Loss.forward = _loss
    out, pin = {}, {'torch': torch.__version__, 'cases': {}}
    for name in LC.LBA_OPT_CASES:
        c = LC.lba_opt_case(name)
        poses, lines = run_reference(c)
        steps = per_step(c)
        out[name + '/poses'] = poses
        out[name + '/printed'] = np.array(lines)
        for k, a in steps.items():
            out[name + '/' + k] = a
        init_u = np.stack([ref_misc.Rotation2UnitQ(T(np.ascontiguousarray(p[:3, :3]))).numpy() for p in c['poses_init']])
        out[name + '/init_u'] = init_u
        out[name + '/init_R'] = np.stack([ref_misc.UnitQ2Rotation(T(u)).numpy() for u in init_u])
        # the oracle against the reference
        rec = []
        o_poses = np.stack(LO.local_ba(c['ref'], c['srcs'], c['dmap'], c['conf'], c['cams'], c['dw_scales'], c['poses_init'], c['max_iter'],
                                       c['step'], c['opt_vars'], c['entry'] == 'parallel', record=rec))
        d = {'final_pose_maxabs': float(np.abs(o_poses - poses).max()),
             'init_pose_error': float(np.abs(c['poses_init'] - c['poses_true']).max()),
             'final_pose_error_reference': float(np.abs(poses - c['poses_true']).max())}
        d.update(one_step_deviation(c, steps))
        pin['cases'][name] = d
        print(name, json.dumps(d), flush=True)
    torch.optim.Adam.step = _adam_step
    torch.nn.L1Loss.forward = _l1_forward
    np.savez_compressed(os.path.join(HERE, 'lba_opt_outputs.npz'), **out)
    with open(os.path.join(HERE, 'PINNING_lba_opt.json'), 'w') as f:
        json.dump(pin, f, indent=1, sort_keys=True)


if __name__ == '__main__':
    main()
