"""Helpers shared by the tests, tests/cases_*.py and tests/reference_driver.py: fixture loaders, the parity-report writer,
small numeric helpers, the engine KVNET the GPU tests build, the reference's re-seeding priors, and the subprocess call
of tests/reference_driver.py."""
import contextlib
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cases
from tests.conftest import maxabs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
DEV = 'cuda:0'
NAMES4 = ['dmap_cur_refined', 'dmap_refined', 'BV_cur', 'DPV']


# ---- fixtures ----------------------------------------------------------------------------------------------------------
def golden(name):
    """tests/golden/<name> (.npz)."""
    return np.load(os.path.join(GOLDEN, name))


def pinning(name):
    """The pinned cases of tests/golden/<name> (PINNING_*.json)."""
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)['cases']


def golden_fixture(name):
    """A module-scoped pytest fixture of golden(name)."""
    return pytest.fixture(scope='module')(lambda: golden(name))


def pinning_fixture(name):
    """A module-scoped pytest fixture of pinning(name)."""
    return pytest.fixture(scope='module')(lambda: pinning(name))


def parity_dump(stem, key, row):
    """Record `row` under `key` in $NRGBD_PARITY_DIR/parity_<stem>.json (read by tools/parity_report.py); nothing without
    the variable. A report that cannot be written does not fail the test."""
    d = os.environ.get('NRGBD_PARITY_DIR')
    if not d:
        return
    try:
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, 'parity_%s.json' % stem)
        cur = json.load(open(path)) if os.path.exists(path) else {}
        cur[key] = row
        with open(path, 'w') as f:
            json.dump(cur, f, indent=1, sort_keys=True)
    except OSError:
        pass


# ---- numeric helpers ---------------------------------------------------------------------------------------------------
def T(a):
    """numpy -> contiguous tensor on the test device."""
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def cam_tensors(cam, device=None):
    """A camera dict (cases.cam_for) with its ray and intrinsic arrays as tensors, on `device` when given."""
    return dict(cam, unit_ray_array_2D=torch.from_numpy(cam['unit_ray_array_2D']).to(device),
                intrinsic_M_cuda=torch.from_numpy(cam['intrinsic_M_cuda']).to(device))


def rel_err(a, b):
    """max |a - b| relative to max |b|, in float64."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def launch_count(fn):
    """-> (kernel launches libnrgbd counted during fn(), fn's result)."""
    from neuralrgbd_b200 import _lib
    L = _lib.lib()
    torch.cuda.synchronize()
    L.nrgbd_reset_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return L.nrgbd_launch_count(), out


# ---- the engine's KVNET ------------------------------------------------------------------------------------------------
def engine_kvnet(c, cam_t, sd, conv_math, train=None, **kvnet_kw):
    """neuralrgbd_b200.models.KVNET.KVNET for case `c` built by keyword (its printout silenced), state dict `sd` (name ->
    array) loaded strictly, on the device with `conv_math`; `train` sets the mode when given."""
    from neuralrgbd_b200.models.KVNET import KVNET
    with contextlib.redirect_stdout(io.StringIO()):
        m = KVNET(feature_dim=64, cam_intrinsics=cam_t, d_candi=c['d'], sigma_soft_max=c['sigma'], KVNet_feature_dim=64,
                  d_upsample_ratio_KV_net=None, t_win_r=c['t_win_r'], **kvnet_kw)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    m = m.to(DEV)
    m.conv_math = conv_math
    if train is not None:
        m.train(train)
    return m


def engine_forward(m, c, cam_t, step, prior):
    """No-grad forward of window t_win_r + step of case `c` (prior: a log-DPV array or None) -> (ref_f, outputs)."""
    ref_f, src_f, poses = cases.window(c, c['t_win_r'] + step)
    assert src_f.shape[1] == 2 * c['t_win_r']
    with torch.no_grad():
        out = m(T(ref_f), T(src_f), T(poses), torch.zeros(1), cam_intrinsics=[cam_t], BV_predict=None if prior is None else T(prior))
    return ref_f, out


def compare_outputs(gold, key, full, d):
    """Max-abs probability deviation on the stored samples (the first window stores BV_cur / dmap_cur_refined, which its
    filtered outputs equal; a steady step its filtered DPV / dmap_refined), the sum of squared probabilities of every full
    array, and the expected depth in mm. The eval and twin fixtures store 8000 strided samples per array, 2000 of depth."""
    row = {}
    aliases = {'DPV': 'BV_cur', 'dmap_refined': 'dmap_cur_refined'} if key.endswith('/step0') else {}
    for nm, a in zip(NAMES4, full):
        a = a.cpu().numpy()
        assert np.isfinite(a).all(), (key, nm)
        k = '%s/%s' % (key, aliases.get(nm, nm))
        if k in gold.files:
            row[nm] = maxabs(np.exp(cases.subsample_to(a, 8000)), np.exp(gold[k]))
        st, gs = cases.stats(np.exp(a.astype(np.float64))), gold['%s/%s_stats' % (key, nm)]
        row[nm + '_sumsq_rel'] = abs(st[1] - gs[1]) / gs[1]
    from neuralrgbd_b200.mutils import misc
    dep = misc.depth_val_regression(full[3], d).cpu().numpy()
    row['depth_mm'] = 1000.0 * maxabs(cases.subsample_to(dep, 2000), gold[key + '/depth'])
    return row


def reference_prior(name, step):
    """The reference's train-mode prior that re-seeds steady step `step` >= 1 of case `name`: from reference_outputs.npz for
    cases.KVNET_CASES, else from configs_priors_<name>.npz, which holds the prior of step 1 only."""
    if name in cases.KVNET_CASES:
        return golden('reference_outputs.npz')['kvnet/%s/step%d/BV_predict_next_full' % (name, step - 1)]
    assert step == 1, step
    return golden('configs_priors_%s.npz' % name)['cfg/%s/step0/BV_predict_next_full' % name]


# ---- the reference in a subprocess -------------------------------------------------------------------------------------
def run_reference_driver(*args, timeout):
    """Run tests/reference_driver.py with the reference copy and `args` (a sub-command and its scenario) -> its JSON line."""
    from oracle import fetch_reference
    ref_code = fetch_reference.code_dir()
    assert ref_code, 'no copy of the reference: oracle/_ref is made by __graft_entry__.build() (oracle/fetch_reference.py)'
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'reference_driver.py'), ref_code] + list(args),
                       capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    return json.loads(r.stdout.strip().splitlines()[-1])
