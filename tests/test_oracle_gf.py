"""CPU checks of tests/oracle_gf.py, the numpy restatement of the reference's models/GF GuidedFilter and BoxFilter, and of
the host side of their mirrors in neuralrgbd_b200.models.GF:
 * the oracle against the unmodified reference's forward and torch autograd (tests/golden/make_golden.py gf) at the
   pinned floor; the forwards are bit-exact;
 * torch.autograd.gradcheck (float64 central differences) of the oracle backwards against their float64 forwards;
 * the mirrors' constructor, attributes, asserts and CPU-tensor error, and the install / uninstall round trip of the
   new install_as_reference_modules() entries on the reference's own modules."""
import json
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cases, cases_gf as CG, oracle_gf as OG, harness
from tests.conftest import ROOT


gold = harness.golden_fixture('gf_outputs.npz')
pin = harness.pinning_fixture('PINNING_gf.json')


def _check(gold, pin, key, mine):
    p = pin[key]
    assert list(mine.shape) == p['shape']
    # the oracle is deterministic: it reproduces the deviation it was pinned at
    assert np.abs(CG.sub(mine).astype(np.float64) - gold[key]).max() <= p['maxabs_oracle']
    s, want = cases.summary(mine), gold[key + '/stats']
    assert s[2] == want[2] and abs(s[3] - want[3]) <= p['maxabs_oracle']
    assert abs(s[1] - want[1]) <= 1e-5 * want[1] + sumsq_allowance(want, p['maxabs_oracle'])
    assert abs(s[0] - want[0]) <= p['maxabs_oracle'] * want[2] + 1e-9 * abs(want[0])


def sumsq_allowance(want, dev):
    """|sum a^2 - sum b^2| <= sum |a - b| |a + b| <= dev (2 sqrt(n sum b^2) + n dev) when |a - b| <= dev everywhere."""
    n, ss = want[2], want[1]
    return dev * (2 * np.sqrt(n * ss) + n * dev)


@pytest.mark.parametrize('name', CG.CASES)
def test_guided_filter_vs_reference(gold, pin, name):
    c = CG.case(name)
    out = OG.guided_filter(c['x'], c['y'], c['r'], c['eps'])
    assert pin['gf/%s/out' % name]['maxabs_oracle'] == 0.0           # bit-exact forward
    _check(gold, pin, 'gf/%s/out' % name, out)
    assert np.array_equal(out, OG.parts(c['x'], c['y'], c['r'], c['eps'])['out'])
    gx, gy = OG.guided_filter_backward(c['g'], c['x'], c['y'], c['r'], c['eps'])
    _check(gold, pin, 'gf/%s/g_x' % name, gx)
    _check(gold, pin, 'gf/%s/g_y' % name, gy)


@pytest.mark.parametrize('name', CG.CASES)
def test_box_filter_vs_reference(gold, pin, name):
    c = CG.case(name)
    assert pin['box/%s/out' % name]['maxabs_oracle'] == 0.0
    _check(gold, pin, 'box/%s/out' % name, OG.box_filter(c['y'], c['r']))
    _check(gold, pin, 'box/%s/g_x' % name, OG.box_filter_backward(c['g_box'], c['r']))


def test_backward_floor_is_small_except_where_A_amplifies(pin):
    """The oracle's float64 backward against the reference's fp32 autograd: within 1e-4 of the largest gradient, except
    the flat guide's d x, where A = cov / (var + eps) amplifies fp32 rounding of var by up to 1/eps."""
    for k, p in pin.items():
        if '/g_' in k and k != 'gf/flat_120x160/g_x':
            assert p['maxabs_oracle'] <= 1e-4 * p['max_ref'], (k, p)
    p = pin['gf/flat_120x160/g_x']
    assert p['maxabs_oracle'] <= 5e-2 * p['max_ref']


# ---- gradcheck of the oracle backwards (float64), small problems ---------------------------------------------------
class _Op(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fwd, bwd):
        ctx.bwd, ctx.x = bwd, x.detach().numpy()
        return torch.from_numpy(np.asarray(fwd(ctx.x), np.float64))

    @staticmethod
    def backward(ctx, g):
        return torch.from_numpy(np.asarray(ctx.bwd(g.detach().numpy(), ctx.x), np.float64)), None, None


def _gradcheck(x0, fwd, bwd):
    x = torch.from_numpy(np.asarray(x0, np.float64)).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda t: _Op.apply(t, fwd, bwd), (x,), eps=1e-6, atol=1e-7, rtol=1e-5)


@pytest.mark.parametrize('r,h,w', [(1, 5, 7), (2, 6, 5), (0, 3, 4)])
def test_gradcheck_box_filter(r, h, w):
    x0 = np.random.RandomState(3).standard_normal((2, 1, h, w))
    _gradcheck(x0, lambda x: OG.box_filter64(x, r), lambda g, x: OG.box_filter_backward(g, r))


@pytest.mark.parametrize('cx,cy', [(1, 1), (1, 2), (2, 2)])
@pytest.mark.parametrize('eps', [1e-2, 1e-1])
def test_gradcheck_guided_filter(cx, cy, eps):
    rng = np.random.RandomState(4)
    N, H, W, r = 1, 5, 6, 1
    x0, y0 = rng.standard_normal((N, cx, H, W)), 2.0 + rng.standard_normal((N, cy, H, W))
    nx = x0.size

    def split(v):
        return v[:nx].reshape(x0.shape), v[nx:].reshape(y0.shape)

    def fwd(v):
        return OG.guided_filter64(*split(v), r, eps)

    def bwd(g, v):
        gx, gy = OG.guided_filter_backward(g, *split(v), r, eps, dtype=np.float64)
        return np.concatenate([gx.reshape(-1), gy.reshape(-1)])
    _gradcheck(np.concatenate([x0.reshape(-1), y0.reshape(-1)]), fwd, bwd)


# ---- the mirrors' host side ---------------------------------------------------------------------------------------
def test_mirror_modules_match_the_reference_surface():
    from neuralrgbd_b200 import _lib
    from neuralrgbd_b200.models.GF.box_filter import BoxFilter
    from neuralrgbd_b200.models.GF.guided_filter import GuidedFilter
    gf = GuidedFilter(2)
    assert gf.r == 2 and gf.eps == 1e-8 and isinstance(gf.boxfilter, BoxFilter) and gf.boxfilter.r == 2
    assert GuidedFilter(1, eps=1e-2).eps == 1e-2
    assert not list(gf.parameters()) and not list(gf.buffers()) and not gf.state_dict()
    x, y = torch.zeros(1, 1, 8, 8), torch.zeros(1, 3, 8, 8)
    # the reference's asserts (guided_filter.py:71-74, box_filter.py:32) come first, then the missing CPU path
    with pytest.raises(AssertionError):
        gf(torch.zeros(2, 1, 8, 8), y)
    with pytest.raises(AssertionError):
        gf(torch.zeros(1, 2, 8, 8), y)
    with pytest.raises(AssertionError):
        gf(x, torch.zeros(1, 3, 8, 9))
    with pytest.raises(AssertionError):
        GuidedFilter(4)(x, y)
    with pytest.raises(ValueError):
        gf(torch.zeros(1, 8, 8), y)
    with pytest.raises(AssertionError):
        BoxFilter(1)(torch.zeros(8, 8))
    with pytest.raises(_lib.NrgbdError):
        gf(x, y)
    with pytest.raises(_lib.NrgbdError):
        BoxFilter(1)(x)


def test_patch_entries_present():
    import neuralrgbd_b200
    table = {r: (m, s) for r, m, s in neuralrgbd_b200._PATCHES}
    assert table['models.GF.guided_filter'] == ('neuralrgbd_b200.models.GF.guided_filter', ('GuidedFilter',))
    assert table['models.GF.box_filter'] == ('neuralrgbd_b200.models.GF.box_filter', ('BoxFilter',))


_ROUND_TRIP = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(1, sys.argv[2])
import neuralrgbd_b200 as nb
import models.GF.guided_filter as G, models.GF.box_filter as B
orig = (G.GuidedFilter, B.BoxFilter)
ns = nb.install_as_reference_modules(sys.argv[2])
import models.Refine as R
from neuralrgbd_b200.models.GF import guided_filter as MG, box_filter as MB
dgf = R.RefineNet_DGF(64)
res = {'patched': G.GuidedFilter is MG.GuidedFilter and B.BoxFilter is MB.BoxFilter,
       'listed': [ns.patched.get('models.GF.guided_filter'), ns.patched.get('models.GF.box_filter')],
       'dgf_is_mirror': type(dgf.dgf) is MG.GuidedFilter,
       'ns_keys': sorted(k for k in vars(ns))}
nb.uninstall_reference_patches()
res['restored'] = (G.GuidedFilter, B.BoxFilter) == orig and not hasattr(G, '_nrgbd_original_GuidedFilter')
dgf2 = R.RefineNet_DGF(64)
res['dgf_restored'] = type(dgf2.dgf) is orig[0]
res['same_keys'] = list(dgf.state_dict()) == list(dgf2.state_dict())
print(json.dumps(res))
'''


def test_install_round_trip_on_the_reference_modules():
    """A reference RefineNet_DGF built after the install carries the mirror; uninstall restores the reference's classes.
    Runs in a subprocess on the reference copy that build() makes under oracle/_ref."""
    from oracle import fetch_reference
    code = fetch_reference.code_dir()
    if not code:
        pytest.skip('no copy of the reference under oracle/_ref (made by __graft_entry__.build())')
    r = subprocess.run([sys.executable, '-c', _ROUND_TRIP, ROOT, code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res['patched'] and res['listed'] == [['GuidedFilter'], ['BoxFilter']]
    assert res['dgf_is_mirror'] and res['restored'] and res['dgf_restored'] and res['same_keys']
    assert res['ns_keys'] == ['KVNET', 'homography', 'misc', 'opt_pose_numerical', 'patched']
