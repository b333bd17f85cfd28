"""The models.GF mirrors on the device: GuidedFilter(r, eps) and BoxFilter(r) (models/GF/guided_filter.py, box_filter.py).

 * Forwards against tests/oracle_gf.py bit for bit on every case, which also holds the parallel scans' fp32 prefixes
   to the sequential double accumulation; BoxFilter on x, y, x*y and x*x of every case, bit for bit.
 * Backwards against the oracle's float64 backward and against the unmodified reference's torch autograd
   (tests/golden/make_golden_gf.py), gated from the oracle-vs-reference floor pinned in PINNING_gf.json.
 * Plain inputs, inputs that require grad and torch.no_grad() give the same launches and bit-identical values; two
   runs give identical results; the reference's asserts are kept.
 * The reference's own models.KVNET.KVNET(refineNet_name='DGF') trained under train_utils/train_KVNet.py's L1 loss with
   the mirrors and GuidedFilter patched in, against the unpatched reference (tests/reference_driver.py grad gf).
Measured deviations are written to $NRGBD_PARITY_DIR/parity_gf.json when that variable is set.
"""
import numpy as np
import pytest
import torch

from tests import cases_gf as CG, oracle_gf as OG, harness
from tests.test_oracle_gf import sumsq_allowance

pytestmark = pytest.mark.gpu
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731

# Backward gates, relative to the largest reference gradient of the array, on top of multiples of the pinned
# oracle-vs-reference floor. The kernels' forward planes are the reference's bit for bit; the backward chains about ten
# fp32 roundings per element and four reverse prefix sums rounded to fp32 per position (the reference's autograd does
# the same in its own order), against the oracle's float64. Where the guide is flat, A = cov / (var + eps) multiplies
# the rounding of var by up to 1/eps: there the fp32 backward is as far from float64 as the reference's own is, so the
# gate is a multiple of that floor.
REL = 2e-5
FLOOR_X = 3.0


gold = harness.golden_fixture('gf_outputs.npz')
pin = harness.pinning_fixture('PINNING_gf.json')


def _gate(gold, pin, key, mine, orc):
    p = pin[key]
    allow = FLOOR_X * p['maxabs_oracle'] + REL * p['max_ref']
    e_orc = float(np.abs(mine.astype(np.float64) - orc).max())
    e_ref = float(np.abs(CG.sub(mine).astype(np.float64) - gold[key]).max())
    s, want = CG.summary(mine), gold[key + '/stats']
    harness.parity_dump('gf', key, {'vs_oracle': e_orc, 'vs_reference_sample': e_ref, 'floor': p['maxabs_oracle'], 'max_ref': p['max_ref'],
                'gate': allow, 'rel_vs_oracle': e_orc / p['max_ref']})
    assert list(mine.shape) == p['shape']
    assert e_orc <= allow, (key, e_orc, allow)
    lim = p['maxabs_oracle'] + allow
    assert e_ref <= lim, (key, e_ref, lim)
    assert s[2] == want[2]
    assert abs(s[3] - want[3]) <= lim
    assert abs(s[1] - want[1]) <= 1e-5 * want[1] + sumsq_allowance(want, lim)
    assert abs(s[0] - want[0]) <= lim * want[2] + 1e-9 * abs(want[0])


def _exact(gold, key, mine, orc):
    assert np.array_equal(mine, orc), (key, int((mine != orc).sum()), float(np.abs(mine.astype(np.float64) - orc).max()))
    assert np.array_equal(CG.sub(mine), gold[key])
    harness.parity_dump('gf', key, {'mismatch_oracle': 0})


@pytest.mark.parametrize('name', CG.CASES)
def test_guided_filter(gold, pin, name):
    from neuralrgbd_b200.models.GF.guided_filter import GuidedFilter
    c = CG.case(name)
    x, y = T(c['x']).requires_grad_(True), T(c['y']).requires_grad_(True)
    out = GuidedFilter(c['r'], c['eps'])(x, y)
    assert out.shape == (c['N'], c['Cy'], c['H'], c['W']) and out.device == x.device
    out.backward(T(c['g']))
    key = 'gf/' + name
    _exact(gold, key + '/out', out.detach().cpu().numpy(), OG.guided_filter(c['x'], c['y'], c['r'], c['eps']))
    gx, gy = OG.guided_filter_backward(c['g'], c['x'], c['y'], c['r'], c['eps'])
    _gate(gold, pin, key + '/g_x', x.grad.cpu().numpy(), gx)
    _gate(gold, pin, key + '/g_y', y.grad.cpu().numpy(), gy)


@pytest.mark.parametrize('name', CG.CASES)
def test_box_filter(gold, pin, name):
    """BoxFilter on its own: the forward on y and on the guide's products bit for bit (every fp32 prefix of the parallel
    scans equals the sequential double accumulation's, or a box sum would differ), the backward at the gate."""
    from neuralrgbd_b200.models.GF.box_filter import BoxFilter
    c = CG.case(name)
    bf = BoxFilter(c['r'])
    y = T(c['y']).requires_grad_(True)
    out = bf(y)
    out.backward(T(c['g_box']))
    key = 'box/' + name
    _exact(gold, key + '/out', out.detach().cpu().numpy(), OG.box_filter(c['y'], c['r']))
    _gate(gold, pin, key + '/g_x', y.grad.cpu().numpy(), OG.box_filter_backward(c['g_box'], c['r']))
    x, yy = c['x'], c['y']
    xb = np.broadcast_to(x, yy.shape) if c['Cx'] == 1 else x
    for what, a in (('x', x), ('xy', (xb * yy).astype(np.float32)), ('xx', (x * x).astype(np.float32))):
        with torch.no_grad():
            mine = bf(T(a)).cpu().numpy()
        want = OG.box_filter(a, c['r'])
        assert np.array_equal(mine, want), (name, what, int((mine != want).sum()))


def test_only_one_input_requires_grad():
    from neuralrgbd_b200.models.GF.guided_filter import GuidedFilter
    c = CG.case('cx1_cy3_60x80')
    gf = GuidedFilter(c['r'], c['eps'])
    gx, gy = OG.guided_filter_backward(c['g'], c['x'], c['y'], c['r'], c['eps'])
    x, y = T(c['x']).requires_grad_(True), T(c['y'])
    gf(x, y).backward(T(c['g']))
    assert y.grad is None and np.abs(x.grad.cpu().numpy() - gx).max() <= REL * np.abs(gx).max()
    x, y = T(c['x']), T(c['y']).requires_grad_(True)
    gf(x, y).backward(T(c['g']))
    assert x.grad is None and np.abs(y.grad.cpu().numpy() - gy).max() <= REL * np.abs(gy).max()


# ---- the no-grad path, determinism, errors -------------------------------------------------------------------------
@pytest.mark.parametrize('op', ['GuidedFilter', 'BoxFilter'])
def test_no_grad_path_unchanged(op):
    from neuralrgbd_b200.models.GF.box_filter import BoxFilter
    from neuralrgbd_b200.models.GF.guided_filter import GuidedFilter
    c = CG.case('textured_480x640')
    if op == 'GuidedFilter':
        m, want = GuidedFilter(1), 5
        fn = lambda rg: m(T(c['x']).requires_grad_(rg), T(c['y']).requires_grad_(rg))      # noqa: E731
    else:
        m, want = BoxFilter(1), 2
        fn = lambda rg: m(T(c['y']).requires_grad_(rg))                                     # noqa: E731
    n0, plain = harness.launch_count(lambda: fn(False))
    with torch.no_grad():
        n1, nog = harness.launch_count(lambda: fn(True))
    n2, withgrad = harness.launch_count(lambda: fn(True))
    assert n0 == n1 == n2 == want, (n0, n1, n2, want)
    assert plain.grad_fn is None and nog.grad_fn is None and withgrad.requires_grad
    assert torch.equal(plain, nog) and torch.equal(plain, withgrad.detach())


def test_backward_launches_and_run_to_run():
    """Two forward + backward runs give identical outputs and gradients (no atomics); the backward is 10 launches."""
    from neuralrgbd_b200.models.GF.guided_filter import GuidedFilter
    c = CG.case('c3_60x80')
    gf = GuidedFilter(c['r'], c['eps'])
    res = []
    for _ in range(2):
        x, y = T(c['x']).requires_grad_(True), T(c['y']).requires_grad_(True)
        out = gf(x, y)
        n, _ = harness.launch_count(lambda: out.backward(T(c['g'])))
        assert n == 10
        res.append((out.detach(), x.grad, y.grad))
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_asserts_and_errors():
    from neuralrgbd_b200 import _lib
    from neuralrgbd_b200.models.GF.box_filter import BoxFilter
    from neuralrgbd_b200.models.GF.guided_filter import GuidedFilter
    gf = GuidedFilter(1)
    x, y = torch.zeros(1, 1, 8, 8, device='cuda'), torch.zeros(1, 3, 8, 8, device='cuda')
    with pytest.raises(AssertionError):
        gf(torch.zeros(1, 2, 8, 8, device='cuda'), y)
    with pytest.raises(AssertionError):
        gf(x, torch.zeros(2, 3, 8, 8, device='cuda'))
    with pytest.raises(AssertionError):
        GuidedFilter(4)(x, y)
    with pytest.raises(AssertionError):
        BoxFilter(1)(torch.zeros(8, 8, device='cuda'))
    with pytest.raises(_lib.NrgbdError):
        gf(x.double(), y.double())
    with pytest.raises(_lib.NrgbdError):
        gf(x, y.cpu())
    with pytest.raises(_lib.NrgbdError):           # box_filter.py's diff changes the shape below 2r + 1
        BoxFilter(3)(torch.zeros(1, 1, 6, 8, device='cuda'))
    assert gf(x, y).shape == (1, 3, 8, 8)


# ---- end to end on the reference's own module and training loss ---------------------------------------------------
def test_reference_kvnet_dgf_training_step():
    """train_utils/train_KVNet.py's L1 loss with its variance terms on the reference's own KVNET(refineNet_name='DGF'),
    a first window and one steady step, with the f-5 mirrors, depth_var and GuidedFilter patched in: every parameter
    gets a gradient within test_gpu_grad.py's gate of the unpatched reference."""
    res = harness.run_reference_driver('grad', 'gf', timeout=1200)
    harness.parity_dump('gf', 'kvnet_dgf_l1_var', res)
    assert res['restored'] is True
    assert res['dgf_is_mirror'] is True and res['same_state_dict_keys'] is True
    assert res['dgf_calls'] > 0
    assert not res['missing'], res['missing']
    la, lb, lp = res['loss']
    assert abs(lb - la) <= 1e-6 * abs(la) and abs(lp - la) <= 1e-5 * abs(la), res['loss']
    params = res['params']
    assert len(params) == 219, len(params)
    gmax = max(p['max'] for p in params.values())
    rel_floor = max(p['floor'] for p in params.values()) / gmax
    assert rel_floor <= 1e-4, rel_floor
    # The guide MLP's first layer gets its gradient only through GuidedFilter's d x, which A = cov / (var + 1e-8)
    # makes ill-conditioned: on the flat-guide case the reference's own fp32 autograd is 1.9e-2 of the largest d x from
    # the float64 value (PINNING_gf.json), and the mirror is as close to float64 as the reference is. Two fp32 orders can
    # then differ by twice that: 5e-2 there (measured 2.6e-2 on an H100), f-5's 2e-2 everywhere else.
    for n, p in params.items():
        if p['max'] >= 1e-4 * gmax:
            assert p['dev'] <= (5e-2 if n.startswith('r_net.feature_ext.0.') else 2e-2) * p['max'], (n, p)
        else:
            assert p['dev'] <= 2e-5 * gmax, (n, p, gmax)
