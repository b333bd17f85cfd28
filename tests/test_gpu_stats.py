"""The depth_var and dpv_statistics mirrors on the device (mutils/misc.py:550-608).

 * Each kernel against tests/oracle_stats.py and against the unmodified reference's forward and torch autograd
   (tests/golden/make_golden_stats.py), gated from the oracle-vs-reference floor pinned in PINNING_stats.json.
 * The plane indices of 'max' / 'min' equal the reference's on the tie case; E_mean inside dpv_statistics is
   depth_val_regression's, bit for bit.
 * Plain inputs, inputs that require grad and torch.no_grad() give the same launches and bit-identical values.
 * A tensor on a second device stays there.
 * The reference's own models.KVNET.KVNET(refineNet_name='DGF') trained with train_utils/train_KVNet.py's L1 loss,
   variance terms included, with the mirrors patched in, against the unpatched reference (tests/reference_driver.py grad stats).
Measured deviations are written to $NRGBD_PARITY_DIR/parity_stats.json when that variable is set.
"""
import numpy as np
import pytest
import torch

from tests import cases_stats as CS, oracle_stats as OS, harness

pytestmark = pytest.mark.gpu
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731

# Gates, relative to the largest reference value of the array, on top of the pinned oracle-vs-reference floor. No kernel
# uses atomics; the forwards round every operation as the reference does, so they differ from the fp32 oracle only by
# expf against numpy's exp (a few ulp of each probability). That moves a squared term by about 2|x|·δx and the variance
# by a few 1e-7 of its largest value: 2e-6. The backwards chain four or five fp32 roundings per element against the
# oracle's float64 (1e-6 of an element); the mean's gradient sums D of them in fp32 (D ulp of the partial sum, 1e-5), and
# dpv_statistics' gradient adds four channels' terms (1e-5).
REL = {'var/out': 2e-6, 'var/g_bv': 2e-6, 'var/g_mean': 1e-5, 'stats/out': 1e-5, 'stats/g_bv': 1e-5}


gold = harness.golden_fixture('stats_outputs.npz')
pin = harness.pinning_fixture('PINNING_stats.json')


def _gate(gold, pin, key, mine, orc):
    kind = '/'.join(key.split('/')[::2])          # 'var/<case>/g_bv' -> 'var/g_bv'
    p = pin[key]
    allow = REL[kind] * p['max_ref']
    e_orc = float(np.abs(mine.astype(np.float64) - orc).max())
    e_ref = float(np.abs(CS.sub(mine).astype(np.float64) - gold[key]).max())
    s, want = CS.summary(mine), gold[key + '/stats']
    harness.parity_dump('stats', key, {'vs_oracle': e_orc, 'vs_reference_sample': e_ref, 'floor': p['maxabs_oracle'], 'max_ref': p['max_ref'],
                'gate': allow})
    assert list(mine.shape) == p['shape']
    assert e_orc <= allow, (key, e_orc, allow)
    assert e_ref <= p['maxabs_oracle'] + allow, (key, e_ref, p['maxabs_oracle'] + allow)
    assert s[2] == want[2]
    assert abs(s[3] - want[3]) <= p['maxabs_oracle'] + allow
    assert abs(s[1] - want[1]) <= 1e-5 * want[1]
    assert abs(s[0] - want[0]) <= (p['maxabs_oracle'] + allow) * want[2]


@pytest.mark.parametrize('name', CS.CASES)
def test_depth_var(gold, pin, name):
    from neuralrgbd_b200.mutils import misc as M
    c = CS.case(name)
    bv, mean = T(c['bv']).requires_grad_(True), T(c['mean']).requires_grad_(True)
    out = M.depth_var(bv, mean, c['d'], BV_log=c['log'], d_sigma=c['sigma'])
    assert out.shape == mean.shape and out.device == bv.device
    out.backward(T(c['g_var']))
    g_bv, g_mu = OS.depth_var_backward(c['g_var'], c['bv'], c['mean'], c['d'], c['log'], c['sigma'])
    key = 'var/' + name
    _gate(gold, pin, key + '/out', out.detach().cpu().numpy(), OS.depth_var(c['bv'], c['mean'], c['d'], c['log'], c['sigma']))
    mine = bv.grad.cpu().numpy()
    assert not mine[1:].any()
    _gate(gold, pin, key + '/g_bv', mine, g_bv)
    _gate(gold, pin, key + '/g_mean', mean.grad.cpu().numpy(), g_mu.reshape(c['mean'].shape))


@pytest.mark.parametrize('name', CS.CASES)
def test_dpv_statistics(gold, pin, name):
    from neuralrgbd_b200.mutils import misc as M
    c = CS.case(name)
    bv = T(c['bv']).requires_grad_(True)
    feats = M.dpv_statistics(bv, c['d'], c['stats'], BV_log=c['log'])
    feats.backward(T(c['g_stats']))
    of, parts = OS.dpv_statistics(c['bv'], c['d'], c['stats'], c['log'])
    key = 'stats/' + name
    _gate(gold, pin, key + '/out', feats.detach().cpu().numpy(), of)
    _gate(gold, pin, key + '/g_bv', bv.grad.cpu().numpy(), OS.dpv_statistics_backward(c['g_stats'], c['bv'], c['d'], parts, c['log']))
    if 'E_mean' in c['stats']:
        with torch.no_grad():
            assert torch.equal(feats[:, c['stats'].index('E_mean')], M.depth_val_regression(bv, c['d'], BV_log=c['log']))


@pytest.mark.parametrize('name', CS.CASES)
def test_extreme_indices(gold, name):
    """On the tie case the kernel's planes are the reference's, every pixel. Elsewhere a plane may differ only where
    expf and the CPU's exp round two planes' probabilities into the other order: the selected values then agree."""
    from neuralrgbd_b200.mutils import misc as M
    c = CS.case(name)
    p = np.exp(c['bv'].astype(np.float64)) if c['log'] else c['bv'].astype(np.float64)
    for kind, is_min in (('argmax', False), ('argmin', c['log'])):
        val, idx = M._extreme_forward(T(c['bv']), c['log'], is_min, True)
        idx = idx.cpu().numpy()
        want = gold['stats/%s/%s' % (name, kind)].astype(np.int64)
        got = idx if want.shape == idx.shape else CS.sub(idx)
        if name == 'prior_pad_120x160_d64':
            assert np.array_equal(got, want), (kind, int((got != want).sum()))
        else:
            st = -(-c['h'] // want.shape[-2])                  # the stride cases_stats.sub chose for the index map
            ps = p[..., ::st, ::st]
            assert ps.shape[-2:] == want.shape[-2:]
            a = np.take_along_axis(ps, got[:, None], 1)[:, 0]
            b = np.take_along_axis(ps, want[:, None], 1)[:, 0]
            assert np.abs(a - b).max() <= 1e-6 * np.abs(p).max()
            harness.parity_dump('stats', 'index/%s/%s' % (name, kind), {'mismatch_sample': int((got != want).sum())})


def test_extreme_nan_and_ties():
    """ATen's CPU max.dim / min.dim rules: the first NaN wins, ties keep the first plane."""
    from neuralrgbd_b200.mutils import misc as M
    x = np.array([[1., 3., 3., 2.], [1., np.nan, 5., np.nan], [0.5, 0.5, 0.2, 0.2], [np.nan, 1., 1., 1.]], np.float32)
    bv = x.T.reshape(1, 4, 2, 2).copy()
    for is_min in (False, True):
        want = torch.min if is_min else torch.max
        v, i = want(torch.from_numpy(bv), dim=1)
        gv, gi = M._extreme_forward(T(bv), False, is_min, True)
        assert torch.equal(gi.cpu().long(), i)
        np.testing.assert_array_equal(gv.cpu().numpy(), v.numpy())          # NaN where ATen has NaN


# ---- the no-grad path -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('op', ['depth_var', 'dpv_statistics'])
def test_no_grad_path_unchanged(op):
    from neuralrgbd_b200.mutils import misc as M
    c = CS.case('sharp_120x160_d64')
    mean = T(c['mean'])
    if op == 'depth_var':
        fn, want = (lambda rg: M.depth_var(T(c['bv']).requires_grad_(rg), mean, c['d'])), 1
    else:
        fn, want = (lambda rg: M.dpv_statistics(T(c['bv']).requires_grad_(rg), c['d'], CS.ALL_STATS)), 4
    n0, plain = harness.launch_count(lambda: fn(False))
    with torch.no_grad():
        n1, nog = harness.launch_count(lambda: fn(True))
    n2, withgrad = harness.launch_count(lambda: fn(True))
    assert n0 == n1 == n2 == want, (n0, n1, n2, want)
    assert plain.grad_fn is None and nog.grad_fn is None and withgrad.requires_grad
    assert torch.equal(plain, nog) and torch.equal(plain, withgrad.detach())


def test_mean_only_requires_grad():
    """A mean that requires grad on its own gets the gradient; BV_measure gets none."""
    from neuralrgbd_b200.mutils import misc as M
    c = CS.case('mean_hw_120x160_d64')
    bv, mean = T(c['bv']), T(c['mean']).requires_grad_(True)
    M.depth_var(bv, mean, c['d']).backward(T(c['g_var']))
    g_mu = OS.depth_var_backward(c['g_var'], c['bv'], c['mean'], c['d'])[1]
    assert bv.grad is None
    assert np.abs(mean.grad.cpu().numpy() - g_mu).max() <= REL['var/g_mean'] * np.abs(g_mu).max()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs a second visible CUDA device')
def test_second_device_stays_put():
    from neuralrgbd_b200.mutils import misc as M
    c = CS.case('n2_37x53_d16')
    dev = torch.device('cuda:1')
    bv = torch.from_numpy(c['bv']).to(dev).requires_grad_(True)
    var = M.depth_var(bv, torch.from_numpy(c['mean']).to(dev), c['d'])
    feats = M.dpv_statistics(bv, c['d'], ['max', 'min'])
    assert var.device == dev and feats.device == dev
    (var.sum() + feats.sum()).backward()
    assert bv.grad.device == dev
    ref = M.depth_var(T(c['bv']), T(c['mean']), c['d'])
    assert torch.equal(var.detach().cpu(), ref.cpu())


# ---- end to end on the reference's own module and training loss ---------------------------------------------------
def test_reference_kvnet_l1_loss_with_variance():
    """train_utils/train_KVNet.py's L1 loss, with weight_var * (var(kv_dpv) + var(d_dpv)), on the reference's own
    KVNET(refineNet_name='DGF') for a first window and one steady step: with the f-5 mirrors and depth_var patched in,
    every parameter gets a gradient and it matches the unpatched reference. The variance terms on their own reach every
    D-Net and K-Net parameter only through depth_var and depth_val_regression: they are checked separately."""
    res = harness.run_reference_driver('grad', 'stats', timeout=1200)
    harness.parity_dump('stats', 'kvnet_dgf_l1_var', res)
    assert res['restored'] is True
    for part in ('full', 'var_only'):
        rr = res[part]
        assert not rr['missing'], (part, rr['missing'])
        la, lb, lp = rr['loss']
        assert abs(lb - la) <= 1e-6 * abs(la) and abs(lp - la) <= 1e-5 * abs(la), (part, rr['loss'])
        params = rr['params']
        assert len(params) > (200 if part == 'full' else 100), (part, len(params))
        # Gate as test_gpu_grad.py's (same model, same mirrors): 2e-2 of each parameter's largest gradient, 2e-5 of the
        # largest overall for parameters whose gradient is zero up to rounding. B - A (two unpatched runs) is the floor.
        gmax = max(p['max'] for p in params.values())
        rel_floor = max(p['floor'] for p in params.values()) / gmax
        assert rel_floor <= 1e-4, (part, rel_floor)
        for n, p in params.items():
            if p['max'] >= 1e-4 * gmax:
                assert p['dev'] <= 2e-2 * p['max'], (part, n, p)
            else:
                assert p['dev'] <= 2e-5 * gmax, (part, n, p, gmax)
    # the variance terms reach D-Net and K-Net, not R-Net
    assert not any(n.startswith('r_net.') for n in res['var_only']['params'])
    assert any(n.startswith('kv_net.') for n in res['var_only']['params'])
