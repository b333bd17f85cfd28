"""CPU checks of tests/oracle_stats.py, the numpy restatement of the reference's depth_var and dpv_statistics, and of the
host-side logic of their mirrors in neuralrgbd_b200.mutils.misc:
 * the oracle against the unmodified reference's forward and torch autograd (tests/golden/make_golden_stats.py), at the
   pinned floor, and the max / min plane indices exactly, the tie case's border pixels included;
 * torch.autograd.gradcheck (float64 central differences) of each oracle backward against its float64 forward;
 * the reference's behaviour the mirror keeps: names selected by identity, 'variance' before 'E_mean', 'min' without
   BV_log, the channel concat over N, the asserts."""
import numpy as np
import pytest
import torch

from tests import cases_stats as CS, oracle_stats as OS, harness


gold = harness.golden_fixture('stats_outputs.npz')
pin = harness.pinning_fixture('PINNING_stats.json')


def _check(gold, pin, key, mine):
    p = pin[key]
    assert list(mine.shape) == p['shape']
    # the oracle is deterministic: it reproduces the deviation it was pinned at
    assert np.abs(CS.sub(mine).astype(np.float64) - gold[key]).max() <= p['maxabs_oracle']
    s, want = CS.summary(mine), gold[key + '/stats']
    assert s[2] == want[2] and abs(s[3] - want[3]) <= p['maxabs_oracle']
    assert abs(s[1] - want[1]) <= 1e-5 * want[1]
    assert abs(s[0] - want[0]) <= p['maxabs_oracle'] * want[2]


@pytest.mark.parametrize('name', CS.CASES)
def test_depth_var_vs_reference(gold, pin, name):
    c = CS.case(name)
    mean = c['mean']
    out = OS.depth_var(c['bv'], mean, c['d'], c['log'], c['sigma'])
    assert out.shape == mean.shape                      # the reference's broadcast shape
    _check(gold, pin, 'var/%s/out' % name, out)
    g_bv, g_mu = OS.depth_var_backward(c['g_var'], c['bv'], mean, c['d'], c['log'], c['sigma'])
    assert not g_bv[1:].any()
    _check(gold, pin, 'var/%s/g_bv' % name, g_bv)
    _check(gold, pin, 'var/%s/g_mean' % name, g_mu.reshape(mean.shape))


@pytest.mark.parametrize('name', CS.CASES)
def test_dpv_statistics_vs_reference(gold, pin, name):
    c = CS.case(name)
    feats, parts = OS.dpv_statistics(c['bv'], c['d'], c['stats'], c['log'])
    _check(gold, pin, 'stats/%s/out' % name, feats)
    _check(gold, pin, 'stats/%s/g_bv' % name, OS.dpv_statistics_backward(c['g_stats'], c['bv'], c['d'], parts, c['log']))
    for kind, is_min in (('argmax', False), ('argmin', c['log'])):
        idx = OS.extreme(c['bv'], c['log'], is_min)[1]
        want = gold['stats/%s/%s' % (name, kind)]
        assert np.array_equal((idx if want.shape == idx.shape else CS.sub(idx)).astype(np.uint8), want)


def test_tie_case_has_whole_pixels_of_ties(gold):
    """The prior's border pixels hold D equal planes: the reference picks plane 0 for both max and min there."""
    c = CS.case('prior_pad_120x160_d64')
    border = np.zeros((c['h'], c['w']), bool)
    border[0] = border[-1] = border[:, 0] = border[:, -1] = True
    for kind in ('argmax', 'argmin'):
        idx = gold['stats/prior_pad_120x160_d64/' + kind][0]
        assert idx.shape == border.shape and not idx[border].any()
        assert idx[~border].any()                        # inside, the planes differ


# ---- gradcheck of the oracle backward (float64), small problems --------------------------------------------------
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
    assert torch.autograd.gradcheck(lambda t: _Op.apply(t, fwd, bwd), (x,), eps=1e-6, atol=1e-8, rtol=1e-6)


def _small(log, N=2, D=5, h=3, w=4, seed=7):
    rng = np.random.RandomState(seed)
    bv = rng.uniform(-3.0, -0.5, (N, D, h, w)) if log else rng.uniform(0.05, 0.6, (N, D, h, w))
    return bv, np.linspace(0.5, 3.0, D)


@pytest.mark.parametrize('log', [True, False])
@pytest.mark.parametrize('sigma', [1.0, 0.7])
def test_gradcheck_depth_var(log, sigma):
    bv, d = _small(log)
    N, D, h, w = bv.shape
    mean = np.random.RandomState(8).uniform(0.5, 2.0, (h, w))
    n_bv = bv.size
    x0 = np.concatenate([bv.reshape(-1), mean.reshape(-1)])
    fwd = lambda x: OS.depth_var64(x[:n_bv].reshape(bv.shape), x[n_bv:], d, log, sigma)        # noqa: E731

    def bwd(g, x):
        g_bv, g_mu = OS.depth_var_backward64(g, x[:n_bv].reshape(bv.shape), x[n_bv:], d, log, sigma)
        return np.concatenate([g_bv.reshape(-1), g_mu.reshape(-1)])
    # the backward reads the mean and BV at fp32 as the kernels do: check on fp32-representable inputs
    _gradcheck(x0.astype(np.float32), fwd, bwd)


@pytest.mark.parametrize('log', [True, False])
@pytest.mark.parametrize('is_min', [False, True])
def test_gradcheck_extreme(log, is_min):
    bv, _ = _small(log)
    idx = OS.extreme(bv, log, is_min)[1]
    _gradcheck(bv.astype(np.float32), lambda x: OS.extreme64(x, log, is_min, idx),
               lambda g, x: OS.extreme_backward64(g, x, idx, log))


@pytest.mark.parametrize('log', [True, False])
def test_gradcheck_dpv_statistics(log):
    """The composed backward (regression + variance through its mean + max + min) against central differences of a
    float64 forward over the same composition."""
    bv, d = _small(log, N=1)
    stats = ['E_mean', 'variance', 'max', 'min']
    _, parts = OS.dpv_statistics(bv, d, stats, log)

    def fwd(x):
        p = np.exp(x) if log else x
        dd = d.astype(np.float32).astype(np.float64).reshape(-1, 1, 1)
        mean = (p[0] * dd).sum(0)
        var = OS.depth_var64(x, mean, d, log)
        return np.stack([mean, var, OS.extreme64(x, log, False, parts[2][1])[0],
                         OS.extreme64(x, log, log, parts[3][1])[0]])[None]
    bwd = lambda g, x: OS.dpv_statistics_backward(g, x, d, parts, log).astype(np.float64)       # noqa: E731
    x = torch.from_numpy(bv.astype(np.float32).astype(np.float64)).requires_grad_(True)
    y = _Op.apply(x, fwd, bwd)
    gy = torch.from_numpy(np.random.RandomState(9).standard_normal(y.shape))
    (ga,) = torch.autograd.grad(y, x, gy)
    num = np.zeros_like(bv)
    eps = 1e-6
    for i in range(bv.size):
        e = np.zeros(bv.size); e[i] = eps
        e = e.reshape(bv.shape)
        num.reshape(-1)[i] = ((fwd(x.detach().numpy() + e) - fwd(x.detach().numpy() - e)) * gy.numpy()).sum() / (2 * eps)
    # the composed backward rounds to fp32 once, as the reference's autograd result is fp32
    assert np.abs(ga.numpy() - num).max() <= 1e-6 * np.abs(num).max()


# ---- the reference's behaviour, on the host side ---------------------------------------------------------------------
def _cpu_ops(monkeypatch):
    """Point the mirror's native pieces at the oracle on CPU tensors, so dpv_statistics' own control flow runs here."""
    from neuralrgbd_b200.mutils import misc as M
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))                     # noqa: E731
    monkeypatch.setattr(M, 'depth_val_regression', lambda bv, d, BV_log=True: t(OS.depth_val_regression(bv.numpy(), d, BV_log)))
    monkeypatch.setattr(M, 'depth_var', lambda bv, mean, d, BV_log=True, d_sigma=1.:
                        t(OS.depth_var(bv.numpy(), mean.numpy(), d, BV_log, d_sigma)))
    monkeypatch.setattr(M, '_dpv_extreme', lambda bv, BV_log, is_min: t(OS.extreme(bv.numpy(), BV_log, is_min)[0]))
    return M


@pytest.mark.parametrize('impl', ['oracle', 'mirror'])
def test_reference_quirks(monkeypatch, impl):
    c = CS.case('n2_37x53_d16')
    bv, d = c['bv'], c['d']
    lin = np.exp(bv).astype(np.float32)
    if impl == 'mirror':
        M = _cpu_ops(monkeypatch)
        run = lambda names, x=bv, log=True: M.dpv_statistics(torch.from_numpy(x), d, names, BV_log=log).numpy()   # noqa: E731
    else:
        run = lambda names, x=bv, log=True: OS.dpv_statistics(x, d, names, log)[0]                                # noqa: E731
    # channels in the order asked for; 'max' / 'min' keep every slice of N
    out = run(['max', 'min'])
    assert out.shape == (2, 2, c['h'], c['w'])
    assert np.array_equal(out[:, 0], lin.max(1)) and np.array_equal(out[:, 1], lin.min(1))
    # 'min' without BV_log is the max over the planes (misc.py:603)
    assert np.array_equal(run(['min'], lin, False)[:, 0], lin.max(1))
    # 'variance' needs an 'E_mean' before it
    with pytest.raises(UnboundLocalError):
        run(['variance', 'E_mean'])
    # names are compared by identity: a name built at run time selects nothing
    with pytest.raises(AssertionError, match='No channels in dpv_feats'):
        run([''.join(['E_', 'mean'])])
    with pytest.raises(AssertionError, match='No channels in dpv_feats'):
        run([])
    # E_mean has one slice, max has N: the concat fails for N > 1
    with pytest.raises(RuntimeError):
        run(['E_mean', 'max'])
    # a repeated name gives a repeated channel
    assert run(['max', 'max']).shape == (2, 2, c['h'], c['w'])


def test_mirror_asserts_and_rejects_cpu_tensors():
    from neuralrgbd_b200 import _lib
    from neuralrgbd_b200.mutils import misc as M
    c = CS.case('n2_37x53_d16')
    bv = torch.from_numpy(c['bv'])
    with pytest.raises(AssertionError, match='same # of slices'):
        M.depth_var(bv, torch.zeros(1, c['h'], c['w']), c['d'][:-1])
    with pytest.raises(_lib.NrgbdError):
        M.depth_var(bv, torch.zeros(1, c['h'], c['w']), c['d'])
    with pytest.raises(_lib.NrgbdError):
        M._dpv_extreme(bv, True, False)


def test_patched_into_the_reference_module():
    import neuralrgbd_b200
    syms = dict((r, s) for r, _, s in neuralrgbd_b200._PATCHES)['mutils.misc']
    assert 'depth_var' in syms and 'dpv_statistics' in syms
