"""GPU parity of the tensor-core convolution's tile schedule (csrc/conv_f16.cu): the 8 x 16 output tile on planes whose
height is a multiple of 8 but not 16, and persistent CTAs with fewer and with many more tiles than CTAs (BatchNorm sums
carried across tiles, ring slots released at each tile's end), against the fp32 numpy oracle at the 6e-6 gate of
test_gpu_conv_h2.py. The development flags that switch each of these off must not change a single output bit: every
element accumulates its products in the same order either way (only the BatchNorm sums may differ, by the order of
their atomics)."""
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import kvnet_oracle as N

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731

# nrgbd_dev_conv_h2_set_flags bits: 8 always the 16 x 8 tile, 32 one tile per CTA
SCHED_FLAGS = (8, 32)


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def set_flags(flags):
    from neuralrgbd_b200 import _lib
    _lib.dev_lib().nrgbd_dev_conv_h2_set_flags(flags)


@pytest.fixture(autouse=True)
def _flags_off():
    set_flags(0)
    yield
    set_flags(0)


def check_stats(st, y):
    """The BatchNorm sums against the float64 sums of the stored output (its values are checked against the oracle
    separately), at the gates of test_gpu_conv_h2.py."""
    st = st.cpu().numpy()
    ref = y.cpu().numpy()
    tol1 = 4e-6 * np.abs(ref).max() * np.sqrt(ref[:, 0].size) * 4 + 1e-5
    assert np.abs(st[0] - ref.sum(axis=(0, 2, 3), dtype=np.float64)).max() <= tol1
    assert np.allclose(st[1], np.square(ref.astype(np.float64)).sum(axis=(0, 2, 3)), rtol=2e-5, atol=1e-3)


CFGS = [
    dict(N=2, Cin=64, Cout=64, H=120, W=160, k=3, p=1, d=1),     # layer2 at 640x480: 8 x 16 tiles, two CTAs per SM
    dict(N=3, Cin=128, Cout=128, H=120, W=160, k=3, p=2, d=2),   # layer4: dilation 2, halo pitch 20; BN = 128, 3+ tiles per CTA
    dict(N=1, Cin=96, Cout=96, H=37, W=45, k=3, p=1, d=1),       # ragged in both directions (8 x 16 pads fewer)
    dict(N=1, Cin=67, Cout=67, H=24, W=40, k=3, p=1, d=1),       # Cout 67: BN = 80
    dict(N=1, Cin=32, Cout=48, H=8, W=16, k=3, p=1, d=1),        # one tile: far fewer tiles than CTAs
    dict(N=2, Cin=64, Cout=32, H=40, W=24, k=1, p=0, d=1),       # one box per tap, 8 x 16
]


@pytest.mark.parametrize('cfg', CFGS)
def test_conv2d_h2_sched_vs_oracle(cfg):
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(7)
    x = rng.standard_normal((cfg['N'], cfg['Cin'], cfg['H'], cfg['W'])).astype(np.float32)
    w = (rng.standard_normal((cfg['Cout'], cfg['Cin'], cfg['k'], cfg['k'])) / math.sqrt(cfg['Cin'] * cfg['k'] ** 2)).astype(np.float32)
    b = rng.standard_normal(cfg['Cout']).astype(np.float32)
    ref = N.leaky_relu(N.conv2d(x, w, b, 1, cfg['p'], cfg['d']))
    y, st = convops.conv_h2(T(x), T(w), T(b), 1, cfg['p'], cfg['d'], leaky=True, want_stats=True)
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
    check_stats(st, y)
    # every combination of the development switches: bit-identical outputs, sums within the gate
    for n in range(1, len(SCHED_FLAGS) + 1):
        for combo in itertools.combinations(SCHED_FLAGS, n):
            set_flags(sum(combo))
            y2, st2 = convops.conv_h2(T(x), T(w), T(b), 1, cfg['p'], cfg['d'], leaky=True, want_stats=True)
            assert torch.equal(y2, y), 'flags %d change the output' % sum(combo)
            check_stats(st2, y2)
    set_flags(0)


@pytest.mark.parametrize('cin,cout,hw', [(128, 128, (120, 160)), (67, 67, (37, 45))])
def test_conv2d_h2_pair_output_sched(cin, cout, hw):
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(cin)
    x = rng.standard_normal((1, cin) + hw).astype(np.float32)
    w = (rng.standard_normal((cout, cin, 3, 3)) / math.sqrt(cin * 9)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    ref = N.leaky_relu(N.conv2d(x, w, b, 1, 1, 1))
    y, yh, yl = convops.conv_h2_pair_out(T(x), T(w), T(b), 1, 1, 1, leaky=True)
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
    for flags in (8, 32, 40):
        set_flags(flags)
        y2, yh2, yl2 = convops.conv_h2_pair_out(T(x), T(w), T(b), 1, 1, 1, leaky=True)
        assert torch.equal(yh2, yh) and torch.equal(yl2, yl) and torch.equal(y2, y)
    set_flags(0)


def test_conv_transpose2d_h2_sched():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(3)
    for cin, cout, h, w_ in ((128, 64, 60, 80), (96, 64, 37, 45)):     # parity planes of 120 / 37 rows
        x = rng.standard_normal((1, cin, h, w_)).astype(np.float32)
        w = (rng.standard_normal((cin, cout, 4, 4)) / math.sqrt(cin * 4)).astype(np.float32)
        b = rng.standard_normal(cout).astype(np.float32)
        ref = N.leaky_relu(N.conv_transpose2d(x, w, b, 2, 1))
        y = convops.conv_transpose2d_h2(T(x), T(w), T(b), leaky=True)
        assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
        for flags in (8, 32, 40):
            set_flags(flags)
            assert torch.equal(convops.conv_transpose2d_h2(T(x), T(w), T(b), leaky=True), y)
        set_flags(0)


def test_conv3d_h2_knet_sched():
    """K-Net's 3-D convolution: 3 depth taps per output plane, 120-row planes (8 x 16 tiles), many tiles per CTA."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(4)
    x = rng.standard_normal((1, 64, 6, 40, 48)).astype(np.float32)
    w = (rng.standard_normal((64, 64, 3, 3, 3)) / math.sqrt(64 * 27)).astype(np.float32)
    ref = N.conv3d(x, w)
    y = convops.conv_h2(T(x), T(w), None, 1, 1, 1)
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
    for flags in (8, 32, 40):
        set_flags(flags)
        assert torch.equal(convops.conv_h2(T(x), T(w), None, 1, 1, 1), y)
    set_flags(0)


@pytest.mark.parametrize('cfg', [CFGS[1], CFGS[2], CFGS[3]])
def test_conv2d_tf32_sched_vs_oracle(cfg):
    """The 3xTF32 path launches the same kernel on TF32 pairs."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(8)
    x = rng.standard_normal((cfg['N'], cfg['Cin'], cfg['H'], cfg['W'])).astype(np.float32)
    w = (rng.standard_normal((cfg['Cout'], cfg['Cin'], 3, 3)) / math.sqrt(cfg['Cin'] * 9)).astype(np.float32)
    b = rng.standard_normal(cfg['Cout']).astype(np.float32)
    ref = N.leaky_relu(N.conv2d(x, w, b, 1, cfg['p'], cfg['d']))
    y, st = convops.conv_tc(T(x), T(w), T(b), 1, cfg['p'], cfg['d'], leaky=True, want_stats=True, impl='v2')
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
    check_stats(st, y)
    for flags in (8, 32, 40):
        set_flags(flags)
        y2 = convops.conv_tc(T(x), T(w), T(b), 1, cfg['p'], cfg['d'], leaky=True, impl='v2')
        assert torch.equal(y2, y)
    set_flags(0)
