"""GPU parity of the second-generation tensor-core convolution (csrc/conv_f16.cu: wgmma on split-fp16
operand pairs, halo tile) against the fp32 numpy oracle, op level. The pair product keeps 22 significand bits per
operand like 3xTF32, so the same 6e-6 gate (relative to the output scale) applies."""
import math

import numpy as np
import pytest
import torch

from oracle import kvnet_oracle as N

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def test_split_f16_pair_keeps_22_bits():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(0)
    x = (rng.standard_normal(8192) * np.exp(rng.uniform(-9, 9, 8192))).astype(np.float32)
    x[:8] = [0.0, -0.0, 1.0, -1.0, 65504.0, 1e-7, 3e-5, -2.5e-6]
    hi, lo = convops.split_f16_pair(T(x))
    rec = hi.cpu().numpy().astype(np.float64) + lo.cpu().numpy().astype(np.float64) / 2048.0
    inr = np.abs(x) <= 60000
    err = np.abs(rec - x)[inr]
    assert (err <= np.abs(x[inr]) * 2.0 ** -21 + 2.0 ** -35).all()        # relative 2^-22 (+ the fp16 subnormal floor)
    big = T(np.array([1e6, -3e38, 7e4, 65504.0], np.float32))
    h2, l2 = convops.split_f16_pair(big)
    assert torch.isfinite(h2).all() and torch.isfinite(l2).all()           # saturates instead of producing inf


CFGS = [
    dict(N=1, Cin=32, Cout=32, H=16, W=8, k=1, s=1, p=0, d=1),       # one tile, one chunk, no halo
    dict(N=1, Cin=64, Cout=64, H=16, W=8, k=1, s=1, p=0, d=1),       # two chunks
    dict(N=1, Cin=32, Cout=64, H=16, W=32, k=3, s=1, p=1, d=1),      # halo tile + zero fill at the borders
    dict(N=2, Cin=64, Cout=64, H=30, W=40, k=3, s=1, p=1, d=1),      # ragged tiles (layer2 shape)
    dict(N=1, Cin=128, Cout=128, H=20, W=28, k=3, s=1, p=2, d=2),    # layer4 dilation 2 (halo pitch 12)
    dict(N=2, Cin=32, Cout=64, H=32, W=48, k=3, s=2, p=1, d=1),      # layer2.0.conv1 stride 2 (one box per tap)
    dict(N=2, Cin=32, Cout=64, H=32, W=48, k=1, s=2, p=0, d=1),      # layer2.0.downsample
    dict(N=1, Cin=320, Cout=128, H=16, W=24, k=3, s=1, p=1, d=1),    # lastconv.0
    dict(N=1, Cin=96, Cout=96, H=24, W=32, k=3, s=1, p=1, d=1),      # R-Net conv1
    dict(N=1, Cin=67, Cout=67, H=24, W=36, k=3, s=1, p=1, d=1),      # R-Net conv2 (padded to 96 / 80)
    dict(N=3, Cin=128, Cout=32, H=1, W=2, k=1, s=1, p=0, d=1),       # SPP branch on a 1x2 map
    dict(N=1, Cin=192, Cout=192, H=20, W=24, k=3, s=1, p=1, d=1),    # R-Net at D=128: Cout split into two chunks of 96
    dict(N=1, Cin=320, Cout=320, H=18, W=16, k=3, s=1, p=1, d=1),    # R-Net at D=256: three chunks of 112
    dict(N=1, Cin=259, Cout=256, H=17, W=20, k=3, s=1, p=1, d=1),    # R-Net conv2_1 at D=256
]


@pytest.mark.parametrize('cfg', CFGS)
def test_conv2d_h2_vs_oracle(cfg):
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(1)
    x = rng.standard_normal((cfg['N'], cfg['Cin'], cfg['H'], cfg['W'])).astype(np.float32)
    w = (rng.standard_normal((cfg['Cout'], cfg['Cin'], cfg['k'], cfg['k'])) / math.sqrt(cfg['Cin'] * cfg['k'] ** 2)).astype(np.float32)
    b = rng.standard_normal(cfg['Cout']).astype(np.float32)
    y, st = convops.conv_h2(T(x), T(w), T(b), cfg['s'], cfg['p'], cfg['d'], leaky=True, want_stats=True)
    torch.cuda.synchronize()
    ref = N.leaky_relu(N.conv2d(x, w, b, cfg['s'], cfg['p'], cfg['d']))
    assert y.shape == ref.shape
    assert rel_err(y.cpu().numpy(), ref) <= 6e-6
    st = st.cpu().numpy()
    tol1 = 4e-6 * np.abs(ref).max() * np.sqrt(ref[:, 0].size) * 4 + 1e-5
    assert np.abs(st[0] - ref.sum(axis=(0, 2, 3), dtype=np.float64)).max() <= tol1
    assert np.allclose(st[1], np.square(ref.astype(np.float64)).sum(axis=(0, 2, 3)), rtol=2e-5, atol=1e-3)


def test_conv3d_h2_vs_oracle():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(2)
    for cin, cout in ((16, 64), (28, 64), (64, 64), (64, 1)):
        x = rng.standard_normal((1, cin, 9, 14, 18)).astype(np.float32)
        w = (rng.standard_normal((cout, cin, 3, 3, 3)) / math.sqrt(cin * 27)).astype(np.float32)
        y = convops.conv_h2(T(x), T(w), None, 1, 1, 1)
        ref = N.conv3d(x, w)
        assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6


def test_conv3d_single_output_channel_tap_gather_vs_oracle():
    """K-Net's last layer (Conv3d(f -> 1, k3), models/basic.py:136-137) in the form the engine runs it: a pointwise conv to one
    channel per tap on the tensor cores + the shifted sum of the taps. Ragged extents exercise every border case of the gather."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(12)
    for cin, shape in ((64, (9, 14, 18)), (28, (5, 33, 41)), (64, (3, 8, 32)), (64, (1, 9, 37))):
        x = rng.standard_normal((1, cin) + shape).astype(np.float32)
        w = (rng.standard_normal((1, cin, 3, 3, 3)) / math.sqrt(cin * 27)).astype(np.float32)
        y = convops.conv_cout1_h2(T(x), T(w))
        ref = N.conv3d(x, w)
        assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
    x = rng.standard_normal((2, 32, 17, 45)).astype(np.float32)          # 2-D form, batch of two
    w = (rng.standard_normal((1, 32, 3, 3)) / math.sqrt(32 * 9)).astype(np.float32)
    y = convops.conv_cout1_h2(T(x), T(w), bias=0.25)
    ref = N.conv2d(x, w, np.array([0.25], np.float32), 1, 1, 1)
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6


@pytest.mark.parametrize('cin,cout,hw', [(128, 128, (30, 40)), (96, 96, (37, 45)), (67, 67, (33, 24)), (64, 64, (16, 8)), (192, 160, (20, 19)),
                                          (131, 131, (18, 25))])
def test_conv2d_h2_pair_output_vs_oracle(cin, cout, hw):
    """R-Net's conv -> conv chains (models/Refine.py:79-107: 3x3 conv + bias + LeakyReLU): the epilogue writes the operand pair
    of the next convolution directly. The pair's value must match the oracle like the fp32 output does, the pad channels must
    be written as zeros, and the halves must be exactly the split of a value (lo within the residual range)."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(cin + cout)
    x = rng.standard_normal((1, cin) + hw).astype(np.float32)
    w = (rng.standard_normal((cout, cin, 3, 3)) / math.sqrt(cin * 9)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    y, yh, yl = convops.conv_h2_pair_out(T(x), T(w), T(b), 1, 1, 1, leaky=True)
    ref = N.conv2d(x, w, b, 1, 1, 1)
    ref = np.where(ref >= 0, ref, ref * np.float32(0.01))
    assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6
    yh_, yl_ = yh.float().cpu().numpy(), yl.float().cpu().numpy()
    assert np.isfinite(yh_).all() and np.isfinite(yl_).all()                  # every element written, pad channels included
    assert not yh_[..., cout:].any() and not yl_[..., cout:].any()
    assert (np.abs(yl_) <= np.maximum(np.abs(yh_), 0.125) * 1.0001).all()        # |lo| <= ulp(hi)/2 * 2^11 <= |hi|


def test_conv_transpose2d_h2_vs_oracle():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(3)
    for cin, cout, h, w_ in ((128, 64, 9, 13), (96, 64, 16, 20), (192, 128, 10, 12), (320, 256, 9, 8)):
        x = rng.standard_normal((1, cin, h, w_)).astype(np.float32)
        w = (rng.standard_normal((cin, cout, 4, 4)) / math.sqrt(cin * 4)).astype(np.float32)
        b = rng.standard_normal(cout).astype(np.float32)
        y = convops.conv_transpose2d_h2(T(x), T(w), T(b), leaky=True)
        ref = N.leaky_relu(N.conv_transpose2d(x, w, b, 2, 1))
        assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6


@pytest.mark.parametrize('shape', [(1, 64, 480, 640, 64), (1, 96, 240, 320, 96), (5, 128, 120, 160, 128), (5, 32, 240, 320, 32)])
def test_h2_large_images_repeatable(shape):
    """Many waves of CTAs on HBM-resident inputs (the regime where ring-recycling races show up)."""
    from neuralrgbd_b200 import convops
    n, cin, h, w_, cout = shape
    g = torch.Generator(device='cuda').manual_seed(11)
    x = torch.randn((n, cin, h, w_), device='cuda', generator=g)
    w = torch.randn((cout, cin, 3, 3), device='cuda', generator=g) / math.sqrt(cin * 9)
    ref = convops.conv(x, w, None, 1, 1, 1)
    scale = float(ref.abs().max())
    first = None
    for _ in range(3):
        y = convops.conv_h2(x, w, None, 1, 1, 1)
        assert float((y - ref).abs().max()) <= 1e-5 * scale
        if first is None:
            first = y
        else:
            assert torch.equal(y, first)
