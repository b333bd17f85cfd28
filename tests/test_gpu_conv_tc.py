"""GPU parity of the wgmma 3xTF32 convolution path against the fp32 numpy oracle, op level.
Expected error of the error-compensated product: ~2^-22 relative per term (vs 2^-11 for plain
TF32), i.e. the same order as an fp32 FFMA chain; gate 6e-6 relative to the output scale."""
import math

import numpy as np
import pytest
import torch

from oracle import kvnet_oracle as N
from tests.conftest import maxabs

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def test_split_tf32_is_exact_to_22_bits():
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(0)
    x = (rng.standard_normal(4096) * np.exp(rng.uniform(-6, 6, 4096))).astype(np.float32)
    hi, lo = convops.split_tf32(T(x))
    hi = hi.cpu().numpy(); lo = lo.cpu().numpy()
    assert (hi.view(np.uint32) & 0x1FFF).max() == 0 and (lo.view(np.uint32) & 0x1FFF).max() == 0
    assert np.abs((hi.astype(np.float64) + lo) - x).max() <= np.abs(x).max() * 2.0 ** -21
    assert (np.abs((hi.astype(np.float64) + lo) - x) <= np.abs(x) * 2.0 ** -21).all()


@pytest.mark.parametrize('cfg', [
    dict(N=1, Cin=32, Cout=32, H=8, W=16, k=1, s=1, p=0, d=1),       # one tile, one K-step
    dict(N=1, Cin=64, Cout=64, H=8, W=16, k=1, s=1, p=0, d=1),       # two K-steps
    dict(N=1, Cin=32, Cout=64, H=16, W=32, k=3, s=1, p=1, d=1),      # taps + halo zero fill
    dict(N=2, Cin=64, Cout=64, H=30, W=40, k=3, s=1, p=1, d=1),      # ragged tiles (layer2 shape)
    dict(N=1, Cin=128, Cout=128, H=20, W=28, k=3, s=1, p=2, d=2),    # layer4 dilation 2
    dict(N=2, Cin=32, Cout=64, H=32, W=48, k=3, s=2, p=1, d=1),      # layer2.0.conv1 stride 2
    dict(N=2, Cin=32, Cout=64, H=32, W=48, k=1, s=2, p=0, d=1),      # layer2.0.downsample
    dict(N=1, Cin=320, Cout=128, H=16, W=24, k=3, s=1, p=1, d=1),    # lastconv.0
    dict(N=1, Cin=96, Cout=96, H=24, W=32, k=3, s=1, p=1, d=1),      # R-Net conv1
    dict(N=1, Cin=67, Cout=67, H=24, W=36, k=3, s=1, p=1, d=1),      # R-Net conv2 (padded to 96 / 80)
    dict(N=3, Cin=128, Cout=32, H=1, W=2, k=1, s=1, p=0, d=1),       # SPP branch on a 1x2 map
])
@pytest.mark.parametrize('impl', ['v1', 'v2'])
def test_conv2d_tc_vs_oracle(cfg, impl):
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(1)
    x = rng.standard_normal((cfg['N'], cfg['Cin'], cfg['H'], cfg['W'])).astype(np.float32)
    w = (rng.standard_normal((cfg['Cout'], cfg['Cin'], cfg['k'], cfg['k'])) / math.sqrt(cfg['Cin'] * cfg['k'] ** 2)).astype(np.float32)
    b = rng.standard_normal(cfg['Cout']).astype(np.float32)
    y, st = convops.conv_tc(T(x), T(w), T(b), cfg['s'], cfg['p'], cfg['d'], leaky=True, want_stats=True, impl=impl)
    torch.cuda.synchronize()
    ref = N.leaky_relu(N.conv2d(x, w, b, cfg['s'], cfg['p'], cfg['d']))
    assert y.shape == ref.shape
    assert rel_err(y.cpu().numpy(), ref) <= 6e-6
    st = st.cpu().numpy()
    # the statistics are sums of the stored outputs: their error is bounded by the summed per-element error
    tol1 = 4e-6 * np.abs(ref).max() * np.sqrt(ref[:, 0].size) * 4 + 1e-5
    assert np.abs(st[0] - ref.sum(axis=(0, 2, 3), dtype=np.float64)).max() <= tol1
    assert np.allclose(st[1], np.square(ref.astype(np.float64)).sum(axis=(0, 2, 3)), rtol=2e-5, atol=1e-3)
    got_sum = y.double().sum(dim=(0, 2, 3)).cpu().numpy()          # stats must equal the sums of what was stored
    assert np.abs(st[0] - got_sum).max() <= 1e-3 * max(1.0, np.abs(got_sum).max()) * 1e-2


@pytest.mark.parametrize('impl', ['v1', 'v2'])
def test_conv3d_tc_vs_oracle(impl):
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(2)
    for cin, cout in ((16, 64), (64, 64), (64, 1)):
        x = rng.standard_normal((1, cin, 9, 14, 18)).astype(np.float32)
        w = (rng.standard_normal((cout, cin, 3, 3, 3)) / math.sqrt(cin * 27)).astype(np.float32)
        y = convops.conv_tc(T(x), T(w), None, 1, 1, 1, impl=impl)
        ref = N.conv3d(x, w)
        assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6


@pytest.mark.parametrize('impl', ['v1', 'v2'])
def test_conv_transpose2d_tc_vs_oracle(impl):
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(3)
    for cin, cout, h, w_ in ((128, 64, 9, 13), (96, 64, 16, 20)):
        x = rng.standard_normal((1, cin, h, w_)).astype(np.float32)
        w = (rng.standard_normal((cin, cout, 4, 4)) / math.sqrt(cin * 4)).astype(np.float32)
        b = rng.standard_normal(cout).astype(np.float32)
        y = convops.conv_transpose2d_tc(T(x), T(w), T(b), leaky=True, impl=impl)
        ref = N.leaky_relu(N.conv_transpose2d(x, w, b, 2, 1))
        assert y.shape == ref.shape and rel_err(y.cpu().numpy(), ref) <= 6e-6


def test_tc_matches_fp32_simt_path():
    """The two conv paths of the engine agree to fp32 rounding on the same input."""
    from neuralrgbd_b200 import convops
    rng = np.random.RandomState(4)
    x = rng.standard_normal((2, 64, 24, 40)).astype(np.float32)
    w = (rng.standard_normal((64, 64, 3, 3)) / 24.0).astype(np.float32)
    a = convops.conv(T(x), T(w), None, 1, 1, 1).cpu().numpy()
    b = convops.conv_tc(T(x), T(w), None, 1, 1, 1).cpu().numpy()
    assert rel_err(b, a) <= 6e-6
    c = convops.conv_tc(T(x), T(w), None, 1, 1, 1, impl='v2').cpu().numpy()
    assert rel_err(c, a) <= 6e-6


@pytest.mark.parametrize('shape', [(1, 64, 480, 640, 64), (1, 96, 240, 320, 96), (5, 128, 120, 160, 128)])
def test_tc2_large_images_repeatable(shape):
    """Many waves of CTAs on HBM-resident inputs: the shared-memory rings are recycled
    hundreds of times per SM with irregular TMA latencies. A slot released before its readers had finished
    showed up only here (a few corrupt tiles per launch), never on the small oracle-sized cases."""
    from neuralrgbd_b200 import convops
    n, cin, h, w_, cout = shape
    g = torch.Generator(device='cuda').manual_seed(11)
    x = torch.randn((n, cin, h, w_), device='cuda', generator=g)
    w = torch.randn((cout, cin, 3, 3), device='cuda', generator=g) / math.sqrt(cin * 9)
    ref = convops.conv(x, w, None, 1, 1, 1)
    scale = float(ref.abs().max())
    for _ in range(3):
        y = convops.conv_tc(x, w, None, 1, 1, 1, impl='v2')
        assert float((y - ref).abs().max()) <= 1e-5 * scale


@pytest.mark.parametrize('cfg', [dict(N=2, C=64, H=24, W=40, Co=64, s=1, p=1, d=1), dict(N=1, C=32, H=37, W=53, Co=32, s=1, p=1, d=1),
                                 dict(N=5, C=128, H=30, W=40, Co=128, s=1, p=2, d=2), dict(N=2, C=32, H=48, W=64, Co=64, s=2, p=1, d=1),
                                 dict(N=1, C=67, H=40, W=56, Co=64, s=1, p=1, d=1)])
def test_conv_with_fused_input_batchnorm(cfg):
    """BasicBlock's conv1 -> BN(batch statistics) -> ReLU -> conv2 with the BN+ReLU folded into conv2's operand converter
    (psm_submodule.py:31-49): bit-identical to the stand-alone BN pass followed by the same convolution - the operands
    the tensor core sees are the same floats - including the zero padding and the running-statistics update."""
    from neuralrgbd_b200 import convops
    g = torch.Generator(device='cuda').manual_seed(21)
    x = torch.randn((cfg['N'], 32, cfg['H'], cfg['W']), device='cuda', generator=g)
    w1 = torch.randn((cfg['C'], 32, 3, 3), device='cuda', generator=g) / math.sqrt(32 * 9)
    w2 = torch.randn((cfg['Co'], cfg['C'], 3, 3), device='cuda', generator=g) / math.sqrt(cfg['C'] * 9)
    gamma = torch.rand(cfg['C'], device='cuda', generator=g) + 0.5
    beta = torch.randn(cfg['C'], device='cuda', generator=g) * 0.3
    y1, st1 = convops.conv_tc(x, w1, None, 1, 1, 1, want_stats=True, impl='v2')         # raw conv1 output + its sums
    ref_in = convops.batch_norm(y1, st1, gamma, beta, relu=True)
    want, st_want = convops.conv_tc(ref_in, w2, None, cfg['s'], cfg['p'], cfg['d'], want_stats=True, impl='v2')
    rm = torch.zeros(cfg['C'], device='cuda'); rv = torch.ones(cfg['C'], device='cuda')
    got, st_got = convops.conv_tc_bn_in(y1, st1, gamma, beta, w2, None, cfg['s'], cfg['p'], cfg['d'], relu=True, want_stats=True,
                                        running=(rm, rv))
    assert torch.equal(got, want)
    assert float((st_got - st_want).abs().max()) <= 1e-9 * float(st_want.abs().max())
    # running statistics as torch's training-mode BatchNorm updates them (momentum 0.1, unbiased variance)
    mean = y1.mean(dim=(0, 2, 3)); var = y1.var(dim=(0, 2, 3), unbiased=True)
    assert float((rm - 0.1 * mean).abs().max()) <= 1e-6 and float((rv - (0.9 + 0.1 * var)).abs().max()) <= 1e-5
    # and against torch itself (fp32 reference of the whole fused op)
    import torch.nn.functional as F
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):        # cuDNN defaults to TF32 convolutions
        t = F.conv2d(F.relu(F.batch_norm(y1, None, None, gamma, beta, True, 0.1, 1e-5)), w2, None, cfg['s'], cfg['p'], cfg['d'])
    assert float((got - t).abs().max()) <= 2e-5 * float(t.abs().max())
