"""numpy restatement of KVNET's guided-filter refinement (refineNet_name='DGF', models/KVNET.py:129-132,176-178):
depth_val_regression of the low-resolution log-DPV, RefineNet_DGF (models/Refine.py:620-641) and GuidedFilter / BoxFilter
(models/GF/guided_filter.py, models/GF/box_filter.py), in the reference's fp32 arithmetic on the CPU:

  * bilinear align-corners upsample: fp32 source index and weights, taps combined as fma(hx, v00, lx*v01), then
    fma(hy, row0, ly*row1) (ATen's CPU kernel);
  * the 1x1 convolutions: accumulator starts at the bias, one FMA per input channel in order (ATen's CPU convolution);
  * cumsum: double accumulation, every prefix rounded to fp32 (ATen's float cumsum); diff_x / diff_y index formulas verbatim;
  * everything else one IEEE fp32 operation at a time.

An FMA is emulated as the exact double product plus the addend, rounded once to fp32 (the product of two fp32 values is exact
in double; the double rounding of the sum is the only departure, and it has not been met on the fixtures).
"""
import numpy as np

from oracle import planesweep_oracle as O

f32 = np.float32


def fma32(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def upsample_ac(x, ratio):
    """F.upsample(x[None, None], scale_factor=ratio, mode='bilinear', align_corners=True)[0, 0] for x [h][w]."""
    x = np.asarray(x, f32)
    h, w = x.shape
    H, W = h * ratio, w * ratio

    def axis(n, N):
        s = f32(n - 1) / f32(N - 1) if n > 1 else f32(0)
        src = (f32(s) * np.arange(N, dtype=f32)).astype(f32)
        i0 = np.minimum(np.floor(src).astype(np.int64), n - 1)
        i1 = i0 + (i0 < n - 1)
        lam = np.clip(src - i0.astype(f32), 0, 1).astype(f32)
        return i0, i1, (f32(1) - lam).astype(f32), lam
    y0, y1, hy, ly = axis(h, H)
    x0, x1, hx, lx = axis(w, W)
    hy, ly, hx, lx = hy[:, None], ly[:, None], hx[None, :], lx[None, :]
    r0 = fma32(hx, x[y0][:, x0], (lx * x[y0][:, x1]).astype(f32))
    r1 = fma32(hx, x[y1][:, x0], (lx * x[y1][:, x1]).astype(f32))
    return fma32(hy, r0, (ly * r1).astype(f32))


def feature_ext(img, w0, b0, w1, b1):
    """Conv2d(64->1, 1x1)(ReLU(Conv2d(3->64, 1x1)(img))) for img [3][H][W]; weights as stored in the state_dict."""
    img = np.asarray(img, f32)
    w0 = np.asarray(w0, f32).reshape(-1, 3); w1 = np.asarray(w1, f32).reshape(-1)
    x = np.full(img.shape[1:], f32(np.asarray(b1).reshape(-1)[0]), f32)
    for k in range(w0.shape[0]):
        a = np.full(img.shape[1:], f32(np.asarray(b0)[k]), f32)
        for c in range(3):
            a = fma32(w0[k, c], img[c], a)
        x = fma32(w1[k], np.maximum(a, f32(0)), x)
    return x


def _diff(cs, r, axis):
    """box_filter.py diff_x (axis 0) / diff_y (axis 1): cat(left, middle, right) of the prefix sums."""
    c = np.moveaxis(cs, axis, 0)
    left = c[r:2 * r + 1]
    middle = c[2 * r + 1:] - c[:-2 * r - 1]
    right = c[-1:] - c[-2 * r - 1:-r - 1]
    return np.moveaxis(np.concatenate([left, middle, right], 0), 0, axis).astype(f32)


def cumsum32(x, axis):
    return np.cumsum(np.asarray(x, np.float64), axis=axis).astype(f32)


def box_filter(x, r):
    """BoxFilter(r).forward for one [H][W] plane."""
    return _diff(cumsum32(_diff(cumsum32(x, 0), r, 0), 1), r, 1)


def guided_filter(x, y, r=1, eps=1e-8):
    """GuidedFilter(r, eps).forward(x, y) for [H][W] planes."""
    x = np.asarray(x, f32); y = np.asarray(y, f32)
    H, W = x.shape
    assert H > 2 * r + 1 and W > 2 * r + 1
    N = box_filter(np.ones((H, W), f32), r)
    mean_x = box_filter(x, r) / N
    mean_y = box_filter(y, r) / N
    cov_xy = box_filter(x * y, r) / N - mean_x * mean_y
    var_x = box_filter(x * x, r) / N - mean_x * mean_x
    A = cov_xy / (var_x + f32(eps))
    b = mean_y - A * mean_x
    mean_A = box_filter(A, r) / N
    mean_b = box_filter(b, r) / N
    return (mean_A * x + mean_b).astype(f32)


def dgf_refine(dmap, img, sd, pre='r_net.'):
    """RefineNet_DGF.forward(dmap [h][w], img [3][H][W]) -> [H][W]."""
    ratio = img.shape[1] // dmap.shape[0]
    y = upsample_ac(dmap, ratio)
    x = feature_ext(img, sd[pre + 'feature_ext.0.weight'], sd[pre + 'feature_ext.0.bias'], sd[pre + 'feature_ext.2.weight'],
                    sd[pre + 'feature_ext.2.bias'])
    return guided_filter(x, y, 1, 1e-8)


# ---- seeded inputs of the guided filter alone (tests/golden/make_golden.py refine, tests/test_gpu_refine.py) -----------
GF_CASES = ['gf_ragged_13x17_x4', 'gf_ragged_37x53_x2', 'gf_textured_120x160_x4', 'gf_flat_120x160_x4']
GF_ENGINE_CASES = ['gf_textured_256x256_x4', 'gf_textured_480x640_x4']     # the engine's sizes, checked against the oracle only


def gf_case(name):
    """-> dict(dmap [h][w], img [3][H][W], sd {r_net.feature_ext.*}) in float32."""
    from neuralrgbd_b200 import synth
    h, w, ratio, seed = {'gf_ragged_13x17_x4': (13, 17, 4, 71), 'gf_ragged_37x53_x2': (37, 53, 2, 72),
                         'gf_textured_120x160_x4': (30, 40, 4, 73), 'gf_flat_120x160_x4': (30, 40, 4, 74),
                         'gf_textured_256x256_x4': (64, 64, 4, 75), 'gf_textured_480x640_x4': (120, 160, 4, 76)}[name]
    rng = np.random.RandomState(seed)
    H, W = h * ratio, w * ratio
    dmap = (2.5 + synth.smooth_image(rng, 1, h, w)[0]).astype(f32)
    img = synth.smooth_image(rng, 3, H, W).astype(f32)
    if name.startswith('gf_flat'):
        # flat over whole regions (var_x = 0 exactly there: A = cov / eps), a textured band and sharp colour edges between
        img = np.zeros((3, H, W), f32)
        for c in range(3):
            img[c, :H // 2, :W // 3] = f32(0.3 * (c + 1))
            img[c, :H // 2, W // 3:] = f32(-0.7 + 0.2 * c)
            img[c, H // 2:, :] = f32(1.1 - 0.4 * c)
        img[:, H // 2 + 8:H // 2 + 16, :] += (0.5 * rng.standard_normal((3, 8, W))).astype(f32)
    sd = {'r_net.feature_ext.0.weight': (rng.standard_normal((64, 3, 1, 1)) * np.sqrt(2. / 64)).astype(f32),
          'r_net.feature_ext.0.bias': (0.1 * rng.standard_normal(64)).astype(f32),
          'r_net.feature_ext.2.weight': (rng.standard_normal((1, 64, 1, 1)) * np.sqrt(2.)).astype(f32),
          'r_net.feature_ext.2.bias': (0.1 * rng.standard_normal(1)).astype(f32)}
    return dict(dmap=dmap, img=img, sd=sd)


def kvnet_dgf_output(log_dpv, ref_frame, d_candi, sd):
    """The DGF refined output of KVNET.forward for one low-resolution log-DPV [D][h][w] and the reference frame [3][H][W]:
    depth_val_regression (mutils/misc.py:532-548, sequential fp32) then RefineNet_DGF."""
    return dgf_refine(O.depth_val_regression(np.asarray(log_dpv)[None], d_candi)[0], ref_frame, sd)
