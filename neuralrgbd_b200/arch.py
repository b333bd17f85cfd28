"""Architecture spec of the KVNET parameter set (names, shapes, roles).

One table drives the host-side nn.Module mirror (parameter registration so that the
reference's checkpoints load: SURVEY.md §5 'Checkpoint / resume'), the synthetic
random-initialised state_dict used by tests/bench (no pretrained weights offline),
and the engine's weight upload order.

Names follow models/KVNET.py:63-85, models/basic.py:13-51,53-110,
models/psm_submodule.py:76-139, models/Refine.py:24-77 of the reference.
"""
import math
import numpy as np


def _convbn(pre, cin, cout, k, track=False):
    out = [(pre + '.0.weight', (cout, cin, k, k), 'conv2d'),
           (pre + '.1.weight', (cout,), 'bn_w'), (pre + '.1.bias', (cout,), 'bn_b')]
    if track:
        out += _bn_track(pre + '.1', cout)
    return out


def _bn_track(pre, c):
    return [(pre + '.running_mean', (c,), 'bn_rm'), (pre + '.running_var', (c,), 'bn_rv'),
            (pre + '.num_batches_tracked', (), 'bn_nb')]


def feature_cnn_specs(pre, feature_dim):
    """psm_submodule.feature_extraction.__init__ :76-139."""
    s = []
    s += _convbn(pre + '.firstconv.0', 3, 32, 3)
    s += _convbn(pre + '.firstconv.2', 32, 32, 3)
    s += _convbn(pre + '.firstconv.4', 32, 32, 3)
    inpl = 32
    for lname, planes, blocks, stride in (('layer1', 32, 3, 1), ('layer2', 64, 16, 2),
                                          ('layer3', 128, 3, 1), ('layer4', 128, 3, 1)):
        for b in range(blocks):
            bp = '%s.%s.%d' % (pre, lname, b)
            cin = inpl if b == 0 else planes
            s += _convbn(bp + '.conv1.0', cin, planes, 3)
            s += _convbn(bp + '.conv2', planes, planes, 3)
            if b == 0 and (stride != 1 or inpl != planes):
                s += [(bp + '.downsample.0.weight', (planes, inpl, 1, 1), 'conv2d'),
                      (bp + '.downsample.1.weight', (planes,), 'bn_w'),
                      (bp + '.downsample.1.bias', (planes,), 'bn_b')]
                s += _bn_track(bp + '.downsample.1', planes)
        inpl = planes
    for br in ('branch1', 'branch2', 'branch3', 'branch4'):
        s += _convbn('%s.%s.1' % (pre, br), 128, 32, 1)
    s += _convbn(pre + '.lastconv.0', 320, 128, 3)
    s += [(pre + '.lastconv.2.weight', (feature_dim, 128, 1, 1), 'conv2d')]
    return s


def kv_net_specs(pre, cin, f):
    """basic.KV_NET_BASIC.__init__ :59-94."""
    def cb(p, a, b):
        return [(p + '.0.weight', (b, a, 3, 3, 3), 'conv3d'), (p + '.1.weight', (b,), 'bn_w'),
                (p + '.1.bias', (b,), 'bn_b')] + _bn_track(p + '.1', b)
    s = cb(pre + '.dres0.0', cin, f) + cb(pre + '.dres0.2', f, f)
    for i in (1, 2, 3, 4):
        s += cb('%s.dres%d.0' % (pre, i), f, f) + cb('%s.dres%d.2' % (pre, i), f, f)
    s += cb(pre + '.classify.0', f, f)
    s += [(pre + '.classify.2.weight', (1, f, 3, 3, 3), 'conv3d')]
    return s


def r_net_specs(pre, C0, C1, C2, D, upsample_D=False):
    """Refine.RefineNet_DPV_upsample.__init__ :30-77. upsample_D widens the two transposed convolutions' outputs to
    D0 = 2D and D1 = 4D planes (:44-48): the refined DPV then has 4D planes."""
    def c(p, a, b):
        return [(p + '.weight', (b, a, 3, 3), 'conv2d'), (p + '.bias', (b,), 'bias')]

    def t(p, a, b):
        return [(p + '.weight', (a, b, 4, 4), 'convT2d'), (p + '.bias', (b,), 'bias')]
    i0 = D + C0
    D0, D1 = (2 * D, 4 * D) if upsample_D else (D, D)
    return (c(pre + '.conv0.0', i0, i0) + c(pre + '.conv0_1.0', i0, i0) + t(pre + '.trans_conv0.0', i0, D0)
            + c(pre + '.conv1.0', D0 + C1, D0 + C1) + c(pre + '.conv1_1.0', D0 + C1, D0 + C1)
            + t(pre + '.trans_conv1.0', D0 + C1, D1)
            + c(pre + '.conv2.0', D1 + C2, D1 + C2) + c(pre + '.conv2_1.0', D1 + C2, D1)
            + c(pre + '.conv2_2', D1, D1))


def dgf_specs(pre):
    """Refine.RefineNet_DGF.__init__ :587-598: feature_ext = Conv2d(3, 64, 1), ReLU, Conv2d(64, 1, 1). The guided filter
    itself has no parameters, and refine_channel does not change these shapes."""
    return [(pre + '.feature_ext.0.weight', (64, 3, 1, 1), 'conv2d'), (pre + '.feature_ext.0.bias', (64,), 'bias'),
            (pre + '.feature_ext.2.weight', (1, 64, 1, 1), 'conv2d'), (pre + '.feature_ext.2.bias', (1,), 'bias')]


def kvnet_param_specs(feature_dim=64, D=64, t_win_r=2, kv_feature_dim=64, refine='DPV', upsample_d=False):
    """Every entry of KVNET(...).state_dict() in registration order. The feature CNN
    appears twice (the extractor object is registered under both `feature_extractor`
    and `d_net.feature_extraction`, KVNET.py:63-67) -- same tensors, two names; its
    parameters do not depend on multi_scale, so every refinement shares them.
    refine: 'DPV' (default), 'DGF' or None (if_refined=False); upsample_d: the DPV R-Net's if_upsample_d (ignored
    unless refine is 'DPV', as in the reference)."""
    fe = feature_cnn_specs('feature_extractor.feature_extraction', feature_dim)
    fe2 = [('d_net.feature_extraction.' + n[len('feature_extractor.'):], shp, kind) for n, shp, kind in fe]
    kv = kv_net_specs('kv_net', 3 * (2 * t_win_r + 1) + 1, kv_feature_dim)
    if refine == 'DPV':
        rn = r_net_specs('r_net', feature_dim, feature_dim // 2, 3, D, upsample_d)
    elif refine == 'DGF':
        rn = dgf_specs('r_net')
    elif refine is None:
        rn = []
    else:
        raise ValueError(refine)
    return fe + fe2 + kv + rn


def synth_state_dict(seed, feature_dim=64, D=64, t_win_r=2, kv_feature_dim=64, refine='DPV', upsample_d=False):
    """Random-initialised weights in the reference's style (He-normal convs,
    basic.py:28-40) with non-trivial BN affine terms so those paths are exercised.
    Transposed convs get the reference's bilinear kernel (Refine.py:121-132) times a
    per-(in,out) random gain / sqrt(Cin) so activations stay O(1) (pretrained weights
    are wget-only and unavailable offline). Returns {name: float32 ndarray}."""
    rng = np.random.RandomState(seed)
    sd = {}
    for name, shp, kind in kvnet_param_specs(feature_dim, D, t_win_r, kv_feature_dim, refine, upsample_d):
        if name.startswith('d_net.feature_extraction.'):
            sd[name] = sd['feature_extractor.' + name[len('d_net.feature_extraction.'):]]
            continue
        if kind in ('conv2d', 'conv3d'):
            n = int(np.prod(shp[2:])) * shp[0]
            v = rng.standard_normal(shp) * math.sqrt(2.0 / n)
            if name.startswith('r_net'):
                v = rng.standard_normal(shp) * math.sqrt(1.0 / (int(np.prod(shp[2:])) * shp[1]))
        elif kind == 'convT2d':
            k = shp[2]; factor = (k + 1) // 2
            center = factor - 1 if k % 2 == 1 else factor - .5
            og = np.ogrid[:k, :k]
            bil = (1 - abs(og[0] - center) / factor) * (1 - abs(og[1] - center) / factor)
            v = bil[None, None] * rng.standard_normal(shp[:2] + (1, 1)) / math.sqrt(shp[0])
        elif kind == 'bn_w':
            v = rng.uniform(0.5, 1.5, shp)
        elif kind in ('bn_b', 'bias'):
            v = 0.1 * rng.standard_normal(shp)
        elif kind == 'bn_rm':
            v = np.zeros(shp)
        elif kind == 'bn_rv':
            v = np.ones(shp)
        elif kind == 'bn_nb':
            sd[name] = np.zeros(shp, np.int64)
            continue
        sd[name] = np.ascontiguousarray(v, dtype=np.float32)
    return sd
