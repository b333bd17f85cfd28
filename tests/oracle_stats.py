"""Numpy restatement of the reference's DPV statistics (mutils/misc.py:550-608) and of what torch autograd computes
through them: depth_var, the max / min over the planes, and dpv_statistics composed of those and depth_val_regression.

Forwards follow the reference's fp32 arithmetic (sequential sum over d, every operation rounded on its own, the divisor
2 d_sigma^2 and D rounded to fp32 as ATen rounds a Python scalar); only exp differs from ATen's by its last bits.
Backwards are accumulated in float64 from the same fp32 inputs and rounded once. Each op also has a float64 forward for
finite-difference checks of its backward.
"""
import numpy as np

f32 = np.float32
f64 = np.float64
_E_MEAN, _VARIANCE, _MAX, _MIN = 'E_mean', 'variance', 'max', 'min'     # interned: `is` as the reference (misc.py:594-602)


def _prob(bv, BV_log):
    return np.exp(bv) if BV_log else bv


def var_div(d_sigma):
    return f32(2 * d_sigma ** 2)


def depth_val_regression(BV, d_candi, BV_log=True):
    """misc.py:532-548 in fp32, sequential over d -> [1, h, w]."""
    BV = np.asarray(BV, f32)
    acc = np.zeros(BV.shape[2:], f32)
    for i, d in enumerate(np.asarray(d_candi).astype(f32)):
        acc = acc + _prob(BV[0, i], BV_log) * d
    return acc[None]


def depth_var(BV, mean, d_candi, BV_log=True, d_sigma=1.):
    """misc.py:550-572 in fp32: the reference's broadcast shape (H x W with an H x W mean, 1 x H x W with 1 x H x W)."""
    BV = np.asarray(BV, f32)
    D = BV.shape[1]
    mean = np.asarray(mean, f32)
    div = var_div(d_sigma)
    acc = np.zeros(BV.shape[2:], f32)
    for i, d in enumerate(np.asarray(d_candi).astype(f32)):
        x = _prob(BV[0, i], BV_log) * d - mean
        acc = acc + (x * x) / div
    return (acc / f32(D)).astype(f32)


def depth_var64(BV, mean, d_candi, BV_log=True, d_sigma=1.):
    BV = np.asarray(BV, f64)
    d = np.asarray(d_candi).astype(f32).astype(f64).reshape(-1, 1, 1)
    x = _prob(BV[0], BV_log) * d - np.asarray(mean, f64).reshape(BV.shape[2:])[None]
    return ((x * x) / f64(var_div(d_sigma))).sum(0) / BV.shape[1]


def depth_var_backward64(grad, BV, mean, d_candi, BV_log=True, d_sigma=1.):
    """grad (the output's shape) -> (d loss / d BV [N,D,h,w], slices after the first zero; d loss / d mean [h, w]) in
    float64. The mean's gradient is -sum_d of the squared term's gradient."""
    N, D, h, w = np.asarray(BV).shape
    p = _prob(np.asarray(BV[0], f32).astype(f64), BV_log)
    d = np.asarray(d_candi).astype(f32).astype(f64).reshape(-1, 1, 1)
    x = p * d - np.asarray(mean, f32).astype(f64).reshape(h, w)[None]
    gx = (np.asarray(grad, f64).reshape(h, w) / (D * f64(var_div(d_sigma))))[None] * 2.0 * x
    g_bv = np.zeros((N, D, h, w), f64)
    g_bv[0] = gx * d * p if BV_log else gx * d
    return g_bv, -gx.sum(0)


def depth_var_backward(grad, BV, mean, d_candi, BV_log=True, d_sigma=1.):
    """depth_var_backward64 rounded to float32 once: (g_bv [N,D,h,w], g_mean [h, w])."""
    g_bv, g_mu = depth_var_backward64(grad, BV, mean, d_candi, BV_log, d_sigma)
    return g_bv.astype(f32), g_mu.astype(f32)


def extreme(BV, BV_log, is_min):
    """torch.max / torch.min over dim 1 of exp(BV) (or BV) -> (value [N,h,w] float32, index [N,h,w]). numpy's
    argmax / argmin keep the first of equal values and return the first NaN, as ATen's max.dim / min.dim on the CPU."""
    p = _prob(np.asarray(BV, f32), BV_log).astype(f32)
    idx = np.argmin(p, axis=1) if is_min else np.argmax(p, axis=1)
    return np.take_along_axis(p, idx[:, None], 1)[:, 0], idx


def extreme64(BV, BV_log, is_min, idx):
    p = _prob(np.asarray(BV, f64), BV_log)
    return np.take_along_axis(p, idx[:, None], 1)[:, 0]


def extreme_backward64(grad, BV, idx, BV_log):
    """grad [N,h,w] -> d loss / d BV [N,D,h,w] (float64): grad * exp(BV) (grad without BV_log) at the selected plane."""
    BV = np.asarray(BV, f32)
    out = np.zeros(BV.shape, f64)
    gv = np.asarray(grad, f64)
    if BV_log:
        gv = gv * np.exp(np.take_along_axis(BV, idx[:, None], 1)[:, 0].astype(f64))
    np.put_along_axis(out, idx[:, None], gv[:, None], 1)
    return out


def extreme_backward(grad, BV, idx, BV_log):
    return extreme_backward64(grad, BV, idx, BV_log).astype(f32)


def dpv_statistics(BV, d_candi, statistics, BV_log=True):
    """misc.py:574-608 with the reference's behaviour: names by identity, 'variance' needs an earlier 'E_mean'
    (UnboundLocalError), 'min' without BV_log is the max, an empty selection fails the assert, mixed N fails the concat.
    -> (features [N', C, h, w] float32, the pieces for dpv_statistics_backward)."""
    feats, parts = [], []
    for name in statistics:
        if name is _E_MEAN:
            depth_regress = depth_val_regression(BV, d_candi, BV_log)
            feats.append(depth_regress[:, None]); parts.append(('E_mean', None))
        if name is _VARIANCE:
            feats.append(depth_var(BV, depth_regress, d_candi, BV_log)[:, None])
            parts.append(('variance', depth_regress))
        if name is _MAX:
            v, i = extreme(BV, BV_log, False)
            feats.append(v[:, None]); parts.append(('max', i))
        if name is _MIN:
            v, i = extreme(BV, BV_log, BV_log)
            feats.append(v[:, None]); parts.append(('min', i))
    assert len(feats) > 0, 'No channels in dpv_feats. Did you specify the right dpv statistics ?'
    if len({f.shape[0] for f in feats}) > 1:
        raise RuntimeError('Sizes of tensors must match except in dimension 1')
    return np.concatenate(feats, axis=1), parts


def dpv_statistics_backward(grad, BV, d_candi, parts, BV_log=True):
    """grad [N', C, h, w] -> d loss / d BV [N,D,h,w] float32 through every channel, the variance's mean included."""
    BV = np.asarray(BV, f32)
    grad = np.asarray(grad, f64)
    out = np.zeros(BV.shape, f64)
    g_mean = np.zeros(BV.shape[2:], f64)
    for c, (kind, aux) in enumerate(parts):
        g = grad[:, c]
        if kind == 'E_mean':
            g_mean += g[0]
        elif kind == 'variance':
            g_bv, g_mu = depth_var_backward64(g[0], BV, aux, d_candi, BV_log)
            out += g_bv
            g_mean += g_mu
        else:
            out += extreme_backward64(g, BV, aux, BV_log)
    d = np.asarray(d_candi).astype(f32).astype(f64).reshape(-1, 1, 1)
    out[0] += g_mean[None] * d * (np.exp(BV[0].astype(f64)) if BV_log else 1.0)
    return out.astype(f32)
