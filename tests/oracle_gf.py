"""numpy restatement of the reference's models/GF GuidedFilter(r, eps) and BoxFilter(r) on N x C x H x W arrays, forward
and backward.

Forward (float32): tests/oracle_refine.py's box_filter / guided_filter, which carry the reference's fp32 arithmetic
(double-accumulated cumsum rounded to fp32 at every prefix, box_filter.py's diffs, one IEEE op at a time), applied per
(n, channel of y) with the guide's channel chosen as the reference's broadcast does (C_x = 1: channel 0). Per-plane
evaluation gives the broadcast's values exactly: every operation is element-wise.

Backward (float64): autograd's order through guided_filter.py:76-97 and box_filter.py - the output's product and sum,
the divisions by N, A = cov / (var + eps), b = mean_y - A * mean_x, cov, var, the products x*y and x*x, then each box
filter's adjoint (the diff's slice / cat backward, then cumsum's backward, a reverse prefix sum; rows before columns).
The intermediate planes come from the float32 forward (what the reference's autograd saw), or from the float64 forward
(`dtype=np.float64`) for gradcheck.
"""
import numpy as np

from tests import oracle_refine as OR

f32, f64 = np.float32, np.float64


def box_filter(a, r):
    """BoxFilter(r).forward of a float32 [..., H, W] array, plane by plane."""
    a = np.asarray(a, f32)
    flat = a.reshape(-1, *a.shape[-2:])
    return np.stack([OR.box_filter(p, r) for p in flat]).reshape(a.shape)


def _cx(Cx, c):
    return 0 if Cx == 1 else c


def guided_filter(x, y, r, eps):
    """GuidedFilter(r, eps).forward(x [N,Cx,H,W], y [N,Cy,H,W]) -> [N,Cy,H,W] float32."""
    x, y = np.asarray(x, f32), np.asarray(y, f32)
    N, Cx, H, W = x.shape
    Cy = y.shape[1]
    assert N == y.shape[0] and (Cx == 1 or Cx == Cy) and y.shape[2:] == (H, W)
    return np.stack([np.stack([OR.guided_filter(x[n, _cx(Cx, c)], y[n, c], r, eps) for c in range(Cy)])
                     for n in range(N)])


# ---- float64 box filter (gradcheck) and the adjoint ------------------------------------------------------------------
def _diff64(cs, r, axis):
    c = np.moveaxis(cs, axis, 0)
    out = np.concatenate([c[r:2 * r + 1], c[2 * r + 1:] - c[:-2 * r - 1], c[-1:] - c[-2 * r - 1:-r - 1]], 0)
    return np.moveaxis(out, 0, axis)


def box_filter64(a, r):
    a = np.asarray(a, f64)
    return _diff64(np.cumsum(_diff64(np.cumsum(a, -2), r, -2), -1), r, -1)


def _diff_adjoint(g, r, axis):
    """Adjoint of box_filter.py's diff along `axis`: d cs[j] = g[j - r] - g[j + r + 1], plus, at the last position, the
    sum of g over the broadcast `right` slice (g[n-r..n-1])."""
    g = np.moveaxis(np.asarray(g, f64), axis, 0)
    n = g.shape[0]
    out = np.zeros_like(g)
    out[r:] += g[:n - r]
    out[:n - r - 1] -= g[r + 1:]
    out[n - 1] += g[n - r:].sum(0)
    return np.moveaxis(out, 0, axis)


def _rcumsum(g, axis):
    return np.ascontiguousarray(np.flip(np.cumsum(np.flip(g, axis), axis), axis))


def box_filter_backward(g, r):
    """Gradient of BoxFilter(r) w.r.t. its input for the upstream gradient g, float64: diff_y's adjoint and the reverse
    cumsum along W, then the same along H (autograd's order)."""
    t = _rcumsum(_diff_adjoint(g, r, -1), -1)
    return _rcumsum(_diff_adjoint(t, r, -2), -2)


# ---- guided filter: intermediates and backward ----------------------------------------------------------------------
def parts(x, y, r, eps, dtype=f32):
    """The planes of guided_filter.py:76-95, as the float32 reference computes them (dtype float32) or in float64."""
    x, y = np.asarray(x, dtype), np.asarray(y, dtype)
    H, W = x.shape[-2:]
    box = box_filter if dtype == f32 else box_filter64
    Nw = box(np.ones((1, 1, H, W), dtype), r).astype(dtype)
    mx, my = (box(x, r) / Nw).astype(dtype), (box(y, r) / Nw).astype(dtype)
    cov = (box(x * y, r) / Nw - mx * my).astype(dtype)
    var = (box(x * x, r) / Nw - mx * mx).astype(dtype)
    ve = (var + dtype(eps)).astype(dtype)
    A = (cov / ve).astype(dtype)
    b = (my - A * mx).astype(dtype)
    mA, mb = (box(A, r) / Nw).astype(dtype), (box(b, r) / Nw).astype(dtype)
    return dict(N=Nw, mx=mx, my=my, cov=cov, ve=ve, A=A, b=b, mA=mA, mb=mb, out=(mA * x + mb).astype(dtype))


def guided_filter64(x, y, r, eps):
    return parts(x, y, r, eps, f64)['out']


def guided_filter_backward(g, x, y, r, eps, dtype=f32):
    """(d x [N,Cx,H,W], d y [N,Cy,H,W]) in float64 for the upstream gradient g [N,Cy,H,W]."""
    P = {k: np.asarray(v, f64) for k, v in parts(x, y, r, eps, dtype).items()}
    x, y, g = np.asarray(x, f64), np.asarray(y, f64), np.asarray(g, f64)
    red = (lambda a: a.sum(1, keepdims=True)) if x.shape[1] == 1 else (lambda a: a)       # noqa: E731 (sum_to_size)
    Nw, mx, my, cov, ve, A = P['N'], P['mx'], P['my'], P['cov'], P['ve'], P['A']
    # out = mean_A * x + mean_b; mean_A = box(A) / N; mean_b = box(b) / N
    gx = red(g * P['mA'])
    gA = box_filter_backward(g * x / Nw, r)
    gb = box_filter_backward(g / Nw, r)
    # b = mean_y - A * mean_x
    gA = gA + (-gb) * mx
    g_mx = red((-gb) * A)
    g_my = gb
    # A = cov / (var + eps)
    g_cov = gA / ve
    g_var = red(-gA * cov / (ve * ve))
    # cov = box(xy) / N - mean_x * mean_y; var = box(xx) / N - mean_x * mean_x
    g_bxy = g_cov / Nw
    g_mx = g_mx + red(-g_cov * my)
    g_my = g_my + (-g_cov) * mx
    g_bxx = g_var / Nw
    g_mx = g_mx + 2 * (-g_var) * mx
    # mean_x = box(x) / N; mean_y = box(y) / N
    G_x, G_y = box_filter_backward(g_mx / Nw, r), box_filter_backward(g_my / Nw, r)
    G_xy, G_xx = box_filter_backward(g_bxy, r), box_filter_backward(g_bxx, r)
    gx = gx + G_x + red(G_xy * y) + 2 * G_xx * x
    gy = G_y + G_xy * x
    return gx, gy
