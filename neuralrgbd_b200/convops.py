"""Op-level host wrappers of the conv-stack entry points (nrgbd_conv_nhwc & co.) taking and
returning NCHW / NCDHW torch tensors. Used by the parity tests to exercise each kernel in
isolation; the engine calls the same C entry points directly from C++."""
import ctypes

import torch

from . import _lib
from ._lib import ptr, check

_F = ctypes.c_float


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def pad4(c):
    return (c + 3) // 4 * 4


def to_cl(x):
    """[N,C,(D,)H,W] -> channels-last [N,(D,)H,W,Cs] with zero pad channels."""
    L = _lib.lib()
    N, C = x.shape[0], x.shape[1]
    P = 1
    for s in x.shape[2:]:
        P *= s
    Cs = pad4(C)
    y = torch.zeros((N,) + tuple(x.shape[2:]) + (Cs,), device=x.device, dtype=torch.float32)
    check(L.nrgbd_nchw_to_nhwc(ptr(x.float().contiguous()), N, C, P, ptr(y), Cs, 0, _st()))
    return y


def from_cl(y, C):
    L = _lib.lib()
    N = y.shape[0]; Cs = y.shape[-1]
    sp = tuple(y.shape[1:-1])
    P = 1
    for s in sp:
        P *= s
    x = torch.empty((N, C) + sp, device=y.device, dtype=torch.float32)
    check(L.nrgbd_nhwc_to_nchw(ptr(y.contiguous()), N, C, P, Cs, 0, ptr(x), _st()))
    return x


def pack_weight(w, transposed=False):
    L = _lib.lib()
    if transposed:
        Cin, Cout = w.shape[0], w.shape[1]
    else:
        Cout, Cin = w.shape[0], w.shape[1]
    taps = 1
    for s in w.shape[2:]:
        taps *= s
    out = torch.empty((taps, pad4(Cin), pad4(Cout)), device=w.device, dtype=torch.float32)
    check(L.nrgbd_pack_conv_weight(ptr(w.float().contiguous()), 1 if transposed else 0, Cout, Cin, taps, pad4(Cin),
                                   pad4(Cout), ptr(out), _st()))
    return out


def conv(x, w, bias=None, stride=1, pad=0, dilation=1, leaky=False, want_stats=False):
    """nn.Conv2d / nn.Conv3d(3x3x3, pad 1) forward on NCHW/NCDHW input. Returns y (same rank) and
    optionally the [2, Cout] float64 (sum, sum of squares) statistics."""
    L = _lib.lib()
    is3d = x.dim() == 5
    xc = to_cl(x)
    N = x.shape[0]
    Din = x.shape[2] if is3d else 1
    Hin, Win = x.shape[-2], x.shape[-1]
    Cout, Cin = w.shape[0], w.shape[1]
    kd = w.shape[2] if is3d else 1
    kh, kw = w.shape[-2], w.shape[-1]
    Ho = (Hin + 2 * pad - dilation * (kh - 1) - 1) // stride + 1
    Wo = (Win + 2 * pad - dilation * (kw - 1) - 1) // stride + 1
    wp = pack_weight(w)
    y = torch.zeros((N,) + ((Din,) if is3d else ()) + (Ho, Wo, pad4(Cout)), device=x.device, dtype=torch.float32)
    stats = torch.zeros((2, Cout), device=x.device, dtype=torch.float64) if want_stats else None
    check(L.nrgbd_conv_nhwc(ptr(xc), N, Din, Hin, Win, pad4(Cin), xc.shape[-1], ptr(wp), ptr(bias), Cout, pad4(Cout), kd,
                            kh, kw, stride, pad, dilation, ptr(y), Ho, Wo, pad4(Cout), 0, 1 if leaky else 0,
                            ctypes.c_void_p(stats.data_ptr()) if want_stats else None, _st()))
    out = from_cl(y, Cout)
    return (out, stats) if want_stats else out


def conv_transpose2d(x, w, bias=None, leaky=False):
    """nn.ConvTranspose2d(kernel 4, stride 2, padding 1) forward on NCHW input."""
    L = _lib.lib()
    xc = to_cl(x)
    N, Cin, Hin, Win = x.shape
    Cout = w.shape[1]
    wp = pack_weight(w, transposed=True)
    y = torch.zeros((N, 2 * Hin, 2 * Win, pad4(Cout)), device=x.device, dtype=torch.float32)
    check(L.nrgbd_conv_transpose2d_k4s2_nhwc(ptr(xc), N, Hin, Win, pad4(Cin), xc.shape[-1], ptr(wp), ptr(bias), Cout,
                                             pad4(Cout), ptr(y), pad4(Cout), 0, 1 if leaky else 0, _st()))
    return from_cl(y, Cout)


def batch_norm(x, stats, gamma, beta, relu=False, residual=None, eps=1e-5):
    """Training-mode BatchNorm from accumulated statistics, optional ReLU / residual add."""
    L = _lib.lib()
    C = x.shape[1]
    xc = to_cl(x)
    n_pos = xc.numel() // xc.shape[-1]
    scale = torch.empty(C, device=x.device); shift = torch.empty(C, device=x.device)
    check(L.nrgbd_bn_finalize(ctypes.c_void_p(stats.data_ptr()), C, float(n_pos), ptr(gamma), ptr(beta), _F(eps), ptr(scale),
                              ptr(shift), None, None, _F(0.1), _st()))
    rc = to_cl(residual) if residual is not None else None
    check(L.nrgbd_bn_apply(ptr(xc), ptr(scale), ptr(shift), ptr(rc), 1 if relu else 0, n_pos, xc.shape[-1], C, ptr(xc),
                           _st()))
    return from_cl(xc, C)


def avg_pool2d(x, k):
    L = _lib.lib()
    N, C, H, W = x.shape
    xc = to_cl(x)
    y = torch.zeros((N, H // k, W // k, pad4(C)), device=x.device, dtype=torch.float32)
    check(L.nrgbd_avgpool_nhwc(ptr(xc), N, H, W, xc.shape[-1], C, k, ptr(y), pad4(C), 0, _st()))
    return from_cl(y, C)


def upsample_bilinear_ac(x, size):
    L = _lib.lib()
    N, C, H, W = x.shape
    xc = to_cl(x)
    y = torch.zeros((N, size[0], size[1], pad4(C)), device=x.device, dtype=torch.float32)
    check(L.nrgbd_upsample_bilinear_ac_nhwc(ptr(xc), N, H, W, xc.shape[-1], C, ptr(y), size[0], size[1], pad4(C), 0, _st()))
    return from_cl(y, C)


# ---------------------------------------------------------------------------------------------
# tensor-core (wgmma, 3xTF32) variants
# ---------------------------------------------------------------------------------------------
def pad_to(c, m):
    return (c + m - 1) // m * m


def to_cl_padded(x, Cs):
    """[N,C,(D,)H,W] -> channels-last with an explicit channel stride Cs (zero pad channels)."""
    L = _lib.lib()
    N, C = x.shape[0], x.shape[1]
    P = 1
    for s in x.shape[2:]:
        P *= s
    y = torch.zeros((N,) + tuple(x.shape[2:]) + (Cs,), device=x.device, dtype=torch.float32)
    check(L.nrgbd_nchw_to_nhwc(ptr(x.float().contiguous()), N, C, P, ptr(y), Cs, 0, _st()))
    return y


def split_tf32(xc, C=None, scale=None, shift=None, relu=False):
    """Channels-last fp32 [..., Cs] -> TF32 pair (hi, lo) of the same shape (nrgbd_split_tf32). Channels below C (default
    Cs) hold x, or relu(x * scale + shift) when scale / shift [C] are given; the others hold zero."""
    L = _lib.lib()
    Cs = xc.shape[-1]
    hi = torch.empty_like(xc); lo = torch.empty_like(xc)
    check(L.nrgbd_split_tf32(ptr(xc), xc.numel() // Cs, Cs, Cs, Cs if C is None else C, ptr(scale), ptr(shift), 1 if relu else 0,
                             ptr(hi), ptr(lo), _st()))
    return hi, lo


def pack_weight_tc(w, transposed=False):
    L = _lib.lib()
    if transposed:
        Cin, Cout = w.shape[0], w.shape[1]
    else:
        Cout, Cin = w.shape[0], w.shape[1]
    taps = 1
    for s in w.shape[2:]:
        taps *= s
    Cin_pad, Cout_pad = pad_to(Cin, 32), pad_to(Cout, 16)
    hi = torch.empty((taps, Cout_pad, Cin_pad), device=w.device, dtype=torch.float32); lo = torch.empty_like(hi)
    check(L.nrgbd_pack_conv_weight_tc(ptr(w.float().contiguous()), 1 if transposed else 0, Cout, Cin, taps, Cin_pad, Cout_pad,
                                      ptr(hi), ptr(lo), _st()))
    return hi, lo


def _conv_tc_pair(xh, xl, x_shape, w, bias, stride, pad, dilation, leaky, want_stats):
    """nrgbd_conv_nhwc_tc on the TF32 pair (xh, xl), channels-last [N,(D,)H,W,Cin_pad], of an input of NCHW / NCDHW shape
    x_shape. Returns what conv_tc returns."""
    L = _lib.lib()
    is3d = len(x_shape) == 5
    N = x_shape[0]
    Din = x_shape[2] if is3d else 1
    Hin, Win = x_shape[-2], x_shape[-1]
    Cout = w.shape[0]
    Cin_pad, Cout_pad = xh.shape[-1], pad_to(Cout, 16)
    kd = w.shape[2] if is3d else 1
    kh, kw = w.shape[-2], w.shape[-1]
    Ho = (Hin + 2 * pad - dilation * (kh - 1) - 1) // stride + 1
    Wo = (Win + 2 * pad - dilation * (kw - 1) - 1) // stride + 1
    wh, wl = pack_weight_tc(w)
    Cs_out = pad4(Cout)
    y = torch.zeros((N,) + ((Din,) if is3d else ()) + (Ho, Wo, Cs_out), device=xh.device, dtype=torch.float32)
    stats = torch.zeros((2, Cout), device=xh.device, dtype=torch.float64) if want_stats else None
    check(L.nrgbd_conv_nhwc_tc(ptr(xh), ptr(xl), N, Din, Hin, Win, Cin_pad, Cin_pad, ptr(wh), ptr(wl), ptr(bias), Cout, Cout_pad,
                               kd, kh, kw, stride, pad, dilation, ptr(y), Ho, Wo, Cs_out, 0, 1 if leaky else 0,
                               ctypes.c_void_p(stats.data_ptr()) if want_stats else None, _st()))
    out = from_cl(y, Cout)
    return (out, stats) if want_stats else out


def conv_tc(x, w, bias=None, stride=1, pad=0, dilation=1, leaky=False, want_stats=False):
    """Tensor-core counterpart of conv() (same arguments / returns): the split, then the GEMM on the TF32 pair."""
    xh, xl = split_tf32(to_cl_padded(x, pad_to(w.shape[1], 32)))
    return _conv_tc_pair(xh, xl, x.shape, w, bias, stride, pad, dilation, leaky, want_stats)


def conv_transpose2d_tc(x, w, bias=None, leaky=False):
    L = _lib.lib()
    N, Cin, Hin, Win = x.shape
    Cout = w.shape[1]
    Cin_pad, Cout_pad = pad_to(Cin, 32), pad_to(Cout, 16)
    xh, xl = split_tf32(to_cl_padded(x, Cin_pad))
    wh, wl = pack_weight_tc(w, transposed=True)
    Cs_out = pad4(Cout)
    y = torch.zeros((N, 2 * Hin, 2 * Win, Cs_out), device=x.device, dtype=torch.float32)
    check(L.nrgbd_conv_transpose2d_k4s2_nhwc_tc(ptr(xh), ptr(xl), N, Hin, Win, Cin_pad, Cin_pad, ptr(wh), ptr(wl), ptr(bias), Cout,
                                                Cout_pad, ptr(y), Cs_out, 0, 1 if leaky else 0, _st()))
    return from_cl(y, Cout)


def conv_tc_bn_in(x_raw, in_stats, gamma, beta, w, bias=None, stride=1, pad=0, dilation=1, relu=True, leaky=False,
                  want_stats=False, eps=1e-5, running=None):
    """conv(relu(batch_norm_train(x_raw))) without a BatchNorm pass: x_raw [N,C,H,W] is the raw output of the producing conv
    and in_stats its [2,C] float64 sums (conv(..., want_stats=True)); nrgbd_bn_finalize turns them into scale / shift and
    the operand split applies them. running = (running_mean, running_var) tensors to update, optional."""
    L = _lib.lib()
    assert x_raw.dim() == 4
    N, Cin, Hin, Win = x_raw.shape
    scale = torch.empty(Cin, device=x_raw.device, dtype=torch.float32); shift = torch.empty_like(scale)
    check(L.nrgbd_bn_finalize(ctypes.c_void_p(in_stats.data_ptr()), Cin, float(N * Hin * Win), ptr(gamma.float().contiguous()),
                              ptr(beta.float().contiguous()), _F(eps), ptr(scale), ptr(shift), ptr(running[0]) if running else None,
                              ptr(running[1]) if running else None, _F(0.1), _st()))
    xh, xl = split_tf32(to_cl_padded(x_raw, pad_to(Cin, 32)), Cin, scale, shift, relu)
    return _conv_tc_pair(xh, xl, x_raw.shape, w, bias, stride, pad, dilation, leaky, want_stats)


# ---------------------------------------------------------------------------------------------
# second-generation tensor-core path (csrc/conv_f16.cu): wgmma on split-fp16 operand pairs
# ---------------------------------------------------------------------------------------------
def h2_plan(Cin, Cout):
    L = _lib.lib()
    a, b, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert L.nrgbd_conv_h2_plan(Cin, Cout, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)) == 1
    return a.value, b.value, c.value          # Cin_pad, Cout_pad, BN


def split_f16_pair(xc, single=False):
    """fp32 tensor -> (hi, lo) float16 tensors of the same shape: x = hi + lo * 2^-11. single: lo = None and hi = RN_f16(x),
    the operand of the single-product convolution (conv_math='f16')."""
    L = _lib.lib()
    hi = torch.empty(xc.shape, device=xc.device, dtype=torch.float16)
    lo = None if single else torch.empty_like(hi)
    check(L.nrgbd_split_f16_pair(ptr(xc), xc.numel(), ptr(hi), ptr(lo), _st()))
    return hi, lo


def pack_weight_h2(w, transposed=False):
    L = _lib.lib()
    if transposed:
        Cin, Cout = w.shape[0], w.shape[1]
    else:
        Cout, Cin = w.shape[0], w.shape[1]
    taps = 1
    for s in w.shape[2:]:
        taps *= s
    Cin_pad, Cout_pad, BN = h2_plan(Cin, Cout)
    out = torch.empty((taps, 2, Cout_pad, Cin_pad), device=w.device, dtype=torch.float16)
    check(L.nrgbd_pack_conv_weight_h2(ptr(w.float().contiguous()), 1 if transposed else 0, Cout, Cin, taps, Cin_pad, Cout_pad,
                                      ptr(out), _st()))
    return out, Cin_pad, Cout_pad, BN


def conv_h2(x, w, bias=None, stride=1, pad=0, dilation=1, leaky=False, want_stats=False, single=False):
    """f16-pair tensor-core counterpart of conv() (same arguments / returns). single: the single-product kernel (x_lo = NULL),
    sum RN_f16(x) * RN_f16(w) in fp32."""
    L = _lib.lib()
    is3d = x.dim() == 5
    N = x.shape[0]
    Din = x.shape[2] if is3d else 1
    Hin, Win = x.shape[-2], x.shape[-1]
    Cout, Cin = w.shape[0], w.shape[1]
    wp, Cin_pad, Cout_pad, BN = pack_weight_h2(w)
    xc = to_cl_padded(x, Cin_pad)
    xh, xl = split_f16_pair(xc, single)
    kd = w.shape[2] if is3d else 1
    kh, kw = w.shape[-2], w.shape[-1]
    Ho = (Hin + 2 * pad - dilation * (kh - 1) - 1) // stride + 1
    Wo = (Win + 2 * pad - dilation * (kw - 1) - 1) // stride + 1
    Cs_out = pad4(Cout)
    y = torch.zeros((N,) + ((Din,) if is3d else ()) + (Ho, Wo, Cs_out), device=x.device, dtype=torch.float32)
    stats = torch.zeros((2, Cout), device=x.device, dtype=torch.float64) if want_stats else None
    check(L.nrgbd_conv_nhwc_h2(ptr(xh), ptr(xl), N, Din, Hin, Win, Cin_pad, Cin_pad, ptr(wp), ptr(bias), Cout, Cout_pad, BN,
                               kd, kh, kw, stride, pad, dilation, ptr(y), Ho, Wo, Cs_out, 0, 1 if leaky else 0,
                               ctypes.c_void_p(stats.data_ptr()) if want_stats else None, _st()))
    out = from_cl(y, Cout)
    return (out, stats) if want_stats else out


def conv_h2_pair_out(x, w, bias=None, stride=1, pad=0, dilation=1, leaky=False, single=False):
    """conv_h2 whose result is written only as the operand pair of the next convolution (nrgbd_conv_nhwc_h2_pair). Returns the
    fp32 value of the pair, hi + lo * 2^-11, as NCHW / NCDHW, and the raw (hi, lo) half tensors (channels-last, Cs = pad32).
    single: x_lo = y_lo = NULL - the single-product kernel, the output stored as hi only (lo returned as None)."""
    L = _lib.lib()
    is3d = x.dim() == 5
    N = x.shape[0]
    Din = x.shape[2] if is3d else 1
    Hin, Win = x.shape[-2], x.shape[-1]
    Cout, Cin = w.shape[0], w.shape[1]
    wp, Cin_pad, Cout_pad, BN = pack_weight_h2(w)
    xh, xl = split_f16_pair(to_cl_padded(x, Cin_pad), single)
    kd = w.shape[2] if is3d else 1
    kh, kw = w.shape[-2], w.shape[-1]
    Ho = (Hin + 2 * pad - dilation * (kh - 1) - 1) // stride + 1
    Wo = (Win + 2 * pad - dilation * (kw - 1) - 1) // stride + 1
    Cs = pad_to(Cout, 32)
    shape = (N,) + ((Din,) if is3d else ()) + (Ho, Wo, Cs)
    # poisoned: every element, pad channels included, must be written by the kernel
    yh = torch.full(shape, float('nan'), device=x.device, dtype=torch.float16)
    yl = None if single else torch.full(shape, float('nan'), device=x.device, dtype=torch.float16)
    check(L.nrgbd_conv_nhwc_h2_pair(ptr(xh), ptr(xl), N, Din, Hin, Win, Cin_pad, Cin_pad, ptr(wp), ptr(bias), Cout, Cout_pad, BN,
                                    kd, kh, kw, stride, pad, dilation, ptr(yh), ptr(yl), Ho, Wo, Cs, 1 if leaky else 0, _st()))
    val = yh.float() if single else yh.float() + yl.float() * (1.0 / 2048.0)
    return from_cl(val.contiguous(), Cout), yh, yl


def bn_eval_coeffs(gamma, beta, running_mean, running_var, eps=1e-5):
    """Eval-mode BatchNorm coefficients on the device (nrgbd_bn_eval_coeffs) -> (scale, shift)."""
    L = _lib.lib()
    C = gamma.numel()
    scale = torch.empty(C, device=gamma.device, dtype=torch.float32); shift = torch.empty_like(scale)
    check(L.nrgbd_bn_eval_coeffs(ptr(gamma.float().contiguous()), ptr(beta.float().contiguous()), ptr(running_mean.float().contiguous()),
                                 ptr(running_var.float().contiguous()), _F(eps), C, ptr(scale), ptr(shift), _st()))
    return scale, shift


def conv_h2_affine(x, w, scale, shift, stride=1, pad=0, dilation=1, res=None, res_pair=False, relu=False, pair_out=False,
                   single=False):
    """Eval-mode convbn in one kernel (nrgbd_conv_nhwc_h2_affine): relu(conv(x, w) * scale + shift + res). res (NCHW / NCDHW,
    the output's shape) is passed as fp32 or, with res_pair, as its split-fp16 operand pair. pair_out: the result is written
    only as the operand pair of the next convolution; returned as its fp32 value hi + lo * 2^-11 plus the raw (hi, lo).
    single: the single-product kernel (x_lo = NULL); a pair output is stored as hi only (y_lo = NULL). The residual keeps
    its pair form."""
    L = _lib.lib()
    is3d = x.dim() == 5
    N = x.shape[0]
    Din = x.shape[2] if is3d else 1
    Hin, Win = x.shape[-2], x.shape[-1]
    Cout = w.shape[0]
    wp, Cin_pad, Cout_pad, BN = pack_weight_h2(w)
    xh, xl = split_f16_pair(to_cl_padded(x, Cin_pad), single)
    kd = w.shape[2] if is3d else 1
    kh, kw = w.shape[-2], w.shape[-1]
    Ho = (Hin + 2 * pad - dilation * (kh - 1) - 1) // stride + 1
    Wo = (Win + 2 * pad - dilation * (kw - 1) - 1) // stride + 1
    Cs = pad_to(Cout, 32) if pair_out else pad4(Cout)
    shape = (N,) + ((Din,) if is3d else ()) + (Ho, Wo, Cs)
    r = rh = rl = None
    if res is not None:
        rc = to_cl_padded(res, Cs)
        if res_pair:
            rh, rl = split_f16_pair(rc)
        else:
            r = rc
    y = yh = yl = None
    if pair_out:
        yh = torch.full(shape, float('nan'), device=x.device, dtype=torch.float16)     # every element must be written
        yl = None if single else torch.full(shape, float('nan'), device=x.device, dtype=torch.float16)
    else:
        y = torch.zeros(shape, device=x.device, dtype=torch.float32)
    check(L.nrgbd_conv_nhwc_h2_affine(ptr(xh), ptr(xl), N, Din, Hin, Win, Cin_pad, Cin_pad, ptr(wp), Cout, Cout_pad, BN, kd, kh, kw,
                                      stride, pad, dilation, ptr(scale), ptr(shift), ptr(r), ptr(rh), ptr(rl), 1 if relu else 0,
                                      ptr(y), ptr(yh), ptr(yl), Ho, Wo, Cs, 0, _st()))
    if pair_out:
        val = yh.float() if single else yh.float() + yl.float() * (1.0 / 2048.0)
        return from_cl(val.contiguous(), Cout), yh, yl
    return from_cl(y, Cout)


def conv_cout1_h2(x, w, bias=0.0, single=False):
    """Single-output-channel k3 convolution (K-Net's last layer, models/basic.py:136-137) the way the engine runs it:
    a pointwise f16-pair conv to one channel per tap + nrgbd_tap_gather_sum. x [N, C, D, H, W] (or [N, C, H, W]),
    w [1, C, 3, 3, 3] (or [1, C, 3, 3]) -> [N, 1, D, H, W] ([N, 1, H, W]). single: the pointwise conv on hi only."""
    L = _lib.lib()
    is3d = x.dim() == 5
    N = x.shape[0]
    D = x.shape[2] if is3d else 1
    H, W = x.shape[-2], x.shape[-1]
    Cin = w.shape[1]
    kd = w.shape[2] if is3d else 1
    taps = kd * 9
    wt = w[0].reshape(Cin, taps, 1, 1)                  # [Cin][Cout' = taps][1][1]: the transposed-kind source layout
    wp, Cin_pad, Cout_pad, BN = pack_weight_h2(wt, transposed=True)
    xh, xl = split_f16_pair(to_cl_padded(x, Cin_pad), single)
    Cs = pad4(taps)
    q = torch.empty((N, D, H, W, Cs), device=x.device, dtype=torch.float32)
    check(L.nrgbd_conv_nhwc_h2(ptr(xh), ptr(xl), N, D, H, W, Cin_pad, Cin_pad, ptr(wp), None, taps, Cout_pad, BN, 1, 1, 1, 1, 0, 1,
                               ptr(q), H, W, Cs, 0, 0, None, _st()))
    out = torch.empty((N, 1) + ((D,) if is3d else ()) + (H, W), device=x.device, dtype=torch.float32)
    check(L.nrgbd_tap_gather_sum(ptr(q), N, D, H, W, Cs, kd, 3, ctypes.c_float(bias), ptr(out), _st()))
    return out


def conv_transpose2d_h2(x, w, bias=None, leaky=False, single=False):
    L = _lib.lib()
    N, Cin, Hin, Win = x.shape
    Cout = w.shape[1]
    wp, Cin_pad, Cout_pad, BN = pack_weight_h2(w, transposed=True)
    xc = to_cl_padded(x, Cin_pad)
    xh, xl = split_f16_pair(xc, single)
    Cs_out = pad4(Cout)
    y = torch.zeros((N, 2 * Hin, 2 * Win, Cs_out), device=x.device, dtype=torch.float32)
    check(L.nrgbd_conv_transpose2d_k4s2_nhwc_h2(ptr(xh), ptr(xl), N, Hin, Win, Cin_pad, Cin_pad, ptr(wp), ptr(bias), Cout,
                                                Cout_pad, BN, ptr(y), Cs_out, 0, 1 if leaky else 0, _st()))
    return from_cl(y, Cout)


def guided_filter_refine(dmap, img, w0, b0, w1, b1, r=1, eps=1e-8):
    """RefineNet_DGF.forward (models/Refine.py:620-641) through nrgbd_guided_filter_refine: dmap [h,w], img [3,H,W]
    (CUDA float32), feature_ext weights as in the state_dict -> [H,W]."""
    L = _lib.lib()
    h, w = dmap.shape
    _, H, W = img.shape
    dmap = dmap.float().contiguous(); img = img.float().contiguous()
    ws = torch.empty(L.nrgbd_guided_filter_workspace_floats(H, W), device=img.device, dtype=torch.float32)
    out = torch.empty((H, W), device=img.device, dtype=torch.float32)
    check(L.nrgbd_guided_filter_refine(ptr(dmap), h, w, ptr(img), H * W, 1, H, W, ptr(w0.float().contiguous()),
                                       ptr(b0.float().contiguous()), ptr(w1.float().contiguous()), ptr(b1.float().contiguous()), r,
                                       _F(eps), ptr(ws), ptr(out), _st()))
    return out
