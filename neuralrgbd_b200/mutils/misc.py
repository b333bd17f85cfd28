"""Mirror of the hot-path helpers of the reference's `mutils.misc`
(/root/reference/code/mutils/misc.py:100-115, 509-517, 532-548, 550-608)."""
import ctypes

import numpy as np
import torch

from .. import _lib
from .._devcache import planes_tensor
from .._lib import ptr, check


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def valid_dpv(dpv_in):
    """misc.py:100-115: a DPV whose first element is NaN marks an invalid batch slot."""
    if dpv_in is None:
        return False
    assert isinstance(dpv_in, torch.Tensor), 'input should a Tensor'
    if dpv_in.dim() not in (2, 3, 4, 5):
        raise Exception('wrong dimension for input dpv !')
    return not bool(torch.isnan(dpv_in.reshape(-1)[0]))


def split_frame_list(frame_list, t_win_r):
    """misc.py:509-517."""
    ref_frame = frame_list[t_win_r]
    src_frames = [frame_list[idx] for idx in range(len(frame_list)) if idx != t_win_r]
    return ref_frame, src_frames


def _regression_forward(bv, dpl, BV_log, return_conf):
    L = _lib.lib()
    D, H, W = bv.shape
    depth = torch.empty((1, H, W), device=bv.device, dtype=torch.float32)
    conf = torch.empty((1, H, W), device=bv.device, dtype=torch.float32) if return_conf else None
    check(L.nrgbd_depth_regression(ptr(bv), H * W, D, H * W, 1, ptr(dpl), 1 if BV_log else 0, ptr(depth),
                                   ptr(conf), _stream()))
    return depth, conf


class _DepthRegression(torch.autograd.Function):
    """depth_val_regression with the gradient autograd gives the reference (misc.py:541-546): slice 0 of BV_measure
    gets g * d (times exp(BV) when BV_log), the other slices zero. The plane depths get no gradient, and the
    `return_conf` output has no backward: differentiating it raises."""

    @staticmethod
    def forward(ctx, BV_measure, dpl, BV_log, return_conf):
        ctx.set_materialize_grads(False)
        bv = BV_measure.detach()[0].float().contiguous()
        ctx.save_for_backward(bv, dpl)
        ctx.meta = (BV_log, tuple(BV_measure.shape), BV_measure.dtype)
        depth, conf = _regression_forward(bv, dpl, BV_log, return_conf)
        return (depth, conf) if return_conf else depth

    @staticmethod
    def backward(ctx, grad_depth, grad_conf=None):
        if grad_conf is not None:
            raise NotImplementedError('depth_val_regression: the confidence output (return_conf=True) has no gradient')
        if grad_depth is None:
            return None, None, None, None
        L = _lib.lib()
        bv, dpl = ctx.saved_tensors
        BV_log, (N, D, H, W), dtype = ctx.meta
        with torch.cuda.device(bv.device):
            g = grad_depth.detach().float().contiguous()
            g_bv = torch.empty((N, D, H, W), device=bv.device, dtype=torch.float32)
            check(L.nrgbd_depth_regression_backward(ptr(g), ptr(bv), H * W, D, H * W, 1, ptr(dpl), 1 if BV_log else 0,
                                                    ptr(g_bv[0]), _stream()))
            if N > 1:          # the reference reads BV_measure[0] only
                g_bv[1:].zero_()
        return g_bv.to(dtype), None, None, None


def depth_val_regression(BV_measure, d_candi_cur, BV_log=True, return_conf=False):
    """misc.py:532-548: depth = sum_d exp(BV[0,d]) * d -> [1,h,w]. One kernel instead of D launches.
    Differentiable w.r.t. BV_measure when it requires grad (the reference trains through it: models/KVNET.py:129,176,
    train_utils/train_KVNet.py:137-142); d_candi_cur gets no gradient, and neither does the `conf` output."""
    assert len(d_candi_cur) == BV_measure.shape[1], \
        'BV_measure should have the same # of slices as len(d_candi_cur) !'
    if not BV_measure.is_cuda:
        raise _lib.NrgbdError('neuralrgbd_b200 has no CPU path: expected a CUDA tensor')
    with torch.cuda.device(BV_measure.device):
        dpl = planes_tensor(d_candi_cur, BV_measure.device)
        if torch.is_grad_enabled() and BV_measure.requires_grad:
            return _DepthRegression.apply(BV_measure, dpl, BV_log, return_conf)
        depth, conf = _regression_forward(BV_measure[0].float().contiguous(), dpl, BV_log, return_conf)
    return (depth, conf) if return_conf else depth


def _var_div(d_sigma):
    """2 * d_sigma**2 as the reference's divisor: computed in double, rounded to fp32 as ATen does with a Python scalar."""
    return float(np.float32(2 * d_sigma ** 2))


def _var_forward(bv, dpl, mean, BV_log, div):
    L = _lib.lib()
    D, H, W = bv.shape
    var = torch.empty((H * W,), device=bv.device, dtype=torch.float32)
    check(L.nrgbd_depth_var(ptr(bv), H * W, D, H * W, 1, ptr(dpl), 1 if BV_log else 0, ptr(mean), div, ptr(var),
                            _stream()))
    return var


class _DepthVar(torch.autograd.Function):
    """depth_var with the gradient autograd gives the reference (misc.py:566-572): slice 0 of BV_measure and the
    (broadcast) mean map get their gradients from one kernel, the other slices zero. The plane depths get none."""

    @staticmethod
    def forward(ctx, BV_measure, mean, dpl, BV_log, div, shape):
        ctx.set_materialize_grads(False)
        bv = BV_measure.detach()[0].float().contiguous()
        mu = mean.detach().to(bv.device, torch.float32).reshape(-1).contiguous()
        ctx.save_for_backward(bv, mu, dpl)
        ctx.meta = (BV_log, div, shape, tuple(BV_measure.shape), BV_measure.dtype, mean.dtype)
        return _var_forward(bv, dpl, mu, BV_log, div).reshape(shape)

    @staticmethod
    def backward(ctx, grad_var):
        if grad_var is None:
            return (None,) * 6
        L = _lib.lib()
        bv, mu, dpl = ctx.saved_tensors
        BV_log, div, shape, (N, D, H, W), bv_dtype, mu_dtype = ctx.meta
        want_bv, want_mu = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        with torch.cuda.device(bv.device):
            g = grad_var.detach().to(bv.device, torch.float32).reshape(-1).contiguous()
            g_bv = torch.empty((N, D, H, W), device=bv.device, dtype=torch.float32) if want_bv else None
            g_mu = torch.empty(shape, device=bv.device, dtype=torch.float32) if want_mu else None
            check(L.nrgbd_depth_var_backward(ptr(g), ptr(bv), H * W, D, H * W, 1, ptr(dpl), 1 if BV_log else 0, ptr(mu), div,
                                             ptr(g_bv[0]) if want_bv else None, ptr(g_mu), _stream()))
            if want_bv and N > 1:      # the reference reads BV_measure[0] only
                g_bv[1:].zero_()
        return (g_bv.to(bv_dtype) if want_bv else None, g_mu.to(mu_dtype) if want_mu else None,
                None, None, None, None)


def depth_var(BV_measure, depth_mean, d_candi_cur, BV_log=True, d_sigma=1.):
    """misc.py:550-572: var = sum_d (p_d * d - depth_mean)^2 / (2 d_sigma^2) / D over slice 0 of BV_measure, in the
    reference's sequential order. One kernel instead of about 6 D launches; the result lives on BV_measure's device and
    has the reference's broadcast shape (1 x H x W for a 1 x H x W depth_mean, H x W for an H x W one).
    Differentiable w.r.t. BV_measure and depth_mean when either requires grad (train_utils/train_KVNet.py:137-145)."""
    assert len(d_candi_cur) == BV_measure.shape[1], 'BV_measure should have the same # of slices as len(d_candi_cur) !'
    N, D, H, W = BV_measure.shape
    if not BV_measure.is_cuda:
        raise _lib.NrgbdError('neuralrgbd_b200 has no CPU path: expected a CUDA tensor')
    with torch.cuda.device(BV_measure.device):
        if not torch.is_tensor(depth_mean):
            depth_mean = torch.as_tensor(depth_mean, dtype=torch.float32, device=BV_measure.device)
        shape = torch.broadcast_shapes((H, W), depth_mean.shape)
        if int(np.prod(shape)) != H * W:
            raise NotImplementedError('depth_var: depth_mean %s broadcasts to %s; one mean per pixel (H x W, 1 x H x W, '
                                      '...) is supported' % (tuple(depth_mean.shape), tuple(shape)))
        # broadcast outside the Function: autograd's expand backward sums the gradient to depth_mean's shape
        mean = depth_mean.expand(shape)
        dpl = planes_tensor(d_candi_cur, BV_measure.device)
        div = _var_div(d_sigma)
        if torch.is_grad_enabled() and (BV_measure.requires_grad or mean.requires_grad):
            return _DepthVar.apply(BV_measure, mean, dpl, BV_log, div, shape)
        mu = mean.to(BV_measure.device, torch.float32).reshape(-1).contiguous()
        return _var_forward(BV_measure[0].float().contiguous(), dpl, mu, BV_log, div).reshape(shape)


def _extreme_forward(bv, BV_log, is_min, want_index):
    L = _lib.lib()
    N, D, H, W = bv.shape
    value = torch.empty((N, H, W), device=bv.device, dtype=torch.float32)
    index = torch.empty((N, H, W), device=bv.device, dtype=torch.int32) if want_index else None
    check(L.nrgbd_dpv_extreme(ptr(bv), H * W, N, D, D * H * W, H * W, 1, 1 if BV_log else 0, 1 if is_min else 0,
                              ptr(value), ptr(index), _stream()))
    return value, index


class _DpvExtreme(torch.autograd.Function):
    """torch.max / torch.min over the planes of exp(BV_measure) (or BV_measure) as misc.py:600-603 uses them: the value's
    gradient goes to the plane ATen's max.dim / min.dim select, times exp(BV) when BV_log."""

    @staticmethod
    def forward(ctx, BV_measure, BV_log, is_min):
        ctx.set_materialize_grads(False)
        bv = BV_measure.detach().float().contiguous()
        value, index = _extreme_forward(bv, BV_log, is_min, True)
        ctx.save_for_backward(bv, index)
        ctx.meta = (BV_log, BV_measure.dtype)
        return value

    @staticmethod
    def backward(ctx, grad_value):
        if grad_value is None:
            return None, None, None
        L = _lib.lib()
        bv, index = ctx.saved_tensors
        BV_log, dtype = ctx.meta
        N, D, H, W = bv.shape
        with torch.cuda.device(bv.device):
            g = grad_value.detach().to(bv.device, torch.float32).contiguous()
            g_bv = torch.empty((N, D, H, W), device=bv.device, dtype=torch.float32)
            check(L.nrgbd_dpv_extreme_backward(ptr(g), ptr(bv), ptr(index), H * W, N, D, D * H * W, H * W, 1,
                                               1 if BV_log else 0, ptr(g_bv), _stream()))
        return g_bv.to(dtype), None, None


def _dpv_extreme(BV_measure, BV_log, is_min):
    """[N, D, H, W] -> [N, H, W]: max_d (is_min: min_d) of exp(BV) (BV_log) or BV, on BV_measure's device."""
    if not BV_measure.is_cuda:
        raise _lib.NrgbdError('neuralrgbd_b200 has no CPU path: expected a CUDA tensor')
    with torch.cuda.device(BV_measure.device):
        if torch.is_grad_enabled() and BV_measure.requires_grad:
            return _DpvExtreme.apply(BV_measure, BV_log, is_min)
        return _extreme_forward(BV_measure.float().contiguous(), BV_log, is_min, False)[0]


# dpv_statistics selects its statistics by identity (`name is 'E_mean'`, misc.py:594-602). These constants are the same
# interned objects as the literals in a caller's code, so `is` against them keeps that behaviour (a name built at run
# time is skipped, as in the reference) without comparing against a literal.
_E_MEAN, _VARIANCE, _MAX, _MIN = 'E_mean', 'variance', 'max', 'min'


def dpv_statistics(BV_measure, d_candi, statistics, BV_log=True):
    """misc.py:574-608: the statistics named in `statistics` stacked as channels, NCHW. Composed of the mirrors
    (depth_val_regression, depth_var, and one kernel per 'max' / 'min'), so autograd sees the reference's graph.
    The reference's behaviour is kept as is: 'variance' needs an 'E_mean' before it (UnboundLocalError otherwise),
    'min' with BV_log=False gives the max over the planes, 'max' / 'min' have N channels where 'E_mean' / 'variance'
    have one (torch.cat fails for N > 1 when both kinds are asked for), and an empty selection fails the same assert."""
    dpv_feats = []
    for name in statistics:
        if name is _E_MEAN:
            depth_regress = depth_val_regression(BV_measure, d_candi, BV_log=BV_log)
            dpv_feats.append(depth_regress.unsqueeze(1))
        if name is _VARIANCE:
            dpv_feats.append(depth_var(BV_measure, depth_regress, d_candi, BV_log=BV_log).unsqueeze(1))
        if name is _MAX:
            dpv_feats.append(_dpv_extreme(BV_measure, BV_log, False).unsqueeze(1))
        if name is _MIN:
            dpv_feats.append(_dpv_extreme(BV_measure, BV_log, BV_log).unsqueeze(1))     # the max without BV_log (:603)

    assert len(dpv_feats) > 0, 'No channels in dpv_feats. Did you specify the right dpv statistics ?'
    return torch.cat(dpv_feats, dim=1)
