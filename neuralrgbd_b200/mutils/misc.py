"""Mirror of the hot-path helpers of the reference's `mutils.misc`
(/root/reference/code/mutils/misc.py:100-115, 509-517, 532-548)."""
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
