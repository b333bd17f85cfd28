"""Mirror of the reference's models/GF/box_filter.py: BoxFilter(r) as two libnrgbd scans (cumsum + diff along H, then
along W), with a backward kernel pair (the diff's adjoint + a reverse prefix sum, along W then H)."""
import ctypes

import torch
from torch import nn

from ... import _lib
from ..._lib import ptr, check


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda_f32(*ts):
    for t in ts:
        if not t.is_cuda:
            raise _lib.NrgbdError('neuralrgbd_b200 has no CPU path: expected a CUDA tensor')
        if t.dtype != torch.float32:
            raise _lib.NrgbdError('models.GF mirrors compute in float32: got %s' % t.dtype)
    if any(t.device != ts[0].device for t in ts):
        raise _lib.NrgbdError('expected all tensors on one device, got %s' % ', '.join(str(t.device) for t in ts))


def _box_forward(x, r):
    L = _lib.lib()
    N, C, H, W = x.shape
    out = torch.empty_like(x)
    ws = torch.empty((L.nrgbd_box_filter_workspace_floats(N, C, H, W),), device=x.device, dtype=torch.float32)
    check(L.nrgbd_box_filter(ptr(x), N, C, H, W, r, ptr(ws), ptr(out), _stream()))
    return out


class _BoxFilter(torch.autograd.Function):
    """BoxFilter.forward with the gradient autograd gives the reference: box_filter.py's diff_y / diff_x adjoints and
    cumsum's backward (a reverse prefix sum), rows first, in one kernel per axis."""

    @staticmethod
    def forward(ctx, x, r):
        ctx.r = r
        return _box_forward(x.detach().contiguous(), r)

    @staticmethod
    def backward(ctx, g):
        L = _lib.lib()
        g = g.detach().contiguous()
        N, C, H, W = g.shape
        with torch.cuda.device(g.device):
            gx = torch.empty_like(g)
            ws = torch.empty((L.nrgbd_box_filter_workspace_floats(N, C, H, W),), device=g.device, dtype=torch.float32)
            check(L.nrgbd_box_filter_backward(ptr(g), N, C, H, W, ctx.r, ptr(ws), ptr(gx), _stream()))
        return gx, None


def box_filter(x, r):
    """box_filter.py:34 on an N x C x H x W float32 CUDA tensor (H, W >= 2r + 1). Differentiable when x requires grad;
    otherwise the same kernels run without autograd, with bit-identical values."""
    require_cuda_f32(x)
    with torch.cuda.device(x.device):
        if torch.is_grad_enabled() and x.requires_grad:
            return _BoxFilter.apply(x, r)
        return _box_forward(x.contiguous(), r)


class BoxFilter(nn.Module):
    """models/GF/box_filter.py BoxFilter(r): no parameters, no buffers."""

    def __init__(self, r):
        super(BoxFilter, self).__init__()

        self.r = r

    def forward(self, x):
        assert x.dim() == 4

        return box_filter(x, self.r)
