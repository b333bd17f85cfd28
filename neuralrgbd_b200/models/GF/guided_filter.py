"""Mirror of the reference's models/GF/guided_filter.py GuidedFilter(r, eps): the whole filter is one libnrgbd forward
(5 launches) and one backward (10 launches), in place of about 75 ATen kernels forward and as many again under autograd.
FastGuidedFilter is not mirrored: nothing in the reference constructs it."""
import ctypes

import torch
from torch import nn

from ... import _lib
from ..._lib import ptr, check
from .box_filter import BoxFilter, require_cuda_f32


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _workspace(N, Cx, Cy, H, W, backward, device):
    n = _lib.lib().nrgbd_gf_workspace_floats(N, Cx, Cy, H, W, 1 if backward else 0)
    return torch.empty((n,), device=device, dtype=torch.float32)


def _gf_forward(x, y, r, eps):
    L = _lib.lib()
    N, Cx, H, W = x.shape
    Cy = y.shape[1]
    out = torch.empty((N, Cy, H, W), device=x.device, dtype=torch.float32)
    ws = _workspace(N, Cx, Cy, H, W, False, x.device)
    check(L.nrgbd_guided_filter(ptr(x), ptr(y), N, Cx, Cy, H, W, r, eps, ptr(ws), ptr(out), _stream()))
    return out


class _GuidedFilter(torch.autograd.Function):
    """GuidedFilter.forward with the gradients autograd gives the reference through guided_filter.py:76-97 and
    box_filter.py. Only x and y are saved: the backward recomputes the box sums (DESIGN §6.7)."""

    @staticmethod
    def forward(ctx, x, y, r, eps):
        ctx.set_materialize_grads(False)
        xs, ys = x.detach().contiguous(), y.detach().contiguous()
        ctx.save_for_backward(xs, ys)
        ctx.meta = (r, eps)
        return _gf_forward(xs, ys, r, eps)

    @staticmethod
    def backward(ctx, g):
        if g is None:
            return None, None, None, None
        L = _lib.lib()
        x, y = ctx.saved_tensors
        r, eps = ctx.meta
        N, Cx, H, W = x.shape
        Cy = y.shape[1]
        want_x, want_y = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        with torch.cuda.device(x.device):
            g = g.detach().to(x.device, torch.float32).contiguous()
            gx = torch.empty_like(x) if want_x else None
            gy = torch.empty_like(y) if want_y else None
            ws = _workspace(N, Cx, Cy, H, W, True, x.device)
            check(L.nrgbd_guided_filter_backward(ptr(g), ptr(x), ptr(y), N, Cx, Cy, H, W, r, eps, ptr(ws), ptr(gx), ptr(gy),
                                                 _stream()))
        return gx, gy, None, None


class GuidedFilter(nn.Module):
    """models/GF/guided_filter.py GuidedFilter(r, eps): same constructor, attributes (r, eps, boxfilter) and forward;
    no parameters or buffers. x (N x C_x x H x W, C_x = 1 or C_y) guides y (N x C_y x H x W); float32 CUDA tensors."""

    def __init__(self, r, eps=1e-8):
        super(GuidedFilter, self).__init__()
        self.r = r
        self.eps = eps
        self.boxfilter = BoxFilter(r)

    def forward(self, x, y):
        '''
        x, y - x: guided signal ( features high res. rgb image)
               y: upsampled target image we want to refine.
               e.g.  This could be an upsampled depth image
        '''
        n_x, c_x, h_x, w_x = x.size()
        n_y, c_y, h_y, w_y = y.size()

        assert n_x == n_y
        assert c_x == 1 or c_x == c_y
        assert h_x == h_y and w_x == w_y
        assert h_x > 2 * self.r + 1 and w_x > 2 * self.r + 1

        require_cuda_f32(x, y)
        with torch.cuda.device(x.device):
            if torch.is_grad_enabled() and (x.requires_grad or y.requires_grad):
                return _GuidedFilter.apply(x, y, self.r, self.eps)
            return _gf_forward(x.contiguous(), y.contiguous(), self.r, self.eps)
