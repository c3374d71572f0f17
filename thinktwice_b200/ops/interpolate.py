"""Training-side bilinear interpolation (align_corners=True) on libtt_b200 (include/tt_b200.h §17).

`interpolate_bilinear(x, size, scale_factor)` is `F.interpolate(x, size, scale_factor, mode='bilinear', align_corners=True)` as an
autograd Function: the forward is ATen's CUDA arithmetic, the backward a gather without atomics, so grad_x is bitwise reproducible
(torch's CUDA bilinear backward scatters with atomics and is refused by `torch.use_deterministic_algorithms(True)`).  `Upsample` is the
`nn.Upsample` that calls it.  `channels_last` fp32 CUDA tensors in and out; there is no fallback: CPU tensors, other dtypes, other
modes and align_corners other than True raise `TTError`.
"""
import ctypes as C
import math

import torch
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import lib
from ..lib import _p


def config_error(mode, align_corners):
    """why the library refuses this interpolation (the parameter named), or None."""
    if mode != 'bilinear':
        return f'mode: {mode!r} (only bilinear)'
    if align_corners is not True:
        return f'align_corners: {align_corners!r} (only True)'
    return None


def _output_size(H, W, size, scale_factor):
    """F.interpolate's output size: `size`, or floor(input size x scale_factor) per dimension."""
    if (size is None) == (scale_factor is None):
        raise ValueError('interpolate_bilinear: give exactly one of size and scale_factor')
    if size is not None:
        oh, ow = (size, size) if isinstance(size, int) else tuple(size)
    else:
        sh, sw = tuple(scale_factor) if isinstance(scale_factor, (tuple, list)) else (scale_factor, scale_factor)
        oh, ow = math.floor(float(H) * sh), math.floor(float(W) * sw)
    return int(oh), int(ow)


def _desc(in_shape, OH, OW):
    d = lib.InterpBilinearTrainDesc()
    d.N, d.C, d.H, d.W = in_shape
    d.OH, d.OW, d.align_corners = OH, OW, 1
    return d


def _check(x):
    if not (x.is_cuda and x.dtype == torch.float32):
        raise lib.TTError('interpolate_bilinear needs fp32 CUDA tensors (no CPU fallback)')
    if x.dim() != 4:
        raise lib.TTError(f'interpolate_bilinear: input of shape {tuple(x.shape)} (only 4-D)')


def _forward(x, OH, OW):
    x = x.contiguous(memory_format=torch.channels_last)
    y = torch.empty((x.shape[0], x.shape[1], OH, OW), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
    lib.call('tt_interp_bilinear_train_forward', C.byref(_desc(x.shape, OH, OW)), _p(x), _p(y))
    return y


class InterpolateBilinearFunction(Function):
    """y = bilinear interpolation of x to OH x OW (align_corners=True), both passes on the library."""

    @staticmethod
    def forward(ctx, x, OH, OW):
        _check(x)
        ctx.in_shape = tuple(x.shape)
        return _forward(x, OH, OW)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_y):
        _check(grad_y)
        grad_y = grad_y.contiguous(memory_format=torch.channels_last)
        grad_x = torch.empty(ctx.in_shape, device=grad_y.device, dtype=grad_y.dtype, memory_format=torch.channels_last)
        d = _desc(ctx.in_shape, grad_y.shape[2], grad_y.shape[3])
        lib.call('tt_interp_bilinear_train_backward', C.byref(d), _p(grad_y), _p(grad_x))
        return grad_x, None, None


def interpolate_bilinear(x, size=None, scale_factor=None, align_corners=True):
    """F.interpolate(x, size, scale_factor, mode='bilinear', align_corners=True) on the library; the output is channels_last."""
    why = config_error('bilinear', align_corners)
    if why is not None:
        raise lib.TTError(f'interpolate_bilinear: unsupported {why}')
    OH, OW = _output_size(x.shape[-2], x.shape[-1], size, scale_factor)
    if torch.is_grad_enabled() and x.requires_grad:
        return InterpolateBilinearFunction.apply(x, OH, OW)
    _check(x)
    return _forward(x, OH, OW)


class Upsample(nn.Upsample):
    """nn.Upsample(mode='bilinear', align_corners=True) on the library; any other mode or align_corners raises TTError."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        why = config_error(self.mode, self.align_corners)
        if why is not None:
            raise lib.TTError(f'Upsample: unsupported {why}')

    def forward(self, x):
        return interpolate_bilinear(x, self.size, self.scale_factor, True)
