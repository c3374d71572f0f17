"""Deformable convolution v1 as an autograd Function and modules on libtt_b200.

Mirror of mmcv 1.7's `mmcv.ops.deform_conv` (`DeformConv2dFunction`, `deform_conv2d`, `DeformConv2d`, `DeformConv2dPack`), which the
reference builds as the DepthNet's `'DCN'` conv layer (open_loop_training/code/model_code/backbones/lss.py:189-197): same arguments,
same saved tensors, same gradient tuple, same parameter names -- with `ext_module.deform_conv_forward / _backward_input /
_backward_parameters` replaced by the C ABI entries `tt_deform_conv_forward / _backward` (include/tt_b200.h §12).  SURVEY.md §8f row f4.
As in mmcv, `conv_offset` is an ordinary zero-initialised `nn.Conv2d`; only the deformable part is the native op.
"""
import ctypes as C
import math

import torch
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

from .. import lib
from ..lib import _p


def _desc(input, weight, stride, padding, dilation, groups, deform_groups, im2col_step):
    def one(v):                                                     # (a, b) with a != b is refused by the library as "not 1"
        return v[0] if v[0] == v[1] else 0
    d = lib.DeformConvDesc()
    d.N, d.C, d.H, d.W = input.shape
    d.Cout, d.groups, d.im2col_step = weight.shape[0], groups, im2col_step
    d.kernel_h, d.kernel_w = weight.shape[2], weight.shape[3]
    d.stride, d.padding, d.dilation, d.deform_groups = one(stride), one(padding), one(dilation), deform_groups
    return d


def _check(d, input, offset, weight):
    for t in (input, offset, weight):
        if not (t.is_cuda and t.dtype == torch.float32):
            raise lib.TTError('deform_conv2d needs fp32 CUDA tensors (no CPU fallback)')
    if weight.shape[1] * d.groups != d.C:
        raise lib.TTError(f'deform_conv2d: weight {tuple(weight.shape)} does not match {d.C} input channels in {d.groups} groups')
    want = (d.N, 2 * d.deform_groups * d.kernel_h * d.kernel_w, d.H, d.W)
    if tuple(offset.shape) != want:
        raise lib.TTError(f'deform_conv2d: offset {tuple(offset.shape)}, expected {want}')


def _workspace(d, device):
    n = int(lib.load().tt_deform_conv_workspace_bytes(C.byref(d)))
    return torch.empty(max(n, 1), dtype=torch.uint8, device=device), n


class DeformConv2dFunction(Function):
    @staticmethod
    def forward(ctx, input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deform_groups=1, bias=False, im2col_step=32):
        if input is not None and input.dim() != 4:
            raise ValueError(f'Expected 4D tensor as input, got {input.dim()}D tensor instead.')
        assert bias is False, 'Only support bias is False.'
        ctx.stride, ctx.padding, ctx.dilation = _pair(stride), _pair(padding), _pair(dilation)
        ctx.groups, ctx.deform_groups, ctx.im2col_step = groups, deform_groups, im2col_step
        input = input.type_as(offset)
        weight = weight.type_as(input)
        ctx.save_for_backward(input, offset, weight)
        cur_im2col_step = min(ctx.im2col_step, input.size(0))
        assert (input.size(0) % cur_im2col_step) == 0, 'batch size must be divisible by im2col_step'
        d = _desc(input, weight, ctx.stride, ctx.padding, ctx.dilation, groups, deform_groups, im2col_step)
        _check(d, input, offset, weight)
        input, offset, weight = input.contiguous(), offset.contiguous(), weight.contiguous()
        output = input.new_empty(d.N, d.Cout, d.H, d.W)
        ws, n = _workspace(d, input.device)
        lib.call('tt_deform_conv_forward', C.byref(d), _p(input), _p(offset), _p(weight), _p(output), _p(ws), C.c_size_t(n))
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        input, offset, weight = ctx.saved_tensors
        cur_im2col_step = min(ctx.im2col_step, input.size(0))
        assert (input.size(0) % cur_im2col_step) == 0, 'batch size must be divisible by im2col_step'
        grad_output = grad_output.contiguous()
        input, offset, weight = input.contiguous(), offset.contiguous(), weight.contiguous()
        need = ctx.needs_input_grad
        grad_input = torch.empty_like(input) if need[0] else None
        grad_offset = torch.empty_like(offset) if need[1] else None
        grad_weight = torch.empty_like(weight) if need[2] else None
        if grad_input is not None or grad_offset is not None or grad_weight is not None:
            d = _desc(input, weight, ctx.stride, ctx.padding, ctx.dilation, ctx.groups, ctx.deform_groups, ctx.im2col_step)
            ws, n = _workspace(d, input.device)
            lib.call('tt_deform_conv_backward', C.byref(d), _p(input), _p(offset), _p(weight), _p(grad_output), _p(grad_input),
                     _p(grad_offset), _p(grad_weight), _p(ws), C.c_size_t(n))
        return grad_input, grad_offset, grad_weight, None, None, None, None, None, None, None


deform_conv2d = DeformConv2dFunction.apply


class DeformConv2d(nn.Module):
    """mmcv.ops.DeformConv2d: `forward(x, offset)`, weight (out_channels, in_channels // groups, kh, kw), no bias."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, deform_groups=1, bias=False,
                 im2col_step=32):
        super().__init__()
        assert not bias, f'bias={bias} is not supported in DeformConv2d.'
        assert in_channels % groups == 0, f'in_channels {in_channels} cannot be divisible by groups {groups}'
        assert out_channels % groups == 0, f'out_channels {out_channels} cannot be divisible by groups {groups}'
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding, self.dilation = _pair(kernel_size), _pair(stride), _pair(padding), _pair(dilation)
        self.groups, self.deform_groups, self.im2col_step = groups, deform_groups, im2col_step
        self.transposed = False
        self.output_padding = (0,)
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        self.reset_parameters()

    def reset_parameters(self):
        n = self.in_channels
        for k in self.kernel_size:
            n *= k
        stdv = 1. / math.sqrt(n)
        self.weight.data.uniform_(-stdv, stdv)

    def forward(self, x, offset):
        return deform_conv2d(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups, self.deform_groups, False,
                             self.im2col_step)


class DeformConv2dPack(DeformConv2d):
    """mmcv.ops.DeformConv2dPack (registered by mmcv as the 'DCN' conv layer): the offsets come from `conv_offset`, a
    zero-initialised nn.Conv2d with the layer's kernel, stride, padding and dilation, so a fresh layer starts as a plain conv."""
    _version = 2

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_offset = nn.Conv2d(self.in_channels, self.deform_groups * 2 * self.kernel_size[0] * self.kernel_size[1],
                                     kernel_size=self.kernel_size, stride=self.stride, padding=self.padding, dilation=self.dilation,
                                     bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset.weight.data.zero_()
        self.conv_offset.bias.data.zero_()

    def forward(self, x):
        offset = self.conv_offset(x)
        return deform_conv2d(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups, self.deform_groups, False,
                             self.im2col_step)
