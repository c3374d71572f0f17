"""Training-side transposed convolution: `torch.nn.ConvTranspose2d` forward and backward on libtt_b200 (include/tt_b200.h §17).

`ConvTranspose2d` is an `nn.ConvTranspose2d` with the same constructor, parameters and `state_dict`, whose passes run the §16
convolution kernels (a transposed convolution is the adjoint of a Conv2d with the same weight tensor) on `channels_last` fp32 tensors:
3xTF32 products, fp32-class accuracy (cuDNN's default single-pass TF32 keeps a 10-bit mantissa), every output and gradient bitwise
reproducible.  `convert_upsampling(module)` swaps every eligible `nn.ConvTranspose2d` and bilinear `nn.Upsample` of a model for the
library's modules, sharing the `Parameter` objects.  There is no fallback: CPU tensors, other dtypes and configurations the library
refuses raise `TTError`.
"""
import ctypes as C

import torch
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import lib
from ..lib import _p
from .conv2d import swap_modules
from .interpolate import Upsample, config_error as interp_config_error


def _desc(N, H, W, Cin, Cout, kernel_size, stride, pad, output_padding, dil, groups, bias):
    d = lib.ConvTranspose2dTrainDesc()
    d.N, d.H, d.W, d.Cin, d.Cout = N, H, W, Cin, Cout
    d.KH, d.KW = kernel_size
    d.stride, d.pad, d.output_padding, d.dil, d.groups, d.bias = stride, pad, output_padding, dil, groups, int(bool(bias))
    d.OH = (H - 1) * stride - 2 * pad + d.KH + output_padding
    d.OW = (W - 1) * stride - 2 * pad + d.KW + output_padding
    return d


def _config_error(in_channels, out_channels, kernel_size, stride, padding, output_padding, dilation, groups, padding_mode):
    """why the library refuses this layer (the parameter named), or None; no tensor and no device needed."""
    if padding_mode != 'zeros':
        return f'padding_mode: {padding_mode!r} (only zeros)'
    for name, v in (('stride', stride), ('padding', padding), ('output_padding', output_padding), ('dilation', dilation)):
        if v[0] != v[1]:
            return f'{name}: {tuple(v)} (only equal height and width)'
    if dilation[0] != 1:
        return f'dilation: {tuple(dilation)} (only 1)'
    H = 2 * padding[0] + 2                                           # large enough for a positive output size
    d = _desc(1, H, H, in_channels, out_channels, kernel_size, stride[0], padding[0], output_padding[0], 1, groups, False)
    if int(lib.load().tt_conv_transpose2d_train_workspace_bytes(C.byref(d))) == 0:
        return lib.load().tt_last_error().decode().split('unsupported ', 1)[-1]
    return None


def _check(tensors):
    for t in tensors:
        if t is not None and not (t.is_cuda and t.dtype == torch.float32):
            raise lib.TTError('conv_transpose2d needs fp32 CUDA tensors (no CPU fallback)')


def _workspace(d, device):
    n = int(lib.load().tt_conv_transpose2d_train_workspace_bytes(C.byref(d)))
    if n == 0:
        raise lib.TTError(f'conv_transpose2d: {lib.load().tt_last_error().decode()}')
    return torch.empty(n, dtype=torch.uint8, device=device), n


def _layer_desc(x, weight, has_bias, stride, pad, output_padding):
    N, Cin, H, W = x.shape
    if weight.shape[0] != Cin:
        raise lib.TTError(f'conv_transpose2d: weight {tuple(weight.shape)} does not match {Cin} input channels')
    return _desc(N, H, W, Cin, weight.shape[1], tuple(weight.shape[2:]), stride, pad, output_padding, 1, 1, has_bias)


def _forward(x, weight, bias, stride, pad, output_padding):
    """y = conv_transpose2d(x, weight, bias) with x channels_last-contiguous."""
    d = _layer_desc(x, weight, bias is not None, stride, pad, output_padding)
    ws, n = _workspace(d, x.device)
    y = torch.empty((d.N, d.Cout, d.OH, d.OW), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
    lib.call('tt_conv_transpose2d_train_forward', C.byref(d), _p(x), _p(weight), _p(bias), _p(y), _p(ws), C.c_size_t(n))
    return y


class ConvTranspose2dFunction(Function):
    """conv_transpose2d(x, weight, bias, stride, padding, output_padding) with both passes on the library; x and the output are
    channels_last."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, output_padding):
        _check((x, weight, bias))
        x = x.contiguous(memory_format=torch.channels_last)
        weight = weight.contiguous()
        y = _forward(x, weight, bias, stride, padding, output_padding)
        ctx.save_for_backward(x, weight)
        ctx.conf = (stride, padding, output_padding, bias is not None)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_y):
        x, weight = ctx.saved_tensors
        stride, pad, output_padding, has_bias = ctx.conf
        need = ctx.needs_input_grad
        _check((grad_y,))
        grad_y = grad_y.contiguous(memory_format=torch.channels_last)
        grad_x = torch.empty_like(x, memory_format=torch.channels_last) if need[0] else None
        grad_w = torch.empty_like(weight) if need[1] else None
        grad_b = weight.new_empty(weight.shape[1]) if has_bias and need[2] else None
        if grad_x is not None or grad_w is not None or grad_b is not None:
            d = _layer_desc(x, weight, has_bias, stride, pad, output_padding)
            ws, n = _workspace(d, x.device)
            lib.call('tt_conv_transpose2d_train_backward', C.byref(d), _p(x), _p(weight), _p(grad_y), _p(grad_x), _p(grad_w), _p(grad_b),
                     _p(ws), C.c_size_t(n))
        return grad_x, grad_w, grad_b, None, None, None


class ConvTranspose2d(nn.ConvTranspose2d):
    """nn.ConvTranspose2d on the library: same constructor, parameters and state_dict.  forward(x, output_size=None) resolves
    output_size as torch does; the output is channels_last; under no_grad (or with nothing requiring a gradient) nothing is saved."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        why = _config_error(self.in_channels, self.out_channels, self.kernel_size, self.stride, self.padding, self.output_padding,
                            self.dilation, self.groups, self.padding_mode)
        if why is not None:
            raise lib.TTError(f'ConvTranspose2d: unsupported {why}')

    def forward(self, x, output_size=None):
        op = self._output_padding(x, output_size, self.stride, self.padding, self.kernel_size, 2, self.dilation)
        if op[0] != op[1]:
            raise lib.TTError(f'ConvTranspose2d: unsupported output_size {list(output_size)}: output padding {tuple(op)} '
                              '(only equal height and width)')
        params = (self.weight, self.bias)
        if torch.is_grad_enabled() and (x.requires_grad or any(t is not None and t.requires_grad for t in params)):
            return ConvTranspose2dFunction.apply(x, self.weight, self.bias, self.stride[0], self.padding[0], op[0])
        _check((x, self.weight, self.bias))
        return _forward(x.contiguous(memory_format=torch.channels_last), self.weight.contiguous(), self.bias, self.stride[0],
                        self.padding[0], op[0])


def convert_upsampling(module, prefix=''):
    """Swap every eligible `nn.ConvTranspose2d` for `ConvTranspose2d` (sharing its weight and bias `Parameter` objects) and every bilinear
    align_corners=True `nn.Upsample` for `Upsample` in `module` (itself included), keeping each layer's training flag.  Returns
    (module, skipped): skipped lists (qualified name, layer, reason) for every `nn.ConvTranspose2d` / `nn.Upsample` left alone.  Other
    module types are untouched; an F.interpolate call inside a forward is out of a module swap's reach (use interpolate_bilinear)."""
    skipped = []

    def swap(m, name):
        if type(m) is nn.ConvTranspose2d:
            why = _config_error(m.in_channels, m.out_channels, m.kernel_size, m.stride, m.padding, m.output_padding, m.dilation, m.groups,
                                m.padding_mode)
            if why is not None:
                skipped.append((name, m, why))
                return m
            new = ConvTranspose2d(m.in_channels, m.out_channels, m.kernel_size, stride=m.stride, padding=m.padding,
                                  output_padding=m.output_padding, groups=m.groups, bias=m.bias is not None, dilation=m.dilation,
                                  padding_mode=m.padding_mode, device='meta')
            new.weight = m.weight
            new.bias = m.bias
        elif type(m) is nn.Upsample:
            why = interp_config_error(m.mode, m.align_corners)
            if why is not None:
                skipped.append((name, m, why))
                return m
            new = Upsample(size=m.size, scale_factor=m.scale_factor, mode=m.mode, align_corners=m.align_corners,
                           recompute_scale_factor=m.recompute_scale_factor)
        else:
            return m
        new.train(m.training)
        return new

    return swap_modules(module, prefix, swap), skipped
