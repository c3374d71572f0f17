"""Training-side dense convolution: `torch.nn.Conv2d` forward and backward on libtt_b200 (include/tt_b200.h §16).

`Conv2d` is an `nn.Conv2d` with the same constructor, parameters and `state_dict`, whose forward and backward run the library's
3xTF32 tensor-core kernels on `channels_last` fp32 tensors: fp32-class accuracy (cuDNN's default single-pass TF32 keeps a 10-bit
mantissa), and every output and gradient bitwise reproducible from run to run.  `convert_conv2d(module)` swaps every eligible
`nn.Conv2d` of a model for it, in the style of `torch.nn.SyncBatchNorm.convert_sync_batchnorm`, sharing the `Parameter` objects.
There is no fallback: CPU tensors, other dtypes and configurations the library refuses raise `TTError`.
"""
import ctypes as C

import torch
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import lib
from ..lib import _p


def _config_error(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, padding_mode):
    """why the library refuses this layer (the parameter named), or None; no tensor and no device needed."""
    if padding_mode != 'zeros':
        return f'padding_mode: {padding_mode!r} (only zeros)'
    if isinstance(padding, str):
        return f'padding: {padding!r} (only integers)'
    for name, v in (('stride', stride), ('padding', padding), ('dilation', dilation)):
        if v[0] != v[1]:
            return f'{name}: {tuple(v)} (only equal height and width)'
    kh, kw = kernel_size
    d = _desc(1, kh * dilation[0] + 2, kw * dilation[1] + 2, in_channels, out_channels, kernel_size, stride[0], padding[0], dilation[0],
              groups, False)
    if int(lib.load().tt_conv2d_train_workspace_bytes(C.byref(d))) == 0:
        return lib.load().tt_last_error().decode().split('unsupported ', 1)[-1]
    return None


def _desc(N, H, W, Cin, Cout, kernel_size, stride, pad, dil, groups, bias):
    d = lib.Conv2dTrainDesc()
    d.N, d.H, d.W, d.Cin, d.Cout = N, H, W, Cin, Cout
    d.KH, d.KW = kernel_size
    d.stride, d.pad, d.dil, d.groups, d.bias = stride, pad, dil, groups, int(bool(bias))
    d.OH = (H + 2 * pad - dil * (d.KH - 1) - 1) // stride + 1
    d.OW = (W + 2 * pad - dil * (d.KW - 1) - 1) // stride + 1
    return d


def _check(tensors):
    for t in tensors:
        if t is not None and not (t.is_cuda and t.dtype == torch.float32):
            raise lib.TTError('conv2d needs fp32 CUDA tensors (no CPU fallback)')


def _workspace(d, device):
    n = int(lib.load().tt_conv2d_train_workspace_bytes(C.byref(d)))
    if n == 0:
        raise lib.TTError(f'conv2d: {lib.load().tt_last_error().decode()}')
    return torch.empty(n, dtype=torch.uint8, device=device), n


def _forward(x, weight, bias, stride, pad, dil):
    """y = conv2d(x, weight, bias) with x channels_last-contiguous; returns (y, descriptor)."""
    N, Cin, H, W = x.shape
    d = _desc(N, H, W, Cin, weight.shape[0], tuple(weight.shape[2:]), stride, pad, dil, 1, bias is not None)
    if weight.shape[1] != Cin:
        raise lib.TTError(f'conv2d: weight {tuple(weight.shape)} does not match {Cin} input channels')
    ws, n = _workspace(d, x.device)
    y = torch.empty((N, d.Cout, d.OH, d.OW), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
    lib.call('tt_conv2d_train_forward', C.byref(d), _p(x), _p(weight), _p(bias), _p(y), _p(ws), C.c_size_t(n))
    return y, d


class Conv2dFunction(Function):
    """conv2d(x, weight, bias, stride, padding, dilation) with both passes on the library; x and the output are channels_last."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, dilation):
        _check((x, weight, bias))
        x = x.contiguous(memory_format=torch.channels_last)
        weight = weight.contiguous()
        y, _ = _forward(x, weight, bias, stride, padding, dilation)
        ctx.save_for_backward(x, weight)
        ctx.conf = (stride, padding, dilation, bias is not None)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_y):
        x, weight = ctx.saved_tensors
        stride, pad, dil, has_bias = ctx.conf
        need = ctx.needs_input_grad
        _check((grad_y,))
        grad_y = grad_y.contiguous(memory_format=torch.channels_last)
        grad_x = torch.empty_like(x, memory_format=torch.channels_last) if need[0] else None
        grad_w = torch.empty_like(weight) if need[1] else None
        grad_b = weight.new_empty(weight.shape[0]) if has_bias and need[2] else None
        if grad_x is not None or grad_w is not None or grad_b is not None:
            N, Cin, H, W = x.shape
            d = _desc(N, H, W, Cin, weight.shape[0], tuple(weight.shape[2:]), stride, pad, dil, 1, has_bias)
            ws, n = _workspace(d, x.device)
            lib.call('tt_conv2d_train_backward', C.byref(d), _p(x), _p(weight), _p(grad_y), _p(grad_x), _p(grad_w), _p(grad_b), _p(ws),
                     C.c_size_t(n))
        return grad_x, grad_w, grad_b, None, None, None


class Conv2d(nn.Conv2d):
    """nn.Conv2d on the library: same constructor, parameters and state_dict.  The input is converted to channels_last once when it
    is not already, the output is channels_last; under no_grad (or with nothing requiring a gradient) nothing is saved."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        why = _config_error(self.in_channels, self.out_channels, self.kernel_size, self.stride, self.padding, self.dilation, self.groups,
                            self.padding_mode)
        if why is not None:
            raise lib.TTError(f'Conv2d: unsupported {why}')

    def forward(self, x):
        params = (self.weight, self.bias)
        if torch.is_grad_enabled() and (x.requires_grad or any(t is not None and t.requires_grad for t in params)):
            return Conv2dFunction.apply(x, self.weight, self.bias, self.stride[0], self.padding[0], self.dilation[0])
        _check((x, self.weight, self.bias))
        return _forward(x.contiguous(memory_format=torch.channels_last), self.weight.contiguous(), self.bias, self.stride[0],
                        self.padding[0], self.dilation[0])[0]


def convert_conv2d(module, prefix=''):
    """Swap every eligible `nn.Conv2d` in `module` (itself included) for `Conv2d`, sharing its weight and bias `Parameter` objects
    (optimizer state and checkpoints are unaffected).  Returns (module, skipped): skipped lists (qualified name, layer, reason) for
    every `nn.Conv2d` left alone, e.g. a 3-channel stem or an 18-channel offset conv.  Other module types are untouched."""
    skipped = []

    def swap(m, name):
        if type(m) is not nn.Conv2d:
            return m
        why = _config_error(m.in_channels, m.out_channels, m.kernel_size, m.stride, m.padding, m.dilation, m.groups, m.padding_mode)
        if why is not None:
            skipped.append((name, m, why))
            return m
        new = Conv2d(m.in_channels, m.out_channels, m.kernel_size, stride=m.stride, padding=m.padding, dilation=m.dilation,
                     groups=m.groups, bias=m.bias is not None, padding_mode=m.padding_mode, device='meta')
        new.weight = m.weight
        new.bias = m.bias
        new.train(m.training)
        return new

    return swap_modules(module, prefix, swap), skipped


def swap_modules(module, prefix, swap):
    """Replace `module` (itself included) and its descendants by swap(m, qualified name), which returns m to keep it; the children of a
    replaced module are not visited.  Returns the (possibly replaced) root."""
    def walk(m, name):
        for child_name, child in list(m.named_children()):
            full = f'{name}.{child_name}' if name else child_name
            new = swap(child, full)
            if new is not child:
                setattr(m, child_name, new)
            else:
                walk(child, full)

    root = swap(module, prefix)
    if root is module:
        walk(module, prefix)
    return root
