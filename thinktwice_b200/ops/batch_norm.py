"""Training-side batch normalization on libtt_b200 (include/tt_b200.h §18): BatchNorm1d / BatchNorm2d / SyncBatchNorm with batch
statistics, forward and backward, with an optional residual add and ReLU fused into the same passes.

`BatchNorm1d`, `BatchNorm2d` and `SyncBatchNorm` subclass torch's classes (same constructor, parameters, buffers, `state_dict` and
`num_batches_tracked`, and `isinstance(m, _BatchNorm)` holds), and their forward takes `forward(x, *, residual=None, relu=False)`:
y = relu(bn(x) + residual) in one pass forward and two backward.  Statistics are fp64 over fixed row chunks folded in a fixed order,
so every output is bitwise reproducible for a fixed split of the batch over ranks.  `SyncBatchNorm` follows torch's rule for when to
synchronize (training, `torch.distributed` initialized, more than one rank in its process group); each synchronized layer gathers a
3-double-per-channel record in the forward and a 2-double one in the backward (`dist.all_gather` with a tensor list, which gloo
supports), and, like torch's, leaves grad_weight / grad_bias per rank for the data-parallel wrapper to average.
`convert_batchnorm(module)` swaps every eligible layer of a model, sharing its `Parameter` and buffer objects, and fuses a directly
following `nn.ReLU`.  4-D input is taken as channels_last (converted once when it is not), 2-D input as (N, C) rows.  There is no
fallback: CPU tensors, other dtypes, 3-D input and configurations the library refuses raise `TTError`.
"""
import ctypes as C

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import lib
from ..lib import _p
from .sparse_conv import SparseSequential


def _desc(M, Cc, R=1, training=True, residual=False, relu=False, eps=1e-5, factor=0.0, count=0, affine=True, track=True):
    d = lib.BatchNormTrainDesc()
    d.M, d.count, d.C, d.R = M, count, Cc, R
    d.affine, d.track_running_stats, d.training, d.residual = int(affine), int(track), int(training), int(residual)
    d.act = lib.ACT_RELU if relu else lib.ACT_NONE
    d.eps, d.factor = eps, factor
    return d


def config_error(num_features, affine, track_running_stats):
    """why the library refuses this layer (the parameter named), or None; no tensor and no device needed."""
    d = _desc(0, num_features, affine=affine, track=track_running_stats)
    if int(lib.load().tt_batch_norm_train_workspace_bytes(C.byref(d))) == 0:
        return lib.load().tt_last_error().decode().split('unsupported ', 1)[-1]
    return None


def _rows(t):
    """(view of t as rows [M][C], t in the layout the rows alias): 4-D as channels_last, 2-D as is."""
    if t.dim() == 4:
        t = t.contiguous(memory_format=torch.channels_last)
        return t.permute(0, 2, 3, 1).view(-1, t.shape[1]), t
    if t.dim() == 2:
        t = t.contiguous()
        return t, t
    raise lib.TTError(f'batch_norm: input of shape {tuple(t.shape)} (only 2-D (N, C) and 4-D (N, C, H, W))')


def _check(tensors):
    for t in tensors:
        if t is not None and not (t.is_cuda and t.dtype == torch.float32):
            raise lib.TTError('batch_norm needs fp32 CUDA tensors (no CPU fallback)')


def _workspace(d, device):
    n = int(lib.load().tt_batch_norm_train_workspace_bytes(C.byref(d)))
    if n == 0:
        raise lib.TTError(f'batch_norm: {lib.load().tt_last_error().decode()}')
    return torch.empty(n, dtype=torch.uint8, device=device), n


def _gather(rec, group, world):
    """the ranks' records [world][len], in rank order (a rank with no rows sends zeros and still joins)."""
    out = rec.new_empty(world, rec.numel())
    dist.all_gather(list(out.unbind(0)), rec, group)
    return out


def _forward(x, r, weight, bias, running_mean, running_var, training, relu, eps, factor, group, world):
    """y = act(bn(x) (+ r)); returns (y, rows of x, rows of r, mean, invstd, count).  In eval mode mean / invstd are the running
    statistics (invstd: the running variance, as the library takes it)."""
    xr, xl = _rows(x)
    rr = None
    if r is not None:
        if r.shape != x.shape:
            raise lib.TTError(f'batch_norm: residual {tuple(r.shape)} does not match the input {tuple(x.shape)}')
        rr, _ = _rows(r)
    M, Cc = xr.shape
    if weight.shape[0] != Cc:
        raise lib.TTError(f'batch_norm: {weight.shape[0]} features, input of {Cc} channels')
    d = _desc(M, Cc, world, training, r is not None, relu, eps, factor)
    if training:
        ws, n = _workspace(d, x.device)
        rec = torch.empty(3 * Cc, dtype=torch.float64, device=x.device)
        lib.call('tt_batch_norm_train_stats', C.byref(d), _p(xr), _p(rec), _p(ws), C.c_size_t(n))
        recs = _gather(rec, group, world) if world > 1 else rec
        count = int(recs.view(world, 3 * Cc)[:, 0].sum().item()) if world > 1 else M
        if count <= 1:
            raise ValueError(f'Expected more than 1 value per channel when training, got input size {count}')
        mean, invstd = torch.empty(Cc, device=x.device), torch.empty(Cc, device=x.device)
        lib.call('tt_batch_norm_train_fold', C.byref(d), _p(recs), _p(running_mean), _p(running_var), _p(mean), _p(invstd))
    else:
        mean, invstd, count = running_mean, running_var, M
    y = torch.empty_like(xl)
    yr, _ = _rows(y)
    lib.call('tt_batch_norm_train_forward', C.byref(d), _p(xr), _p(rr), _p(weight), _p(bias), _p(mean), _p(invstd), _p(yr))
    return y, xr, rr, mean, invstd, count


class BatchNormFunction(Function):
    """y = act(batch_norm(x) (+ r)) with both passes on the library; the SyncBatchNorm gathers run in `group` when world > 1."""

    @staticmethod
    def forward(ctx, x, r, weight, bias, running_mean, running_var, training, relu, eps, factor, group, world):
        _check((x, r, weight, bias, running_mean, running_var))
        y, xr, rr, mean, invstd, count = _forward(x, r, weight, bias, running_mean, running_var, training, relu, eps, factor, group,
                                                  world)
        if not training:                                                  # the running statistics may change before the backward
            mean, invstd = mean.clone(), invstd.clone()
        ctx.save_for_backward(xr, rr, weight, bias, mean, invstd)
        ctx.conf = (training, relu, eps, count, group, world)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_y):
        xr, rr, weight, bias, mean, invstd = ctx.saved_tensors
        training, relu, eps, count, group, world = ctx.conf
        need = ctx.needs_input_grad
        _check((grad_y,))
        gyr, gyl = _rows(grad_y)
        M, Cc = xr.shape
        d = _desc(M, Cc, world, training, rr is not None, relu, eps, 0.0, count)
        grad_w = torch.empty_like(weight) if need[2] else None
        grad_b = torch.empty_like(bias) if need[3] else None
        recs = None
        if training or grad_w is not None or grad_b is not None:
            ws, n = _workspace(d, xr.device)
            rec = torch.empty(2 * Cc, dtype=torch.float64, device=xr.device)
            lib.call('tt_batch_norm_train_backward_reduce', C.byref(d), _p(xr), _p(rr), _p(weight), _p(bias), _p(mean), _p(invstd), _p(gyr),
                     _p(rec), _p(grad_w), _p(grad_b), _p(ws), C.c_size_t(n))
            recs = _gather(rec, group, world) if world > 1 else rec
        grad_x = torch.empty_like(gyl) if need[0] else None
        grad_r = torch.empty_like(gyl) if rr is not None and need[1] else None
        lib.call('tt_batch_norm_train_backward', C.byref(d), _p(xr), _p(rr), _p(weight), _p(bias), _p(mean), _p(invstd), _p(gyr), _p(recs),
                 _p(_rows(grad_x)[0] if grad_x is not None else None), _p(_rows(grad_r)[0] if grad_r is not None else None))
        return grad_x, grad_r, grad_w, grad_b, None, None, None, None, None, None, None, None


class _LibBatchNorm:
    """The forward shared by the three classes.  `fused_relu` (set by convert_batchnorm when the layer was followed by an nn.ReLU)
    applies the ReLU on every call, like relu=True."""

    fused_relu = False

    def _sync(self):
        """(process group, world size) of the gathers: world 1 unless torch's SyncBatchNorm would synchronize."""
        return None, 1

    def _check_config(self):
        why = config_error(self.num_features, self.affine, self.track_running_stats)
        if why is not None:
            raise lib.TTError(f'{type(self).__name__}: unsupported {why}')

    def forward(self, x, *, residual=None, relu=False):
        self._check_input_dim(x)
        factor = 0.0 if self.momentum is None else self.momentum
        if self.training:
            self.num_batches_tracked.add_(1)
            if self.momentum is None:
                factor = 1.0 / float(self.num_batches_tracked)
        group, world = self._sync() if self.training else (None, 1)
        relu = bool(relu or self.fused_relu)
        args = (x, residual, self.weight, self.bias, self.running_mean, self.running_var, self.training, relu, self.eps, factor, group,
                world)
        if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, residual, self.weight, self.bias)):
            return BatchNormFunction.apply(*args)
        _check((x, residual, self.weight, self.bias, self.running_mean, self.running_var))
        return _forward(*args)[0]

    def extra_repr(self):
        return super().extra_repr() + (', fused_relu=True' if self.fused_relu else '')


class BatchNorm1d(_LibBatchNorm, nn.BatchNorm1d):
    """nn.BatchNorm1d on the library, on (N, C) input (3-D (N, C, L) input raises TTError)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._check_config()


class BatchNorm2d(_LibBatchNorm, nn.BatchNorm2d):
    """nn.BatchNorm2d on the library; the output is channels_last."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._check_config()


class SyncBatchNorm(_LibBatchNorm, nn.SyncBatchNorm):
    """nn.SyncBatchNorm on the library, on 2-D (N, C) or 4-D input; synchronizes exactly when torch's would."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._check_config()

    def _sync(self):
        if not (dist.is_available() and dist.is_initialized()):
            return None, 1
        group = self.process_group if self.process_group else dist.group.WORLD
        world = dist.get_world_size(group)
        return (group, world) if world > 1 else (None, 1)


_SWAP = {nn.BatchNorm1d: BatchNorm1d, nn.BatchNorm2d: BatchNorm2d, nn.SyncBatchNorm: SyncBatchNorm}


def convert_batchnorm(module, fuse_relu=True, prefix=''):
    """Swap every eligible `nn.BatchNorm1d` / `nn.BatchNorm2d` / `nn.SyncBatchNorm` in `module` (itself included) for the library's
    class of the same kind, sharing its weight, bias and buffer objects (optimizer state and checkpoints are unaffected) and keeping
    its training flag and process group.  With fuse_relu, a swapped layer directly followed by an `nn.ReLU` in an `nn.Sequential` or
    a `SparseSequential` applies the ReLU itself and the ReLU becomes `nn.Identity` (the state_dict is unchanged).  Returns
    (module, skipped, fused): skipped lists (qualified name, layer, reason) for every batch norm left on torch, fused the qualified
    names of the layers that took the ReLU."""
    skipped, fused = [], []

    def swap(m, name):
        cls = _SWAP.get(type(m))
        if cls is None:
            return m
        why = config_error(m.num_features, m.affine, m.track_running_stats)
        if why is not None:
            skipped.append((name, m, why))
            return m
        kw = dict(process_group=m.process_group) if cls is SyncBatchNorm else {}
        new = cls(m.num_features, eps=m.eps, momentum=m.momentum, affine=True, track_running_stats=True, device='meta', **kw)
        new.weight, new.bias = m.weight, m.bias
        new.running_mean, new.running_var, new.num_batches_tracked = m.running_mean, m.running_var, m.num_batches_tracked
        new.train(m.training)
        return new

    from .conv2d import swap_modules
    root = swap_modules(module, prefix, swap)
    if fuse_relu:
        for name, m in root.named_modules(prefix=prefix):
            if not isinstance(m, (nn.Sequential, SparseSequential)):
                continue
            kids = list(m.named_children())
            for (bn_name, bn), (relu_name, relu) in zip(kids, kids[1:]):
                if isinstance(bn, _LibBatchNorm) and type(relu) is nn.ReLU:
                    bn.fused_relu = True
                    setattr(m, relu_name, nn.Identity())
                    fused.append(f'{name}.{bn_name}' if name else bn_name)
    return root, skipped, fused
