"""Trainable sparse 3-D convolutions (spconv 2.x `SubMConv3d` / `SparseConv3d`) and mmdet3d's `SparseEncoder` on libtt_b200.

The spconv 2.x surface that mmdet3d's `SparseEncoder` / `SparseBasicBlock` use (lidarnet.py:24-58, cfg thinktwice.py:167-176):
`SparseConvTensor` (`features`, `indices`, `spatial_shape`, `batch_size`, `indice_dict`, `replace_feature()`, `dense()`),
`SparseModule`, `SparseSequential`, `SubMConv3d` and `SparseConv3d` with spconv's constructor arguments and the spconv 2.x weight
layout `(Cout, kd, kh, kw, Cin)`.  Rulebooks are built on the device (`tt_sparse_rulebook`, then `tt_sparse_pairs_ordered` for pair
lists in a fixed order); forward and backward are `tt_sparse_conv_train_forward / _backward` (include/tt_b200.h §13).  SURVEY.md §8f
row f4.  What the reference does not build (dilation, groups, bias, transposed / inverse convolutions, other kernels) is refused
when the module is constructed; CPU tensors are refused with `TTError` (no fallback).
"""
import ctypes as C
import math

import torch
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import lib
from ..lib import _p


def _t3(v):
    return tuple(int(a) for a in v) if isinstance(v, (list, tuple)) else (int(v),) * 3


def _pow2(v):
    t = 1024
    while t < v:
        t <<= 1
    return t


class SparseConvTensor:
    """spconv.pytorch.SparseConvTensor: features (N, C) fp32, indices (N, 4) int32 (b, z, y, x), spatial_shape (D, H, W)."""

    def __init__(self, features, indices, spatial_shape, batch_size, indice_dict=None):
        self._features = features
        self.indices = indices if indices.dtype == torch.int32 and indices.is_contiguous() else indices.int().contiguous()
        self.spatial_shape = [int(v) for v in spatial_shape]
        self.batch_size = int(batch_size)
        self.indice_dict = {} if indice_dict is None else indice_dict

    @property
    def features(self):
        return self._features

    @features.setter
    def features(self, value):
        self._features = value

    def replace_feature(self, feature):
        """a tensor with the same sites, rulebooks and shape and new features (spconv 2.x)."""
        return SparseConvTensor(feature, self.indices, self.spatial_shape, self.batch_size, self.indice_dict)

    def find_indice_pair(self, key):
        return self.indice_dict.get(key) if key is not None else None

    def dense(self, channels_first=True):
        """(N, C, D, H, W) (or (N, D, H, W, C)), zero at empty sites; differentiable with respect to the features."""
        D, H, W = self.spatial_shape
        Cf = self.features.shape[1]
        i = self.indices.long()
        flat = ((i[:, 0] * D + i[:, 1]) * H + i[:, 2]) * W + i[:, 3]
        out = self.features.new_zeros(self.batch_size * D * H * W, Cf).index_copy(0, flat, self.features)
        out = out.view(self.batch_size, D, H, W, Cf)
        return out.permute(0, 4, 1, 2, 3).contiguous() if channels_first else out


class SparseModule(nn.Module):
    """Marks modules that take a SparseConvTensor (spconv.pytorch.SparseModule)."""


class SparseSequential(SparseModule):
    """spconv.pytorch.SparseSequential: a SparseModule gets the SparseConvTensor, any other module (BatchNorm1d, ReLU, ...) its
    `.features` (skipped when there are no sites, as in spconv)."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        if len(args) == 1 and isinstance(args[0], dict):
            for name, module in args[0].items():
                self.add_module(name, module)
        else:
            for idx, module in enumerate(args):
                self.add_module(str(idx), module)
        for name, module in kwargs.items():
            self.add_module(name, module)

    def __len__(self):
        return len(self._modules)

    def __getitem__(self, idx):
        return list(self._modules.values())[idx]

    def __iter__(self):
        return iter(self._modules.values())

    def forward(self, input):
        for module in self._modules.values():
            if isinstance(module, SparseModule):
                input = module(input)
            elif isinstance(input, SparseConvTensor):
                if input.indices.shape[0] != 0:
                    input = input.replace_feature(module(input.features))
            else:
                input = module(input)
        return input


class Rulebook:
    """the pairs of one convolution: out_indices / n_out, the device row counts, and tap-major pair lists in ascending output row."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _out_shape(in_shape, k, s, p, subm):
    return list(in_shape) if subm else [(in_shape[a] + 2 * p[a] - k[a]) // s[a] + 1 for a in range(3)]


def build_rulebook(indices, batch_size, in_shape, k, s, p, subm):
    """tt_sparse_rulebook (neighbour table) + tt_sparse_pairs_ordered.  A strided conv reads its output site count on the host once,
    to size its output (spconv synchronises there too); a SubM conv does not synchronise."""
    dev = indices.device
    n_in = int(indices.shape[0])
    kvol = k[0] * k[1] * k[2]
    out_shape = _out_shape(in_shape, k, s, p, subm)
    in_count = torch.full((1,), n_in, dtype=torch.int32, device=dev)
    if n_in == 0:
        return Rulebook(out_indices=indices.new_zeros((0, 4)), out_shape=out_shape, n_in=0, n_out=0, in_count=in_count, out_count=in_count,
                        pairs_in=None, pairs_out=None, pair_count=None, pair_cap=1, kvol=kvol)
    reach = math.prod(-(-k[a] // s[a]) for a in range(3))                 # output sites one input site can reach
    cap_out = n_in if subm else min(n_in * reach, batch_size * math.prod(out_shape))
    d = lib.RulebookDesc()
    d.B = batch_size
    d.in_shape, d.out_shape, d.k, d.s, d.p = lib.i3(in_shape), lib.i3(out_shape), lib.i3(k), lib.i3(s), lib.i3(p)
    d.subm, d.cap_in, d.cap_out = int(subm), n_in, cap_out
    d.table_size = _pow2(2 * max(n_in, cap_out))
    L = lib.load()
    ws = torch.empty(max(int(L.tt_rulebook_workspace_bytes(C.byref(d))), 1), dtype=torch.uint8, device=dev)
    out_coords = torch.empty((cap_out, 4), dtype=torch.int32, device=dev)
    out_count = torch.empty((1,), dtype=torch.int32, device=dev)
    nbr = torch.empty((cap_out, kvol), dtype=torch.int32, device=dev)
    lib.call('tt_sparse_rulebook', C.byref(d), _p(indices), _p(in_count), _p(out_coords), _p(out_count), _p(nbr), _p(None), _p(None),
             _p(None), _p(ws))
    n_out = n_in if subm else int(out_count.item())
    pair_cap = max(1, min(n_in, n_out))
    pin = torch.empty((kvol, pair_cap), dtype=torch.int32, device=dev)
    pout = torch.empty((kvol, pair_cap), dtype=torch.int32, device=dev)
    pcount = torch.empty((kvol,), dtype=torch.int32, device=dev)
    nb = int(L.tt_sparse_pairs_ordered_workspace_bytes(cap_out, kvol))
    ws2 = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
    lib.call('tt_sparse_pairs_ordered', _p(nbr), _p(out_count), cap_out, kvol, pair_cap, _p(pin), _p(pout), _p(pcount), _p(ws2), C.c_size_t(nb))
    return Rulebook(out_indices=out_coords[:n_out], out_shape=out_shape, n_in=n_in, n_out=n_out, in_count=in_count, out_count=out_count,
                    pairs_in=pin, pairs_out=pout, pair_count=pcount, pair_cap=pair_cap, kvol=kvol)


def conv_desc(Cin, Cout, kernel_size, stride, padding, dilation=1, groups=1, bias=False, subm=False, transposed=False, inverse=False,
              n_in=0, n_out=0, pair_cap=1):
    d = lib.SparseConvTrainDesc()
    k = _t3(kernel_size)
    d.Cin, d.Cout, d.kvol = Cin, Cout, k[0] * k[1] * k[2]
    d.cap_in, d.cap_out, d.pair_cap, d.in_ld, d.out_ld = n_in, n_out, pair_cap, Cin, Cout
    d.k, d.stride, d.padding, d.dilation = lib.i3(k), lib.i3(_t3(stride)), lib.i3(_t3(padding)), lib.i3(_t3(dilation))
    d.subm, d.groups, d.bias, d.transposed, d.inverse = int(subm), groups, int(bool(bias)), int(transposed), int(inverse)
    return d


def workspace_bytes(d):
    """the library's workspace for `d`; raises TTError naming the parameter when the library refuses the convolution."""
    n = int(lib.load().tt_sparse_conv_train_workspace_bytes(C.byref(d)))
    if n == 0:
        raise lib.TTError(f'sparse convolution refused: {lib.load().tt_last_error().decode()}')
    return n


def _check_tensor(t, what):
    if not t.is_cuda:
        raise lib.TTError(f'sparse convolution: {what} must be a CUDA tensor (no CPU fallback)')
    if t.dtype != torch.float32:
        raise lib.TTError(f'sparse convolution: {what} must be float32, got {t.dtype}')


class SparseConvFunction(Function):
    """features (n_in, Cin), weight (Cout, kd, kh, kw, Cin) -> features (n_out, Cout) over the pairs of `rb`."""

    @staticmethod
    def forward(ctx, features, weight, rb, geom):
        _check_tensor(features, 'features')
        _check_tensor(weight, 'weight')
        features, weight = features.contiguous(), weight.contiguous()
        Cout, Cin = weight.shape[0], weight.shape[-1]
        ctx.rb, ctx.geom = rb, geom
        ctx.save_for_backward(features, weight)
        if rb.n_in == 0 or rb.n_out == 0:
            return features.new_zeros((rb.n_out, Cout))
        d = conv_desc(Cin, Cout, **geom, n_in=rb.n_in, n_out=rb.n_out, pair_cap=rb.pair_cap)
        n = workspace_bytes(d)
        ws = torch.empty(n, dtype=torch.uint8, device=features.device)
        out = features.new_empty((rb.n_out, Cout))
        lib.call('tt_sparse_conv_train_forward', C.byref(d), _p(features), _p(weight), _p(rb.pairs_in), _p(rb.pairs_out), _p(rb.pair_count),
                 _p(rb.out_count), _p(out), _p(ws), C.c_size_t(n))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        features, weight = ctx.saved_tensors
        rb = ctx.rb
        need = ctx.needs_input_grad
        if rb.n_in == 0 or rb.n_out == 0:
            return (torch.zeros_like(features) if need[0] else None, torch.zeros_like(weight) if need[1] else None, None, None)
        grad_in = torch.empty_like(features) if need[0] else None
        grad_w = torch.empty_like(weight) if need[1] else None
        if grad_in is None and grad_w is None:
            return None, None, None, None
        Cout, Cin = weight.shape[0], weight.shape[-1]
        d = conv_desc(Cin, Cout, **ctx.geom, n_in=rb.n_in, n_out=rb.n_out, pair_cap=rb.pair_cap)
        n = workspace_bytes(d)
        ws = torch.empty(n, dtype=torch.uint8, device=features.device)
        grad_out = grad_out.contiguous()
        lib.call('tt_sparse_conv_train_backward', C.byref(d), _p(features), _p(weight), _p(grad_out), _p(rb.pairs_in), _p(rb.pairs_out),
                 _p(rb.pair_count), _p(rb.in_count), _p(rb.out_count), _p(grad_in), _p(grad_w), _p(ws), C.c_size_t(n))
        return grad_in, grad_w, None, None


class SparseConvolution(SparseModule):
    """spconv 2.x SparseConvolution (3-D): parameter `weight` (Cout, kd, kh, kw, Cin)."""

    def __init__(self, ndim, in_channels, out_channels, kernel_size=3, stride=1, padding=0, dilation=1, groups=1, bias=True, subm=False,
                 output_padding=0, transposed=False, inverse=False, indice_key=None, algo=None, fp32_accum=None, name=None):
        super().__init__()
        assert ndim == 3, 'only 3-D sparse convolutions are provided'
        self.ndim, self.in_channels, self.out_channels = ndim, in_channels, out_channels
        self.kernel_size, self.stride, self.padding, self.dilation = _t3(kernel_size), _t3(stride), _t3(padding), _t3(dilation)
        self.output_padding = _t3(output_padding)
        self.groups, self.subm, self.transposed, self.inverse, self.indice_key = groups, subm, transposed, inverse, indice_key
        self.algo, self.fp32_accum, self.name = algo, fp32_accum, name
        self.geom = dict(kernel_size=self.kernel_size, stride=self.stride, padding=self.padding, dilation=self.dilation, groups=groups,
                         bias=bias, subm=subm, transposed=transposed, inverse=inverse)
        workspace_bytes(conv_desc(in_channels, out_channels, **self.geom))     # refuse what the library does not run, here
        self.weight = nn.Parameter(torch.empty(out_channels, *self.kernel_size, in_channels))
        self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight.view(self.out_channels, -1), a=math.sqrt(5))

    def forward(self, input):
        if not isinstance(input, SparseConvTensor):
            raise TypeError('sparse convolutions take a SparseConvTensor')
        _check_tensor(input.features, 'features')
        if not input.indices.is_cuda:
            raise lib.TTError('sparse convolution: indices must be a CUDA tensor (no CPU fallback)')
        if input.features.shape[1] != self.in_channels:
            raise lib.TTError(f'sparse convolution: {input.features.shape[1]} input channels, expected {self.in_channels}')
        rb = input.find_indice_pair(self.indice_key) if self.subm else None
        if rb is None:
            rb = build_rulebook(input.indices, input.batch_size, input.spatial_shape, self.kernel_size, self.stride, self.padding, self.subm)
            if self.indice_key is not None:
                input.indice_dict[self.indice_key] = rb
        out = SparseConvFunction.apply(input.features, self.weight, rb, self.geom)
        return SparseConvTensor(out, rb.out_indices, rb.out_shape, input.batch_size, input.indice_dict)


class SubMConv3d(SparseConvolution):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True, indice_key=None,
                 algo=None, fp32_accum=None, name=None):
        super().__init__(3, in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias, True, indice_key=indice_key,
                         algo=algo, fp32_accum=fp32_accum, name=name)


class SparseConv3d(SparseConvolution):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True, indice_key=None,
                 algo=None, fp32_accum=None, name=None):
        super().__init__(3, in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias, indice_key=indice_key,
                         algo=algo, fp32_accum=fp32_accum, name=name)


class SparseConvTranspose3d(SparseConvolution):
    """spconv's transposed convolution: the reference does not build it, so construction is refused (TTError)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True, indice_key=None,
                 algo=None, fp32_accum=None, name=None):
        super().__init__(3, in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias, transposed=True,
                         indice_key=indice_key, algo=algo, fp32_accum=fp32_accum, name=name)


class SparseInverseConv3d(SparseConvolution):
    """spconv's inverse convolution: the reference does not build it, so construction is refused (TTError)."""

    def __init__(self, in_channels, out_channels, kernel_size, indice_key=None, bias=True, algo=None, fp32_accum=None, name=None):
        super().__init__(3, in_channels, out_channels, kernel_size, bias=bias, inverse=True, indice_key=indice_key, algo=algo,
                         fp32_accum=fp32_accum, name=name)


def _bn(c):
    return nn.BatchNorm1d(c, eps=1e-3, momentum=0.01)


class SparseBasicBlock(SparseModule):
    """mmdet3d SparseBasicBlock: conv1 / bn1 / relu / conv2 / bn2, + identity, relu (SubM 3x3x3, padding 1, no bias)."""

    def __init__(self, inplanes, planes, indice_key=None):
        super().__init__()
        self.conv1 = SubMConv3d(inplanes, planes, 3, padding=1, bias=False, indice_key=indice_key)
        self.bn1 = _bn(planes)
        self.conv2 = SubMConv3d(planes, planes, 3, padding=1, bias=False, indice_key=indice_key)
        self.bn2 = _bn(planes)
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        identity = x.features
        out = self.conv1(x)
        out = out.replace_feature(self.relu(self.bn1(out.features)))
        out = self.conv2(out)
        return out.replace_feature(self.relu(self.bn2(out.features) + identity))


class SparseEncoder(nn.Module):
    """mmdet3d SparseEncoder(block_type='basicblock', order=('conv', 'norm', 'act')), trainable; forward = lidarnet.py:28-58.
    BatchNorm1d(eps 1e-3, momentum 0.01) after every convolution; SubM convs of one resolution share a rulebook (indice_key)."""

    def __init__(self, in_channels, sparse_shape, output_channels=128, order=('conv', 'norm', 'act'), norm_cfg=None, base_channels=16,
                 encoder_channels=((16,), (32, 32, 32), (64, 64, 64), (64, 64, 64)), encoder_paddings=((1,), (1, 1, 1), (1, 1, 1),
                 ((0, 1, 1), 1, 1)), block_type='basicblock'):
        super().__init__()
        assert block_type == 'basicblock' and tuple(order) == ('conv', 'norm', 'act')
        self.sparse_shape = list(sparse_shape)
        self.in_channels, self.output_channels, self.base_channels = in_channels, output_channels, base_channels
        self.encoder_channels, self.encoder_paddings = encoder_channels, encoder_paddings
        self.conv_input = SparseSequential(SubMConv3d(in_channels, base_channels, 3, padding=1, bias=False, indice_key='subm1'),
                                           _bn(base_channels), nn.ReLU(inplace=True))
        self.encoder_layers = SparseSequential()
        cin = base_channels
        for i, blocks in enumerate(encoder_channels):
            stage = []
            for j, cout in enumerate(blocks):
                if j == len(blocks) - 1 and i != len(encoder_channels) - 1:
                    stage.append(SparseSequential(SparseConv3d(cin, cout, 3, stride=2, padding=encoder_paddings[i][j], bias=False,
                                                               indice_key=f'spconv{i + 1}'), _bn(cout), nn.ReLU(inplace=True)))
                else:
                    stage.append(SparseBasicBlock(cout, cout, indice_key=f'subm{i + 1}'))
                cin = cout
            self.encoder_layers.add_module(f'encoder_layer{i + 1}', SparseSequential(*stage))
        self.conv_out = SparseSequential(SparseConv3d(cin, output_channels, (3, 1, 1), stride=(2, 1, 1), padding=0, bias=False,
                                                      indice_key='spconv_down2'), _bn(output_channels), nn.ReLU(inplace=True))

    def forward(self, voxel_features, coors, batch_size):
        """voxel_features (N, in_channels) fp32, coors (N, 4) (b, z, y, x) on the device -> the (B, C * D, H, W) BEV map."""
        x = SparseConvTensor(voxel_features, coors.int(), self.sparse_shape, batch_size)
        x = self.conv_input(x)
        for stage in self.encoder_layers:
            x = stage(x)
        d = self.conv_out(x).dense()
        N, Cd, D, H, W = d.shape
        return d.view(N, Cd * D, H, W)
