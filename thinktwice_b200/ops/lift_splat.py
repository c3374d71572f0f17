"""The camera branch's lift-splat with a gradient: depth softmax, outer product with the context and voxel pooling as one op.

A training fork's `_forward_single_sweep` (open_loop_training/code/model_code/backbones/lss.py:583-615) forms
`depth.softmax(1).unsqueeze(1) * img_feature.unsqueeze(2)`, a (B*N, C, D, fH, fW) fp32 tensor (514 MB per frame at thinktwice.py
shapes), makes a permuted copy of it and pools it through `voxel_pooling`; autograd then carries tensors of the same size through
the backward.  `lift_splat` returns the same (B, C, Y, X) `feature_map` through the C ABI entries `tt_lift_splat_train_forward /
_backward` (include/tt_b200.h §14), which never form that tensor: the forward keeps only the cell of every bin (4 bytes per bin)
and the backward gathers both gradients from dL/dbev along those cells, bitwise reproducibly.  SURVEY.md §8f row f4.
"""
import ctypes as C

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import lib
from ..lib import _p


def _workspace(d, device):
    n = int(lib.load().tt_lift_splat_train_workspace_bytes(C.byref(d)))
    if n == 0:                                                      # the descriptor is refused: tt_last_error names why
        raise lib.TTError(f'lift_splat: {lib.load().tt_last_error().decode()}')
    return torch.empty(n, dtype=torch.uint8, device=device), n


class LiftSplatFunction(Function):
    """forward(depth_logits (BN, D, fH, fW), context (BN, C, fH, fW), mats [BN][32], frustum_u, frustum_v, frustum_d, desc, record) ->
    (B, C, Y, X), a permuted view of the [B][Y][X][C] map.  Gradients w.r.t. the logits and the context only.  `record`: grad mode
    was on at the call (inside forward it is off, and needs_input_grad does not see torch.no_grad), so bin_cell is worth keeping."""

    @staticmethod
    def forward(ctx, depth, context, mats, fu, fv, fd, d, record):
        need = record and (ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        bev = context.new_empty(d.B, d.Y, d.X, d.C)
        bin_cell = torch.empty(d.B * d.N * d.fH * d.fW, d.D, dtype=torch.int32, device=context.device) if need else None
        ws, n = _workspace(d, context.device)
        lib.call('tt_lift_splat_train_forward', C.byref(d), _p(depth), _p(context), _p(mats), _p(fu), _p(fv), _p(fd), _p(bev), _p(bin_cell),
                 _p(ws), C.c_size_t(n))
        if need:
            ctx.save_for_backward(depth, context, bin_cell)
        ctx.d = d
        return bev.permute(0, 3, 1, 2)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_bev):
        depth, context, bin_cell = ctx.saved_tensors
        d = ctx.d
        if not (grad_bev.is_cuda and grad_bev.dtype == torch.float32):
            raise lib.TTError('lift_splat backward needs an fp32 CUDA gradient (no CPU fallback)')
        need = ctx.needs_input_grad
        grad_depth = depth.new_empty(d.B * d.N, d.D, d.fH, d.fW) if need[0] else None
        grad_context = torch.empty_like(context) if need[1] else None
        if grad_depth is not None or grad_context is not None:
            ws, n = _workspace(d, context.device)
            sb, sc, sy, sx = grad_bev.stride()
            lib.call('tt_lift_splat_train_backward', C.byref(d), _p(depth), _p(context), _p(bin_cell), _p(grad_bev), C.c_longlong(sb),
                     C.c_longlong(sc), C.c_longlong(sy), C.c_longlong(sx), _p(grad_depth), _p(grad_context), _p(ws), C.c_size_t(n))
        return grad_depth, grad_context, None, None, None, None, None, None


def lift_splat(depth, img_feature, sensor2ego, intrin, ida, frustum, voxel_coord, voxel_size, voxel_num, bda_mat=None):
    """`feature_map` of lss.py:593-615 for one sweep, (B, C, Y, X), differentiable w.r.t. `depth` and `img_feature`.

    depth       : the depth LOGITS, (B*N, D, fH, fW) fp32 CUDA, e.g. the view `depth_feature[:, :D]` (passed without a copy);
                  the softmax over D is part of the op.
    img_feature : the merged context, (B*N, C, fH, fW) fp32 CUDA.
    sensor2ego, intrin, ida : the sweep's (B, N, 4, 4) matrices (`mats_dict[...][:, sweep_index]`); their 4x4 inverses are taken
                  in fp32 on the host, as LSS.stage takes them.  No gradient flows to them.
    frustum, voxel_coord, voxel_size, voxel_num : the LSS module's buffers of those names.  The voxel index is
                  trunc((geom - (voxel_coord - voxel_size / 2)) / voxel_size) with the lower bound computed in fp32 (lss.py:630-631).
    bda_mat     : not supported (the reference's dataset never provides one).
    """
    if bda_mat is not None:
        raise ValueError('lift_splat: bda_mat is not supported')
    for name, t in (('depth', depth), ('img_feature', img_feature)):
        if not t.is_cuda:
            raise lib.TTError(f'lift_splat: {name} is not a CUDA tensor (no CPU fallback)')
        if t.dtype != torch.float32:
            raise lib.TTError(f'lift_splat: {name} is {t.dtype}, only torch.float32 is supported')
        if t.dim() != 4:
            raise ValueError(f'lift_splat: {name} must be (B*N, channels, fH, fW), got {tuple(t.shape)}')
    B, N = sensor2ego.shape[:2]
    BN, D, fH, fW = depth.shape
    Cc = img_feature.shape[1]
    if frustum.dim() != 4 or tuple(frustum.shape) != (D, fH, fW, 4):
        raise ValueError(f'lift_splat: frustum {tuple(frustum.shape)} does not match logits {tuple(depth.shape)} ((D, fH, fW, 4) expected)')
    if BN != B * N or tuple(img_feature.shape) != (BN, Cc, fH, fW):
        raise ValueError(f'lift_splat: logits {tuple(depth.shape)}, img_feature {tuple(img_feature.shape)} and {B} x {N} cameras disagree')
    for name, m in (('sensor2ego', sensor2ego), ('intrin', intrin), ('ida', ida)):
        if tuple(m.shape) != (B, N, 4, 4):
            raise ValueError(f'lift_splat: {name} {tuple(m.shape)}, expected {(B, N, 4, 4)}')
    dev = img_feature.device
    if depth.stride()[1:] != (fH * fW, fW, 1):                # a channel slice of an NCHW map passes as is
        depth = depth.contiguous()
    img_feature = img_feature.contiguous()
    h = lambda m: m.detach().to('cpu', torch.float32)
    mats = torch.stack([torch.inverse(h(ida)), h(sensor2ego).matmul(torch.inverse(h(intrin)))], 2).reshape(B * N, 32)
    fr = h(frustum)
    fu, fv, fd = fr[0, 0, :, 0], fr[0, :, 0, 1], fr[:, 0, 0, 2]
    vsize = h(voxel_size)
    lower = h(voxel_coord) - vsize / 2.0
    d = lib.LiftSplatTrainDesc()
    d.B, d.N, d.D, d.fH, d.fW, d.C = B, N, D, fH, fW, Cc
    d.depth_bstride = depth.stride(0) if BN > 0 else D * fH * fW
    d.lower, d.size = lib.f3(lower.tolist()), lib.f3(vsize.tolist())
    d.X, d.Y, d.Z = (int(v) for v in voxel_num)
    return LiftSplatFunction.apply(depth, img_feature, mats.to(dev), fu.contiguous().to(dev), fv.contiguous().to(dev),
                                   fd.contiguous().to(dev), d, torch.is_grad_enabled())
