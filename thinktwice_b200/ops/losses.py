"""The reference's training losses with gradients: the camera branch's seg / depth supervision and `ThinkTwiceDecoder.loss`.

A training fork's `forward_train` (open_loop_training/code/encoder_decoder_framework.py:147-191) computes its losses with torch ops.
For the camera half that is the largest memory consumer left on the step: `F.cross_entropy` keeps a log-softmax of the (B*N, 12,
224, 448) logits for its backward, and the depth target is a one-hot of every foreground cell.  For the decoder half it is about
twenty terms of a few small ops each, forward and backward.

  * `camera_losses(model, batch, cam_feat)` replaces framework:171-190.  One `tt_camera_loss_train_forward` launch reads the NCHW
    logits in place and keeps one byte per logit pixel (its class or bin); one `tt_camera_loss_train_backward` launch writes both
    logit gradients from those bytes (include/tt_b200.h §15).
  * `decoder_loss(decoder, batch, pred, mid_BEV_feature)` replaces `self.decoder.loss(batch, pred, mid_BEV_feature)`.  The values
    come from one `tt_loss_reduce` launch, the gradients of every prediction from one `tt_loss_backward` launch (§10, §10b); the
    predictions are read in place through their strides.

SURVEY.md §8f row f4.
"""
import ctypes as C
from collections import OrderedDict

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import lib
from ..lib import _p

_STATS_BYTES = C.sizeof(lib.CameraLossStats)
SPLIT_ELEMENTS = 1 << 18


def _need_cuda_fp32(name, t):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise lib.TTError(f'{name} is not a CUDA tensor (no CPU fallback)')
    if t.dtype != torch.float32:
        raise lib.TTError(f'{name} is {t.dtype}, only torch.float32 is supported')


def _cfg(config, key):
    return getattr(config, key) if hasattr(config, key) else config[key]


# ------------------------------------------------------------------------------------------------------------ camera supervision
class CameraLossFunction(Function):
    """forward(seg (BN, C, h, w) or None, depth (BN, D, h', w') or None, seg_gt, depth_gt, fields, record) -> (seg_loss, depth_loss),
    0-d views of one (2,) result (a half that is off gives an undefined value, not returned by camera_losses).  `record`: grad mode
    was on at the call, so the per-pixel targets are worth keeping."""

    @staticmethod
    def forward(ctx, seg, depth, seg_gt, depth_gt, fields, record):
        ref = seg if seg is not None else depth
        d = lib.CameraLossTrainDesc()
        for k, v in fields.items():
            setattr(d, k, v)
        d.seg_logits, d.seg_gt, d.depth_logits, d.depth_gt = _p(seg), _p(seg_gt), _p(depth), _p(depth_gt)
        if seg is not None:
            d.seg_stride = (C.c_longlong * 4)(*seg.stride())
        if depth is not None:
            d.depth_stride = (C.c_longlong * 4)(*depth.stride())
        dev = ref.device
        out = torch.empty(2, device=dev)
        stats = torch.empty(_STATS_BYTES, dtype=torch.uint8, device=dev)
        keep = record and any(ctx.needs_input_grad[:2])
        st = torch.empty(d.BN, d.seg_h, d.seg_w, dtype=torch.uint8, device=dev) if keep and seg is not None else None
        dt = torch.empty(d.BN, d.depth_h, d.depth_w, dtype=torch.uint8, device=dev) if keep and depth is not None else None
        if d.BN == 0:                                               # torch's values: a mean over no pixel, a sum over no cell
            out.copy_(torch.tensor([float('nan'), 0.0]))
        else:
            n = int(lib.load().tt_camera_loss_train_workspace_bytes(C.byref(d)))
            ws = torch.empty(n, dtype=torch.uint8, device=dev)
            lib.call('tt_camera_loss_train_forward', C.byref(d), _p(out), _p(stats), _p(st), _p(dt), _p(ws), C.c_size_t(n))
        if keep:
            ctx.save_for_backward(seg, depth, stats, st, dt)
        ctx.d = d
        return out[0], out[1]

    @staticmethod
    @once_differentiable
    def backward(ctx, g_seg, g_depth):
        seg, depth, stats, st, dt = ctx.saved_tensors
        need = ctx.needs_input_grad
        grad_seg = torch.empty(seg.shape, device=seg.device) if need[0] and seg is not None else None
        grad_depth = torch.empty(depth.shape, device=depth.device) if need[1] and depth is not None else None
        if (grad_seg is None and grad_depth is None) or ctx.d.BN == 0:
            return None, None, None, None, None, None
        ref = seg if seg is not None else depth
        zero = torch.zeros((), device=ref.device)
        for g in (g_seg, g_depth):
            if g is not None and not (g.is_cuda and g.dtype == torch.float32):
                raise lib.TTError('camera_losses backward needs fp32 CUDA gradients (no CPU fallback)')
        up = torch.stack([g_seg if g_seg is not None else zero, g_depth if g_depth is not None else zero])
        lib.call('tt_camera_loss_train_backward', C.byref(ctx.d), _p(stats), _p(st), _p(dt), _p(up), _p(grad_seg), _p(grad_depth))
        return grad_seg, grad_depth, None, None, None, None


def _check_seg_labels(lab, classes, ignore):
    """the labels the loss reads (nearest-resized) against CrossEntropyLoss's bounds: ValueError where torch raises."""
    if not bool(torch.isfinite(lab).all()):
        raise ValueError('seg: a label the loss reads is not finite')
    t = lab.trunc()
    if not bool((((t >= 0) & (t < classes)) | (t == ignore)).all()):
        raise ValueError(f'seg: labels must truncate into [0, {classes}) or to {ignore} (ignored)')


def camera_losses(model, batch, cam_feat):
    """framework:171-190 with a gradient: an OrderedDict of the enabled terms in the reference's order, 'seg_loss' (use_seg; seg_loss
    * 10) and 'depth_loss' (use_depth), 0-d fp32 tensors differentiable w.r.t. cam_feat['seg'] and cam_feat['depth'].

    model    : the reference's EncoderDecoder (or anything with its attributes): use_seg, use_depth, downsample_factor,
               seg_downsample_factor, dbound, depth_channels and seg_loss_func.{alpha, gamma, ignore_index}.
    batch    : batch['seg'] / batch['depth'], (B, N, H, W) full-resolution labels / depths (any device and float dtype).
    cam_feat : cam_feat['seg'] (B*N, C, H / s, W / s) and cam_feat['depth'] (B*N, depth_channels, H / f, W / f) logits, fp32 CUDA;
               the plane must be dense, any batch / channel stride passes without a copy (the view depth_feature[:, :D])."""
    use_seg, use_depth = bool(getattr(model, 'use_seg', False)), bool(getattr(model, 'use_depth', False))
    if not (use_seg or use_depth):
        return OrderedDict()
    seg = cam_feat['seg'] if use_seg else None
    depth = cam_feat['depth'] if use_depth else None
    f = dict()
    dev = None
    for name, t, key in (('seg', seg, 'seg'), ('depth', depth, 'depth')):
        if t is None:
            continue
        _need_cuda_fp32(f"cam_feat['{name}']", t)
        dev = t.device
        if t.dim() != 4:
            raise ValueError(f"cam_feat['{name}'] must be (B*N, channels, h, w), got {tuple(t.shape)}")
        if key not in batch:
            raise ValueError(f"{name}_loss needs batch['{key}']")
        if batch[key].dim() != 4:
            raise ValueError(f"batch['{key}'] must be (B, N, H, W), got {tuple(batch[key].shape)}")
    BN = (seg if seg is not None else depth).shape[0]
    f['BN'] = BN
    seg_gt = depth_gt = None
    if seg is not None:
        gt = batch['seg']
        s = int(model.seg_downsample_factor)
        B, N, H, W = gt.shape
        _, Cs, h, w = seg.shape
        if B * N != BN or H // s != h or W // s != w:
            raise ValueError(f"seg: logits {tuple(seg.shape)} do not match labels {tuple(gt.shape)} at downsample factor {s}")
        loss_fn = model.seg_loss_func
        if getattr(loss_fn, 'weight', None) is not None:
            raise ValueError('seg: a class-weighted FocalLoss is not supported')
        seg_gt = gt.to(dev, torch.float32).reshape(BN, H, W).contiguous()
        if BN:
            _check_seg_labels(torch.nn.functional.interpolate(seg_gt[:, None], size=(h, w), mode='nearest'), Cs,
                              int(loss_fn.ignore_index))
        f.update(seg_h=h, seg_w=w, seg_H=H, seg_W=W, seg_classes=Cs, seg_ignore=int(loss_fn.ignore_index),
                 seg_alpha=float(loss_fn.alpha), seg_gamma=float(loss_fn.gamma), seg_weight=10.0)
    if depth is not None:
        gt = batch['depth']
        fd = int(model.downsample_factor)
        D = int(model.depth_channels)
        B, N, H, W = gt.shape
        _, Dd, h, w = depth.shape
        if Dd != D or B * N != BN or (H, W) != (h * fd, w * fd):
            raise ValueError(f'depth: logits {tuple(depth.shape)} do not match depths {tuple(gt.shape)} with {D} bins and '
                             f'{fd}x{fd} blocks')
        depth_gt = gt.to(dev, torch.float32).reshape(BN, H, W).contiguous()
        d0, _, step = (float(v) for v in model.dbound)
        f.update(depth_h=h, depth_w=w, depth_factor=fd, depth_bins=D, depth_offset=d0 - step, depth_step=step)
    vals = CameraLossFunction.apply(seg, depth, seg_gt, depth_gt, f, torch.is_grad_enabled())
    d = OrderedDict()
    if use_seg:
        d['seg_loss'] = vals[0]
    if use_depth:
        d['depth_loss'] = vals[1]
    return d


# ------------------------------------------------------------------------------------------------------------ the decoder's terms
class DecoderLossFunction(Function):
    """forward(plan, *inputs) -> one tensor per key of plan['keys'] (0-d, value_loss (B, 1)), views of one result vector.
    plan['terms']: the tt_loss_term dicts, each with 'grad' = (input index, index into that input) or None; plan['grads']: per term,
    None or (up_slot, up_count).  The inputs are the prediction tensors the terms read."""

    @staticmethod
    def forward(ctx, plan, *inputs):
        terms = plan['terms']
        n_slots = plan['n_slots']
        dev = inputs[0].device
        out = torch.empty(n_slots, device=dev)
        n = int(lib.load().tt_loss_workspace_bytes(len(terms)))
        ws = torch.empty(n, dtype=torch.uint8, device=dev)
        lib.call('tt_loss_reduce', lib.pack_loss_terms(terms), len(terms), _p(out), n_slots, _p(ws), C.c_size_t(n))
        ctx.plan = plan
        ctx.save_for_backward(*inputs)
        outs = [out[s0:s0 + c].view(c, 1) if shape == 'column' else out[s0] for _, s0, c, shape in plan['keys']]
        ctx.mark_non_differentiable(*[o for o, (name, *_) in zip(outs, plan['keys']) if name in plan['detached']])
        return tuple(outs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        inputs = ctx.saved_tensors
        plan = ctx.plan
        need = ctx.needs_input_grad[1:]
        if not any(need):
            return (None,) * (1 + len(inputs))
        dev = inputs[0].device
        parts = []
        for g, (_, s0, c, _) in zip(grads, plan['keys']):
            if g is None:
                parts.append(torch.zeros(c, device=dev))
            else:
                parts.append(g.reshape(c))
        grad_out = torch.cat(parts)
        if grad_out.dtype != torch.float32:
            raise lib.TTError(f'decoder_loss backward needs fp32 gradients, got {grad_out.dtype}')
        gin = [torch.empty(t.shape, device=dev) if need[j] or j in plan['paired'] else None for j, t in enumerate(inputs)]
        gl = []
        for t in plan['terms']:
            spec = t['grad']
            if spec is None or gin[spec[0]] is None:
                gl.append(dict(grad_pred=_p(None), grad_pred2=_p(None), grad_stride=[0] * len(t['shape']), up_slot=0, up_count=1))
                continue
            j, idx, j2, up_slot, up_count = spec
            gv = gin[j][idx]
            gl.append(dict(grad_pred=_p(gv), grad_pred2=_p(gin[j2][idx]) if j2 is not None else _p(None), grad_stride=list(gv.stride()),
                           up_slot=up_slot, up_count=up_count))
        n = int(lib.load().tt_loss_backward_workspace_bytes(len(gl)))
        ws = torch.empty(n, dtype=torch.uint8, device=dev)
        lib.call('tt_loss_backward', lib.pack_loss_terms(plan['terms']), len(gl), lib.pack_loss_grads(gl), _p(grad_out),
                 plan['n_slots'], _p(ws), C.c_size_t(n))
        return (None,) + tuple(g if need[j] else None for j, g in enumerate(gin))


def _beta_ok(*ts):
    return bool(torch.stack([(torch.isfinite(t) & (t > 0)).all() for t in ts]).all())


def decoder_loss(decoder, batch, pred, mid_BEV_feature):
    """ThinkTwiceDecoder.loss (thinktwice_decoder.py:535-620) with gradients: the reference's dict, same keys, order and shapes
    (value_loss (B, 1), every other entry 0-d), differentiable w.r.t. every prediction the reference's loss differentiates.  The four
    open-loop offsets are detached, as the reference's no_grad block leaves them.

    decoder : the reference's ThinkTwiceDecoder (or anything with action_loss_weight, wp_loss_weight, distil_index,
              distil_kl_loss_weight_dict and config.{value_weight, features_weight}).
    pred    : the reference's teacher-forced `pred` dict, fp32 CUDA tensors (any strides: they are read in place).
    mid_BEV_feature : the fusion's pyramid list; entries distil_index are supervised."""
    keys_in = ('mu_branches', 'sigma_branches', 'pred_speed', 'pred_value_traj', 'pred_value_ctrl', 'pred_features_traj',
               'pred_features_ctrl', 'future_mu', 'future_sigma', 'pred_wp', 'refine_BEV_feature', 'refine_flattned_BEV_feature',
               'teacher_pred_wp_offset', 'teacher_pred_ctrl_offset_lis', 'teacher_future_BEV_feature', 'teacher_refine_BEV_feature',
               'teacher_refine_flattned_BEV_feature')
    P = {k: pred[k] for k in keys_in}
    distil = list(decoder.distil_index)
    for i in distil:
        P[f'mid{i}'] = mid_BEV_feature[i]
    for k, t in P.items():
        _need_cuda_fp32(f'pred[{k!r}]' if not k.startswith('mid') else f'mid_BEV_feature[{k[3:]}]', t)
    for a, b in (('mu_branches', 'sigma_branches'), ('future_mu', 'future_sigma')):   # pred2 is read with pred's strides
        if P[a].shape != P[b].shape:
            raise ValueError(f'pred[{a!r}] {tuple(P[a].shape)} and pred[{b!r}] {tuple(P[b].shape)} differ')
        if P[a].stride() != P[b].stride():
            P[a], P[b] = P[a].contiguous(), P[b].contiguous()
    dev = P['mu_branches'].device
    names = list(P)
    inputs = [P[k] for k in names]
    col = {k: j for j, k in enumerate(names)}
    g32 = lambda t: t.to(dev, torch.float32).contiguous()
    B = P['pred_speed'].shape[0]
    gt_speed = g32(batch['speed']).view(-1, 1) / 12.
    gt_value = g32(batch['value']).view(-1, 1)
    gt_feat = g32(batch['feature'])
    gt_wp = g32(batch['waypoints'])
    a_mu, a_sigma = g32(batch['action_mu']), g32(batch['action_sigma'])
    f_mu = torch.stack([g32(t) for t in batch['future_action_mu'][:-1]], 1).unsqueeze(1)
    f_sigma = torch.stack([g32(t) for t in batch['future_action_sigma'][:-1]], 1).unsqueeze(1)
    if not _beta_ok(a_mu, a_sigma, f_mu, f_sigma, P['mu_branches'].detach(), P['sigma_branches'].detach(), P['future_mu'].detach(),
                    P['future_sigma'].detach()):
        raise ValueError('Beta parameters (action_mu / action_sigma, future_action_mu / future_action_sigma and the predicted '
                         'mu / sigma) must be finite and > 0')
    cfg = decoder.config
    fw, vw = float(_cfg(cfg, 'features_weight')), float(_cfg(cfg, 'value_weight'))
    aw, ww = float(decoder.action_loss_weight), float(decoder.wp_loss_weight)
    dw = decoder.distil_kl_loss_weight_dict
    terms, keys, detached = [], [], set()
    paired, hold = set(), []                                        # hold: the ground-truth tensors the terms point at

    def key(name, count=1, shape='scalar'):
        s0 = sum(c for _, _, c, _ in keys)
        keys.append((name, s0, count, shape))
        return s0

    def term(kind, slot, scale, name, idx=(), pred2=None, gt=None, gt2=None, aux=0, grad=None):
        """pred = P[name][idx]; pred2 = P[pred2][idx]; gt / gt2 broadcast to pred's shape; grad = (up_slot, up_count) or None"""
        p = P[name][idx]
        shape = list(p.shape) or [1]
        gt_v = None
        if gt is not None:
            try:
                gt_v = gt.expand(p.shape)
            except RuntimeError:
                raise ValueError(f'{name}: ground truth {tuple(gt.shape)} does not broadcast to the prediction {tuple(p.shape)}') from None
        gt2_v = gt2.expand(p.shape) if gt2 is not None else None
        hold.extend((gt_v, gt2_v))
        if gt2_v is not None and gt2_v.stride() != gt_v.stride():
            raise ValueError(f'{name}: the two Beta targets differ in layout')
        if grad is not None and idx == () and p.dim() > 1 and p.numel() > SPLIT_ELEMENTS:
            # tt_loss_reduce gives every term the same CTA count: a large term goes in as one term per leading index (same slot)
            for b in range(p.shape[0]):
                term(kind, slot, scale, name, (b,), pred2, None if gt_v is None else gt_v[b], None if gt2_v is None else gt2_v[b], aux, grad)
            return
        flat = lambda st: list(st) or [1]
        spec = None
        if grad is not None:
            j2 = col[pred2] if pred2 is not None else None
            if j2 is not None:
                paired.update((col[name], j2))
            spec = (col[name], idx, j2, grad[0], grad[1])
        terms.append(dict(kind=kind, slot=slot, scale=scale, shape=shape, aux=aux, pred=_p(p), pred_stride=flat(p.stride()),
                          pred2=_p(P[pred2][idx]) if pred2 is not None else _p(None), gt=_p(gt_v), gt2=_p(gt2_v),
                          gt_stride=flat(gt_v.stride()) if gt_v is not None else [0] * len(shape), grad=spec))

    L1, SL1, CLAMP, KL, ACT = lib.LOSS_L1, lib.LOSS_SMOOTH_L1, lib.LOSS_SMOOTH_L1_CLAMP, lib.LOSS_BETA_KL, lib.LOSS_ACTION_L1
    mu, wp = P['mu_branches'], P['pred_wp']
    for c, name in enumerate(('current_throttle_brake_offset', 'current_steer_offset')):
        s = key(name)
        detached.add(name)
        term(ACT, s, 1.0 / B, 'mu_branches', (slice(None), -1, c), pred2='sigma_branches', gt=a_mu[:, c], gt2=a_sigma[:, c], aux=c)
    for c, name in enumerate(('longitudinal_offset', 'lateral_offset')):
        s = key(name)
        detached.add(name)
        term(L1, s, 1.0 / (B * wp.shape[2]), 'pred_wp', (slice(None), -1, slice(None), c), gt=gt_wp[:, :, c])
    s = key('action_loss')
    term(KL, s, aw / mu.numel(), 'mu_branches', pred2='sigma_branches', gt=a_mu.unsqueeze(1), gt2=a_sigma.unsqueeze(1), grad=(s, 1))
    s = key('speed_loss')
    term(SL1, s, 1.0 / P['pred_speed'].numel(), 'pred_speed', gt=gt_speed, grad=(s, 1))
    v0 = key('value_loss', B, 'column')                             # (B, 1): mean_b sl1(v_traj) + sl1(v_ctrl)[b], one slot per frame
    vt, vc = P['pred_value_traj'], P['pred_value_ctrl']
    if vc.numel() != B:
        raise ValueError(f"pred['pred_value_ctrl'] {tuple(vc.shape)}: one value per frame expected")
    for b in range(B):
        term(SL1, v0 + b, vw / vt.numel(), 'pred_value_traj', gt=gt_value, grad=(v0, B) if b == 0 else None)
        term(SL1, v0 + b, vw, 'pred_value_ctrl', (slice(b, b + 1),), gt=gt_value[b:b + 1], grad=(v0 + b, 1))
    s = key('flattened_feature_loss')
    for k in ('pred_features_traj', 'pred_features_ctrl'):
        term(SL1, s, fw / P[k].numel(), k, gt=gt_feat, grad=(s, 1))
    s = key('future_action_loss')
    term(KL, s, aw * 0.25 / P['future_mu'].numel(), 'future_mu', pred2='future_sigma', gt=f_mu, gt2=f_sigma, grad=(s, 1))
    s = key('wp_loss')
    term(SL1, s, ww / wp.numel(), 'pred_wp', gt=gt_wp.unsqueeze(1), grad=(s, 1))
    for i in distil:
        s = key(f'BEV_feature_loss{i}')
        term(CLAMP, s, float(dw[i]) / P[f'mid{i}'].numel(), f'mid{i}', gt=g32(batch['grid_feature'][i]), grad=(s, 1))
    g2 = g32(batch['grid_feature'][2]).unsqueeze(1)
    s = key('refine_BEV_feature_loss2')
    term(CLAMP, s, float(dw[2]) / P['refine_BEV_feature'].numel(), 'refine_BEV_feature', gt=g2, grad=(s, 1))
    s = key('refine_flattened_feature_loss')
    term(CLAMP, s, fw * 0.1 / P['refine_flattned_BEV_feature'].numel(), 'refine_flattned_BEV_feature', gt=gt_feat.unsqueeze(1),
         grad=(s, 1))
    for k, name in (('teacher_pred_wp_offset', 'teacher_wp_loss'), ('teacher_pred_ctrl_offset_lis', 'teacher_action_loss')):
        s = key(name)
        term(SL1, s, 1.0 / P[k].numel(), k, grad=(s, 1))
    gf = torch.stack([g32(t[2]) for t in batch['future_grid_feature']], 1).unsqueeze(1)
    s = key('teacher_future_BEV_feature_loss2')
    term(CLAMP, s, float(dw[2]) / P['teacher_future_BEV_feature'].numel(), 'teacher_future_BEV_feature', gt=gf, grad=(s, 1))
    s = key('teacher_refine_BEV_feature_loss2')
    term(CLAMP, s, float(dw[2]) / P['teacher_refine_BEV_feature'].numel(), 'teacher_refine_BEV_feature', gt=g2, grad=(s, 1))
    s = key('teacher_refine_flattened_feature_loss')
    term(CLAMP, s, fw / P['teacher_refine_flattned_BEV_feature'].numel(), 'teacher_refine_flattned_BEV_feature', gt=gt_feat.unsqueeze(1),
         grad=(s, 1))
    plan = dict(terms=terms, keys=keys, detached=detached, paired=paired, n_slots=sum(c for _, _, c, _ in keys), hold=hold)
    outs = DecoderLossFunction.apply(plan, *inputs)
    return OrderedDict((name, o) for (name, *_), o in zip(keys, outs))
