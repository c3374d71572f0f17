"""Plain-PyTorch restatement of the reference's open-loop validation path — TEST INFRASTRUCTURE ONLY.  Built on the oracle's modules
(oracle/decoder.py, oracle/model.py), it adds what the inference oracle lacks:

  * teacher_pass     thinktwice_decoder.py:491-533  (the K layers fed the ground truth; only BEV / flat / future features chain)
  * decoder_loss     thinktwice_decoder.py:535-636  (every term of ThinkTwiceDecoder.loss, torch.distributions.Beta KLs)
  * forward_train    encoder_decoder_framework.py:147-191 with use_depth = use_seg = False
  * parse_losses     encoder_decoder_framework.py:409-440

tests/golden/ref_losses_*.npz pin it to the reference's own code (tests/test_losses_cpu.py).
"""
from collections import OrderedDict

import torch
import torch.nn.functional as F
from torch.distributions import Beta, kl_divergence

TEACHER_INPUTS = ('waypoints', 'action_sigma', 'action_mu', 'future_action_sigma', 'future_action_mu')
DISTIL = {2: 0.25, 3: 1.0 / 3.0, 4: 1.0 / 4.0, 5: 1 / 11.0}


def inv_softplus(x):
    return x + torch.log(-torch.expm1(-x))


def teacher_pass(dec, flat, bev, meas, parent, look_meta, tf):
    lidar2img, ida, fpn, lidar_hi = look_meta
    mlvl = [getattr(dec, f'fpn_linear{i}')(fpn[i]) for i in range(4)]
    shapes, fpn_flat = dec.transform_fpn_feats(mlvl)
    wp = tf['waypoints'].float()
    sp = torch.cat([torch.cat([tf['action_mu'], tf['action_sigma']], -1).unsqueeze(1),
                    torch.cat([torch.stack(tf['future_action_mu'][:-1], 1), torch.stack(tf['future_action_sigma'][:-1], 1)], -1)], 1).float()
    ctrl = inv_softplus(sp)
    fut, cur_bev, cur_flat = None, bev.clone(), flat.clone()
    off_wp, off_ctrl, s_bev, s_flat, s_fut = [], [], [], [], []
    for layer in dec.decoder_layers:
        t_off, c_off, fut, cur_bev, cur_flat = layer(cur_bev, wp, ctrl, fut, parent, dec.grid2feat, meas, cur_flat, lidar2img, ida,
                                                     dec.config['img_size'], mlvl, fpn_flat, shapes, lidar_hi, dec.temporal_embedding,
                                                     dec.static_embedding, False)
        off_wp.append(t_off); off_ctrl.append(c_off); s_bev.append(cur_bev); s_flat.append(cur_flat); s_fut.append(fut)
    return dict(teacher_pred_wp_offset=torch.stack(off_wp, 1), teacher_pred_ctrl_offset_lis=torch.stack(off_ctrl, 1),
                teacher_future_BEV_feature=torch.stack(s_fut, 1), teacher_refine_flattned_BEV_feature=torch.stack(s_flat, 1),
                teacher_refine_BEV_feature=torch.stack(s_bev, 1))


def action_beta(alpha, beta):
    x = torch.zeros_like(alpha)
    x[:, 1] += 0.5
    m1 = (alpha > 1) & (beta > 1)
    x[m1] = (alpha[m1] - 1) / (alpha[m1] + beta[m1] - 2)
    x[(alpha <= 1) & (beta > 1)] = 0.0
    x[(alpha > 1) & (beta <= 1)] = 1.0
    m4 = (alpha <= 1) & (beta <= 1)
    x[m4] = alpha[m4] / torch.clamp(alpha[m4] + beta[m4], min=1e-5)
    return x * 2 - 1


def _clamped(p, g):
    return torch.clamp(F.smooth_l1_loss(p, g, reduction='none'), min=-5.0, max=5.0).mean()


def decoder_loss(config, batch, pred, mid):
    d = OrderedDict()
    gt_speed = batch['speed'].to(dtype=torch.float32).view(-1, 1) / 12.
    gt_value = batch['value'].view(-1, 1)
    gt_feat = batch['feature']
    gt_wp = batch['waypoints']
    a = F.l1_loss(action_beta(pred['mu_branches'][:, -1, :], pred['sigma_branches'][:, -1, :]),
                  action_beta(batch['action_mu'], batch['action_sigma']), reduction='none').mean(0)
    d['current_throttle_brake_offset'], d['current_steer_offset'] = a[0], a[1]
    w = F.l1_loss(pred['pred_wp'][:, -1], gt_wp, reduction='none').mean(0).mean(0)
    d['longitudinal_offset'], d['lateral_offset'] = w[0], w[1]
    kl = kl_divergence(Beta(batch['action_mu'].unsqueeze(1), batch['action_sigma'].unsqueeze(1)), Beta(pred['mu_branches'], pred['sigma_branches']))
    d['action_loss'] = kl.mean() * 15.0
    d['speed_loss'] = F.smooth_l1_loss(pred['pred_speed'], gt_speed)
    d['value_loss'] = (F.smooth_l1_loss(pred['pred_value_traj'], gt_value) +
                       F.smooth_l1_loss(pred['pred_value_ctrl'], gt_value, reduction='none')) * config['value_weight']
    d['flattened_feature_loss'] = (F.smooth_l1_loss(pred['pred_features_traj'], gt_feat) +
                                   F.smooth_l1_loss(pred['pred_features_ctrl'], gt_feat)) * config['features_weight']
    fm = torch.stack(batch['future_action_mu'][:-1], 1).unsqueeze(1)
    fs = torch.stack(batch['future_action_sigma'][:-1], 1).unsqueeze(1)
    d['future_action_loss'] = kl_divergence(Beta(fm, fs), Beta(pred['future_mu'], pred['future_sigma'])).mean() * 15.0 * 0.25
    d['wp_loss'] = F.smooth_l1_loss(pred['pred_wp'], gt_wp.unsqueeze(1).expand_as(pred['pred_wp'])) * 15.0
    for i, wt in DISTIL.items():
        d[f'BEV_feature_loss{i}'] = _clamped(mid[i], batch['grid_feature'][i]) * wt
    g2 = batch['grid_feature'][2]
    rb = pred['refine_BEV_feature']
    d['refine_BEV_feature_loss2'] = _clamped(rb, g2.unsqueeze(1).expand_as(rb)) * DISTIL[2]
    rf = pred['refine_flattned_BEV_feature']
    d['refine_flattened_feature_loss'] = _clamped(rf, gt_feat.unsqueeze(1).expand_as(rf)) * config['features_weight'] * 0.1
    d['teacher_wp_loss'] = F.smooth_l1_loss(pred['teacher_pred_wp_offset'], torch.zeros_like(pred['teacher_pred_wp_offset']))
    d['teacher_action_loss'] = F.smooth_l1_loss(pred['teacher_pred_ctrl_offset_lis'], torch.zeros_like(pred['teacher_pred_ctrl_offset_lis']))
    tfut = pred['teacher_future_BEV_feature']
    gf = torch.stack([f[2] for f in batch['future_grid_feature']], 1).unsqueeze(1).expand_as(tfut)
    d['teacher_future_BEV_feature_loss2'] = _clamped(tfut, gf) * DISTIL[2]
    tb = pred['teacher_refine_BEV_feature']
    d['teacher_refine_BEV_feature_loss2'] = _clamped(tb, g2.unsqueeze(1).expand_as(tb)) * DISTIL[2]
    tf = pred['teacher_refine_flattned_BEV_feature']
    d['teacher_refine_flattened_feature_loss'] = _clamped(tf, gt_feat.unsqueeze(1).expand_as(tf)) * config['features_weight']
    return d


def _frame(batch, j):
    def cut(v):
        if torch.is_tensor(v):
            return v[j:j + 1]
        if isinstance(v, list):
            return [cut(x) for x in v]
        return v
    return {k: v[j:j + 1] if k == 'img_metas' else cut(v) for k, v in batch.items()}


@torch.no_grad()
def predict_train(o, batch):
    """the oracle's teacher-forced forward: (pred dict with the teacher_* outputs, mid_BEV_feature)."""
    keep = {}
    pred = o.forward_inference(batch, keep=keep)
    cam = keep['cam']
    pred.update(teacher_pass(o.decoder, keep['flat'], keep['bev32'], keep['meas'], o,
                             [cam['lidar2img'], cam['ida_mat'], cam['fpn_feats'], keep['lidar'][0]], batch))
    return pred, keep['mid']


@torch.no_grad()
def forward_train(o, batch, independent_frames=False):
    """framework:147-191 on the oracle.  independent_frames: every frame's predictions as the frame computes them alone (B = 1), the
    losses over the whole batch (EncoderDecoder.enable_independent_frames)."""
    if not independent_frames:
        pred, mid = predict_train(o, batch)
    else:
        B = batch['img'].shape[0]
        parts = [predict_train(o, _frame(batch, j)) for j in range(B)]
        pred = {k: torch.cat([p[k] for p, _ in parts]) for k in parts[0][0] if torch.is_tensor(parts[0][0][k])}
        mid = [None, None] + [torch.cat([m[i] for _, m in parts]) for i in range(2, 6)]
    return decoder_loss(o.config, batch, pred, mid), pred


def parse_losses(losses):
    log_vars = OrderedDict((k, v.mean()) for k, v in losses.items())
    log_vars['loss'] = sum(v for k, v in log_vars.items() if 'loss' in k)
    return log_vars['loss'], OrderedDict((k, v.item()) for k, v in log_vars.items())
