"""Plain-PyTorch restatement of the camera branch's supervision in the reference's open-loop validation path — TEST INFRASTRUCTURE ONLY.
Built on tests/loss_oracle.py (the decoder's teacher-forced pass and losses) and the oracle's modules, it adds:

  * downsampled_gt_depth  encoder_decoder_framework.py:443-482 (min_pooling=True)
  * downsampled_gt_seg    encoder_decoder_framework.py:485-491 (T.Resize NEAREST, .long())
  * focal_loss            utils.py:31-47
  * camera_loss           encoder_decoder_framework.py:171-190 (seg_loss, depth_loss of the key frame)
  * forward_train         encoder_decoder_framework.py:147-191 honouring train_cfg use_seg / use_depth

tests/golden/ref_camera_losses_*.npz pin it to the reference's own code (tests/test_camera_losses_cpu.py).
"""
from collections import OrderedDict

import torch
import torch.nn.functional as F

import loss_oracle


def downsampled_gt_depth(gt, f, dbound, D):
    """framework:443-482 with min_pooling=True: (B, N, H, W) depths -> (B*N*h*w, D) one-hot bins (class 0 dropped)."""
    B, N, H, W = gt.shape
    g = gt.view(B * N, H // f, f, W // f, f, 1).permute(0, 1, 3, 5, 2, 4).contiguous().view(-1, f * f)
    g = torch.where(g == 0.0, 1e5 * torch.ones_like(g), g)
    g = torch.min(g, dim=-1).values.view(B * N, H // f, W // f)
    g = (g - (dbound[0] - dbound[2])) / dbound[2]
    g = torch.where((g < D + 1) & (g >= 0.0), g, torch.zeros_like(g))
    return F.one_hot(g.long(), num_classes=D + 1).view(-1, D + 1)[:, 1:].float()


def downsampled_gt_seg(gt, s):
    """framework:485-491: T.Resize((H // s, W // s), NEAREST) of the (B*N, H, W) labels (F.interpolate 'nearest' underneath), .long()."""
    B, N, H, W = gt.shape
    return F.interpolate(gt.reshape(B * N, 1, H, W), size=(H // s, W // s), mode='nearest')[:, 0].long()


def focal_loss(logits, labels, alpha=0.5, gamma=2, ignore_index=255):
    """utils.py:31-47: the focal transform of the batch-mean cross entropy over the non-ignored pixels."""
    logpt = -F.cross_entropy(logits, labels, ignore_index=ignore_index)
    pt = torch.exp(logpt)
    return -((1 - pt) ** gamma) * alpha * logpt


def camera_loss(config, batch, seg, depth, dbound, f=16, s=2):
    """framework:171-190: seg (B*N, C, h, w) and depth (B*N, D, h', w') logits of the key frame; the enabled terms in the reference's order."""
    d = OrderedDict()
    if config.get('use_seg', False):
        d['seg_loss'] = focal_loss(seg, downsampled_gt_seg(batch['seg'], s)) * 10
    if config.get('use_depth', False):
        D = depth.shape[1]
        gt = downsampled_gt_depth(batch['depth'], f, dbound, D)
        pred = depth.permute(0, 2, 3, 1).contiguous().view(-1, D)
        fg = torch.max(gt, dim=1).values > 0.0
        d['depth_loss'] = F.binary_cross_entropy_with_logits(pred[fg], gt[fg].to(pred.dtype), reduction='none').sum() / max(1.0, fg.sum())
    return d


@torch.no_grad()
def predict_train(o, batch):
    """loss_oracle.predict_train plus the key frame's segmentation / depth logits (pred['cam_seg'], pred['cam_depth'])."""
    keep = {}
    pred = o.forward_inference(batch, keep=keep)
    cam = keep['cam']
    pred.update(loss_oracle.teacher_pass(o.decoder, keep['flat'], keep['bev32'], keep['meas'], o,
                                         [cam['lidar2img'], cam['ida_mat'], cam['fpn_feats'], keep['lidar'][0]], batch))
    pred['cam_seg'], pred['cam_depth'] = cam['seg'], cam['depth']
    return pred, keep['mid']


@torch.no_grad()
def forward_train(o, batch, independent_frames=False):
    """framework:147-191 on the oracle: the decoder's terms (loss_oracle.decoder_loss), then seg_loss / depth_loss where o.config turns
    them on.  The depth / segmentation factors are the model's defaults, 16 and 2.  independent_frames as loss_oracle.forward_train."""
    if not independent_frames:
        pred, mid = predict_train(o, batch)
    else:
        B = batch['img'].shape[0]
        parts = [predict_train(o, loss_oracle._frame(batch, j)) for j in range(B)]
        pred = {k: torch.cat([p[k] for p, _ in parts]) for k in parts[0][0] if torch.is_tensor(parts[0][0][k])}
        mid = [None, None] + [torch.cat([m[i] for _, m in parts]) for i in range(2, 6)]
    losses = loss_oracle.decoder_loss(o.config, batch, pred, mid)
    losses.update(camera_loss(o.config, batch, pred['cam_seg'], pred['cam_depth'], o.img_encoder.d_bound))
    return losses, pred
