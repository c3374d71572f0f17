"""Golden vectors of the camera branch's supervision, produced by the REFERENCE'S OWN Python behind the import stubs of
make_reference_golden.py (run where the reference tree is available):

    python tests/golden/make_camera_loss_golden.py        -> tests/golden/ref_camera_losses_plumbing_seed{0,1}.npz

The reference's EncoderDecoder.forward_train (encoder_decoder_framework.py:147-191: the decoder's losses, then seg_loss through
get_downsampled_gt_seg and utils.FocalLoss, then depth_loss through get_downsampled_gt_depth and BCE-with-logits) and _parse_losses at
the plumbing shape with train_cfg use_depth = use_seg = True, as the shipped configuration trains; the reference LSS as camera encoder and
oracle.lidar.LidarNet standing in for the LiDAR encoder, the oracle's seeded, BatchNorm-calibrated weights (as make_loss_golden.py).
The ground truth is thinktwice_b200.synthetic.make_supervision + make_camera_supervision.  Stored: every loss term, every log var and
the log vars' order.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

CASES = ((0, 1), (1, 2))                                               # (seed, B)


def camera_config():
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    cfg = Config.fromfile(PLUMBING_CONFIG)
    cfg.merge_from_dict({'model.train_cfg.use_seg': True, 'model.train_cfg.use_depth': True})
    return cfg


def main():
    from make_reference_golden import load_reference, load_reference_lss
    from oracle.lidar import LidarNet
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.synthetic import make_batch, make_camera_supervision, make_supervision
    fw, regs = load_reference()
    cfg = camera_config()
    mc = cfg.model
    lss = sys.modules.get('olt_code.model_code.backbones.lss') or load_reference_lss(regs)
    regs['BACKBONES'].classes['LSS'], regs['BACKBONES'].classes['LidarNet'] = lss.LSS, LidarNet
    for seed, B in CASES:
        batch = make_batch(cfg, B, seed=seed, num_points=1500)
        o = Oracle(**{k: v for k, v in mc.items() if k != 'type'})
        init_oracle_weights(o, seed)
        calibrate_bn(o, batch)
        ref = fw.EncoderDecoder(img_encoder=dict(mc['img_encoder']), decoder=dict(mc['decoder']), lidar_encoder=dict(mc['lidar_encoder']),
                                train_cfg=mc['train_cfg'], test_cfg=mc.get('test_cfg')).eval()
        ref.load_state_dict(o.state_dict())
        assert ref.use_seg and ref.use_depth
        batch.update(make_supervision(cfg, B, seed=seed))
        batch.update(make_camera_supervision(cfg, B, seed=seed))
        with torch.no_grad():
            losses = ref.forward_train(batch)
            _, log_vars = ref._parse_losses(losses)
        arrs = {'loss.' + k: np.asarray(v.detach().cpu().numpy()) for k, v in losses.items()}
        arrs.update({'log.' + k: np.asarray(v, dtype=np.float64) for k, v in log_vars.items()})
        np.savez_compressed(os.path.join(HERE, f'ref_camera_losses_plumbing_seed{seed}.npz'), keys=np.array(list(losses.keys())),
                            log_keys=np.array(['log.' + k for k in log_vars]), batch=np.array(B), **arrs)
        print(f'seed {seed}, B {B}: loss {log_vars["loss"]:.6f}  seg_loss {log_vars["seg_loss"]:.6g}  depth_loss {log_vars["depth_loss"]:.6g}')
    regs['BACKBONES'].classes['LSS'] = regs['stub_encoder']
    regs['BACKBONES'].classes['LidarNet'] = regs['stub_encoder']


if __name__ == '__main__':
    main()
