"""Golden vectors of the open-loop validation losses, produced by the REFERENCE'S OWN Python behind the import stubs of
make_reference_golden.py (run where the reference tree is available):

    python tests/golden/make_loss_golden.py        -> tests/golden/ref_losses_*.npz

  * plumbing_seed{0,1,2}: the reference's EncoderDecoder.forward_train (framework:147-191: state assembly, extract_sensor_feat,
    fusion, ThinkTwiceDecoder.forward with teacher forcing, ThinkTwiceDecoder.loss) and _parse_losses at the plumbing shape, with
    train_cfg use_depth = use_seg = False, the reference LSS as camera encoder and oracle.lidar.LidarNet standing in for the LiDAR
    encoder (third-party glue, as in make_reference_golden.e2e_case).  Weights: the oracle's seeded, BatchNorm-calibrated ones
    (make_reference_golden.calibrated_case), so that the predictions, and with them the losses, are of a sane size.
  * decoder_k5: the reference's fusion + ThinkTwiceDecoder.forward with teacher forcing + loss at the full config (K = 5, B = 2) on
    the seeded encoder stand-ins of make_reference_golden.synthetic_inputs.

The supervision is thinktwice_b200.synthetic.make_supervision (seeded, GT Beta parameters in U(0.5, 20)); torch.distributions.Beta
is the reference's own import.  Stored: every loss term, every log var, and the teacher-forced tensors (the bulky 21x21 maps of the
B = 2 cases as channel means + a strided sub-grid).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

TEACHER_KEYS = ('teacher_pred_wp_offset', 'teacher_pred_ctrl_offset_lis', 'teacher_refine_flattned_BEV_feature', 'teacher_refine_BEV_feature',
                'teacher_future_BEV_feature')
TEACHER_INPUTS = ('waypoints', 'action_sigma', 'action_mu', 'future_action_sigma', 'future_action_mu')
PLUMBING_CASES = ((0, 1), (1, 2), (2, 1))                              # (seed, B)


def loss_config(path):
    """a config with the camera branch's depth / segmentation supervision off (framework:42-43)."""
    from thinktwice_b200.config import Config
    cfg = Config.fromfile(path)
    for k in ('use_depth', 'use_seg'):
        cfg.merge_from_dict({f'model.train_cfg.{k}': False, f'model.decoder.config.{k}': False})
    return cfg


def digest(pred, full):
    """teacher tensors as stored: whole, or (full=False) the 21x21 maps as channel means + every 4th row / column."""
    out = {}
    for k in TEACHER_KEYS:
        v = pred[k].detach()
        if full or v.dim() < 5:
            out[k] = v
        else:
            out[k + '.mean_hw'] = v.mean((-2, -1))
            out[k + '.sub'] = v[..., ::4, ::4]
    return out


def save(name, losses, log_vars, teacher, **extra):
    arrs = {'loss.' + k: np.asarray(v.detach().cpu().numpy()) for k, v in losses.items()}
    arrs.update({'log.' + k: np.asarray(v, dtype=np.float64) for k, v in log_vars.items()})
    arrs.update({'teacher.' + k: v.cpu().numpy() for k, v in teacher.items()})
    np.savez_compressed(os.path.join(HERE, f'ref_losses_{name}.npz'), keys=np.array(list(losses.keys())), **arrs, **extra)
    print(f'{name}: loss {log_vars["loss"]:.6f}  ' + '  '.join(f'{k}={log_vars[k]:.4g}' for k in list(log_vars)[:6]))


def plumbing_case(fw, regs):
    from make_reference_golden import load_reference_lss
    from oracle.lidar import LidarNet
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import PLUMBING_CONFIG
    from thinktwice_b200.synthetic import make_batch, make_supervision
    cfg = loss_config(PLUMBING_CONFIG)
    mc = cfg.model
    lss = sys.modules.get('olt_code.model_code.backbones.lss') or load_reference_lss(regs)
    regs['BACKBONES'].classes['LSS'], regs['BACKBONES'].classes['LidarNet'] = lss.LSS, LidarNet
    for seed, B in PLUMBING_CASES:
        batch = make_batch(cfg, B, seed=seed, num_points=1500)
        o = Oracle(**{k: v for k, v in mc.items() if k != 'type'})
        init_oracle_weights(o, seed)
        calibrate_bn(o, batch)
        ref = fw.EncoderDecoder(img_encoder=dict(mc['img_encoder']), decoder=dict(mc['decoder']), lidar_encoder=dict(mc['lidar_encoder']),
                                train_cfg=mc['train_cfg'], test_cfg=mc.get('test_cfg')).eval()
        ref.load_state_dict(o.state_dict())
        batch.update(make_supervision(cfg, B, seed=seed))
        seen = {}
        h = ref.decoder.register_forward_hook(lambda m, a, out: seen.setdefault('pred', out))
        with torch.no_grad():
            losses = ref.forward_train(batch)
            _, log_vars = ref._parse_losses(losses)
        h.remove()
        save(f'plumbing_seed{seed}', losses, log_vars, digest(seen['pred'], B == 1), batch=np.array(B))
    regs['BACKBONES'].classes['LSS'] = regs['stub_encoder']
    regs['BACKBONES'].classes['LidarNet'] = regs['stub_encoder']


def decoder_k5_case(fw, regs, seed=3, B=2):
    from make_reference_golden import named_init, synthetic_inputs
    from thinktwice_b200.config import DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_supervision
    cfg = loss_config(DEFAULT_CONFIG)
    mc = cfg.model
    torch.manual_seed(seed)
    ref = fw.EncoderDecoder(img_encoder=dict(mc['img_encoder']), decoder=dict(mc['decoder']), lidar_encoder=dict(mc['lidar_encoder']),
                            train_cfg=mc['train_cfg'], test_cfg=mc.get('test_cfg')).eval()
    named_init(ref, seed)
    x = synthetic_inputs(cfg, seed, B)
    batch = dict(speed=x['speed'], **make_supervision(cfg, B, seed=seed))
    with torch.no_grad():
        state = torch.cat([x['speed'].float().view(-1, 1) / 12., x['target_point'].float(), x['target_command']], -1)
        meas = ref.measurements_encoder(state)
        flat, bev32, mid, lidar_hi = ref.get_fusion_feat({'bev': x['cam_bev']}, [x['lidar']])
        teacher = {k: batch[k] for k in TEACHER_INPUTS}
        pred = ref.decoder(flat, bev32, meas, x['target_point'], ref, teacher, [x['lidar2img'], x['ida_mat'], x['fpn'], lidar_hi])
        losses = ref.decoder.loss(batch, pred, mid)
        _, log_vars = ref._parse_losses(losses)
    save(f'decoder_k5_seed{seed}', losses, log_vars, digest(pred, False), batch=np.array(B), seed=np.array(seed))


def main():
    from make_reference_golden import load_reference
    fw, regs = load_reference()
    plumbing_case(fw, regs)
    decoder_k5_case(fw, regs)


if __name__ == '__main__':
    main()
