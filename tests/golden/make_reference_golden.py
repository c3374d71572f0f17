"""Golden vectors produced by the REFERENCE'S OWN Python (run in the build container, where /root/reference is mounted):

    python tests/golden/make_reference_golden.py        -> tests/golden/ref_*.npz

The reference cannot be imported as a package here (mmcv / mmdet / mmdet3d / spconv are absent), but its in-tree files can:
`_ref_stubs.py` supplies import-time plumbing only (registries, BaseModule, fp16 decorators), after which
`open_loop_training/code/encoder_decoder_framework.py`, `code/utils.py`, `model_code/dense_heads/{thinktwice_decoder,
multi_scale_deformable_attn_function,utils}.py` load and run unmodified.  What is exercised is the reference's own arithmetic for

  * BEV fusion + SE pyramid + flatten MLP        (framework:81-138, 213-235; code/utils.py:84-121)
  * the whole ThinkTwiceDecoder forward           (thinktwice_decoder.py:26-489; msda:197-526; dense_heads/utils.py:53-106)
  * process_action / control_pid / PIDController  (framework:268-390; code/utils.py:7-29)

with ONE third-party leaf supplied from its published semantics: mmcv's `multi_scale_deformable_attn_pytorch`
(= oracle.decoder.msda_pytorch, itself checked against brute-force bilinear loops in tests/test_oracle_selfcheck.py).
The camera / LiDAR encoders are replaced by seeded random feature maps of the real shapes' aspect (they are pinned elsewhere).

Weights are NOT stored (the decoder alone is ~50 M parameters): both sides fill every state_dict entry from a generator seeded by
the entry's NAME (`named_init`), which also checks that the oracle and the reference expose the same names and shapes.
"""
import importlib
import os
import sys
import types
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = '/root/reference/open_loop_training/code'
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)


_REGS = None                                                       # registries of an already-loaded reference (tests reuse it)


def named_init(module, seed, prefix=''):
    """fill every state_dict entry of `module` from a generator seeded by crc32(prefix + name) ^ seed."""
    sd = module.state_dict()
    params = {n for n, _ in module.named_parameters()} if hasattr(module, 'named_parameters') else None
    out = {}
    for name, t in sd.items():
        if params is not None and name not in params and not name.endswith(('running_mean', 'running_var')):
            out[name] = t.clone()                                      # geometry buffers (frustum, voxel_*), step counters: keep
            continue
        g = torch.Generator().manual_seed((zlib.crc32((prefix + name).encode()) ^ (seed * 2654435761)) & 0x7FFFFFFF)
        if name.endswith('num_batches_tracked'):
            out[name] = t.clone()
        elif name.endswith('running_var'):
            out[name] = 0.8 + 0.4 * torch.rand(t.shape, generator=g)
        elif name.endswith('running_mean'):
            out[name] = 0.1 * torch.randn(t.shape, generator=g)
        elif t.dim() >= 2:
            fan_in = t[0].numel()
            out[name] = torch.randn(t.shape, generator=g) * (2.0 / fan_in) ** 0.5
        elif name.endswith('weight'):
            out[name] = 1.0 + 0.05 * torch.randn(t.shape, generator=g)          # norm scales
        else:
            out[name] = 0.02 * torch.randn(t.shape, generator=g)                # biases
        out[name] = out[name].to(t.dtype)
    module.load_state_dict(out)
    return out


def synthetic_inputs(cfg, seed, B=1):
    """seeded stand-ins for what the encoders hand to fusion + decoder (shapes of thinktwice.py, FPN maps at 1/4 linear size)."""
    from thinktwice_b200.synthetic import make_batch
    g = torch.Generator().manual_seed(7000 + seed)
    r = lambda *s: torch.randn(*s, generator=g)
    batch = make_batch(cfg, B, seed=seed, num_points=100)
    metas = batch['img_metas']
    l2i = torch.stack([torch.as_tensor(np.asarray(m[-1]['lidar2img']), dtype=torch.float32) for m in metas])     # (B, 4, 4, 4)
    ida = torch.stack([torch.as_tensor(np.asarray(m[-1]['ida_mats']), dtype=torch.float32) for m in metas])
    fpn = [0.5 * r(B * 4, 256, h, w) for (h, w) in ((28, 56), (14, 28), (7, 14), (4, 7))]
    return dict(cam_bev=0.5 * r(B, 256, 21, 21), lidar=0.5 * r(B, 512, 84, 84), fpn=fpn, lidar2img=l2i, ida_mat=ida,
                speed=batch['speed'], target_point=batch['target_point'], target_command=batch['target_command'])


def load_reference():
    import _ref_stubs
    regs = _ref_stubs.install()
    from oracle.decoder import msda_pytorch
    sys.modules['mmcv.ops.multi_scale_deform_attn'].multi_scale_deformable_attn_pytorch = msda_pytorch
    for name, path in (('olt_code', REF), ('olt_code.model_code', REF + '/model_code'),
                       ('olt_code.model_code.dense_heads', REF + '/model_code/dense_heads')):
        m = types.ModuleType(name)
        m.__path__ = [path]
        sys.modules[name] = m                                          # synthetic packages: the real __init__.py files are not run

    class _StubEncoder(torch.nn.Module):                               # stands where LSS / LidarNet would be built
        def __init__(self, d_bound=(1.0, 41.0, 0.5), **kw):
            super().__init__()
            self.d_bound = d_bound
    regs['stub_encoder'] = _StubEncoder
    regs['BACKBONES'].classes['LSS'] = _StubEncoder
    regs['BACKBONES'].classes['LidarNet'] = _StubEncoder
    importlib.import_module('olt_code.model_code.dense_heads.thinktwice_decoder')          # registers ThinkTwiceDecoder
    return importlib.import_module('olt_code.encoder_decoder_framework'), regs


def load_reference_lss(regs):
    """model_code/backbones/lss.py behind stubs.  Reference-own code exercised: DepthNet / ASPP / Mlp / SELayer / UNet /
    seg->feature stack / PAFPN forward (the in-tree restatement lss.py:286-348) / create_frustum / get_geometry / the lift /
    sweep handling / LSS.forward's matrix assembly.  Third-party LEAVES supplied from published semantics (all named in the fixture):
    mmdet ResNet-50 and PAFPN layer CONSTRUCTION, mmdet BasicBlock, mmcv DCN pack (torchvision deform_conv2d) = oracle.camera.*;
    ops.voxel_pooling (CUDA-only) = oracle.voxel_pool.voxel_pooling_ref, itself checked against the reference's compiled kernel on
    the GPU box (tests/test_ops_gpu.py)."""
    import _ref_stubs
    from oracle import camera as oc, voxel_pool as ovp
    for n in ['mmdet.models.backbones', 'mmdet.models.backbones.resnet', 'mmdet.models.necks', 'mmdet.models.necks.pafpn', 'ops',
              'ops.voxel_pooling']:
        _ref_stubs._mod(n)
    S = sys.modules

    class _ResNet(oc.ResNet50):
        def __init__(self, **cfg):
            super().__init__()

        def init_weights(self):
            pass

    class _PAFPNBase(_ref_stubs.BaseModule):                           # mmdet FPN/PAFPN __init__: layer construction only
        def __init__(self, in_channels, out_channels, num_outs, start_level=0, add_extra_convs=False,
                     relu_before_extra_convs=False, **kw):
            super().__init__()
            n = len(in_channels)
            self.in_channels, self.out_channels, self.num_outs, self.start_level = in_channels, out_channels, num_outs, start_level
            self.backbone_end_level, self.add_extra_convs, self.relu_before_extra_convs = n, add_extra_convs, relu_before_extra_convs
            self.lateral_convs = torch.nn.ModuleList([oc.ConvModule(c, out_channels, 1) for c in in_channels])
            self.fpn_convs = torch.nn.ModuleList([oc.ConvModule(out_channels, out_channels, 3, padding=1) for _ in range(n)])
            self.downsample_convs = torch.nn.ModuleList([oc.ConvModule(out_channels, out_channels, 3, stride=2, padding=1) for _ in range(n - 1)])
            self.pafpn_convs = torch.nn.ModuleList([oc.ConvModule(out_channels, out_channels, 3, padding=1) for _ in range(n - 1)])

        def init_weights(self):
            pass

    S['mmdet.models'].build_backbone = lambda cfg: _ResNet(**cfg)
    S['mmdet.models.backbones.resnet'].BasicBlock = lambda cin, cout: oc.BasicBlock(cin)
    S['mmdet.models.necks.pafpn'].PAFPN = _PAFPNBase
    S['mmdet3d.models'].build_neck = lambda cfg: regs['NECKS'].build(cfg)
    S['mmcv.cnn'].build_conv_layer = lambda cfg, *a, **k: oc.DeformConv2dPack(cfg['in_channels'], cfg['out_channels'], cfg['groups'])
    S['ops.voxel_pooling'].voxel_pooling = ovp.voxel_pooling_ref
    m = types.ModuleType('olt_code.model_code.backbones')
    m.__path__ = [REF + '/model_code/backbones']
    sys.modules['olt_code.model_code.backbones'] = m
    lss = importlib.import_module('olt_code.model_code.backbones.lss')
    regs['NECKS'].classes['PAFPN'] = lss.PAFPN_fp32                    # cfg type 'PAFPN' (mmdet's): same forward, restated in-tree
    return lss


def lss_digest(out):
    """what the fixture keeps of an LSS output dict: small tensors whole, big maps as channel means + a strided sub-grid."""
    keep = {'bev': out['bev'], 'depth': out['depth'], 'lidar2img': out['lidar2img'], 'ida_mat': out['ida_mat'],
            'seg.mean_hw': out['seg'].mean((-2, -1)), 'seg.sub8': out['seg'][..., ::8, ::8]}
    for i, f in enumerate(out['fpn_feats']):
        keep[f'fpn{i}.mean_hw'] = f.mean((-2, -1))
        keep[f'fpn{i}.sub'] = f[..., ::4, ::4][:, ::8]
    return keep


def lss_case(regs):
    """camera encoder at the plumbing shape: reference LSS.forward vs the same inputs, name-keyed weights."""
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(PLUMBING_CONFIG)
    lss = load_reference_lss(regs)
    kw = {k: v for k, v in dict(cfg.model['img_encoder']).items() if k != 'type'}
    for seed, B in ((0, 1), (1, 2)):
        torch.manual_seed(seed)
        ref = lss.LSS(**kw).eval()
        named_init(ref, seed, prefix='img_encoder.')
        batch = make_batch(cfg, B, seed=seed, num_points=10)
        with torch.no_grad():
            out = ref(batch['img'], batch['img_metas'], is_return_depth=True)
        names = sorted(ref.state_dict().keys())
        keep = lss_digest(out)
        np.savez_compressed(os.path.join(HERE, f'ref_lss_plumbing_seed{seed}.npz'), batch=np.array(B), names=np.array(names),
                            shapes=np.array([str(tuple(ref.state_dict()[n].shape)) for n in names]),
                            **{k: v.detach().cpu().numpy().astype(np.float32) for k, v in keep.items()})
        print(f'lss seed {seed} B {B}: bev {tuple(out["bev"].shape)} |bev| {float(out["bev"].abs().max()):.3f} seg {tuple(out["seg"].shape)} '
              f'depth {tuple(out["depth"].shape)}')


PRED_KEYS = ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'pred_value_traj', 'pred_value_ctrl',
             'refine_flattned_BEV_feature', 'refine_BEV_feature')


def e2e_case(fw, regs):
    """the reference's EncoderDecoder.forward_inference end to end at the plumbing shape (framework:194-250: state assembly,
    extract_sensor_feat with its rot90(flip), fusion, decoder) with the reference LSS as camera encoder.  The LiDAR encoder is
    third-party glue over mmdet3d / spconv (lidarnet.py:28-96): oracle.lidar.LidarNet stands in for it on both sides."""
    from oracle.lidar import LidarNet
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(PLUMBING_CONFIG)
    mc = cfg.model
    lss = sys.modules['olt_code.model_code.backbones.lss']
    regs['BACKBONES'].classes['LSS'] = lss.LSS
    regs['BACKBONES'].classes['LidarNet'] = LidarNet
    for seed, B in ((0, 1), (1, 2)):
        torch.manual_seed(seed)
        ref = fw.EncoderDecoder(img_encoder=dict(mc['img_encoder']), decoder=dict(mc['decoder']), lidar_encoder=dict(mc['lidar_encoder']),
                                train_cfg=mc['train_cfg'], test_cfg=mc.get('test_cfg')).eval()
        named_init(ref, seed)
        batch = make_batch(cfg, B, seed=seed, num_points=1500)
        batch['target_command_raw'] = batch['target_command'].argmax(-1)
        with torch.no_grad():
            pred = ref.forward_inference(batch)
        names = sorted(ref.state_dict().keys())
        np.savez_compressed(os.path.join(HERE, f'ref_e2e_plumbing_seed{seed}.npz'), batch=np.array(B), names=np.array(names),
                            shapes=np.array([str(tuple(ref.state_dict()[n].shape)) for n in names]),
                            **{k: pred[k].detach().cpu().numpy() for k in PRED_KEYS})
        print(f'e2e seed {seed} B {B}: pred_wp[-1] = {[round(float(v), 4) for v in pred["pred_wp"][0, -1].flatten()]}')
    regs['BACKBONES'].classes['LSS'] = regs['stub_encoder']
    regs['BACKBONES'].classes['LidarNet'] = regs['stub_encoder']


def calibrated_case(fw, regs):
    """the reference's EncoderDecoder.forward_inference (its framework, LSS and decoder; LiDAR encoder = oracle stand-in) with the
    oracle's seeded, BatchNorm-calibrated weights: the plumbing config at seeds 0..2 (the weights of tests/golden/plumbing_seed*.npz)
    and the full thinktwice.py config at seed 0 (the bench workload, B = 1)."""
    from oracle.lidar import LidarNet
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG, PLUMBING_CONFIG
    from thinktwice_b200.synthetic import make_batch
    lss = sys.modules['olt_code.model_code.backbones.lss']
    regs['BACKBONES'].classes['LSS'], regs['BACKBONES'].classes['LidarNet'] = lss.LSS, LidarNet
    for name, path, seeds, points in (('plumbing', PLUMBING_CONFIG, (0, 1, 2), 2000), ('full', DEFAULT_CONFIG, (0,), 40000)):
        mc = Config.fromfile(path).model
        for seed in seeds:
            o = Oracle(**{k: v for k, v in mc.items() if k != 'type'})
            init_oracle_weights(o, seed)
            batch = make_batch(Config.fromfile(path), 1, seed=seed, num_points=points)
            calibrate_bn(o, batch)
            ref = fw.EncoderDecoder(img_encoder=dict(mc['img_encoder']), decoder=dict(mc['decoder']), lidar_encoder=dict(mc['lidar_encoder']),
                                    train_cfg=mc['train_cfg'], test_cfg=mc.get('test_cfg')).eval()
            ref.load_state_dict(o.state_dict())
            batch['target_command_raw'] = batch['target_command'].argmax(-1)
            with torch.no_grad():
                pred = ref.forward_inference(batch)
            keys = PRED_KEYS if name == 'full' else PRED_KEYS[:-1]
            np.savez_compressed(os.path.join(HERE, f'ref_calibrated_{name}_seed{seed}.npz'), **{k: pred[k].detach().cpu().numpy() for k in keys})
            print(f'calibrated {name} seed {seed}: pred_wp[-1] = {[round(float(v), 4) for v in pred["pred_wp"][0, -1].flatten()]}')
    regs['BACKBONES'].classes['LSS'] = regs['stub_encoder']
    regs['BACKBONES'].classes['LidarNet'] = regs['stub_encoder']


GEOM_SAMPLE = 8192


def camera_geometry_case(regs):
    """what the reference LSS computes on the host side of the camera branch, for the plumbing and the full config (B = 2, batch
    seed 3): create_frustum, the voxel grid constants, get_geometry per sweep (on the matrices LSS.forward assembles; a seeded sample of
    GEOM_SAMPLE points and their integer voxel indices) and the 22-wide tensor DepthNet feeds its BatchNorm1d."""
    from thinktwice_b200.config import Config, DEFAULT_CONFIG, PLUMBING_CONFIG
    from thinktwice_b200.registry import BACKBONES
    from thinktwice_b200.synthetic import make_batch
    lss = sys.modules['olt_code.model_code.backbones.lss']
    for which, path in (('plumbing', PLUMBING_CONFIG), ('full', DEFAULT_CONFIG)):
        cfg = Config.fromfile(path)
        kw = {k: v for k, v in dict(cfg.model['img_encoder']).items() if k != 'type'}
        ref = lss.LSS(**kw).eval()
        prod = BACKBONES.build(dict(cfg.model['img_encoder']))          # (only its build_mats: the matrices LSS.forward assembles)
        B = 2
        batch = make_batch(cfg, B, seed=3, num_points=10)
        metas = batch['img_metas']
        N = batch['img'].shape[2]
        mats = prod.build_mats(metas, N)
        out = dict(frustum=ref.frustum.numpy(), lower=(ref.voxel_coord - ref.voxel_size / 2.0).numpy(), voxel_size=ref.voxel_size.numpy(),
                   voxel_num=np.array([int(v) for v in ref.voxel_num]))
        lower = ref.voxel_coord - ref.voxel_size / 2.0
        for s in range(len(metas[0])):
            idx = -1 if s == 0 else -s                                  # the sweep index LSS.forward passes (lss.py:689, 712)
            geom = ref.get_geometry(mats['sensor2ego_mats'][:, idx], mats['intrin_mats'][:, idx], mats['ida_mats'][:, idx], None)
            flat = geom.reshape(-1, 3)
            pos = torch.randperm(flat.shape[0], generator=torch.Generator().manual_seed(s))[:GEOM_SAMPLE].sort().values
            out[f'geom{s}_pos'] = pos.numpy()
            out[f'geom{s}'] = flat[pos].numpy()
            out[f'geom{s}_voxel'] = ((flat[pos] - lower) / ref.voxel_size).int().numpy()
        seen = {}
        h = ref.depth_net.bn.register_forward_pre_hook(lambda m, inp: seen.setdefault('x', inp[0].detach().clone()))
        with torch.no_grad():
            ref.depth_net(torch.zeros(B * N, kw['depth_net_conf']['in_channels'], 2, 2), {k: v for k, v in mats.items()})
        h.remove()
        out['depthnet_bn_input'] = seen['x'].reshape(B * N, 22).numpy()
        np.savez_compressed(os.path.join(HERE, f'ref_camera_geometry_{which}.npz'), **out)
        print(f'camera geometry {which}: frustum {tuple(ref.frustum.shape)}, {len(metas[0])} sweeps')


def main():
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    cfg = Config.fromfile(DEFAULT_CONFIG)
    fw, regs = load_reference()
    lss_case(regs)
    e2e_case(fw, regs)
    calibrated_case(fw, regs)
    camera_geometry_case(regs)
    mc = cfg.model
    regs['BACKBONES'].classes['LSS'] = regs['stub_encoder']            # (importing lss.py registered the real LSS)
    for seed, B in ((0, 1), (1, 1), (2, 2)):                           # B = 2: the Look module couples the frames of a batch (SURVEY fact 4)
        torch.manual_seed(seed)
        ref = fw.EncoderDecoder(img_encoder=dict(mc['img_encoder']), decoder=dict(mc['decoder']), lidar_encoder=dict(mc['lidar_encoder']),
                                train_cfg=mc['train_cfg'], test_cfg=mc.get('test_cfg'))
        ref.eval()
        named_init(ref, seed)
        x = synthetic_inputs(cfg, seed, B)
        with torch.no_grad():
            state = torch.cat([x['speed'].float().view(-1, 1) / 12., x['target_point'].float(), x['target_command']], -1)
            meas = ref.measurements_encoder(state)
            flat, bev32, mid, lidar_hi = ref.get_fusion_feat({'bev': x['cam_bev']}, [x['lidar']])
            pred = ref.decoder(flat, bev32, meas, x['target_point'], ref, None, [x['lidar2img'], x['ida_mat'], x['fpn'], lidar_hi])
            # call-site types of leaderboard/team_code/thinktwice_agent.py:458-461: speed = FloatTensor([v]), target = numpy (2,)
            tp = x['target_point'][0].numpy()
            p0 = {k: v[:1] for k, v in pred.items() if torch.is_tensor(v)}   # the agent runs B = 1 (control_pid asserts it)
            steer, throttle, brake, meta = ref.process_action(p0, 3, x['speed'][:1], tp)
            pid = ref.control_pid(p0['pred_wp'][:, -1], x['speed'][:1], tp)
        out = {'meas': meas, 'flat': flat, 'bev32': bev32, 'mid10': mid[3], 'mid4': mid[4], 'mid2': mid[5]}
        for k in ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'pred_value_traj',
                  'pred_value_ctrl', 'refine_flattned_BEV_feature', 'refine_BEV_feature'):
            out['pred.' + k] = pred[k]
        out['pred.refine_future_BEV_feature.mean_hw'] = pred['refine_future_BEV_feature'].mean((-2, -1))   # (B, K, T, 32): keeps the fixture small
        out['action'] = torch.tensor([steer, throttle, brake], dtype=torch.float64)
        out['pid'] = torch.tensor([float(v) for v in pid[:3]] + [pid[3][k] for k in ('desired_speed', 'angle', 'angle_last', 'angle_target', 'angle_final', 'delta')], dtype=torch.float64)
        names = sorted(ref.state_dict().keys())
        np.savez_compressed(os.path.join(HERE, f'ref_fusion_decoder_seed{seed}.npz'),
                            batch=np.array(B), names=np.array(names), shapes=np.array([str(tuple(ref.state_dict()[n].shape)) for n in names]),
                            **{k: v.detach().cpu().numpy() for k, v in out.items()})
        print(f'seed {seed} B {B}: pred_wp[-1] = {pred["pred_wp"][0, -1].flatten().tolist()}  action = {steer:.4f} {throttle:.4f} {brake:.4f}')


if __name__ == '__main__':
    main()
