"""GPU: the H100 path reproduces the committed golden vectors (end-to-end plumbing config + per-op cases)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def rel(a, b):
    return float(np.abs(np.asarray(a) - b).max() / (np.abs(b).max() + 1e-12))


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_plumbing_forward_matches_golden(seed):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(PLUMBING_CONFIG)
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})        # only as the source of weights
    init_oracle_weights(o, seed)
    batch = make_batch(cfg, 1, seed=seed, num_points=2000)
    calibrate_bn(o, batch)
    m = build_model(cfg.model)
    m.load_state_dict(o.state_dict())
    m.prepare('cuda:0', impl=3)
    pred = m.forward_inference(batch)
    ref = np.load(os.path.join(G, f'plumbing_seed{seed}.npz'))
    for k in ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'refine_flattned_BEV_feature'):
        assert rel(pred[k].cpu().numpy(), ref[k]) < 1e-3, k
    cam = m.last_cam_feat
    assert rel(cam['bev'].nchw().sum((2, 3)).cpu().numpy(), ref['cam_bev_sum']) < 1e-3
    assert rel(cam['seg'].nchw().mean((2, 3)).cpu().numpy(), ref['seg_mean']) < 1e-3


def test_ops_match_golden_vectors():
    from thinktwice_b200 import lib
    from thinktwice_b200.lib import MsdaDesc, _p
    from thinktwice_b200.ops.voxel_pooling import voxel_pooling
    o = np.load(os.path.join(G, 'ops.npz'))
    out = voxel_pooling(torch.from_numpy(o['vp_geom']).cuda().contiguous(), torch.from_numpy(o['vp_feats']).cuda().contiguous(),
                        torch.tensor([6, 5, 1]))
    assert rel(out.cpu().numpy(), o['vp_out']) < 1e-5
    # MSDA: the golden stores sampling locations / softmaxed weights; feed offsets = loc - ref with ref = 0 and log-weights
    shapes = [(6, 8), (3, 4), (2, 2), (1, 2)]
    value, loc, aw = (torch.from_numpy(o[k]) for k in ('msda_value', 'msda_loc', 'msda_aw'))
    BN, nq = loc.shape[0], loc.shape[1]
    norm = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float32)
    off = (loc * norm[None, None, None, :, None, :]).reshape(BN * nq, -1).contiguous().cuda()       # ref point = 0
    logits = aw.clamp_min(1e-30).log().reshape(BN * nq, -1).contiguous().cuda()
    d = MsdaDesc()
    d.BN, d.rows_cap, d.heads, d.levels, d.points, d.dh = BN, nq, 8, 4, 8, 32
    d.lvl_h, d.lvl_w = lib.i4([s[0] for s in shapes]), lib.i4([s[1] for s in shapes])
    starts = np.cumsum([0] + [h * w for h, w in shapes])[:4]
    d.lvl_start, d.num_keys = lib.i4(starts), int(sum(h * w for h, w in shapes))
    v = value.reshape(BN, d.num_keys, 256).contiguous().cuda()
    ref_pts = torch.zeros(BN * nq, 2, device='cuda')
    res = torch.zeros(BN * nq, 256, device='cuda')
    ml = torch.tensor([nq], dtype=torch.int32, device='cuda')
    lib.call('tt_msda_forward', C.byref(d), _p(v), _p(off), _p(logits), _p(ref_pts), _p(ml), _p(res))
    assert rel(res.view(BN, nq, 256).cpu().numpy(), o['msda_out']) < 1e-4
