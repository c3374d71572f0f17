"""Generate the committed golden vectors (run once, on CPU):  python tests/golden/make_golden.py

The reference ships no tests or fixtures (SURVEY.md §4), so these vectors are produced by the oracle
(oracle/ = plain-PyTorch restatement of the reference).  They pin (a) the oracle against accidental edits and
(b) the H100 path against a stored answer that does not depend on re-running the oracle.  The end-to-end vectors are
re-derived with the reference's OWN code (same weights loaded into the reference EncoderDecoder behind import stubs) by
tests/test_reference_golden_cpu.py::test_committed_plumbing_golden_is_reproduced_by_the_reference_code; vectors made
directly by the reference's code live beside them as ref_*.npz (make_reference_golden.py).
  plumbing_seed{0,1,2}.npz : end-to-end outputs at the plumbing config (weights/inputs regenerated from the seed)
  ops.npz                  : per-op cases with their INPUTS stored (voxel pool, MSDA, hard voxelisation, sparse conv)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import decoder, lidar, voxel_pool  # noqa: E402
from oracle.model import EncoderDecoder, calibrate_bn, init_oracle_weights  # noqa: E402
from thinktwice_b200.config import Config, PLUMBING_CONFIG  # noqa: E402
from thinktwice_b200.synthetic import make_batch  # noqa: E402

KEYS = ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'pred_value_traj',
        'refine_flattned_BEV_feature')


def plumbing(seed):
    cfg = Config.fromfile(PLUMBING_CONFIG)
    m = EncoderDecoder(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(m, seed)
    batch = make_batch(cfg, 1, seed=seed, num_points=2000)
    calibrate_bn(m, batch)
    keep = {}
    with torch.no_grad():
        pred = m.forward_inference(batch, keep=keep)
    out = {k: pred[k].numpy() for k in KEYS}
    out['cam_bev_sum'] = keep['cam']['bev'].sum((2, 3)).numpy()
    out['lidar_bev_sum'] = keep['lidar'][0].sum((2, 3)).numpy()
    out['seg_mean'] = keep['cam']['seg'].mean((2, 3)).numpy()
    return out


def ops():
    g = torch.Generator().manual_seed(123)
    o = {}
    geom = torch.stack([torch.randint(-2, 8, (2, 300), generator=g), torch.randint(-2, 7, (2, 300), generator=g),
                        torch.randint(-1, 2, (2, 300), generator=g)], -1).int()
    feats = torch.randn(2, 300, 12, generator=g)
    o['vp_geom'], o['vp_feats'] = geom.numpy(), feats.numpy()
    o['vp_out'] = voxel_pool.voxel_pooling_ref(geom, feats, torch.tensor([6, 5, 1])).numpy()
    shapes = [(6, 8), (3, 4), (2, 2), (1, 2)]
    nk = sum(h * w for h, w in shapes)
    value = torch.randn(2, nk, 8, 32, generator=g)
    loc = torch.rand(2, 7, 8, 4, 8, 2, generator=g) * 1.3 - 0.15
    aw = torch.rand(2, 7, 8, 32, generator=g).softmax(-1).view(2, 7, 8, 4, 8)
    o['msda_value'], o['msda_loc'], o['msda_aw'] = value.numpy(), loc.numpy(), aw.numpy()
    o['msda_out'] = decoder.msda_pytorch(value, torch.tensor(shapes), loc, aw).numpy()
    pts = torch.rand(500, 5, generator=g)
    pts[:, :3] = pts[:, :3] * torch.tensor([2.4, 2.4, 1.2]) - 0.2
    pts[:120, :3] = pts[120:240, :3]
    v, c, n = lidar.hard_voxelize(pts, [0.2, 0.2, 0.4], [0.0, 0.0, 0.0, 2.0, 2.0, 0.8], 3, 1000)
    o['vox_pts'], o['vox_coors'], o['vox_num'] = pts.numpy(), c.numpy(), n.numpy()
    o['vox_mean'] = (v.sum(1) / n.float().view(-1, 1)).numpy()
    mask = torch.rand(1, 7, 10, 9, generator=g) < 0.2
    coords = mask.nonzero()
    f = torch.randn(coords.shape[0], 4, generator=g)
    conv = lidar.SparseConvBase(4, 8, 3, stride=2, padding=1)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * 0.2)
        y = conv(lidar.SparseTensor(f, coords, (7, 10, 9), 1))
    o['sp_coords'], o['sp_feats'], o['sp_weight'], o['sp_dense'] = coords.numpy(), f.numpy(), conv.weight.detach().numpy(), y.dense().numpy()
    return o


if __name__ == '__main__':
    for s in (0, 1, 2):
        np.savez_compressed(os.path.join(HERE, f'plumbing_seed{s}.npz'), **plumbing(s))
        print('seed', s, 'done')
    np.savez_compressed(os.path.join(HERE, 'ops.npz'), **ops())
    print('ops done')
