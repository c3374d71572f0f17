"""Seeded synthetic batch in the reference's input contract (SURVEY.md §8b "Batch dict in", §8d).

The rig constants are the CARLA camera rig the reference hard-codes as data in
open_loop_training/code/datasets/pipelines/transform.py:25-51 (LIDAR2CAM, UNDISTORT_LIDAR2IMG,
newcameramtx); camera order is thinktwice.py:102.  The ida matrix is the test-time branch of
`sample_ida_augmentation` / `img_transform` (transform.py:264-272, 346-378) for 900x1600 -> final_dim.
"""
import numpy as np
import torch

CAMERAS = ('rgb_front', 'rgb_left', 'rgb_right', 'rgb_back')

LIDAR2CAM = {
    'rgb_front': [[0.0, 1.0, 0.0, 0.0], [0.0, 0.0, -1.0, 2.5], [1.0, 0.0, 0.0, -1.5], [0.0, 0.0, 0.0, 1.0]],
    'rgb_back': [[0.0, -1.0, 0.0, 0.0], [0.0, 0.0, -1.0, 2.5], [-1.0, 0.0, 0.0, -1.6], [0.0, 0.0, 0.0, 1.0]],
    'rgb_left': [[1.0, 0.0, 0.0, 0.0], [0.0, 0.0, -1.0, 2.5], [0.0, -1.0, 0.0, -0.3], [0.0, 0.0, 0.0, 1.0]],
    'rgb_right': [[-1.0, 0.0, 0.0, 0.0], [0.0, 0.0, -1.0, 2.5], [0.0, 1.0, 0.0, -0.3], [0.0, 0.0, 0.0, 1.0]],
}
UNDISTORT_LIDAR2IMG = {
    'rgb_front': [[788.25758876, 304.14395142, 0.0, -1182.38638314], [449.78972161, 0.0, -221.49429321, -120.94884939000008],
                  [1.0, 0.0, 0.0, -1.5], [0.0, 0.0, 0.0, 1.0]],
    'rgb_left': [[304.14395142, -788.25758876, 0.0, -236.47727662799997], [0.0, -449.78972161, -221.49429321, 418.79881654199994],
                 [0.0, -1.0, 0.0, -0.3], [0.0, 0.0, 0.0, 1.0]],
    'rgb_right': [[-304.14395142, 788.25758876, 0.0, -236.47727662799997], [0.0, 449.78972161, -221.49429321, 418.79881654199994],
                  [0.0, 1.0, 0.0, -0.3], [0.0, 0.0, 0.0, 1.0]],
    'rgb_back': [[-788.25758876, -304.14395142, 0.0, -1261.2121420160001], [-449.78972161, 0.0, -221.49429321, -165.9278215510001],
                 [-1.0, 0.0, 0.0, -1.6], [0.0, 0.0, 0.0, 1.0]],
}
NEW_CAMERA_MTX = [[304.14395142, 0.0, 788.25758876], [0.0, 221.49429321, 449.78972161], [0.0, 0.0, 1.0]]
SRC_H, SRC_W = 900, 1600


def test_time_ida(final_dim):
    """4x4 image-data-augmentation matrix of the evaluation branch (no flip / rotate)."""
    fH, fW = final_dim
    resize = max(fH / SRC_H, fW / SRC_W)
    newW, newH = int(SRC_W * resize), int(SRC_H * resize)
    crop_h = int(newH) - fH
    crop_w = int(max(0, newW - fW) / 2)
    m = torch.eye(4)
    m[0, 0] = m[1, 1] = resize
    m[0, 3] = -float(crop_w)
    m[1, 3] = -float(crop_h)
    return m


def rig_metas(final_dim, num_sweeps):
    """img_metas for one sample: list[T] of dicts with the keys LSS.forward reads (lss.py:668-680,705)."""
    n = len(CAMERAS)
    intr = torch.tensor([NEW_CAMERA_MTX] * n, dtype=torch.float32)
    l2c = torch.tensor([LIDAR2CAM[c] for c in CAMERAS], dtype=torch.float32)
    l2i = torch.tensor(np.array([UNDISTORT_LIDAR2IMG[c] for c in CAMERAS]).astype(np.float32))
    ida = test_time_ida(final_dim)[None].repeat(n, 1, 1)
    return [dict(cam_intrinsic=intr.clone(), ida_mats=ida.clone(), lidar2cam=l2c.clone(), lidar2img=l2i.clone(),
                 currlidar2keycam=l2c.clone()) for _ in range(num_sweeps)]


def make_batch(cfg, batch_size=1, seed=0, num_points=40000, device='cpu'):
    """Batch dict for `EncoderDecoder.forward_inference` (framework:194-206); one generator per frame,
    seed = 1000*seed + frame, so frame j of any batch size is the same tensor."""
    tcfg = cfg.model.train_cfg
    H, W = tcfg['img_size']
    T = tcfg['queue_length']
    n = len(CAMERAS)
    lo = cfg.point_cloud_range[:3]
    hi = [cfg.point_cloud_range[3], cfg.point_cloud_range[4], 4.2]      # z < 4.2: inside sparse_shape z=41 (SURVEY A9)
    imgs, pts, speed, tp, cmd = [], [], [], [], []
    for j in range(batch_size):
        g = torch.Generator().manual_seed(1000 * seed + j)
        imgs.append(torch.randn(T, n, 3, H, W, generator=g))
        u = torch.rand(num_points, 3, generator=g)
        xyz = torch.stack([lo[i] + (hi[i] - lo[i]) * u[:, i] for i in range(3)], 1)
        ground = torch.rand(num_points, generator=g) < 0.7
        xyz[:, 2] = torch.where(ground, 0.05 * torch.randn(num_points, generator=g), xyz[:, 2])
        inten = torch.rand(num_points, 1, generator=g)
        ts = -(torch.rand(num_points, 1, generator=g) < 0.5).float()
        pts.append(torch.cat([xyz, inten, ts], 1)[None])
        speed.append(8.0 * torch.rand(1, generator=g))
        tp.append(10.0 * torch.randn(2, generator=g))
        c = int(torch.randint(0, 6, (1,), generator=g))
        cmd.append(torch.nn.functional.one_hot(torch.tensor(c), 6).float())
    batch = dict(
        img=torch.stack(imgs).to(device),
        img_metas=[rig_metas((H, W), T) for _ in range(batch_size)],
        points=torch.stack(pts).to(device),
        speed=torch.cat(speed).to(device),
        target_point=torch.stack(tp).to(device),
        target_command=torch.stack(cmd).to(device),
    )
    batch['target_command_raw'] = batch['target_command'].argmax(-1)
    return batch


def make_supervision(cfg, batch_size=1, seed=0, device='cpu'):
    """Seeded ground truth in the reference's training-batch contract (the keys ThinkTwiceDecoder.loss and the teacher-forced pass
    read, thinktwice_decoder.py:496-619): waypoints (B, T, 2); Beta parameters action_mu / action_sigma (B, 2) and T future ones
    (lists of (B, 2)), drawn from U(0.5, 20) independently of any prediction so that no loss term is near zero; value (B,); the
    flattened feature (B, 256); the BEV pyramid targets grid_feature = [None, None, 32x21x21, 64x10x10, 128x4x4, 256x2x2] and T
    future 21x21 targets future_grid_feature[t] = [None, None, 32x21x21].  One generator per frame, as make_batch."""
    T = cfg.model.train_cfg['pred_len']
    shapes = {2: (32, 21, 21), 3: (64, 10, 10), 4: (128, 4, 4), 5: (256, 2, 2)}
    frames = []
    for j in range(batch_size):
        g = torch.Generator().manual_seed(5000 + 1000 * seed + j)
        beta = lambda *s: 0.5 + 19.5 * torch.rand(*s, generator=g)
        f = dict(waypoints=torch.cumsum(torch.stack([1.0 + 2.0 * torch.rand(T, generator=g), 0.5 * torch.randn(T, generator=g)], -1), 0),
                 action_mu=beta(2), action_sigma=beta(2), future_action_mu=beta(T, 2), future_action_sigma=beta(T, 2),
                 value=torch.randn(1, generator=g), feature=torch.rand(256, generator=g))
        for i, s in shapes.items():
            f[f'grid{i}'] = 2.0 * torch.rand(*s, generator=g)
        f['future_grid'] = 2.0 * torch.rand(T, *shapes[2], generator=g)
        frames.append(f)
    st = lambda k: torch.stack([f[k] for f in frames]).to(device)
    grid = [None, None] + [st(f'grid{i}') for i in shapes]
    fut = st('future_grid')
    return dict(waypoints=st('waypoints'), action_mu=st('action_mu'), action_sigma=st('action_sigma'),
                future_action_mu=list(st('future_action_mu').unbind(1)), future_action_sigma=list(st('future_action_sigma').unbind(1)),
                value=st('value').view(-1), feature=st('feature'), grid_feature=grid,
                future_grid_feature=[[None, None, fut[:, t]] for t in range(T)])


def make_camera_supervision(cfg, batch_size=1, seed=0, device='cpu'):
    """Seeded ground truth of the camera branch's supervision (encoder_decoder_framework.py:171-190): depth and seg, (B, N, H, W) fp32 at the
    image size.  Depth: dense over the d_bound range and beyond, about 30 % zero pixels (no measurement), in camera 0 one all-zero block,
    one block holding a NaN, and blocks whose minimum lies exactly on the bin value v = (d - (d_bound[0] - d_bound[2])) / d_bound[2]
    = 0, 1, 2, D, D + 1 or just below 1 and D + 1.  Seg: labels of the C classes as the data pipeline's grid-sample leaves them, with
    fractional parts (some just below the next integer) and about 10 % ignored pixels (255, some 255.5).  One generator per frame."""
    tcfg, enc = cfg.model.train_cfg, cfg.model.img_encoder
    H, W = tcfg['img_size']
    n = len(CAMERAS)
    d0, d1, step = (float(v) for v in enc['d_bound'])
    D = int((d1 - d0) / step)
    f = int(cfg.model.get('downsample_factor', 16))
    C = int(enc['seg_net_conf']['out_channels'])
    edges = [0.0, 1.0, 2.0, float(D), float(D + 1), 1.0 - 2.0 ** -10, D + 1 - 2.0 ** -10]
    depth, seg = [], []
    for j in range(batch_size):
        g = torch.Generator().manual_seed(9000 + 1000 * seed + j)
        d = (d0 - 2 * step) + (d1 - d0 + 8 * step) * torch.rand(n, H, W, generator=g)
        d[torch.rand(n, H, W, generator=g) < 0.3] = 0.0
        d[0, :f, :f] = 0.0                                        # a block with no measurement: background
        d[0, :f, f:2 * f] = 0.5 * (d0 + d1)
        d[0, 3, f + 5] = float('nan')                              # torch.min propagates it: background
        for k, v in enumerate(edges):                              # minimum exactly on a bin value
            blk = d[0, f:2 * f, k * f:(k + 1) * f]
            blk.copy_(d1 + 4 * step + torch.rand(f, f, generator=g))
            blk[int(torch.randint(0, f, (1,), generator=g)), int(torch.randint(0, f, (1,), generator=g))] = (d0 - step) + v * step
        depth.append(d)
        lab = torch.randint(0, C, (n, H, W), generator=g).float() + 0.999 * torch.rand(n, H, W, generator=g)
        below = torch.rand(n, H, W, generator=g) < 0.05
        lab = torch.where(below, lab.floor() + (1 - 2.0 ** -10), lab)           # just below the next integer: still truncates down
        ign = torch.rand(n, H, W, generator=g)
        lab = torch.where(ign < 0.1, torch.full_like(lab, 255.0), lab)
        lab = torch.where(ign < 0.02, torch.full_like(lab, 255.5), lab)
        seg.append(lab)
    return dict(depth=torch.stack(depth).to(device), seg=torch.stack(seg).to(device))
