"""Agent-side pre-processing on the GPU (SURVEY.md §8f row f1).

The reference agent turns each tick's sensor data into the batch dict on the CPU: four 900 x 1600 uint8 frames per queue entry go
through `IDAImageTransform` (float conversion, `grid_sample` undistortion, `T.Resize`, crop) and `ImageTransformMulti` (/255,
Normalize) — open_loop_training/code/datasets/pipelines/transform.py:275-341, 149-163, called from
leaderboard/team_code/thinktwice_agent.py:445 — and the LiDAR half sweeps are stitched with numpy (thinktwice_agent.py:340-352).
Here both are one kernel each of libtt_b200 (csrc/preprocess.cu): the frames cross PCIe as uint8 and the network input (or directly
the stem convolution's operand planes) is produced on the device.  Same constructor arguments as the reference transform.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import lib
from .lib import _p

# rig constants of the reference pipeline (transform.py:47-51, 144): calibration data, not code
MTX = np.array([[214.35935394, 0, 800], [0, 214.35935394, 450], [0, 0, 1]])
DIST = np.array([[0.00888296, -0.00130899, 0.00012061, -0.00338673, 0.00028834]])
NEWCAMERAMTX = np.array([[304.14395142, 0, 788.25758876], [0, 221.49429321, 449.78972161], [0, 0, 1]])
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def undistort_grid(size=(1600, 900)):
    """the normalised sampling grid of IDAImageTransform.__init__ (transform.py:233-236), (H, W, 2) fp32 on the host."""
    import cv2
    mapx, mapy = cv2.initUndistortRectifyMap(MTX, DIST, None, NEWCAMERAMTX, size, 5)
    return torch.stack([(torch.from_numpy(mapx) - 800) / 800, (torch.from_numpy(mapy) - 450) / 450], dim=-1).contiguous()


def test_time_ida(conf):
    """sample_ida_augmentation with is_train=False (transform.py:264-272): (resize, (newW, newH), crop)."""
    H, W = conf['H'], conf['W']
    fH, fW = conf['final_dim']
    resize = max(fH / H, fW / W)
    newW, newH = int(W * resize), int(H * resize)
    crop_h = int((1 - np.mean(conf['bot_pct_lim'])) * newH) - fH
    crop_w = int(max(0, newW - fW) / 2)
    return resize, (newW, newH), (crop_w, crop_h, crop_w + fW, crop_h + fH)


def obtain_transform_matrix(x, y, yaw):
    """thinktwice_agent.py:47-60 with zero roll / pitch."""
    cy, sy = math.cos(yaw), math.sin(yaw)
    return np.array([[cy, -sy, 0.0, x], [sy, cy, 0.0, y], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]])


def obtain_inv_transform_matrix(x, y, yaw):
    """thinktwice_agent.py:62-90 with zero roll / pitch."""
    cy, sy = math.cos(yaw), math.sin(yaw)
    x, y = -x, -y
    ox, oy = cy * x + sy * y, -sy * x + cy * y                        # InverseRotateVector (roll = pitch = 0)
    return np.array([[cy, sy, 0.0, ox], [-sy, cy, 0.0, oy], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]])


def get_ego_shift(delta_x, delta_y, ego_angle):
    """code/datasets/carla_dataset.py:250-257."""
    length = np.sqrt(delta_x ** 2 + delta_y ** 2)
    bev_angle = ego_angle - np.arctan2(delta_y, delta_x) / np.pi * 180
    return length * np.sin(bev_angle / 180 * np.pi), length * np.cos(bev_angle / 180 * np.pi)


def union_metas(can_bus_list, lidar2cam):
    """The matrix half of `union2one` (code/datasets/carla_dataset.py:261-312): one meta dict per queue entry (oldest first, key frame last)
    with the can_bus deltas, `prev_bev`, `curr2key` and `currlidar2keycam` (host: a handful of 4 x 4 products per tick)."""
    n = len(can_bus_list)
    metas, prev_pos, prev_angle = [], None, None
    for i, cb in enumerate(can_bus_list):
        cb = np.array(cb, dtype=np.float64, copy=True)
        pos, ang = cb[:3].copy(), float(cb[-1])
        if i == 0:
            cb[:3] = 0
            cb[-1] = 0
        else:
            cb[:3] -= prev_pos
            cb[-1] -= prev_angle
        prev_pos, prev_angle = pos, ang
        metas.append({'can_bus': cb, 'prev_bev': i > 0, 'lidar2cam': lidar2cam})
    metas[-1]['curr2key'] = torch.eye(4)
    metas[-1]['currlidar2keycam'] = lidar2cam
    key_x, key_y, key_yaw = can_bus_list[-1][0], can_bus_list[-1][1], can_bus_list[-1][-2]
    for i in range(n - 2, -1, -1):
        sx, sy = get_ego_shift(key_x - can_bus_list[i][0], key_y - can_bus_list[i][1], key_yaw / np.pi * 180)
        ang = key_yaw - can_bus_list[i][-2]
        R = torch.eye(4)
        R[:2, :2] = torch.Tensor([[np.cos(ang), np.sin(ang)], [-np.sin(ang), np.cos(ang)]])
        T = torch.eye(4)
        T[0, 3], T[1, 3] = sx, sy
        metas[i]['curr2key'] = R @ T
        metas[i]['currlidar2keycam'] = lidar2cam @ metas[i]['curr2key']
    return metas


class AgentPreprocessor:
    """GPU stand-in for `IDAImageTransform(cfg, ida_aug_conf, is_train=False)` + `ImageTransformMulti(aug=False)` and the LiDAR
    stitching of the agent's `tick()`.  cfg keys used: 'undistort' (default True), 'num_cams'."""

    def __init__(self, cfg, ida_aug_conf, device='cuda:0', map_grid=None):
        lib.require_cuda(device)
        self.device = torch.device(device)
        self.conf = dict(ida_aug_conf)
        self.undistort = bool(cfg.get('undistort', True))
        self.num_cams = int(cfg.get('num_cams', 4))
        self.H, self.W = int(self.conf['H']), int(self.conf['W'])
        self.fH, self.fW = (int(v) for v in self.conf['final_dim'])
        self.resize, (self.newW, self.newH), self.crop = test_time_ida(self.conf)
        if self.undistort:
            g = map_grid if map_grid is not None else undistort_grid((self.W, self.H))
            assert tuple(g.shape) == (self.H, self.W, 2), g.shape
            self.grid = g.to(self.device, torch.float32).contiguous()
        else:
            self.grid = None
        # what the reference puts into img_metas (transform.py:244, 333-340)
        self.cam_intrinsic = torch.from_numpy(np.stack([(NEWCAMERAMTX if self.undistort else MTX).copy()] * self.num_cams).astype(np.float32))
        m = torch.zeros(4, 4)
        m[0, 0] = m[1, 1] = self.resize
        m[0, 3], m[1, 3] = -float(self.crop[0]), -float(self.crop[1])
        m[2, 2] = m[3, 3] = 1
        self.ida_mat = m                                              # img_transform with flip=False, rotate=0 (transform.py:360-378)

    def desc(self, n_img, pad=None):
        d = lib.PreprocDesc()
        d.n_img, d.H, d.W, d.newH, d.newW, d.outH, d.outW = n_img, self.H, self.W, self.newH, self.newW, self.fH, self.fW
        d.crop_x, d.crop_y, d.undistort, d.div = self.crop[0], self.crop[1], int(self.undistort), 255.0
        d.mean, d.std = lib.f3(MEAN), lib.f3(STD)
        if pad is not None:
            d.pad_H, d.pad_W, d.pad_top, d.pad_left = pad
        return d

    def _raw(self, raw):
        raw = torch.as_tensor(raw)
        if raw.dtype != torch.uint8 or raw.shape[-3:] != (self.H, self.W, 3):
            raise lib.TTError(f'raw frames must be uint8 (..., {self.H}, {self.W}, 3), got {raw.dtype} {tuple(raw.shape)}')
        return raw.to(self.device, non_blocking=True).contiguous()

    def images(self, raw, out=None):
        """raw uint8 (..., H, W, 3) RGB frames (host or device) -> normalised fp32 (..., 3, fH, fW): the batch dict's `img`."""
        raw = self._raw(raw)
        lead = tuple(raw.shape[:-3])
        n = int(np.prod(lead)) if lead else 1
        if out is None:
            out = torch.empty(lead + (3, self.fH, self.fW), dtype=torch.float32, device=self.device)
        assert out.is_contiguous() and out.numel() == n * 3 * self.fH * self.fW and out.dtype == torch.float32
        lib.call('tt_preprocess_u8', C.byref(self.desc(n)), _p(raw), _p(self.grid), _p(out), None, C.c_longlong(0))
        return out

    def images_to_stem(self, raw, planes, plane_halves, pad):
        """raw uint8 device tensor (n, H, W, 3) -> the row-packed stem's operand planes (see tt_image_to_split8); pad = (pad_H, pad_W, top, left).
        Frames of another size are refused (TTError), and so are n slots that do not fit a plane of `plane_halves` halves (the C ABI)."""
        raw = self._raw(raw)
        n = raw.numel() // (self.H * self.W * 3)
        lib.call('tt_preprocess_u8', C.byref(self.desc(n, pad)), _p(raw), _p(self.grid), None, _p(planes), C.c_longlong(plane_halves))

    def ida_mats(self, T):
        return self.ida_mat.expand(T, self.num_cams, 4, 4).clone()

    @staticmethod
    def relative_matrix(pose_prev, pose_now):
        """(x, y, compass) of the previous and the current tick -> now_inv_mat @ prev_matrix (thinktwice_agent.py:343-344, 352)."""
        prev = obtain_transform_matrix(pose_prev[1], -pose_prev[0], pose_prev[2] - np.pi / 2)
        now_inv = obtain_inv_transform_matrix(pose_now[1], -pose_now[0], pose_now[2] - np.pi / 2)
        return np.dot(now_inv, prev)

    def union_points(self, points_list, metas):
        """The point half of `union2one` (carla_dataset.py:314-328): points_list — one (n_i, 4) cloud per queue entry (oldest first, key frame
        last; host or device), metas from union_metas() -> (1, sum n_i, 5) on the device: key frame first with timestamp 0, then the earlier
        frames (newest first) moved by their `curr2key`, timestamp i - (T - 1)."""
        clouds = [torch.as_tensor(p).to(self.device, torch.float32).contiguous() for p in points_list]
        n = len(clouds)
        out = torch.empty(1, sum(c.shape[0] for c in clouds), 5, dtype=torch.float32, device=self.device)
        off = 0
        for i in [n - 1] + list(range(n - 2, -1, -1)):
            mat = None if i == n - 1 else metas[i]['curr2key'].to(self.device, torch.float32).contiguous()
            lib.call('tt_points_union', _p(clouds[i]), clouds[i].shape[0], _p(mat), C.c_float(float(i - (n - 1))), _p(out, off * 5))
            off += clouds[i].shape[0]
        return out

    def stitch_lidar(self, prev, now, rel_mat, z_add=2.5):
        """prev / now: (n, 4) float32 half sweeps (host or device; prev may be None on the first tick) -> (n_prev + n_now, 4) on the device."""
        now = torch.as_tensor(now).to(self.device, torch.float32).contiguous()
        n_prev = 0
        if prev is not None:
            prev = torch.as_tensor(prev).to(self.device, torch.float32).contiguous()
            n_prev = prev.shape[0]
            rel = torch.as_tensor(np.asarray(rel_mat, dtype=np.float64)).to(self.device).contiguous()
        out = torch.empty(n_prev + now.shape[0], 4, dtype=torch.float32, device=self.device)
        lib.call('tt_lidar_stitch', _p(prev) if n_prev else None, n_prev, _p(now), now.shape[0], _p(rel) if n_prev else None,
                 C.c_double(z_add), _p(out))
        return out
