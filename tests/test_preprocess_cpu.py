"""SURVEY §8f row f1 (agent-side pre-processing), CPU side: the oracle restatement against golden vectors produced by the
reference's OWN classes (tests/golden/make_preprocess_golden.py), the product's host-side geometry against the same vectors, and
the kernel's written operation order (a torch restatement of csrc/preprocess.cu) against torch's CPU kernels, bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
CONF = {'resize_lim': (0.56, 0.6255), 'final_dim': (448, 896), 'rot_lim': (0, 0), 'H': 900, 'W': 1600, 'rand_flip': True,
        'bot_pct_lim': (0.0, 0.0)}


@pytest.fixture(scope='module')
def golden():
    return np.load(os.path.join(HERE, 'golden', 'ref_preprocess.npz'))


def test_oracle_reproduces_the_reference_pipeline(golden):
    from make_preprocess_golden import STRIDE, raw_frames
    from oracle import preprocess as op
    grid = op.undistort_grid((1600, 900))
    assert np.array_equal(grid[::50, ::50].numpy(), golden['grid_sub']) and abs(float(grid.double().sum()) - float(golden['grid_sum'])) < 1e-9
    img, ida = op.ida_image_transform(raw_frames(), grid, CONF)
    img = op.image_normalize(img)
    assert tuple(img.shape) == (2, 4, 3, 448, 896)
    assert np.array_equal(img[..., ::STRIDE, ::STRIDE].numpy(), golden['img_sub'])            # same torch kernels underneath: bit-exact
    assert abs(float(img.double().sum()) - float(golden['img_sum'])) <= 1e-9 * float(golden['img_abs_sum'])
    assert np.array_equal(ida.numpy(), golden['ida_mats'])


def test_oracle_stitching_reproduces_the_agent_lines(golden):
    from make_preprocess_golden import lidar_case
    from oracle.preprocess import stitch_lidar
    prev, now, _, _ = lidar_case()
    out = stitch_lidar(prev, now, golden['rel_mat'])
    assert out.dtype == np.float32 and out.shape == (prev.shape[0] + now.shape[0], 4)
    assert np.array_equal(out[::7], golden['stitched_sub']) and float(out.astype(np.float64).sum()) == float(golden['stitched_sum'])
    first = stitch_lidar(None, now, None)
    assert np.array_equal(first[:, 2], (now[:, 2].astype(np.float64) + 2.5).astype(np.float32))


def test_product_host_geometry_matches_the_reference(golden):
    """the rectification map, the test-time resize / crop, the ida matrix, the intrinsics and the relative LiDAR transform the product
    computes on the host (thinktwice_b200/preprocess.py) against what the reference's classes produced."""
    from make_preprocess_golden import lidar_case
    from thinktwice_b200 import preprocess as pp
    g = pp.undistort_grid((1600, 900))
    assert np.array_equal(g[::50, ::50].numpy(), golden['grid_sub']) and abs(float(g.double().sum()) - float(golden['grid_sum'])) < 1e-9
    resize, (newW, newH), crop = pp.test_time_ida(CONF)
    assert (newW, newH, crop) == (896, 504, (0, 56, 896, 504)) and resize == 0.56
    pre = pp.AgentPreprocessor.__new__(pp.AgentPreprocessor)           # host half only (the constructor wants a CUDA device)
    pre.resize, pre.crop, pre.num_cams = resize, crop, 4
    m = torch.zeros(4, 4)
    m[0, 0] = m[1, 1] = resize
    m[0, 3], m[1, 3], m[2, 2], m[3, 3] = -crop[0], -crop[1], 1, 1
    assert np.array_equal(m.expand(2, 4, 4, 4).numpy(), golden['ida_mats'])
    assert np.array_equal(np.stack([pp.NEWCAMERAMTX] * 4).astype(np.float32), golden['cam_intrinsic'])
    _, _, pose_prev, pose_now = lidar_case()
    assert np.array_equal(pp.AgentPreprocessor.relative_matrix(pose_prev, pose_now), golden['rel_mat'])


def kernel_order_restatement(raw, grid, conf, undistort=True):
    """csrc/preprocess.cu's arithmetic, operation for operation (fused multiply-adds written as float64 round trips), in torch."""
    from thinktwice_b200.preprocess import MEAN, STD, test_time_ida
    f32, f64 = torch.float32, torch.float64

    def fma(a, b, c):                                                   # single rounding: exact in float64 for float32 inputs
        return (a.to(f64) * b.to(f64) + c.to(f64)).to(f32)
    n, H, W, _ = raw.shape
    img = raw.to(f32)
    _, (newW, newH), crop = test_time_ida(conf)
    fH, fW = conf['final_dim']

    def U(y, x):                                                        # (n, len(y), len(x), 3) undistorted pixel values
        if not undistort:
            return img[:, y][:, :, x]
        g = grid[y][:, x]
        ix = fma(g[..., 0] + 1, torch.tensor(0.5 * W, dtype=f32), torch.tensor(-0.5, dtype=f32))
        iy = fma(g[..., 1] + 1, torch.tensor(0.5 * H, dtype=f32), torch.tensor(-0.5, dtype=f32))
        fx, fy = ix.floor(), iy.floor()
        w, nn = ix - fx, iy - fy
        e, s = 1 - w, 1 - nn
        out = None
        for t, wt in enumerate((s * e, s * w, nn * e, nn * w)):
            xx, yy = fx.long() + (t & 1), fy.long() + (t >> 1)
            ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
            v = img[:, yy.clamp(0, H - 1), xx.clamp(0, W - 1)] * ok[None, ..., None]
            out = v * wt[None, ..., None] if out is None else fma(v, wt[None, ..., None].expand_as(v), out)
        return out

    def axis(S, newS, off, O):
        o = torch.arange(O, dtype=f32) + off
        sc = torch.tensor(S, dtype=f32) / torch.tensor(newS, dtype=f32)
        f = fma(sc.expand_as(o), o + 0.5, torch.tensor(-0.5, dtype=f32)).clamp_min(0)
        i0 = f.floor().long()
        i1 = i0 + (i0 < S - 1).long()
        l1 = f - i0.to(f32)
        return i0, i1, 1 - l1, l1
    y0, y1, ly0, ly1 = axis(H, newH, crop[1], fH)
    x0, x1, lx0, lx1 = axis(W, newW, crop[0], fW)
    LX0, LX1 = lx0[None, None, :, None], lx1[None, None, :, None]
    LY0, LY1 = ly0[None, :, None, None], ly1[None, :, None, None]
    p00, p01, p10, p11 = U(y0, x0), U(y0, x1), U(y1, x0), U(y1, x1)
    r0 = fma(p00, LX0.expand_as(p00), p01 * LX1)
    r1 = fma(p10, LX0.expand_as(p00), p11 * LX1)
    r = fma(LY0.expand_as(r0), r0, LY1 * r1)
    out = ((r / 255.0) - torch.tensor(MEAN, dtype=f32)) / torch.tensor(STD, dtype=f32)
    return out.permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize('undistort', [True, False])
def test_kernel_operation_order_equals_torch_bit_for_bit(undistort):
    """where the fused multiply-adds sit in ATen's CPU grid_sample / upsample_bilinear2d kernels was determined empirically; this pins the
    restatement the CUDA kernel was written from (small frames, a distortion that leaves the image on two sides)."""
    from oracle import preprocess as op
    conf = dict(CONF, H=90, W=160, final_dim=(44, 88))
    raw = torch.from_numpy(np.random.default_rng(3).integers(0, 256, size=(2, 3, 90, 160, 3), dtype=np.uint8))
    ys, xs = torch.meshgrid(torch.arange(90.), torch.arange(160.), indexing='ij')
    grid = torch.stack([(xs + 3 * torch.sin(ys / 17) + 2.37 - 80) / 80, (ys + 2 * torch.cos(xs / 23) - 1.21 - 45) / 45], -1)
    want, _ = op.ida_image_transform(raw, grid if undistort else None, conf)
    want = op.image_normalize(want).reshape(6, 3, 44, 88)
    got = kernel_order_restatement(raw.reshape(6, 90, 160, 3), grid, conf, undistort)
    assert torch.equal(got, want), float((got - want).abs().max())


def test_stem_plane_checker_rejects_each_corruption():
    """negative controls of tests/stem_plane_checks.py (the full-shape GPU test's judge): planes built here from an independent split
    (the emulated ABI's) pass; a flipped lo' bit in the last image, one written border pixel, a non-zero pad channel and a write into the
    guard gap are each rejected, by the property they break."""
    from emu_lib import _split_f16
    from stem_plane_checks import sentinel_planes, stem_plane_failures
    n, H0, W0 = 3, 5, 7
    pad = (H0 + 3, W0 + 4, 1, 2)
    slot = pad[0] * pad[1] * 8
    split_plane = n * slot + 8 * 5
    v = torch.from_numpy(np.random.default_rng(4).standard_normal((n, 3, H0, W0)).astype(np.float32))
    v[0, 0, 0, 0], v[1, 2, 4, 6] = 1e5, -3e-9                          # saturating and subnormal-lo values
    planes = sentinel_planes(split_plane, 'cpu')
    view = planes.view(2, split_plane)[:, :n * slot].view(2, n, pad[0], pad[1], 8)
    for p, half in enumerate(_split_f16(v.permute(0, 2, 3, 1))):
        view[p, :, 1:1 + H0, 2:2 + W0, :3] = half
        view[p, :, 1:1 + H0, 2:2 + W0, 3:] = 0
    assert stem_plane_failures(planes, split_plane, v, pad) == []

    def corrupted(edit):
        bad = planes.clone()
        edit(bad.view(torch.int16).view(2, split_plane))
        return stem_plane_failures(bad, split_plane, v, pad)

    def flip_lo(b):
        b[1, (n - 1) * slot + ((1 + H0 - 1) * pad[1] + 2 + W0 - 1) * 8 + 2] ^= 1      # last image, last interior pixel, channel 2
    fails = corrupted(flip_lo)
    assert len(fails) == 1 and fails[0].startswith("lo' plane") and '[2, 4, 6, 2]' in fails[0], fails

    def write_border(b):
        b[0, slot + (pad[0] - 1) * pad[1] * 8 + 3] = 0                   # image 1, bottom border row, channel 3
    fails = corrupted(write_border)
    assert len(fails) == 1 and fails[0].startswith('border pixels'), fails

    def pad_channel(b):
        b[0, ((1 + 2) * pad[1] + 2 + 3) * 8 + 5] = 0x3C00                # image 0, interior pixel, channel 5 = 1.0
    fails = corrupted(pad_channel)
    assert len(fails) == 1 and fails[0].startswith('pad channels'), fails

    def gap(b):
        b[1, n * slot + 7] = 0
    fails = corrupted(gap)
    assert len(fails) == 1 and fails[0].startswith('guard gap'), fails


def test_union2one_restatements_match_the_reference_function(golden):
    """carla_dataset.py:250-334 run from its own source text (golden) vs the oracle restatement and vs the product's host half (union_metas)."""
    from make_preprocess_golden import union_case
    from oracle import preprocess as op
    from thinktwice_b200 import preprocess as pp
    can, pts = union_case()
    l2c = torch.from_numpy(op.LIDAR2CAM_ALL.astype(np.float32))
    metas, points = op.union2one(can, l2c, pts)
    assert np.array_equal(points.numpy(), golden['u_points'])
    for got in (metas, pp.union_metas(can, l2c)):
        assert np.array_equal(np.stack([m['curr2key'].numpy() for m in got]), golden['u_curr2key'])
        assert np.array_equal(np.stack([m['currlidar2keycam'].numpy() for m in got]), golden['u_l2kc'])
        assert np.array_equal(np.stack([m['can_bus'] for m in got]), golden['u_can_bus'])
        assert [bool(m['prev_bev']) for m in got] == [bool(v) for v in golden['u_prev_bev']]
