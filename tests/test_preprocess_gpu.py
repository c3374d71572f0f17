"""SURVEY §8f row f1 on the GPU: tt_preprocess_u8 / tt_lidar_stitch through the C ABI against the CPU oracle (oracle/preprocess.py,
pinned to the reference's classes by tests/test_preprocess_cpu.py) and against the committed reference golden vectors; the model fed
with raw uint8 frames against the model fed with the oracle's pre-processed tensor."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
CONF = {'resize_lim': (0.56, 0.6255), 'final_dim': (448, 896), 'rot_lim': (0, 0), 'H': 900, 'W': 1600, 'rand_flip': True,
        'bot_pct_lim': (0.0, 0.0)}
TOL = 2e-6            # fp32: the kernel follows torch's operation order; a few ulp of slack for the byte -> float products


def test_full_size_tick_matches_the_oracle_and_the_reference_golden():
    from make_preprocess_golden import STRIDE, raw_frames
    from oracle import preprocess as op
    from thinktwice_b200.preprocess import AgentPreprocessor
    raw = raw_frames()
    pre = AgentPreprocessor(dict(undistort=True, num_cams=4), CONF, 'cuda:0')
    got = pre.images(raw).cpu()
    want, ida = op.ida_image_transform(raw, op.undistort_grid((1600, 900)), CONF)
    want = op.image_normalize(want)
    assert got.shape == want.shape == (2, 4, 3, 448, 896)
    assert float((got - want).abs().max()) <= TOL * float(want.abs().max())
    golden = np.load(os.path.join(HERE, 'golden', 'ref_preprocess.npz'))
    assert float(np.abs(got[..., ::STRIDE, ::STRIDE].numpy() - golden['img_sub']).max()) <= TOL * float(np.abs(golden['img_sub']).max())
    assert np.array_equal(pre.ida_mats(2).numpy(), golden['ida_mats']) and np.array_equal(pre.cam_intrinsic.numpy(), golden['cam_intrinsic'])


@pytest.mark.parametrize('undistort', [True, False])
def test_small_frames_edges_and_stem_planes(undistort):
    """a distortion map that leaves the frame on two sides (zero padding of grid_sample), odd sizes, and the direct stem-plane output:
    hi + lo / 2048 reproduces the fp32 result to 2^-21, the zero border is never written."""
    from oracle import preprocess as op
    from thinktwice_b200 import lib
    from thinktwice_b200.preprocess import AgentPreprocessor
    import ctypes as C
    conf = dict(CONF, H=90, W=160, final_dim=(44, 88))
    raw = torch.from_numpy(np.random.default_rng(3).integers(0, 256, size=(3, 2, 90, 160, 3), dtype=np.uint8))
    ys, xs = torch.meshgrid(torch.arange(90.), torch.arange(160.), indexing='ij')
    grid = torch.stack([(xs + 3 * torch.sin(ys / 17) + 2.37 - 80) / 80, (ys + 2 * torch.cos(xs / 23) - 1.21 - 45) / 45], -1)
    pre = AgentPreprocessor(dict(undistort=undistort, num_cams=2), conf, 'cuda:0', map_grid=grid)
    want, _ = op.ida_image_transform(raw, grid if undistort else None, conf)
    want = op.image_normalize(want)
    got = pre.images(raw.cuda()).cpu()
    assert float((got - want).abs().max()) <= TOL * float(want.abs().max())
    n, H0, W0 = 6, 44, 88
    padH, padW = H0 + 6, W0 + 8
    planes = torch.full((2, n * padH * padW * 8), 7.0, dtype=torch.float16, device='cuda')
    planes.zero_()
    pre.images_to_stem(raw.cuda().reshape(n, 90, 160, 3), planes, planes.numel() // 2, (padH, padW, 3, 3))
    torch.cuda.synchronize()
    hi, lo = planes[0].float().view(n, padH, padW, 8).cpu(), planes[1].float().view(n, padH, padW, 8).cpu()
    rebuilt = (hi + lo / 2048.0)[:, 3:3 + H0, 3:3 + W0, :3].permute(0, 3, 1, 2)
    assert float((rebuilt - want.reshape(n, 3, H0, W0)).abs().max()) <= 2.0 ** -20 * float(want.abs().max())
    border = (hi + lo / 2048.0).clone()
    border[:, 3:3 + H0, 3:3 + W0, :3] = 0
    assert float(border.abs().max()) == 0.0                             # border pixels and the 5 padding channels stay zero
    # argument checking: a crop window outside the resized frame is refused, not clamped
    d = pre.desc(n)
    d.crop_y = 10 ** 6
    rc = lib.load().tt_preprocess_u8(C.byref(d), lib._p(raw.cuda()), lib._p(pre.grid), lib._p(got.cuda()), None, C.c_longlong(0), lib._stream())
    assert rc == -1 and b'crop' in lib.load().tt_last_error()


def agent_frames(n, seed):
    """n random 900 x 1600 frames, with whole frames and blocks at 0 and 255: frame 0 black, frame n - 1 white, frame 1 with saturated
    corner blocks on the frame's edges, frame n - 2 a white block holding a black one (sharp 0 / 255 edges inside the crop)."""
    raw = np.random.default_rng(seed).integers(0, 256, size=(n, 900, 1600, 3), dtype=np.uint8)
    raw[0], raw[n - 1] = 0, 255
    raw[1, :300, :500], raw[1, 600:, 1100:] = 0, 255
    raw[n - 2, 200:700, 400:1200] = 255
    raw[n - 2, 350:550, 700:900] = 0
    return torch.from_numpy(raw)


@pytest.mark.parametrize('n', [8, 128])
def test_stem_planes_at_the_agent_shape(n):
    """the mode the f16s forward uses (`img.nhwc#s8`) at thinktwice.py's geometry — real rectification map, 900 x 1600 -> resize 0.56 ->
    crop 448 x 896, stem slot 454 x 904 x 8 — for n = 8 images (B = 1 x 2 sweeps x 4 cams) and n = 128 (B = 16).  One call writes both
    outputs into planes pre-filled with a sentinel, with a guard gap after the last slot of each plane: hi / lo' are bitwise split_h of
    the NCHW value the same call wrote, the pad channels +0, every border pixel and the gap untouched; the NCHW result is within TOL of
    the oracle on all n images.  A plane capacity one slot short is refused before any launch."""
    import ctypes as C
    import time
    from oracle import preprocess as op
    from stem_plane_checks import sentinel_planes, stem_plane_failures
    from thinktwice_b200 import lib
    from thinktwice_b200.preprocess import AgentPreprocessor
    raw = agent_frames(n, 100 + n)
    grid = op.undistort_grid((1600, 900))
    pre = AgentPreprocessor(dict(undistort=True, num_cams=4), CONF, 'cuda:0', map_grid=grid)
    H0, W0 = CONF['final_dim']
    pad = (H0 + 6, W0 + 8, 3, 3)                                        # lss.py _single_sweep: 3 px top / bottom / left, 5 right
    slot = pad[0] * pad[1] * 8
    split_plane = n * slot + 8 * 4096                                   # guard gap: 4096 pixels after the last slot of each plane
    planes = sentinel_planes(split_plane, 'cuda')
    nchw = torch.empty(n, 3, H0, W0, device='cuda')
    dev = raw.cuda()
    lib.call('tt_preprocess_u8', C.byref(pre.desc(n, pad)), lib._p(dev), lib._p(pre.grid), lib._p(nchw), lib._p(planes), C.c_longlong(split_plane))
    torch.cuda.synchronize()
    bad = stem_plane_failures(planes, split_plane, nchw, pad)
    assert not bad, bad
    t0 = time.perf_counter()
    got, vmax, err = nchw.cpu(), 0.0, 0.0
    for i in range(0, n, 16):                                           # the oracle in chunks of 16 frames: bounded host memory
        want = op.image_normalize(op.ida_image_transform(raw[None, i:i + 16], grid, CONF)[0])[0]
        vmax, err = max(vmax, float(want.abs().max())), max(err, float((got[i:i + 16] - want).abs().max()))
    print(f'n = {n}: NCHW max error {err:.3g} = {err / vmax:.3g} of max |oracle| (bound {TOL}); oracle on the CPU {time.perf_counter() - t0:.1f} s')
    assert err <= TOL * vmax
    # argument checking: planes one slot short of n slots are refused before any launch (and the planes stay as the first call left them)
    launches = lib.launch_count()
    rc = lib.load().tt_preprocess_u8(C.byref(pre.desc(n, pad)), lib._p(dev), lib._p(pre.grid), None, lib._p(planes), C.c_longlong(n * slot - slot),
                                     lib._stream())
    assert rc == -1 and b'stem-plane capacity' in lib.load().tt_last_error()
    torch.cuda.synchronize()
    assert lib.launch_count() == launches
    assert not stem_plane_failures(planes, split_plane, nchw, pad)


def test_lidar_stitch_matches_the_agent_arithmetic():
    from make_preprocess_golden import lidar_case
    from oracle.preprocess import stitch_lidar
    from thinktwice_b200.preprocess import AgentPreprocessor
    prev, now, pose_prev, pose_now = lidar_case()
    rel = AgentPreprocessor.relative_matrix(pose_prev, pose_now)
    pre = AgentPreprocessor(dict(undistort=False, num_cams=1), dict(CONF, H=8, W=8, final_dim=(4, 4)), 'cuda:0')
    got = pre.stitch_lidar(prev, now, rel).cpu().numpy()
    want = stitch_lidar(prev, now, rel)
    golden = np.load(os.path.join(HERE, 'golden', 'ref_preprocess.npz'))
    assert got.shape == want.shape
    # float64 accumulation on both sides, rounded to float32 once: at most one float32 ulp where numpy's einsum sums in another order
    assert np.all(np.abs(got - want) <= np.spacing(np.abs(want)))
    assert np.mean(got != want) < 1e-3
    assert np.all(np.abs(got[::7] - golden['stitched_sub']) <= np.spacing(np.abs(golden['stitched_sub'])))
    first = pre.stitch_lidar(None, now, None).cpu().numpy()
    assert np.array_equal(first, stitch_lidar(None, now, None))


def test_model_fed_with_raw_frames_equals_model_fed_with_the_preprocessed_tensor():
    """forward_inference(batch with `img_raw`) — uint8 frames uploaded, undistort / resize / crop / normalise fused into the stem's input
    staging — against forward_inference(batch with `img` = the oracle's pre-processed tensor); host inputs, eager and CUDA-graph modes."""
    from oracle import preprocess as op
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.preprocess import AgentPreprocessor
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(PLUMBING_CONFIG)
    cfg.model['img_encoder']['queue_len'] = 2
    cfg.model['train_cfg']['queue_length'] = 2
    fH, fW = cfg.model['img_encoder']['final_dim']
    N = cfg.model['num_cams']
    conf = dict(CONF, H=300, W=400, final_dim=(fH, fW))
    ys, xs = torch.meshgrid(torch.arange(300.), torch.arange(400.), indexing='ij')
    grid = torch.stack([(xs + 2 * torch.sin(ys / 31) - 200) / 200, (ys + 1.5 * torch.cos(xs / 47) - 150) / 150], -1)
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, 8)
    batches = []
    for t in range(2):
        b = make_batch(cfg, 2, seed=80 + t, num_points=1500)
        raw = torch.from_numpy(np.random.default_rng(90 + t).integers(0, 256, size=(2, 2, N, 300, 400, 3), dtype=np.uint8))
        img = torch.stack([op.image_normalize(op.ida_image_transform(raw[i], grid, conf)[0]) for i in range(2)])
        assert img.shape == b['img'].shape
        b['img'] = img
        batches.append((b, raw))
    calibrate_bn(oracle, batches[0][0])
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    model.attach_preprocessor(AgentPreprocessor(dict(undistort=True, num_cams=N), conf, 'cuda:0', map_grid=grid))
    keys = ('pred_wp', 'mu_branches', 'refine_BEV_feature')
    want = [{k: model.forward_inference(b)[k].clone() for k in keys} for b, _ in batches]
    for use_graph in (False, True):
        if use_graph:
            model.enable_cuda_graph()
        for i, (b, raw) in enumerate(batches):
            rb = {k: v for k, v in b.items() if k != 'img'}
            rb['img_raw'] = raw.pin_memory()
            pred = model.forward_inference(rb)
            for k in keys:
                err = float((pred[k] - want[i][k]).abs().max() / want[i][k].abs().max())
                assert err < 1e-4, (use_graph, i, k, err)
    model.use_graph = False
    assert model.f16s_saturations() == 0


def test_union_points_matches_the_reference_union2one():
    """carla_dataset.py:314-328 on the device against the golden output of the reference's own function."""
    from make_preprocess_golden import union_case
    from oracle.preprocess import LIDAR2CAM_ALL
    from thinktwice_b200.preprocess import AgentPreprocessor, union_metas
    can, pts = union_case()
    metas = union_metas(can, torch.from_numpy(LIDAR2CAM_ALL.astype(np.float32)))
    pre = AgentPreprocessor(dict(undistort=False, num_cams=1), dict(CONF, H=8, W=8, final_dim=(4, 4)), 'cuda:0')
    got = pre.union_points(pts, metas).cpu().numpy()
    golden = np.load(os.path.join(HERE, 'golden', 'ref_preprocess.npz'))['u_points']
    assert got.shape == golden.shape
    assert np.array_equal(got[..., 4], golden[..., 4]) and np.array_equal(got[0, :pts[1].shape[0], :4], pts[1].numpy())
    assert float(np.abs(got - golden).max()) <= 1e-5 * float(np.abs(golden).max())     # fp32 4-term dot products: order of summation only
