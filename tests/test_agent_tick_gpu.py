"""The closed-loop agent tick at the thinktwice.py shape (SURVEY §8f rows f1 / f2), the way tools/agent_tick.py times it: uint8 900 x 1600
camera frames through tt_preprocess_u8 straight into the stem's split planes (`img.nhwc#s8`), with the pipelined or graph-replayed
forward and the streaming BEV cache on top.

Four consecutive ticks, B = 1: pinned host frames (1, 2, 4, 900, 1600, 3) whose history sweep is the previous tick's key frame (the
agent's queue of two), a static rig (the same img_metas every tick), LiDAR points from make_batch.  The reference run is the product
fed the oracle's pre-processed `img` on the device, eager, cache off; it is held to the oracle stage by stage on ticks 0 and 3.  Every
execution mode of the raw frames must then reproduce it on every tick within 1e-4 (DESIGN §3's bound for graph replay and
re-ordered schedules: red.add accumulation order is the only difference)."""
import numpy as np
import pytest
import torch

from test_model_gpu import compare_all, relerr

pytestmark = pytest.mark.gpu
CONF = {'final_dim': (448, 896), 'H': 900, 'W': 1600, 'bot_pct_lim': (0.0, 0.0)}
KEYS = ('pred_wp', 'mu_branches', 'sigma_branches', 'pred_speed', 'refine_BEV_feature')
TICKS = 4
TOL = 1e-4
PRE_TOL = 2e-6                      # tests/test_preprocess_gpu.py TOL: the kernel's NCHW result against the oracle, relative to max |x|
MODES = {                           # img_raw on the device?, graph replay?, streaming BEV cache?
    'host_eager': (False, False, False),        # the pipelined three-stream forward
    'host_graph': (False, True, False),         # the same as four CUDA graphs
    'cache_eager': (False, False, True),
    'cache_graph': (False, True, True),         # tools/agent_tick.py's streaming line
    'device_graph': (True, True, False),
}


def _on(batch, device):
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in batch.items()}


def _pinned(batch):
    return {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in batch.items()}


@pytest.fixture(scope='module')
def tick():
    from oracle import preprocess as op
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.preprocess import AgentPreprocessor
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    assert tuple(cfg.model['img_encoder']['final_dim']) == CONF['final_dim'] and cfg.model['img_encoder']['queue_len'] == 2
    grid = op.undistort_grid((1600, 900))
    # sweep s of the stream: sweeps[t] / sweeps[t + 1] are tick t's history / key frames
    sweeps = torch.from_numpy(np.random.default_rng(7).integers(0, 256, size=(TICKS + 1, 4, 900, 1600, 3), dtype=np.uint8))
    imgs = op.image_normalize(op.ida_image_transform(sweeps, grid, CONF)[0])          # (TICKS + 1, 4, 3, 448, 896)
    metas = make_batch(cfg, 1, seed=200)['img_metas']
    ticks = []
    for t in range(TICKS):
        b = make_batch(cfg, 1, seed=200 + t, num_points=40000)
        b['img_metas'] = metas                                         # static rig: what the streaming cache relies on
        b['img'] = imgs[t:t + 2][None].clone()
        ticks.append((b, sweeps[t:t + 2][None].clone()))
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, 0)
    calibrate_bn(oracle, ticks[0][0])
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    model.attach_preprocessor(AgentPreprocessor(dict(undistort=True, num_cams=4), CONF, 'cuda:0', map_grid=grid))
    want = []
    for b, _ in ticks:                                                 # the reference run: `img` on the device, eager, cache off
        pred = model.forward_inference(_on(b, 'cuda'))
        want.append({k: pred[k].clone() for k in KEYS})
    assert model.f16s_saturations() == 0
    return dict(cfg=cfg, oracle=oracle, model=model, ticks=ticks, want=want, key_imgs=imgs[1:])


def test_reference_run_matches_the_oracle(tick):
    """ticks 0 and 3 stage by stage against the oracle on the same `img` (1e-3, the north star).  compare_all hands both sides the host
    batch; with the upload pipeline off the product stages it into the same device buffers and runs the one-stream eager forward the
    reference run is."""
    model = tick['model']
    model.pipeline_uploads = False
    try:
        for t in (0, 3):
            errs = compare_all(tick['oracle'], model, tick['ticks'][t][0])
            print(f'tick {t}: worst stage against the oracle {max(errs.values()):.2e} ({max(errs, key=errs.get)})')
    finally:
        del model.pipeline_uploads


def _stem_plane_error(model, key_img):
    """the key sweep's images in `img.nhwc#s8` (the last sweep the forward staged) against the split of the oracle's key-frame images:
    max of |decoded - decoded split(oracle)| / (PRE_TOL * max |oracle| + 2^-21 |v|); <= 1 passes.  Border and pad channels must be +0."""
    from stem_plane_checks import split_h
    n, _, H0, W0 = key_img.shape
    planes = model.eng.static_named('img.nhwc#s8').view(2, n, H0 + 6, W0 + 8, 8)
    dec = (planes[0].double() + planes[1].double() / 2048.0)
    got = dec[:, 3:3 + H0, 3:3 + W0, :3]
    v = key_img.cuda().permute(0, 2, 3, 1)
    hi, lo = split_h(v)
    want = hi.double() + lo.double() / 2048.0
    bound = PRE_TOL * float(v.abs().max()) + 2.0 ** -21 * torch.maximum(got.abs(), want.abs())
    rest = planes.clone()
    rest[:, :, 3:3 + H0, 3:3 + W0, :3] = 0
    assert int((rest.view(torch.int16) != 0).sum()) == 0, 'stem border or pad channels written'
    return float(((got - want).abs() / bound).max())


@pytest.mark.parametrize('mode', list(MODES))
def test_raw_frame_ticks_reproduce_the_reference_run(tick, mode):
    """TICKS consecutive ticks of raw frames in one execution mode against the reference run, tick by tick, within 1e-4 on pred_wp,
    mu / sigma_branches, pred_speed and refine_BEV_feature.  With the streaming cache, ticks 1.. must really be warm (only the key
    frame encoded).  In the eager host mode the stem planes are also checked after every tick against the oracle's key frame."""
    on_device, graph, cache = MODES[mode]
    model = tick['model']
    model.enable_streaming_bev_cache(cache)
    model.enable_cuda_graph(graph)
    worst, plane_worst = {k: 0.0 for k in KEYS}, 0.0
    try:
        for t, (b, raw) in enumerate(tick['ticks']):
            rb = {k: v for k, v in b.items() if k != 'img'}
            rb['img_raw'] = raw
            rb = _on(rb, 'cuda') if on_device else _pinned(rb)
            assert model.img_encoder.cache_ready(1) == (cache and t > 0), (mode, t)       # a silently cold cache cannot pass
            pred = model.forward_inference(rb)
            for k in KEYS:
                worst[k] = max(worst[k], relerr(pred[k], tick['want'][t][k]))
            if mode == 'host_eager':
                torch.cuda.synchronize()
                plane_worst = max(plane_worst, _stem_plane_error(model, tick['key_imgs'][t]))
        if graph:
            assert model._graphs, mode                                  # the ticks after the first really were graph replays
            assert any(k[0] == 'pipe' for k in model._graphs) == (not on_device), mode
    finally:
        model.enable_cuda_graph(False)
        model.enable_streaming_bev_cache(False)
    print(f'{mode}: worst error against the reference run {max(worst.values()):.2e} ({max(worst, key=worst.get)}), bound {TOL}'
          + (f'; stem planes at {plane_worst:.3f} of their bound' if mode == 'host_eager' else ''))
    assert all(v < TOL for v in worst.values()), (mode, worst)
    assert plane_worst <= 1.0
    assert model.f16s_saturations() == 0


def test_two_agents_raw_frames_keep_batch_order(tick):
    """B = 2, two agents' different frames (ticks 1 and 3 of the stream) as raw frames from the host, eager and as graphs (capture, then a
    replay), against the same batch fed as `img` on the device: a b / t / n mix-up in the `in.raw.{t}` staging shows at the full shape."""
    from thinktwice_b200.synthetic import make_batch
    model = tick['model']
    (b1, r1), (b3, r3) = tick['ticks'][1], tick['ticks'][3]
    batch = make_batch(tick['cfg'], 2, seed=300, num_points=40000)
    batch['img'] = torch.cat([b1['img'], b3['img']])
    raw = torch.cat([r1, r3])
    assert not torch.equal(raw[0], raw[1])
    pred = model.forward_inference(_on(batch, 'cuda'))
    want = {k: pred[k].clone() for k in KEYS}
    rb = {k: v for k, v in batch.items() if k != 'img'}
    rb['img_raw'] = raw
    rb = _pinned(rb)
    worst = 0.0
    try:
        for graph, calls in ((False, 1), (True, 2)):
            model.enable_cuda_graph(graph)
            for _ in range(calls):
                pred = model.forward_inference(rb)
                for k in KEYS:
                    err = relerr(pred[k], want[k])
                    worst = max(worst, err)
                    assert err < TOL, (graph, k, err)
    finally:
        model.enable_cuda_graph(False)
    print(f'B = 2 raw frames: worst error against the `img` batch {worst:.2e}, bound {TOL}')
    assert model.f16s_saturations() == 0
