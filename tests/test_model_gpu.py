"""End-to-end parity of the H100 path against the CPU oracle on the same seeded synthetic inputs and weights.

Metric (SURVEY.md §8d): per output tensor max|x - x_ref| / max|x_ref| <= 1e-3 (BASELINE.json north_star: "within
1e-3 relative fp32").  Stage-wise comparisons localise a failure (camera BEV, seg, LiDAR BEV, fusion, decoder)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-3


def relerr(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def build_pair(cfg_path, B, num_points, seed=0, impl=1, refine_num=None):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(cfg_path)
    if refine_num is not None:                                      # BASELINE.json configs[4]: decoder-depth sweep
        for c in (cfg.model.decoder.config, cfg.model.train_cfg, cfg.model.test_cfg):
            c['refine_num'] = refine_num
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, seed)
    batch = make_batch(cfg, B, seed=seed, num_points=num_points)
    calibrate_bn(oracle, batch)
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0', impl=impl)
    return cfg, oracle, model, batch


def compare_all(oracle, model, batch, tol=TOL):
    keep = {}
    with torch.no_grad():
        ref = oracle.forward_inference(batch, keep=keep)
    pred = model.forward_inference(batch)
    torch.cuda.synchronize()
    cam = model.last_cam_feat
    errs = {}
    errs['fpn0'] = relerr(cam['fpn_feats'][0].nchw(), keep['cam']['fpn_feats'][0])
    errs['fpn3'] = relerr(cam['fpn_feats'][3].nchw(), keep['cam']['fpn_feats'][3])
    errs['depth_logits'] = relerr(cam['depth'].nchw(), keep['cam']['depth'])
    errs['seg'] = relerr(cam['seg'].nchw(), keep['cam']['seg'])
    errs['img_feature'] = relerr(cam['img_feature'].nchw(), keep['cam_keep']['img_feature'])
    errs['cam_bev'] = relerr(cam['bev'].nchw(), keep['cam']['bev'])
    errs['lidar_bev'] = relerr(model.eng.static_named('lidar.out.at').permute(0, 3, 1, 2), keep['lidar'][0])
    for k in ('bev_feature', 'pred_speed', 'pred_features_traj', 'pred_wp', 'mu_branches', 'sigma_branches', 'future_mu',
              'future_sigma', 'refine_flattned_BEV_feature', 'refine_BEV_feature', 'refine_future_BEV_feature'):
        errs[k] = relerr(pred[k], ref[k])
    print({k: f'{v:.1e}' for k, v in errs.items()})
    bad = {k: v for k, v in errs.items() if not v <= tol}
    assert not bad, bad
    assert model.f16s_saturations() == 0
    return errs


@pytest.mark.parametrize('impl', [1, 3, 4])
def test_plumbing_config_b1_matches_oracle(impl):
    """impl 1: every contraction on the SIMT fp32 kernel; impl 3: dense convs on tensor-core 3xTF32; impl 4: on tensor-core scaled-split fp16."""
    from thinktwice_b200.config import PLUMBING_CONFIG
    _, oracle, model, batch = build_pair(PLUMBING_CONFIG, 1, 2000, impl=impl)
    compare_all(oracle, model, batch)


def test_plumbing_config_b2_keeps_batch_coupled_look_semantics():
    """fact 4 of SURVEY.md: max_len over the batch, first B rows zeroed, divide by B — same on both sides."""
    from thinktwice_b200.config import PLUMBING_CONFIG
    _, oracle, model, batch = build_pair(PLUMBING_CONFIG, 2, 1500, seed=1, impl=0)
    compare_all(oracle, model, batch)


def test_repeat_forward_is_bitwise_stable_where_deterministic():
    from thinktwice_b200.config import PLUMBING_CONFIG
    _, _, model, batch = build_pair(PLUMBING_CONFIG, 1, 2000)
    a = model.forward_inference(batch)['pred_wp'].clone()
    b = model.forward_inference(batch)['pred_wp'].clone()
    assert float((a - b).abs().max()) < 1e-4 * float(a.abs().max())


@pytest.mark.parametrize('K', [2, 3, 10])
def test_decoder_depth_sweep_matches_oracle(K):
    """BASELINE.json configs[4] (K in {1,2,3,5,10}): K=1 and K=5 are the plumbing / full configs, here K=2,3,10."""
    from thinktwice_b200.config import PLUMBING_CONFIG
    _, oracle, model, batch = build_pair(PLUMBING_CONFIG, 1, 1000, seed=3, impl=0, refine_num=K)
    errs = compare_all(oracle, model, batch)
    assert oracle.decoder.config['refine_num'] == K and len(model.decoder.layers) == K


def test_cuda_graph_replay_equals_eager():
    from thinktwice_b200.config import PLUMBING_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg, _, model, batch = build_pair(PLUMBING_CONFIG, 1, 2000, impl=0)
    eager = {k: model.forward_inference(batch)[k].clone() for k in ('pred_wp', 'mu_branches', 'refine_BEV_feature')}
    model.enable_cuda_graph()
    for _ in range(2):                                              # capture, then a pure replay
        pred = model.forward_inference(batch)
    for k, v in eager.items():                                      # red.add accumulation (sparse convs, split-K) is order-dependent:
        assert relerr(pred[k], v) < 1e-4, k                         # runs agree to amplified fp32 rounding, not bitwise
    other = make_batch(cfg, 1, seed=7, num_points=2000)             # new inputs through the same graph
    p2 = model.forward_inference(other)['pred_wp'].clone()
    model.use_graph = False
    assert relerr(p2, model.forward_inference(other)['pred_wp']) < 1e-4


@pytest.fixture(scope='module')
def full():
    """the thinktwice.py model pair (oracle + product, tensor-core engine), built once for the full-shape tests."""
    from thinktwice_b200.config import DEFAULT_CONFIG
    cfg, oracle, model, batch = build_pair(DEFAULT_CONFIG, 1, 40000, impl=0)   # 0 = the product's default engine
    return dict(cfg=cfg, oracle=oracle, model=model, batch=batch)


def test_full_thinktwice_config_b1_matches_oracle(full):
    """BASELINE.json configs[1]: thinktwice.py, 4 cams x 2 sweeps 448x896 + 40k LiDAR points, K=5, batch 1."""
    full['model'].use_graph = False
    full['errs_b1'] = compare_all(full['oracle'], full['model'], full['batch'])


def test_full_config_graph_replay_matches_oracle_and_eager(full):
    """the BENCHMARKED execution mode (bench.py: CUDA-graph replay, LiDAR encoder on a side stream) at the full shape:
    graph replay vs the oracle (1e-3) and vs the eager launch sequence (red.add accumulation order differs: 1e-4)."""
    model, batch = full['model'], full['batch']
    model.use_graph = False
    eager = {k: model.forward_inference(batch)[k].clone() for k in ('pred_wp', 'mu_branches', 'sigma_branches', 'refine_BEV_feature')}
    model.enable_cuda_graph()
    try:
        for _ in range(3):                                          # warm-up + capture, then pure replays
            model.forward_inference(batch)
        compare_all(full['oracle'], model, batch)                   # forward_inference inside = a graph replay
        pred = model.forward_inference(batch)
        for k, v in eager.items():
            assert relerr(pred[k], v) < 1e-4, k
    finally:
        model.use_graph = False


def test_full_config_b2_with_collate_padding_matches_oracle(full):
    """B = 2 at the full shape (batch-coupled Look semantics, msda:338-342) with unequal clouds: frame 1 has 31k real
    points, zero-padded to 40k the way mmcv's collate pads (SURVEY A9 hazard: the zeros ARE points, they land in one voxel)."""
    from thinktwice_b200.synthetic import make_batch
    batch = make_batch(full['cfg'], 2, seed=11, num_points=40000)
    batch['points'][1, :, 31000:] = 0
    full['model'].use_graph = False
    compare_all(full['oracle'], full['model'], batch)


def test_throughput_config_b16_encoder_is_batch_invariant_and_decoder_matches_oracle(full):
    """BASELINE.json configs[2] (and the per-GPU shard of configs[3]): 16 frames in one forward (what fits an 80 GB GPU).
    The CPU oracle needs ~10 s per frame, so the batch is checked in two parts, both at B = 16:
      * encoder (per-frame independent, SURVEY §8e): frames 0 / 9 / 15 of the B = 16 forward equal the same frames run
        alone (B = 1) — the B = 1 path is the one held to the oracle above;
      * decoder (frames COUPLED through the Look module: batch-wide max_len, first-B-rows / divide-by-B): the oracle's
        decoder is run on the CPU at B = 16 on the product's own encoder outputs and every decoder output compared."""
    from thinktwice_b200.synthetic import make_batch
    cfg, oracle, model = full['cfg'], full['oracle'], full['model']
    model.use_graph = False
    B = 16
    batch = make_batch(cfg, B, seed=21, num_points=40000)
    pred = model.forward_inference(batch)
    torch.cuda.synchronize()
    e = model.eng
    cam = model.last_cam_feat
    keep32 = dict(cam_bev=cam['bev'].nchw().cpu().clone(), seg=cam['seg'].nchw().cpu().clone(),
                  lidar=e.static_named('lidar.out.at').permute(0, 3, 1, 2).cpu().clone())
    fpn = [f.nchw().cpu().clone() for f in cam['fpn_feats']]
    flat = e.static_named('fu.py.flat').view(B, 256).cpu().clone()
    bev32 = e.static_named('fu.m21.out').permute(0, 3, 1, 2).cpu().clone()
    meas = e.static_named('meas').view(B, 128).cpu().clone()
    lidar_hi = keep32['lidar']
    out32 = {k: pred[k].float().cpu().clone() for k in ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed',
                                                        'refine_flattned_BEV_feature', 'refine_BEV_feature')}
    # ---- decoder at B = 16 against the oracle decoder on the same inputs
    lidar2img = torch.stack([m[-1]['lidar2img'] for m in batch['img_metas']], 0).float()
    ida = torch.stack([m[-1]['ida_mats'] for m in batch['img_metas']], 0).float()
    with torch.no_grad():
        ref = oracle.decoder(flat, bev32, meas, oracle, [lidar2img, ida, fpn, lidar_hi], False, None)
    errs = {k: relerr(out32[k], ref[k]) for k in out32}
    print({k: f'{v:.1e}' for k, v in errs.items()})
    assert all(v <= TOL for v in errs.values()), errs
    # ---- encoder: frame j of the batch == frame j alone
    for j in (0, 9, 15):
        one = {k: (v[j:j + 1] if torch.is_tensor(v) else v[j:j + 1]) for k, v in batch.items()}
        model.forward_inference(one)
        torch.cuda.synchronize()
        c1 = model.last_cam_feat
        assert relerr(c1['bev'].nchw(), keep32['cam_bev'][j:j + 1]) < 5e-4, j
        assert relerr(c1['seg'].nchw(), keep32['seg'][j * 4:(j + 1) * 4]) < 5e-4, j
        assert relerr(e.static_named('lidar.out.at').permute(0, 3, 1, 2), keep32['lidar'][j:j + 1]) < 5e-4, j


def test_streaming_bev_cache_equals_the_full_forward_on_a_consecutive_stream():
    """SURVEY §8f f2 (closed loop): the history sweep's BEV is the previous tick's key-frame BEV.  Three consecutive ticks with the
    cache (eager, then as CUDA-graph replays) against full forwards of the same ticks."""
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(PLUMBING_CONFIG)
    cfg.model['img_encoder']['queue_len'] = 2
    cfg.model['train_cfg']['queue_length'] = 2
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, 4)
    ticks = [make_batch(cfg, 1, seed=40 + t, num_points=1500) for t in range(4)]
    for t in range(1, 4):
        ticks[t]['img'][:, 0] = ticks[t - 1]['img'][:, 1]
    calibrate_bn(oracle, ticks[0])
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    full = [{k: model.forward_inference(b)[k].clone() for k in ('pred_wp', 'mu_branches', 'refine_BEV_feature')} for b in ticks]
    for use_graph in (False, True):
        model.enable_streaming_bev_cache()
        if use_graph:
            model.enable_cuda_graph()
        for t, b in enumerate(ticks):
            pred = model.forward_inference(b)
            for k, v in full[t].items():
                assert relerr(pred[k], v) < 1e-4, (use_graph, t, k)
        model.use_graph = False
    assert model.f16s_saturations() == 0


def test_pipelined_host_input_forward_equals_the_single_stream_forward():
    """host-resident batch (the agent / bench e2e case): uploads ordered by first use and overlapped with the kernels on three
    streams (EncoderDecoder._pipelined_forward), eagerly and as three CUDA graphs, against the same batch resident on the device
    run on one stream; different frames on consecutive calls so that a stale input buffer or a missing stream dependency shows."""
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    cfg = Config.fromfile(PLUMBING_CONFIG)
    cfg.model['img_encoder']['queue_len'] = 2
    cfg.model['train_cfg']['queue_length'] = 2
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, 6)
    frames = [make_batch(cfg, 2, seed=60 + t, num_points=1500) for t in range(3)]
    calibrate_bn(oracle, frames[0])
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    keys = ('pred_wp', 'mu_branches', 'refine_BEV_feature', 'pred_speed')
    resident = [{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b.items()} for b in frames]
    want = [{k: model.forward_inference(b)[k].clone() for k in keys} for b in resident]
    assert not any(k[0] == 'pipe' for k in getattr(model, '_graphs', {}))
    pinned = [{k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in b.items()} for b in frames]
    for use_graph in (False, True):
        if use_graph:
            model.enable_cuda_graph()
        for rnd in range(2):
            for t, b in enumerate(pinned):
                pred = model.forward_inference(b)
                for k, v in want[t].items():
                    assert relerr(pred[k], v) < 1e-4, (use_graph, rnd, t, k)
    assert any(k[0] == 'pipe' for k in model._graphs)              # the graph rounds really took the three-graph path
    model.use_graph = False
    assert model.f16s_saturations() == 0
