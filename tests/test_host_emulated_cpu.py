"""The PRODUCT's host code run end to end on the CPU over a torch emulation of the C ABI (tests/emu_lib.py) and compared
with the oracle: weight repacking / BatchNorm folding / concat, scatter and slice layouts / descriptor filling / the forward
orchestration are exercised numerically without a GPU.  (The CUDA kernels are the `-m gpu` suite's job.)"""
import numpy as np
import pytest
import torch


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-12))


def _pair(cfg_path, B, points, seed, impl, sweeps=None):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(cfg_path)
    if sweeps is not None:                                             # plumbing shape with a history sweep (lss.py:710-717)
        cfg.model['img_encoder']['queue_len'] = sweeps
        cfg.model['train_cfg']['queue_length'] = sweeps
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, seed)
    batch = make_batch(cfg, B, seed=seed, num_points=points)
    calibrate_bn(o, batch)
    m = build_model(cfg.model)
    m.load_state_dict(o.state_dict())
    m.prepare('cpu', impl=impl)
    return o, m, batch


@pytest.mark.parametrize('impl,B,seed,sweeps', [(1, 1, 0, None), (3, 1, 0, None), (3, 2, 1, None), (3, 1, 2, 2), (4, 1, 0, None), (4, 2, 1, None), (4, 1, 2, 2)])
def test_plumbing_forward_through_the_emulated_abi_matches_the_oracle(emulated, impl, B, seed, sweeps):
    """impl 1: SIMT weight layouts; impl 3: the tensor-core layouts (hi / lo planes, row-packed stem, padded thin convs, per-group
    DCN GEMMs, sparse-conv planes); B = 2 exercises the batch-coupled Look semantics on the product side; sweeps = 2 the history
    sweep (key-frame matrices, no_grad BEV, sweep merge conv)."""
    from thinktwice_b200.config import PLUMBING_CONFIG
    o, m, batch = _pair(PLUMBING_CONFIG, B, 1500, seed, impl, sweeps)
    keep = {}
    with torch.no_grad():
        ref = o.forward_inference(batch, keep=keep)
    pred = m.forward_inference(batch)
    for k in ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'refine_flattned_BEV_feature'):
        assert rel(pred[k], ref[k]) < 5e-4, k                         # fp32 oracle vs fp64-contraction emulation, amplified ~1e3
    cam = m.last_cam_feat
    assert rel(cam['seg'].nchw(), keep['cam']['seg']) < 5e-4
    assert rel(cam['bev'].nchw(), keep['cam']['bev']) < 5e-4
    assert rel(cam['depth'].nchw().softmax(1), keep['cam_keep']['depth_prob']) < 1e-3


def test_value_proj_layer_by_layer_path_matches_the_merged_one(emulated):
    """the K layers' value_proj run as ONE projection per FPN level when the K-fold value tensor fits the budget (latency configs),
    layer by layer into one reused buffer otherwise (B = 32): both against the oracle."""
    from thinktwice_b200.config import PLUMBING_CONFIG
    o, m, batch = _pair(PLUMBING_CONFIG, 2, 900, 5, 4)
    with torch.no_grad():
        ref = o.forward_inference(batch)
    merged = {k: m.forward_inference(batch)[k].clone() for k in ('pred_wp', 'mu_branches')}
    m.decoder.value_all_budget = 0
    layered = m.forward_inference(batch)
    for k, v in merged.items():
        assert rel(v, ref[k]) < 5e-4 and rel(layered[k], ref[k]) < 5e-4, k


def test_full_thinktwice_config_through_the_emulated_abi_matches_the_oracle(emulated):
    """the bench workload (thinktwice.py: 4 cams x 2 sweeps 448x896, 40k LiDAR points, K = 5, B = 1) with the tensor-core weight
    layouts: ~1000 emulated launches, ~70 s of CPU."""
    from thinktwice_b200.config import DEFAULT_CONFIG
    o, m, batch = _pair(DEFAULT_CONFIG, 1, 40000, 0, 3)
    keep = {}
    with torch.no_grad():
        ref = o.forward_inference(batch, keep=keep)
    pred = m.forward_inference(batch)
    for k in ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'refine_flattned_BEV_feature'):
        assert rel(pred[k], ref[k]) < 5e-4, k
    cam = m.last_cam_feat
    assert rel(cam['seg'].nchw(), keep['cam']['seg']) < 5e-4
    assert rel(cam['bev'].nchw(), keep['cam']['bev']) < 5e-4


@pytest.mark.parametrize('impl', [4, 1])
def test_raw_uint8_frames_through_the_emulated_abi_match_the_preprocessed_tensor(emulated, impl):
    """SURVEY 8f f1 host plumbing on the CPU: a batch carrying `img_raw` (uint8 frames; per-sweep uint8 staging buffers, the pre-processor
    writing the stem's operand planes — impl 4 — or the NCHW tensor the fp32 engines stage themselves — impl 1) against the same model fed
    with the oracle's pre-processed `img`.  Frames of another size than the pre-processor's, and a pre-processor whose final_dim is not
    the model's, are refused with TTError before anything is pre-processed (the f16s stem slots are sized by the model: a mismatch would
    leave stale bytes in them, or write past the planes)."""
    import ctypes as C
    from oracle import preprocess as op
    from thinktwice_b200 import lib
    from thinktwice_b200.config import PLUMBING_CONFIG
    from thinktwice_b200.preprocess import AgentPreprocessor
    o, m, batch = _pair(PLUMBING_CONFIG, 1, 1200, 7, impl, sweeps=2)
    conf = {'final_dim': (256, 256), 'H': 300, 'W': 400, 'bot_pct_lim': (0.0, 0.0)}
    ys, xs = torch.meshgrid(torch.arange(300.), torch.arange(400.), indexing='ij')
    grid = torch.stack([(xs + 2 * torch.sin(ys / 31) - 200) / 200, (ys + 1.5 * torch.cos(xs / 47) - 150) / 150], -1)
    raw = torch.from_numpy(np.random.default_rng(5).integers(0, 256, size=(1, 2, 4, 300, 400, 3), dtype=np.uint8))
    batch['img'] = op.image_normalize(op.ida_image_transform(raw[0], grid, conf)[0])[None]
    want = {k: m.forward_inference(batch)[k].clone() for k in ('pred_wp', 'mu_branches', 'refine_BEV_feature')}
    m.attach_preprocessor(AgentPreprocessor(dict(undistort=True, num_cams=4), conf, 'cpu', map_grid=grid))
    rb = {k: v for k, v in batch.items() if k != 'img'}
    rb['img_raw'] = raw
    got = m.forward_inference(rb)
    for k, v in want.items():
        assert rel(got[k], v) < 1e-5, k
    calls = []
    emu_pre = emulated.tt_preprocess_u8
    emulated.tt_preprocess_u8 = lambda *a: calls.append(a) or emu_pre(*a)
    for h in (200, 400):                                                # fewer bytes than 8 frames / more than the 8 stem slots hold
        bad = dict(rb, img_raw=torch.from_numpy(np.random.default_rng(h).integers(0, 256, size=(1, 2, 4, h, 400, 3), dtype=np.uint8)))
        with pytest.raises(lib.TTError, match='raw frames must be uint8'):
            m.forward_inference(bad)
        assert not calls, h
    pre = m.img_encoder.pre
    with pytest.raises(lib.TTError, match='final_dim'):                 # a 128 x 256 image in a 256 x 256 slot: refused at attach time
        m.attach_preprocessor(AgentPreprocessor(dict(undistort=True, num_cams=4), dict(conf, final_dim=(128, 256)), 'cpu', map_grid=grid))
    assert m.img_encoder.pre is pre
    # the emulated C ABI refuses stem planes one slot short, as the kernel does, and takes them at exactly n slots
    n, pad = 8, (256 + 6, 256 + 8, 3, 3)
    slot = pad[0] * pad[1] * 8
    planes = torch.zeros(2, n * slot, dtype=torch.float16)
    frames = raw.reshape(n, 300, 400, 3).contiguous()
    for cap, rc in ((n * slot - slot, -1), (n * slot, 0)):
        got_rc = emulated.tt_preprocess_u8(C.byref(pre.desc(n, pad)), lib._p(frames), lib._p(pre.grid), lib._p(None), lib._p(planes),
                                           C.c_longlong(cap), None)
        assert got_rc == rc, cap
    assert b'stem-plane capacity' in emulated.tt_last_error()
    with pytest.raises(Exception):                                      # without a pre-processor the raw batch is refused, not guessed at
        m.img_encoder.pre = None
        m.forward_inference(rb)
