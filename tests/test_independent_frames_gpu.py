"""Independent-frames mode on the H100: the two per-frame Look entry points (tt_msda_forward_frames, tt_look_reduce_frames)
against float64 references, and the whole model at the thinktwice.py shape, where frame j of an independent-mode batch of 16
must equal frame j run alone at B = 1."""
import pytest
import torch

pytestmark = pytest.mark.gpu

KEYS = ('pred_wp', 'mu_branches', 'sigma_branches', 'future_mu', 'future_sigma', 'pred_speed', 'refine_flattned_BEV_feature',
        'refine_BEV_feature', 'refine_future_BEV_feature')
# frame j in a batch of 16 against frame j alone: the same kernels, only the tile and split-K choices that depend on the row count
# differ (fp32 summation order), amplified through the K = 5 cascade
FRAME_TOL = 1e-4
ORACLE_TOL = 1e-3


def relerr(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def frame_errs(batched, alone, keys=KEYS):
    """{key: max over frames j of |batched[j] - alone[j]|, relative to the output's largest magnitude over the frames}"""
    out = {}
    for k in keys:
        scale = max(float(a[k].abs().max()) for a in alone) + 1e-12
        out[k] = max(float((batched[k][j:j + 1].double().cpu() - a[k].double().cpu()).abs().max()) for j, a in enumerate(alone)) / scale
    return out


# ------------------------------------------------------------------ kernel level
def _msda_problem(counts, cap=120, seed=0):
    from thinktwice_b200 import lib
    g = torch.Generator().manual_seed(seed)
    B, cams = counts.shape
    BN, heads, L, P, dh = B * cams, 8, 4, 8, 32
    shapes = [(28, 56), (14, 28), (7, 14), (4, 7)]
    nk = sum(h * w for h, w in shapes)
    value = torch.randn(BN, nk, heads * dh, generator=g)
    off = torch.randn(BN, cap, heads * L * P * 2, generator=g) * 3
    logits = torch.randn(BN, cap, heads * L * P, generator=g)
    ref = torch.rand(BN, cap, 2, generator=g) * 1.2 - 0.1
    ml = counts.amax(1)
    for b in range(B):                                                 # rows at or past max_len_b: NaN, so a read past the bound shows
        for t in (off, logits, ref):
            t[b * cams:(b + 1) * cams, int(ml[b]):] = float('nan')
    d = lib.MsdaDesc()
    d.BN, d.rows_cap, d.heads, d.levels, d.points, d.dh = BN, cap, heads, L, P, dh
    d.lvl_h, d.lvl_w = lib.i4([h for h, _ in shapes]), lib.i4([w for _, w in shapes])
    starts, acc = [], 0
    for h, w in shapes:
        starts.append(acc); acc += h * w
    d.lvl_start, d.num_keys = lib.i4(starts), nk
    return d, shapes, value, off, logits, ref, ml


# frame 0 reaches the cap (120), the others have different max_len_b, frame 2 has none, frame 3 one row (row 0 only)
COUNTS = torch.tensor([[120, 3, 50, 0], [10, 37, 5, 7], [0, 0, 0, 0], [1, 0, 1, 1], [64, 64, 63, 2]], dtype=torch.int32)


def test_msda_forward_frames_matches_fp64_and_the_coupled_entry():
    from oracle.decoder import msda_pytorch
    from thinktwice_b200 import lib
    counts = COUNTS
    B, cams = counts.shape
    d, shapes, value, off, logits, ref, ml = _msda_problem(counts)
    BN, cap = d.BN, d.rows_cap
    dev = [t.cuda() for t in (value, off, logits, ref)]
    sentinel = 12345.0
    out = torch.full((BN, cap, 256), sentinel, device='cuda')
    lib.call('tt_msda_forward_frames', lib.ref(d), *[lib._p(t) for t in dev], lib._p(counts.cuda()), cams, lib._p(out))
    # the coupled entry with the batch-wide max_len on the same inputs computes every row up to 120 (NaN past the frames' bounds)
    out_c = torch.full_like(out, sentinel)
    lib.call('tt_msda_forward', lib.ref(d), *[lib._p(t) for t in dev], lib._p(counts.max().view(1).int().cuda()), lib._p(out_c))
    torch.cuda.synchronize()
    out, out_c = out.cpu(), out_c.cpu()
    # float64 reference (mmcv's pure-torch formulation) on the rows below the bounds (the NaN rows zeroed: not compared)
    ref, off, logits = (torch.nan_to_num(t.double()) for t in (ref, off, logits))
    loc = ref.view(BN, cap, 1, 1, 1, 2) + off.view(BN, cap, 8, 4, 8, 2) / torch.tensor(
        [[w, h] for h, w in shapes], dtype=torch.float64)[None, None, None, :, None, :]
    aw = logits.view(BN, cap, 8, 32).softmax(-1).view(BN, cap, 8, 4, 8)
    want = msda_pytorch(value.double().view(BN, -1, 8, 32), torch.tensor(shapes), loc, aw)
    for b in range(B):
        rows = slice(b * cams, (b + 1) * cams)
        n = int(ml[b])
        assert torch.all(out[rows, n:] == sentinel), b                # nothing written at or past max_len_b
        if n:
            assert not torch.isnan(out[rows, :n]).any(), b
            assert relerr(out[rows, :n], want[rows, :n]) < 2e-5, b    # fp32 sample positions: ~1e-6 px at 56 px
            assert torch.equal(out[rows, :n], out_c[rows, :n]), b     # one kernel body: bitwise the coupled entry's rows


def test_look_reduce_frames_matches_fp64():
    from thinktwice_b200 import lib
    counts = COUNTS
    B, cams = counts.shape
    cap, C = 120, 256
    g = torch.Generator().manual_seed(1)
    rows = torch.randn(B, cams, cap, C, generator=g)
    ml = counts.amax(1)
    for b in range(B):
        rows[b, :, int(ml[b]):] = float('nan')
    out = torch.full((B, cams * C), 777.0, device='cuda')
    lib.call('tt_look_reduce_frames', lib._p(rows.cuda()), B, cams, cap, C, lib._p(counts.cuda()), lib._p(out))
    torch.cuda.synchronize()
    out = out.cpu()
    for b in range(B):
        want = rows[b, :, 1:int(ml[b])].double().sum(1).reshape(-1)   # row 0 zeroed, divisor 1 (B = 1 semantics)
        if int(ml[b]) <= 1:
            assert torch.equal(out[b], torch.zeros(cams * C)), b
        else:
            assert relerr(out[b], want) < 1e-5, b


def test_frames_entries_equal_the_coupled_entries_at_b1():
    """at B = 1 the per-frame bound is the batch-wide max_len and the divisor is 1: bitwise the same results."""
    from thinktwice_b200 import lib
    for counts in (COUNTS[0:1], COUNTS[1:2], COUNTS[3:4]):
        d, _, value, off, logits, ref, ml = _msda_problem(counts, seed=2)
        dev = [t.cuda() for t in (value, off, logits, ref)]
        a, b = (torch.zeros(d.BN, 120, 256, device='cuda') for _ in range(2))
        lib.call('tt_msda_forward_frames', lib.ref(d), *[lib._p(t) for t in dev], lib._p(counts.cuda()), 4, lib._p(a))
        lib.call('tt_msda_forward', lib.ref(d), *[lib._p(t) for t in dev], lib._p(ml.int().cuda()), lib._p(b))
        rows = torch.randn(1, 4, 120, 256).cuda()
        r1, r2 = (torch.zeros(1, 1024, device='cuda') for _ in range(2))
        lib.call('tt_look_reduce_frames', lib._p(rows), 1, 4, 120, 256, lib._p(counts.cuda()), lib._p(r1))
        lib.call('tt_look_reduce', lib._p(rows), 1, 4, 120, 256, lib._p(ml.int().cuda()), lib._p(r2))
        torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(r1, r2)


def test_frames_entries_refuse_bad_arguments():
    from thinktwice_b200 import lib
    d, *_ = _msda_problem(COUNTS[:1])
    x = torch.zeros(16, device='cuda')
    with pytest.raises(lib.TTError):
        lib.call('tt_msda_forward_frames', lib.ref(d), lib._p(x), lib._p(x), lib._p(x), lib._p(x), lib._p(x), 3, lib._p(x))
    with pytest.raises(lib.TTError):
        lib.call('tt_look_reduce_frames', lib._p(x), 1, 4, 120, 256, None, lib._p(x))


# ------------------------------------------------------------------ the model at the thinktwice.py shape, B = 16
LENGTHS = [40000, 31000, 5000, 40000, 31000, 5000, 40000, 40000, 31000, 5000, 40000, 31000, 5000, 40000, 31000, 40000]
EMPTY = 4                                                              # the frame whose cloud has no point in range


@pytest.fixture(scope='module')
def full16():
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, 0)
    calibrate_bn(oracle, make_batch(cfg, 1, seed=0, num_points=40000))
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    batch = make_batch(cfg, 16, seed=31, num_points=40000)
    clouds = [batch['points'][j, :, :n].clone() for j, n in enumerate(LENGTHS)]
    clouds[EMPTY][..., 0] = 1000.0                                     # x far outside point_cloud_range: zero voxels
    batch['points'] = clouds
    model.enable_independent_frames()
    pred = model.forward_inference(batch)
    torch.cuda.synchronize()
    e, cam = model.eng, model.last_cam_feat
    B = 16
    enc = dict(fpn=[f.nchw().cpu().clone() for f in cam['fpn_feats']], flat=e.static_named('fu.py.flat').view(B, 256).cpu().clone(),
               bev32=e.static_named('fu.m21.out').permute(0, 3, 1, 2).cpu().clone(), meas=e.static_named('meas').view(B, 128).cpu().clone(),
               lidar=e.static_named('lidar.out.at').permute(0, 3, 1, 2).cpu().clone())
    out16 = {k: pred[k].float().cpu().clone() for k in KEYS}
    sat16 = model.f16s_saturations()
    counts = e.static_named('look.counts').view(B, 4).cpu().clone()
    alone = []
    for j in range(B):
        p1 = model.forward_inference({k: v[j:j + 1] for k, v in batch.items()})
        alone.append({k: p1[k].float().cpu().clone() for k in KEYS})
    return dict(cfg=cfg, oracle=oracle, model=model, batch=batch, out16=out16, enc=enc, sat16=sat16, alone=alone, counts=counts)


def test_full_config_b16_independent_frames_equal_each_frame_alone(full16):
    errs = frame_errs(full16['out16'], full16['alone'])
    print('independent B = 16 vs each frame alone:', {k: f'{v:.2e}' for k, v in errs.items()}, 'max', f'{max(errs.values()):.2e}')
    print('max_len_b per frame (last layer):', full16['counts'].amax(1).tolist())
    assert len(set(full16['counts'].amax(1).tolist())) > 1
    assert max(errs.values()) <= FRAME_TOL, errs
    assert full16['sat16'] == 0


def test_full_config_b16_independent_decoder_matches_the_oracle_at_b1(full16):
    """frames 0, 7, 15: the oracle's decoder run alone (B = 1) on the product's own encoder outputs of that frame."""
    oracle, batch, enc, out16 = full16['oracle'], full16['batch'], full16['enc'], full16['out16']
    for j in (0, 7, 15):
        s = slice(j, j + 1)
        l2i = batch['img_metas'][j][-1]['lidar2img'][None].float()
        ida = batch['img_metas'][j][-1]['ida_mats'][None].float()
        fpn = [f[4 * j:4 * j + 4] for f in enc['fpn']]
        with torch.no_grad():
            ref = oracle.decoder(enc['flat'][s], enc['bev32'][s], enc['meas'][s], oracle, [l2i, ida, fpn, enc['lidar'][s]], False, None)
        errs = {k: relerr(out16[k][s], ref[k]) for k in KEYS}
        print(j, {k: f'{v:.1e}' for k, v in errs.items()})
        assert all(v <= ORACLE_TOL for v in errs.values()), (j, errs)


def test_full_config_b16_coupled_mode_differs_from_each_frame_alone(full16):
    model = full16['model']
    model.enable_independent_frames(False)
    try:
        pred = model.forward_inference(full16['batch'])
        errs = frame_errs({k: pred[k].float().cpu() for k in KEYS}, full16['alone'])
    finally:
        model.enable_independent_frames(True)
    print('coupled B = 16 vs each frame alone:', {k: f'{v:.2e}' for k, v in errs.items()})
    assert max(errs.values()) > 10 * FRAME_TOL, errs


def test_full_config_two_shards_of_8_equal_the_b16_batch(full16):
    from thinktwice_b200.parallel import shard_batch
    model, out16 = full16['model'], full16['out16']
    worst = 0.0
    for r in range(2):
        part = shard_batch(full16['batch'], r, 2)
        pred = model.forward_inference(part)
        errs = frame_errs({k: pred[k].float().cpu() for k in KEYS}, [{k: out16[k][j:j + 1] for k in KEYS} for j in range(8 * r, 8 * r + 8)])
        worst = max(worst, max(errs.values()))
    print(f'two shards of 8 vs B = 16: {worst:.2e}')
    assert worst <= FRAME_TOL


def test_b1_the_two_modes_are_bitwise_the_same_computation(full16):
    """one frame at B = 1: the fusion + decoder tail run in both modes on the same encoder outputs.  Split-K (red.add partial sums) is
    switched off for the test so that the tail is deterministic: a repeat in the first mode is the control."""
    from thinktwice_b200 import lib
    model, batch = full16['model'], full16['batch']
    model.forward_inference({k: v[7:8] for k, v in batch.items()})
    lib.check(lib.load().tt_debug_set(128), 'tt_debug_set')
    try:
        lidar = model._phase_lidar()
        cam, meas = model._phase_key()
        outs = []
        for mode in (False, True, False):
            model.enable_independent_frames(mode)
            p = model._phase_tail(cam, meas, lidar)
            torch.cuda.synchronize()
            outs.append({k: p[k].clone() for k in KEYS})
    finally:
        lib.check(lib.load().tt_debug_set(0), 'tt_debug_set')
        model.enable_independent_frames(True)
    for k in KEYS:
        assert torch.equal(outs[0][k], outs[2][k]), ('control', k)
        assert torch.equal(outs[0][k], outs[1][k]), k


# ------------------------------------------------------------------ CUDA graphs (plumbing config with a history sweep, B = 4)
def test_graph_replay_equals_eager_in_independent_mode_and_modes_alternate():
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(PLUMBING_CONFIG)
    cfg.model['img_encoder']['queue_len'] = 2
    cfg.model['train_cfg']['queue_length'] = 2
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(oracle, 1)
    host = make_batch(cfg, 4, seed=1, num_points=1500)
    calibrate_bn(oracle, host)
    model = build_model(cfg.model)
    model.load_state_dict(oracle.state_dict())
    model.prepare('cuda:0')
    keys = ('pred_wp', 'mu_branches', 'refine_BEV_feature', 'pred_speed')
    resident = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in host.items()}
    pinned = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in host.items()}
    eager = {}
    for mode in (False, True):
        model.enable_independent_frames(mode)
        p = model.forward_inference(resident)
        eager[mode] = {k: p[k].clone() for k in keys}
    assert max(relerr(eager[True][k], eager[False][k]) for k in keys) > 10 * FRAME_TOL      # the alternation below discriminates
    model.enable_cuda_graph()
    for mode in (True, False, True, False, True):                      # capture each mode, then replays alternating with the other
        model.enable_independent_frames(mode)
        for b in (resident, pinned):
            for _ in range(2):
                p = model.forward_inference(b)
                for k in keys:
                    assert relerr(p[k], eager[mode][k]) < FRAME_TOL, (mode, b is pinned, k)
    assert any(k[0] == 'pipe' for k in model._graphs) and any(k[0] != 'pipe' for k in model._graphs)
    assert {k[-1] for k in model._graphs} == {False, True}
    model.use_graph = False
    assert model.f16s_saturations() == 0
