"""Open-loop validation losses on the GPU: tt_loss_reduce against fp64 on crafted inputs, the teacher-forced pass and every loss term
end to end against the oracle (tests/loss_oracle.py, itself pinned to the reference's code by tests/test_losses_cpu.py), a
self-consistency check that needs no oracle, and the inference path left as it was."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-3                # predictions and teacher tensors vs the oracle (the north star)
TERM_TOL = 5e-3           # loss terms vs the oracle: smooth-L1 / L1 of (pred - gt) turn a relative prediction difference e into up to
                          # e * |pred| / |pred - gt| (speed_loss at the plumbing shape, B = 1: 1.6e-3 from a 5e-4 pred_speed difference)
EXACT = 1e-5              # loss terms vs the same losses computed in torch from the product's own outputs: the kernel itself


def relerr(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-6))


# ---------------------------------------------------------------------------------------------- the kernel on crafted inputs
def reduce(terms, n_slots):
    from thinktwice_b200 import lib
    out = torch.full((n_slots,), float('nan'), device='cuda')
    ws = torch.empty(int(lib.load().tt_loss_workspace_bytes(len(terms))), dtype=torch.uint8, device='cuda')
    import ctypes
    lib.call('tt_loss_reduce', lib.pack_loss_terms(terms), len(terms), lib._p(out), n_slots, lib._p(ws), ctypes.c_size_t(ws.numel()))
    torch.cuda.synchronize()
    return out.cpu()


def term(kind, slot, scale, shape, pred, pstride, gt=None, gstride=None, pred2=None, gt2=None, aux=0, poff=0, goff=0):
    from thinktwice_b200 import lib
    return dict(kind=kind, slot=slot, scale=scale, shape=list(shape), aux=aux, pred=lib._p(pred, poff), pred_stride=list(pstride),
                pred2=lib._p(pred2, poff) if pred2 is not None else lib._p(None), gt=lib._p(gt, goff) if gt is not None else lib._p(None),
                gt_stride=list(gstride) if gstride is not None else [0] * len(shape), gt2=lib._p(gt2, goff) if gt2 is not None else lib._p(None))


def test_smooth_l1_edges_and_the_clamp():
    from thinktwice_b200 import lib
    p = torch.tensor([0.0, 1.0, -1.0, 0.5, 5.5, -5.5, 100.0], device='cuda')
    g = torch.tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0], device='cuda')
    want = torch.where(p.abs() < 1, 0.5 * p.double() ** 2, p.double().abs() - 0.5).cpu()          # |x| = 1: 0.5 on both branches
    terms = [term(lib.LOSS_SMOOTH_L1, i, 1.0, [1], p, [1], g, [1], poff=i, goff=i) for i in range(7)]
    terms += [term(lib.LOSS_SMOOTH_L1_CLAMP, 7 + i, 1.0, [1], p, [1], poff=i) for i in range(7)]     # null gt: zero target
    terms += [term(lib.LOSS_L1, 14, 1.0 / 7, [7], p, [1])]
    out = reduce(terms, 15).double()
    assert torch.allclose(out[:7], want, rtol=1e-7, atol=0)
    assert out[7 + 4] == 5.0 and out[7 + 6] == 5.0 and out[7 + 3] == 0.125                         # clamp at exactly 5
    assert abs(float(out[14]) - float(p.double().abs().mean())) < 1e-6


def test_broadcast_strides_and_channels_last_against_nchw():
    from thinktwice_b200 import lib
    g = torch.Generator().manual_seed(0)
    N, C, H, W, ld, coff = 3, 32, 21, 21, 40, 4
    buf = torch.randn(N, H, W, ld, generator=g).cuda()                  # channels-last map, C channels at coff of ld
    gt = (2 * torch.rand(N, C, H, W, generator=g)).cuda()               # NCHW
    row = torch.randn(C, generator=g).cuda()                             # broadcast over N, H, W
    want_cl = torch.clamp(torch.nn.functional.smooth_l1_loss(buf[..., coff:coff + C].permute(0, 3, 1, 2).double(), gt.double(),
                                                             reduction='none'), -5, 5).mean()
    want_bc = torch.nn.functional.smooth_l1_loss(buf[..., coff:coff + C].permute(0, 3, 1, 2).double(), row.double()[None, :, None, None].expand(N, C, H, W))
    n = N * C * H * W
    out = reduce([term(lib.LOSS_SMOOTH_L1_CLAMP, 0, 1.0 / n, [N, C, H, W], buf, [H * W * ld, 1, W * ld, ld], gt, gt.stride(), poff=coff),
                  term(lib.LOSS_SMOOTH_L1, 1, 1.0 / n, [N, C, H, W], buf, [H * W * ld, 1, W * ld, ld], row, [0, 1, 0, 0], poff=coff),
                  term(lib.LOSS_SMOOTH_L1, 1, 1.0 / n, [N, C, H, W], buf, [H * W * ld, 1, W * ld, ld], row, [0, 1, 0, 0], poff=coff)], 2)
    assert abs(float(out[0]) - float(want_cl)) <= 1e-6 * float(want_cl)
    assert abs(float(out[1]) - 2 * float(want_bc)) <= 1e-6 * float(want_bc)                       # a shared slot adds its terms


def test_beta_kl_against_scipy_on_a_grid():
    from scipy.special import digamma, gammaln
    from thinktwice_b200 import lib
    v = np.logspace(-3, 3, 7).astype(np.float32)
    grid = np.array(np.meshgrid(v, v, v, v, indexing='ij')).reshape(4, -1).T                        # (a1, b1, a2, b2)
    a1, b1, a2, b2 = (torch.from_numpy(np.ascontiguousarray(grid[:, i])).cuda() for i in range(4))
    n = grid.shape[0]
    out = reduce([term(lib.LOSS_BETA_KL, i, 1.0, [1], a2, [1], a1, [1], pred2=b2, gt2=b1, poff=i, goff=i) for i in range(n)], n).double().numpy()
    x = grid.astype(np.float64)
    A1, B1, A2, B2 = x.T
    want = (gammaln(A2) + gammaln(B2) + gammaln(A1 + B1) - gammaln(A1) - gammaln(B1) - gammaln(A2 + B2) + (A1 - A2) * digamma(A1)
            + (B1 - B2) * digamma(B1) + (A2 + B2 - A1 - B1) * digamma(A1 + B1))
    err = np.abs(out - want) / np.maximum(np.abs(want), 1e-3)
    assert err.max() < 2e-6, (err.max(), grid[err.argmax()], out[err.argmax()], want[err.argmax()])


def test_action_beta_every_branch():
    import loss_oracle
    from thinktwice_b200 import lib
    v = torch.tensor([0.25, 1.0, 1.0 + 2 ** -20, 3.0, 40.0])
    grid = torch.cartesian_prod(v, v, v, v)                                                         # (pred a, pred b, gt a, gt b)
    n = grid.shape[0]
    pa, pb, ga, gb = (grid[:, i].contiguous().cuda() for i in range(4))
    terms = [term(lib.LOSS_ACTION_L1, 2 * i + c, 1.0, [1], pa, [1], ga, [1], pred2=pb, gt2=gb, aux=c, poff=i, goff=i)
             for i in range(n) for c in (0, 1)]
    out = reduce(terms, 2 * n).view(n, 2).double()
    col = lambda a, b: torch.stack([a, b], 1)
    for c in (0, 1):                                                                                # the same value in either column
        want = (loss_oracle.action_beta(col(grid[:, 0], grid[:, 0]), col(grid[:, 1], grid[:, 1]))[:, c] -
                loss_oracle.action_beta(col(grid[:, 2], grid[:, 2]), col(grid[:, 3], grid[:, 3]))[:, c]).abs().double()
        assert torch.allclose(out[:, c], want, rtol=0, atol=1e-6), c


def test_nan_and_out_of_domain_values_give_nan():
    """a NaN element keeps a clamped term NaN (torch.clamp propagates it), and Beta parameters outside (0, inf) give NaN, not a number."""
    from thinktwice_b200 import lib
    p = torch.tensor([0.5, float('nan'), 9.0], device='cuda')
    a = torch.tensor([2.0, 3.0, -0.5, 0.0, float('nan')], device='cuda')
    b = torch.tensor([2.0, 2.0, 2.0, 2.0, 2.0], device='cuda')
    terms = [term(lib.LOSS_SMOOTH_L1_CLAMP, 0, 1.0, [3], p, [1]), term(lib.LOSS_SMOOTH_L1_CLAMP, 1, 1.0, [1], p, [1], poff=2)]
    terms += [term(lib.LOSS_BETA_KL, 2 + i, 1.0, [1], b, [1], a, [1], pred2=b, gt2=b, poff=i, goff=i) for i in range(5)]
    out = reduce(terms, 7)
    assert torch.isnan(out[0]) and out[1] == 5.0
    assert out[2] == 0.0 and torch.isfinite(out[3]) and torch.isnan(out[4:]).all()


def test_two_launches_are_bitwise_equal():
    from thinktwice_b200 import lib
    g = torch.Generator().manual_seed(1)
    p, q = torch.randn(1 << 20, generator=g).cuda(), torch.randn(1 << 20, generator=g).cuda()
    terms = [term(lib.LOSS_SMOOTH_L1, 0, 1e-6, [1 << 20], p, [1], q, [1]), term(lib.LOSS_L1, 1, 1.0, [1024, 1024], p, [1024, 1], q, [1, 1024])]
    a, b = reduce(terms, 2), reduce(terms, 2)
    assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------- end to end
def loss_config(path):
    from thinktwice_b200.config import Config
    cfg = Config.fromfile(path)
    for k in ('use_depth', 'use_seg'):
        cfg.merge_from_dict({f'model.train_cfg.{k}': False, f'model.decoder.config.{k}': False})
    return cfg


def build(path, B, seed, points, independent=False):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch, make_supervision
    cfg = loss_config(path)
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, seed)
    batch = make_batch(cfg, B, seed=seed, num_points=points)
    calibrate_bn(o, batch)
    batch.update(make_supervision(cfg, B, seed=seed))
    m = build_model(cfg.model)
    m.load_state_dict(o.state_dict())
    m.prepare('cuda:0')
    return cfg, o.eval(), m.enable_independent_frames(independent), batch


TEACHER = ('teacher_pred_wp_offset', 'teacher_pred_ctrl_offset_lis', 'teacher_future_BEV_feature', 'teacher_refine_flattned_BEV_feature',
           'teacher_refine_BEV_feature')


PRED = ('pred_speed', 'pred_value_traj', 'pred_value_ctrl', 'pred_features_traj', 'pred_features_ctrl', 'pred_wp', 'mu_branches', 'sigma_branches', 'future_mu',
        'future_sigma', 'refine_flattned_BEV_feature', 'refine_BEV_feature')


def check_losses(m, got, want, pred_o, batch, train_cfg, layer0_only=()):
    """got: the product's loss dict; want / pred_o: the oracle's losses and predictions.  Three checks: every prediction the losses read
    within TOL of the oracle, every term within EXACT of the reference's loss formulas applied (in torch, fp32) to the product's OWN
    outputs — which isolates tt_loss_reduce and its descriptors — and every term within TERM_TOL of the oracle's."""
    import loss_oracle
    t = m.last_train
    pred = {k: t['pred'][k].float().cpu() for k in PRED + TEACHER}
    mid = [None, None] + [f.nchw().float().cpu() for f in t['mid'][2:]]
    errs = {k: relerr(pred[k][:, :1] if k in layer0_only else pred[k], pred_o[k][:, :1] if k in layer0_only else pred_o[k])
            for k in PRED + TEACHER}
    own = loss_oracle.decoder_loss(train_cfg, batch, pred, mid)

    def cmp(a, b):                                                   # value_loss: (B, 1) where both sides have it, else the logged mean
        a, b = torch.as_tensor(a), torch.as_tensor(b)
        return relerr(a, b) if a.shape == b.shape else relerr(a.double().mean(), b.double().mean())
    exact = {k: cmp(got[k], v) for k, v in own.items()}
    terms = {k: cmp(got[k], v) for k, v in want.items()}
    print({k: f'{v:.1e}' for k, v in errs.items()}, {k: f'{v:.1e}' for k, v in exact.items()}, {k: f'{v:.1e}' for k, v in terms.items()})
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    bad.update({'exact.' + k: v for k, v in exact.items() if not v <= EXACT})
    bad.update({'term.' + k: v for k, v in terms.items() if not v <= TERM_TOL})
    assert not bad, bad


def check_against_oracle(o, m, batch):
    import loss_oracle
    want, pred_o = loss_oracle.forward_train(o, batch)
    _, want_log = loss_oracle.parse_losses(want)
    out = m.forward(is_eval=True, **batch)
    torch.cuda.synchronize()
    assert set(out) == {'loss', 'log_vars', 'num_samples'} and list(out['log_vars']) == list(want_log)
    got = {k: torch.as_tensor(out['log_vars'][k]) for k in want}
    check_losses(m, got, {k: v.mean() for k, v in want.items()}, pred_o, batch, o.config)
    assert relerr(out['log_vars']['loss'], want_log['loss']) <= TERM_TOL
    assert m.f16s_saturations() == 0


@pytest.mark.parametrize('B', [1, 2])
def test_plumbing_losses_match_the_oracle(B):
    from thinktwice_b200.config import PLUMBING_CONFIG
    _, o, m, batch = build(PLUMBING_CONFIG, B, seed=B, points=2000)
    check_against_oracle(o, m, batch)


def test_full_config_b2_losses_match_the_oracle():
    from thinktwice_b200.config import DEFAULT_CONFIG
    _, o, m, batch = build(DEFAULT_CONFIG, 2, seed=0, points=40000)
    check_against_oracle(o, m, batch)


@pytest.mark.parametrize('independent', [False, True], ids=['coupled', 'independent'])
def test_b16_decoder_terms_match_the_oracle_decoder_on_the_products_encoder_outputs(independent):
    """B = 16 at the full config: the oracle's teacher-forced decoder + loss run on the CPU on the product's own fusion outputs (as
    test_model_gpu.py does for inference, with its model); every term compared.  The future-BEV stacks are held to TOL at layer 0: the
    4-step GRU recurrence of the seeded network amplifies fp32-level differences about 7x per step and the later layers compound it
    (refine_future_BEV_feature of the MAIN pass, not a loss input, shows the same growth); their loss terms are compared at every layer."""
    import loss_oracle
    from thinktwice_b200.config import DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_batch, make_supervision
    cfg, o, m, _ = build(DEFAULT_CONFIG, 1, seed=0, points=40000, independent=independent)
    B = 16
    batch = make_batch(cfg, B, seed=21, num_points=40000)
    batch.update(make_supervision(cfg, B, seed=21))
    got = m.forward_train(batch)
    torch.cuda.synchronize()
    t = m.last_train
    cpu = lambda x: x.float().cpu().clone()
    flat, bev32, meas = cpu(t['flat'].t.view(B, 256)), cpu(t['bev32'].nchw()), cpu(t['meas'].t.view(B, 128))
    mid = [None, None] + [cpu(f.nchw()) for f in t['mid'][2:]]
    fpn = [cpu(f.nchw()) for f in m.last_cam_feat['fpn_feats']]
    lidar_hi = cpu(t['lidar_hi'].nchw())
    l2i = torch.stack([mm[-1]['lidar2img'] for mm in batch['img_metas']], 0).float()
    ida = torch.stack([mm[-1]['ida_mats'] for mm in batch['img_metas']], 0).float()

    def decode(sl):
        meta = [l2i[sl], ida[sl], [f[sl.start * 4:sl.stop * 4] for f in fpn], lidar_hi[sl]]
        sub = {k: batch[k][sl] if torch.is_tensor(batch[k]) else [x[sl] for x in batch[k]] for k in loss_oracle.TEACHER_INPUTS}
        with torch.no_grad():
            p = o.decoder(flat[sl], bev32[sl], meas[sl], o, meta, False, None)
            p.update(loss_oracle.teacher_pass(o.decoder, flat[sl], bev32[sl], meas[sl], o, meta, sub))
        return p
    if independent:
        parts = [decode(slice(j, j + 1)) for j in range(B)]
        pred = {k: torch.cat([p[k] for p in parts]) for k in parts[0] if torch.is_tensor(parts[0][k])}
    else:
        pred = decode(slice(0, B))
    want = loss_oracle.decoder_loss(o.config, batch, pred, mid)
    check_losses(m, got, want, pred, batch, o.config, layer0_only=('teacher_future_BEV_feature', 'teacher_pred_wp_offset',
                                                                    'teacher_pred_ctrl_offset_lis'))


def test_teacher_layer0_fed_the_coarse_prediction_equals_the_main_pass_layer0():
    """No oracle: with the ground truth set to the model's own coarse prediction, the teacher pass's first layer sees exactly the
    main pass's first-layer inputs (through an inv_softplus / softplus round trip) and must produce its outputs."""
    from thinktwice_b200.config import PLUMBING_CONFIG
    _, _, m, batch = build(PLUMBING_CONFIG, 2, seed=3, points=2000)
    pred = m.forward_inference(batch)
    T = pred['pred_wp'].shape[2]
    gt = dict(batch, waypoints=pred['pred_wp'][:, 0].cpu(), action_mu=pred['mu_branches'][:, 0].cpu(),
              action_sigma=pred['sigma_branches'][:, 0].cpu(),
              future_action_mu=[pred['future_mu'][:, 0, t].cpu() for t in range(T - 1)] + [batch['future_action_mu'][-1]],
              future_action_sigma=[pred['future_sigma'][:, 0, t].cpu() for t in range(T - 1)] + [batch['future_action_sigma'][-1]])
    m.forward_train(gt)
    torch.cuda.synchronize()
    p = m.last_train['pred']
    assert relerr(p['teacher_pred_wp_offset'][:, 0], p['pred_wp'][:, 1] - p['pred_wp'][:, 0]) < 1e-4
    assert relerr(p['teacher_refine_BEV_feature'][:, 0], p['refine_BEV_feature'][:, 0]) < 1e-4
    assert relerr(p['teacher_refine_flattned_BEV_feature'][:, 0], p['refine_flattned_BEV_feature'][:, 0]) < 1e-4


def test_inference_is_unaffected_by_a_loss_call():
    """eager, one-stream graph replay, the pipelined four-graph replay of a host-resident batch (the default graph mode for host inputs)
    and the streaming BEV cache: forward_inference after forward(**batch_with_gt) is what it was — bitwise where two inference calls in a
    row are bitwise equal, else within 1e-5 (fp32 red.add accumulation can reorder between launches: two eager calls in a row differ by
    ~1e-6 on their own)."""
    from thinktwice_b200.config import DEFAULT_CONFIG
    _, _, m, batch = build(DEFAULT_CONFIG, 1, seed=5, points=20000)
    plain = {k: v for k, v in batch.items() if k not in m.SUPERVISION_KEYS}
    keys = ('pred_wp', 'mu_branches', 'sigma_branches', 'pred_speed')
    run = lambda: {k: v.clone() for k, v in m.forward_inference(plain).items() if k in keys}
    assert plain['img'].device.type == 'cpu' and plain['img'].shape[1] == 2    # host inputs with a history sweep: pipelined when allowed
    for mode in ('eager', 'graph', 'pipelined graph', 'stream'):
        m.pipeline_uploads = mode == 'pipelined graph'
        m.enable_cuda_graph(mode in ('graph', 'pipelined graph'))
        if mode == 'stream':
            m.enable_streaming_bev_cache()
        first = run()                                                # (graph modes: the capture call; stream mode: a cold tick)
        before = run()
        if mode == 'pipelined graph':
            assert any(k[0] == 'pipe' for k in m._graphs)            # the four-graph pipelined form is what was captured and replayed
        out = m.forward(is_eval=True, **batch)
        assert out['loss'] is not None and np.isfinite(out['log_vars']['loss'])
        after = run()
        if mode == 'stream':                                         # the loss call reset the cache: the next tick is a cold one again
            first, before = before, first
        for k in keys:
            if torch.equal(first[k], before[k]):
                assert torch.equal(after[k], before[k]), (mode, k)
            else:
                assert relerr(after[k], before[k]) <= 1e-5, (mode, k)
    assert m.f16s_saturations() == 0
