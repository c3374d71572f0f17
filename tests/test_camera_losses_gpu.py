"""The camera branch's supervision on the GPU: tt_camera_loss against float64 on crafted inputs (tests/camera_loss_checks.py), seg_loss /
depth_loss end to end against the oracle (tests/camera_loss_oracle.py, pinned to the reference's code by tests/test_camera_losses_cpu.py) and
against the reference's formulas on the product's own logits, the decoder's terms left as they were, inference after a validation
call left as it was, and the happens-before audit of a validation call with both terms mixed with inference."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-3                # the key frame's logits vs the oracle
TERM_TOL = 5e-3           # the two terms vs the oracle (as the decoder's terms, tests/test_losses_gpu.py)
EXACT = 1e-5              # the two terms vs the reference's formulas on the product's own logits: the kernel and the staging
DECODER = 1e-4            # the decoder's terms with and without the camera terms (run-to-run red.add order, not bitwise)


def relerr(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-6))


def test_kernel_on_crafted_inputs_against_float64():
    import camera_loss_checks
    out = camera_loss_checks.check_all('cuda')
    for name, (got, want) in out.items():
        print(name, got, want)


def camera_config(path):
    from thinktwice_b200.config import Config
    cfg = Config.fromfile(path)
    cfg.merge_from_dict({'model.train_cfg.use_seg': True, 'model.train_cfg.use_depth': True})
    return cfg


def build(path, B, seed, points):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch, make_camera_supervision, make_supervision
    cfg = camera_config(path)
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, seed)
    batch = make_batch(cfg, B, seed=seed, num_points=points)
    calibrate_bn(o, batch)
    batch.update(make_supervision(cfg, B, seed=seed))
    batch.update(make_camera_supervision(cfg, B, seed=seed))
    m = build_model(cfg.model)
    m.load_state_dict(o.state_dict())
    m.prepare('cuda:0')
    return cfg, o.eval(), m, batch


def own_logits(m):
    """the key frame's (B*N, C, h, w) segmentation and (B*N, D, h', w') depth logits as the product computed them."""
    cam = m.last_cam_feat
    D = m.img_encoder.depth_channels
    return cam['seg'].nchw().float(), cam['depth'].slice(0, D).nchw().float()


def own_formulas(m, batch, device='cpu'):
    """the reference's seg_loss / depth_loss (fp32 torch, as the reference computes them) on the product's own logits."""
    import camera_loss_oracle
    seg, depth = own_logits(m)
    gt = {k: batch[k].to(device) for k in ('seg', 'depth')}
    return camera_loss_oracle.camera_loss(m.config, gt, seg.to(device).contiguous(), depth.to(device).contiguous(), m.dbound,
                                          m.downsample_factor, m.seg_downsample_factor)


def decoder_terms_unchanged(m, batch, got):
    """the decoder's terms of the same batch with the camera flags off, within DECODER of the ones computed with them on."""
    m.config['use_seg'] = m.config['use_depth'] = False
    try:
        off = m.forward_train(batch)
    finally:
        m.config['use_seg'] = m.config['use_depth'] = True
    assert list(off) == [k for k in got if k not in ('seg_loss', 'depth_loss')]
    bad = {k: relerr(got[k], v) for k, v in off.items() if not relerr(got[k], v) <= DECODER}
    assert not bad, bad


def check_against_oracle(o, m, batch):
    import camera_loss_oracle
    import loss_oracle
    want, pred_o = camera_loss_oracle.forward_train(o, batch)
    _, want_log = loss_oracle.parse_losses(want)
    out = m.forward(is_eval=True, **batch)
    torch.cuda.synchronize()
    assert list(out['log_vars']) == list(want_log) and list(want_log)[-3:] == ['seg_loss', 'depth_loss', 'loss']
    seg, depth = own_logits(m)
    errs = dict(seg_logits=relerr(seg, pred_o['cam_seg']), depth_logits=relerr(depth, pred_o['cam_depth']))
    own = own_formulas(m, batch)
    exact = {k: relerr(out['log_vars'][k], own[k]) for k in own}
    terms = {k: relerr(out['log_vars'][k], want[k]) for k in own}
    print(errs, exact, terms, {k: out['log_vars'][k] for k in own})
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    bad.update({'exact.' + k: v for k, v in exact.items() if not v <= EXACT})
    bad.update({'term.' + k: v for k, v in terms.items() if not v <= TERM_TOL})
    assert not bad, bad
    assert np.isfinite(out['log_vars']['loss']) and m.f16s_saturations() == 0
    decoder_terms_unchanged(m, batch, m.forward_train(batch))


@pytest.mark.parametrize('B', [1, 2])
def test_plumbing_camera_losses_match_the_oracle(B):
    from thinktwice_b200.config import PLUMBING_CONFIG
    _, o, m, batch = build(PLUMBING_CONFIG, B, seed=B, points=2000)
    check_against_oracle(o, m, batch)


def test_full_config_b2_camera_losses_match_the_oracle():
    from thinktwice_b200.config import DEFAULT_CONFIG
    _, o, m, batch = build(DEFAULT_CONFIG, 2, seed=0, points=40000)
    check_against_oracle(o, m, batch)


def test_b16_full_config_with_the_shipped_flags():
    """B = 16 at the full config, flags as shipped, the camera ground truth on the host: both terms within EXACT of the reference's
    formulas evaluated on the GPU on the product's own logits; an eager inference call after it is what it was before."""
    from thinktwice_b200.config import DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_batch, make_camera_supervision, make_supervision
    cfg, _, m, _ = build(DEFAULT_CONFIG, 1, seed=0, points=40000)
    assert m.config['use_seg'] and m.config['use_depth']
    B = 16
    batch = make_batch(cfg, B, seed=21, num_points=40000)
    plain = dict(batch)
    before = {k: v.clone() for k, v in m.forward_inference(plain).items() if k in ('pred_wp', 'mu_branches', 'pred_speed')}
    again = {k: v.clone() for k, v in m.forward_inference(plain).items() if k in before}
    camera_gt = make_camera_supervision(cfg, B, seed=21)
    out = m.forward(is_eval=True, **batch, **make_supervision(cfg, B, seed=21), **camera_gt)
    torch.cuda.synchronize()
    print('peak GB', torch.cuda.max_memory_allocated() / 1e9, {k: out['log_vars'][k] for k in ('seg_loss', 'depth_loss', 'loss')})
    own = own_formulas(m, camera_gt, 'cuda')
    for k, v in own.items():
        assert relerr(out['log_vars'][k], v) <= EXACT, (k, out['log_vars'][k], float(v))
    after = {k: v.clone() for k, v in m.forward_inference(plain).items() if k in before}
    for k in before:
        if torch.equal(before[k], again[k]):
            assert torch.equal(after[k], before[k]), k
        else:
            assert relerr(after[k], before[k]) <= 1e-5, k


@pytest.mark.parametrize('order', ['validation_first', 'inference_first'])
def test_audit_validation_with_camera_terms_and_inference_mixed(order):
    """tests/stream_audit.py finds no unordered conflict in a validation call with both camera terms (ground truth on the host) mixed with
    a pipelined inference call."""
    from test_stream_order_gpu import audit_clean, frames, plumbing_q2
    from thinktwice_b200.synthetic import make_camera_supervision, make_supervision
    cfg, model = plumbing_q2(12)
    assert model.config['use_seg'] and model.config['use_depth']
    b1, = frames(cfg, 2, (121,), 1500, 'cpu')
    b1.update(make_supervision(cfg, 2, seed=121))
    b1.update(make_camera_supervision(cfg, 2, seed=121))
    b2, = frames(cfg, 2, (122,), 1500, 'pinned')

    def run():
        if order == 'validation_first':
            model.forward(**b1)
            model.forward_inference(b2)
        else:
            model.forward_inference(b2)
            model.forward(**b1)
    rec = audit_clean(model, run, f'validation with camera terms / inference, {order}')
    assert any(op.what.startswith('tt_camera_loss.') for op in rec.trace if hasattr(op, 'what') and op.what)
