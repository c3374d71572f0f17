"""Open-loop validation losses without a GPU.

  * tests/loss_oracle.py (the plain-PyTorch restatement) reproduces tests/golden/ref_losses_*.npz, which the reference's own
    forward_train / decoder.loss / _parse_losses produced (tests/golden/make_loss_golden.py);
  * the product's host code — teacher-forced pass, supervision staging, the loss descriptors, forward_train, _parse_losses, the
    `forward(is_eval=True, **batch)` route — through the emulated C ABI (tests/emu_lib.py + tests/emu_losses.py) matches the oracle,
    in both Look modes;
  * the ctypes mirror of tt_loss_term has the header's layout; a batch without supervision keeps the inference route; depth /
    segmentation supervision raises; two gloo ranks average the log vars as the reference does.
The kernels themselves are tests/test_losses_gpu.py's job."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
G = os.path.join(HERE, 'golden')
sys.path.insert(0, G)

TOL = 5e-4                                                             # fp32 oracle vs fp64-contraction emulation (as the other emulated tests)


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-6))


def loss_config(path=None):
    from make_loss_golden import loss_config as lc
    from thinktwice_b200.config import PLUMBING_CONFIG
    return lc(path or PLUMBING_CONFIG)


def oracle_and_batch(cfg, B, seed, points=1500):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.synthetic import make_batch, make_supervision
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, seed)
    batch = make_batch(cfg, B, seed=seed, num_points=points)
    calibrate_bn(o, batch)
    batch.update(make_supervision(cfg, B, seed=seed))
    return o, batch


# ---------------------------------------------------------------------------------------------- the oracle vs the reference's code
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_oracle_forward_train_equals_the_reference_code(seed):
    import loss_oracle
    from make_loss_golden import PLUMBING_CASES
    f = np.load(os.path.join(G, f'ref_losses_plumbing_seed{seed}.npz'))
    B = dict(PLUMBING_CASES)[seed]
    assert int(f['batch']) == B
    o, batch = oracle_and_batch(loss_config(), B, seed)
    losses, pred = loss_oracle.forward_train(o.eval(), batch)
    assert list(losses) == list(f['keys'])                             # the reference's keys, in its order
    for k, v in losses.items():
        assert rel(v.numpy(), f['loss.' + k]) < 1e-5, k                # camera encoder: index_add order, not bitwise (as the e2e golden)
    _, log_vars = loss_oracle.parse_losses(losses)
    for k, v in log_vars.items():
        assert rel(v, f['log.' + k]) < 1e-5, k
    for k in [n[len('teacher.'):] for n in f.files if n.startswith('teacher.')]:
        got = pred[k.split('.')[0]]
        got = got.mean((-2, -1)) if k.endswith('.mean_hw') else got[..., ::4, ::4] if k.endswith('.sub') else got
        assert rel(got.numpy(), f['teacher.' + k]) < 1e-5, k


def test_oracle_teacher_forced_decoder_equals_the_reference_code_at_k5():
    """fusion + decoder with teacher forcing + loss at the full config (K = 5, B = 2) on the seeded encoder stand-ins."""
    import loss_oracle
    from make_reference_golden import named_init, synthetic_inputs
    from oracle.model import EncoderDecoder as Oracle
    from thinktwice_b200.config import DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_supervision
    f = np.load(os.path.join(G, 'ref_losses_decoder_k5_seed3.npz'))
    seed, B = int(f['seed']), int(f['batch'])
    cfg = loss_config(DEFAULT_CONFIG)
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'}).eval()
    sub = {k: v for k, v in o.state_dict().items() if not k.startswith(('img_encoder.', 'lidar_encoder.'))}

    class Shared:                                                      # the fusion + decoder part the golden covers
        def state_dict(self):
            return sub

        def load_state_dict(self, d):
            o.load_state_dict(d, strict=False)
    named_init(Shared(), seed)
    x = synthetic_inputs(cfg, seed, B)
    batch = dict(speed=x['speed'], **make_supervision(cfg, B, seed=seed))
    with torch.no_grad():
        state = torch.cat([x['speed'].float().view(-1, 1) / 12., x['target_point'].float(), x['target_command']], -1)
        meas = o.measurements_encoder(state)
        flat, bev32, mid, lidar_hi = o.get_fusion_feat(x['cam_bev'], x['lidar'])
        meta = [x['lidar2img'], x['ida_mat'], x['fpn'], lidar_hi]
        pred = o.decoder(flat, bev32, meas, o, meta, False, None)
        pred.update(loss_oracle.teacher_pass(o.decoder, flat, bev32, meas, o, meta, batch))
        losses = loss_oracle.decoder_loss(cfg.model.train_cfg, batch, pred, mid)
    assert list(losses) == list(f['keys'])
    for k, v in losses.items():
        assert rel(v.numpy(), f['loss.' + k]) < 1e-6, k                # same torch ops in the same order
    for k in [n[len('teacher.'):] for n in f.files if n.startswith('teacher.')]:
        got = pred[k.split('.')[0]]
        got = got.mean((-2, -1)) if k.endswith('.mean_hw') else got[..., ::4, ::4] if k.endswith('.sub') else got
        assert rel(got.numpy(), f['teacher.' + k]) < 1e-6, k


# ---------------------------------------------------------------------------------------------- the product's host code, emulated ABI
@pytest.fixture
def emu(emulated, monkeypatch):
    import gc
    import emu_frames
    import emu_lib
    import emu_losses
    emu_lib._by_addr.clear()                                          # the emulation's address book keeps every tensor it saw alive
    gc.collect()
    yield emu_losses.install(emu_frames.install(emulated), monkeypatch)
    emu_lib._by_addr.clear()
    gc.collect()


def product(cfg, o, independent=False):
    from thinktwice_b200.registry import build_model
    m = build_model(cfg.model)
    m.load_state_dict(o.state_dict())
    m.prepare('cpu', impl=4)
    return m.enable_independent_frames(independent)


@pytest.mark.parametrize('independent', [False, True], ids=['coupled', 'independent'])
@pytest.mark.parametrize('B', [1, 2])
def test_emulated_forward_with_supervision_matches_the_oracle(emu, B, independent):
    import loss_oracle
    cfg = loss_config()
    o, batch = oracle_and_batch(cfg, B, seed=1)
    want, _ = loss_oracle.forward_train(o.eval(), batch, independent_frames=independent)
    _, want_log = loss_oracle.parse_losses(want)
    m = product(cfg, o, independent)
    out = m.forward(is_eval=True, **batch)
    assert set(out) == {'loss', 'log_vars', 'num_samples'} and out['num_samples'] == B
    assert list(out['log_vars']) == list(want_log)
    for k, v in want_log.items():
        assert rel(out['log_vars'][k], v) < TOL, (k, out['log_vars'][k], v)
    assert rel(float(out['loss']), want_log['loss']) < TOL
    got = m.forward_train(batch)
    assert got['value_loss'].shape == (B, 1) and all(v.dim() == 0 for k, v in got.items() if k != 'value_loss')
    for k, v in want.items():
        assert rel(got[k].numpy(), v.numpy()) < TOL, k


def test_teacher_outputs_match_the_oracle(emu):
    import loss_oracle
    cfg = loss_config()
    o, batch = oracle_and_batch(cfg, 2, seed=2)
    _, want = loss_oracle.forward_train(o.eval(), batch)
    m = product(cfg, o)
    m.forward_train(batch)
    pred = m.last_train['pred']
    for k in ('teacher_pred_wp_offset', 'teacher_pred_ctrl_offset_lis', 'teacher_future_BEV_feature', 'teacher_refine_flattned_BEV_feature',
              'teacher_refine_BEV_feature', 'refine_BEV_feature', 'pred_wp'):
        assert pred[k].shape == want[k].shape, k
        assert rel(pred[k].numpy(), want[k].numpy()) < TOL, k


def test_a_batch_without_supervision_keeps_the_inference_route(emu):
    cfg = loss_config()
    o, batch = oracle_and_batch(cfg, 1, seed=0)
    plain = {k: v for k, v in batch.items() if k not in ('waypoints', 'action_mu')}
    m = product(cfg, o)
    out = m.forward(is_eval=True, **plain)
    assert out['loss'] is None and out['log_vars'] == {} and 'pred' in out
    with pytest.raises(NotImplementedError):
        m.forward(is_eval=False, return_loss=True, **plain)


def test_depth_or_segmentation_supervision_raises(emu):
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    for key in ('use_depth', 'use_seg'):
        cfg = loss_config()
        cfg.merge_from_dict({f'model.train_cfg.{key}': True})
        o, batch = oracle_and_batch(cfg, 1, seed=0)
        m = product(cfg, o)
        with pytest.raises(NotImplementedError, match='depth_loss' if key == 'use_depth' else 'seg_loss'):
            m.forward(is_eval=True, **batch)
    assert Config.fromfile(PLUMBING_CONFIG).model.train_cfg['use_depth']      # the shipped config trains the camera branch


def test_loss_term_struct_matches_the_header(tmp_path):
    """offsets and size of every tt_loss_term field as a C compiler lays the header out vs the ctypes mirror in lib.py."""
    from thinktwice_b200 import lib
    cc = shutil.which('cc') or shutil.which('gcc')
    if cc is None:
        pytest.skip('no C compiler')
    fields = [n for n, _ in lib.LossTerm._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "tt_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof(tt_loss_term, {n}));\n' for n in fields) +
                   '  printf("%zu\\n%d\\n", sizeof(tt_loss_term), TT_LOSS_MAX_DIM);\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call([cc, '-I', os.path.join(os.path.dirname(HERE), 'include'), str(src), '-o', str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    want = [getattr(lib.LossTerm, n).offset for n in fields] + [ctypes.sizeof(lib.LossTerm), lib.LOSS_MAX_DIM]
    assert got == want
    assert (lib.LOSS_SMOOTH_L1, lib.LOSS_SMOOTH_L1_CLAMP, lib.LOSS_L1, lib.LOSS_BETA_KL, lib.LOSS_ACTION_L1) == (0, 1, 2, 3, 4)


def test_new_entry_points_fail_loudly_without_cuda():
    """the wrappers refuse host tensors, and the entry point itself, given well-formed arguments, returns an error status (no device)."""
    from thinktwice_b200 import lib
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    assert {'tt_loss_workspace_bytes', 'tt_loss_reduce'} <= set(lib.EXPORTS)
    with pytest.raises(lib.TTError):
        lib._p(torch.zeros(1))
    if not os.path.exists(lib.LIB_PATH):
        pytest.skip('libtt_b200.so not built')
    L = lib.load()
    terms = lib.pack_loss_terms([dict(kind=lib.LOSS_L1, slot=0, scale=0.25, shape=[4], aux=0, pred=ctypes.c_void_p(256), pred_stride=[1],
                                      pred2=None, gt=None, gt_stride=[0], gt2=None)])
    rc = L.tt_loss_reduce(terms, 1, ctypes.c_void_p(512), 1, ctypes.c_void_p(4096), ctypes.c_size_t(L.tt_loss_workspace_bytes(1)),
                          ctypes.c_void_p(0))
    with pytest.raises(lib.TTError, match='tt_loss_reduce'):
        lib.check(rc, 'tt_loss_reduce')


def _bad(batch, key, value):
    return dict(batch, **{key: value})


def test_malformed_ground_truth_raises(emu):
    """ground truth that does not match the prediction it is compared with, or Beta parameters outside (0, inf), raise ValueError
    before anything is staged (the reference raises in F.smooth_l1_loss / torch.distributions.Beta); nothing reaches the kernel."""
    cfg = loss_config()
    o, batch = oracle_and_batch(cfg, 2, seed=0)
    m = product(cfg, o)
    grid = list(batch['grid_feature'])
    grid[2] = grid[2][..., :20, :20].contiguous()
    fut_grid = [list(f) for f in batch['future_grid_feature']]
    fut_grid[1][2] = fut_grid[1][2][:, :16]
    neg_mu = batch['action_mu'].clone()
    neg_mu[1, 0] = -0.5
    fut_sigma = list(batch['future_action_sigma'])
    fut_sigma[0] = fut_sigma[0].clone()
    fut_sigma[0][0, 1] = float('-inf')
    zero_sigma = batch['action_sigma'].clone()
    zero_sigma[0, 0] = 0.0
    cases = [('feature', batch['feature'][:, :128], 'feature'), ('grid_feature', grid, r'grid_feature\[2\]'),
             ('future_grid_feature', fut_grid, r'future_grid_feature\[1\]'), ('waypoints', batch['waypoints'][:, :3], 'waypoints'),
             ('value', batch['value'][:1], 'value'), ('action_mu', neg_mu, 'action_mu'),
             ('future_action_sigma', fut_sigma, r'future_action_sigma\[0\]'), ('action_sigma', zero_sigma, 'action_sigma')]
    calls = []
    reduce = emu.tt_loss_reduce
    emu.tt_loss_reduce = lambda *a: calls.append(1) or reduce(*a)
    for key, value, match in cases:
        with pytest.raises(ValueError, match=match):
            m.forward(is_eval=True, **_bad(batch, key, value))
    assert not calls
    out = m.forward(is_eval=True, **batch)                             # the same model still validates a well-formed batch
    assert calls == [1] and np.isfinite(out['log_vars']['loss'])


# ---------------------------------------------------------------------------------------------- _parse_losses across ranks
def _rank(rank, world, path, q):
    import torch.distributed as dist
    from thinktwice_b200.encoder_decoder_framework import EncoderDecoder
    dist.init_process_group('gloo', init_method=f'file://{path}', rank=rank, world_size=world)
    try:
        losses = {'a_loss': torch.tensor(1.0 + rank), 'value_loss': torch.tensor([[2.0 * rank], [4.0]]), 'lateral_offset': torch.tensor(3.0 * rank)}
        loss, log_vars = EncoderDecoder._parse_losses(losses)
        q.put((rank, float(loss), dict(log_vars)))
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_average_the_log_vars(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, 2, str(tmp_path / 'rdv'), q)) for r in range(2)]
    for p in procs:
        p.start()
    out = dict((r, (l, v)) for r, l, v in (q.get(timeout=120) for _ in procs))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r, (loss, lv) in out.items():
        # rank r: a_loss 1 + r, value_loss mean (r + 2), lateral_offset 3r; loss = a_loss + value_loss (the offset is not a loss)
        assert loss == pytest.approx((1.0 + r) + (r + 2.0))              # the local total is returned as is
        assert lv['a_loss'] == pytest.approx(1.5) and lv['value_loss'] == pytest.approx(2.5)
        assert lv['lateral_offset'] == pytest.approx(1.5) and lv['loss'] == pytest.approx(4.0)
