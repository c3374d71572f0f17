"""The camera branch's supervision (seg_loss, depth_loss) without a GPU.

  * tests/camera_loss_oracle.py reproduces tests/golden/ref_camera_losses_*.npz, which the reference's own forward_train / _parse_losses produced
    with train_cfg use_depth = use_seg = True (tests/golden/make_camera_loss_golden.py);
  * the product's host code — ground-truth checks, staging, the tt_camera_loss descriptor, forward_train's key order — through the
    emulated C ABI (tests/emu_lib.py + tests/emu_losses.py + tests/emu_camera_losses.py) matches the oracle, in both Look modes;
  * tests/camera_loss_checks.py, the GPU test's checks of the kernel, accept the emulation and reject each of its seeded bugs;
  * the nearest-index formula is torchvision's T.Resize(NEAREST), the fp32 bin arithmetic is torch's at the bin edges, and the ctypes
    mirror of tt_camera_loss_desc has the header's layout."""
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

TOL = 5e-4


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-6))


def camera_config(use_seg=True, use_depth=True):
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    cfg = Config.fromfile(PLUMBING_CONFIG)
    cfg.merge_from_dict({'model.train_cfg.use_seg': use_seg, 'model.train_cfg.use_depth': use_depth})
    return cfg


def oracle_and_batch(cfg, B, seed, points=1500):
    from test_losses_cpu import oracle_and_batch as ob
    from thinktwice_b200.synthetic import make_camera_supervision
    o, batch = ob(cfg, B, seed, points)
    batch.update(make_camera_supervision(cfg, B, seed=seed))
    return o, batch


# ---------------------------------------------------------------------------------------------- the oracle vs the reference's code
@pytest.mark.parametrize('seed', [0, 1])
def test_oracle_camera_losses_equal_the_reference_code(seed):
    import camera_loss_oracle
    import loss_oracle
    from make_camera_loss_golden import CASES
    f = np.load(os.path.join(G, f'ref_camera_losses_plumbing_seed{seed}.npz'))
    B = dict(CASES)[seed]
    assert int(f['batch']) == B
    o, batch = oracle_and_batch(camera_config(), B, seed)
    losses, _ = camera_loss_oracle.forward_train(o.eval(), batch)
    assert list(losses) == list(f['keys']) and list(losses)[-2:] == ['seg_loss', 'depth_loss']
    for k, v in losses.items():
        assert rel(v.numpy(), f['loss.' + k]) < 1e-5, k
    _, log_vars = loss_oracle.parse_losses(losses)
    assert list(log_vars) == [n[len('log.'):] for n in f['log_keys']]
    for k, v in log_vars.items():
        assert rel(v, f['log.' + k]) < 1e-5, k


# ---------------------------------------------------------------------------------------------- the product's host code, emulated ABI
@pytest.fixture
def emu(emulated, monkeypatch):
    import gc
    import emu_frames
    import emu_lib
    import emu_camera_losses
    import emu_losses
    emu_lib._by_addr.clear()
    gc.collect()
    yield emu_camera_losses.install(emu_losses.install(emu_frames.install(emulated), monkeypatch), monkeypatch)
    emu_lib._by_addr.clear()
    gc.collect()


def product(cfg, o, independent=False):
    from test_losses_cpu import product as p
    return p(cfg, o, independent)


@pytest.mark.parametrize('independent', [False, True], ids=['coupled', 'independent'])
@pytest.mark.parametrize('B', [1, 2])
def test_emulated_forward_with_camera_supervision_matches_the_oracle(emu, B, independent):
    import camera_loss_oracle
    import loss_oracle
    cfg = camera_config()
    o, batch = oracle_and_batch(cfg, B, seed=1)
    want, _ = camera_loss_oracle.forward_train(o.eval(), batch, independent_frames=independent)
    _, want_log = loss_oracle.parse_losses(want)
    m = product(cfg, o, independent)
    out = m.forward(is_eval=True, **batch)
    assert list(out['log_vars']) == list(want_log) and list(want_log)[-3:] == ['seg_loss', 'depth_loss', 'loss']
    for k, v in want_log.items():
        assert rel(out['log_vars'][k], v) < TOL, (k, out['log_vars'][k], v)
    assert rel(float(out['loss']), want_log['loss']) < TOL
    got = m.forward_train(batch)
    for k in ('seg_loss', 'depth_loss'):
        assert got[k].dim() == 0 and got[k].dtype == torch.float32
        assert rel(got[k].numpy(), want[k].numpy()) < TOL, k


@pytest.mark.parametrize('flag', ['use_seg', 'use_depth'])
def test_only_the_enabled_term_appears(emu, flag):
    import camera_loss_oracle
    import loss_oracle
    cfg = camera_config(use_seg=flag == 'use_seg', use_depth=flag == 'use_depth')
    o, batch = oracle_and_batch(cfg, 1, seed=0)
    want, _ = camera_loss_oracle.forward_train(o.eval(), batch)
    m = product(cfg, o)
    got = m.forward_train(batch)
    name = 'seg_loss' if flag == 'use_seg' else 'depth_loss'
    assert list(got) == list(want) and list(got)[-1] == name and ({'seg_loss', 'depth_loss'} - {name}).isdisjoint(got)
    assert rel(got[name].numpy(), want[name].numpy()) < TOL


def test_a_batch_without_the_camera_ground_truth_raises(emu):
    cfg = camera_config()
    o, batch = oracle_and_batch(cfg, 1, seed=0)
    m = product(cfg, o)
    for key, name in (('depth', 'depth_loss'), ('seg', 'seg_loss')):
        with pytest.raises(NotImplementedError, match=name):
            m.forward(is_eval=True, **{k: v for k, v in batch.items() if k != key})


def test_malformed_camera_ground_truth_raises_before_anything_is_staged(emu):
    """depth not (B, N, 16 h, 16 w), seg not (B, N, H, W) with H // 2 = h and W // 2 = w, a non-finite label the loss reads, a label that
    truncates outside [0, C) and is not 255: ValueError, and neither loss kernel nor any ground-truth upload has run."""
    cfg = camera_config()
    o, batch = oracle_and_batch(cfg, 2, seed=0)
    m = product(cfg, o)
    d, s = batch['depth'], batch['seg']
    nan_lab, big_lab, neg_lab, ok_lab = s.clone(), s.clone(), s.clone(), s.clone()
    nan_lab[1, 2, 10, 6] = float('nan')                               # an even row / column: a pixel the resize reads
    big_lab[0, 0, 0, 0] = 12.0                                        # C = 12 classes
    neg_lab[0, 3, 4, 4] = -1.0
    ok_lab[1, 2, 11, 7] = float('nan')                                # an odd row / column: never read, as in the reference
    ok_lab[0, 0, 2, 2] = -0.5                                         # truncates to class 0
    cases = [('depth', d[..., :-16], 'depth'), ('depth', d[:, :3], 'depth'), ('seg', s[..., :-2, :], 'seg'), ('seg', s[:1], 'seg'),
             ('seg', nan_lab, 'not finite'), ('seg', big_lab, 'labels'), ('seg', neg_lab, 'labels')]
    calls = []
    for fn in ('tt_loss_reduce', 'tt_camera_loss'):
        real = getattr(emu, fn)
        setattr(emu, fn, lambda *a, real=real, fn=fn: calls.append(fn) or real(*a))
    for key, value, match in cases:
        m.eng.cur.pop('gt.seg', None), m.eng.cur.pop('gt.depth', None), m.eng.cur.pop('gt.speed', None)
        with pytest.raises(ValueError, match=match):
            m.forward(is_eval=True, **dict(batch, **{key: value}))
        assert not calls and not {'gt.seg', 'gt.depth', 'gt.speed'} & set(m.eng.cur), key
    out = m.forward(is_eval=True, **dict(batch, seg=ok_lab))          # an odd (+0.5 scale) pixel is not read; -0.5 is class 0
    assert calls == ['tt_loss_reduce', 'tt_camera_loss'] and np.isfinite(out['log_vars']['seg_loss'])
    # a shape one odd pixel larger still downsamples to the map: H // 2 == h
    odd = torch.cat([s, s[..., -1:, :]], 2)
    out = m.forward(is_eval=True, **dict(batch, seg=odd))
    assert np.isfinite(out['log_vars']['seg_loss'])


# ---------------------------------------------------------------------------------------------- the kernel's checks on the emulation
def test_the_kernel_checks_accept_the_emulation(emu):
    import camera_loss_checks
    out = camera_loss_checks.check_all('cpu')
    (got, want) = out['edges']
    assert np.isfinite(want).all() and want[1] > 0                    # the crafted case has foreground cells and valid pixels


@pytest.mark.parametrize('bug', ['nan_dropping_min', 'ce_all_pixels', 'no_max1', 'bin_off_by_one', 'read_past_C', 'per_pixel_focal'])
def test_the_kernel_checks_reject_a_seeded_bug(emu, monkeypatch, bug):
    import camera_loss_checks
    import emu_camera_losses
    monkeypatch.setattr(emu_camera_losses, 'BUG', bug)
    with pytest.raises(AssertionError):
        camera_loss_checks.check_all('cpu')


@pytest.mark.parametrize('H', [256, 257, 448, 449, 33])
def test_nearest_index_is_torchvisions_resize(H):
    """the kernel's source index (identity / k >> 1 / floor(k * (float)H / h) clamped) is the pixel T.Resize(NEAREST) picks, for even
    and odd H."""
    T = pytest.importorskip('torchvision.transforms')
    from emu_camera_losses import nearest_index
    h, W = H // 2, 6
    src = torch.arange(H, dtype=torch.float32).view(1, H, 1).expand(1, H, W).contiguous()
    got = T.Resize((h, W // 2), interpolation=T.InterpolationMode.NEAREST)(src)[0, :, 0].long()
    assert torch.equal(got, nearest_index(h, H))
    assert torch.equal(nearest_index(H, H), torch.arange(H)) and torch.equal(nearest_index(2 * H, H), torch.arange(2 * H) >> 1)


@pytest.mark.parametrize('d_bound', [[1.0, 9.0, 1.0], [1.0, 41.0, 0.5]])
def test_fp32_bin_arithmetic_equals_torch_at_the_edges(d_bound):
    """(d - (d0 - step)) / step in fp32, then [0, D + 1) and .long(): the bins of the oracle's get_downsampled_gt_depth (torch) and of
    the emulation's kernel formula agree at every bin edge and one fp32 ulp either side."""
    import camera_loss_oracle
    import loss_oracle
    d0, d1, step = d_bound
    D = int((d1 - d0) / step)
    edges = torch.tensor([(d0 - step) + v * step for v in range(D + 3)], dtype=torch.float32)
    vals = torch.cat([edges, torch.nextafter(edges, edges + 1), torch.nextafter(edges, edges - 1), torch.tensor([0.0, float('nan'), -1.0])])
    f = 1
    gt = vals.view(1, 1, 1, -1)
    onehot = camera_loss_oracle.downsampled_gt_depth(gt, f, d_bound, D)            # (n, D): class 0 dropped
    want = torch.where(onehot.sum(1) > 0, onehot.argmax(1) + 1, torch.zeros(len(vals), dtype=torch.long))
    v = (torch.where(vals == 0, torch.full_like(vals, 1e5), vals) - torch.tensor(d0 - step, dtype=torch.float32)) / torch.tensor(step, dtype=torch.float32)
    got = torch.where((v >= 0) & (v < D + 1), v, torch.zeros_like(v)).long()
    assert torch.equal(got, want)
    assert int(got[0]) == 0 and int(got[1]) == 1 and int(got[D]) == D and int(got[D + 1]) == 0      # v = 0, 1, D, D + 1


def test_camera_loss_desc_matches_the_header(tmp_path):
    from thinktwice_b200 import lib
    cc = shutil.which('cc') or shutil.which('gcc')
    if cc is None:
        pytest.skip('no C compiler')
    fields = [n for n, _ in lib.CameraLossDesc._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "tt_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof(tt_camera_loss_desc, {n}));\n' for n in fields) +
                   '  printf("%zu\\n", sizeof(tt_camera_loss_desc));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call([cc, '-I', os.path.join(os.path.dirname(HERE), 'include'), str(src), '-o', str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [getattr(lib.CameraLossDesc, n).offset for n in fields] + [ctypes.sizeof(lib.CameraLossDesc)]


def test_camera_loss_entry_fails_loudly_without_cuda():
    from thinktwice_b200 import lib
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    assert {'tt_camera_loss_workspace_bytes', 'tt_camera_loss'} <= set(lib.EXPORTS)
    if not os.path.exists(lib.LIB_PATH):
        pytest.skip('libtt_b200.so not built')
    L = lib.load()
    d = lib.camera_loss_desc(BN=1, seg_logits=ctypes.c_void_p(256), seg_gt=ctypes.c_void_p(512), seg_h=1, seg_w=1, seg_H=2, seg_W=2,
                             seg_ld=12, seg_classes=12, seg_ignore=255, seg_alpha=0.5, seg_gamma=2.0, seg_weight=10.0)
    rc = L.tt_camera_loss(lib.ref(d), ctypes.c_void_p(1024), ctypes.c_void_p(4096), ctypes.c_size_t(1 << 20), ctypes.c_void_p(0))
    with pytest.raises(lib.TTError, match='tt_camera_loss'):
        lib.check(rc, 'tt_camera_loss')
