"""CPU side of the training losses (include/tt_b200.h §10b and §15, thinktwice_b200/ops/losses.py): the float64 gradient references
of tests/loss_train_reference.py pinned against the header's per-element formulas on crafted edge cases, the gradient check rejecting
seeded bugs, the ctypes layouts against gcc, and every refusal of the library and of the Python ops."""
import ctypes as C
import os
import subprocess

import pytest
import torch

import loss_train_reference as R
from thinktwice_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------------ camera
def camera_case(BN=3, Cn=12, h=6, w=8, D=80, f=4, seed=0):
    """small logits / ground truth with the edge cases in place: frame 1 all ignored, a NaN depth block, depths on bin edges (bin
    value exactly an integer, 0 and D + 1), zero depths (1e5: background)"""
    g = torch.Generator().manual_seed(seed)
    seg = torch.randn(BN, Cn, h, w, generator=g, dtype=torch.float64) * 3
    lab = torch.randint(0, Cn, (BN, 1, 2 * h, 2 * w), generator=g).double()
    lab[:, :, ::3] = R.IGNORE
    lab[1] = R.IGNORE                                                  # an all-ignored frame
    depth = torch.randn(BN, D, h, w, generator=g, dtype=torch.float64) * 2
    d0, _, step = R.DBOUND
    k = torch.randint(-2, D + 3, (BN, 1, f * h, f * w), generator=g).double()
    dg = (d0 - step) + step * k                                        # every bin value an integer: the bin edges
    dg[0, 0, :f, :f] = (d0 - step) + step * 7
    dg[0, 0, 1, 2] = float('nan')                                      # one NaN pixel makes its block background
    dg[0, 0, f:2 * f, :f] = 0.0                                        # all zero -> 1e5 -> background
    dg[0, 0, :f, f:2 * f] = (d0 - step) + step * (D + 1)               # the top edge: excluded
    dg[0, 0, f:2 * f, f:2 * f] = (d0 - step)                           # bin value 0: background
    return seg, depth, lab.float(), dg.float(), f


@pytest.mark.parametrize('nan_logit', [False, True])
def test_camera_reference_equals_the_formula(nan_logit):
    seg, depth, lab, dg, f = camera_case()
    if nan_logit:
        seg[2, 3, 1, 1] = float('nan')                                 # a counted pixel: every counted pixel's gradient NaN
    up = (0.7, -1.3)
    vals, gs, gd = R.camera_ref(seg, depth, lab, dg, f=f, up=up)
    fs, fd = R.camera_formula(seg, depth, lab, dg, f=f, up=up)
    assert torch.equal(torch.isnan(gs), torch.isnan(fs)) and bool(torch.isnan(gs).any()) == nan_logit
    assert (gs[:, :, 0] == 0).all()                                    # ignored pixels get 0 even then
    assert torch.allclose(gs.nan_to_num(), fs.nan_to_num(), rtol=1e-12, atol=1e-15)
    assert torch.allclose(gd, fd, rtol=1e-12, atol=1e-15)
    assert (gs[1] == 0).all()                                          # the all-ignored frame
    bins = R.depth_bins(dg, f, 80).reshape(3, 6, 8)
    assert bins[0, 0, 0] == 0 and bins[0, 1, 0] == 0 and bins[0, 0, 1] == 0 and bins[0, 1, 1] == 0
    assert (gd[0, :, 0, 0] == 0).all() and (gd[0, :, 1, 1] == 0).all()  # NaN block, bin value 0


def test_camera_reference_all_ignored_batch():
    seg, depth, lab, dg, f = camera_case()
    lab[:] = R.IGNORE
    vals, gs, _ = R.camera_ref(seg, depth, lab, dg, f=f)
    fs, _ = R.camera_formula(seg, depth, lab, dg, f=f)
    assert vals[0] != vals[0] and (gs == 0).all() and (fs == 0).all()   # a NaN loss (0 / 0) whose gradient is 0: no pixel counted


def test_camera_check_rejects_seeded_bugs():
    seg, depth, lab, dg, f = camera_case()
    _, gs, gd = R.camera_ref(seg, depth, lab, dg, f=f)
    ss, sd = R.camera_scale(seg, depth, lab, dg, f=f)
    fs, fd = R.camera_formula(seg.float().double(), depth.float().double(), lab, dg, f=f)
    assert R.ratio(fs.float(), gs, R.EPS * ss) < 1 and R.ratio(fd.float(), gd, R.EPS * sd) < 1
    for bug in ('gradient on ignored pixels', "f' second term missing", 'gradient on background cells', 'NaN block treated as foreground'):
        bs, bd = R.camera_formula(seg, depth, lab, dg, f=f, bug=bug)
        worst = max(R.ratio(bs.float(), gs, R.EPS * ss), R.ratio(bd.float(), gd, R.EPS * sd))
        assert worst > 1, bug


# ------------------------------------------------------------------------------------------------------------------ decoder
def test_decoder_reference_equals_the_formula():
    pred, mid, batch = R.make_inputs(2, seed=3, quarter=True)
    pred['refine_BEV_feature'][0, 0, 0, 0, :6] = batch['grid_feature'][2][0, 0, 0, :6] + torch.tensor([0, 1, -1, 5.5, -5.5, 5.75],
                                                                                                        dtype=torch.float64)
    pred['teacher_pred_wp_offset'][0, 0, 0] = torch.tensor([0.0, 1.0], dtype=torch.float64)
    pred['pred_speed'][0, 0] = batch['speed'][0] / 12 + 5.5
    vals, G, w = R.decoder_ref(pred, mid, batch)
    Fm = R.decoder_formula(pred, mid, batch, w)
    for k in G:
        assert torch.allclose(G[k], Fm[k], rtol=1e-10, atol=1e-16), k
    rb = G['refine_BEV_feature'][0, 0, 0, 0, :6] / (w['refine_BEV_feature_loss2'] * R.LO.DISTIL[2] / pred['refine_BEV_feature'].numel())
    assert rb.tolist() == [0.0, 1.0, -1.0, 1.0, -1.0, 0.0]             # smooth-L1 at 0, 1; the clamp passes 5 (|d| = 5.5), not 5.25
    assert G['teacher_pred_wp_offset'][0, 0, 0].tolist()[0] == 0.0
    assert float(G['pred_speed'][0, 0]) > 0                            # plain smooth-L1 at |d| = 5.5: no clamp


def test_decoder_nan_and_clamp_boundary_against_torch():
    d = torch.tensor([5.5, -5.5, 5.5 + 2 ** -20, float('nan'), 1.0, -1.0, 0.0], dtype=torch.float64, requires_grad=True)
    torch.clamp(torch.nn.functional.smooth_l1_loss(d, torch.zeros_like(d), reduction='none'), min=-5.0, max=5.0).sum().backward()
    ours = torch.where(R.clamp_pass(d.detach()), 1.0, 0.0) * R.sl1p(d.detach())
    assert torch.equal(torch.isnan(ours), torch.isnan(d.grad)) and torch.equal(ours.nan_to_num(), d.grad.nan_to_num())
    assert d.grad[:3].tolist() == [1.0, -1.0, 0.0] and d.grad[3] != d.grad[3]


def test_decoder_check_rejects_seeded_bugs():
    pred, mid, batch = R.make_inputs(3, seed=5, quarter=True)
    pred['refine_BEV_feature'][0, 0, 0, 0, :2] = batch['grid_feature'][2][0, 0, 0, :2] + torch.tensor([5.5, -5.5], dtype=torch.float64)
    _, G, w = R.decoder_ref(pred, mid, batch)
    S = R.decoder_scale(pred, mid, batch, w)
    good = R.decoder_formula(pred, mid, batch, w)
    assert max(R.ratio(good[k].float(), G[k], R.EPS * S[k]) for k in G) < 1
    for bug in ('clamp boundary excluded', 'v_traj fed by one slot'):
        bad = R.decoder_formula(pred, mid, batch, w, bug=bug)
        assert max(R.ratio(bad[k].float(), G[k], R.EPS * S[k]) for k in G) > 1, bug


# ------------------------------------------------------------------------------------------------------------------ the C ABI
def _layout(tmp_path, struct, cls):
    fields = [n for n, _ in cls._fields_]
    src = tmp_path / f'{struct}.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "tt_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof({struct}, {n}));\n' for n in fields) +
                   f'  printf("%zu\\n", sizeof({struct}));\n  return 0;\n}}\n')
    exe = tmp_path / struct
    subprocess.check_call(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(cls, n).offset for n in fields] + [C.sizeof(cls)], struct


def test_ctypes_layouts_match_the_c_header_and_the_entries_are_exported(tmp_path):
    _layout(tmp_path, 'tt_camera_loss_train_desc', lib.CameraLossTrainDesc)
    _layout(tmp_path, 'tt_camera_loss_stats', lib.CameraLossStats)
    _layout(tmp_path, 'tt_loss_grad', lib.LossGrad)
    names = ('tt_loss_backward_workspace_bytes', 'tt_loss_backward', 'tt_camera_loss_train_workspace_bytes', 'tt_camera_loss_train_forward',
             'tt_camera_loss_train_backward')
    assert set(names) <= set(lib.EXPORTS)
    L = lib.load()
    assert all(hasattr(L, n) for n in names)


def _cam_desc(**kw):
    d = lib.CameraLossTrainDesc()
    base = dict(BN=64, seg_h=224, seg_w=448, seg_H=448, seg_W=896, seg_classes=12, seg_ignore=255, seg_alpha=0.5, seg_gamma=2.0,
                seg_weight=10.0, depth_h=28, depth_w=56, depth_factor=16, depth_bins=80, depth_offset=0.5, depth_step=0.5,
                seg_logits=16, seg_gt=16, depth_logits=16, depth_gt=16)
    base.update(kw)
    d.seg_stride = (C.c_longlong * 4)(*base.pop('seg_stride', (12 * 224 * 448, 224 * 448, 448, 1)))
    d.depth_stride = (C.c_longlong * 4)(*base.pop('depth_stride', (336 * 28 * 56, 28 * 56, 56, 1)))
    for k, v in base.items():
        setattr(d, k, v)
    return d


def _cam_calls(L, d, ws_bytes=0):
    null = C.c_void_p(0)
    return (lambda: L.tt_camera_loss_train_forward(C.byref(d), null, null, null, null, null, C.c_size_t(ws_bytes), null),
            lambda: L.tt_camera_loss_train_backward(C.byref(d), null, null, null, null, null, null, null))


@pytest.mark.parametrize('kw,named', [
    (dict(seg_classes=33), 'seg_classes'), (dict(depth_bins=256), 'depth_bins'),
    (dict(seg_stride=(12 * 224 * 448, 224 * 448, 448, 2)), 'seg_stride'), (dict(seg_stride=(12 * 224 * 448, 224 * 448, 450, 1)), 'seg_stride'),
    (dict(depth_stride=(80, 1, 56 * 80, 80)), 'depth_stride'), (dict(BN=2000), 'BN, seg_classes, seg_h, seg_w'),
    (dict(BN=6000, seg_logits=0), 'BN, depth_factor')])
def test_the_camera_entries_refuse_what_they_cannot_index(kw, named):
    """checked before any pointer or device is touched: no GPU needed, nothing launched"""
    L = lib.load()
    d = _cam_desc(**kw)
    n0 = L.tt_launch_count()
    for call in _cam_calls(L, d, 1 << 20):
        assert call() == -3
        assert f'unsupported {named}' in L.tt_last_error().decode()
    assert L.tt_launch_count() == n0


def test_a_short_camera_workspace_is_refused_and_an_empty_batch_launches_nothing():
    L = lib.load()
    d = _cam_desc()
    n = L.tt_camera_loss_train_workspace_bytes(C.byref(d))
    n0 = L.tt_launch_count()
    assert _cam_calls(L, d, n - 1)[0]() == -3 and 'unsupported ws_bytes' in L.tt_last_error().decode()
    e = _cam_desc(BN=0)
    assert all(call() == 0 for call in _cam_calls(L, e, n))
    assert L.tt_launch_count() == n0


def _term(kind=lib.LOSS_SMOOTH_L1, shape=(4,), slot=0):
    return dict(kind=kind, slot=slot, scale=0.25, shape=list(shape), aux=0, pred=C.c_void_p(256), pred_stride=[1] * len(shape),
                pred2=C.c_void_p(512), gt=C.c_void_p(1024), gt2=C.c_void_p(2048), gt_stride=[1] * len(shape))


def _grad(ptr, stride=(1,), slot=0, count=1, ptr2=0):
    return dict(grad_pred=C.c_void_p(ptr), grad_pred2=C.c_void_p(ptr2), grad_stride=list(stride), up_slot=slot, up_count=count)


@pytest.mark.parametrize('case,rc,msg', [
    ('l1 with a gradient', -3, 'L1 / ACTION_L1'), ('two terms overlap', -3, 'overlaps term 0'),
    ('pred and pred2 overlap', -3, 'term 1 overlaps term 1'), ('broadcast gradient', -3, 'two elements to one address'),
    ('slots past n_slots', -1, 'bad term'), ('short workspace', -1, 'workspace too small')])
def test_tt_loss_backward_refusals(case, rc, msg):
    L = lib.load()
    terms, grads, n_slots, ws = [_term(), _term()], [_grad(4096), _grad(8192)], 2, None
    if case == 'l1 with a gradient':
        terms[1]['kind'] = lib.LOSS_L1
    elif case == 'two terms overlap':
        grads[1] = _grad(4096 + 12)
    elif case == 'pred and pred2 overlap':
        terms[1]['kind'] = lib.LOSS_BETA_KL
        grads[1] = _grad(8192, ptr2=8192 + 8)
    elif case == 'broadcast gradient':
        grads[1] = _grad(8192, stride=(0,))
    elif case == 'slots past n_slots':
        grads[1] = _grad(8192, slot=1, count=2)
    elif case == 'short workspace':
        ws = L.tt_loss_backward_workspace_bytes(2) - 1
    n = ws if ws is not None else L.tt_loss_backward_workspace_bytes(2)
    n0 = L.tt_launch_count()
    got = L.tt_loss_backward(lib.pack_loss_terms(terms), 2, lib.pack_loss_grads(grads), C.c_void_p(64), n_slots, C.c_void_p(128),
                             C.c_size_t(n), C.c_void_p(0))
    assert got == rc and msg in L.tt_last_error().decode()
    assert L.tt_launch_count() == n0


def test_ops_refuse_cpu_tensors():
    from thinktwice_b200.ops.losses import camera_losses, decoder_loss
    model = type('M', (), dict(use_seg=True, use_depth=False, seg_downsample_factor=2))()
    with pytest.raises(lib.TTError, match='CUDA'):
        camera_losses(model, dict(seg=torch.zeros(1, 1, 4, 4)), dict(seg=torch.zeros(1, 12, 2, 2)))
    pred, mid, batch = R.make_inputs(1, seed=0)
    with pytest.raises(lib.TTError, match='CUDA'):
        decoder_loss(R.decoder_module(), batch, {k: v.float() for k, v in pred.items()}, [m if m is None else m.float() for m in mid])
