"""CPU side of the training-side batch norm (include/tt_b200.h §18, thinktwice_b200/ops/batch_norm.py): the ctypes descriptor against
gcc, the library's refusals (each named, before any pointer or device is touched), the float64 restatement against torch autograd in
float64 (forward, running statistics, the backward with ReLU and residual, SyncBatchNorm's per-rank grad_weight over an R-way split),
seeded bugs each caught, and convert_batchnorm on the oracle model."""
import ctypes as C
import os
import subprocess

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.modules.batchnorm import _BatchNorm

import batch_norm_train_reference as RB
from thinktwice_b200 import lib
from thinktwice_b200.ops import batch_norm as bn
from thinktwice_b200.ops.sparse_conv import SparseEncoder

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ctypes_descriptor_matches_the_c_header(tmp_path):
    cls, cname = lib.BatchNormTrainDesc, 'tt_batch_norm_train_desc'
    fields = [n for n, _ in cls._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "tt_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof({cname}, {n}));\n' for n in fields) +
                   f'  printf("%zu\\n", sizeof({cname}));\n  return 0;\n}}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(cls, n).offset for n in fields] + [C.sizeof(cls)]


def test_new_entries_are_exported():
    names = {'tt_batch_norm_train_workspace_bytes', 'tt_batch_norm_train_stats', 'tt_batch_norm_train_fold', 'tt_batch_norm_train_forward',
             'tt_batch_norm_train_backward_reduce', 'tt_batch_norm_train_backward'}
    assert names <= set(lib.EXPORTS)
    L = lib.load()
    assert all(hasattr(L, n) for n in names)


def _d(**kw):
    d = bn._desc(100, 64, R=2, count=150)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


REFUSED = [(dict(affine=0), 'affine'), (dict(track_running_stats=0), 'track_running_stats'), (dict(C=22), 'C'), (dict(C=0), 'C'),
           (dict(M=-1), 'M'), (dict(R=0), 'R'), (dict(eps=0.0), 'eps'), (dict(eps=float('nan')), 'eps'), (dict(act=2), 'act'),
           (dict(residual=2), 'residual'), (dict(training=3), 'training')]


@pytest.mark.parametrize('kw,named', REFUSED)
def test_the_library_refuses_batch_norms_it_does_not_build(kw, named):
    d = _d(**kw)
    L = lib.load()
    null = C.c_void_p(0)
    assert L.tt_batch_norm_train_workspace_bytes(C.byref(d)) == 0
    calls = (lambda: L.tt_batch_norm_train_stats(C.byref(d), null, null, null, C.c_size_t(1 << 30), null),
             lambda: L.tt_batch_norm_train_fold(C.byref(d), null, null, null, null, null, null),
             lambda: L.tt_batch_norm_train_forward(C.byref(d), null, null, null, null, null, null, null, null),
             lambda: L.tt_batch_norm_train_backward_reduce(C.byref(d), null, null, null, null, null, null, null, null, null, null, null,
                                                           C.c_size_t(1 << 30), null),
             lambda: L.tt_batch_norm_train_backward(C.byref(d), null, null, null, null, null, null, null, null, null, null, null))
    for call in calls:
        assert call() == -3                                              # TT_ERR_UNSUPPORTED
        assert named in L.tt_last_error().decode()


def test_a_short_workspace_and_a_training_backward_without_rows_are_refused():
    d = _d()
    L = lib.load()
    n = L.tt_batch_norm_train_workspace_bytes(C.byref(d))
    assert n > 0
    null = C.c_void_p(0)
    assert L.tt_batch_norm_train_stats(C.byref(d), null, null, null, C.c_size_t(n - 1), null) == -3
    assert 'ws_bytes' in L.tt_last_error().decode()
    assert L.tt_batch_norm_train_backward_reduce(C.byref(d), null, null, null, null, null, null, null, null, null, null, null,
                                                 C.c_size_t(n - 1), null) == -3
    assert 'ws_bytes' in L.tt_last_error().decode()
    d.count = 0
    assert L.tt_batch_norm_train_backward(C.byref(d), null, null, null, null, null, null, null, null, null, null, null) == -3
    assert 'count' in L.tt_last_error().decode()


@pytest.mark.parametrize('cls,kw,named', [(bn.BatchNorm2d, dict(num_features=22), 'C'), (bn.BatchNorm1d, dict(num_features=6), 'C'),
                                          (bn.BatchNorm2d, dict(num_features=16, affine=False), 'affine'),
                                          (bn.SyncBatchNorm, dict(num_features=16, track_running_stats=False), 'track_running_stats')])
def test_the_modules_refuse_at_construction_naming_the_parameter(cls, kw, named):
    with pytest.raises(lib.TTError, match=named):
        cls(**kw)


def test_cpu_non_fp32_and_3d_inputs_are_refused():
    m = bn.BatchNorm2d(8)
    with pytest.raises(lib.TTError):
        m(torch.randn(2, 8, 3, 3))
    with pytest.raises(lib.TTError):
        m(torch.randn(2, 8, 3, 3, requires_grad=True))
    with pytest.raises(lib.TTError):
        m.double()(torch.randn(2, 8, 3, 3, dtype=torch.float64))
    with pytest.raises(lib.TTError):
        bn.BatchNorm1d(8)(torch.randn(2, 8, 5))


# ----------------------------------------------------------------------------------------- the float64 restatement, pinned
def _case(M, Cc, seed=0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, Cc, generator=g, dtype=torch.float64) * 2 + shift
    r = torch.randn(M, Cc, generator=g, dtype=torch.float64)
    w = 1 + 0.3 * torch.randn(Cc, generator=g, dtype=torch.float64)
    b = 0.3 * torch.randn(Cc, generator=g, dtype=torch.float64)
    gy = torch.randn(M, Cc, generator=g, dtype=torch.float64)
    return x, r, w, b, gy


def _torch(x, r, w, b, gy, eps, relu, momentum=0.1, rm=None, rv=None):
    """torch autograd in float64: (y, grad_x, grad_r, grad_w, grad_b, running_mean, running_var)."""
    x, w, b = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    r = r.clone().requires_grad_(True) if r is not None else None
    rm = torch.zeros(x.shape[1], dtype=torch.float64) if rm is None else rm.clone()
    rv = torch.ones(x.shape[1], dtype=torch.float64) if rv is None else rv.clone()
    z = F.batch_norm(x, rm, rv, w, b, training=True, momentum=momentum, eps=eps)
    if r is not None:
        z = z + r
    y = torch.relu(z) if relu else z
    y.backward(gy)
    return y.detach(), x.grad, (r.grad if r is not None else None), w.grad, b.grad, rm, rv


def _close(a, b):
    return torch.allclose(a, b, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('relu,res', [(False, False), (True, False), (True, True), (False, True)])
@pytest.mark.parametrize('M,Cc,shift', [(37, 8, 0.0), (5, 4, 3.0), (200, 12, -20.0), (2, 4, 0.0)])
def test_the_restatement_equals_torch_autograd(relu, res, M, Cc, shift):
    x, r, w, b, gy = _case(M, Cc, shift=shift)
    r = r if res else None
    eps = 1e-3
    y, gx, gr, gw, gb, rm, rv = _torch(x, r, w, b, gy, eps, relu, momentum=0.01)
    assert _close(RB.forward(x, r, w, b, eps, relu), y)
    m0, v0 = RB.running(torch.zeros(Cc, dtype=torch.float64), torch.ones(Cc, dtype=torch.float64), x, eps, 0.01)
    assert _close(m0, rm) and _close(v0, rv)
    rgx, rgr, rgw, rgb = RB.backward(x, r, w, b, gy, eps, relu)
    assert _close(rgx, gx) and _close(rgw[0], gw) and _close(rgb[0], gb)
    assert (rgr is None) == (r is None) and (gr is None or _close(rgr, gr))


def test_momentum_none_is_the_cumulative_average():
    x, _, w, b, gy = _case(30, 8)
    rm, rv = torch.randn(8, dtype=torch.float64), torch.rand(8, dtype=torch.float64) + 0.5
    for nbt in (1, 2, 7):
        m = nn.BatchNorm1d(8, momentum=None).double().train()
        m.running_mean.copy_(rm)
        m.running_var.copy_(rv)
        m.num_batches_tracked.fill_(nbt - 1)
        m(x)
        want = RB.running(rm, rv, x, 1e-5, 1.0 / nbt)
        assert _close(want[0], m.running_mean) and _close(want[1], m.running_var)


@pytest.mark.parametrize('splits', [(30,), (12, 18), (7, 0, 23), (1, 1, 28)])
@pytest.mark.parametrize('relu,res', [(False, False), (True, True)])
def test_the_r_way_split_has_sync_batch_norms_gradient_semantics(splits, relu, res):
    """Each rank's grad_weight / grad_bias is the gradient through its own rows only (torch's SyncBatchNorm backward leaves them per
    rank), while grad_x is the gradient of the whole batch: autograd with one leaf copy of the affine parameters per rank."""
    x, r, w, b, gy = _case(sum(splits), 8, seed=2)
    r = r if res else None
    eps = 1e-5
    xl = x.clone().requires_grad_(True)
    mean, invstd, _, _ = RB.stats(xl, eps)
    xhat = (xl - mean) * invstd
    ws = [w.clone().requires_grad_(True) for _ in splits]
    bs = [b.clone().requires_grad_(True) for _ in splits]
    parts, lo = [], 0
    for m, wk, bk in zip(splits, ws, bs):
        z = wk * xhat[lo:lo + m] + bk + (r[lo:lo + m] if r is not None else 0)
        parts.append(torch.relu(z) if relu else z)
        lo += m
    torch.cat(parts).backward(gy)
    gx, _, gw, gb = RB.backward(x, r, w, b, gy, eps, relu, splits=splits)
    assert _close(gx, xl.grad)
    for k in range(len(splits)):
        assert _close(gw[k], ws[k].grad) and _close(gb[k], bs[k].grad), k


def test_each_seeded_bug_is_caught():
    x, r, w, b, gy = _case(40, 8, seed=3)
    b = b - 0.8                                                           # residual-dependent mask decisions
    eps = 1e-5
    _, gx, gr, gw, gb, rm, rv = _torch(x, r, w, b, gy, eps, True, momentum=0.1)
    m, v = RB.running(torch.zeros(8, dtype=torch.float64), torch.ones(8, dtype=torch.float64), x, eps, 0.1, bug='biased_running_var')
    assert _close(m, rm) and not torch.allclose(v, rv, rtol=1e-6, atol=1e-6)
    bgx, _, _, _ = RB.backward(x, r, w, b, gy, eps, True, bug='mask_without_residual')
    assert not torch.allclose(bgx, gx, rtol=1e-6, atol=1e-6)
    splits = (15, 25)
    _, _, good, _ = RB.backward(x, r, w, b, gy, eps, True, splits=splits)
    _, _, bad, _ = RB.backward(x, r, w, b, gy, eps, True, splits=splits, bug='global_grad_weight')
    assert _close(good[0] + good[1], gw)
    assert not torch.allclose(bad[0], good[0], rtol=1e-6, atol=1e-6)


# ----------------------------------------------------------------------------------------- convert_batchnorm
def _oracle():
    from oracle.model import EncoderDecoder as Oracle
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    cfg = Config.fromfile(DEFAULT_CONFIG)
    torch.manual_seed(0)
    return Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})


FUSED = (['img_encoder.depth_net.reduce_conv.1', 'img_encoder.depth_net.depth_conv.3.global_avg_pool.2'] +
         [f'img_encoder.seg_res_to_image_feature.{i}' for i in range(1, 20, 3)] +
         [f'lidar_encoder.pts_backbone.blocks.{j}.{i}' for j in (0, 1) for i in range(1, 17, 3)] +
         ['lidar_encoder.pts_neck.deblocks.0.1', 'lidar_encoder.pts_neck.deblocks.1.1', 'conv_cam.1', 'conv_lidar.1', 'conv_lidar.4',
          'conv_fusion.1'])


def test_convert_batchnorm_on_the_oracle_model():
    model = _oracle()
    before = {n: m for n, m in model.named_modules() if isinstance(m, _BatchNorm)}
    tensors = {n: (m.weight, m.bias, m.running_mean, m.running_var, m.num_batches_tracked) for n, m in before.items()}
    state = {k: v.clone() for k, v in model.state_dict().items()}
    out, skipped, fused = bn.convert_batchnorm(model)
    assert out is model
    assert [(n, why.split(':')[0]) for n, _, why in skipped] == [('img_encoder.depth_net.bn', 'C')]
    assert type(skipped[0][1]) is nn.BatchNorm1d and skipped[0][1].num_features == 22
    assert sorted(fused) == sorted(FUSED)
    after = dict(model.named_modules())
    assert len(before) == 124
    for n, m in before.items():
        new = after[n]
        assert isinstance(new, _BatchNorm), n
        if n == 'img_encoder.depth_net.bn':
            assert new is m
            continue
        assert type(new) is {nn.BatchNorm1d: bn.BatchNorm1d, nn.BatchNorm2d: bn.BatchNorm2d}[type(m)], n
        assert all(a is b for a, b in zip((new.weight, new.bias, new.running_mean, new.running_var, new.num_batches_tracked), tensors[n]))
        assert new.fused_relu == (n in FUSED) and (new.eps, new.momentum) == (m.eps, m.momentum)
    for n in FUSED:                                                       # the ReLU after each fused layer is gone
        parent, idx = n.rsplit('.', 1)
        assert type(after[f'{parent}.{int(idx) + 1}']) is nn.Identity
    assert list(model.state_dict()) == list(state)
    for k, v in model.state_dict().items():
        assert torch.equal(v, state[k]), k


def test_convert_batchnorm_on_the_trainable_sparse_encoder_and_sync_layers():
    enc = SparseEncoder(4, [41, 1600, 1408])
    _, skipped, fused = bn.convert_batchnorm(enc)
    assert skipped == [] and sorted(fused) == sorted(['conv_input.1', 'encoder_layers.encoder_layer1.0.1', 'encoder_layers.encoder_layer2.2.1',
                                                      'encoder_layers.encoder_layer3.2.1', 'conv_out.1'])
    assert type(enc.encoder_layers.encoder_layer2[0].bn2) is bn.BatchNorm1d and not enc.encoder_layers.encoder_layer2[0].bn2.fused_relu
    group = object()
    seq = nn.Sequential(nn.SyncBatchNorm(8, momentum=None, process_group=group), nn.ReLU(), nn.BatchNorm2d(8, affine=False), nn.ReLU(),
                        nn.SyncBatchNorm(16))
    seq[0].eval()
    _, skipped, fused = bn.convert_batchnorm(seq, fuse_relu=False)
    assert fused == [] and type(seq[1]) is nn.ReLU
    assert type(seq[0]) is bn.SyncBatchNorm and seq[0].process_group is group and seq[0].momentum is None and not seq[0].training
    assert isinstance(seq[0], nn.SyncBatchNorm) and isinstance(seq[4], _BatchNorm)
    assert [(n, why.split(':')[0]) for n, _, why in skipped] == [('2', 'affine')]
    _, _, fused = bn.convert_batchnorm(seq)
    assert fused == ['0'] and type(seq[1]) is nn.Identity and type(seq[3]) is nn.ReLU
    bare, skipped, fused = bn.convert_batchnorm(nn.BatchNorm2d(8))
    assert type(bare) is bn.BatchNorm2d and skipped == [] and fused == []
