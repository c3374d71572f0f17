"""CPU side of the training-side upsampling (include/tt_b200.h §17, thinktwice_b200/ops/conv_transpose2d.py and interpolate.py): the
ctypes descriptors against gcc, the library's refusals (each named, before any pointer or device is touched), the float64 restatements
of the transposed convolution (as the adjoint Conv2d) and of the gather-form bilinear backward against torch autograd in float64, seeded
bugs each caught, and convert_upsampling on the oracle model."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import conv_transpose2d_train_reference as RT
import interpolate_train_reference as RI
from thinktwice_b200 import lib
from thinktwice_b200.ops import conv_transpose2d as ct
from thinktwice_b200.ops import interpolate as ip

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('cls,cname', [(lib.ConvTranspose2dTrainDesc, 'tt_conv_transpose2d_train_desc'),
                                       (lib.InterpBilinearTrainDesc, 'tt_interp_bilinear_train_desc')])
def test_ctypes_descriptors_match_the_c_header(tmp_path, cls, cname):
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
    assert {'tt_conv_transpose2d_train_workspace_bytes', 'tt_conv_transpose2d_train_forward', 'tt_conv_transpose2d_train_backward',
            'tt_interp_bilinear_train_forward', 'tt_interp_bilinear_train_backward'} <= set(lib.EXPORTS)


def _t(**kw):
    g = dict(N=2, H=7, W=9, Cin=16, Cout=32, k=(2, 2), s=2, p=0, op=0, dil=1, groups=1, bias=True)
    g.update(kw)
    return ct._desc(g['N'], g['H'], g['W'], g['Cin'], g['Cout'], g['k'], g['s'], g['p'], g['op'], g['dil'], g['groups'], g['bias'])


def _with(d, **kw):
    for k, v in kw.items():
        setattr(d, k, v)
    return d


T_REFUSED = [(lambda: _t(op=2), 'output_padding'), (lambda: _t(s=1, op=1), 'output_padding'), (lambda: _t(groups=2), 'groups'),
             (lambda: _t(dil=2), 'dil'), (lambda: _t(s=3), 'stride'), (lambda: _t(Cin=6), 'Cin'), (lambda: _t(Cout=18), 'Cout'),
             (lambda: _t(p=-1), 'pad'), (lambda: _with(_t(), OH=15), 'OH'), (lambda: _with(_t(), OW=17), 'OW'),
             (lambda: _t(k=(3, 3), p=5, H=1, W=1, s=1), 'OH'), (lambda: _t(N=4096, H=512, W=512, Cin=16), 'N')]


@pytest.mark.parametrize('make,named', T_REFUSED)
def test_the_library_refuses_transposed_convolutions_it_does_not_build(make, named):
    d = make()
    L = lib.load()
    assert L.tt_conv_transpose2d_train_workspace_bytes(C.byref(d)) == 0
    null = C.c_void_p(0)
    for call in (lambda: L.tt_conv_transpose2d_train_forward(C.byref(d), null, null, null, null, null, C.c_size_t(0), null),
                 lambda: L.tt_conv_transpose2d_train_backward(C.byref(d), null, null, null, null, null, null, null, C.c_size_t(0), null)):
        assert call() == -3                                              # TT_ERR_UNSUPPORTED
        assert named in L.tt_last_error().decode()


def test_a_short_workspace_is_refused_before_anything_is_touched():
    d = _t()
    L = lib.load()
    n = L.tt_conv_transpose2d_train_workspace_bytes(C.byref(d))
    assert n > 0
    null = C.c_void_p(0)
    assert L.tt_conv_transpose2d_train_forward(C.byref(d), null, null, null, null, null, C.c_size_t(n - 1), null) == -3
    assert 'ws_bytes' in L.tt_last_error().decode()
    assert L.tt_conv_transpose2d_train_backward(C.byref(d), null, null, null, null, null, null, null, C.c_size_t(n - 1), null) == -3
    assert 'ws_bytes' in L.tt_last_error().decode()


def _i(**kw):
    d = lib.InterpBilinearTrainDesc()
    for k, v in {**dict(N=2, C=16, H=5, W=6, OH=10, OW=12, align_corners=1), **kw}.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize('make,named', [(lambda: _i(align_corners=0), 'align_corners'), (lambda: _i(C=6), 'C'), (lambda: _i(OH=0), 'OH'),
                                        (lambda: _i(H=0), 'H'), (lambda: _i(N=4096, C=512, OH=1024, OW=1024), 'N')])
def test_the_library_refuses_interpolations_it_does_not_build(make, named):
    d = make()
    L = lib.load()
    null = C.c_void_p(0)
    assert L.tt_interp_bilinear_train_forward(C.byref(d), null, null, null) == -3
    assert named in L.tt_last_error().decode()
    assert L.tt_interp_bilinear_train_backward(C.byref(d), null, null, null) == -3
    assert named in L.tt_last_error().decode()


@pytest.mark.parametrize('kw,named', [(dict(groups=2), 'groups'), (dict(stride=3), 'stride'), (dict(output_padding=2), 'output_padding'),
                                      (dict(dilation=2), 'dilation'), (dict(padding=(1, 0)), 'padding'), (dict(stride=(1, 2)), 'stride')])
def test_the_modules_refuse_at_construction_naming_the_parameter(kw, named):
    with pytest.raises(lib.TTError, match=named):
        ct.ConvTranspose2d(16, 32, 3, **{'stride': 2, **kw})
    with pytest.raises(lib.TTError, match='Cout'):
        ct.ConvTranspose2d(16, 18, 2, stride=2)
    with pytest.raises(lib.TTError, match='align_corners'):
        ip.Upsample(scale_factor=2, mode='bilinear', align_corners=False)
    with pytest.raises(lib.TTError, match='align_corners'):
        ip.Upsample(scale_factor=2, mode='bilinear')
    with pytest.raises(lib.TTError, match='mode'):
        ip.Upsample(scale_factor=2, mode='nearest')
    with pytest.raises(lib.TTError, match='align_corners'):
        ip.interpolate_bilinear(torch.randn(1, 4, 3, 3), scale_factor=2, align_corners=False)


def test_output_size_follows_torch_and_a_mismatch_is_refused():
    m = ct.ConvTranspose2d(8, 8, 3, stride=2, padding=1)
    x = torch.randn(1, 8, 5, 6)
    with pytest.raises(ValueError, match='output size'):                 # torch's own range check
        m(x, output_size=(12, 11))
    with pytest.raises(lib.TTError, match='output_size'):                # output padding (1, 0): not one value for both dimensions
        m(x, output_size=(10, 11))
    with pytest.raises(lib.TTError):                                     # valid, but a CPU tensor
        m(x, output_size=(10, 12))


def test_cpu_and_non_fp32_tensors_are_refused():
    m = ct.ConvTranspose2d(4, 8, 2, stride=2)
    with pytest.raises(lib.TTError):
        m(torch.randn(1, 4, 5, 5))
    with pytest.raises(lib.TTError):
        m(torch.randn(1, 4, 5, 5, requires_grad=True))
    with pytest.raises(lib.TTError):
        m.double()(torch.randn(1, 4, 5, 5, dtype=torch.float64))
    up = ip.Upsample(scale_factor=2, mode='bilinear', align_corners=True)
    with pytest.raises(lib.TTError):
        up(torch.randn(1, 4, 5, 5))
    with pytest.raises(lib.TTError):
        up(torch.randn(1, 4, 5, 5, requires_grad=True))


# ----------------------------------------------------------------------------------------- the float64 restatements, pinned
T_GEOMETRIES = [(2, 2, 0, 0), (2, 2, 0, 1), (3, 2, 1, 1), (3, 2, 1, 0), (3, 1, 1, 0), (1, 2, 0, 0), (1, 2, 0, 1), (4, 2, 1, 0), (5, 2, 3, 1),
                (1, 1, 0, 0)]


def _tcase(k, s, p, op, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 8, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(8, 12, k, k, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(12, generator=g, dtype=torch.float64, requires_grad=True)
    return x, w, b


@pytest.mark.parametrize('k,s,p,op', T_GEOMETRIES)
def test_the_transposed_restatement_equals_torch_autograd(k, s, p, op):
    for H, W in ((7, 9), (8, 6), (1, 1), (14, 28)):
        if RT.out_size(H, k, s, p, op) < 1 or RT.out_size(W, k, s, p, op) < 1:
            continue
        x, w, b = _tcase(k, s, p, op, H, W)
        y = F.conv_transpose2d(x, w, b, stride=s, padding=p, output_padding=op)
        gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
        y.backward(gy)
        assert torch.allclose(RT.forward(x.detach(), w.detach(), b.detach(), s, p, op), y.detach(), rtol=1e-12, atol=1e-12), (H, W)
        assert torch.allclose(RT.grad_input(gy, w.detach(), s, p), x.grad, rtol=1e-12, atol=1e-12), (H, W)
        assert torch.allclose(RT.grad_weight(x.detach(), gy, k, s, p), w.grad, rtol=1e-12, atol=1e-12), (H, W)
        assert torch.allclose(gy.sum((0, 2, 3)), b.grad, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('bug,k,s,p,op,H,W', [('swapped_phase', 2, 2, 0, 0, 7, 9), ('swapped_phase', 3, 2, 1, 1, 8, 6),
                                               ('flipped_tap', 3, 2, 1, 1, 7, 9), ('flipped_tap', 3, 1, 1, 0, 5, 4),
                                               ('flipped_tap', 4, 2, 1, 0, 6, 6)])
def test_each_seeded_transposed_bug_is_caught_by_the_torch_comparison(bug, k, s, p, op, H, W):
    x, w, b = _tcase(k, s, p, op, H, W, seed=3)
    want = F.conv_transpose2d(x, w, b, stride=s, padding=p, output_padding=op).detach()
    assert torch.allclose(RT.forward(x.detach(), w.detach(), b.detach(), s, p, op), want, rtol=1e-12, atol=1e-12)
    assert not torch.allclose(RT.forward(x.detach(), w.detach(), b.detach(), s, p, op, bug=bug), want, rtol=1e-6, atol=1e-6)


I_SHAPES = [(112, 224, 224, 448), (14, 28, 28, 56), (7, 9, 14, 18), (1, 1, 28, 56), (1, 3, 5, 7), (5, 6, 1, 1), (5, 6, 1, 12),
            (9, 8, 4, 3), (2, 2, 7, 7)]


@pytest.mark.parametrize('H,W,OH,OW', I_SHAPES)
def test_the_bilinear_restatement_equals_torch_autograd(H, W, OH, OW):
    g = torch.Generator().manual_seed(0)
    n = 1 if H * W > 1000 else 2
    x = torch.randn(n, 3, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    y = F.interpolate(x, size=(OH, OW), mode='bilinear', align_corners=True)
    gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(gy)
    assert torch.allclose(RI.forward(x.detach(), OH, OW), y.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(RI.backward(gy, H, W), x.grad, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('H,OH', [(112, 224), (14, 28), (7, 14), (5, 7), (9, 4), (1, 28), (28, 1)])
def test_the_gather_ranges_hold_every_output_that_reads_an_input_in_both_coordinate_types(H, OH):
    for coord in (np.float64, np.float32):
        A = RI.forward_matrix(H, OH, coord)
        assert torch.equal(RI.gather_matrix(H, OH, coord), A.t())
        reached = [set(RI.reach(i, H, OH, coord)) for i in range(H)]
        for o in range(OH):
            for i in range(H):
                if A[o, i] != 0:
                    assert o in reached[i], (coord, o, i)


@pytest.mark.parametrize('H,W,OH,OW', [(7, 9, 14, 18), (1, 1, 28, 56), (14, 28, 28, 56)])
def test_the_seeded_reach_bug_is_caught_by_the_torch_comparison(H, W, OH, OW):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 2, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    y = F.interpolate(x, size=(OH, OW), mode='bilinear', align_corners=True)
    gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(gy)
    assert torch.allclose(RI.backward(gy, H, W), x.grad, rtol=1e-12, atol=1e-12)
    assert not torch.allclose(RI.backward(gy, H, W, bug='reach'), x.grad, rtol=1e-6, atol=1e-6)


# ----------------------------------------------------------------------------------------- convert_upsampling on the oracle model
def _oracle():
    from oracle.model import EncoderDecoder as Oracle
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    cfg = Config.fromfile(DEFAULT_CONFIG)
    torch.manual_seed(0)
    return Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})


def test_convert_upsampling_on_the_oracle_model():
    model = _oracle()
    kinds = (nn.ConvTranspose2d, nn.Upsample)
    before = {n: m for n, m in model.named_modules() if isinstance(m, kinds)}
    params = {n: (m.weight, m.bias) for n, m in before.items() if isinstance(m, nn.ConvTranspose2d)}
    state = {k: v.clone() for k, v in model.state_dict().items()}
    other = {n: m for n, m in model.named_modules() if not isinstance(m, kinds)}
    out, skipped = ct.convert_upsampling(model)
    assert out is model and skipped == []
    after = dict(model.named_modules())
    assert sorted(before) == sorted(['img_encoder.seg_net.unet_layer4.up', 'img_encoder.seg_net.unet_layer3.up',
                                     'img_encoder.seg_net.unet_layer2.up', 'img_encoder.seg_net.unet_layer0.0',
                                     'lidar_encoder.pts_neck.deblocks.1.0'])
    for n in before:
        assert type(after[n]) is (ip.Upsample if n.endswith('unet_layer0.0') else ct.ConvTranspose2d), n
    for n, (w, b) in params.items():
        assert after[n].weight is w and after[n].bias is b, n                # the same Parameter objects
    assert all(after[n] is m for n, m in other.items() if n in after)         # other modules untouched
    assert list(model.state_dict()) == list(state)
    for k, v in model.state_dict().items():
        assert torch.equal(v, state[k]), k


def test_convert_upsampling_swaps_a_bare_layer_keeps_its_training_flag_and_names_what_it_skips():
    m = nn.ConvTranspose2d(8, 16, 2, stride=2).eval()
    new, skipped = ct.convert_upsampling(m)
    assert type(new) is ct.ConvTranspose2d and new.weight is m.weight and new.bias is m.bias and not new.training and skipped == []
    seq = nn.Sequential(nn.Upsample(scale_factor=2, mode='nearest'), nn.ConvTranspose2d(8, 18, 2, stride=2),
                        nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True))
    same, skipped = ct.convert_upsampling(seq)
    assert same is seq and type(seq[2]) is ip.Upsample and seq[2].scale_factor == 2.0
    assert [(n, why.split(':')[0]) for n, _, why in skipped] == [('0', 'mode'), ('1', 'Cout')]
