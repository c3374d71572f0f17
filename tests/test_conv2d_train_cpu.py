"""CPU side of the training-side dense convolution (include/tt_b200.h §16, thinktwice_b200/ops/conv2d.py): the ctypes descriptor, the
library's refusals (each named, before any pointer or device is touched), the float64 restatement of the phase-decomposed grad_x and
the implicit-convolution grad_weight against torch.nn.grad for every geometry the reference builds, seeded bugs each caught, and
convert_conv2d on the oracle model."""
import ctypes as C
import os
import subprocess

import pytest
import torch
import torch.nn as nn

import conv2d_train_reference as R
from thinktwice_b200 import lib
from thinktwice_b200.ops import conv2d as cv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ctypes_descriptor_matches_the_c_header(tmp_path):
    fields = [n for n, _ in lib.Conv2dTrainDesc._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "tt_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof(tt_conv2d_train_desc, {n}));\n' for n in fields) +
                   '  printf("%zu\\n", sizeof(tt_conv2d_train_desc));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(lib.Conv2dTrainDesc, n).offset for n in fields] + [C.sizeof(lib.Conv2dTrainDesc)]


def test_new_entries_are_exported():
    assert {'tt_conv2d_train_workspace_bytes', 'tt_conv2d_train_forward', 'tt_conv2d_train_backward'} <= set(lib.EXPORTS)


def _d(**kw):
    g = dict(N=2, H=9, W=8, Cin=16, Cout=32, kernel_size=(3, 3), stride=2, pad=1, dil=1, groups=1, bias=True)
    g.update(kw)
    return cv._desc(g['N'], g['H'], g['W'], g['Cin'], g['Cout'], g['kernel_size'], g['stride'], g['pad'], g['dil'], g['groups'], g['bias'])


def _with(d, **kw):
    for k, v in kw.items():
        setattr(d, k, v)
    return d


REFUSED = [(lambda: _d(groups=2), 'groups'), (lambda: _d(stride=3), 'stride'), (lambda: _d(Cin=6), 'Cin'), (lambda: _d(Cout=18), 'Cout'),
           (lambda: _with(_d(), OH=4), 'OH'), (lambda: _with(_d(), OW=5), 'OW'),
           (lambda: _d(N=4096, H=1024, W=1024, Cin=16), 'N'), (lambda: _d(kernel_size=(0, 3)), 'KH')]


@pytest.mark.parametrize('make,named', REFUSED)
def test_the_library_refuses_what_the_reference_does_not_build(make, named):
    """checked before any pointer or device is touched: the refusal works without a GPU."""
    d = make()
    L = lib.load()
    assert L.tt_conv2d_train_workspace_bytes(C.byref(d)) == 0
    null = C.c_void_p(0)
    for call in (lambda: L.tt_conv2d_train_forward(C.byref(d), null, null, null, null, null, C.c_size_t(0), null),
                 lambda: L.tt_conv2d_train_backward(C.byref(d), null, null, null, null, null, null, null, C.c_size_t(0), null)):
        assert call() == -3                                              # TT_ERR_UNSUPPORTED
        assert named in L.tt_last_error().decode()


def test_a_short_workspace_is_refused_before_anything_is_touched():
    d = _d()
    L = lib.load()
    n = L.tt_conv2d_train_workspace_bytes(C.byref(d))
    assert n > 0
    null = C.c_void_p(0)
    assert L.tt_conv2d_train_forward(C.byref(d), null, null, null, null, null, C.c_size_t(n - 1), null) == -3
    assert 'ws_bytes' in L.tt_last_error().decode()
    assert L.tt_conv2d_train_backward(C.byref(d), null, null, null, null, null, null, null, C.c_size_t(n - 1), null) == -3
    assert 'ws_bytes' in L.tt_last_error().decode()


@pytest.mark.parametrize('kw,named', [(dict(groups=2), 'groups'), (dict(stride=3), 'stride'), (dict(padding=(1, 0)), 'padding'),
                                      (dict(stride=(1, 2)), 'stride'), (dict(dilation=(1, 2)), 'dilation'),
                                      (dict(padding_mode='reflect'), 'padding_mode'), (dict(padding='same'), 'padding')])
def test_the_module_refuses_at_construction_naming_the_parameter(kw, named):
    with pytest.raises(lib.TTError, match=named):
        cv.Conv2d(16, 32, 3, **kw)
    with pytest.raises(lib.TTError, match='Cin'):
        cv.Conv2d(3, 64, 7, stride=2, padding=3)
    with pytest.raises(lib.TTError, match='Cout'):
        cv.Conv2d(512, 18, 3, padding=1)


def test_cpu_and_non_fp32_tensors_are_refused():
    m = cv.Conv2d(4, 8, 3, padding=1)
    with pytest.raises(lib.TTError):
        m(torch.randn(1, 4, 5, 5))
    with pytest.raises(lib.TTError):
        m(torch.randn(1, 4, 5, 5, requires_grad=True))
    with pytest.raises(lib.TTError):
        m.double()(torch.randn(1, 4, 5, 5, dtype=torch.float64))


# ----------------------------------------------------------------------------------------- the float64 restatement, pinned
def _oracle():
    from oracle.model import EncoderDecoder as Oracle
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    cfg = Config.fromfile(DEFAULT_CONFIG)
    torch.manual_seed(0)
    return Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})


def _geometries():
    """every (kernel, stride, padding, dilation) of an eligible nn.Conv2d the reference builds (thinktwice.py)."""
    got = set()
    for m in _oracle().modules():
        if type(m) is nn.Conv2d and m.in_channels % 4 == 0 and m.out_channels % 4 == 0:
            got.add((m.kernel_size[0], m.stride[0], m.padding[0], m.dilation[0]))
    return sorted(got)


GEOMETRIES = [(1, 1, 0, 1), (1, 2, 0, 1), (3, 1, 0, 1), (3, 1, 1, 1), (3, 1, 6, 6), (3, 1, 12, 12), (3, 1, 18, 18), (3, 2, 0, 1), (3, 2, 1, 1)]


def test_the_geometry_list_is_what_the_reference_builds():
    assert _geometries() == GEOMETRIES


def _maps(k, s, p, d):
    maps = [(7, 9), (8, 6), (1, 1) if d * (k - 1) <= 2 * p else (d * (k - 1) + 1 - 2 * p, 3)]
    if s == 2 and p == 0:
        maps += [(21, 21), (10, 10)]
    return maps


def _case(k, s, p, d, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 8, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(12, 8, k, k, generator=g, dtype=torch.float64)
    OH, OW = (H + 2 * p - d * (k - 1) - 1) // s + 1, (W + 2 * p - d * (k - 1) - 1) // s + 1
    gy = torch.randn(2, 12, OH, OW, generator=g, dtype=torch.float64)
    return x, w, gy


@pytest.mark.parametrize('k,s,p,d', GEOMETRIES)
def test_the_phase_decomposition_and_the_implicit_weight_gradient_equal_torch(k, s, p, d):
    for H, W in _maps(k, s, p, d):
        x, w, gy = _case(k, s, p, d, H, W)
        want_x = torch.nn.grad.conv2d_input(x.shape, w, gy, stride=s, padding=p, dilation=d)
        want_w = torch.nn.grad.conv2d_weight(x, w.shape, gy, stride=s, padding=p, dilation=d)
        assert torch.allclose(R.grad_input(gy, w, H, W, s, p, d), want_x, rtol=1e-12, atol=1e-12), (H, W)
        assert torch.allclose(R.grad_weight(x, gy, k, k, s, p, d), want_w, rtol=1e-12, atol=1e-12), (H, W)


def test_empty_phases_and_unreached_rows_occur_where_expected():
    """the 1x1 stride-2 downsample reaches only phase (0, 0); conv10_4 (3x3, stride 2, no padding) on 10 x 10 reaches no tap in the last
    row and column: (10 + 0 - 2 - 1) mod 2 = 1 > pad = 0."""
    assert [R.phase_dim(q, 1, 2, 0, 1, 28)[1] for q in (0, 1)] == [1, 0]
    x, w, gy = _case(3, 2, 0, 1, 10, 10)
    gx = R.grad_input(gy, w, 10, 10, 2, 0, 1)
    assert torch.equal(gx[:, :, 9], torch.zeros_like(gx[:, :, 9])) and torch.equal(gx[:, :, :, 9], torch.zeros_like(gx[:, :, :, 9]))
    assert bool((gx[:, :, :9, :9] != 0).any())


@pytest.mark.parametrize('bug,k,s,p,d,H,W', [('origin', 3, 2, 1, 1, 8, 6), ('origin', 3, 1, 6, 6, 7, 9), ('zero_phase', 1, 2, 0, 1, 7, 9),
                                             ('zero_phase', 1, 2, 0, 1, 8, 6), ('unflipped', 3, 1, 1, 1, 7, 9), ('unflipped', 3, 2, 1, 1, 8, 6),
                                             ('tap_order', 3, 1, 1, 1, 7, 9), ('tap_order', 3, 2, 0, 1, 21, 21)])
def test_each_seeded_bug_is_caught_by_the_torch_comparison(bug, k, s, p, d, H, W):
    x, w, gy = _case(k, s, p, d, H, W, seed=3)
    if bug == 'tap_order':
        want = torch.nn.grad.conv2d_weight(x, w.shape, gy, stride=s, padding=p, dilation=d)
        assert torch.allclose(R.grad_weight(x, gy, k, k, s, p, d), want, rtol=1e-12, atol=1e-12)
        assert not torch.allclose(R.grad_weight(x, gy, k, k, s, p, d, bug=bug), want, rtol=1e-6, atol=1e-6)
    else:
        want = torch.nn.grad.conv2d_input(x.shape, w, gy, stride=s, padding=p, dilation=d)
        assert torch.allclose(R.grad_input(gy, w, H, W, s, p, d), want, rtol=1e-12, atol=1e-12)
        assert not torch.allclose(R.grad_input(gy, w, H, W, s, p, d, bug=bug), want, rtol=1e-6, atol=1e-6)


# ----------------------------------------------------------------------------------------- convert_conv2d on the oracle model
def test_convert_conv2d_on_the_oracle_model():
    model = _oracle()
    before = {n: (type(m), m.weight, m.bias) for n, m in model.named_modules() if isinstance(m, nn.Conv2d)}
    state = {k: v.clone() for k, v in model.state_dict().items()}
    other = {n: m for n, m in model.named_modules() if not isinstance(m, nn.Conv2d)}
    out, skipped = cv.convert_conv2d(model)
    assert out is model
    after = dict(model.named_modules())
    skipped_names = {n for n, _, _ in skipped}
    for n, (t, w, b) in before.items():
        m = after[n]
        eligible = m.in_channels % 4 == 0 and m.out_channels % 4 == 0
        if t is nn.Conv2d and eligible:
            assert type(m) is cv.Conv2d, n
            assert m.weight is w and m.bias is b, n                          # the same Parameter objects
        else:
            assert type(m) is t, n
    for n, m, why in skipped:
        assert type(m) is nn.Conv2d and after[n] is m
        assert ('Cin' in why) == (m.in_channels % 4 != 0) and ('Cout' in why) == (m.in_channels % 4 == 0), (n, why)
    assert 'img_encoder.img_backbone.conv1' in skipped_names                  # the stem: Cin = 3
    assert 'img_encoder.depth_net.depth_conv.4.conv_offset' in skipped_names   # the DCN's offsets: Cout = 18
    assert all(after[n] is m for n, m in other.items() if n in after)         # other modules (DCN, deconvs, BN) untouched
    assert list(model.state_dict()) == list(state)
    for k, v in model.state_dict().items():
        assert torch.equal(v, state[k]), k
    with pytest.raises(lib.TTError):                                           # CPU tensors: no fallback
        model.img_encoder.img_backbone.layer1[0].conv2(torch.randn(1, 64, 8, 8))


def test_convert_conv2d_swaps_a_bare_layer_and_keeps_its_training_flag():
    m = nn.Conv2d(8, 16, 3, padding=1).eval()
    new, skipped = cv.convert_conv2d(m)
    assert type(new) is cv.Conv2d and new.weight is m.weight and new.bias is m.bias and not new.training and skipped == []
    stem = nn.Conv2d(3, 64, 7, stride=2, padding=3)
    same, skipped = cv.convert_conv2d(stem)
    assert same is stem and skipped[0][0] == '' and 'Cin' in skipped[0][2]
