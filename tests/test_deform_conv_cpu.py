"""CPU side of the training-side deformable convolution (include/tt_b200.h §12, thinktwice_b200/ops/deform_conv.py): mmcv's refusals,
the library's refusals of what the reference does not build, the module's parameter names, the ctypes descriptor, and the float64
reference the GPU tests compare against (torchvision's deform_conv2d) pinned to a literal loop."""
import ctypes as C
import math
import os
import subprocess

import pytest
import torch
from torchvision.ops import deform_conv2d as tv_deform_conv2d

from deform_conv_reference import outside, reference
from thinktwice_b200 import lib
from thinktwice_b200.ops.deform_conv import DeformConv2d, DeformConv2dFunction, DeformConv2dPack, deform_conv2d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_only():
    if torch.cuda.is_available():
        pytest.skip('CUDA present')


def test_function_and_modules_refuse_cpu_tensors():
    _cpu_only()
    x, off, w = torch.randn(2, 8, 5, 6), torch.randn(2, 18, 5, 6), torch.randn(8, 2, 3, 3)
    with pytest.raises(lib.TTError):
        DeformConv2dFunction.apply(x, off, w, 1, 1, 1, 4, 1, False, 2)
    with pytest.raises(lib.TTError):
        deform_conv2d(x, off, w, 1, 1, 1, 4)
    with pytest.raises(lib.TTError):
        DeformConv2dPack(8, 8, 3, padding=1, groups=4)(x)
    with pytest.raises(lib.TTError):
        DeformConv2d(8, 8, 3, padding=1, groups=4)(x, off)


def test_mmcv_assertions_are_reproduced():
    """mmcv 1.7 DeformConv2dFunction.forward: 4-D input (ValueError), bias False, batch divisible by min(im2col_step, N)."""
    w = torch.randn(8, 2, 3, 3)
    with pytest.raises(ValueError, match='4D'):
        deform_conv2d(torch.randn(8, 5, 6), torch.randn(1, 18, 5, 6), w, 1, 1, 1, 4)
    with pytest.raises(AssertionError, match='bias'):
        deform_conv2d(torch.randn(2, 8, 5, 6), torch.randn(2, 18, 5, 6), w, 1, 1, 1, 4, 1, True)
    with pytest.raises(AssertionError, match='divisible by im2col_step'):
        deform_conv2d(torch.randn(3, 8, 5, 6), torch.randn(3, 18, 5, 6), w, 1, 1, 1, 4, 1, False, 2)
    with pytest.raises(AssertionError):
        DeformConv2d(8, 8, 3, bias=True)
    with pytest.raises(AssertionError):
        DeformConv2d(6, 8, 3, groups=4)


def _desc(**kw):
    d = lib.DeformConvDesc()
    base = dict(N=2, C=512, H=28, W=56, Cout=512, groups=4, im2col_step=128, kernel_h=3, kernel_w=3, stride=1, padding=1, dilation=1,
                deform_groups=1)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize('field,value,named', [
    ('kernel_h', 5, 'kernel_size'), ('kernel_w', 1, 'kernel_size'), ('stride', 2, 'stride'), ('padding', 0, 'padding'),
    ('dilation', 2, 'dilation'), ('deform_groups', 2, 'deform_groups'), ('groups', 3, 'groups'), ('C', 40, 'groups'),
    ('Cout', 520, 'groups'), ('im2col_step', 0, 'im2col_step')])
def test_the_library_refuses_what_the_reference_does_not_build(field, value, named):
    """checked before any pointer or device is touched: the refusal works without a GPU."""
    L = lib.load()
    d = _desc(**{field: value})
    assert L.tt_deform_conv_workspace_bytes(C.byref(d)) == 0
    null = C.c_void_p(0)
    for call in (lambda: L.tt_deform_conv_forward(C.byref(d), null, null, null, null, null, C.c_size_t(0), null),
                 lambda: L.tt_deform_conv_backward(C.byref(d), null, null, null, null, null, null, null, null, C.c_size_t(0), null)):
        assert call() == -3                                          # TT_ERR_UNSUPPORTED
        assert named in L.tt_last_error().decode()


def test_workspace_is_bounded_by_the_chunk():
    """the columns of one chunk of im2col_step images, not of the batch: 32 images at step 8 need a quarter of step 32's columns."""
    L = lib.load()
    big = L.tt_deform_conv_workspace_bytes(C.byref(_desc(N=32, im2col_step=32)))
    small = L.tt_deform_conv_workspace_bytes(C.byref(_desc(N=32, im2col_step=8)))
    col = 32 * 28 * 56 * 9 * 512 * 4
    assert col < big < 1.5 * col and small < big / 3                   # + channels-last input, output and grad_input copies


def test_ctypes_descriptor_matches_the_c_header(tmp_path):
    fields = [n for n, _ in lib.DeformConvDesc._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "tt_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof(tt_deform_conv_desc, {n}));\n' for n in fields) +
                   '  printf("%zu\\n", sizeof(tt_deform_conv_desc));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(lib.DeformConvDesc, n).offset for n in fields] + [C.sizeof(lib.DeformConvDesc)]


def test_state_dict_matches_the_oracle_pack_and_a_checkpoint_loads():
    from mmcv_loader import load_checkpoint
    from oracle.camera import DeformConv2dPack as OraclePack
    ours = DeformConv2dPack(512, 512, 3, padding=1, groups=4, im2col_step=128)
    ref = OraclePack(512, 512, groups=4)
    assert [(k, tuple(v.shape)) for k, v in ours.state_dict().items()] == [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    assert float(ours.conv_offset.weight.abs().sum()) == 0 and float(ours.conv_offset.bias.abs().sum()) == 0


def test_depth_conv_dcn_tensors_of_a_checkpoint_load_through_mmcvs_loader(tmp_path):
    """the `depth_conv.4.*` tensors of a model checkpoint (lss.py:189: the DCN is the fifth module of depth_conv)."""
    from mmcv_loader import load_checkpoint
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.registry import build_model
    m = build_model(dict(Config.fromfile(PLUMBING_CONFIG).model, seed=3))
    pre = 'img_encoder.depth_net.depth_conv.4.'
    sd = {k[len(pre):]: v.clone() for k, v in m.state_dict().items() if k.startswith(pre)}
    assert sorted(sd) == ['conv_offset.bias', 'conv_offset.weight', 'weight']
    cout, cg = sd['weight'].shape[:2]
    pack = DeformConv2dPack(cg * 4, cout, 3, padding=1, groups=4, im2col_step=128)
    f = tmp_path / 'dcn.pth'
    torch.save({'state_dict': sd}, f)
    rep = load_checkpoint(pack, str(f), map_location='cpu')['_load_report']
    assert rep['missing'] == [] and rep['unexpected'] == [] and rep['err'] == []
    for k, v in pack.state_dict().items():
        assert torch.equal(v, sd[k]), k


# ----------------------------------------------------------------------------------------- the float64 reference, pinned
def _bilinear(img, h, w):
    """mmcv's deformable_im2col_bilinear on one channel: zero outside (-1, H) x (-1, W), out-of-image corners zero."""
    H, W = img.shape
    if not (-1 < h < H and -1 < w < W):
        return 0.0
    hl, wl = math.floor(h), math.floor(w)
    lh, lw = h - hl, w - wl
    v = 0.0
    for hh, wh, wt in ((hl, wl, (1 - lh) * (1 - lw)), (hl, wl + 1, (1 - lh) * lw), (hl + 1, wl, lh * (1 - lw)), (hl + 1, wl + 1, lh * lw)):
        if 0 <= hh < H and 0 <= wh < W:
            v += wt * float(img[hh, wh])
    return v


def _coord_weight(img, h, w, axis):
    """mmcv's get_coordinate_weight: d(bilinear sample) / dh (axis 0) or / dw (axis 1), 0 outside (-1, H) x (-1, W)."""
    H, W = img.shape
    if not (-1 < h < H and -1 < w < W):
        return 0.0
    hl, wl = math.floor(h), math.floor(w)

    def at(a, b):
        return float(img[a, b]) if 0 <= a < H and 0 <= b < W else 0.0
    if axis == 0:
        return (wl + 1 - w) * (at(hl + 1, wl) - at(hl, wl)) + (w - wl) * (at(hl + 1, wl + 1) - at(hl, wl + 1))
    return (hl + 1 - h) * (at(hl, wl + 1) - at(hl, wl)) + (h - hl) * (at(hl + 1, wl + 1) - at(hl + 1, wl))


def _literal(x, off, wt, gout, groups):
    """forward and the three gradients of mmcv's DCNv1 (3x3, stride 1, padding 1) as literal loops over every contribution."""
    N, Cin, H, W = x.shape
    Cout, Cg = wt.shape[:2]
    Cog = Cout // groups
    out, gx, goff, gw = torch.zeros(N, Cout, H, W, dtype=torch.float64), torch.zeros_like(x), torch.zeros_like(off), torch.zeros_like(wt)
    for n in range(N):
        for ho in range(H):
            for wo in range(W):
                for tap in range(9):
                    i, j = divmod(tap, 3)
                    h = ho - 1 + i + float(off[n, 2 * tap, ho, wo])
                    w = wo - 1 + j + float(off[n, 2 * tap + 1, ho, wo])
                    inside = -1 < h < H and -1 < w < W
                    for c in range(Cin):
                        g, cg = divmod(c, Cg)
                        img = x[n, c]
                        col = _bilinear(img, h, w)
                        dcol_dh, dcol_dw = _coord_weight(img, h, w, 0), _coord_weight(img, h, w, 1)
                        for o in range(g * Cog, (g + 1) * Cog):
                            k = float(wt[o, cg, i, j])
                            go = float(gout[n, o, ho, wo])
                            out[n, o, ho, wo] += k * col
                            gw[o, cg, i, j] += go * col
                            goff[n, 2 * tap, ho, wo] += go * k * dcol_dh
                            goff[n, 2 * tap + 1, ho, wo] += go * k * dcol_dw
                            if inside:                               # the column gradient scattered to the four corners
                                hl, wl = math.floor(h), math.floor(w)
                                lh, lw = h - hl, w - wl
                                for hh, wh, cw in ((hl, wl, (1 - lh) * (1 - lw)), (hl, wl + 1, (1 - lh) * lw), (hl + 1, wl, lh * (1 - lw)),
                                                   (hl + 1, wl + 1, lh * lw)):
                                    if 0 <= hh < H and 0 <= wh < W:
                                        gx[n, c, hh, wh] += go * k * cw
    return out, gx, goff, gw


def test_the_float64_reference_equals_a_literal_loop():
    """torchvision's deform_conv2d (float64 autograd on the CPU) is what the GPU tests compare against; here it is pinned to mmcv's
    semantics spelled out as loops, with samples in (-1, 0), past H - 1, outside, and exactly on integers."""
    g = torch.Generator().manual_seed(7)
    N, Cin, Cout, H, W, groups = 2, 4, 4, 4, 5, 2
    x = torch.randn(N, Cin, H, W, generator=g, dtype=torch.float64)
    wt = torch.randn(Cout, Cin // groups, 3, 3, generator=g, dtype=torch.float64)
    off = torch.randn(N, 18, H, W, generator=g, dtype=torch.float64) * 1.5
    off[0, :, 0, :] = torch.randint(-2, 3, (18, W), generator=g).double()       # exactly on integers
    off[0, 0::2, 1, :] = -torch.arange(3).repeat_interleave(3)[:, None].double() - 0.4          # row 1, tap row i: h = i + dy = -0.4
    off[1, 0::2, 3, :] = 0.6                                                    # rows 3 + (i - 1) + 0.6: past H - 1
    off[1, 1::2, 2, :] = 9.0                                                    # outside
    gout = torch.randn(N, Cout, H, W, generator=g, dtype=torch.float64)
    lit = _literal(x, off, wt, gout, groups)
    for a, b in zip(reference(x, off, wt, gout), lit):
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-10)
    # the one correction the reference makes: torchvision's own offset gradient is nonzero at some samples mmcv reads as zero
    t = off.clone().requires_grad_(True)
    tv_deform_conv2d(x, t, wt, padding=1).backward(gout)
    out = outside(off).repeat_interleave(2, dim=1)
    assert torch.allclose(t.grad[~out], lit[2][~out], rtol=1e-10, atol=1e-10)
    assert float(t.grad[out].abs().max()) > 0 and float(lit[2][out].abs().max()) == 0
    hs = torch.stack([off[:, 2 * t] + torch.arange(H).view(1, H, 1) - 1 + t // 3 for t in range(9)])
    assert bool(((hs > -1) & (hs < 0)).any()) and bool(((hs > H - 1) & (hs < H)).any()) and bool((hs == hs.round()).any())


def test_the_float64_reference_passes_gradcheck():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 4, 4, 5, generator=g, dtype=torch.float64, requires_grad=True)
    off = (torch.randn(1, 18, 4, 5, generator=g, dtype=torch.float64) * 1.3).requires_grad_(True)
    wt = torch.randn(4, 2, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, b, c: tv_deform_conv2d(a, b, c, padding=1), (x, off, wt))
