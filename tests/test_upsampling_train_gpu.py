"""Training-side upsampling on the GPU (include/tt_b200.h §17, thinktwice_b200/ops/conv_transpose2d.py and interpolate.py) against
float64.

Every output element is held to |got - ref| <= 1e-5 * S, S the float64 sum of |terms| of that element (the §16 convention): y, grad_x,
grad_weight and grad_bias of every distinct nn.ConvTranspose2d, and y and grad_x of every bilinear interpolation (nn.Upsample and the
ASPP's F.interpolate), of one thinktwice.py forward of the oracle (collected with hooks; the UNet head at 32 images), corner cases,
bitwise repeatability, skipped NULL gradients, empty batches, and the oracle's UNet under autograd after convert_conv2d +
convert_upsampling.  The bilinear reference weighs in float64 the fp32 source coordinates the op defines (ATen's fp32 arithmetic)."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import interpolate_train_reference as RI
from thinktwice_b200 import lib
from thinktwice_b200.ops import conv2d as cv
from thinktwice_b200.ops import conv_transpose2d as ct
from thinktwice_b200.ops import interpolate as ip

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope='module', autouse=True)
def report():
    yield
    if WORST:
        print('\n[upsampling_train] worst |err| / (1e-5 S): ' + ', '.join(f'{k} {v:.3g}' for k, v in sorted(WORST.items())))


def _ratio(name, got, ref, S):
    err = (got.double() - ref).abs()
    bound = 1e-5 * S
    r = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), r)
    assert r <= 1.0, (name, r)
    assert bool((err[S == 0] == 0).all()), name                            # nothing reaches: exactly zero


def _layer_shapes():
    """('t', Cin, Cout, k, s, p, op, bias, H, W) of every nn.ConvTranspose2d and ('i', C, H, W, OH, OW) of every bilinear interpolation
    in one thinktwice.py forward of the oracle, with the camera branch's flag."""
    import oracle.camera as cam
    from oracle.model import EncoderDecoder as Oracle, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, 0)
    o.eval()
    seen = set()

    def hook(m, inp):
        if type(m) is nn.ConvTranspose2d:
            seen.add(('t', m.in_channels, m.out_channels, m.kernel_size[0], m.stride[0], m.padding[0], m.output_padding[0],
                      m.bias is not None, *inp[0].shape[2:]))
    for m in o.modules():
        if type(m) is nn.ConvTranspose2d:
            m.register_forward_pre_hook(hook)
    interp = F.interpolate

    def record(x, size=None, scale_factor=None, mode='nearest', align_corners=None, *args, **kw):
        y = interp(x, size, scale_factor, mode, align_corners, *args, **kw)
        if mode == 'bilinear':
            assert align_corners is True
            seen.add(('i', x.shape[1], *x.shape[2:], *y.shape[2:]))
        return y
    cam.F.interpolate = record                                           # nn.Upsample and the ASPP's call both go through it
    try:
        with torch.no_grad():
            o.forward_inference(make_batch(cfg, 1, seed=0, num_points=40000))
    finally:
        cam.F.interpolate = interp
    return sorted(seen)


def check_t(Cin, Cout, k, s, p, op, bias, H, W, N, seed=0, tag='layer'):
    g = torch.Generator(device='cuda').manual_seed(seed)
    dev = 'cuda'
    m = ct.ConvTranspose2d(Cin, Cout, k, stride=s, padding=p, output_padding=op, bias=bias).to(dev)
    with torch.no_grad():
        m.weight.copy_(torch.randn(m.weight.shape, generator=g, device=dev) / (Cin * k * k / (s * s)) ** 0.5)
        if bias:
            m.bias.copy_(torch.randn(Cout, generator=g, device=dev))
    x = torch.randn(N, Cin, H, W, generator=g, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = m(x)
    assert y.is_contiguous(memory_format=torch.channels_last)
    gy = torch.randn(y.shape, generator=g, device=dev).contiguous(memory_format=torch.channels_last)
    y.backward(gy)
    xd, wd, gyd = x.detach().double(), m.weight.detach().double(), gy.double()
    bd = m.bias.detach().double() if bias else None
    conv = dict(stride=s, padding=p)
    _ratio(f'{tag} y', y.detach(), F.conv_transpose2d(xd, wd, bd, output_padding=op, **conv),
           F.conv_transpose2d(xd.abs(), wd.abs(), bd.abs() if bias else None, output_padding=op, **conv))
    _ratio(f'{tag} grad_x', x.grad, F.conv2d(gyd, wd, **conv), F.conv2d(gyd.abs(), wd.abs(), **conv))
    _ratio(f'{tag} grad_weight', m.weight.grad, torch.nn.grad.conv2d_weight(gyd, wd.shape, xd, **conv),
           torch.nn.grad.conv2d_weight(gyd.abs(), wd.shape, xd.abs(), **conv))
    if bias:
        _ratio(f'{tag} grad_bias', m.bias.grad, gyd.sum((0, 2, 3)), gyd.abs().sum((0, 2, 3)))


def check_i(Cc, H, W, OH, OW, N, seed=0, tag='layer'):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(N, Cc, H, W, generator=g, device='cuda').contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = ip.interpolate_bilinear(x, size=(OH, OW))
    assert y.shape == (N, Cc, OH, OW) and y.is_contiguous(memory_format=torch.channels_last)
    gy = torch.randn(y.shape, generator=g, device='cuda').contiguous(memory_format=torch.channels_last)
    y.backward(gy)
    xd = x.detach().double()
    _ratio(f'{tag} y', y.detach(), RI.forward(xd, OH, OW, np.float32), RI.forward(xd.abs(), OH, OW, np.float32))
    _ratio(f'{tag} grad_x', x.grad, RI.backward(gy, H, W, np.float32), RI.backward_abs(gy, H, W, np.float32))


def test_every_upsampling_layer_of_the_model_against_float64():
    shapes = _layer_shapes()
    ts = [s[1:] for s in shapes if s[0] == 't']
    its = [s[1:] for s in shapes if s[0] == 'i']
    assert (256, 128, 2, 2, 0, 0, True, 56, 112) in ts and any(not t[6] for t in ts)   # UNet up, the SECONDFPN deblock
    assert (128, 112, 224, 224, 448) in its and (512, 1, 1, 28, 56) in its             # unet_layer0, the ASPP broadcast
    for t in ts:
        check_t(*t, N=32 if t[6] else 4, tag='deconv')
        torch.cuda.empty_cache()
    for i in its:
        check_i(*i, N=32, tag='broadcast' if i[1:3] == (1, 1) else 'bilinear')
        torch.cuda.empty_cache()


@pytest.mark.parametrize('Cin,Cout,k,s,p,op,bias,H,W,N', [
    (4, 4, 2, 2, 0, 0, True, 5, 7, 2),            # k2s2 at odd sizes, the smallest channel counts
    (36, 68, 2, 2, 0, 0, False, 11, 13, 3),       # tails in K, N and M
    (8, 12, 3, 2, 1, 1, True, 7, 9, 2),           # output_padding
    (8, 12, 3, 2, 1, 0, True, 6, 5, 1),
    (8, 12, 3, 1, 1, 0, True, 6, 5, 2),           # stride 1
    (8, 12, 1, 2, 0, 1, True, 5, 6, 2),           # k1s2: three phases no tap reaches, written with the bias
    (8, 12, 1, 2, 0, 0, False, 5, 6, 2),
    (8, 12, 4, 2, 1, 0, True, 6, 6, 2),
    (8, 12, 5, 2, 3, 1, True, 4, 7, 2),           # padding past the kernel's reach
    (8, 12, 1, 1, 0, 0, True, 129, 3, 1),         # 1x1: the plain weight-gradient contraction
])
def test_transposed_corner_cases_against_float64(Cin, Cout, k, s, p, op, bias, H, W, N):
    check_t(Cin, Cout, k, s, p, op, bias, H, W, N, tag='deconv corner')


@pytest.mark.parametrize('Cc,H,W,OH,OW,N', [
    (16, 7, 9, 14, 18, 2), (4, 5, 6, 1, 1, 2), (8, 5, 6, 1, 12, 2), (8, 5, 6, 12, 1, 2),   # OH = 1 / OW = 1
    (512, 1, 1, 28, 56, 4), (20, 1, 1, 9, 7, 3),                                         # the broadcast (split lanes, C4 < 32)
    (8, 1, 3, 5, 7, 2), (12, 9, 8, 4, 3, 2), (20, 3, 2, 64, 40, 2), (132, 14, 28, 28, 56, 2)])
def test_bilinear_corner_cases_against_float64(Cc, H, W, OH, OW, N):
    check_i(Cc, H, W, OH, OW, N, tag='bilinear corner')


def test_empty_batches_launch_nothing():
    m = ct.ConvTranspose2d(8, 16, 2, stride=2).cuda()
    x = torch.randn(0, 8, 5, 5, device='cuda', requires_grad=True)
    n0 = lib.launch_count()
    y = m(x)
    y.backward(torch.randn_like(y))
    z = ip.interpolate_bilinear(torch.randn(0, 8, 5, 5, device='cuda', requires_grad=True), scale_factor=2)
    z.backward(torch.randn_like(z))
    torch.cuda.synchronize()
    assert y.shape == (0, 16, 10, 10) and z.shape == (0, 8, 10, 10) and lib.launch_count() == n0
    assert torch.equal(m.weight.grad, torch.zeros_like(m.weight)) and torch.equal(m.bias.grad, torch.zeros_like(m.bias))


def _raw(d, x, w, b, gy, want):
    """one tt_conv_transpose2d_train_backward with the gradients in `want`; returns (grads, launches)."""
    gx = torch.empty_like(x) if 'x' in want else None
    gw = torch.empty_like(w) if 'w' in want else None
    gb = torch.empty_like(b) if 'b' in want else None
    ws, n = ct._workspace(d, x.device)
    n0 = lib.launch_count()
    lib.call('tt_conv_transpose2d_train_backward', C.byref(d), lib._p(x), lib._p(w), lib._p(gy), lib._p(gx), lib._p(gw), lib._p(gb),
             lib._p(ws), C.c_size_t(n))
    torch.cuda.synchronize()
    return (gx, gw, gb), lib.launch_count() - n0


@pytest.mark.parametrize('k,s,p,op', [(2, 2, 0, 0), (3, 2, 1, 1), (3, 1, 1, 0), (1, 2, 0, 1)])
def test_transposed_repeatable_bitwise_and_null_gradients_skipped(k, s, p, op):
    torch.manual_seed(1)
    N, Cin, Cout, H, W = 3, 48, 40, 23, 17
    x = torch.randn(N, Cin, H, W, device='cuda').contiguous(memory_format=torch.channels_last)
    w = torch.randn(Cin, Cout, k, k, device='cuda')
    b = torch.randn(Cout, device='cuda')
    d = ct._desc(N, H, W, Cin, Cout, (k, k), s, p, op, 1, 1, True)
    y1, y2 = ct._forward(x, w, b, s, p, op), ct._forward(x, w, b, s, p, op)
    assert torch.equal(y1, y2)
    gy = torch.randn(y1.shape, device='cuda').contiguous(memory_format=torch.channels_last)
    full1, n_all = _raw(d, x, w, b, gy, 'xwb')
    full2, _ = _raw(d, x, w, b, gy, 'xwb')
    for a, c in zip(full1, full2):
        assert torch.equal(a, c)
    counts = {}
    for want in ('', 'x', 'w', 'b'):
        got, counts[want] = _raw(d, x, w, b, gy, want)
        for name, g, f in zip('xwb', got, full1):
            assert (g is None) == (name not in want)
            if g is not None:
                assert torch.equal(g, f)
    assert counts[''] == 0 and counts['b'] == 2
    assert counts['x'] + counts['w'] + counts['b'] == n_all and counts['x'] > 0 and counts['w'] > 0


@pytest.mark.parametrize('Cc,H,W,OH,OW', [(128, 56, 112, 112, 224), (512, 1, 1, 28, 56)])
def test_bilinear_repeatable_bitwise(Cc, H, W, OH, OW):
    torch.manual_seed(2)
    x = torch.randn(4, Cc, H, W, device='cuda').contiguous(memory_format=torch.channels_last)
    gy = torch.randn(4, Cc, OH, OW, device='cuda').contiguous(memory_format=torch.channels_last)
    outs = []
    for _ in range(2):
        xr = x.clone().requires_grad_(True)
        y = ip.interpolate_bilinear(xr, size=(OH, OW))
        y.backward(gy)
        outs.append((y.detach(), xr.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_no_grad_saves_nothing_and_matches_the_autograd_path():
    m = ct.ConvTranspose2d(16, 32, 2, stride=2).cuda()
    up = ip.Upsample(scale_factor=2, mode='bilinear', align_corners=True)
    x = torch.randn(2, 16, 9, 11, device='cuda')
    with torch.no_grad():
        y0, z0 = m(x), up(x)
    assert y0.grad_fn is None and z0.grad_fn is None and y0.is_contiguous(memory_format=torch.channels_last)
    y1, z1 = m(x), up(x.requires_grad_(True))
    assert y1.grad_fn is not None and z1.grad_fn is not None and torch.equal(y0, y1) and torch.equal(z0, z1)


def test_unet_under_autograd_after_convert_conv2d_and_convert_upsampling():
    """The oracle's UNet seg head (three k2s2 deconvs, the bilinear x2, the convolutions between) at 4 images of the thinktwice.py
    feature maps, every parameter and input gradient against the float64 module.  Each is held to max(1e-4 max|ref|, 2 x torch fp32's
    error) (TF32 off): as close as fp32.  The worst ratios are printed, with torch's default single-pass TF32 error beside them."""
    from oracle.camera import UNet
    torch.manual_seed(0)
    ref = UNet(12, (256, 256, 256, 256)).cuda().train()
    f32, t32 = copy.deepcopy(ref), copy.deepcopy(ref)
    ours, _ = cv.convert_conv2d(copy.deepcopy(ref))
    ours, skipped = ct.convert_upsampling(ours)
    assert skipped == []
    assert not any(type(m) in (nn.ConvTranspose2d, nn.Upsample) for m in ours.modules())
    ref = ref.double()
    feats = [torch.randn(4, 256, h, w, device='cuda') for h, w in ((112, 224), (56, 112), (28, 56), (14, 28))]
    out = ref([f.double() for f in feats])
    wt = torch.randn(out.shape, device='cuda', dtype=torch.float64)

    def run(model, dtype):
        xs = [f.to(dtype, copy=True).requires_grad_(True) for f in feats]      # a fresh leaf per run: no gradient accumulates
        (model(xs) * wt.to(dtype)).sum().backward()
        g = {n: p.grad.double() for n, p in model.named_parameters()}
        g.update({f'input{i}': x.grad.double() for i, x in enumerate(xs)})
        return g
    want = run(ref, torch.float64)
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
        g_t32 = run(t32, torch.float32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        g_f32, got = run(f32, torch.float32), run(ours, torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    rel = {}
    for n in want:
        scale = float(want[n].abs().max())
        rel[n] = [float((h[n] - want[n]).abs().max()) / scale for h in (got, g_f32, g_t32)]
    ratio = {n: r[0] / max(1e-4, 2 * r[1]) for n, r in rel.items()}
    n = max(ratio, key=ratio.get)
    print(f'\n[upsampling_train] UNet, worst error / max|ref| (ours, torch fp32, torch tf32): {n} {tuple(f"{v:.2e}" for v in rel[n])}')
    WORST['unet autograd err / bound'] = ratio[n]
    assert ratio[n] <= 1.0, (n, rel[n])
