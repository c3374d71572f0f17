"""Training-side dense convolution on the GPU (include/tt_b200.h §16, thinktwice_b200/ops/conv2d.py) against float64.

Every output element is held to |got - ref| <= 1e-5 * S, S the float64 sum of |terms| of that element (the convention of the
deformable- and sparse-convolution tests): y, grad_x, grad_weight and grad_bias of every distinct eligible nn.Conv2d of the oracle
model at thinktwice.py shapes (collected with forward hooks), corner cases, bitwise repeatability, skipped NULL gradients, and the
camera trunk under autograd after convert_conv2d.  About 40 s on an H100, most of it the oracle's CPU forward for the shapes."""
import ctypes as C

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from thinktwice_b200 import lib
from thinktwice_b200.ops import conv2d as cv

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope='module', autouse=True)
def report():
    yield
    if WORST:
        print('\n[conv2d_train] worst |err| / (1e-5 S): ' + ', '.join(f'{k} {v:.3g}' for k, v in sorted(WORST.items())))


def _ratio(name, got, ref, S):
    err = (got.double() - ref).abs()
    bound = 1e-5 * S
    r = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), r)
    assert r <= 1.0, (name, r)
    assert bool((err[S == 0] == 0).all()), name                            # nothing reaches: exactly zero


def _layer_shapes():
    """distinct (Cin, Cout, k, stride, pad, dil, bias, H, W) of every eligible nn.Conv2d in one thinktwice.py forward of the oracle."""
    from oracle.model import EncoderDecoder as Oracle, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, 0)
    o.eval()
    seen = set()

    def hook(m, inp):
        if m.in_channels % 4 == 0 and m.out_channels % 4 == 0:
            seen.add((m.in_channels, m.out_channels, m.kernel_size[0], m.stride[0], m.padding[0], m.dilation[0], m.bias is not None,
                      *inp[0].shape[2:]))
    for m in o.modules():
        if type(m) is nn.Conv2d:
            m.register_forward_pre_hook(hook)
    with torch.no_grad():
        o.forward_inference(make_batch(cfg, 1, seed=0, num_points=40000))
    return sorted(seen)


LAYERS = None


def layers():
    global LAYERS
    if LAYERS is None:
        shapes = _layer_shapes()
        flops = sorted(shapes, key=lambda s: -(s[0] * s[1] * s[2] ** 2 * ((s[7] + 2 * s[4] - s[5] * (s[2] - 1) - 1) // s[3] + 1) *
                                               ((s[8] + 2 * s[4] - s[5] * (s[2] - 1) - 1) // s[3] + 1)))
        big = set(flops[:3])
        LAYERS = [(s, 32 if s in big else 4) for s in shapes]
    return LAYERS


def check(Cin, Cout, k, s, p, d, bias, H, W, N, seed=0, nchw_grad=False, tag='layer'):
    g = torch.Generator(device='cuda').manual_seed(seed)
    dev = 'cuda'
    m = cv.Conv2d(Cin, Cout, k, stride=s, padding=p, dilation=d, bias=bias).to(dev)
    with torch.no_grad():
        m.weight.copy_(torch.randn(m.weight.shape, generator=g, device=dev) / (Cin * k * k) ** 0.5)
        if bias:
            m.bias.copy_(torch.randn(Cout, generator=g, device=dev))
    x = torch.randn(N, Cin, H, W, generator=g, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = m(x)
    assert y.is_contiguous(memory_format=torch.channels_last)
    gy = torch.randn(y.shape, generator=g, device=dev)
    if not nchw_grad:
        gy = gy.contiguous(memory_format=torch.channels_last)
    y.backward(gy)
    xd, wd, gyd = x.detach().double(), m.weight.detach().double(), gy.double()
    conv = dict(stride=s, padding=p, dilation=d)
    ref_y = F.conv2d(xd, wd, m.bias.detach().double() if bias else None, **conv)
    S_y = F.conv2d(xd.abs(), wd.abs(), m.bias.detach().double().abs() if bias else None, **conv)
    _ratio(f'{tag} y', y.detach(), ref_y, S_y)
    del ref_y, S_y
    _ratio(f'{tag} grad_x', x.grad, torch.nn.grad.conv2d_input(xd.shape, wd, gyd, **conv),
           torch.nn.grad.conv2d_input(xd.shape, wd.abs(), gyd.abs(), **conv))
    _ratio(f'{tag} grad_weight', m.weight.grad, torch.nn.grad.conv2d_weight(xd, wd.shape, gyd, **conv),
           torch.nn.grad.conv2d_weight(xd.abs(), wd.shape, gyd.abs(), **conv))
    if bias:
        _ratio(f'{tag} grad_bias', m.bias.grad, gyd.sum((0, 2, 3)), gyd.abs().sum((0, 2, 3)))


def test_every_distinct_layer_of_the_model_against_float64():
    ls = layers()
    assert len(ls) > 60
    assert any(sh[2] == 3 and sh[5] in (6, 12, 18) and sh[7:] == (28, 56) for sh, _ in ls)        # ASPP
    assert any(sh[3] == 2 and sh[4] == 0 and sh[7:] == (10, 10) for sh, _ in ls)                  # conv10_4
    for sh, n in ls:
        check(*sh, N=n, tag=f'{sh[2]}x{sh[2]}/s{sh[3]}' + ('/d' if sh[5] > 1 else ''))
        torch.cuda.empty_cache()


@pytest.mark.parametrize('Cin,Cout,k,s,p,d,bias,H,W,N', [
    (4, 4, 3, 1, 1, 1, True, 6, 7, 2),            # the smallest channel counts
    (4, 4, 1, 2, 0, 1, False, 9, 8, 1),           # N = 1, empty phases
    (36, 68, 3, 2, 1, 1, True, 11, 13, 3),        # tails in K (36 = 32 + 4), N (68 = 64 + 4) and M (odd maps)
    (132, 20, 3, 2, 0, 1, False, 21, 21, 2),      # stride 2, no padding, unreached last row / column
    (64, 128, 3, 2, 0, 1, True, 10, 10, 2),
    (16, 8, 3, 1, 6, 6, True, 4, 5, 2),           # a dilation halo larger than the map
    (16, 8, 3, 1, 18, 18, False, 5, 3, 1),
    (8, 12, 1, 1, 0, 1, True, 129, 3, 1),         # 1x1: the plain weight-gradient contraction, M tail
    (8, 12, 5, 2, 2, 1, True, 9, 10, 2),          # 5x5: 3x3 / 3x2 / 2x3 / 2x2 phases
    (8, 12, 3, 2, 1, 2, False, 12, 9, 2),         # stride 2 with an even dilation: two empty phases
])
def test_corner_cases_against_float64(Cin, Cout, k, s, p, d, bias, H, W, N):
    check(Cin, Cout, k, s, p, d, bias, H, W, N, tag='corner')


def test_grad_y_arriving_nchw_contiguous():
    check(32, 64, 3, 2, 1, 1, True, 14, 15, 2, nchw_grad=True, tag='nchw grad_y')


def test_an_empty_batch_launches_nothing_and_zeroes_the_parameter_gradients():
    m = cv.Conv2d(8, 16, 3, padding=1).cuda()
    x = torch.randn(0, 8, 5, 5, device='cuda', requires_grad=True)
    n0 = lib.launch_count()
    y = m(x)
    y.backward(torch.randn_like(y))
    torch.cuda.synchronize()
    assert y.shape == (0, 16, 5, 5) and lib.launch_count() == n0
    assert torch.equal(m.weight.grad, torch.zeros_like(m.weight)) and torch.equal(m.bias.grad, torch.zeros_like(m.bias))


def _raw(d, x, w, b, gy, want):
    """one tt_conv2d_train_backward with the gradients in `want`; returns (grads, launches)."""
    gx = torch.empty_like(x) if 'x' in want else None
    gw = torch.empty_like(w) if 'w' in want else None
    gb = torch.empty_like(b) if 'b' in want else None
    ws, n = cv._workspace(d, x.device)
    n0 = lib.launch_count()
    lib.call('tt_conv2d_train_backward', C.byref(d), lib._p(x), lib._p(w), lib._p(gy), lib._p(gx), lib._p(gw), lib._p(gb), lib._p(ws),
             C.c_size_t(n))
    torch.cuda.synchronize()
    return (gx, gw, gb), lib.launch_count() - n0


@pytest.mark.parametrize('k,s', [(3, 1), (3, 2), (1, 2)])
def test_repeatable_bitwise_and_null_gradients_skipped(k, s):
    torch.manual_seed(1)
    N, Cin, Cout, H, W, p = 3, 48, 40, 23, 17, k // 2
    x = torch.randn(N, Cin, H, W, device='cuda').contiguous(memory_format=torch.channels_last)
    w = torch.randn(Cout, Cin, k, k, device='cuda')
    b = torch.randn(Cout, device='cuda')
    d = cv._desc(N, H, W, Cin, Cout, (k, k), s, p, 1, 1, True)
    y1, _ = cv._forward(x, w, b, s, p, 1)
    y2, _ = cv._forward(x, w, b, s, p, 1)
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


def test_no_grad_saves_nothing_and_matches_the_autograd_path():
    m = cv.Conv2d(16, 32, 3, stride=2, padding=1).cuda()
    x = torch.randn(2, 16, 9, 11, device='cuda')
    with torch.no_grad():
        y0 = m(x)
    assert y0.grad_fn is None and y0.is_contiguous(memory_format=torch.channels_last)
    y1 = m(x)
    assert y1.grad_fn is not None and torch.equal(y0, y1)


def test_camera_trunk_under_autograd_after_convert_conv2d():
    """ResNet-50 + PAFPN + neck_conv of oracle.camera in train mode (BatchNorm batch statistics) at 4 images of 224 x 448, every parameter
    gradient against float64.  This trunk at random initialisation amplifies rounding strongly (torch fp32 with TF32 off misses float64 by
    ~2 % of a tensor's max), so each gradient is held to max(1e-3 max|ref|, 2 x torch fp32's error, torch TF32's error / 4): as close as
    fp32 or clearly closer than single-pass TF32 cuDNN.  The per-element fp32-class check is the per-layer test above; the worst ratios
    against each yardstick are printed."""
    import copy
    from oracle.camera import PAFPN, ResNet50
    torch.manual_seed(0)

    class Trunk(nn.Module):
        def __init__(self):
            super().__init__()
            self.img_backbone, self.img_neck, self.neck_conv = ResNet50(), PAFPN(), nn.Conv2d(256, 512, 1)

        def forward(self, x):
            f = self.img_neck(self.img_backbone(x))
            return list(f) + [self.neck_conv(f[2])]
    ref = Trunk().cuda().train()
    f32, t32 = copy.deepcopy(ref), copy.deepcopy(ref)
    ours, skipped = cv.convert_conv2d(copy.deepcopy(ref))
    assert [n for n, _, _ in skipped] == ['img_backbone.conv1']
    ref = ref.double()
    x = torch.randn(4, 3, 224, 448, device='cuda')             # layer4's BatchNorm sees 4 x 7 x 14 values per channel
    outs = ref(x.double())
    wts = [torch.randn(o.shape, device='cuda', dtype=torch.float64) for o in outs]

    def run(model):
        sum((o.float() * w.float()).sum() for o, w in zip(model(x), wts)).backward()
        return {n: p.grad.double() for n, p in model.named_parameters()}
    sum((o * w).sum() for o, w in zip(outs, wts)).backward()
    want = {n: p.grad for n, p in ref.named_parameters()}
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
        g_t32 = run(t32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False      # the stem stays on torch: fp32 for both
        g_f32, got = run(f32), run(ours)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    rel = {}
    for n, g in got.items():
        scale = float(want[n].abs().max())
        rel[n] = [float((h[n] - want[n]).abs().max()) / scale for h in (got, g_f32, g_t32)]
    worst = {k: max(rel, key=lambda n: rel[n][0] / v(rel[n])) for k, v in
             (('1e-3', lambda r: 1e-3), ('fp32', lambda r: r[1]), ('tf32', lambda r: r[2]))}
    print('\n[conv2d_train] trunk, error / max|ref| (ours, torch fp32, torch tf32): ' +
          ', '.join(f'worst vs {k}: {n} {tuple(round(v, 5) for v in rel[n])}' for k, n in worst.items()))
    ratio = {n: r[0] / max(1e-3, 2 * r[1], r[2] / 4) for n, r in rel.items()}
    n = max(ratio, key=ratio.get)
    WORST['trunk autograd err / bound'] = ratio[n]
    assert ratio[n] <= 1.0, (n, rel[n])
