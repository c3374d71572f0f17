"""Training-side deformable convolution on the GPU (include/tt_b200.h §12) against the float64 reference of
tests/deform_conv_reference.py (torchvision's deform_conv2d on the CPU, mmcv's border rule for the offset gradient).

Error bound: |got - ref| / S <= 1e-5 per element, S = the float64 sum of |contribution| of that element.  Every product is formed in
3xTF32 (operands split x = hi + lo, hi*hi + hi*lo + lo*hi: ~2^-21 relative per product), accumulated in fp32 over K (the tensor core
truncates within a 64-deep chunk, chunks are added with round-to-nearest) and, for grad_weight, partial sums over pixel ranges are
folded in a fixed order: each step errs by a few 2^-24 of the running |sum| <= S, and the 50 176-deep reductions random-walk far below
1e-5 S.  The offsets are multiples of 2^-12, so every float32 sampling coordinate (ho - 1 + i) + dy is exact and the comparison
measures the arithmetic, not a rounding of the input coordinate."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from deform_conv_reference import abs_bounds, reference, sample_coords, worst

pytestmark = pytest.mark.gpu
BOUND = 1e-5


def _quant(t):
    return torch.round(t * 4096) / 4096


def _inputs(N, Cin, Cout, H, W, groups, seed, crafted=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin // groups, 3, 3, generator=g) * (2.0 / (9 * Cin / groups)) ** 0.5
    off = torch.randn(N, 18, H, W, generator=g) * 2.0
    if crafted:                                        # image 0, small blocks: under 1 % of all samples sit on an integer
        ti = (torch.arange(9) // 3).view(9, 1, 1).float()
        off[0, :, 0:2, 0:8] = torch.randint(-3, 4, (18, 2, 8), generator=g).float()               # integer offsets
        off[0, :, 2:4, 0:8] = torch.randint(-3, 4, (18, 2, 8), generator=g).float() + 0.5         # half-integer offsets
        ho = torch.arange(4, 6).view(1, 2, 1).float()
        off[0, 0::2, 4:6, 8:16] = -(ho - 1 + ti) - torch.rand(9, 2, 8, generator=g) * 0.98 - 0.01  # h in (-1, 0)
        ho = torch.arange(H - 2, H).view(1, 2, 1).float()
        off[0, 0::2, H - 2:H, 8:16] = (H - 1) - (ho - 1 + ti) + torch.rand(9, 2, 8, generator=g) * 0.98 + 0.01   # h in (H - 1, H)
        off[0, :, 6:8, 0:16] = torch.where(torch.rand(18, 2, 16, generator=g) < 0.5, -30.0, 30.0)                # far outside
    gout = torch.randn(N, Cout, H, W, generator=g)
    return x, _quant(off), w, gout


def _ours(x, off, w, gout, groups, step):
    from thinktwice_b200.ops.deform_conv import deform_conv2d
    t = [v.cuda().requires_grad_(True) for v in (x, off, w)]
    y = deform_conv2d(t[0], t[1], t[2], 1, 1, 1, groups, 1, False, step)
    y.backward(gout.cuda())
    torch.cuda.synchronize()
    return y.detach().cpu(), t[0].grad.cpu(), t[1].grad.cpu(), t[2].grad.cpu()


def _check_all(x, off, w, gout, groups, got, near_ok=True):
    ref = reference(x, off, w, gout)
    bnd = abs_bounds(x, off, w, gout, groups)
    names = ('output', 'grad_input', 'grad_offset', 'grad_weight')
    # grad_offset: the sampled value is piecewise bilinear in the coordinate, its derivative jumps where a coordinate is an integer.
    # Samples within 1e-4 of one are compared with float32 autograd (same float32 coordinate, same side of the jump), the rest
    # against float64.
    hs, ws = sample_coords(off)
    near = (((hs - hs.round()).abs() < 1e-4) | ((ws - ws.round()).abs() < 1e-4)).repeat_interleave(2, dim=1)
    assert int(near[:, 0::2].sum()) < near[:, 0::2].numel() // 100
    for k, name in enumerate(names):
        if k == 2:
            r32 = reference(x, off, w, gout, dtype=torch.float32)[2].double()
            e = worst(got[2][~near], ref[2][~near], bnd[2][~near])
            assert e <= BOUND, (name, e)
            if bool(near.any()):
                e32 = worst(got[2][near], r32[near], bnd[2][near])
                assert e32 <= 1e-3, (name + ' at integer coordinates', e32)
        else:
            e = worst(got[k], ref[k], bnd[k])
            assert e <= BOUND, (name, e)
    return ref, bnd


def test_training_shape_of_the_reference():
    """the key sweep at B = 2: 8 images x 512 x 28 x 56, groups 4, im2col_step 128 (lss.py:189-197), crafted offsets included."""
    x, off, w, gout = _inputs(8, 512, 512, 28, 56, 4, seed=1, crafted=True)
    got = _ours(x, off, w, gout, 4, 128)
    _check_all(x, off, w, gout, 4, got)


@pytest.mark.parametrize('N,Cin,Cout,H,W,groups,step', [(2, 64, 64, 13, 17, 1, 2), (1, 64, 32, 9, 11, 4, 128), (3, 16, 48, 7, 5, 4, 1)])
def test_small_shapes(N, Cin, Cout, H, W, groups, step):
    x, off, w, gout = _inputs(N, Cin, Cout, H, W, groups, seed=N * 100 + Cin)
    _check_all(x, off, w, gout, groups, _ours(x, off, w, gout, groups, step))


def test_zero_offsets_are_a_grouped_convolution():
    x, _, w, gout = _inputs(2, 128, 128, 14, 28, 4, seed=9)
    off = torch.zeros(2, 18, 14, 28)
    y, gx, _, _ = _ours(x, off, w, gout, 4, 128)
    xd, wd, gd = x.double(), w.double(), gout.double()
    _, gxa, _, _ = abs_bounds(x, off, w, gout, 4)
    ya = F.conv2d(xd.abs(), wd.abs(), padding=1, groups=4)
    assert worst(y, F.conv2d(xd, wd, padding=1, groups=4), ya) <= BOUND
    assert worst(gx, F.conv_transpose2d(gd, wd, padding=1, groups=4), gxa) <= BOUND


def test_reproducibility_and_chunking():
    """grad_weight / grad_offset: fixed-order reductions, bitwise equal from call to call; output / grad_offset: independent of
    im2col_step (every pixel's sum has one order); grad_input (fp32 atomics) stays within the bound."""
    x, off, w, gout = _inputs(4, 128, 128, 28, 56, 4, seed=4)
    a = _ours(x, off, w, gout, 4, 128)
    b = _ours(x, off, w, gout, 4, 128)
    assert torch.equal(a[3], b[3]) and torch.equal(a[2], b[2]) and torch.equal(a[0], b[0])
    c = _ours(x, off, w, gout, 4, 1)
    assert torch.equal(a[0], c[0]) and torch.equal(a[2], c[2])
    ref = reference(x, off, w, gout)
    bnd = abs_bounds(x, off, w, gout, 4)
    for got in (a, c):
        assert worst(got[1], ref[1], bnd[1]) <= BOUND
        assert worst(got[3], ref[3], bnd[3]) <= BOUND


def test_null_gradients_are_skipped_and_the_others_unchanged():
    from thinktwice_b200 import lib
    from thinktwice_b200.lib import _p
    x, off, w, gout = (t.cuda() for t in _inputs(2, 64, 64, 12, 20, 4, seed=6))
    d = lib.DeformConvDesc()
    for k, v in dict(N=2, C=64, H=12, W=20, Cout=64, groups=4, im2col_step=2, kernel_h=3, kernel_w=3, stride=1, padding=1, dilation=1,
                     deform_groups=1).items():
        setattr(d, k, v)
    n = int(lib.load().tt_deform_conv_workspace_bytes(C.byref(d)))
    ws = torch.empty(n, dtype=torch.uint8, device='cuda')

    def run(mask):
        outs = [torch.full_like(t, float('nan')) if m else None for t, m in zip((x, off, w), mask)]
        lib.call('tt_deform_conv_backward', C.byref(d), _p(x), _p(off), _p(w), _p(gout), *[_p(o) for o in outs], _p(ws), C.c_size_t(n))
        torch.cuda.synchronize()
        return outs
    full = run((True, True, True))
    assert all(bool(torch.isfinite(t).all()) for t in full)
    for mask in [(False, True, True), (True, False, True), (True, True, False), (True, False, False), (False, False, True),
                 (False, False, False)]:
        outs = run(mask)
        for k, o in enumerate(outs):
            if o is None:
                continue
            if k == 0:                                                 # fp32 atomics: same values up to the summation order
                assert torch.allclose(o, full[0], rtol=1e-5, atol=1e-6)
            else:
                assert torch.equal(o, full[k]), (mask, k)


class _TorchvisionMmcvBorder(torch.autograd.Function):
    """torchvision's CUDA deform_conv2d with mmcv's offset-gradient border rule (tests/deform_conv_reference.py)."""
    @staticmethod
    def forward(ctx, x, off, w):
        ctx.save_for_backward(x, off, w)
        from torchvision.ops import deform_conv2d
        return deform_conv2d(x, off, w, padding=1)

    @staticmethod
    def backward(ctx, g):
        from deform_conv_reference import outside
        from torchvision.ops import deform_conv2d
        x, off, w = ctx.saved_tensors
        with torch.enable_grad():
            t = [v.detach().requires_grad_(True) for v in (x, off, w)]
            gx, goff, gw = torch.autograd.grad(deform_conv2d(t[0], t[1], t[2], padding=1), t, g)
        return gx, goff.masked_fill(outside(off.cpu()).repeat_interleave(2, dim=1).to(goff.device), 0.0), gw


def test_end_to_end_pack_in_a_torch_graph():
    """a DeformConv2dPack between torch layers; loss.backward(): the gradients of weight, conv_offset.* and the input against the same
    graph on torchvision's CUDA deform_conv2d (fp32) and a float64 CPU run of it: ours must err no more than twice torchvision's."""
    from thinktwice_b200.ops.deform_conv import DeformConv2dPack
    torch.manual_seed(0)
    pack = DeformConv2dPack(64, 64, 3, padding=1, groups=4, im2col_step=128)
    with torch.no_grad():
        pack.conv_offset.weight.normal_(0, 0.05)
        pack.conv_offset.bias.normal_(0, 0.5)
    pre = torch.nn.Conv2d(32, 64, 3, padding=1)
    x0 = torch.randn(2, 32, 20, 36)
    target = torch.randn(2, 64, 20, 36)

    def graph(dcn, dev, dtype):
        p = {k: v.detach().to(dev, dtype).requires_grad_(True) for k, v in pack.state_dict().items()}
        q = {k: v.detach().to(dev, dtype) for k, v in pre.state_dict().items()}
        xi = x0.to(dev, dtype).requires_grad_(True)
        h = F.relu(F.conv2d(xi, q['weight'], q['bias'], padding=1))
        off = F.conv2d(h, p['conv_offset.weight'], p['conv_offset.bias'], padding=1)
        y = dcn(h, off, p['weight'])
        loss = ((F.relu(y) - target.to(dev, dtype)) ** 2).mean()
        loss.backward()
        return [xi.grad, p['weight'].grad, p['conv_offset.weight'].grad, p['conv_offset.bias'].grad]

    from thinktwice_b200.ops.deform_conv import deform_conv2d
    ours = graph(lambda h, o, w: deform_conv2d(h, o, w, 1, 1, 1, 4, 1, False, 128), 'cuda', torch.float32)
    tvc = graph(lambda h, o, w: _TorchvisionMmcvBorder.apply(h, o, w), 'cuda', torch.float32)
    ref = graph(lambda h, o, w: _TorchvisionMmcvBorder.apply(h, o, w), 'cpu', torch.float64)
    for a, b, r, name in zip(ours, tvc, ref, ('input', 'weight', 'conv_offset.weight', 'conv_offset.bias')):
        scale = float(r.abs().max())
        e_ours = float((a.cpu().double() - r).abs().max()) / scale
        e_tv = float((b.cpu().double() - r).abs().max()) / scale
        assert e_ours <= max(2 * e_tv, 1e-5), (name, e_ours, e_tv)
