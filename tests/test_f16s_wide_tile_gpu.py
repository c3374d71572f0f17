"""128-column tiles of the scaled-split fp16 convolution (csrc/gemm_conv_f16s.cu, BN = 128) against an fp64 torch reference.
tt_conv2d_f16s takes 128-column tiles when Cout > 64 and the 128-column tiles alone cover every SM of an H100 (132), so every
case here but the split-K one is sized to clear that bar; the numbers in the comments are those tiles.  Each case is run
again with debug bit 0x400000, which forces 64-column tiles: both tiles walk K in the same order with the same fold schedule per
output element, so the two results must agree to 1e-6 (they are expected to be bit-identical outside split-K)."""
import pytest
import torch
import torch.nn.functional as F

from test_f16s_gpu import IMPL, TOL, engine, saturations, split_value, to_fmap_s
from test_tc_gpu import relerr, to_fmap

pytestmark = pytest.mark.gpu
FORCE_BN64 = 0x400000


def set_knobs(flags):
    from thinktwice_b200 import lib
    lib.check(lib.load().tt_debug_set(flags), 'tt_debug_set')


def both_tiles(run):
    """run() -> dict of output tensors; returns (default tiles, forced 64-column tiles), each cloned before the next run."""
    outs = []
    try:
        for flags in (0, FORCE_BN64):
            set_knobs(flags)
            got = run()
            torch.cuda.synchronize()
            outs.append({k: v.detach().double().cpu().clone() for k, v in got.items()})
    finally:
        set_knobs(0)
    return outs


def check_same(wide, narrow):
    for k in wide:
        assert relerr(wide[k], narrow[k]) <= 1e-6, k


def pack(w, b=None):
    from thinktwice_b200.weights import Packer
    sd = {'c.weight': w}
    if b is not None:
        sd['c.bias'] = b
    return Packer(sd, torch.device('cuda:0'), tc_mode=IMPL).conv('c')


@pytest.mark.parametrize('case', [
    # N, H, W, Cin, Cout, k, pad, stride, bias, act
    (2, 96, 96, 64, 96, 1, 0, 1, True, 1),        # 1x1 flat, partial N tile (96 of 128): 144 tiles
    (2, 48, 96, 96, 192, 3, 1, 1, False, 1),      # 3x3, one full and one partial N tile: 144 tiles
    (8, 96, 96, 64, 128, 3, 1, 2, True, 0),       # 3x3 stride 2 (TMA element strides): 144 tiles
    (4, 112, 112, 256, 512, 1, 0, 2, False, 1),   # 1x1 stride 2 (ResNet downsample): 448 tiles
    (1, 28, 56, 512, 2048, 1, 0, 1, True, 0),     # 1x1 flat, 16 N tiles: 208 tiles
])
def test_f16s_wide_tile_matches_fp64(case):
    N, H, W, Cin, Cout, k, p, stride, bias, act = case
    gen = torch.Generator().manual_seed(sum(case))
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen) * (Cin * k * k) ** -0.5
    b = torch.randn(Cout, generator=gen) if bias else None
    eng = engine()
    pw = pack(w, b)
    xf = to_fmap_s(eng, 'wt.x', x.cuda(), ld=-(-Cin // 8) * 8)
    saturations()

    def run():
        y = eng.conv(xf, pw, name='wt.y', stride=stride, pad=p, act=act)
        return {'y': y.nchw(), 'planes': split_value(y)}

    wide, narrow = both_tiles(run)
    ref = F.conv2d(x.double(), w.double(), b.double() if bias else None, stride=stride, padding=p)
    ref = F.relu(ref) if act else ref
    err = relerr(wide['y'], ref)
    print(case, err, 'bit-identical' if torch.equal(wide['y'], narrow['y']) else 'differs')
    assert err < TOL
    assert relerr(wide['planes'], wide['y']) < 6e-7
    check_same(wide, narrow)
    assert saturations() == 0


def test_f16s_underfilled_layer_keeps_narrow_split_k():
    """an under-filled layer (B = 1 layer4 3x3, 512 -> 512 at 14 x 28) would have 4 x 4 tiles of 128 columns: too few for the SMs,
    so it keeps 64-column tiles and splits K (4 x 8 tiles, 5 splits) with or without the knob — and gives the same result."""
    from thinktwice_b200 import lib
    gen = torch.Generator().manual_seed(31)
    N, H, W, Cin, Cout = 1, 14, 28, 512, 512
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, 3, 3, generator=gen) * (Cin * 9) ** -0.5
    b = torch.randn(Cout, generator=gen)
    r = torch.randn(N, Cout, H, W, generator=gen)
    eng = engine()
    pw = pack(w, b)
    xf = to_fmap_s(eng, 'wk.x', x.cuda())
    rf = to_fmap(r.cuda())

    def run():
        n0 = lib.launch_count()
        y = eng.conv(xf, pw, name='wk.y', pad=1, act=1, res=rf)
        assert lib.launch_count() - n0 == 3                          # init + split-K kernel + finish
        return {'y': y.nchw(), 'planes': split_value(y)}

    wide, narrow = both_tiles(run)
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1) + r.double())
    assert relerr(wide['y'], ref) < TOL
    assert relerr(wide['planes'], wide['y']) < 6e-7
    check_same(wide, narrow)                                         # red.add order of the splits: equal to rounding, not bitwise


def test_f16s_wide_tile_epilogue_residuals_concat_upsample_and_scatter():
    from thinktwice_b200 import lib
    from thinktwice_b200.engine import FMap
    gen = torch.Generator().manual_seed(37)
    eng = engine()
    N, H, W, Cin = 2, 96, 96, 64
    x = torch.randn(N, Cin, H, W, generator=gen)
    xs = to_fmap_s(eng, 'we.x', x.cuda())

    # 3x3, Cout 192 into a concat slice at channel offset 32 of a 256-channel buffer; fp32 residual + split-plane residual
    # (a residual stored as planes only): 144 x 2 tiles
    w = torch.randn(192, Cin, 3, 3, generator=gen) * (Cin * 9) ** -0.5
    r1, r2 = torch.randn(N, 192, H, W, generator=gen), torch.randn(N, 192, H, W, generator=gen)
    pw = pack(w)
    r1f = to_fmap(r1.cuda(), ld=200, coff=8)
    r2s = to_fmap_s(eng, 'we.r2', r2.cuda())
    r2f = FMap(None, r2s.N, r2s.H, r2s.W, r2s.C, r2s.ld, r2s.coff, r2s.s)
    out = eng.fmap('we.cat', N, H, W, 256, split=True)

    def run_cat():
        eng.fill(out.t, 5.0)
        eng.sync_split(out)
        y = eng.conv(xs, pw, out=out.slice(32, 192), pad=1, act=1, res=r1f, res2=r2f)
        return {'y': y.nchw(), 'buf': out.nchw(), 'planes': split_value(out)}

    wide, narrow = both_tiles(run_cat)
    ref = F.relu(F.conv2d(x.double(), w.double(), padding=1) + r1.double() + r2.double())
    assert relerr(wide['y'], ref) < TOL
    assert float((wide['buf'][:, :32] - 5).abs().max()) == 0 and float((wide['buf'][:, 224:] - 5).abs().max()) == 0
    assert relerr(wide['planes'], wide['buf']) < 6e-7
    check_same(wide, narrow)

    # 1x1 lateral with a nearest-upsampled top map (RES_UP2): Cout 256, 144 x 2 tiles
    w1 = torch.randn(256, Cin, 1, 1, generator=gen) * Cin ** -0.5
    top = torch.randn(N, 256, H // 2, W // 2, generator=gen)
    pw1 = pack(w1)
    topf = to_fmap(top.cuda())

    def run_up():
        y = eng.conv(xs, pw1, name='we.lat', res=topf, res_mode=lib.RES_UP2)
        return {'y': y.nchw()}

    wide, narrow = both_tiles(run_up)
    ref = F.conv2d(x.double(), w1.double()) + F.interpolate(top.double(), size=(H, W), mode='nearest')
    assert relerr(wide['y'], ref) < TOL
    check_same(wide, narrow)

    # 2x2 stride-2 transposed conv as four pixel-scattered 1x1 convs into one map: Cout 128, 144 tiles each
    wt = torch.randn(Cin, 128, 2, 2, generator=gen) * Cin ** -0.5
    from thinktwice_b200.weights import Packer
    ups = Packer({'u.weight': wt}, torch.device('cuda:0'), tc_mode=IMPL).convT('u')
    up = eng.fmap('we.up', N, 2 * H, 2 * W, 128, split=True)

    def run_scatter():
        for i in range(2):
            for j in range(2):
                eng.conv(xs, ups[i][j], out=up, scatter=(2, i, 2, j))
        return {'y': up.nchw(), 'planes': split_value(up)}

    wide, narrow = both_tiles(run_scatter)
    refT = F.conv_transpose2d(x.double(), wt.double(), stride=2)
    assert relerr(wide['y'], refT) < TOL
    assert relerr(wide['planes'], wide['y']) < 6e-7
    check_same(wide, narrow)
