"""wgmma implicit-GEMM convolution (TMA + register accumulators, 3xTF32 / single-pass TF32) against an fp64 torch reference."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def relerr(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def to_fmap(x_nchw, ld=None, coff=0):
    from thinktwice_b200.engine import FMap
    N, Cc, H, W = x_nchw.shape
    ld = ld or Cc
    t = torch.zeros(N, H, W, ld, device='cuda')
    t[..., coff:coff + Cc] = x_nchw.permute(0, 2, 3, 1)
    return FMap(t, N, H, W, Cc, ld, coff)


CASES = [
    # N, H, W, Cin, Cout, k, pad, dil, bias, act [, stride]
    (2, 32, 32, 64, 128, 3, 1, 1, True, 1, 2),    # 3x3 stride 2 (ResNet conv2 / PAFPN down): TMA element strides
    (1, 28, 56, 256, 512, 1, 0, 1, False, 0, 2),  # 1x1 stride 2 (ResNet downsample)
    (2, 21, 21, 32, 64, 3, 0, 1, True, 1, 2),     # conv21_10: odd map, no padding
    (1, 84, 84, 64, 64, 3, 1, 1, False, 1, 2),    # conv_lidar / SECOND stride 2
    (2, 16, 32, 64, 128, 1, 0, 1, True, 0),       # 1x1, flat path, exact tiles
    (1, 28, 56, 256, 64, 1, 0, 1, False, 1),      # BN = 64
    (3, 13, 17, 96, 80, 1, 0, 1, True, 2),        # ragged pixel count, Cout = 80
    (1, 16, 16, 48, 32, 1, 0, 1, True, 0),        # Cin = 48: partial K slab (zero-filled by TMA)
    (2, 16, 16, 64, 128, 3, 1, 1, True, 1),       # 3x3, exact rectangle tiles
    (1, 28, 56, 128, 256, 3, 1, 1, False, 1),     # DepthNet shape, two N tiles
    (2, 21, 21, 32, 64, 3, 1, 1, True, 0),        # odd map, ragged tiles
    (1, 14, 28, 64, 64, 3, 6, 6, False, 1),       # dilated (ASPP), halo larger than the tile
    (1, 84, 84, 128, 128, 3, 1, 1, False, 1),     # SECOND shape
    (1, 40, 40, 36, 32, 3, 1, 1, True, 3),        # Cin = 36
]


@pytest.mark.parametrize('impl,tol', [(3, 3e-6), (2, 3e-3)])
@pytest.mark.parametrize('case', CASES)
def test_tc_conv_matches_fp64(case, impl, tol):
    from thinktwice_b200 import lib
    from thinktwice_b200.engine import Engine
    from thinktwice_b200.weights import Packer
    N, H, W, Cin, Cout, k, p, dil, bias, act = case[:10]
    stride = case[10] if len(case) > 10 else 1
    gen = torch.Generator().manual_seed(sum(case))
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen) * (Cin * k * k) ** -0.5
    b = torch.randn(Cout, generator=gen) if bias else None
    sd = {'c.weight': w}
    if bias:
        sd['c.bias'] = b
    eng = Engine('cuda:0', impl=impl)
    eng.tc_min_rows = 1
    pw = Packer(sd, torch.device('cuda:0'), tc_mode=impl).conv('c')
    assert pw.w_tc is not None
    n0 = lib.launch_count()
    y = eng.conv(to_fmap(x.cuda()), pw, name='tc.y', stride=stride, pad=p, dil=dil, act=act)
    torch.cuda.synchronize()
    assert 1 <= lib.launch_count() - n0 <= 3       # one tensor-core kernel (+ split-K init / activation passes)
    ref = F.conv2d(x.double(), w.double(), b.double() if bias else None, stride=stride, padding=p, dilation=dil)
    ref = {0: ref, 1: F.relu(ref), 2: F.gelu(ref), 3: torch.sigmoid(ref)}[act]
    err = relerr(y.nchw(), ref)
    print(case, impl, err)
    assert err < tol


def test_tc_conv_epilogue_offsets_residuals_scatter():
    from thinktwice_b200 import lib
    from thinktwice_b200.engine import Engine
    from thinktwice_b200.weights import Packer
    gen = torch.Generator().manual_seed(5)
    eng = Engine('cuda:0', impl=3)
    eng.tc_min_rows = 1
    x = torch.randn(2, 32, 12, 16, generator=gen)
    w = torch.randn(64, 32, 3, 3, generator=gen) * 0.06
    r1, r2 = torch.randn(2, 64, 12, 16, generator=gen), torch.randn(2, 64, 12, 16, generator=gen)
    pw = Packer({'c.weight': w}, torch.device('cuda:0'), tc_mode=3).conv('c')
    out = eng.fmap('tc.cat', 2, 12, 16, 96)
    eng.fill(out.t, 5.0)
    y = eng.conv(to_fmap(x.cuda(), ld=40, coff=8), pw, out=out.slice(32, 64), pad=1, act=1, res=to_fmap(r1.cuda()),
                 res2=to_fmap(r2.cuda(), ld=72, coff=8))
    ref = F.relu(F.conv2d(x.double(), w.double(), padding=1) + r1.double() + r2.double())
    assert relerr(y.nchw(), ref) < 2e-5
    assert float((out.t[..., :32] - 5).abs().max()) == 0
    top = torch.randn(2, 64, 6, 8, generator=gen)
    w1 = torch.randn(64, 32, 1, 1, generator=gen) * 0.2
    pw1 = Packer({'c.weight': w1}, torch.device('cuda:0'), tc_mode=3).conv('c')
    y = eng.conv(to_fmap(x.cuda()), pw1, name='tc.lat', res=to_fmap(top.cuda()), res_mode=lib.RES_UP2)
    ref = F.conv2d(x.double(), w1.double()) + F.interpolate(top.double(), size=(12, 16), mode='nearest')
    assert relerr(y.nchw(), ref) < 2e-5
    wt = torch.randn(32, 64, 2, 2, generator=gen) * 0.2
    ups = Packer({'u.weight': wt}, torch.device('cuda:0'), tc_mode=3).convT('u')
    up = eng.fmap('tc.up', 2, 24, 32, 64)
    for i in range(2):
        for j in range(2):
            eng.conv(to_fmap(x.cuda()), ups[i][j], out=up, scatter=(2, i, 2, j))
    assert relerr(up.nchw(), F.conv_transpose2d(x.double(), wt.double(), stride=2)) < 2e-5


@pytest.mark.parametrize('case', [
    # N, H, W, Cin, Cout, k, pad, bias, act, residual
    (1, 14, 28, 512, 512, 3, 1, False, 1, True),      # ResNet stage 4 3x3: 4 tiles x 4 N tiles, K = 144 slabs
    (1, 21, 21, 544, 128, 3, 1, True, 1, False),      # decoder BEV update: 441 rows, long K
    (2, 8, 8, 2048, 512, 1, 0, True, 0, False),       # 1x1 with one M tile: flat mode, no activation -> no finish kernel
    (1, 28, 56, 512, 32, 3, 1, True, 0, False),       # DCN offset conv (18 -> 32 padded), BN = 64
])
def test_tc_split_k_for_underfilled_layers(case):
    from thinktwice_b200 import lib
    from thinktwice_b200.engine import Engine
    from thinktwice_b200.weights import Packer
    N, H, W, Cin, Cout, k, p, bias, act, use_res = case
    gen = torch.Generator().manual_seed(sum(case[:6]))
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen) * (Cin * k * k) ** -0.5
    sd = {'c.weight': w}
    if bias:
        sd['c.bias'] = torch.randn(Cout, generator=gen)
    r = torch.randn(N, Cout, H, W, generator=gen) if use_res else None
    eng = Engine('cuda:0', impl=3)
    eng.tc_min_rows = 1
    pw = Packer(sd, torch.device('cuda:0'), tc_mode=3).conv('c')
    n0 = lib.launch_count()
    y = eng.conv(to_fmap(x.cuda()), pw, name='tc.sk', pad=p, act=act, res=to_fmap(r.cuda()) if use_res else None)
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 == (3 if act else 2)          # init + split-K tensor-core kernel (+ activation pass)
    ref = F.conv2d(x.double(), w.double(), sd['c.bias'].double() if bias else None, padding=p)
    if use_res:
        ref = ref + r.double()
    ref = F.relu(ref) if act else ref
    assert relerr(y.nchw(), ref) < 5e-6


@pytest.mark.parametrize('impl,tol', [(1, 2e-6), (3, 3e-6)])
def test_rowpacked_stem_conv_matches_fp64(impl, tol):
    """7x7 s2 p3 conv on 3 channels as a 7x1 conv over 32 row-packed "channels" of a zero-bordered channels-last image
    (tt_conv_desc.x_hstride, x_ld < Cin): SIMT and tensor cores against torch fp64."""
    from thinktwice_b200 import lib
    from thinktwice_b200.engine import Engine, FMap
    from thinktwice_b200.weights import Packer
    gen = torch.Generator().manual_seed(21)
    N, H, W, Cout = 2, 36, 52, 64
    x = torch.randn(N, 3, H, W, generator=gen)
    w = torch.randn(Cout, 3, 7, 7, generator=gen) * 0.08
    eng = Engine('cuda:0', impl=impl)
    eng.tc_min_rows = 1
    pw = Packer({'c.weight': w}, torch.device('cuda:0'), tc_mode=impl).conv_rowpacked('c')
    pb = eng.nchw_to_nhwc_padded(x.cuda(), 't.img', 4, 3, 3, 3, 5)
    assert float(pb[:, :3].abs().max()) == 0 and float(pb[:, :, :3].abs().max()) == 0 and float(pb[:, :, W + 3:].abs().max()) == 0
    Wp = W + 8
    n0 = lib.launch_count()
    y = eng.conv(FMap(pb, N, H + 6, W, 32, ld=4), pw, name='t.stem', stride=2, act=1, x_hstride=Wp * 4, x_nstride=(H + 6) * Wp * 4)
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 == 1
    ref = F.relu(F.conv2d(x.double(), w.double(), stride=2, padding=3))
    assert y.H == ref.shape[2] and y.W == ref.shape[3]
    assert relerr(y.nchw(), ref) < tol
