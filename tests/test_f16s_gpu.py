"""Tensor-core (wgmma) convolution on scaled-split fp16 operands (csrc/gemm_conv_f16s.cu, impl 4) against an fp64 torch reference.
Same case list as the 3xTF32 kernel (tests/test_tc_gpu.py): the two engines share the tiling and the epilogue contract.
Every case also checks the split planes the epilogue writes (hi + lo'/2048 == the fp32 output to 2^-22)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from test_tc_gpu import CASES, relerr

pytestmark = pytest.mark.gpu
IMPL = 4
TOL = 5e-6


def split_value(fm):
    """fp32 value held by the split companion of an FMap, (N, C, H, W)."""
    plane = fm.s.numel() // 2
    hi = fm.s[0].view(-1)[: fm.N * fm.H * fm.W * fm.ld].view(fm.N, fm.H, fm.W, fm.ld)[..., fm.coff:fm.coff + fm.C]
    lo = fm.s[1].view(-1)[: fm.N * fm.H * fm.W * fm.ld].view(fm.N, fm.H, fm.W, fm.ld)[..., fm.coff:fm.coff + fm.C]
    assert plane == fm.s[0].numel()
    return (hi.double() + lo.double() / 2048.0).permute(0, 3, 1, 2)


def to_fmap_s(eng, name, x_nchw, ld=None, coff=0):
    """channels-last FMap WITH a split companion, filled from an NCHW tensor."""
    N, Cc, H, W = x_nchw.shape
    ld = ld or Cc
    fm = eng.fmap(name, N, H, W, ld, ld, zero=True, split=True)
    assert fm.s is not None
    fm.t[..., coff:coff + Cc] = x_nchw.permute(0, 2, 3, 1)
    eng.sync_split(fm)
    return fm.slice(coff, Cc)


def engine():
    from thinktwice_b200.engine import Engine
    eng = Engine('cuda:0', impl=IMPL)
    eng.tc_min_rows = 1
    return eng


def saturations():
    from thinktwice_b200 import lib
    n = C.c_uint(0)
    lib.check(lib.load().tt_f16s_saturation_count(C.byref(n), 1, lib._stream()), 'tt_f16s_saturation_count')
    return n.value


@pytest.mark.parametrize('case', CASES)
def test_f16s_conv_matches_fp64(case):
    from thinktwice_b200 import lib
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
    eng = engine()
    pw = Packer(sd, torch.device('cuda:0'), tc_mode=IMPL).conv('c')
    assert pw.w_h is not None and pw.w_h.dtype == torch.float16
    ld = -(-Cin // 8) * 8                                            # TMA strides: multiples of 16 bytes = 8 halves
    xf = to_fmap_s(eng, 'h.x', x.cuda(), ld=ld)
    saturations()
    n0 = lib.launch_count()
    y = eng.conv(xf, pw, name='h.y', stride=stride, pad=p, dil=dil, act=act)
    torch.cuda.synchronize()
    assert 1 <= lib.launch_count() - n0 <= 3
    assert eng.stats['late_split'] == 0
    ref = F.conv2d(x.double(), w.double(), b.double() if bias else None, stride=stride, padding=p, dilation=dil)
    ref = {0: ref, 1: F.relu(ref), 2: F.gelu(ref), 3: torch.sigmoid(ref)}[act]
    err = relerr(y.nchw(), ref)
    print(case, err)
    assert err < TOL
    assert y.s is not None and relerr(split_value(y), y.nchw()) < 6e-7      # the planes the NEXT conv will read
    assert saturations() == 0


def test_f16s_conv_epilogue_offsets_residuals_scatter_and_late_split():
    from thinktwice_b200 import lib
    from thinktwice_b200.weights import Packer
    from test_tc_gpu import to_fmap
    gen = torch.Generator().manual_seed(5)
    eng = engine()
    x = torch.randn(2, 32, 12, 16, generator=gen)
    w = torch.randn(64, 32, 3, 3, generator=gen) * 0.06
    r1, r2 = torch.randn(2, 64, 12, 16, generator=gen), torch.randn(2, 64, 12, 16, generator=gen)
    pw = Packer({'c.weight': w}, torch.device('cuda:0'), tc_mode=IMPL).conv('c')
    out = eng.fmap('h.cat', 2, 12, 16, 96, split=True)
    eng.fill(out.t, 5.0)
    eng.sync_split(out)
    y = eng.conv(to_fmap_s(eng, 'h.x2', x.cuda(), ld=40, coff=8), pw, out=out.slice(32, 64), pad=1, act=1, res=to_fmap(r1.cuda()),
                 res2=to_fmap(r2.cuda(), ld=72, coff=8))
    ref = F.relu(F.conv2d(x.double(), w.double(), padding=1) + r1.double() + r2.double())
    assert relerr(y.nchw(), ref) < 2e-5
    assert float((out.t[..., :32] - 5).abs().max()) == 0
    assert relerr(split_value(out), out.nchw()) < 6e-7               # concat slice written next to untouched neighbours
    # an input WITHOUT a companion (a raw tensor wrapped by the caller): converted on the fly, same result
    y2 = eng.conv(to_fmap(x.cuda(), ld=40, coff=8), pw, name='h.late', pad=1, act=1, res=to_fmap(r1.cuda()), res2=to_fmap(r2.cuda()))
    assert eng.stats['late_split'] == 1 and relerr(y2.nchw(), ref) < 2e-5
    top = torch.randn(2, 64, 6, 8, generator=gen)
    w1 = torch.randn(64, 32, 1, 1, generator=gen) * 0.2
    pw1 = Packer({'c.weight': w1}, torch.device('cuda:0'), tc_mode=IMPL).conv('c')
    y = eng.conv(to_fmap_s(eng, 'h.x3', x.cuda()), pw1, name='h.lat', res=to_fmap(top.cuda()), res_mode=lib.RES_UP2)
    ref = F.conv2d(x.double(), w1.double()) + F.interpolate(top.double(), size=(12, 16), mode='nearest')
    assert relerr(y.nchw(), ref) < 2e-5
    wt = torch.randn(32, 64, 2, 2, generator=gen) * 0.2
    ups = Packer({'u.weight': wt}, torch.device('cuda:0'), tc_mode=IMPL).convT('u')
    up = eng.fmap('h.up', 2, 24, 32, 64, split=True)
    xs = to_fmap_s(eng, 'h.x4', x.cuda())
    for i in range(2):
        for j in range(2):
            eng.conv(xs, ups[i][j], out=up, scatter=(2, i, 2, j))
    refT = F.conv_transpose2d(x.double(), wt.double(), stride=2)
    assert relerr(up.nchw(), refT) < 2e-5 and relerr(split_value(up), up.nchw()) < 6e-7


@pytest.mark.parametrize('case', [
    (1, 14, 28, 512, 512, 3, 1, False, 1, True),
    (1, 21, 21, 544, 128, 3, 1, True, 1, False),
    (2, 8, 8, 2048, 512, 1, 0, True, 0, False),
    (1, 28, 56, 512, 32, 3, 1, True, 0, False),
])
def test_f16s_split_k_for_underfilled_layers(case):
    from thinktwice_b200 import lib
    from thinktwice_b200.weights import Packer
    from test_tc_gpu import to_fmap
    N, H, W, Cin, Cout, k, p, bias, act, use_res = case
    gen = torch.Generator().manual_seed(sum(case[:6]))
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen) * (Cin * k * k) ** -0.5
    sd = {'c.weight': w}
    if bias:
        sd['c.bias'] = torch.randn(Cout, generator=gen)
    r = torch.randn(N, Cout, H, W, generator=gen) if use_res else None
    eng = engine()
    pw = Packer(sd, torch.device('cuda:0'), tc_mode=IMPL).conv('c')
    xf = to_fmap_s(eng, 'h.skx', x.cuda())
    n0 = lib.launch_count()
    y = eng.conv(xf, pw, name='h.sk', pad=p, act=act, res=to_fmap(r.cuda()) if use_res else None)
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 == 3                              # init + split-K kernel + finish (activation and / or split planes)
    ref = F.conv2d(x.double(), w.double(), sd['c.bias'].double() if bias else None, padding=p)
    if use_res:
        ref = ref + r.double()
    ref = F.relu(ref) if act else ref
    assert relerr(y.nchw(), ref) < TOL
    assert relerr(split_value(y), y.nchw()) < 6e-7


def test_f16s_rowpacked_stem_conv_matches_fp64():
    """7x7 s2 p3 conv on 3 channels as a 7x1 conv over 64 row-packed halves (8 per pixel) of a zero-bordered image."""
    from thinktwice_b200 import lib
    from thinktwice_b200.engine import FMap
    from thinktwice_b200.lib import _p
    from thinktwice_b200.weights import Packer
    gen = torch.Generator().manual_seed(21)
    N, H, W, Cout = 2, 36, 52, 64
    x = torch.randn(N, 3, H, W, generator=gen)
    w = torch.randn(Cout, 3, 7, 7, generator=gen) * 0.08
    eng = engine()
    pw = Packer({'c.weight': w}, torch.device('cuda:0'), tc_mode=IMPL).conv_rowpacked('c', cpad=8, kslab=64)
    Wp = W + 8
    rows = N * (H + 6) * Wp
    pbs = eng.buf('h.img#s8', (2, rows * 8), torch.float16, zero=True)
    xd = x.cuda().contiguous()
    lib.call('tt_image_to_split8', _p(xd), _p(pbs), C.c_longlong(rows * 8), N, 3, H, W, H + 6, Wp, 3, 3)
    img = (pbs[0].float() + pbs[1].float() / 2048.0).view(N, H + 6, Wp, 8)
    assert float((img[:, 3:3 + H, 3:3 + W, :3] - xd.permute(0, 2, 3, 1)).abs().max()) < 1e-6 * float(xd.abs().max())
    assert float(img[:, :3].abs().max()) == 0 and float(img[:, :, :3].abs().max()) == 0 and float(img[..., 3:].abs().max()) == 0
    n0 = lib.launch_count()
    y = eng.conv(FMap(None, N, H + 6, W, 64, ld=8, s=pbs), pw, name='h.stem', stride=2, act=1, x_hstride=Wp * 8, x_nstride=(H + 6) * Wp * 8)
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 == 1
    ref = F.relu(F.conv2d(x.double(), w.double(), stride=2, padding=3))
    assert y.H == ref.shape[2] and y.W == ref.shape[3]
    assert relerr(y.nchw(), ref) < TOL


def test_f16s_saturation_is_counted_not_silent():
    """|x| >= 65504 cannot be carried by the split format: the epilogue clamps and counts (tt_f16s_saturation_count)."""
    from thinktwice_b200.weights import Packer
    eng = engine()
    x = torch.full((1, 32, 16, 16), 300.0)
    w = torch.ones(32, 32, 1, 1)
    pw = Packer({'c.weight': w}, torch.device('cuda:0'), tc_mode=IMPL).conv('c')
    saturations()
    y = eng.conv(to_fmap_s(eng, 'h.big', x.cuda()), pw, name='h.sat')
    torch.cuda.synchronize()
    assert relerr(y.nchw(), torch.full((1, 32, 16, 16), 9600.0)) < 1e-6 and saturations() == 0
    pw2 = Packer({'c.weight': w * 10}, torch.device('cuda:0'), tc_mode=IMPL).conv('c')
    y = eng.conv(to_fmap_s(eng, 'h.big', x.cuda()), pw2, name='h.sat')
    torch.cuda.synchronize()
    assert float(y.t.max()) == 96000.0                               # the fp32 output is exact ...
    assert saturations() > 0 and float(split_value(y).max()) < 65505  # ... its split planes are clamped, and say so


@pytest.mark.parametrize('form', ['tap', 'os'])
@pytest.mark.parametrize('Cin,Cout,density', [(64, 128, 0.25), (32, 32, 0.3), (128, 64, 0.15)])
def test_f16s_sparse_conv_layers_match_oracle(Cin, Cout, density, form):
    """form 'tap': tap-major pair lists + red.add (3 launches); 'os': output-stationary over the neighbour table, ONE launch with
    bias / residual / activation / split planes fused."""
    from oracle.lidar import SparseConvBase, SparseTensor
    from thinktwice_b200.lib import RulebookDesc, _p
    from thinktwice_b200 import lib
    from thinktwice_b200.engine import PackedConv
    from thinktwice_b200.weights import f16s_split
    eng = engine()
    gen = torch.Generator().manual_seed(13)
    B, shape = 2, (9, 24, 20)
    mask = torch.rand(B, *shape, generator=gen) < density
    coords = mask.nonzero().int()
    coords = coords[torch.randperm(coords.shape[0], generator=gen)]
    n = coords.shape[0]
    feats = torch.randn(n, Cin, generator=gen)
    x = SparseTensor(feats.double(), coords, shape, B)
    for (k, s, p, subm) in [((3, 3, 3), (1, 1, 1), (1, 1, 1), True), ((3, 3, 3), (2, 2, 2), (1, 1, 1), False),
                            ((3, 1, 1), (2, 1, 1), (0, 0, 0), False)]:
        conv = SparseConvBase(Cin, Cout, k, stride=s, padding=p, subm=subm)
        w = conv.weight.detach().clone()                         # fp32 weights; the reference runs them in float64
        with torch.no_grad():
            ref = conv.double()(x).dense()
        cap_in = n + 7
        out_shape = shape if subm else tuple((shape[i] + 2 * p[i] - k[i]) // s[i] + 1 for i in range(3))
        cap_out = cap_in if subm else min(cap_in * 8, B * out_shape[0] * out_shape[1] * out_shape[2])
        d = RulebookDesc()
        d.B, d.in_shape, d.out_shape, d.k, d.s, d.p = B, lib.i3(shape), lib.i3(out_shape), lib.i3(k), lib.i3(s), lib.i3(p)
        d.subm, d.cap_in, d.cap_out = int(subm), cap_in, cap_out
        t = 1024
        while t < 2 * max(cap_in, cap_out):
            t <<= 1
        d.table_size = t
        ws = torch.empty(lib.load().tt_rulebook_workspace_bytes(C.byref(d)), dtype=torch.uint8, device='cuda')
        ic = torch.zeros(cap_in, 4, dtype=torch.int32, device='cuda'); ic[:n] = coords.cuda()
        icount = torch.tensor([n], dtype=torch.int32, device='cuda')
        oc = torch.zeros(cap_out, 4, dtype=torch.int32, device='cuda'); ocount = torch.zeros(1, dtype=torch.int32, device='cuda')
        kvol = k[0] * k[1] * k[2]
        pin, pout = (torch.zeros(kvol, cap_out, dtype=torch.int32, device='cuda') for _ in range(2))
        pcount = torch.zeros(kvol, dtype=torch.int32, device='cuda')
        nbr = torch.zeros(cap_out, kvol, dtype=torch.int32, device='cuda') if form == 'os' else None
        lib.call('tt_sparse_rulebook', C.byref(d), _p(ic), _p(icount), _p(oc), _p(ocount), _p(nbr), _p(pin), _p(pout), _p(pcount), _p(ws))
        w_h = torch.stack(f16s_split(w.reshape(Cout, kvol, Cin))).contiguous().cuda()
        pw = PackedConv(w.reshape(Cout, kvol, Cin).permute(1, 2, 0).reshape(kvol * Cin, Cout).contiguous().cuda(), None, Cin, Cout, w_h=w_h)
        fin = torch.zeros(cap_in, Cin, device='cuda'); fin[:n] = feats.cuda()
        fin_s = torch.zeros(2, cap_in * Cin, dtype=torch.float16, device='cuda')
        lib.call('tt_split_f16', _p(fin), C.c_longlong(Cin), _p(fin_s), C.c_longlong(cap_in * Cin), C.c_longlong(Cin), C.c_longlong(cap_in), Cin, None)
        out = torch.zeros(cap_out, Cout, device='cuda')
        out_s = torch.zeros(2, cap_out * Cout, dtype=torch.float16, device='cuda')
        rule = dict(kvol=kvol, cap=cap_out, pairs_in=pin, pairs_out=pout, pair_count=pcount, count=ocount, nbr=nbr)
        n0 = lib.launch_count()
        eng.sparse_conv(fin, pw, rule, out, feats_s=fin_s, out_s=out_s)
        assert lib.launch_count() - n0 == (1 if form == 'os' else 3)
        m = int(ocount.item())
        D, H, W = out_shape
        dense = torch.zeros(B, H, W, Cout * D, device='cuda')
        lib.call('tt_sparse_to_bev', _p(out), _p(oc), _p(ocount), cap_out, Cout, D, H, W, 0, _p(dense))
        got = dense.view(B, H, W, Cout, D).permute(0, 3, 4, 1, 2)
        assert relerr(got, ref) < TOL
        val = out_s[0].view(cap_out, Cout)[:m].double() + out_s[1].view(cap_out, Cout)[:m].double() / 2048.0
        assert relerr(val, out[:m]) < 6e-7


def test_f16s_split_only_tensors_chain_through_convs_residuals_and_copies():
    """fmt='s': a tensor only convolutions read is stored as split planes alone — operands AND residuals come from the planes
    (tt_f16s_io.res_split), under-filled layers still split-K through a lent fp32 workspace, concat copies move planes, and
    tt_merge_f16 rebuilds fp32 where a map keeps both forms."""
    from thinktwice_b200.weights import Packer
    gen = torch.Generator().manual_seed(9)
    eng = engine()
    eng.tc_min_rows = 128
    N, H, W = 2, 24, 32
    x = torch.randn(N, 64, H, W, generator=gen)
    w1 = torch.randn(64, 64, 3, 3, generator=gen) * 0.05
    w2 = torch.randn(64, 64, 1, 1, generator=gen) * 0.12
    w3 = torch.randn(128, 128, 3, 3, generator=gen) * 0.03
    dev = torch.device('cuda:0')
    p1, p2, p3 = (Packer({'c.weight': w}, dev, tc_mode=IMPL).conv('c') for w in (w1, w2, w3))
    xf = to_fmap_s(eng, 'so.x', x.cuda())
    y1 = eng.conv(xf, p1, name='so.y1', pad=1, act=1, fmt='s')
    assert y1.t is None and y1.s is not None
    y2 = eng.conv(y1, p2, name='so.y2', act=1, res=y1, fmt='s')             # split operand, split residual, split-only output
    cat = eng.fmap('so.cat', N, H, W, 128, fmt='fs')
    eng.copy_cols(y2, cat.slice(0, 64))                                       # planes -> planes (+ fp32 rebuilt by tt_merge_f16)
    eng.copy_cols(y1, cat.slice(64, 64))
    y3 = eng.conv(cat, p3, name='so.y3', stride=2, pad=1, res2=None, fmt='s')
    torch.cuda.synchronize()
    r1 = F.relu(F.conv2d(x.double(), w1.double(), padding=1))
    r2 = F.relu(F.conv2d(r1, w2.double()) + r1)
    r3 = F.conv2d(torch.cat([r2, r1], 1), w3.double(), stride=2, padding=1)
    assert relerr(y1.nchw(), r1) < TOL and relerr(y2.nchw(), r2) < TOL
    assert relerr(cat.nchw(), torch.cat([r2, r1], 1)) < TOL                   # the fp32 side of the concat buffer
    assert relerr(split_value(cat), torch.cat([r2, r1], 1)) < TOL
    assert y3.t is None and relerr(y3.nchw(), r3) < 2 * TOL
    assert eng.stats['late_split'] == 0
    # an fp32 kernel asked to read a split-only map fails loudly
    from thinktwice_b200 import lib
    with pytest.raises(lib.TTError):
        eng.maxpool3x3s2(y1, 'so.pool')
    # a non-conv producer with a split-only result: fp32 lives in the lane scratch only until it is converted
    up = eng.upsample2x(cat.slice(0, 128), 'so.up', fmt='s')
    assert up.t is None
    ref_up = F.interpolate(torch.cat([r2, r1], 1), scale_factor=2, mode='bilinear', align_corners=True)
    assert relerr(up.nchw(), ref_up) < TOL


@pytest.mark.parametrize('Cin,Cout,act', [(12, 64, 1), (64, 32, 0), (64, 12, 0), (32, 32, 1), (64, 64, 1)])
def test_f16s_thin_pointwise_conv_matches_fp64(Cin, Cout, act):
    """tt_pointwise_f16s: thin 1x1 heads over large maps as a per-pixel fp32 mat-vec (one thread per pixel, planes in, fp32 + planes out)."""
    from thinktwice_b200 import lib
    from thinktwice_b200.weights import Packer
    gen = torch.Generator().manual_seed(Cin * 100 + Cout)
    N, H, W = 2, 96, 160
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, 1, 1, generator=gen) * Cin ** -0.5
    b = torch.randn(Cout, generator=gen)
    eng = engine()
    eng.thin_min_rows = 1
    cp = 32 if Cout < 32 else None                                       # the model pads thin heads to 32 output channels
    pw = Packer({'c.weight': w, 'c.bias': b}, torch.device('cuda:0'), tc_mode=IMPL).conv('c', cout_pad=cp)
    xf = to_fmap_s(eng, 'pw.x', x.cuda(), ld=max(32, -(-Cin // 8) * 8))
    n0 = lib.launch_count()
    y = eng.conv(xf, pw, name='pw.y', act=act)
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 == (2 if pw.Cout > 32 else 1)
    ref = F.conv2d(x.double(), w.double(), b.double())
    ref = F.relu(ref) if act else ref
    got = y.nchw()[:, :Cout]
    assert relerr(got, ref) < 2e-6
    assert relerr(split_value(y)[:, :Cout], got) < 6e-7
    if pw.Cout > Cout:
        assert float(y.nchw()[:, Cout:].abs().max()) == 0
