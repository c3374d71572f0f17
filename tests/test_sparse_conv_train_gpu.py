"""Training-side sparse convolution on the GPU (include/tt_b200.h §13, thinktwice_b200/ops/sparse_conv.py) against the float64
reference of tests/sparse_conv_reference.py (the oracle's explicit-rulebook SparseConvBase under autograd, run in float64).

Error bound: |got - ref| <= TOL * S per element, S = the float64 sum of |term| of that element.  The tensor-core layers form every product
in 3xTF32 (~2^-21 relative) and accumulate in fp32; the thin layers multiply in fp32 FFMA.  Both add at most 27 * Cin (forward), 27 * Cout
(grad_input) or one tap's pairs (grad_weight, folded in fixed-size pieces) terms, each addition erring by 2^-24 of the running |sum| <= S,
so the observed error stays far below TOL = 1e-5 (the DCN tests' bound, for reductions of the same depth)."""
import ctypes as C

import pytest
import torch

import lidar_sparse_checks as L
from sparse_conv_reference import abs_bounds, reference, site_keys, worst

pytestmark = pytest.mark.gpu
TOL = 1e-5
SHAPE = (41, 672, 672)
B = 2


@pytest.fixture(scope='module')
def levels():
    """the voxelised seeded cloud (B = 2) and the site sets of every resolution of the thinktwice.py encoder."""
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.ops.sparse_conv import build_rulebook
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    vl, shape = L.voxel_layer(cfg)
    pts = make_batch(cfg, B, seed=0, num_points=40000)['points'][:, 0].float().contiguous().cuda()
    pts[1, 31000:] = 0                                           # frames of unequal size (collate padding)
    vox = L.run_voxelize(pts, vl)
    n = int(vox['count'].item())
    coords, feats = vox['coords'][:n].contiguous(), vox['feats'][:n].contiguous()
    out = {'l0': (coords, list(shape))}
    c, s = coords, list(shape)
    for i, pad in enumerate([(1, 1, 1), (1, 1, 1), (0, 1, 1)]):
        rb = build_rulebook(c, B, s, (3, 3, 3), (2, 2, 2), pad, False)
        c, s = rb.out_indices.contiguous(), rb.out_shape
        out[f'l{i + 1}'] = (c, s)
    return dict(levels=out, feats=feats)


# every distinct convolution of the reference encoder: (name, level, Cin, Cout, kernel, stride, padding, subm)
LAYERS = [('conv_input', 'l0', 5, 16, (3, 3, 3), (1, 1, 1), (1, 1, 1), True),
          ('subm16', 'l0', 16, 16, (3, 3, 3), (1, 1, 1), (1, 1, 1), True),
          ('down16_32', 'l0', 16, 32, (3, 3, 3), (2, 2, 2), (1, 1, 1), False),
          ('subm32', 'l1', 32, 32, (3, 3, 3), (1, 1, 1), (1, 1, 1), True),
          ('down32_64', 'l1', 32, 64, (3, 3, 3), (2, 2, 2), (1, 1, 1), False),
          ('subm64', 'l2', 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), True),
          ('down64_128', 'l2', 64, 128, (3, 3, 3), (2, 2, 2), (0, 1, 1), False),
          ('subm128', 'l3', 128, 128, (3, 3, 3), (1, 1, 1), (1, 1, 1), True),
          ('conv_out', 'l3', 128, 128, (3, 1, 1), (2, 1, 1), (0, 0, 0), False)]


def _module(Cin, Cout, k, s, p, subm, seed):
    from thinktwice_b200.ops.sparse_conv import SparseConv3d, SubMConv3d
    torch.manual_seed(seed)
    cls = SubMConv3d if subm else SparseConv3d
    return cls(Cin, Cout, k, stride=s, padding=p, bias=False).cuda()


def _run(conv, x, coords, shape, seed, gy=None):
    """ours: (y, out_coords, grad_x, grad_w, gy) through the module and autograd."""
    from thinktwice_b200.ops.sparse_conv import SparseConvTensor
    xs = x.detach().clone().requires_grad_(True)
    conv.weight.grad = None
    out = conv(SparseConvTensor(xs, coords, shape, B))
    if gy is None:
        g = torch.Generator(device='cuda').manual_seed(seed)
        gy = torch.randn(out.features.shape, generator=g, device='cuda')
    out.features.backward(gy)
    torch.cuda.synchronize()
    return out.features.detach(), out.indices, xs.grad, conv.weight.grad.clone(), gy


def _check(conv, x, coords, shape, k, s, p, subm, got, name):
    y, oc, gx, gw, gy = got
    ry, roc, rgx, rgw = reference(x, coords, shape, B, conv.weight.detach(), k, s, p, subm, gy)
    by, bgx, bgw = abs_bounds(x, coords, shape, B, conv.weight.detach(), k, s, p, subm, gy)
    out_shape = shape if subm else [(shape[a] + 2 * p[a] - k[a]) // s[a] + 1 for a in range(3)]
    ko, kr = site_keys(oc, out_shape), site_keys(roc, out_shape)
    assert torch.equal(ko.sort()[0], kr.sort()[0]), name + ': output sites'
    o1, o2 = ko.argsort(), kr.argsort()
    errs = (worst(y[o1], ry[o2], by[o2]), worst(gx, rgx, bgx), worst(gw, rgw, bgw))
    for e, what in zip(errs, ('forward', 'grad_input', 'grad_weight')):
        assert e <= TOL, (name, what, e)
    return errs


@pytest.mark.parametrize('layer', LAYERS, ids=[l[0] for l in LAYERS])
def test_every_layer_of_the_reference_encoder(levels, layer):
    name, lvl, Cin, Cout, k, s, p, subm = layer
    coords, shape = levels['levels'][lvl]
    g = torch.Generator(device='cuda').manual_seed(Cin * 7 + Cout)
    x = levels['feats'] if Cin == 5 else torch.randn(coords.shape[0], Cin, generator=g, device='cuda')
    conv = _module(Cin, Cout, k, s, p, subm, seed=Cin + Cout)
    got = _run(conv, x, coords, shape, seed=1)
    errs = _check(conv, x, coords, shape, k, s, p, subm, got, name)
    print(f'{name}: {coords.shape[0]} sites, err / bound forward {errs[0]:.3g} grad_input {errs[1]:.3g} grad_weight {errs[2]:.3g}')
    again = _run(conv, x, coords, shape, seed=1, gy=got[4])
    assert torch.equal(again[3], got[3]), name + ': grad_weight is not bitwise reproducible'
    assert torch.equal(again[1], got[1])


def _corner_cloud(kind):
    D, H, W = SHAPE
    if kind == 'one_frame_empty':                               # frame 1 has no site
        c = [[0, z, y, x] for z in (0, 1, 2) for y in (10, 11, 12) for x in (20, 21, 22, 30)]
    elif kind == 'isolated':                                    # sites 4 apart: SubM has pairs on the centre tap only
        c = [[b, 4 * i % D, 4 * i, 8 + 4 * (i % 5)] for b in range(B) for i in range(1, 40)]
    elif kind == 'border':                                      # every corner and edge of the grid, both frames
        c = [[b, z, y, x] for b in range(B) for z in (0, 1, D - 2, D - 1) for y in (0, 1, H - 1) for x in (0, W - 2, W - 1)]
    else:                                                       # unequal frames: a dense block in frame 0, a few sites in frame 1
        c = [[0, z, y, x] for z in range(5) for y in range(6) for x in range(7)] + [[1, 3, 100, 200], [1, 4, 100, 201], [1, 40, 671, 0]]
    return torch.tensor(c, dtype=torch.int32, device='cuda')


@pytest.mark.parametrize('kind', ['one_frame_empty', 'isolated', 'border', 'unequal'])
@pytest.mark.parametrize('Cin,Cout', [(5, 16), (32, 64)])
def test_corner_cases(kind, Cin, Cout):
    coords = _corner_cloud(kind)
    g = torch.Generator(device='cuda').manual_seed(3)
    x = torch.randn(coords.shape[0], Cin, generator=g, device='cuda')
    for k, s, p, subm in [((3, 3, 3), (1, 1, 1), (1, 1, 1), True), ((3, 3, 3), (2, 2, 2), (1, 1, 1), False),
                          ((3, 3, 3), (2, 2, 2), (0, 1, 1), False), ((3, 1, 1), (2, 1, 1), (0, 0, 0), False)]:
        conv = _module(Cin, Cout, k, s, p, subm, seed=5)
        _check(conv, x, coords, list(SHAPE), k, s, p, subm, _run(conv, x, coords, list(SHAPE), seed=2), f'{kind} {k} {s} {p}')
    if kind == 'isolated':
        from thinktwice_b200.ops.sparse_conv import build_rulebook
        pc = build_rulebook(coords, B, list(SHAPE), (3, 3, 3), (1, 1, 1), (1, 1, 1), True).pair_count.tolist()
        assert pc[13] == coords.shape[0] and sum(pc) == pc[13]      # every other tap has zero pairs


def test_a_batch_with_no_sites():
    from thinktwice_b200.ops.sparse_conv import SparseConvTensor
    for subm in (True, False):
        conv = _module(32, 32, 3, 1 if subm else 2, 1, subm, seed=1)
        x = torch.zeros(0, 32, device='cuda', requires_grad=True)
        out = conv(SparseConvTensor(x, torch.zeros(0, 4, dtype=torch.int32, device='cuda'), list(SHAPE), B))
        assert out.features.shape == (0, 32)
        out.features.sum().backward()
        assert x.grad.shape == (0, 32) and float(conv.weight.grad.abs().sum()) == 0


def _abi(coords_buf, count, cap, Cin, Cout, k, s, p, subm):
    """the ABI chain with capacity-sized buffers: tt_sparse_rulebook (nbr), tt_sparse_pairs_ordered."""
    from thinktwice_b200 import lib
    from thinktwice_b200.lib import _p
    from thinktwice_b200.ops.sparse_conv import _out_shape, _pow2
    kvol = k[0] * k[1] * k[2]
    out_shape = _out_shape(list(SHAPE), k, s, p, subm)
    cap_out = cap if subm else cap * 8
    d = lib.RulebookDesc()
    d.B, d.in_shape, d.out_shape, d.k, d.s, d.p = B, lib.i3(SHAPE), lib.i3(out_shape), lib.i3(k), lib.i3(s), lib.i3(p)
    d.subm, d.cap_in, d.cap_out, d.table_size = int(subm), cap, cap_out, _pow2(2 * cap_out)
    Lb = lib.load()
    ws = torch.empty(Lb.tt_rulebook_workspace_bytes(C.byref(d)), dtype=torch.uint8, device='cuda')
    oc = torch.full((cap_out, 4), -7, dtype=torch.int32, device='cuda')
    ocount = torch.empty(1, dtype=torch.int32, device='cuda')
    nbr = torch.full((cap_out, kvol), 12345, dtype=torch.int32, device='cuda')
    lib.call('tt_sparse_rulebook', C.byref(d), _p(coords_buf), _p(count), _p(oc), _p(ocount), _p(nbr), _p(None), _p(None), _p(None), _p(ws))
    return dict(oc=oc, ocount=ocount, nbr=nbr, cap_out=cap_out, kvol=kvol)


def test_a_larger_clouds_buffers_reused_by_a_smaller_one(levels):
    """capacity-sized buffers written by a large cloud, then a small one through the same buffers with device counts: the small
    cloud's pair lists, grad_weight (bitwise) and forward / grad_input rows equal those of fresh buffers; rows past the counts are
    not written."""
    from thinktwice_b200 import lib
    from thinktwice_b200.lib import _p
    from thinktwice_b200.ops.sparse_conv import conv_desc
    big, _ = levels['levels']['l1']
    n_big = big.shape[0]
    n_small = n_big // 3
    Cin, Cout, k, s, p = 32, 64, (3, 3, 3), (2, 2, 2), (1, 1, 1)
    cap = n_big
    g = torch.Generator(device='cuda').manual_seed(9)
    x = torch.randn(cap, Cin, generator=g, device='cuda')
    w = torch.randn(Cout, 27, Cin, generator=g, device='cuda') * 0.05
    cap_out = cap * 8
    gy = torch.randn(cap_out, Cout, generator=g, device='cuda')

    def run(coords_buf, n, bufs=None):
        count = torch.full((1,), n, dtype=torch.int32, device='cuda')
        rb = _abi(coords_buf, count, cap, Cin, Cout, k, s, p, False)
        if bufs is None:
            bufs = dict(pin=torch.full((27, cap), -5, dtype=torch.int32, device='cuda'), pout=torch.full((27, cap), -5, dtype=torch.int32, device='cuda'),
                        pc=torch.empty(27, dtype=torch.int32, device='cuda'), y=torch.full((cap_out, Cout), 777.0, device='cuda'),
                        gx=torch.full((cap, Cin), 777.0, device='cuda'), gw=torch.empty(Cout, 27, Cin, device='cuda'))
        nb = int(lib.load().tt_sparse_pairs_ordered_workspace_bytes(rb['cap_out'], 27))
        ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
        lib.call('tt_sparse_pairs_ordered', _p(rb['nbr']), _p(rb['ocount']), rb['cap_out'], 27, cap, _p(bufs['pin']), _p(bufs['pout']),
                 _p(bufs['pc']), _p(ws), C.c_size_t(nb))
        d = conv_desc(Cin, Cout, k, s, p, n_in=cap, n_out=cap_out, pair_cap=cap)
        n2 = int(lib.load().tt_sparse_conv_train_workspace_bytes(C.byref(d)))
        ws2 = torch.empty(n2, dtype=torch.uint8, device='cuda')
        lib.call('tt_sparse_conv_train_forward', C.byref(d), _p(x), _p(w), _p(bufs['pin']), _p(bufs['pout']), _p(bufs['pc']), _p(rb['ocount']),
                 _p(bufs['y']), _p(ws2), C.c_size_t(n2))
        lib.call('tt_sparse_conv_train_backward', C.byref(d), _p(x), _p(w), _p(gy), _p(bufs['pin']), _p(bufs['pout']), _p(bufs['pc']),
                 _p(count), _p(rb['ocount']), _p(bufs['gx']), _p(bufs['gw']), _p(ws2), C.c_size_t(n2))
        torch.cuda.synchronize()
        return bufs, int(rb['ocount'].item())

    buf_big = torch.zeros(cap, 4, dtype=torch.int32, device='cuda')
    buf_big.copy_(big)
    reused, _ = run(buf_big, n_big)
    small = big[:n_small].clone()
    buf_big[:n_small] = small                                        # the small cloud over the big one's buffer (stale rows after it)
    reused, m = run(buf_big, n_small, reused)
    fresh_coords = torch.zeros(cap, 4, dtype=torch.int32, device='cuda')
    fresh_coords[:n_small] = small
    fresh, m2 = run(fresh_coords, n_small)
    assert m == m2
    pc = reused['pc'].tolist()
    assert pc == fresh['pc'].tolist()
    for t, c in enumerate(pc):
        assert torch.equal(reused['pin'][t, :c], fresh['pin'][t, :c]) and torch.equal(reused['pout'][t, :c], fresh['pout'][t, :c])
        assert bool((reused['pout'][t, 1:c] > reused['pout'][t, :c - 1]).all())       # ascending output row
    assert torch.equal(reused['gw'], fresh['gw'])
    assert torch.allclose(reused['y'][:m], fresh['y'][:m], rtol=1e-5, atol=1e-5)
    assert torch.allclose(reused['gx'][:n_small], fresh['gx'][:n_small], rtol=1e-5, atol=1e-5)
    assert bool((fresh['y'][m:] == 777.0).all()) and bool((fresh['gx'][n_small:] == 777.0).all())   # rows past the counts untouched


@pytest.mark.parametrize('Cin,Cout', [(5, 16), (64, 64)])
def test_null_gradients_are_skipped_and_the_others_unchanged(levels, Cin, Cout):
    from thinktwice_b200 import lib
    from thinktwice_b200.lib import _p
    from thinktwice_b200.ops.sparse_conv import build_rulebook, conv_desc
    coords, shape = levels['levels']['l0']
    rb = build_rulebook(coords, B, shape, (3, 3, 3), (1, 1, 1), (1, 1, 1), True)
    n = coords.shape[0]
    g = torch.Generator(device='cuda').manual_seed(4)
    x, gy = torch.randn(n, Cin, generator=g, device='cuda'), torch.randn(n, Cout, generator=g, device='cuda')
    w = torch.randn(Cout, 27, Cin, generator=g, device='cuda') * 0.05
    d = conv_desc(Cin, Cout, 3, 1, 1, subm=True, n_in=n, n_out=n, pair_cap=rb.pair_cap)
    nb = int(lib.load().tt_sparse_conv_train_workspace_bytes(C.byref(d)))
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')

    def run(gin, gw):
        a = torch.full_like(x, float('nan')) if gin else None
        b = torch.full_like(w, float('nan')) if gw else None
        lib.call('tt_sparse_conv_train_backward', C.byref(d), _p(x), _p(w), _p(gy), _p(rb.pairs_in), _p(rb.pairs_out), _p(rb.pair_count),
                 _p(rb.in_count), _p(rb.out_count), _p(a), _p(b), _p(ws), C.c_size_t(nb))
        torch.cuda.synchronize()
        return a, b
    full = run(True, True)
    assert bool(torch.isfinite(full[0]).all()) and bool(torch.isfinite(full[1]).all())
    gi, _ = run(True, False)
    _, gw = run(False, True)
    assert torch.allclose(gi, full[0], rtol=1e-5, atol=1e-6) and torch.equal(gw, full[1])
    before = lib.launch_count()
    run(False, False)
    assert lib.launch_count() == before                              # nothing requested: nothing launched
    # autograd: an unrequested gradient is not computed
    from thinktwice_b200.ops.sparse_conv import SparseConvFunction
    geom = dict(kernel_size=(3, 3, 3), stride=(1, 1, 1), padding=(1, 1, 1), dilation=(1, 1, 1), groups=1, bias=False, subm=True,
                transposed=False, inverse=False)
    wp = w.view(Cout, 3, 3, 3, Cin).clone().requires_grad_(True)
    SparseConvFunction.apply(x, wp, rb, geom).backward(gy)
    assert torch.equal(wp.grad.view(Cout, 27, Cin), full[1])


def _encoder_inputs(levels):
    coords, _ = levels['levels']['l0']
    return levels['feats'], coords


def test_subm_convs_sharing_an_indice_key_build_one_rulebook(levels, monkeypatch):
    from thinktwice_b200 import lib
    from thinktwice_b200.ops.sparse_conv import SparseEncoder
    from test_sparse_conv_train_cpu import CFG
    enc = SparseEncoder(**CFG).cuda()
    calls = []
    inner = lib.call

    def spy(name, *a):
        calls.append(name)
        return inner(name, *a)
    monkeypatch.setattr(lib, 'call', spy)
    feats, coords = _encoder_inputs(levels)
    enc(feats, coords, B)
    # 17 SubM convs on 4 resolutions share 4 rulebooks; 3 downsamplings and conv_out have their own
    assert calls.count('tt_sparse_rulebook') == 8 and calls.count('tt_sparse_pairs_ordered') == 8
    assert calls.count('tt_sparse_conv_train_forward') == 21


def test_encoder_forward_and_backward_against_the_oracle_in_float64(levels):
    """SparseEncoder at the full thinktwice.py shape, BatchNorm in train mode, against oracle.lidar.SparseEncoder in float64 with
    the same state dict: the dense output, grad(voxel_features) and every parameter gradient within 1e-3 of the reference's max.
    Twenty train-mode BatchNorms and ReLUs deep, fp32 itself can miss that bound on a tensor (a ReLU whose input rounds to the other
    side of 0, the cancellation of the train-mode BatchNorm backward over ~10^5 rows): on an H100 the oracle run in plain fp32 (TF32 off)
    errs by up to 1.6e-2 on a weight gradient, and which tensor errs most changes from run to run (index_add_ and red.add orders).  So
    each tensor must be within max(1e-3, 2 x the plain-fp32 oracle's worst error over all tensors).  Every single layer is held to 1e-5
    of S above."""
    from oracle.lidar import SparseEncoder as OracleEncoder
    from thinktwice_b200.ops.sparse_conv import SparseEncoder
    from test_sparse_conv_train_cpu import CFG
    torch.manual_seed(0)
    ref = OracleEncoder(**CFG)
    with torch.no_grad():
        for m in ref.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
    ours, r32 = SparseEncoder(**CFG), OracleEncoder(**CFG)
    ours.load_state_dict(ref.state_dict())
    r32.load_state_dict(ref.state_dict())
    ref, r32, ours = ref.cuda().double().train(), r32.cuda().train(), ours.cuda().train()
    feats, coords = _encoder_inputs(levels)
    g = torch.Generator(device='cuda').manual_seed(1)
    G = torch.randn((B, 256, 84, 84), generator=g, device='cuda', dtype=torch.float64)

    def run(model, dtype):
        x = feats.to(dtype).clone().requires_grad_(True)
        y = model(x, coords, B)
        assert y.shape == (B, 256, 84, 84)
        (y * G.to(dtype)).sum().backward()
        return [y.detach(), x.grad] + [p.grad for _, p in model.named_parameters()]
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        got, want, plain = run(ours, torch.float32), run(ref, torch.float64), run(r32, torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    names = ['output', 'grad(voxel_features)'] + [n for n, _ in ours.named_parameters()]
    report = []
    for name, a, b, c in zip(names, got, want, plain):
        scale = float(b.abs().max())
        e, e32 = float((a.double() - b).abs().max()) / scale, float((c.double() - b).abs().max()) / scale
        report.append((name, e, e32))
    print('encoder |err| / max|ref| (fp32 oracle):\n  ' + '\n  '.join(f'{n}: {e:.3g} ({e32:.3g})' for n, e, e32 in report))
    bound = max(1e-3, 2 * max(e32 for _, _, e32 in report))
    for name, e, e32 in report:
        assert e <= bound, (name, e, bound)
