"""Training lift-splat (tt_lift_splat_train_forward / _backward, thinktwice_b200.ops.lift_splat) at the thinktwice.py shapes against
the float64 reference of tests/lift_splat_train_reference.py: the forward BEV within check_lift's bound, every recorded cell equal to
the float64 cell, both gradients within the derived bound, bitwise repeatable backward over every layout of the BEV gradient, the
whole op under autograd between two convolutions, and its memory.  Each test prints its largest error-to-bound ratio."""
import ctypes as C

import numpy as np
import pytest
import torch

import camera_look_checks as K
import lift_splat_train_reference as R
from thinktwice_b200 import lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def geo():
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    return K.lift_geometry(Config.fromfile(DEFAULT_CONFIG))


def _mats(geo, B):
    from thinktwice_b200.synthetic import rig_metas
    return K.sweep_mats([rig_metas(geo['final_dim'], geo['queue_len']) for _ in range(B)], geo['N'], 0)


def _inputs(geo, B, seed):
    """NCHW logits (the flat / sharp / one-hot mix) as the [:, :D] view of a wider map, context, and G, on the GPU."""
    gen = torch.Generator().manual_seed(seed)
    BN, D, fH, fW, Cc = B * geo['N'], geo['D'], geo['fH'], geo['fW'], geo['C']
    dl = K.depth_logits(gen, BN, fH, fW, D).permute(0, 3, 1, 2)
    wide = torch.full((BN, D + Cc, fH, fW), float('nan'))
    wide[:, :D] = dl
    ctx = torch.randn(BN, Cc, fH, fW, generator=gen)
    G = torch.randn(B, Cc, geo['Y'], geo['X'], generator=gen)
    return wide.cuda()[:, :D], ctx.cuda(), G.cuda()


def _check_all(geo, B, s2e, intr, ida, logits, ctx, G, name):
    """forward (+ the inference tt_lift_splat on the same inputs), cells, gradients.  Returns (bev ratio, inference ratio, gl, gc)."""
    Cc, D = geo['C'], geo['D']
    mats = K.kernel_mats(s2e, intr, ida)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
    ref = K.ref_lift(nhwc(logits).cpu().numpy(), nhwc(ctx).cpu().numpy(), s2e, intr, ida, mats, geo)
    d = R.train_desc(geo, B, Cc, logits.stride(0))
    bev = torch.full((B, geo['Y'], geo['X'], Cc), float('nan'), device='cuda')
    cells = torch.full((B * geo['N'] * geo['fH'] * geo['fW'], D), -7, dtype=torch.int32, device='cuda')
    R.run_forward(d, geo, logits, ctx, mats, bev, cells)
    nan = np.full(bev.shape, np.nan, np.float32)
    r_bev = K.check_lift(bev.cpu().numpy(), nan, ref, geo, 0, name=f'{name} forward')
    inf = torch.full_like(bev, float('nan'))
    K.run_lift(K.lift_desc(geo, B, Cc, D, 0, Cc, 0, Cc, 0), geo, nhwc(logits), nhwc(ctx), mats.cuda(), inf)
    r_inf = K.check_lift(inf.cpu().numpy(), nan, ref, geo, 0, name=f'{name} tt_lift_splat')
    rc = R.ref_cells(s2e, intr, ida, mats, geo)
    R.check_bin_cell(cells.cpu().numpy(), rc, name=f'{name} bin_cell')
    gl, gc = torch.full_like(logits, float('nan')), torch.full_like(ctx, float('nan'))
    R.run_backward(d, logits, ctx, cells, G, gl, gc)
    rg = R.ref_grads(logits, ctx, cells.cpu().numpy(), G)
    r_gl, r_gc = R.check_grads(gl, gc, rg, name=name)
    print(f'[lift-train] {name}: {rc["in_bins"]} bins in the grid, {rc["amb_bins"]} ambiguous; err/bound forward {r_bev:.4f}, '
          f'tt_lift_splat {r_inf:.4f}, grad_logits {r_gl:.4f}, grad_context {r_gc:.4f}')
    return dict(d=d, cells=cells, gl=gl, gc=gc, rg=rg, ref=ref)


@pytest.mark.parametrize('B', [1, 8])
def test_forward_cells_and_gradients_at_the_model_shape(geo, B):
    s2e, intr, ida = _mats(geo, B)
    logits, ctx, G = _inputs(geo, B, 30 + B)
    _check_all(geo, B, s2e, intr, ida, logits, ctx, G, f'B={B}')


def _crafted(geo, B):
    """frame 0: cam 0 pixel (i, j) -> cell (x i, y j); cam 1 on the truncation band t_x in (-0.9, -0.1), t_z = -0.5; cam 2 misses
    the grid (t_z = -3); cam 3 is the rig.  Frame 1: every camera misses (an empty BEV).  Frames >= 2: the rig.  Set up like the
    crafted rays of test_camera_look_gpu.py: ida swaps rows 2 and 3 and intrin = I, so every bin of a pixel lands on one point."""
    N = geo['N']
    lower, size = geo['lower'].astype(np.float64), geo['size'].astype(np.float64)
    su, sv, umax = float(geo['fu'][1] - geo['fu'][0]), float(geo['fv'][1] - geo['fv'][0]), float(geo['fu'][-1])
    s2e, intr, ida = (t.clone() for t in _mats(geo, B))
    P = torch.eye(4)[[0, 1, 3, 2]]

    def mc(tx, ty, tz):
        m = torch.zeros(4, 4, dtype=torch.float64)
        for r, (cu, cv, c0) in enumerate((tx, ty, tz)):
            m[r, 0], m[r, 1], m[r, 2] = cu * size[r], cv * size[r], lower[r] + c0 * size[r]
        m[3, 3] = 1
        return m.float()
    cams = {(0, 0): mc((1 / su, 0, 0.5), (0, 1 / sv, 0.5), (0, 0, 0.5)),
            (0, 1): mc((0.8 / umax, 0, -0.9), (0, 1 / sv, 0.5), (0, 0, -0.5)),
            (0, 2): mc((1 / su, 0, 0.5), (0, 1 / sv, 0.5), (0, 0, -3.0))}
    for n in range(N):
        cams[(1, n)] = mc((0, 0, -5.5), (0, 1 / sv, 0.5), (0, 0, 0.5))
    for (b, n), m in cams.items():
        s2e[b, n], intr[b, n], ida[b, n] = m, torch.eye(4), P
    return s2e, intr, ida


def test_crafted_rays_empty_frame_truncation_band_and_one_hot_pixels(geo):
    B, N, D = 3, geo['N'], geo['D']
    s2e, intr, ida = _crafted(geo, B)
    logits, ctx, G = _inputs(geo, B, 41)
    out = _check_all(geo, B, s2e, intr, ida, logits, ctx, G, 'crafted')
    HW = geo['fH'] * geo['fW']
    cells = out['cells'].cpu().numpy().reshape(B * N, HW, D)
    assert (cells[2] == -1).all() and (cells[N:2 * N] == -1).all()            # the missing camera, the empty frame
    assert (out['gl'][2] == 0).all() and (out['gc'][2] == 0).all()             # their gradients are exactly 0
    assert (out['gl'][N:2 * N] == 0).all() and (out['gc'][N:2 * N] == 0).all()
    assert not out['ref']['reached'][1].any()
    assert (cells[1] % geo['X'] == 0)[cells[1] >= 0].all() and (cells[1] >= 0).any()   # the band lands in cell column x 0
    hot = (logits.max(1).values == 0) & ((logits == -200).sum(1) == D - 1)     # one-hot pixels: the other weights underflow to 0
    assert hot.any()
    gl = out['gl'].permute(0, 2, 3, 1)[hot]
    assert (gl[logits.permute(0, 2, 3, 1)[hot] == -200] == 0).all()


def test_backward_is_bitwise_repeatable_over_layouts_and_skips_null_gradients(geo):
    B, Cc = 2, geo['C']
    s2e, intr, ida = _mats(geo, B)
    logits, ctx, G = _inputs(geo, B, 50)
    d = R.train_desc(geo, B, Cc, logits.stride(0))
    cells = torch.empty(B * geo['N'] * geo['fH'] * geo['fW'], geo['D'], dtype=torch.int32, device='cuda')
    R.run_forward(d, geo, logits, ctx, K.kernel_mats(s2e, intr, ida), torch.empty(B, geo['Y'], geo['X'], Cc, device='cuda'), cells)
    cat = torch.cat([torch.randn_like(G), G, torch.randn_like(G)], 1)
    layouts = {'contiguous': G, 'permuted NHWC': G.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2), 'concat slice': cat[:, Cc:2 * Cc]}
    outs = []
    for name, g in list(layouts.items()) + [('contiguous again', G)]:
        gl, gc = torch.full_like(logits, float('nan')), torch.full_like(ctx, float('nan'))
        R.run_backward(d, logits, ctx, cells, g, gl, gc)
        outs.append((name, gl, gc))
    for name, gl, gc in outs[1:]:
        assert torch.equal(gl, outs[0][1]) and torch.equal(gc, outs[0][2]), name
    buf = torch.full((logits.numel() + ctx.numel(),), K.SENT, device='cuda')      # [grad_logits | grad_context] in one buffer
    gl, gc = buf[:logits.numel()].view(logits.shape), buf[logits.numel():].view(ctx.shape)
    R.run_backward(d, logits, ctx, cells, G, gl, None)
    assert torch.equal(gl, outs[0][1]) and (gc == K.SENT).all()
    gl.fill_(K.SENT)
    R.run_backward(d, logits, ctx, cells, G, None, gc)
    assert torch.equal(gc, outs[0][2]) and (gl == K.SENT).all()
    n0 = lib.launch_count()
    R.run_backward(d, logits, ctx, cells, G, None, None)
    assert lib.launch_count() == n0


def test_empty_batch_launches_nothing(geo):
    d = R.train_desc(geo, 0, geo['C'])
    n0 = lib.launch_count()
    null = C.c_void_p(0)
    L = lib.load()
    assert L.tt_lift_splat_train_forward(C.byref(d), null, null, null, null, null, null, null, null, null, C.c_size_t(0), null) == 0
    assert L.tt_lift_splat_train_backward(C.byref(d), null, null, null, null, C.c_longlong(0), C.c_longlong(0), C.c_longlong(0),
                                          C.c_longlong(0), null, null, null, C.c_size_t(0), null) == 0
    torch.cuda.synchronize()
    assert lib.launch_count() == n0


def _composition(geo, B, logits, ctx, s2e, intr, ida, dtype, pool):
    """lss.py:583-615 as torch ops: softmax, outer product, permute + contiguous, voxel pooling of the geometry's cells."""
    from oracle.camera import LSS as OLSS
    import types
    m = geo['lss']
    dev = ctx.device
    ns = types.SimpleNamespace(frustum=geo['frustum'].to(dev, dtype), voxel_coord=m.voxel_coord.to(dev, dtype),
                               voxel_size=m.voxel_size.to(dev, dtype))
    geom = OLSS.get_geometry(ns, s2e.to(dev, dtype), intr.to(dev, dtype), ida.to(dev, dtype))
    idx = OLSS.geom_index(ns, geom).contiguous()
    N, Cc, D, fH, fW = geo['N'], ctx.shape[1], geo['D'], geo['fH'], geo['fW']
    lifted = logits.softmax(1).unsqueeze(1) * ctx.unsqueeze(2)
    lifted = lifted.reshape(B, N, Cc, D, fH, fW).permute(0, 1, 3, 4, 5, 2).contiguous()
    return pool(idx, lifted, m.voxel_num.to(dev))


def test_end_to_end_through_autograd_between_two_convolutions(geo):
    """a conv makes depth_feature (D + 16 channels), a second conv the context; the op runs on the [:, :D] view and a fixed G is
    backpropagated.  Conv weight and input gradients against the float64 composition, within max(1e-4 max|ref|, 2 x the fp32
    composition's own worst error)."""
    from oracle.voxel_pool import voxel_pooling_ref
    from thinktwice_b200.ops.lift_splat import lift_splat
    B, N, D, Cc = 1, geo['N'], geo['D'], geo['C']
    m = geo['lss']
    gen = torch.Generator().manual_seed(60)
    x0 = torch.randn(B * N, 32, geo['fH'], geo['fW'], generator=gen)
    w10, w20 = torch.randn(D + 16, 32, 3, 3, generator=gen) * 0.3, torch.randn(Cc, 32, 3, 3, generator=gen) * 0.1
    G = torch.randn(B, Cc, geo['Y'], geo['X'], generator=gen).cuda()
    s2e, intr, ida = _mats(geo, B)

    def run(dtype, op):
        x, w1, w2 = (t.cuda().to(dtype).requires_grad_(True) for t in (x0, w10, w20))
        df = torch.nn.functional.conv2d(x, w1, padding=1)
        feat = torch.nn.functional.conv2d(x, w2, padding=1)
        op(df[:, :D], feat).backward(G.to(dtype))
        return [t.grad.double() for t in (x, w1, w2)]
    ours = run(torch.float32, lambda lg, f: lift_splat(lg, f, s2e.cuda(), intr.cuda(), ida.cuda(), m.frustum, m.voxel_coord, m.voxel_size,
                                                        m.voxel_num))
    comp = lambda dtype: (lambda lg, f: _composition(geo, B, lg, f, s2e, intr, ida, dtype, voxel_pooling_ref))
    ref = run(torch.float64, comp(torch.float64))
    f32 = run(torch.float32, comp(torch.float32))
    for name, a, b, c in zip(('x', 'depth conv weight', 'context conv weight'), ours, ref, f32):
        own = float((c - b).abs().max())
        tol = max(1e-4 * float(b.abs().max()), 2 * own)
        err = float((a - b).abs().max())
        print(f'[lift-train] autograd {name}: max err {err:.3e}, fp32 composition {own:.3e}, limit {tol:.3e}')
        assert err <= tol, name


def test_memory_at_batch_8(geo):
    """peak increment of forward + backward from a reset_peak_memory_stats baseline: the op within the buffers it declares (workspace,
    bin_cell, BEV, both gradients; G is staged inside the workspace) + 1 MiB; the composition's increment printed beside it."""
    from thinktwice_b200.ops.lift_splat import lift_splat
    from thinktwice_b200.ops.voxel_pooling import voxel_pooling
    B, N, D, Cc = 8, geo['N'], geo['D'], geo['C']
    m = geo['lss']
    s2e, intr, ida = _mats(geo, B)
    logits, ctx, G = _inputs(geo, B, 70)
    mc = lambda: (s2e.cuda(), intr.cuda(), ida.cuda())
    peaks = {}
    for name in ('op', 'composition'):
        lg, f = logits.clone().requires_grad_(True), ctx.clone().requires_grad_(True)
        mats = mc()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        if name == 'op':
            out = lift_splat(lg, f, *mats, m.frustum, m.voxel_coord, m.voxel_size, m.voxel_num)
        else:
            pool = lambda idx, lifted, vn: voxel_pooling(idx, lifted, vn)
            out = _composition(geo, B, lg, f, *mats, torch.float32, pool)
        out.backward(G)
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del out, lg, f
    d = R.train_desc(geo, B, Cc)
    pixels = B * N * geo['fH'] * geo['fW']
    declared = (lib.load().tt_lift_splat_train_workspace_bytes(C.byref(d)) + pixels * D * 4 + B * geo['X'] * geo['Y'] * Cc * 4
                + pixels * (D + Cc) * 4)
    mib = lambda v: v / 2 ** 20
    print(f'[lift-train] B=8 forward + backward peak increment: op {mib(peaks["op"]):.1f} MiB (declared {mib(declared):.1f} MiB), '
          f'composition {mib(peaks["composition"]):.1f} MiB')
    assert peaks['op'] <= declared + 2 ** 20
