"""CPU side of the training lift-splat (include/tt_b200.h §14, thinktwice_b200/ops/lift_splat.py): the ctypes descriptor, the exports,
every refusal of the library and of the Python op, and the float64 reference of tests/lift_splat_train_reference.py pinned against
the oracle composition under autograd and against a literal loop; the gradient check rejects seeded bugs."""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest
import torch

import camera_look_checks as K
import lift_splat_train_reference as R
from thinktwice_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ctypes_descriptor_matches_the_c_header_and_the_entries_are_exported(tmp_path):
    fields = [n for n, _ in lib.LiftSplatTrainDesc._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "tt_b200.h"\nint main(void) {\n' +
                   ''.join(f'  printf("%zu\\n", offsetof(tt_lift_splat_train_desc, {n}));\n' for n in fields) +
                   '  printf("%zu\\n", sizeof(tt_lift_splat_train_desc));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(lib.LiftSplatTrainDesc, n).offset for n in fields] + [C.sizeof(lib.LiftSplatTrainDesc)]
    names = ('tt_lift_splat_train_workspace_bytes', 'tt_lift_splat_train_forward', 'tt_lift_splat_train_backward')
    assert set(names) <= set(lib.EXPORTS)
    L = lib.load()
    assert all(hasattr(L, n) for n in names)


def _desc(**kw):
    d = lib.LiftSplatTrainDesc()
    base = dict(B=8, N=4, D=80, fH=28, fW=56, C=256, X=21, Y=21, Z=1)
    base.update(kw)
    base.setdefault('depth_bstride', 336 * base['fH'] * base['fW'])     # the logits view of a (BN, 80 + 256, fH, fW) map
    for k, v in base.items():
        setattr(d, k, v)
    d.lower, d.size = lib.f3([-8.0, -19.2, -4.0]), lib.f3([1.8285, 1.8285, 14.0])
    return d


@pytest.mark.parametrize('field,value,named', [
    ('D', 129, 'D'), ('C', 258, 'C'), ('C', 516, 'C'), ('X', 20000000, 'X, Y'), ('B', 6000, 'B, N, fH, fW, D'),
    ('depth_bstride', 80 * 28 * 56 - 1, 'depth_bstride'), ('fW', 400, 'C, D, fW')])
def test_the_library_refuses_what_it_cannot_index(field, value, named):
    """checked before any pointer or device is touched: no GPU needed, nothing launched."""
    L = lib.load()
    d = _desc(**{field: value})
    n0 = L.tt_launch_count()
    assert L.tt_lift_splat_train_workspace_bytes(C.byref(d)) == 0
    null = C.c_void_p(0)
    calls = (lambda: L.tt_lift_splat_train_forward(C.byref(d), null, null, null, null, null, null, null, null, null, C.c_size_t(0), null),
             lambda: L.tt_lift_splat_train_backward(C.byref(d), null, null, null, null, C.c_longlong(0), C.c_longlong(0), C.c_longlong(0),
                                                     C.c_longlong(0), null, null, null, C.c_size_t(0), null))
    for call in calls:
        assert call() == -3                                          # TT_ERR_UNSUPPORTED
        assert f'unsupported {named}' in L.tt_last_error().decode()
    assert L.tt_launch_count() == n0


def test_a_short_workspace_is_refused_and_an_empty_batch_launches_nothing():
    L = lib.load()
    d = _desc()
    n = L.tt_lift_splat_train_workspace_bytes(C.byref(d))
    pixels = 8 * 4 * 28 * 56
    assert n >= pixels * 256 * 4 + 4 * pixels * 80 * 4 and n < 8 * 4 * 256 * 80 * 28 * 56 * 4 // 20   # far below the frustum tensor
    null, bogus = C.c_void_p(0), C.c_void_p(16)
    n0 = L.tt_launch_count()
    assert L.tt_lift_splat_train_forward(C.byref(d), bogus, bogus, bogus, bogus, bogus, bogus, bogus, bogus, bogus, C.c_size_t(n - 1), null) == -3
    assert 'unsupported ws_bytes' in L.tt_last_error().decode()
    assert L.tt_lift_splat_train_backward(C.byref(d), bogus, bogus, bogus, bogus, C.c_longlong(1), C.c_longlong(1), C.c_longlong(1),
                                          C.c_longlong(1), bogus, bogus, bogus, C.c_size_t(n - 1), null) == -3
    assert 'unsupported ws_bytes' in L.tt_last_error().decode()
    e = _desc(B=0)
    assert L.tt_lift_splat_train_forward(C.byref(e), null, null, null, null, null, null, null, null, null, C.c_size_t(0), null) == 0
    assert L.tt_lift_splat_train_backward(C.byref(e), null, null, null, null, C.c_longlong(0), C.c_longlong(0), C.c_longlong(0),
                                          C.c_longlong(0), null, null, null, C.c_size_t(0), null) == 0
    assert L.tt_launch_count() == n0


def test_the_op_refuses_cpu_tensors_other_dtypes_bda_and_shapes_off_the_frustum():
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.ops.lift_splat import lift_splat
    geo = K.lift_geometry(Config.fromfile(PLUMBING_CONFIG))
    m = geo['lss']
    BN, D, fH, fW = 4, geo['D'], geo['fH'], geo['fW']
    eye = torch.eye(4).expand(1, 4, 4, 4)
    args = lambda dep, ctx, fr=m.frustum: (dep, ctx, eye, eye, eye, fr, m.voxel_coord, m.voxel_size, m.voxel_num)
    dep, ctx = torch.randn(BN, D, fH, fW), torch.randn(BN, 8, fH, fW)
    with pytest.raises(ValueError, match='bda_mat'):
        lift_splat(*args(dep, ctx), bda_mat=torch.eye(4))
    if not torch.cuda.is_available():
        with pytest.raises(lib.TTError, match='CUDA'):
            lift_splat(*args(dep, ctx))
        return
    dep, ctx = dep.cuda(), ctx.cuda()
    with pytest.raises(lib.TTError, match='float32'):
        lift_splat(*args(dep.half(), ctx))
    with pytest.raises(ValueError, match='frustum'):
        lift_splat(*args(dep[:, 1:], ctx))
    with pytest.raises(ValueError, match='frustum'):
        lift_splat(*args(dep, ctx, m.frustum[:, :, 1:]))


# ----------------------------------------------------------------------------------------- the float64 reference, pinned
@pytest.fixture(scope='module')
def small():
    """the plumbing config (4 cameras, 16 x 16 feature maps, 8 bins) with rig matrices, B = 2, C = 8."""
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.synthetic import rig_metas
    geo = K.lift_geometry(Config.fromfile(PLUMBING_CONFIG))
    B, N, Cc = 2, geo['N'], 8
    metas = [rig_metas(geo['final_dim'], geo['queue_len']) for _ in range(B)]
    s2e, intr, ida = K.sweep_mats(metas, N, 0)
    gen = torch.Generator().manual_seed(5)
    dl = K.depth_logits(gen, B * N, geo['fH'], geo['fW'], geo['D']).permute(0, 3, 1, 2).contiguous().double()
    ctx = torch.randn(B * N, Cc, geo['fH'], geo['fW'], generator=gen, dtype=torch.float64)
    G = torch.randn(B, Cc, geo['Y'], geo['X'], generator=gen, dtype=torch.float64)
    cells = R.ref_cells(s2e, intr, ida, K.kernel_mats(s2e, intr, ida), geo)
    return dict(geo=geo, B=B, N=N, C=Cc, s2e=s2e, intr=intr, ida=ida, dl=dl, ctx=ctx, G=G, cells=cells)


def test_reference_cells_and_gradients_equal_the_oracle_composition_under_autograd(small):
    """oracle.camera.LSS.get_geometry / geom_index in float64, softmax, the outer product, voxel_pooling_ref, .backward(G)."""
    from oracle.camera import LSS as OLSS
    from oracle.voxel_pool import voxel_pooling_ref
    s, geo = small, small['geo']
    B, N, Cc, D, fH, fW = s['B'], s['N'], s['C'], geo['D'], geo['fH'], geo['fW']
    ns = types.SimpleNamespace(frustum=geo['frustum'].double(), voxel_coord=geo['lss'].voxel_coord.double(),
                               voxel_size=geo['lss'].voxel_size.double())
    geom = OLSS.get_geometry(ns, s['s2e'].double(), s['intr'].double(), s['ida'].double())
    idx = OLSS.geom_index(ns, geom)                                         # (B, N, D, fH, fW, 3)
    dl, ctx = s['dl'].clone().requires_grad_(True), s['ctx'].clone().requires_grad_(True)
    lifted = dl.softmax(1).unsqueeze(1) * ctx.unsqueeze(2)
    lifted = lifted.reshape(B, N, Cc, D, fH, fW).permute(0, 1, 3, 4, 5, 2).contiguous()
    bev = voxel_pooling_ref(idx.contiguous(), lifted, geo['lss'].voxel_num)
    bev.backward(s['G'])
    # the composition's cells, pixel-major, as the kernel records them
    X, Y, Z = geo['X'], geo['Y'], geo['Z']
    i = idx.permute(0, 1, 3, 4, 2, 5).reshape(B * N * fH * fW, D, 3).long()
    ok = (i >= 0).all(-1) & (i[..., 0] < X) & (i[..., 1] < Y) & (i[..., 2] < Z)
    cells = torch.where(ok, i[..., 1] * X + i[..., 0], -1).numpy()
    R.check_bin_cell(cells, s['cells'], name='geom_index')
    assert s['cells']['in_bins'] > 0.05 * cells.size
    ref = R.ref_grads(s['dl'], s['ctx'], cells, s['G'])
    assert torch.allclose(ref['gl'], dl.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(ref['gc'], ctx.grad, rtol=1e-10, atol=1e-12)


def test_reference_gradients_equal_a_literal_loop():
    g = torch.Generator().manual_seed(11)
    B, N, D, fH, fW, Cc, X, Y = 2, 2, 5, 2, 3, 4, 3, 2
    dl = torch.randn(B * N, D, fH, fW, generator=g, dtype=torch.float64) * 2
    ctx = torch.randn(B * N, Cc, fH, fW, generator=g, dtype=torch.float64)
    G = torch.randn(B, Cc, Y, X, generator=g, dtype=torch.float64)
    cells = torch.randint(-1, X * Y, (B * N * fH * fW, D), generator=g).numpy()
    cells[3] = [2, 2, -1, 2, 5]                                              # a cell left and re-entered
    ref = R.ref_grads(dl, ctx, cells, G)
    gl, gc = torch.zeros_like(dl), torch.zeros_like(ctx)
    for bn in range(B * N):
        b = bn // N
        for h in range(fH):
            for w in range(fW):
                p = (bn * fH + h) * fW + w
                e = [np.exp(float(dl[bn, d, h, w])) for d in range(D)]
                pi = [v / sum(e) for v in e]
                gv = []
                for d in range(D):
                    c = int(cells[p, d])
                    gv.append(0.0 if c < 0 else sum(float(ctx[bn, k, h, w] * G[b, k, c // X, c % X]) for k in range(Cc)))
                    if c >= 0:
                        for k in range(Cc):
                            gc[bn, k, h, w] += pi[d] * float(G[b, k, c // X, c % X])
                S = sum(pi[d] * gv[d] for d in range(D))
                for d in range(D):
                    gl[bn, d, h, w] = pi[d] * (gv[d] - S)
    assert torch.allclose(ref['gl'], gl, rtol=1e-12, atol=1e-14) and torch.allclose(ref['gc'], gc, rtol=1e-12, atol=1e-14)


def _last_run_dropped(cells):
    c = cells.copy()
    for p in range(c.shape[0]):
        d = np.nonzero(c[p] >= 0)[0]
        if len(d):
            last, k = c[p, d[-1]], d[-1]
            while k >= 0 and c[p, k] == last:
                c[p, k] = -1
                k -= 1
    return c


def test_the_gradient_check_rejects_seeded_bugs(small):
    s = small
    cells = s['cells']['cell']
    dl, ctx, G = s['dl'].float(), s['ctx'].float(), s['G'].float()
    ref = R.ref_grads(dl, ctx, cells, G)
    gl, gc = ref['gl'].float(), ref['gc'].float()                            # a correct fp32 result
    assert all(r < 0.5 for r in R.check_grads(gl, gc, ref))
    B, Cc, Y, X = G.shape
    Gt = G.reshape(B, Cc * X * Y).reshape(B, X * Y, Cc).permute(0, 2, 1).reshape(B, Cc, Y, X)   # [C][cells] read as [cells][C]
    shifted = np.concatenate([np.full_like(cells[:, :1], -1), cells[:, :-1]], 1)
    outside = np.where(cells < 0, 0, cells)
    bugs = {
        'bins shifted by one run position': R.ref_grads(dl, ctx, shifted, G),
        'sum_j pi g dropped': dict(ref, gl=_pi_g(dl, ctx, cells, G)),
        'last run dropped': R.ref_grads(dl, ctx, _last_run_dropped(cells), G),
        'G read transposed': R.ref_grads(dl, ctx, cells, Gt),
        'neighbouring camera': {k: torch.roll(v, 1, 0) for k, v in ref.items()},
        'out-of-grid bin given a gradient': R.ref_grads(dl, ctx, outside, G),
    }
    for name, bad in bugs.items():
        for key in ('gl', 'gc'):
            if torch.equal(bad[key], ref[key]):
                continue
            got = dict(gl=gl, gc=gc)
            got[key] = bad[key].float()
            with pytest.raises(AssertionError):
                R.check_grads(got['gl'], got['gc'], ref, name=name)
            break
        else:
            raise AssertionError(f'seeded bug "{name}" changed nothing')


def _pi_g(dl, ctx, cells, G):
    """grad_logits without the softmax's sum_j pi g term: pi g."""
    pi = torch.softmax(dl.double(), 1)
    BN, D, fH, fW = dl.shape
    B, Cc = G.shape[:2]
    c = torch.as_tensor(cells).reshape(BN, fH, fW, D).permute(0, 3, 1, 2)
    g = torch.zeros_like(pi)
    for bn in range(BN):
        rows = G[bn // (BN // B)].double().reshape(Cc, -1)[:, c[bn].clamp(min=0).reshape(-1)].reshape(Cc, D, fH, fW)
        g[bn] = (ctx[bn].double()[:, None] * rows).sum(0) * (c[bn] >= 0)
    return pi * g
