"""Reference semantics and comparison helpers for the camera-branch and Look-module kernels: the fused lift-splat
(csrc/lift_splat.cu), Look projection + ordered compaction and query rebatching (csrc/look.cu), the deformable-conv column
builder (csrc/dcn.cu) and the GRU input plane (csrc/elementwise.cu).

tests/test_camera_look_gpu.py runs these checks on the CUDA kernels at the thinktwice.py shapes; tests/test_camera_look_cpu.py
runs them on the torch emulation of the C ABI and shows that each one rejects a corrupted copy of a correct result.  The
references are written from the reference semantics (lss.py get_geometry / geom_index / voxel pooling, thinktwice_decoder.py
cam_ref_points_query, mmcv deformable im2col) in float64, never from a kernel's intermediate values.  The runners call the C ABI
through thinktwice_b200.lib, so they work on either backend."""
import ctypes as C
import types

import numpy as np
import torch

U = 2.0 ** -24            # unit roundoff of fp32 (round to nearest)
SENT = -1234.5            # fp32 sentinel of columns / rows a kernel must not write
EPS = float(np.float32(1e-5))   # depth clamp and validity threshold of cam_ref_points_query, as the fp32 reference holds it


def gamma(n):
    """bound on the relative error of an n-rounding fp32 dot product or sum, relative to the sum of |terms|."""
    return n * U / (1 - n * U)


def same_bits(a, b):
    """element-wise bitwise equality of two fp32 arrays (NaN sentinels compare equal to themselves)."""
    return np.asarray(a, np.float32).view(np.int32) == np.asarray(b, np.float32).view(np.int32)


def check_sentinel(after, before, keep, what):
    """every element of `after` where `keep` is True is bitwise what it was before the call.  after, before: host arrays of
    the whole buffer; keep: boolean array broadcastable to them.  `what(index)` names the first changed element."""
    bad = keep & ~same_bits(after, before)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f'{what(i)}: outside the written range, changed from {before[i]!r} to {after[i]!r}')


# ---------------------------------------------------------------------------------------------------------- lift-splat
def lift_geometry(cfg, final_dim=None):
    """camera-branch shapes and voxel grid of a model config, through the product's LSS (no weights are built); final_dim
    overrides the image size (smaller feature maps for the CPU checks)."""
    from thinktwice_b200.lss import LSS
    kw = {k: v for k, v in cfg.model['img_encoder'].items() if k != 'type'}
    if final_dim is not None:
        kw['final_dim'] = tuple(final_dim)
    m = LSS(**kw)
    m.h_vsize = m.voxel_size.float()
    lower = (m.voxel_coord.float() - m.h_vsize / 2.0)                # lss.py:630 in fp32, as LSS.prepare hands it to the kernel
    return dict(lss=m, D=m.depth_channels, fH=m.fH, fW=m.fW, C=m.output_channels, N=len(cfg.model['decoder']['config']['camera_names']),
                X=int(m.voxel_num[0]), Y=int(m.voxel_num[1]), Z=int(m.voxel_num[2]), lower=lower.numpy(), size=m.h_vsize.numpy(),
                final_dim=tuple(m.final_dim), queue_len=m.queue_len, fu=m.frustum_u, fv=m.frustum_v, fd=m.frustum_d,
                frustum=m.make_frustum(), mid=m.mid)


def sweep_mats(metas, N, s):
    """(sensor2ego, intrin, ida) of sweep s, each (B, N, 4, 4) fp32, as LSS.stage picks them (key frame -1, history sweep -s)."""
    from thinktwice_b200.lss import LSS
    m = LSS.build_mats(metas, N)
    idx = -1 if s == 0 else -s
    return m['sensor2ego_mats'][:, idx], m['intrin_mats'][:, idx], m['ida_mats'][:, idx]


def kernel_mats(s2e, intrin, ida):
    """[BN][32] fp32 matrices of tt_lift_splat (ida^-1 | sensor2ego @ intrin^-1), computed as LSS.stage computes them."""
    B, N = s2e.shape[:2]
    return torch.stack([torch.inverse(ida), s2e.matmul(torch.inverse(intrin))], 2).reshape(B * N, 32).contiguous()


def ref_lift(depth, ctx, s2e, intrin, ida, mats32, geo):
    """float64 lift-splat of frames (B, N): depth logits (BN, fH, fW, D) and context (BN, fH, fW, C) host fp32 arrays,
    s2e / intrin / ida (B, N, 4, 4) fp32 camera matrices, mats32 the [BN][32] matrices the kernel is given (used for the
    bound only).  Returns dict(val, bound (B, cells, C), W (frame*cell, pixel) fp64 weights, reached (B, cells), in_bins,
    amb_bins).

    Geometry: oracle.camera.LSS.get_geometry in float64 on the same matrices, cell = trunc((g - lower) / size) as geom_index
    (so t in (-1, 0) lands in cell 0).  Weights: fp64 softmax over D.  The bins of a pixel that share a cell are summed into
    one entry of a sparse (frame*cell, pixel) matrix W, and the BEV is W @ context, never the (pixels, D, C) tensor.

    Bound of one output element (frame, cell, c), two terms:
    (1) rounding, u = 2^-24.  A weight is expf(l - max) * (1 / sum): the argument rounds once (relative |a| u on the exp,
        a = max - l), CUDA's expf is within 2 ulp (4u), the sum of D positive terms within (D - 1)u plus the terms' own
        errors (their softmax-weighted |a| is at most log D < 5), 1 / sum and the product u each: (|a| + D + 14) u.  The run sum
        of at most D weights adds (D - 1) u, and the SpMM chains ceil(n / 8) fmaf per warp (n entries in the cell) and reduces
        8 warps with 7 adds.  So |err| <= u * sum over the cell's bins of w |ctx| (|a| + 2D + 22 + ceil(n / 8)).  Weights
        below fp32's normal range (2^-126) may flush to 0 in expf: their whole w |ctx| is added.
    (2) ambiguous mass.  The kernel evaluates the geometry in fp32.  Per bin and axis, an upper bound on the error of the
        normalised coordinate t = (g - lower) / size is carried through the kernel's operations: q = Mi (u, v, d, 1) as
        4-term fp32 dot products (gamma_4 |Mi| |x|) plus the rounding of the fp32 inverse Mi itself (|Mi32 - Mi64| |x|);
        p = (q0 q2, q1 q2, q2, q3), whose products add the first-order error terms and one rounding; g = Mc p as 4-term
        dot products plus |Mc32 - Mc64| |p|; then the subtraction and the division, 2u |t|.  At the full config the
        magnitudes are |p| ~ 6e4 (pixel x depth) and |Mc| |p| ~ 320 m, so the bound is about 1e-4 of a cell.  Where t +- that
        bound truncates to two different cells on some axis, the bin's w |ctx| is added to the bound of every cell it could
        fall in.  Truncation is constant across t = 0, so only t near -1 and near k >= 1 is ambiguous.  The checks require
        ambiguous bins to be under 0.1 % of the in-grid bins, so the term keeps its teeth."""
    from oracle.camera import LSS as OLSS
    import scipy.sparse as sp
    BN, fH, fW, D = depth.shape
    B, N = s2e.shape[:2]
    Cc = ctx.shape[-1]
    X, Y, Z = geo['X'], geo['Y'], geo['Z']
    cells = X * Y
    npix = fH * fW
    lower, size = geo['lower'].astype(np.float64), geo['size'].astype(np.float64)
    hi_ = np.array([X, Y, Z])
    lg = depth.astype(np.float64).reshape(BN * npix, D)
    a = lg.max(1, keepdims=True) - lg
    e = np.exp(-a)
    w = e / e.sum(1, keepdims=True)                               # (pixels, D)
    x = geo['frustum'].double().numpy()                           # (D, fH, fW, 4): the kernel's u, v, d floats
    ns = types.SimpleNamespace(frustum=geo['frustum'].double())
    m32 = mats32.detach().cpu().double().numpy().reshape(B, N, 2, 4, 4)
    ent = dict(W=([], [], []), Wa=([], [], []), S=([], [], []))
    in_bins = amb_bins = 0
    g4 = gamma(4)
    for b in range(B):
        g = OLSS.get_geometry(ns, s2e[b:b + 1].double(), intrin[b:b + 1].double(), ida[b:b + 1].double())[0].numpy()
        Mi = torch.inverse(ida[b].double()).numpy()                                   # (N, 4, 4)
        Mc = s2e[b].double().matmul(torch.inverse(intrin[b].double())).numpy()
        dMi, dMc = np.abs(m32[b, :, 0] - Mi), np.abs(m32[b, :, 1] - Mc)
        ax = np.abs(x)
        A = np.einsum('nij,dhwj->ndhwi', np.abs(Mi), ax)
        eq = g4 * A + np.einsum('nij,dhwj->ndhwi', dMi, ax)
        P = np.stack([A[..., 0] * A[..., 2], A[..., 1] * A[..., 2], A[..., 2], A[..., 3]], -1)
        ep = np.stack([A[..., 0] * eq[..., 2] + A[..., 2] * eq[..., 0] + eq[..., 0] * eq[..., 2] + U * P[..., 0],
                       A[..., 1] * eq[..., 2] + A[..., 2] * eq[..., 1] + eq[..., 1] * eq[..., 2] + U * P[..., 1],
                       eq[..., 2], eq[..., 3]], -1)
        aMc = np.abs(Mc[:, :3])
        ee = (g4 * np.einsum('nij,ndhwj->ndhwi', aMc, P) + np.einsum('nij,ndhwj->ndhwi', aMc, ep)
              + np.einsum('nij,ndhwj->ndhwi', dMc[:, :3], P))
        t = (g - lower) / size
        et = ee / size + 2 * U * np.abs(t) + 1e-12
        # pixel-major (N, fH, fW, D, 3), as the kernel walks a pixel's ray
        t, et = (v.transpose(0, 2, 3, 1, 4).reshape(N * npix, D, 3) for v in (t, et))
        idx, lo, hi = np.trunc(t).astype(np.int64), np.trunc(t - et).astype(np.int64), np.trunc(t + et).astype(np.int64)
        inside = ((idx >= 0) & (idx < hi_)).all(-1)
        pix = np.broadcast_to((b * N * npix + np.arange(N * npix))[:, None], inside.shape)
        wb, ab = w[b * N * npix:(b + 1) * N * npix], a[b * N * npix:(b + 1) * N * npix]
        row = b * cells + idx[..., 1] * X + idx[..., 0]
        for key, data in (('W', wb), ('Wa', wb * ab)):
            ent[key][0].append(row[inside]); ent[key][1].append(pix[inside]); ent[key][2].append(data[inside])
        tiny = inside & (wb < 2.0 ** -126)
        ent['S'][0].append(row[tiny]); ent['S'][1].append(pix[tiny]); ent['S'][2].append(wb[tiny])
        amb = (lo != hi).any(-1)
        any_in = np.zeros_like(amb)
        for k in range(8):                                        # every cell an ambiguous bin could fall in
            bit = np.array([(k >> i) & 1 for i in range(3)], bool)
            sel = amb & ((lo != hi) | ~bit).all(-1)
            cand = np.where(bit, hi, lo)
            ok = sel & ((cand >= 0) & (cand < hi_)).all(-1)
            any_in |= ok
            r = b * cells + cand[..., 1] * X + cand[..., 0]
            ent['S'][0].append(r[ok]); ent['S'][1].append(pix[ok]); ent['S'][2].append(wb[ok])
        in_bins += int(inside.sum())
        amb_bins += int(any_in.sum())
    shape = (B * cells, BN * npix)
    mat = {k: sp.coo_matrix((np.concatenate(v[2]), (np.concatenate(v[0]), np.concatenate(v[1]))), shape=shape).tocsr()
           for k, v in ent.items()}
    c64 = ctx.astype(np.float64).reshape(BN * npix, Cc)
    ac = np.abs(c64)
    n = mat['W'].getnnz(1) + mat['S'].getnnz(1)
    coef = 2 * D + 22 + np.ceil(n / 8)
    val = mat['W'] @ c64
    bound = U * (mat['Wa'] @ ac + coef[:, None] * (mat['W'] @ ac)) + mat['S'] @ ac
    return dict(val=val.reshape(B, cells, Cc), bound=bound.reshape(B, cells, Cc), W=mat['W'], reached=(n > 0).reshape(B, cells),
                in_bins=in_bins, amb_bins=amb_bins, bins=BN * npix * D)


def check_lift(after, before, ref, geo, coff, anti=False, name='lift_splat'):
    """after / before: host fp32 copies (B, Y, X, ld) of the whole BEV buffer after and before the call.  The C columns at
    `coff` must be within the bound of the float64 reference (exactly 0 where no ray reaches), every other column untouched.
    anti: the kernel stored the rot90(flip) layout (cell (y, x) at [X-1-x][Y-1-y]).  Returns the largest |err| / bound."""
    B, Y, X, ld = after.shape
    Cc = ref['val'].shape[-1]
    amb, ins = ref['amb_bins'], ref['in_bins']
    assert amb <= 1e-3 * ins, f'{name}: {amb} ambiguous bins of {ins} in the grid: the bound would lose its teeth'
    got = after[..., coff:coff + Cc].astype(np.float64)
    if anti:
        got = got.transpose(0, 2, 1, 3)[:, ::-1, ::-1]
    got = got.reshape(B, Y * X, Cc)
    cell = lambda i: f'{name}: frame {i[0]} cell (y {i[1] // X}, x {i[1] % X}) channel {i[2]}'
    nan = np.isnan(got)
    if nan.any():
        raise AssertionError(f'{cell(np.argwhere(nan)[0])}: not written (still the sentinel)')
    err = np.abs(got - ref['val'])
    over = err > ref['bound']
    if over.any():
        i = tuple(np.argwhere(over)[0])
        raise AssertionError(f'{cell(i)}: |err| {err[i]:.3e} > bound {ref["bound"][i]:.3e} (ref {ref["val"][i]:.4e})')
    keep = np.ones(ld, bool)
    keep[coff:coff + Cc] = False
    check_sentinel(after, before, keep, lambda i: f'{name}: frame {i[0]} row {i[1]} col {i[2]} column {i[3]}')
    pos = ref['bound'] > 0
    return float((err[pos] / ref['bound'][pos]).max()) if pos.any() else 0.0


def lift_desc(geo, B, C_, ld_d, d_coff, ld_c, c_coff, bev_ld, bev_coff, anti=0):
    from thinktwice_b200 import lib
    d = lib.LiftSplatDesc()
    d.B, d.N, d.D, d.fH, d.fW, d.C = B, geo['N'], geo['D'], geo['fH'], geo['fW'], C_
    d.ld_d, d.d_coff, d.ld_c, d.c_coff = ld_d, d_coff, ld_c, c_coff
    d.lower, d.size = lib.f3(geo['lower']), lib.f3(geo['size'])
    d.X, d.Y, d.Z = geo['X'], geo['Y'], geo['Z']
    d.bev_ld, d.bev_coff, d.anti_transpose = bev_ld, bev_coff, anti
    return d


def lift_workspace(d, dev):
    from thinktwice_b200 import lib
    return torch.empty(lib.load().tt_lift_splat_workspace_bytes(C.byref(d)), dtype=torch.uint8, device=dev)


def run_lift(d, geo, depth, ctx, mats, bev, bev_ptr_off=0, ws=None):
    """tt_lift_splat into `bev` (written at element offset bev_ptr_off, like LSS passes a concat slice)."""
    from thinktwice_b200 import lib
    dev = bev.device
    ws = lift_workspace(d, dev) if ws is None else ws
    fu, fv, fd = geo['fu'].to(dev), geo['fv'].to(dev), geo['fd'].to(dev)
    lib.call('tt_lift_splat', C.byref(d), lib._p(depth), lib._p(ctx), lib._p(mats.to(dev)), lib._p(fu), lib._p(fv), lib._p(fd),
             lib._p(bev, bev_ptr_off), lib._p(ws))
    return ws


def depth_logits(gen, BN, fH, fW, D):
    """logits mixing flat (scale 0.5), medium (3) and sharp (20) softmaxes, plus one-hot pixels (one bin, the others at -200:
    exp underflows to 0 in fp32)."""
    x = torch.randn(BN, fH, fW, D, generator=gen)
    kind = torch.randint(0, 4, (BN, fH, fW, 1), generator=gen)
    x = x * torch.where(kind == 0, 0.5, torch.where(kind == 1, 3.0, 20.0))
    hot = torch.randint(0, D, (BN, fH, fW), generator=gen)
    oh = torch.full_like(x, -200.0).scatter_(-1, hot[..., None], 0.0)
    return torch.where(kind == 3, oh, x).contiguous()


# ---------------------------------------------------------------------------------------------------------- Look module
def look_desc(cfg, B):
    """the product's tt_look_desc (ThinkTwiceDecoder._look_meta) at the config's image size and FPN level sizes, and the
    level sizes.  The FPN levels are the ResNet-50 c2..c5 maps, strides 4..32; level 2 is the depth net's input."""
    from thinktwice_b200.thinktwice_decoder import ThinkTwiceDecoder
    dc = cfg.model['decoder']['config']
    H, W = dc['img_size']
    lv = [(H // s, W // s) for s in (4, 8, 16, 32)]
    ds = cfg.model['img_encoder']['downsample_factor']
    assert lv[2] == (H // ds, W // ds)
    stub = types.SimpleNamespace(config=dc, T=dc['pred_len'], eng=types.SimpleNamespace(static=lambda name: None))
    meta = ThinkTwiceDecoder._look_meta(stub, B, [types.SimpleNamespace(H=h, W=w) for h, w in lv])
    return meta['look_desc'], lv


def look_points(wp):
    """(B, Q, 3) fp32 look points of thinktwice_decoder.py:155-160: waypoints then the 4 static points, 15 z levels each."""
    B, T = wp.shape[:2]
    st = np.array([[5.0, 0.0], [0.0, -5.0], [0.0, 5.0], [-5.0, 0.0]], np.float32)
    look = np.concatenate([np.asarray(wp, np.float32), np.broadcast_to(st, (B, 4, 2))], 1)
    z = np.arange(-4, 11, dtype=np.float32)
    pts = np.concatenate([np.repeat(look[:, :, None], 15, 2), np.broadcast_to(z[None, None, :, None], (B, look.shape[1], 15, 1))], -1)
    return pts.reshape(B, -1, 3).astype(np.float32)


def ref_project(wp, l2i, ida, img_w, img_h):
    """float64 cam_ref_points_query (oracle/decoder.py:167-204) on fp32 inputs wp (B, T, 2), l2i / ida (B, N, 4, 4).
    Returns dict(xy (B, N, Q, 2), depth, valid (surely valid), maybe (possibly valid), dxy (B, N, Q, 2) fp32 error bound).

    Bound: c = l2i (x, y, z, 1) is a 4-term fp32 dot product (gamma_4 |l2i| |p|); dividing by dz = max(c2, eps) adds
    (err c0 + |c0 / dz| err dz) / dz + u |c0 / dz|; e = ida c' adds gamma_4 |ida| |c'| + |ida| err c'; the division by the image
    size one more u.  Doubled to cover the second-order terms.  A query whose x, y or depth lies within its bound of a
    threshold (0 or 1, eps) may go either way."""
    p = look_points(wp).astype(np.float64)
    B, Q = p.shape[:2]
    ph = np.concatenate([p, np.ones((B, Q, 1))], -1)
    L = np.asarray(l2i, np.float64)
    A = np.asarray(ida, np.float64)
    g4 = gamma(4)
    cam = np.einsum('bnij,bqj->bnqi', L, ph)
    ecam = g4 * np.einsum('bnij,bqj->bnqi', np.abs(L), np.abs(ph))
    dz = np.maximum(cam[..., 2], EPS)
    edz = ecam[..., 2]                                            # max(c2, eps) is 1-Lipschitz in c2
    xi, yi = cam[..., 0] / dz, cam[..., 1] / dz
    exi = (ecam[..., 0] + np.abs(xi) * edz) / dz + U * np.abs(xi)
    eyi = (ecam[..., 1] + np.abs(yi) * edz) / dz + U * np.abs(yi)
    c2 = np.stack([xi, yi, cam[..., 2], cam[..., 3]], -1)
    ec2 = np.stack([exi, eyi, ecam[..., 2], ecam[..., 3]], -1)
    e = np.einsum('bnij,bnqj->bnqi', A, c2)
    ee = g4 * np.einsum('bnij,bnqj->bnqi', np.abs(A), np.abs(c2)) + np.einsum('bnij,bnqj->bnqi', np.abs(A), ec2)
    x, y = e[..., 0] / img_w, e[..., 1] / img_h
    dx, dy, dd = 2 * (ee[..., 0] / img_w + U * np.abs(x)), 2 * (ee[..., 1] / img_h + U * np.abs(y)), 2 * ee[..., 2]
    depth = e[..., 2]
    valid = (depth - dd > EPS) & (x - dx > 0) & (x + dx < 1) & (y - dy > 0) & (y + dy < 1)
    maybe = (depth + dd > EPS) & (x + dx > 0) & (x - dx < 1) & (y + dy > 0) & (y - dy < 1)
    return dict(xy=np.stack([x, y], -1), depth=depth, valid=valid, maybe=maybe, dxy=np.stack([dx, dy], -1))


def check_project(got, ref, name='look_project'):
    """got: dict of host arrays ref_cam (B, N, Q, 2), order (B, N, Q), counts (B, N), max_len (scalar).  Per (frame, camera):
    the count lies between the surely-valid and the possibly-valid queries, order[:count] is strictly ascending, holds every
    surely-valid query and no surely-invalid one; max_len = max(counts); ref_cam within its bound for every query.  Returns
    the largest ref_cam |err| / bound."""
    B, N, Q = ref['valid'].shape
    counts, order = np.asarray(got['counts']).reshape(B, N), np.asarray(got['order']).reshape(B, N, Q)
    for b in range(B):
        for n in range(N):
            cnt, nv, nm = int(counts[b, n]), int(ref['valid'][b, n].sum()), int(ref['maybe'][b, n].sum())
            assert nv <= cnt <= nm, f'{name}: (b {b}, cam {n}): count {cnt}, expected {nv}' + (f'..{nm}' if nm > nv else '')
            o = order[b, n, :cnt].astype(np.int64)
            assert ((o >= 0) & (o < Q)).all(), f'{name}: (b {b}, cam {n}): order holds {o[(o < 0) | (o >= Q)][0]}, not a query id'
            miss = np.setdiff1d(np.nonzero(ref['valid'][b, n])[0], o)
            assert not len(miss), f'{name}: (b {b}, cam {n}, query {miss[0]}): valid but missing from order'
            extra = o[~ref['maybe'][b, n][o]]
            assert not len(extra), f'{name}: (b {b}, cam {n}, query {extra[0]}): invalid but in order'
            if cnt > 1 and not (np.diff(o) > 0).all():
                r = int(np.argmax(np.diff(o) <= 0))
                raise AssertionError(f'{name}: (b {b}, cam {n}): order not strictly ascending at rows {r}, {r + 1} ({o[r]}, {o[r + 1]})')
    ml = int(np.asarray(got['max_len']).reshape(-1)[0])
    assert ml == int(counts.max()), f'{name}: max_len {ml}, expected max(counts) = {int(counts.max())}'
    rc = np.asarray(got['ref_cam'], np.float64).reshape(B, N, Q, 2)
    err = np.abs(rc - ref['xy'])
    bad = ~(err <= ref['dxy'])
    if bad.any():
        b, n, q, k = np.argwhere(bad)[0]
        raise AssertionError(f'{name}: (b {b}, cam {n}, query {q}): ref_cam[{k}] {rc[b, n, q, k]:.9g}, expected {ref["xy"][b, n, q, k]:.9g} '
                             f'+- {ref["dxy"][b, n, q, k]:.2e}')
    return float((err / np.maximum(ref['dxy'], 1e-300)).max())


def run_project(d, wp, l2i, ida, out=None):
    """tt_look_project; outputs into fresh buffers (NaN / -7 filled) or into `out` from an earlier call."""
    from thinktwice_b200 import lib
    dev = wp.device
    B, N, Q = d.B, d.num_cams, d.num_query
    o = out or dict(ref_cam=torch.full((B, N, Q, 2), float('nan'), device=dev), order=torch.full((B, N, Q), -7, dtype=torch.int32, device=dev),
                    counts=torch.full((B, N), -7, dtype=torch.int32, device=dev), max_len=torch.full((1,), -7, dtype=torch.int32, device=dev))
    lib.call('tt_look_project', C.byref(d), lib._p(wp), lib._p(l2i), lib._p(ida), lib._p(o['ref_cam']), lib._p(o['order']),
             lib._p(o['counts']), lib._p(o['max_len']))
    return o


def host(o):
    return {k: v.detach().cpu().numpy() for k, v in o.items()}


def query_rows(d, wp, ctrl_sp, temb, semb, meas, flat):
    """(B, Q, q_dim) fp32 query of every look point (thinktwice_decoder.py:164-171): [softplus ctrl of its waypoint (0 for
    the static points) | xyz | temporal (waypoints) or static embedding | measurement feature | flattened BEV feature]."""
    B, T, Q = d.B, d.T, d.num_query
    wp, cs = np.asarray(wp, np.float32), np.asarray(ctrl_sp, np.float32)
    te, se = np.asarray(temb, np.float32), np.asarray(semb, np.float32)
    ctrl = np.concatenate([np.repeat(cs, 15, 1), np.zeros((B, 4 * 15, 4), np.float32)], 1)
    emb = np.broadcast_to(np.concatenate([np.repeat(te, 15, 0), np.repeat(se, 15, 0)], 0)[None], (B, Q, te.shape[1]))
    rep = lambda v: np.broadcast_to(np.asarray(v, np.float32)[:, None], (B, Q, v.shape[-1]))
    return np.concatenate([ctrl, look_points(wp), emb, rep(meas), rep(flat)], -1)


def ref_samples(levels, bn, xy):
    """float64 F.grid_sample(level, 2 xy - 1, bilinear, zeros, align_corners=False) of every level at the positions xy (R, 2)
    of images bn (R,), feature index c * L + l.  levels: list of (BN, H, W, C) fp32 tensors (any device).  Returns
    (val, mag, lim) (R, C * L) float64 tensors: mag = sum of |corners| used, lim = the bound of the kernel's fp32 sample.

    Bound: the kernel forms x = rx W - 0.5 in fp32, off by at most u (|rx W| + |x|) <= 2u (W + 1); the sample's slope in x is
    at most the sum of |corners|, the same for y.  The weights (1 - l) * (1 - l') round twice and the 4-term fp32 sum is within
    gamma_4: |err| <= u (2W + 2H + 12) * sum |corners|.  Sampling at the kernel's own rx means fp32 rounding of rx cannot switch
    a corner; a switch through the rounding of x moves a weight near 0 only, which the slope term covers."""
    dev = levels[0].device
    bn = torch.as_tensor(bn, dtype=torch.long, device=dev)
    xy = torch.as_tensor(np.asarray(xy, np.float64), device=dev)
    vals, mags, lims = [], [], []
    for f in levels:
        BN, H, W, Cc = f.shape
        x, y = xy[:, 0] * W - 0.5, xy[:, 1] * H - 0.5
        x0, y0 = torch.floor(x), torch.floor(y)
        lx, ly = x - x0, y - y0
        val = torch.zeros(len(bn), Cc, dtype=torch.float64, device=dev)
        mag = torch.zeros_like(val)
        for dy, dx, wgt in ((0, 0, (1 - ly) * (1 - lx)), (0, 1, (1 - ly) * lx), (1, 0, ly * (1 - lx)), (1, 1, ly * lx)):
            yy, xx = (y0 + dy).long(), (x0 + dx).long()
            ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            v = f[bn, yy.clamp(0, H - 1), xx.clamp(0, W - 1)].double() * ok[:, None]
            val += wgt[:, None] * v
            mag += v.abs()
        vals.append(val); mags.append(mag); lims.append(U * (2 * W + 2 * H + 12) * mag)
    st = lambda v: torch.stack(v, -1).reshape(len(bn), -1)
    return st(vals), st(mags), st(lims)


def check_rebatch(rows_after, rows_before, re_after, d, proj, qrows, levels, rows_ld, name='look_rebatch'):
    """rows_after / rows_before: the whole rows buffer (BN * cap, rows_ld) after / before the call (host fp32); re_after:
    ref_rebatch (BN * cap, 2); proj: host outputs of tt_look_project the rebatch read; qrows: query_rows().  For rows below
    the count the query part is bitwise the fp32 inputs and the sampled part within the bound of the float64 sample at the
    kernel's own ref_cam; rows at or past the count are exactly 0; ref_rebatch rows are ref_cam[order] bitwise (0 past the
    count); the tail columns past q_dim + levels * C keep their sentinels.  Returns the largest sample |err| / bound."""
    B, N, Q, cap = d.B, d.num_cams, d.num_query, d.max_len_cap
    width = d.q_dim + d.levels * d.C
    rows = rows_after.reshape(B * N, cap, rows_ld)
    re = re_after.reshape(B * N, cap, 2)
    counts, order, rc = proj['counts'].reshape(-1), proj['order'].reshape(B * N, Q), proj['ref_cam'].reshape(B * N, Q, 2)
    idx = [(bn, r, int(order[bn, r])) for bn in range(B * N) for r in range(int(counts[bn]))]
    row_of = lambda bn, r: f'{name}: (b {bn // N}, cam {bn % N}, row {r}' + (f' = query {order[bn, r]})' if r < counts[bn] else ')')
    # rows at or past the count: exact zeros, ref_rebatch too
    past = np.arange(cap)[None, :] >= counts[:, None]
    nz = past[..., None] & (rows[..., :width] != 0)
    if nz.any():
        bn, r, i = np.argwhere(nz)[0]
        raise AssertionError(f'{row_of(bn, r)}: past the count {counts[bn]} but column {i} is {rows[bn, r, i]!r}, expected 0')
    nz = past[..., None] & (re != 0)
    if nz.any():
        bn, r, _ = np.argwhere(nz)[0]
        raise AssertionError(f'{row_of(bn, r)}: ref_rebatch past the count is {re[bn, r].tolist()}, expected 0')
    ratio = 0.0
    if idx:
        bn, r, q = (np.array(v) for v in zip(*idx))
        want = rc[bn, q]
        bad = ~same_bits(re[bn, r], want)
        if bad.any():
            i = int(np.argwhere(bad)[0, 0])
            raise AssertionError(f'{row_of(bn[i], r[i])}: ref_rebatch {re[bn[i], r[i]].tolist()}, expected ref_cam {want[i].tolist()}')
        qw = qrows[bn // N, q]
        bad = ~same_bits(rows[bn, r, :d.q_dim], qw)
        if bad.any():
            i, c = np.argwhere(bad)[0]
            raise AssertionError(f'{row_of(bn[i], r[i])}: query column {c} is {rows[bn[i], r[i], c]!r}, expected {qw[i, c]!r}')
        val, _, lim = ref_samples(levels, bn, want)
        got = torch.as_tensor(np.ascontiguousarray(rows[bn, r, d.q_dim:width]), device=val.device).double()
        err = (got - val).abs()
        over = ~(err <= lim)
        if over.any():
            i, k = (int(v) for v in torch.nonzero(over)[0])
            raise AssertionError(f'{row_of(bn[i], r[i])}: sampled feature (c {k // d.levels}, level {k % d.levels}) is {float(got[i, k]):.7g}, '
                                 f'expected {float(val[i, k]):.7g} +- {float(lim[i, k]):.2e}')
        pos = lim > 0
        ratio = float((err[pos] / lim[pos]).max()) if pos.any() else 0.0
    keep = np.zeros(rows_ld, bool)
    keep[width:] = True
    check_sentinel(rows_after.reshape(-1, rows_ld), rows_before.reshape(-1, rows_ld), keep,
                   lambda i: f'{name}: row {i[0]} tail column {i[1]}')
    return ratio


def run_rebatch(d, wp, ctrl_sp, temb, semb, meas, flat, levels, proj, rows, rows_ld, ref_re):
    from thinktwice_b200 import lib
    for f in levels:
        lib._p(f)                                                 # (registers the maps with the emulated ABI; no-op on the GPU)
    ptrs = (C.c_void_p * 4)(*[f.data_ptr() for f in levels])
    lib.call('tt_look_rebatch', C.byref(d), lib._p(wp), lib._p(ctrl_sp), lib._p(temb), lib._p(semb), lib._p(meas), lib._p(flat),
             ptrs, lib._p(proj['ref_cam']), lib._p(proj['order']), lib._p(proj['counts']), lib._p(rows), rows_ld, lib._p(ref_re))


# ---------------------------------------------------------------------------------------------------------- DCN columns
def dcn_positions(off, H, W):
    """fp32 sampling positions (n, H, W, 9) of mmcv's deformable im2col (3x3, pad 1, stride 1, dilation 1, one offset
    group): h = fl32((ho - 1 + kh) + dh), w = fl32((wo - 1 + kw) + dw), offsets (dh, dw) per tap at channels 2 tap, 2 tap + 1.
    off: (n, H, W, >= 18) fp32 tensor.  The fp32 sum is the position the kernel computes."""
    dev = off.device
    k = torch.arange(9, device=dev)
    bh = (torch.arange(H, device=dev)[:, None] - 1 + k[None] // 3).float()       # (H, 9)
    bw = (torch.arange(W, device=dev)[:, None] - 1 + k[None] % 3).float()       # (W, 9)
    h = bh[None, :, None, :] + off[..., 0:18:2]
    w = bw[None, None, :, :] + off[..., 1:18:2]
    return h, w


def ref_dcn_image(x, h, w):
    """float64 deformable columns of one image: x (H, W, C) fp32, positions h, w (H, W, 9) fp32.  mmcv semantics: a sample
    is zero unless h > -1 && w > -1 && h < H && w < W; each of the 4 corners outside the map counts as zero.  Returns (val,
    lim) (H, W, 9, C): lim = 8u * sum |corners used| bounds the kernel's fp32 weights (1 - l)(1 - l') and 4-term sum (the
    positions are the same floats, so every border decision matches exactly)."""
    H, W, Cc = x.shape
    xf = x.reshape(H * W, Cc).double()
    h, w = h.double(), w.double()
    inside = (h > -1) & (w > -1) & (h < H) & (w < W)
    hl, wl = torch.floor(h), torch.floor(w)
    lh, lw = h - hl, w - wl
    val = torch.zeros(H, W, 9, Cc, dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(val)
    for dh, dw, wgt in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
        yy, xx = (hl + dh).long(), (wl + dw).long()
        ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
        v = xf[(yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).reshape(-1)].reshape(H, W, 9, Cc) * ok[..., None]
        val += wgt[..., None] * v
        mag += v.abs()
    return val, 8 * U * mag


def dcn_columns(col, n, N, H, W, C_, G):
    """image n of the kernel's columns [N*H*W][G][9][C/G] as (H, W, 9, C) (channel g * C/G + c)."""
    return col.view(N, H, W, G, 9, C_ // G)[n].permute(0, 1, 3, 2, 4).reshape(H, W, 9, C_)


def check_dcn(x, off, col, G, images, name='dcn_im2col'):
    """every column element of the listed images within the bound of the float64 reference (exactly 0 where mmcv gives 0).
    x (N, H, W, C), off (N, H, W, off_ld), col: the kernel's output, all tensors on one device.  Returns the largest
    |err| / bound."""
    N, H, W, Cc = x.shape
    ratio = 0.0
    for n in images:
        h, w = dcn_positions(off[n:n + 1], H, W)
        val, lim = ref_dcn_image(x[n], h[0], w[0])
        got = dcn_columns(col, n, N, H, W, Cc, G).double()
        err = (got - val).abs()
        over = ~(err <= lim)
        if over.any():
            ho, wo, k, c = (int(v) for v in torch.nonzero(over)[0])
            raise AssertionError(f'{name}: image {n} pixel (h {ho}, w {wo}) tap {k} channel {c}: {float(got[ho, wo, k, c]):.7g}, expected '
                                 f'{float(val[ho, wo, k, c]):.7g} +- {float(lim[ho, wo, k, c]):.2e} (position h {float(h[0, ho, wo, k]):.7g}, '
                                 f'w {float(w[0, ho, wo, k]):.7g})')
        pos = lim > 0
        if pos.any():
            ratio = max(ratio, float((err[pos] / lim[pos]).max()))
    return ratio


def run_dcn(x, off, off_ld, col, G):
    from thinktwice_b200 import lib
    N, H, W, Cc = x.shape
    lib.call('tt_dcn_im2col', lib._p(x), lib._p(off), off_ld, lib._p(col), N, H, W, Cc, G)


def craft_dcn_offsets(off, H, W, n, gen):
    """overwrite the offsets of image n with border cases, tap by tap in a cycle over the pixels: integer offsets, positions
    in (-1, 0) and in (H-1, H) / (W-1, W) on each axis, and positions exactly at -1 and at H / W (which must give 0)."""
    dev = off.device
    k = torch.arange(9, device=dev)
    bh = (torch.arange(H, device=dev)[:, None, None] - 1 + k // 3).float().expand(H, W, 9)
    bw = (torch.arange(W, device=dev)[None, :, None] - 1 + k % 3).float().expand(H, W, 9)
    u = torch.rand(H, W, 9, generator=gen).to(dev) * 0.98 + 0.01                     # strictly inside (0, 1)
    r = torch.randn(H, W, 9, generator=gen).to(dev) * 3
    cat = (torch.arange(H * W, device=dev).view(H, W, 1) + k) % 7
    band_lo, band_hi_h, band_hi_w = u - 1, (H - 1) + u, (W - 1) + u
    th = [torch.round(bh + r), band_lo, band_hi_h, bh + r, torch.full_like(u, -1.0), torch.full_like(u, float(H)), bh + r]
    tw = [torch.round(bw + r.flip(-1)), bw + r, band_lo, band_hi_w, bw + r, bw + r, torch.full_like(u, float(W))]
    th, tw = torch.stack(th, -1), torch.stack(tw, -1)
    pick = lambda t: torch.gather(t, -1, cat[..., None])[..., 0]
    off[n, ..., 0:18:2] = pick(th) - bh
    off[n, ..., 1:18:2] = pick(tw) - bw
    return cat


# ---------------------------------------------------------------------------------------------------------- GRU input plane
def check_gru(after, before, wp, ctrl_sp, t, col0, name='gru_input'):
    """after / before: host (B, HW, ld) buffers; columns col0..col0+5 of every pixel of frame b are exactly (wp[b, t],
    ctrl_sp[b, t]); every other column keeps its sentinel."""
    B, HW, ld = after.shape
    want = np.concatenate([np.asarray(wp)[:, t], np.asarray(ctrl_sp)[:, t]], 1)            # (B, 6)
    got = after[..., col0:col0 + 6]
    bad = ~same_bits(got, np.broadcast_to(want[:, None], got.shape))
    if bad.any():
        b, p, c = np.argwhere(bad)[0]
        raise AssertionError(f'{name}: frame {b} pixel {p} column {col0 + c} is {got[b, p, c]!r}, expected {want[b, c]!r}')
    keep = np.ones(ld, bool)
    keep[col0:col0 + 6] = False
    check_sentinel(after, before, keep, lambda i: f'{name}: frame {i[0]} pixel {i[1]} column {i[2]}')


def run_gru(wp, ctrl_sp, t, buf, col0):
    from thinktwice_b200 import lib
    B, H, W, ld = buf.shape
    T = wp.shape[1]
    lib.call('tt_gru_input', lib._p(wp), lib._p(ctrl_sp), t, T, lib._p(buf, col0), ld, B, H * W)
