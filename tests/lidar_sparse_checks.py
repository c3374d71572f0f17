"""Reference semantics and comparison helpers for the LiDAR sparse-encoder kernels: hard voxelisation + mean VFE and the
sparse-conv rulebooks (csrc/lidar.cu), and the sparse modes of the scaled-split fp16 convolution (csrc/gemm_conv_f16s.cu).

tests/test_lidar_sparse_gpu.py runs these checks on the CUDA kernels; tests/test_lidar_sparse_cpu.py runs them on the torch
emulation of the C ABI and shows that each one rejects a corrupted copy of a correct result.  The references are written from
the semantics (mmcv hard voxelisation, spconv SubMConv3d / SparseConv3d): numpy on the host, float64 wherever arithmetic happens.
The runners drive the product's own host code (LidarNet._rulebook, Engine.sparse_conv), so they work on either backend."""
import ctypes as C
import itertools
import types

import numpy as np
import torch

VOX_TOL = 1e-6           # voxel means, relative to the mean |p| of the averaged points
GLOBAL_TOL = 5e-6        # sparse convs: max |err| / max |ref| (DESIGN.md §2)
SPLIT = 2.0 ** -22       # hi + lo'/2048 carries an fp32 value to 2^-22 relative
ACC = 2.0 ** -23         # one fp32 accumulation step, counted as a full ulp (tensor-core adders truncate)
BM, BN = 128, 64         # output rows / columns of one work item of the f16s sparse modes
SENT = -1234.5           # fp32 sentinel of rows past the count
SENT_H = -77.0           # fp16 sentinel of split planes past the count
ONE_TAP = 0x200000       # debug bit: one tap per 64-half K slab (turns off the two-tap slabs of Cin = 32)


# ---------------------------------------------------------------------------------------------------------- common
def site_keys(coords, shape):
    """linear (b, z, y, x) key of each row of coords (n, 4) in a grid of `shape` (D, H, W)."""
    c = np.asarray(coords, np.int64).reshape(-1, 4)
    return ((c[:, 0] * shape[0] + c[:, 1]) * shape[1] + c[:, 2]) * shape[2] + c[:, 3]


def decode_keys(k, shape):
    D, H, W = shape
    return np.stack([k // (D * H * W), (k // (H * W)) % D, (k // W) % H, k % W], 1).astype(np.int64)


def split_round(x):
    """float64 value of the split planes (hi, lo') of an fp32 tensor: what a kernel reading the planes sees."""
    from thinktwice_b200.weights import f16s_split
    hi, lo = f16s_split(x.cpu())
    return hi.double() + lo.double() / 2048.0


def planes_value(planes, rows, cols):
    """float64 value hi + lo'/2048 of the first `rows` rows of a [2][cap * cols] split companion."""
    p = planes.detach().cpu().view(2, -1)[:, :rows * cols].double().view(2, rows, cols)
    return (p[0] + p[1] / 2048.0).numpy()


def os_items(count, cout):
    """work items of the output-stationary form: 128-row output tiles x 64-column tiles."""
    return -(-int(count) // BM) * -(-cout // BN)


def tap_items(pair_count, cout):
    """work items of the tap-major form: 128-row tiles of each tap's pair list x 64-column tiles."""
    return int(sum(-(-int(c) // BM) for c in np.asarray(pair_count).reshape(-1))) * -(-cout // BN)


# ---------------------------------------------------------------------------------------------------------- voxelisation
def point_cells(pts, lower, vsize):
    """(P, 3) integer (x, y, z) cell of each point: floor((p - lower) / vsize) in float32, as mmcv computes it."""
    p = np.asarray(pts, np.float32)[:, :3]
    return np.floor((p - np.asarray(lower, np.float32)) / np.asarray(vsize, np.float32)).astype(np.int64)


def ref_voxelize(points, lower, vsize, grid, zmax, max_points):
    """points (B, P, F) -> dict(coords (n, 4) [b, z, y, x] in ascending key order, feats (n, F) float64 mean of the FIRST
    `max_points` points of each voxel in input order, scale (n, F) mean |p| of the same points, members: per site the point
    ids that were averaged).  Points outside the grid or at z >= zmax are dropped."""
    pts = np.asarray(points, np.float32)
    B, P, F = pts.shape
    gx, gy, gz = grid
    cs, fs, ss, members = [], [], [], []
    for b in range(B):
        c = point_cells(pts[b], lower, vsize)
        ok = ((c >= 0) & (c < np.asarray(grid))).all(1) & (c[:, 2] < zmax)
        idx = np.nonzero(ok)[0]
        key = (c[idx, 2] * gy + c[idx, 1]) * gx + c[idx, 0]
        o = np.argsort(key, kind='stable')                     # grouped by voxel, input order kept inside a voxel
        k, ids = key[o], idx[o]
        uk, start, cnt = np.unique(k, return_index=True, return_counts=True)
        rank = np.arange(len(k)) - np.repeat(start, cnt)
        sel = rank < max_points
        grp = np.repeat(np.arange(len(uk)), cnt)[sel]
        v = pts[b][ids[sel]].astype(np.float64)
        n = np.minimum(cnt, max_points)[:, None].astype(np.float64)
        f = np.zeros((len(uk), F)); np.add.at(f, grp, v)
        s = np.zeros((len(uk), F)); np.add.at(s, grp, np.abs(v))
        cs.append(np.stack([np.full_like(uk, b), uk // (gx * gy), (uk // gx) % gy, uk % gx], 1))
        fs.append(f / np.maximum(n, 1))
        ss.append(s / np.maximum(n, 1))
        members += np.split(ids[sel], np.cumsum(np.minimum(cnt, max_points))[:-1]) if len(uk) else []
    return dict(coords=np.concatenate(cs).reshape(-1, 4), feats=np.concatenate(fs).reshape(-1, F),
                scale=np.concatenate(ss).reshape(-1, F), members=members)


def check_voxelize(got, ref, name='voxelize'):
    """site count, coordinates and order exact; features within VOX_TOL * mean|p| of the float64 mean.

    Bound: the kernel sums n <= 10 fp32 points in input order and divides by n.  Each addition rounds by at most 2^-24 of the
    running sum of magnitudes, the division by 2^-24 of the result, so |err| <= ((n - 1) + 1) * 2^-24 * mean|p| = n * 6e-8 * mean|p|,
    below 1e-6 * mean|p| for n <= 16.  Averaging any other point than the first max_points moves the mean by |p_a - p_b| / n."""
    n, m = int(got['count']), len(ref['coords'])
    assert n == m, f'{name}: {n} sites, expected {m}'
    c = np.asarray(got['coords'])[:n].astype(np.int64)
    bad = np.nonzero((c != ref['coords']).any(1))[0]
    assert not len(bad), f'{name}: site {bad[0]} is {c[bad[0]].tolist()}, expected {ref["coords"][bad[0]].tolist()}'
    err = np.abs(np.asarray(got['feats'])[:n].astype(np.float64) - ref['feats'])
    lim = VOX_TOL * ref['scale']
    if err.size and not (err <= lim).all():
        r, f = np.unravel_index(np.argmax(err - lim), err.shape)
        raise AssertionError(f'{name}: site {r} feature {f}: |err| {err[r, f]:.3e} > {lim[r, f]:.3e}')
    return float(err.max()) if err.size else 0.0


# ---------------------------------------------------------------------------------------------------------- rulebooks
def out_shape_of(in_shape, k, s, p, subm):
    return tuple(in_shape) if subm else tuple((in_shape[i] + 2 * p[i] - k[i]) // s[i] + 1 for i in range(3))


def ref_rulebook(in_coords, in_shape, k, s, p, subm):
    """spconv rulebook of a conv over the sites in_coords (n, 4).  SubMConv3d: the output sites are the input sites, in their
    order.  SparseConv3d: every output cell some input reaches, in ascending (b, z, y, x) order; along an axis, input cell i
    feeds output cell o iff o * s - p <= i <= o * s - p + k - 1.  nbr[o][tap] = input row at o * s - p + tap, or -1."""
    c = np.asarray(in_coords, np.int64).reshape(-1, 4)
    k, s, p = (np.asarray(v, np.int64) for v in (k, s, p))
    oshape = out_shape_of(in_shape, k, s, p, subm)
    if subm:
        oc = c.copy()
    else:
        lo = np.maximum(-((k - 1 - p - c[:, 1:]) // s), 0)        # ceil((i + p - k + 1) / s)
        hi = np.minimum((c[:, 1:] + p) // s, np.asarray(oshape) - 1)
        cand = [np.zeros((0, 4), np.int64)]
        for dd in itertools.product(*(range(-(-int(k[a]) // int(s[a]))) for a in range(3))):
            o = lo + np.asarray(dd)
            ok = (o <= hi).all(1)
            cand.append(np.concatenate([c[ok, :1], o[ok]], 1))
        oc = decode_keys(np.unique(site_keys(np.concatenate(cand), oshape)), oshape)
    kin = site_keys(c, in_shape)
    order = np.argsort(kin)
    sk = kin[order]
    kvol = int(np.prod(k))
    nbr = np.full((len(oc), kvol), -1, np.int64)
    for t, tap in enumerate(itertools.product(*(range(int(v)) for v in k))):
        src = oc[:, 1:] * s - p + np.asarray(tap)
        ok = ((src >= 0) & (src < np.asarray(in_shape))).all(1)
        q = site_keys(np.concatenate([oc[:, :1], src], 1), in_shape)
        pos = np.minimum(np.searchsorted(sk, q), max(len(sk) - 1, 0))
        hit = ok & (sk[pos] == q) if len(sk) else ok & False
        nbr[hit, t] = order[pos[hit]]
    return dict(coords=oc, nbr=nbr, shape=oshape, kvol=kvol)


def rulebook_host(rb):
    """host copy of a rulebook dict from LidarNet._rulebook."""
    h = lambda t: None if t is None else t.detach().cpu().numpy().astype(np.int64)
    return dict(coords=h(rb['coords']), count=int(rb['count'].item()), nbr=h(rb['nbr']), pairs_in=h(rb['pairs_in']),
                pairs_out=h(rb['pairs_out']), pair_count=h(rb['pair_count']))


def check_rulebook(got, ref, name='rulebook'):
    """output sites exact and in order; nbr entry by entry; each tap's pair list equal to the reference as a set (its order
    within a tap comes from atomics).  got: rulebook_host()."""
    n, m = got['count'], len(ref['coords'])
    assert n == m, f'{name}: {n} output sites, expected {m}'
    c = got['coords'][:n]
    bad = np.nonzero((c != ref['coords']).any(1))[0]
    assert not len(bad), f'{name}: output site {bad[0]} is {c[bad[0]].tolist()}, expected {ref["coords"][bad[0]].tolist()}'
    if got['nbr'] is not None:
        bad = np.argwhere(got['nbr'][:n] != ref['nbr'])
        if len(bad):
            r, t = bad[0]
            raise AssertionError(f'{name}: nbr[{r}][{t}] = {got["nbr"][r, t]}, expected {ref["nbr"][r, t]}')
    if got['pair_count'] is not None:
        for t in range(ref['kvol']):
            rows = np.nonzero(ref['nbr'][:, t] >= 0)[0]                # ascending, unique
            cnt = int(got['pair_count'][t])
            assert cnt == len(rows), f'{name}: tap {t} has {cnt} pairs, expected {len(rows)}'
            po, pi = got['pairs_out'][t, :cnt], got['pairs_in'][t, :cnt]
            o = np.argsort(po, kind='stable')
            assert (po[o] == rows).all(), f'{name}: tap {t}: output rows of the pairs differ from the reference set'
            assert (pi[o] == ref['nbr'][rows, t]).all(), f'{name}: tap {t}: an input row of a pair differs from the reference'


# ---------------------------------------------------------------------------------------------------------- sparse convs
def ref_sparse_conv(x, in_coords, in_shape, B, w, k, s, p, subm, ref_rb):
    """float64 oracle (oracle.lidar.SparseConvBase) of the conv without bias / residual / activation.
    x (n_in, Cin) float64 (the split-rounded rows the kernel reads), w (Cout, kvol, Cin).  Returns dict(acc = conv(x),
    mag = conv(|x|) with |w|, K = Cin * taps with an input, per output row)."""
    from oracle.lidar import SparseConvBase, SparseTensor
    Cout, kvol, Cin = w.shape
    conv = SparseConvBase(Cin, Cout, k, stride=s, padding=p, subm=subm).double()
    xc = torch.as_tensor(np.asarray(in_coords, np.int64))
    x = torch.as_tensor(x, dtype=torch.float64)
    w = torch.as_tensor(w, dtype=torch.float64).reshape(Cout, *k, Cin)
    with torch.no_grad():
        conv.weight.copy_(w)
        y = conv(SparseTensor(x, xc, in_shape, B))
        conv.weight.copy_(w.abs())
        mag = conv(SparseTensor(x.abs(), xc, in_shape, B)).feats
    assert np.array_equal(y.coords.numpy(), ref_rb['coords']), 'oracle and rulebook reference disagree on the output sites'
    return dict(acc=y.feats.numpy(), mag=mag.numpy(), K=Cin * (ref_rb['nbr'] >= 0).sum(1))


def expected(ref, bias=None, res=None, act=0, planes=False):
    """reference output act(acc + bias + res) and its per-element error bound.

    Each product x * w is formed from the split operands as xh*wh + (xh*wl' + xl'*wh) / 2048, exactly in fp32 (11-bit
    significands).  The reference reads the same split-rounded x, so the operand errors are the weight split, |w - wh - wl'/2048|
    <= 2^-22 |w|, and the dropped lo*lo term, |xl'*wl'| / 2048^2 <= 2^-11 |x| * 2^-11 |w| = 2^-22 |x||w|.  Summing the row's
    K = Cin * (taps with an input) terms in fp32 costs at most K * 2^-23 * sum |x||w| (one ulp per step, whatever the order,
    chunking or folding).  Adding bias and residual in fp32 rounds twice: 2^-23 (|acc| + |bias| + |res|).  Reading the result
    back from its split planes adds 2^-22 |y|.  ReLU is 1-Lipschitz.  So, with mag = sum |x||w| per output element,
        |got - ref| <= (2 * 2^-22 + K * 2^-23) * mag + 2^-23 (|acc| + |bias| + |res|) [+ 2^-22 |y|].
    A wrong input row, a dropped tap or a missing residual changes an element by about sqrt(Cin) |x||w|, far above this bound."""
    acc = ref['acc']
    b = np.zeros(acc.shape[1]) if bias is None else np.asarray(bias, np.float64)
    r = np.zeros_like(acc) if res is None else np.asarray(res, np.float64)
    pre = acc + b + r
    y = np.maximum(pre, 0) if act else pre
    bound = (2 * SPLIT + ref['K'][:, None] * ACC) * ref['mag'] + ACC * (np.abs(acc) + np.abs(b) + np.abs(r))
    if planes:
        bound = bound + SPLIT * np.abs(y)
    return y, bound


def check_conv(got, y, bound, name='conv', scale=1.0):
    """global error <= GLOBAL_TOL of max |ref| and every element within `scale` x its bound.  Returns (global rel. error,
    largest err / bound)."""
    got = np.asarray(got, np.float64)
    assert got.shape == y.shape, f'{name}: shape {got.shape}, expected {y.shape}'
    if not y.size:
        return 0.0, 0.0
    err = np.abs(got - y)
    ratio = err / np.maximum(scale * bound, 1e-300)
    if not (ratio <= 1).all():                                   # first: it names the row
        r, c = np.unravel_index(np.argmax(ratio), ratio.shape)
        raise AssertionError(f'{name}: row {r} col {c}: |err| {err[r, c]:.3e} > bound {scale * bound[r, c]:.3e}')
    g = float(err.max() / max(np.abs(y).max(), 1e-30))
    assert g <= GLOBAL_TOL, f'{name}: max error {g:.2e} of max |ref| > {GLOBAL_TOL:.0e}'
    return g, float(ratio.max())


def check_untouched(buf, count, cols, name='rows'):
    """rows from `count` up to the capacity still hold the sentinel: buf (cap, cols) fp32 or a [2][cap * cols] split companion."""
    t = buf.detach().cpu()
    if t.dtype == torch.float16:
        bad = (t.view(2, -1, cols)[:, count:] != SENT_H).any(0).any(1)
    else:
        bad = (t.view(-1, cols)[count:] != SENT).any(1)
    if bad.any():
        raise AssertionError(f'{name}: row {count + int(bad.nonzero()[0, 0])} past the count {count} was written')


def sentinel_rows(cap, cols, dev):
    return torch.full((cap, cols), SENT, device=dev)


def sentinel_planes(cap, cols, dev):
    return torch.full((2, cap * cols), SENT_H, dtype=torch.float16, device=dev)


# ---------------------------------------------------------------------------------------------------------- runners
def voxel_layer(cfg):
    """voxelisation parameters of the LiDAR encoder of a model config (lower, vsize, grid (x, y, z), zmax, max_points,
    max_voxels) and its sparse shape (D, H, W)."""
    le = cfg.model['lidar_encoder']
    v = le['pts_voxel_layer']
    shape = tuple(le['pts_middle_encoder']['sparse_shape'])
    vs, r = np.asarray(v['voxel_size'], np.float32), np.asarray(v['point_cloud_range'], np.float32)
    mv = v['max_voxels']
    return dict(lower=list(r[:3]), vsize=list(vs), grid=[int(g) for g in np.round((r[3:] - r[:3]) / vs)], zmax=shape[0],
                max_points=v['max_num_points'], max_voxels=int(mv[1] if isinstance(mv, (list, tuple)) else mv)), shape


def run_voxelize(points, vl, into=None):
    """tt_voxelize_mean on points (B, P, F) into fresh buffers (the rows past the count hold sentinels), or into the buffers
    of an earlier result `into`."""
    from thinktwice_b200 import lib
    B, P, F = points.shape
    dev = points.device
    d = lib.VoxelizeDesc()
    d.B, d.P, d.F = B, P, F
    d.lower, d.vsize, d.grid = lib.f3(vl['lower']), lib.f3(vl['vsize']), lib.i3(vl['grid'])
    d.zmax, d.max_points, d.max_voxels, d.cap = vl['zmax'], vl['max_points'], vl['max_voxels'], B * P
    ws = torch.empty(lib.load().tt_voxelize_workspace_bytes(C.byref(d)), dtype=torch.uint8, device=dev)
    if into is not None:
        feats, coords, count = into['feats'], into['coords'], into['count']
    else:
        feats = sentinel_rows(B * P, F, dev)
        coords = torch.full((B * P, 4), -9, dtype=torch.int32, device=dev)
        count = torch.full((1,), -1, dtype=torch.int32, device=dev)
    pts = points.contiguous()
    lib.call('tt_voxelize_mean', C.byref(d), lib._p(pts), lib._p(feats), lib._p(coords), lib._p(count), lib._p(ws))
    return dict(feats=feats, coords=coords, count=count, cap=B * P)


def rulebook(eng, tag, B, coords, count, cap, shape, k, s, p, subm, form):
    """the product's rulebook (LidarNet._rulebook) in buffers of `eng` named after `tag`."""
    from thinktwice_b200.lidarnet import LidarNet
    return LidarNet._rulebook(types.SimpleNamespace(eng=eng), tag, B, coords, count, cap, tuple(shape), tuple(k), tuple(s), tuple(p),
                              subm, form)


def pack(w, bias=None):
    """PackedConv of a sparse conv weight w (Cout, kvol, Cin) on the device of w, with its split planes."""
    from thinktwice_b200.engine import PackedConv
    from thinktwice_b200.weights import f16s_split
    Cout, kvol, Cin = w.shape
    w_h = torch.stack(f16s_split(w.cpu())).contiguous().to(w.device)
    return PackedConv(w.permute(1, 2, 0).reshape(kvol * Cin, Cout).contiguous(), bias, Cin, Cout, w_h=w_h)


def set_debug(flags):
    from thinktwice_b200 import lib
    lib.check(lib.load().tt_debug_set(flags), 'tt_debug_set')


def run_conv(eng, rb, x_s, pw, act=0, res=None, res_s=None, f32_out=True, flags=0, into=None):
    """one sparse conv through Engine.sparse_conv into sentinel-filled outputs (or into the (rows, planes) pair `into`): the
    output-stationary form when rb carries `nbr`, else the tap-major form.  x_s: split planes of the input rows.
    Returns (fp32 rows or None, split planes)."""
    dev = x_s.device
    if into is not None:
        out, out_s = into
    else:
        out = sentinel_rows(rb['cap'], pw.Cout, dev) if f32_out else None
        out_s = sentinel_planes(rb['cap'], pw.Cout, dev)
    set_debug(flags)
    try:
        eng.sparse_conv(None if rb['nbr'] is not None else torch.empty(0, device=dev), pw, rb, out, act=act, res=res, name='t',
                        feats_s=x_s, out_s=out_s, res_s=res_s)
    finally:
        set_debug(0)
    return out, out_s
