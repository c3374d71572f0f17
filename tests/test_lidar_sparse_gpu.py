"""LiDAR sparse-encoder kernels at the full thinktwice.py shape against exact and float64 references: hard voxelisation + mean
VFE (tt_voxelize_mean), the rulebooks of every conv LidarNet issues (tt_sparse_rulebook, neighbour-table and pair-list forms) and
the sparse modes of the scaled-split fp16 convolution (tt_sparse_conv_os_f16s output-stationary, tt_sparse_conv_f16s
tap-major).  The clouds are thinktwice_b200.synthetic frames of 40000 points, frame 1 zero-padded from point 31000 on the way
mmcv's collate pads, plus crafted points at the voxelisation edges.  At that size the first strided level has more output tiles
than an H100 has SMs in both forms, so the persistent work loop and the cross-tile neighbour prefetch run (the log prints the
site counts and work items).  The last test runs the whole encoder of the calibrated model and compares it level by level with
the oracle's SparseEncoder in float64.  The checks are in tests/lidar_sparse_checks.py; tests/test_lidar_sparse_cpu.py shows
that each of them rejects a corrupted result.

Wall time on one H100 machine: about 2 minutes, nearly all of it float64 references on the CPU (about 1 minute for the
kernel-level tests, about 1 minute for the encoder chain, including building and calibrating the model pair)."""
import numpy as np
import pytest
import torch

import lidar_sparse_checks as L

pytestmark = pytest.mark.gpu
NUM_POINTS = 40000
PAD_FROM = 31000
SEED = 0


def craft(points, vl):
    """write the edge cases into frame 0 (in place) and return the ids of the 40-point voxel's points."""
    lower, vs = np.asarray(vl['lower'], np.float64), np.asarray(vl['vsize'], np.float64)
    P = points.shape[1]
    g = np.random.default_rng(5)
    # one voxel holding 40 points spread over the whole index range: the hash chain (atomicExch) meets them out of input order
    ids = np.linspace(300, P - 300, 40).astype(np.int64)
    cell = np.array([100, 200, 30])
    xyz = (lower + (cell + 0.25 + 0.5 * g.random((40, 3))) * vs).astype(np.float32)
    points[0, ids, :3] = torch.from_numpy(xyz)
    points[0, ids, 3] = torch.from_numpy((0.01 * np.arange(40) + 0.005).astype(np.float32))   # distinct: any other choice shows
    points[0, ids, 4] = 0.0
    f32 = np.float32
    below = [f32(lower[a] - 1e-6) if f32(lower[a] - 1e-6) != f32(lower[a]) else np.nextafter(f32(lower[a]), f32(-np.inf))
             for a in range(3)]                                  # 1e-6 under -19.2 is below half an fp32 ulp: take the next float
    upper = f32(lower[0] + vl['grid'][0] * vs[0])
    mid = (lower + np.array([50.5, 60.5, 20.5]) * vs).astype(np.float32)
    z40, z41 = f32(lower[2] + 40.5 * vs[2]), f32(lower[2] + 41.5 * vs[2])
    edge = np.array([[lower[0], mid[1], mid[2]],                 # x = lower: cell 0, kept
                     [upper, mid[1] + vs[1], mid[2]],            # x = upper: cell grid[0], dropped
                     [below[0], mid[1] + 2 * vs[1], mid[2]],     # just below lower on each axis: floor -> -1, dropped
                     [mid[0], below[1], mid[2]],
                     [mid[0] + vs[0], mid[1], below[2]],
                     [mid[0] + 2 * vs[0], mid[1], z40],          # z cell 40: kept
                     [mid[0] + 3 * vs[0], mid[1], z41]], np.float32)   # z cell 41 >= sparse_shape[0]: dropped
    eids = np.arange(len(edge)) * 11 + 7
    points[0, eids, :3] = torch.from_numpy(edge)
    cells = L.point_cells(edge, vl['lower'], vl['vsize'])
    assert cells[0, 0] == 0 and cells[1, 0] == vl['grid'][0] and (cells[[2, 3, 4], [0, 1, 2]] == -1).all()
    assert cells[5, 2] == 40 and cells[6, 2] == 41
    return ids


def cloud(cfg, vl, num_points=NUM_POINTS):
    from thinktwice_b200.synthetic import make_batch
    pts = make_batch(cfg, 2, seed=SEED, num_points=num_points)['points'][:, 0].float().contiguous()   # (B, P, 5)
    pts[1, PAD_FROM:] = 0
    return pts


def split_rows(x):
    """[2][rows * C] split planes of fp32 rows x (rows, C) on the device, and their float64 value on the host."""
    from thinktwice_b200.weights import f16s_split
    hi, lo = f16s_split(x.cpu())
    return torch.stack([hi.reshape(-1), lo.reshape(-1)]).cuda(), L.split_round(x).numpy()


# the rulebooks LidarNet._rulebook builds at the thinktwice.py shape: (level, tag, kernel, stride, padding, subm)
CHAIN = [('l0', (3, 3, 3), (1, 1, 1), (1, 1, 1), True), ('d0', (3, 3, 3), (2, 2, 2), (1, 1, 1), False),
         ('l1', (3, 3, 3), (1, 1, 1), (1, 1, 1), True), ('d1', (3, 3, 3), (2, 2, 2), (1, 1, 1), False),
         ('l2', (3, 3, 3), (1, 1, 1), (1, 1, 1), True), ('d2', (3, 3, 3), (2, 2, 2), (0, 1, 1), False),
         ('l3', (3, 3, 3), (1, 1, 1), (1, 1, 1), True), ('out', (3, 1, 1), (2, 1, 1), (0, 0, 0), False)]


def build_chain(eng, vox, shape, B=2):
    """every rulebook of the encoder in both forms, chained on the product's own output sites.  Returns {tag: dict(nbr=...,
    pairs=..., in_coords, in_count, in_cap, in_shape, spec)}."""
    coords, count, cap, shp = vox['coords'], vox['count'], vox['cap'], shape
    out = {}
    for tag, k, s, p, subm in CHAIN:
        rbs = {f: L.rulebook(eng, f'{tag}.{f}', B, coords, count, cap, shp, k, s, p, subm, f) for f in ('nbr', 'pairs')}
        out[tag] = dict(rbs, in_coords=coords, in_count=count, in_cap=cap, in_shape=shp, spec=(k, s, p, subm))
        if not subm:
            rb = rbs['nbr']
            coords, count, cap, shp = rb['coords'], rb['count'], rb['cap'], rb['shape']
    return out


@pytest.fixture(scope='module')
def full():
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.engine import Engine
    cfg = Config.fromfile(DEFAULT_CONFIG)
    vl, shape = L.voxel_layer(cfg)
    pts = cloud(cfg, vl)
    crafted = craft(pts, vl)
    eng = Engine('cuda:0', impl=4)
    vox = L.run_voxelize(pts.cuda(), vl)
    chain = build_chain(eng, vox, shape)
    torch.cuda.synchronize()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f'\nsites: l0 {int(vox["count"].item())}', ' '.join(f'{t} {int(c["nbr"]["count"].item())}' for t, c in chain.items()
                                                            if not c['spec'][3]), f'| SMs {sms}')
    return dict(cfg=cfg, vl=vl, shape=shape, pts=pts, crafted=crafted, eng=eng, vox=vox, chain=chain, sms=sms)


def test_voxelize_matches_hard_voxelize_and_the_fp64_mean_of_the_first_points(full):
    from oracle.lidar import hard_voxelize
    vl, pts, vox = full['vl'], full['pts'], full['vox']
    v = full['cfg'].model['lidar_encoder']['pts_voxel_layer']
    ref = L.ref_voxelize(pts.numpy(), vl['lower'], vl['vsize'], vl['grid'], vl['zmax'], vl['max_points'])
    # the oracle's site set per frame (first-seen order there, ascending (z, y, x) in the product), with the z >= 41 drop
    for b in range(2):
        _, c, _ = hard_voxelize(pts[b], v['voxel_size'], v['point_cloud_range'], v['max_num_points'], vl['max_voxels'])
        c = c.numpy().astype(np.int64)
        c = c[c[:, 0] < vl['zmax']]
        c = np.concatenate([np.full((len(c), 1), b), c], 1)
        c = c[np.argsort(L.site_keys(c, (vl['zmax'], vl['grid'][1], vl['grid'][0])))]
        assert np.array_equal(ref['coords'][ref['coords'][:, 0] == b], c), b
    err = L.check_voxelize({k: vox[k].cpu() for k in ('coords', 'feats', 'count')}, ref)
    n = len(ref['coords'])
    L.check_untouched(vox['feats'], n, 5, 'voxel feats')
    # the 40-point voxel averages exactly its first 10 points in input order, and another choice would be rejected
    row = [i for i, m in enumerate(ref['members']) if ref['coords'][i, 0] == 0 and np.isin(full['crafted'][0], m).any()]
    assert len(row) == 1 and np.array_equal(ref['members'][row[0]], full['crafted'][:vl['max_points']])
    p0 = pts[0].numpy().astype(np.float64)
    for alt in (full['crafted'][1:vl['max_points'] + 1], np.r_[full['crafted'][:vl['max_points'] - 1], full['crafted'][-1]]):
        assert (np.abs(p0[alt].mean(0) - ref['feats'][row[0]]) > L.VOX_TOL * ref['scale'][row[0]]).any()
    print(f'voxelize: {n} sites, max |err| {err:.2e} (bound {L.VOX_TOL:.0e} x mean|p|)')


def test_voxelize_with_a_frame_without_points_in_range(full):
    vl = full['vl']
    pts = full['pts'].clone()
    pts[1, :, 0] = 1000.0                                        # frame 1: every point outside the range
    vox = L.run_voxelize(pts.cuda(), vl)
    ref = L.ref_voxelize(pts.numpy(), vl['lower'], vl['vsize'], vl['grid'], vl['zmax'], vl['max_points'])
    assert (ref['coords'][:, 0] == 0).all()
    L.check_voxelize({k: vox[k].cpu() for k in ('coords', 'feats', 'count')}, ref)
    L.check_untouched(vox['feats'], len(ref['coords']), 5, 'voxel feats')


def test_rulebooks_match_the_reference(full):
    """every rulebook kind LidarNet builds (subm k3 at each level, the three down convs with their paddings, conv_out), in the
    neighbour-table and the pair-list form, against ref_rulebook on the same input sites."""
    for tag, c in full['chain'].items():
        k, s, p, subm = c['spec']
        n_in = int(c['in_count'].item())
        ref = L.ref_rulebook(c['in_coords'][:n_in].cpu().numpy(), c['in_shape'], k, s, p, subm)
        if not subm:
            assert (np.diff(L.site_keys(ref['coords'], ref['shape'])) > 0).all()
        for form in ('nbr', 'pairs'):
            rb = c[form]
            assert tuple(rb['shape']) == ref['shape']
            L.check_rulebook(L.rulebook_host(rb), ref, f'{tag}.{form}')
        print(f'rulebook {tag}: {n_in} -> {len(ref["coords"])} sites, {int((ref["nbr"] >= 0).sum())} pairs')


# (name, rulebook tag, Cin, Cout): every wide sparse conv LidarNet issues at thinktwice.py
CONVS = [('subm32', 'l1', 32, 32), ('subm64', 'l2', 64, 64), ('subm128', 'l3', 128, 128), ('down32_64', 'd1', 32, 64),
         ('down64_128', 'd2', 64, 128), ('conv_out', 'out', 128, 128)]


@pytest.mark.parametrize('name,tag,Cin,Cout', CONVS)
def test_f16s_sparse_conv_matches_fp64(full, name, tag, Cin, Cout):
    """both forms against the float64 oracle on the real site sets: bias + ReLU; fp32 and split-plane residuals; planes-only
    rows; the tap-major form's rows split by tt_split_f16 over the first *count rows; one tap per slab (0x200000) against the
    default.  Rows from *count up to the capacity keep their sentinels."""
    from thinktwice_b200 import lib
    from thinktwice_b200.lib import _p
    import ctypes as C
    c = full['chain'][tag]
    k, s, p, subm = c['spec']
    eng, sms = full['eng'], full['sms']
    rbo, rbt = c['nbr'], c['pairs']
    n_in, n = int(c['in_count'].item()), int(rbo['count'].item())
    kvol = rbo['kvol']
    gen = torch.Generator().manual_seed(Cin * 7 + Cout + kvol)
    x = torch.randn(c['in_cap'], Cin, generator=gen)
    w = torch.randn(Cout, kvol, Cin, generator=gen) * (kvol * Cin / 4) ** -0.5
    bias = torch.randn(Cout, generator=gen) * 0.1
    x_s, x64 = split_rows(x)
    ref_rb = L.ref_rulebook(c['in_coords'][:n_in].cpu().numpy(), c['in_shape'], k, s, p, subm)
    ref = L.ref_sparse_conv(x64[:n_in], c['in_coords'][:n_in].cpu().numpy(), c['in_shape'], 2, w.numpy(), k, s, p, subm, ref_rb)
    pw, pwb = L.pack(w.cuda()), L.pack(w.cuda(), bias.cuda())
    oi, ti = L.os_items(n, Cout), L.tap_items(rbt['pair_count'].cpu(), Cout)
    print(f'\n{name}: {n_in} -> {n} rows, work items os {oi} / tap {ti} against {sms} SMs')
    report = []

    def host(rows):
        return rows.detach().cpu().numpy()[:n].astype(np.float64)

    def check(label, out, out_s, y, bnd, scale=1.0):
        if out is not None:
            g, r = L.check_conv(host(out), y, bnd, f'{name} {label}', scale)
            L.check_untouched(out, n, Cout, f'{name} {label}')
            report.append((label, g, r))
        g, r = L.check_conv(L.planes_value(out_s, n, Cout), y, bnd + L.SPLIT * np.abs(y), f'{name} {label} planes', scale)
        L.check_untouched(out_s, n, Cout, f'{name} {label} planes')
        report.append((label + ' planes', g, r))

    # bias + ReLU, both forms; they agree with each other within the sum of their bounds
    y, bnd = L.expected(ref, bias.numpy(), act=1)
    oo, oo_s = L.run_conv(eng, rbo, x_s, pwb, act=1)
    ot, ot_s = L.run_conv(eng, rbt, x_s, pwb, act=1)
    torch.cuda.synchronize()
    check('os bias+relu', oo, oo_s, y, bnd)
    check('tap bias+relu', ot, ot_s, y, bnd)
    L.check_conv(host(oo), host(ot), 2 * bnd, f'{name} os vs tap')
    # the tap-major rows split again by tt_split_f16 limited to the first *count rows
    sp = L.sentinel_planes(rbt['cap'], Cout, 'cuda')
    lib.call('tt_split_f16', _p(ot), C.c_longlong(Cout), _p(sp), C.c_longlong(sp.numel() // 2), C.c_longlong(Cout),
             C.c_longlong(rbt['cap']), Cout, _p(rbt['count']))
    torch.cuda.synchronize()
    assert np.abs(L.planes_value(sp, n, Cout) - host(ot)).max() <= L.SPLIT * np.abs(host(ot)).max()
    L.check_untouched(sp, n, Cout, f'{name} tt_split_f16')
    if Cin == 32:                                                # two taps per K slab (default) against one tap per slab
        o1, o1_s = L.run_conv(eng, rbo, x_s, pwb, act=1, flags=L.ONE_TAP)
        torch.cuda.synchronize()
        check('os one-tap', o1, o1_s, y, bnd)
        L.check_conv(host(o1), host(oo), 2 * bnd, f'{name} one-tap vs two-tap')
    if subm and Cin == Cout:
        r = torch.randn(rbo['cap'], Cout, generator=gen)
        r_s, r64 = split_rows(r)
        y, bnd = L.expected(ref, bias.numpy(), res=r.numpy()[:n].astype(np.float64), act=1)
        for form, rb in (('os', rbo), ('tap', rbt)):             # fp32 residual
            o, o_s = L.run_conv(eng, rb, x_s, pwb, act=1, res=r.cuda())
            torch.cuda.synchronize()
            check(f'{form} res', o, o_s, y, bnd)
        y, bnd = L.expected(ref, bias.numpy(), res=r64[:n], act=1)
        o, o_s = L.run_conv(eng, rbo, x_s, pwb, act=1, res_s=r_s)   # split-plane residual
        torch.cuda.synchronize()
        check('os res_s', o, o_s, y, bnd)
        o, o_s = L.run_conv(eng, rbo, x_s, pwb, act=1, res_s=r_s, f32_out=False)   # planes-only rows
        torch.cuda.synchronize()
        check('os planes-only', None, o_s, y, bnd)
    else:
        y, bnd = L.expected(ref)                                 # no bias, no activation
        o, o_s = L.run_conv(eng, rbo, x_s, pw, f32_out=False)
        torch.cuda.synchronize()
        check('os planes-only', None, o_s, y, bnd)
    for label, g, r in report:
        print(f'  {label:<22} max err {g:.2e} of max|ref| (<= {L.GLOBAL_TOL:.0e}), max err/bound {r:.3f}')


def test_work_items_exceed_the_sm_count_in_both_forms(full):
    """the persistent loop, the barrier phases across tiles and the next-tap prefetch across a tile boundary need more work
    items than SMs: at 40000 points per frame the first wide level gives that in both forms."""
    sms = full['sms']
    wide = [(full['chain'][tag], Cout) for _, tag, _, Cout in CONVS]
    best_os = max(L.os_items(c['nbr']['count'].item(), Cout) for c, Cout in wide)
    best_tap = max(L.tap_items(c['pairs']['pair_count'].cpu(), Cout) for c, Cout in wide)
    print(f'most work items: os {best_os}, tap {best_tap}, SMs {sms}')
    assert best_os > sms and best_tap > sms


def _edge_pipeline(eng, pts, vl, shape, tag_sfx='', keep=None):
    """voxelise, build the subm (l0) and down (d0) rulebooks in both forms and run a 32 -> 32 subm and a 32 -> 64 down conv on
    fixed random rows in both forms; every result checked against its reference.  Rulebooks live in buffers of `eng`; the
    voxelisation and conv outputs in the dict `keep` when one is passed (filled on the first call, written again on the next,
    where rows past the count still hold the previous cloud's)."""
    reuse = keep is not None and 'vox' in keep
    vox = L.run_voxelize(pts.cuda(), vl, into=keep['vox'] if reuse else None)
    if keep is not None:
        keep['vox'] = vox
    ref_v = L.ref_voxelize(pts.numpy(), vl['lower'], vl['vsize'], vl['grid'], vl['zmax'], vl['max_points'])
    L.check_voxelize({k: vox[k].cpu() for k in ('coords', 'feats', 'count')}, ref_v)
    n0 = len(ref_v['coords'])
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(vox['cap'], 32, generator=gen)
    x_s, x64 = split_rows(x)
    res = {}
    for tag, k, s, p, subm, Cout in (('l0', (3, 3, 3), (1, 1, 1), (1, 1, 1), True, 32), ('d0', (3, 3, 3), (2, 2, 2), (1, 1, 1), False, 64)):
        w = torch.randn(Cout, 27, 32, generator=gen) * (27 * 8) ** -0.5
        ref_rb = L.ref_rulebook(ref_v['coords'], shape, k, s, p, subm)
        ref = L.ref_sparse_conv(x64[:n0], ref_v['coords'], shape, 2, w.numpy(), k, s, p, subm, ref_rb)
        y, bnd = L.expected(ref, act=1)
        pw = L.pack(w.cuda())
        for form in ('nbr', 'pairs'):
            rb = L.rulebook(eng, f'e{tag}.{form}', 2, vox['coords'], vox['count'], vox['cap'], shape, k, s, p, subm, form)
            o, o_s = L.run_conv(eng, rb, x_s, pw, act=1, into=keep.get((tag, form)) if reuse else None)
            if keep is not None:
                keep[(tag, form)] = (o, o_s)
            torch.cuda.synchronize()
            h = L.rulebook_host(rb)
            L.check_rulebook(h, ref_rb, f'{tag}.{form}{tag_sfx}')
            n = h['count']
            L.check_conv(o.cpu().numpy()[:n], y, bnd, f'{tag}.{form}{tag_sfx}')
            L.check_conv(L.planes_value(o_s, n, Cout), y, bnd + L.SPLIT * np.abs(y), f'{tag}.{form}{tag_sfx} planes')
            if not reuse:
                L.check_untouched(o, n, Cout, f'{tag}.{form}{tag_sfx}')
                L.check_untouched(o_s, n, Cout, f'{tag}.{form}{tag_sfx} planes')
            res[(tag, form)] = dict(rb=h, out=o.cpu()[:n].clone(), bound=bnd)
    return res


def test_zero_sites_in_one_frame_and_in_the_whole_batch(full):
    from thinktwice_b200.engine import Engine
    vl, shape = full['vl'], full['shape']
    pts = full['pts'][:, :5000].clone().contiguous()
    pts[1, :, 0] = -1000.0                                       # frame 1: no site
    res = _edge_pipeline(Engine('cuda:0', impl=4), pts, vl, shape, ' (frame 1 empty)')
    assert all((r['rb']['coords'][:r['rb']['count'], 0] == 0).all() for r in res.values())
    pts[0, :, 0] = -1000.0                                       # no site at all
    res = _edge_pipeline(Engine('cuda:0', impl=4), pts, vl, shape, ' (empty batch)')
    assert all(r['rb']['count'] == 0 and int(r['rb']['pair_count'].sum() if r['rb']['pair_count'] is not None else 0) == 0
               for r in res.values())


def test_a_smaller_cloud_in_the_buffers_of_a_larger_one_leaves_nothing_stale(full):
    """graph replay reuses the buffers of one capture for every cloud: run the full clouds, then a 5000-point cloud (the same
    capacity, the rest of its points out of range) in the same buffers, and compare with a run in fresh buffers.  The
    output-stationary conv has no atomics: bitwise equal.  The tap-major conv red.adds: within twice the bound."""
    from thinktwice_b200.engine import Engine
    vl, shape = full['vl'], full['shape']
    small = full['pts'].clone()
    small[:, 5000:, 0] = -1000.0
    reused, keep = Engine('cuda:0', impl=4), {}
    _edge_pipeline(reused, full['pts'], vl, shape, ' (full)', keep)
    again = _edge_pipeline(reused, small, vl, shape, ' (reused buffers)', keep)
    fresh = _edge_pipeline(Engine('cuda:0', impl=4), small, vl, shape, ' (fresh buffers)')
    for key in again:
        a, f = again[key], fresh[key]
        if key[1] == 'nbr':
            assert torch.equal(a['out'], f['out']), key
        else:
            L.check_conv(a['out'].numpy(), f['out'].numpy().astype(np.float64), 2 * a['bound'], f'{key} reused vs fresh')


# the encoder's levels in lidarnet.py order: (label, rulebook tag of the rows' sites, buffer, channels, convs from the voxels)
LEVELS = [('conv_input', 'l0', 'sp.l0.x', 16, 1), ('l0 blocks', 'l0', 'sp.l0.o1', 16, 5), ('d0', 'd0', 'sp.l1.x', 32, 6),
          ('l1 blocks', 'l1', 'sp.l1.o1', 32, 10), ('d1', 'd1', 'sp.l2.x', 64, 11), ('l2 blocks', 'l2', 'sp.l2.o1', 64, 15),
          ('d2', 'd2', 'sp.l3.x', 128, 16), ('l3 blocks', 'l3', 'sp.l3.o1', 128, 20), ('conv_out', 'out', 'sp.out.x', 128, 21)]


def test_encoder_layer_by_layer_matches_the_fp64_oracle():
    """the whole sparse encoder as lidarnet.py wires it (conv_input 5 -> 16, the 16-channel blocks on the tap-major SIMT path, the
    16 -> 32 down conv, the wide levels on the output-stationary f16s form with the conv1 -> conv2 residual handed over through
    planes-only rows, conv_out, tt_sparse_to_bev) on the calibrated model pair at B = 2 with collate padding, against the
    oracle's SparseEncoder run in float64 on the product's own voxel features and sites.  The sites of every level must be
    exact.  Each level's rows (the fp32 buffer, or the split planes where the product keeps no fp32 copy) and the densified
    output must be within depth x 5e-6 of the level's max |ref|, where depth is the number of convs from the voxels to that
    level (21 at conv_out): every conv is held to 5e-6 above (DESIGN.md §2), and the error of a chain of them grows at most by
    about one such bound per conv.  A failure names its level."""
    import copy
    from oracle.lidar import SparseTensor
    from test_model_gpu import build_pair
    from thinktwice_b200.config import DEFAULT_CONFIG
    cfg, oracle, model, batch = build_pair(DEFAULT_CONFIG, 2, NUM_POINTS, impl=0)
    batch['points'][1, :, PAD_FROM:] = 0
    model.use_graph = False
    model.forward_inference(batch)
    torch.cuda.synchronize()
    e = model.eng
    dev = lambda name: e.static_named(name).detach().cpu()
    n = int(dev('vox.count')[0])
    feats, coords = dev('vox.feats')[:n].double(), dev('vox.coords')[:n].long()
    enc = copy.deepcopy(oracle.lidar_encoder.pts_middle_encoder).double().eval()
    B = 2
    errs = []

    def compare(level, x):
        label, tag, buf, Cc, depth = level
        m = int(dev(f'sp.{tag}.count')[0])
        got_c = dev(f'sp.{tag}.coords')[:m].long()
        assert m == x.coords.shape[0] and torch.equal(got_c, x.coords), f'{label}: sites differ from the oracle'
        if buf in e.last_buf:
            got = dev(buf)[:m].double()
        else:                                                    # planes-only rows: hi + lo'/2048
            got = torch.from_numpy(L.planes_value(dev(buf + '#s'), m, Cc))
        tol = depth * L.GLOBAL_TOL
        err = float((got - x.feats).abs().max() / x.feats.abs().max().clamp_min(1e-30)) if m else 0.0
        errs.append((label, m, err, tol))
        assert err <= tol, f'{label}: error {err:.2e} of max |ref| > {tol:.1e} ({depth} convs x {L.GLOBAL_TOL:.0e})'

    with torch.no_grad():
        x = enc.conv_input(SparseTensor(feats, coords, enc.sparse_shape, B))
        li = iter(LEVELS)
        compare(next(li), x)
        for stage in enc.encoder_layers.children():
            mods = list(stage.children())
            for mod in mods[:2]:
                x = mod(x)
            compare(next(li), x)
            if len(mods) > 2:
                x = mods[2](x)
                compare(next(li), x)
        x = enc.conv_out(x)
        compare(next(li), x)
        d = x.dense()
    N, Cc, D, H, W = d.shape
    ref = d.view(N, Cc * D, H, W).permute(0, 2, 3, 1)
    got = dev('lidar.dense').double()
    err = float((got - ref).abs().max() / ref.abs().max())
    errs.append(('lidar.dense', N * H * W, err, 21 * L.GLOBAL_TOL))
    for label, m, er, tol in errs:
        print(f'  {label:<12} {m:>7} rows  error {er:.2e} of max|ref| (<= {tol:.1e})')
    assert err <= 21 * L.GLOBAL_TOL, f'lidar.dense: error {err:.2e}'
