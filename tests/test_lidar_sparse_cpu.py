"""The checks of tests/test_lidar_sparse_gpu.py (tests/lidar_sparse_checks.py) run on the torch emulation of the C ABI at a
reduced size: each accepts the emulated (correct) result and rejects a corrupted copy of it — a dropped site, a missing tap
in one row, a count off by one, a stale row past the count, a wrong neighbour-table entry."""
import numpy as np
import pytest
import torch

import lidar_sparse_checks as L

NUM_POINTS = 3000


@pytest.fixture
def emu(emulated):
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.engine import Engine
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    vl, shape = L.voxel_layer(cfg)
    pts = make_batch(cfg, 2, seed=0, num_points=NUM_POINTS)['points'][:, 0].float().contiguous()   # (B, P, 5)
    pts[1, 2000:] = 0                                            # mmcv collate padding
    eng = Engine('cpu', impl=4)
    vox = L.run_voxelize(pts, vl)
    ref_v = L.ref_voxelize(pts.numpy(), vl['lower'], vl['vsize'], vl['grid'], vl['zmax'], vl['max_points'])
    n0 = len(ref_v['coords'])
    rbs, refs = {}, {}
    for tag, k, s, p, subm in (('l0', (3, 3, 3), (1, 1, 1), (1, 1, 1), True), ('d0', (3, 3, 3), (2, 2, 2), (1, 1, 1), False)):
        refs[tag] = L.ref_rulebook(ref_v['coords'], shape, k, s, p, subm)
        for form in ('nbr', 'pairs'):
            rbs[(tag, form)] = L.rulebook(eng, f'{tag}.{form}', 2, vox['coords'], vox['count'], vox['cap'], shape, k, s, p, subm, form)
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(vox['cap'], 32, generator=gen)
    w = torch.randn(64, 27, 32, generator=gen) * (27 * 8) ** -0.5
    from thinktwice_b200.weights import f16s_split
    hi, lo = f16s_split(x)
    x_s, x64 = torch.stack([hi.reshape(-1), lo.reshape(-1)]), L.split_round(x).numpy()
    ref = L.ref_sparse_conv(x64[:n0], ref_v['coords'], shape, 2, w.numpy(), (3, 3, 3), (2, 2, 2), (1, 1, 1), False, refs['d0'])
    out, out_s = L.run_conv(eng, rbs[('d0', 'nbr')], x_s, L.pack(w), act=1)
    return dict(vox=vox, ref_v=ref_v, rbs=rbs, refs=refs, ref=ref, x64=x64, w=w.double().numpy(), out=out, out_s=out_s)


def _vox(e):
    return {k: e['vox'][k].clone() for k in ('coords', 'feats', 'count')}


def test_voxelize_check_accepts_the_result_and_rejects_a_dropped_site_and_an_off_count(emu):
    L.check_voxelize(_vox(emu), emu['ref_v'])
    L.check_untouched(emu['vox']['feats'], len(emu['ref_v']['coords']), 5, 'feats')
    v = _vox(emu)
    n = int(v['count'])
    v['coords'][5:n - 1] = v['coords'][6:n].clone()              # site 5 dropped
    v['feats'][5:n - 1] = v['feats'][6:n].clone()
    v['count'] -= 1
    with pytest.raises(AssertionError, match='sites'):
        L.check_voxelize(v, emu['ref_v'])
    v = _vox(emu)
    v['coords'][5:n - 1] = v['coords'][6:n].clone()              # site 5 dropped, the count kept (last row repeated)
    v['feats'][5:n - 1] = v['feats'][6:n].clone()
    with pytest.raises(AssertionError, match='site 5 is .* expected'):
        L.check_voxelize(v, emu['ref_v'])
    v = _vox(emu)
    v['count'] += 1
    with pytest.raises(AssertionError, match='sites'):
        L.check_voxelize(v, emu['ref_v'])
    v = _vox(emu)
    v['feats'][3, 3] += 2e-6 * max(1.0, float(v['feats'][3, 3].abs()))   # a mean over another set of points
    with pytest.raises(AssertionError, match='feature'):
        L.check_voxelize(v, emu['ref_v'])


@pytest.mark.parametrize('tag', ['l0', 'd0'])
@pytest.mark.parametrize('form', ['nbr', 'pairs'])
def test_rulebook_check_accepts_the_result_and_rejects_each_corruption(emu, tag, form):
    ref = emu['refs'][tag]
    h = L.rulebook_host(emu['rbs'][(tag, form)])
    L.check_rulebook(h, ref, tag)
    n = h['count']
    bad = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in h.items()}
    bad['coords'][7:n - 1] = h['coords'][8:n]                    # one site dropped
    bad['count'] = n - 1
    with pytest.raises(AssertionError):
        L.check_rulebook(bad, ref, tag)
    bad['count'] = n                                             # the same drop with the count kept (last row repeated)
    with pytest.raises(AssertionError, match='output site 7 is .* expected'):
        L.check_rulebook(bad, ref, tag)
    bad = dict(h, count=n + 1)                                   # count off by one
    with pytest.raises(AssertionError, match='output sites'):
        L.check_rulebook(bad, ref, tag)
    if form == 'nbr':                                            # one neighbour-table entry wrong
        nb = h['nbr'].copy()
        r, t = np.argwhere(nb[:n] >= 0)[len(np.argwhere(nb[:n] >= 0)) // 2]
        nb[r, t] = (nb[r, t] + 1) % n
        with pytest.raises(AssertionError, match='nbr'):
            L.check_rulebook(dict(h, nbr=nb), ref, tag)
    else:                                                        # one pair pointing at the wrong input row
        pi = h['pairs_in'].copy()
        pi[13, 0] = (pi[13, 0] + 1) % n
        with pytest.raises(AssertionError, match='input row'):
            L.check_rulebook(dict(h, pairs_in=pi), ref, tag)


def test_conv_check_accepts_the_result_and_rejects_a_missing_tap_and_a_stale_row(emu):
    ref, rb = emu['ref'], L.rulebook_host(emu['rbs'][('d0', 'nbr')])
    n = rb['count']
    y, bnd = L.expected(ref, act=1)
    L.check_conv(emu['out'].numpy()[:n], y, bnd, 'd0')
    L.check_untouched(emu['out'], n, 64, 'd0')
    L.check_untouched(emu['out_s'], n, 64, 'd0 planes')
    # one tap's contribution missing from one row (before the ReLU)
    r = int(np.argmax((rb['nbr'][:n] >= 0).sum(1)))
    t = int(np.nonzero(rb['nbr'][r] >= 0)[0][0])
    acc = ref['acc'].copy()
    acc[r] -= emu['x64'][rb['nbr'][r, t]] @ emu['w'][:, t, :].T
    with pytest.raises(AssertionError, match=f'row {r} '):
        L.check_conv(np.maximum(acc, 0), y, bnd, 'd0')
    # a row past the count written (stale data from a larger cloud)
    out = emu['out'].clone()
    out[n] = 0.5
    with pytest.raises(AssertionError, match='past the count'):
        L.check_untouched(out, n, 64, 'd0')
    planes = emu['out_s'].clone()
    planes.view(2, -1, 64)[1, n + 2] = 0
    with pytest.raises(AssertionError, match='past the count'):
        L.check_untouched(planes, n, 64, 'd0 planes')
