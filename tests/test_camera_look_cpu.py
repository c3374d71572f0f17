"""The checks of tests/test_camera_look_gpu.py (tests/camera_look_checks.py) run on the torch emulation of the C ABI at a
reduced size: each accepts the emulated (correct) result and rejects a corrupted copy of it, with a message that names the
frame / cell, the (frame, camera, query) or the pixel / tap."""
import numpy as np
import pytest
import torch

import camera_look_checks as K


@pytest.fixture
def cfg():
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    return Config.fromfile(DEFAULT_CONFIG)


# ---------------------------------------------------------------------------------------------------------- lift-splat
@pytest.fixture
def lift(emulated, cfg):
    from thinktwice_b200.synthetic import rig_metas
    geo = K.lift_geometry(cfg, final_dim=(128, 256))
    B, Cc, N = 2, 32, geo['N']
    metas = [rig_metas(geo['final_dim'], 2) for _ in range(B)]
    s2e, intr, ida = K.sweep_mats(metas, N, 1)
    mats = K.kernel_mats(s2e, intr, ida)
    gen = torch.Generator().manual_seed(0)
    dl = K.depth_logits(gen, B * N, geo['fH'], geo['fW'], geo['D'])
    ctx = torch.randn(B * N, geo['fH'], geo['fW'], Cc, generator=gen)
    ref = K.ref_lift(dl.numpy(), ctx.numpy(), s2e, intr, ida, mats, geo)
    bev = torch.full((B, geo['Y'], geo['X'], 2 * Cc), float('nan'))
    before = bev.numpy().copy()
    K.run_lift(K.lift_desc(geo, B, Cc, geo['D'], 0, Cc, 0, 2 * Cc, 0), geo, dl, ctx, mats, bev, bev_ptr_off=Cc)
    return dict(geo=geo, ref=ref, ctx=ctx.double().numpy().reshape(-1, Cc), after=bev.numpy().copy(), before=before, C=Cc)


def _cell_msg(b, cell, X):
    return f'frame {b} cell \\(y {cell // X}, x {cell % X}\\)'


def test_lift_check_accepts_the_result_and_rejects_each_corruption(lift):
    geo, ref, Cc, X = lift['geo'], lift['ref'], lift['C'], lift['geo']['X']
    check = lambda after: K.check_lift(after, lift['before'], ref, geo, Cc)
    assert 0.05 < ref['in_bins'] / ref['bins'] < 0.95
    check(lift['after'])
    W = ref['W'].tocoo()
    k = int(np.argmax(W.data))                                   # the heaviest (pixel, cell) run: a one-hot pixel's bin
    row, pix, w = int(W.row[k]), int(W.col[k]), float(W.data[k])
    assert w > 0.99
    b, cell = divmod(row, X * X)
    y, x = divmod(cell, X)
    # one bin's weight dropped
    a = lift['after'].copy()
    a[b, y, x, Cc:] -= (w * lift['ctx'][pix]).astype(np.float32)
    with pytest.raises(AssertionError, match=_cell_msg(b, cell, X)):
        check(a)
    # the same run put in the neighbouring cell
    nx = x + 1 if x + 1 < X else x - 1
    a[b, y, nx, Cc:] += (w * lift['ctx'][pix]).astype(np.float32)
    with pytest.raises(AssertionError, match=f'frame {b} cell \\(y {y}, x ({x}|{nx})\\)'):
        check(a)
    # an empty cell left at its sentinel
    cold = np.argwhere(~ref['reached'])
    b2, c2 = (int(v) for v in (cold[0] if len(cold) else (1, 0)))
    a = lift['after'].copy()
    a[b2, c2 // X, c2 % X, Cc + 3] = np.nan
    with pytest.raises(AssertionError, match=_cell_msg(b2, c2, X) + ' channel 3: not written'):
        check(a)
    # a write into the other half of the concat buffer
    a = lift['after'].copy()
    a[1, 4, 5, 7] = 0.0
    with pytest.raises(AssertionError, match='frame 1 row 4 col 5 column 7: outside the written range'):
        check(a)


# ---------------------------------------------------------------------------------------------------------- Look module
LEVELS = [(16, 32), (8, 16), (4, 8), (2, 4)]


@pytest.fixture
def look(emulated, cfg):
    from thinktwice_b200 import lib
    from thinktwice_b200.lss import LSS
    from thinktwice_b200.synthetic import rig_metas
    B = 2
    d, _ = K.look_desc(cfg, B)
    d.C = 8
    d.lvl_h, d.lvl_w = lib.i4([h for h, _ in LEVELS]), lib.i4([w for _, w in LEVELS])
    N, T = d.num_cams, d.T
    H, W = int(d.img_h), int(d.img_w)
    metas = [rig_metas((H, W), 2) for _ in range(B)]
    l2i = torch.stack([m[-1]['lidar2img'] for m in metas]).float().clone()
    ida = LSS.build_mats(metas, N)['ida_mats'][:, -1].clone().float()
    gen = torch.Generator().manual_seed(1)
    wp = torch.stack([torch.randn(B, T, generator=gen) * 8 + 6, torch.randn(B, T, generator=gen) * 4], -1)
    l2i[1, 3] = torch.tensor([[1.0, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1], [0, 0, 0, 1]])   # x = px / W, y = py / H
    ida[1, 3] = torch.eye(4)
    f = 0.3 / LEVELS[0][1]                                      # the outer half pixel of every level
    wp[1] = torch.tensor([[f * W, H / 2], [W - f * W, H / 2], [W / 2, f * H], [W / 2, H - f * H]])
    wp = wp.contiguous()
    l2i, ida = l2i.reshape(B, N, 16).contiguous(), ida.reshape(B, N, 16).contiguous()
    ref = K.ref_project(wp.numpy(), l2i.view(B, N, 4, 4).numpy(), ida.view(B, N, 4, 4).numpy(), d.img_w, d.img_h)
    proj = K.run_project(d, wp, l2i, ida)
    ctrl_sp = torch.nn.functional.softplus(torch.randn(B, T, 4, generator=gen))
    temb, semb = torch.randn(T, d.emb_dim, generator=gen), torch.randn(4, d.emb_dim, generator=gen)
    meas, flat = torch.randn(B, d.meas_dim, generator=gen), torch.randn(B, d.flat_dim, generator=gen)
    levels = [torch.randn(B * N, h, w, d.C, generator=gen) for h, w in LEVELS]
    rows_ld = d.q_dim + d.levels * d.C + 5
    rows = torch.full((B * N * d.max_len_cap, rows_ld), K.SENT)
    rows[:, :rows_ld - 5] = float('nan')
    before = rows.numpy().copy()
    ref_re = torch.full((B * N * d.max_len_cap, 2), float('nan'))
    K.run_rebatch(d, wp, ctrl_sp, temb, semb, meas, flat, levels, proj, rows, rows_ld, ref_re)
    qrows = K.query_rows(d, wp.numpy(), ctrl_sp.numpy(), temb.numpy(), semb.numpy(), meas.numpy(), flat.numpy())
    return dict(d=d, ref=ref, ph=K.host(proj), rows=rows.numpy().copy(), before=before, re=ref_re.numpy().copy(), qrows=qrows,
                levels=levels, rows_ld=rows_ld)


def test_look_project_check_accepts_the_result_and_rejects_each_corruption(look):
    ref, ph = look['ref'], look['ph']
    K.check_project(ph, ref)
    n_cams = ph['counts'].shape[1]
    exact = [(b, n) for b in range(ph['counts'].shape[0]) for n in range(n_cams)
             if ref['valid'][b, n].sum() == ref['maybe'][b, n].sum() and ph['counts'][b, n] >= 3]
    b, n = exact[0]
    cnt = int(ph['counts'][b, n])
    # a valid query dropped from order, the count kept (the last entry repeated)
    bad = {k: v.copy() for k, v in ph.items()}
    q = int(bad['order'][b, n, 1])
    bad['order'][b, n, 1:cnt - 1] = ph['order'][b, n, 2:cnt]
    with pytest.raises(AssertionError, match=f'\\(b {b}, cam {n}, query {q}\\): valid but missing'):
        K.check_project(bad, ref)
    # two entries swapped
    bad = {k: v.copy() for k, v in ph.items()}
    bad['order'][b, n, [0, 1]] = ph['order'][b, n, [1, 0]]
    with pytest.raises(AssertionError, match=f'\\(b {b}, cam {n}\\): order not strictly ascending'):
        K.check_project(bad, ref)
    # a count off by one (max_len kept consistent)
    bad = {k: v.copy() for k, v in ph.items()}
    bad['counts'][b, n] += 1
    bad['max_len'][0] = bad['counts'].max()
    with pytest.raises(AssertionError, match=f'\\(b {b}, cam {n}\\): count {cnt + 1}, expected {cnt}'):
        K.check_project(bad, ref)
    # max_len of a different call
    bad = {k: v.copy() for k, v in ph.items()}
    bad['max_len'][0] += 1
    with pytest.raises(AssertionError, match='max_len'):
        K.check_project(bad, ref)


def test_look_rebatch_check_accepts_the_result_and_rejects_each_corruption(look):
    d, ph, rows_ld = look['d'], look['ph'], look['rows_ld']
    N, cap, Q = d.num_cams, d.max_len_cap, d.num_query
    check = lambda rows, re=look['re']: K.check_rebatch(rows, look['before'], re, d, ph, look['qrows'], look['levels'], rows_ld)
    check(look['rows'])
    # a nonzero row past the count
    bn = int(np.argmin(ph['counts'].reshape(-1)))
    c0 = int(ph['counts'].reshape(-1)[bn])
    rows = look['rows'].copy()
    rows.reshape(-1, cap, rows_ld)[bn, c0, 11] = 0.5
    with pytest.raises(AssertionError, match=f'\\(b {bn // N}, cam {bn % N}, row {c0}\\): past the count'):
        check(rows)
    # a bilinear corner dropped at a map border: frame 1 camera 3, waypoint 0 samples x0 = -1 on level 0; drop corner (y0, x0 + 1)
    bn = 1 * N + 3
    order = ph['order'].reshape(-1, Q)[bn]
    r = int(np.nonzero(order[:ph['counts'].reshape(-1)[bn]] < 15)[0][0])          # a row of waypoint 0
    rx, ry = ph['ref_cam'].reshape(-1, Q, 2)[bn, order[r]].astype(np.float64)
    Hl, Wl = LEVELS[0]
    x, y = rx * Wl - 0.5, ry * Hl - 0.5
    assert np.floor(x) == -1
    y0 = int(np.floor(y))
    f = look['levels'][0][bn, y0, 0, 2].double().item()
    rows = look['rows'].copy()
    rows.reshape(-1, cap, rows_ld)[bn, r, d.q_dim + 2 * d.levels + 0] -= np.float32((1 - (y - y0)) * (x + 1) * f)
    with pytest.raises(AssertionError, match=f'\\(b 1, cam 3, row {r} = query {order[r]}\\): sampled feature \\(c 2, level 0\\)'):
        check(rows)
    # a ref_rebatch row that is not ref_cam[order]
    re = look['re'].copy()
    re.reshape(-1, cap, 2)[bn, r, 0] += 1e-3
    with pytest.raises(AssertionError, match=f'\\(b 1, cam 3, row {r} = query {order[r]}\\): ref_rebatch'):
        check(look['rows'], re)
    # a write into the tail columns
    rows = look['rows'].copy()
    rows[5, rows_ld - 2] = 0.0
    with pytest.raises(AssertionError, match=f'row 5 tail column {rows_ld - 2}'):
        check(rows)


# ---------------------------------------------------------------------------------------------------------- DCN columns
def test_dcn_check_accepts_the_result_and_rejects_each_corruption(emulated):
    N, H, W, Cc, G, off_ld = 2, 6, 9, 16, 4, 20
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(N, H, W, Cc, generator=gen)
    off = torch.full((N, H, W, off_ld), float('nan'))
    off[..., :18] = torch.randn(N, H, W, 18, generator=gen) * 3
    K.craft_dcn_offsets(off, H, W, 0, gen)
    col = torch.full((N * H * W * 9 * Cc,), float('nan'))
    K.run_dcn(x, off, off_ld, col, G)
    K.check_dcn(x, off, col, G, range(N))
    h, w = K.dcn_positions(off[:1], H, W)
    h, w = h[0], w[0]
    Cg = Cc // G

    def at(ho, wo, k, c):                                        # flat index of column element (image 0, pixel, tap, channel)
        return ((ho * W + wo) * G + c // Cg) * 9 * Cg + k * Cg + c % Cg
    # a corner dropped at the border: h in (-1, 0) keeps only the row-0 corners; drop (0, wl)
    ho, wo, k = (int(v) for v in torch.nonzero((h > -1) & (h < 0) & (w > 0) & (w < W - 1))[0])
    lh, wl = float(h[ho, wo, k]) + 1, int(np.floor(float(w[ho, wo, k])))
    lw = float(w[ho, wo, k]) - wl
    bad = col.clone()
    bad[at(ho, wo, k, 5)] -= lh * (1 - lw) * float(x[0, 0, wl, 5])
    with pytest.raises(AssertionError, match=f'image 0 pixel \\(h {ho}, w {wo}\\) tap {k} channel 5'):
        K.check_dcn(x, off, bad, G, [0])
    # the validity test at -1 made inclusive: a sample exactly at h = -1 reads the border row instead of giving 0
    ho, wo, k = (int(v) for v in torch.nonzero((h == -1) & (w > 0) & (w < W - 1))[0])
    bad = col.clone()
    bad[at(ho, wo, k, 3)] = x[0, 0, int(np.floor(float(w[ho, wo, k]))), 3]
    with pytest.raises(AssertionError, match=f'image 0 pixel \\(h {ho}, w {wo}\\) tap {k} channel 3'):
        K.check_dcn(x, off, bad, G, [0])


# ---------------------------------------------------------------------------------------------------------- GRU input plane
def test_gru_check_accepts_the_result_and_rejects_each_corruption(emulated):
    B, T, ld, col0 = 2, 4, 40, 32
    gen = torch.Generator().manual_seed(3)
    wp, cs = torch.randn(B, T, 2, generator=gen), torch.randn(B, T, 4, generator=gen)
    buf = torch.full((B, 5, 5, ld), K.SENT)
    before = buf.numpy().reshape(B, -1, ld).copy()
    K.run_gru(wp, cs, 2, buf, col0)
    after = buf.numpy().reshape(B, -1, ld).copy()
    K.check_gru(after, before, wp.numpy(), cs.numpy(), 2, col0)
    bad = after.copy()
    bad[1, 7, 38] = 0.0
    with pytest.raises(AssertionError, match='frame 1 pixel 7 column 38: outside the written range'):
        K.check_gru(bad, before, wp.numpy(), cs.numpy(), 2, col0)
    bad = after.copy()
    bad[0, 3, 34] = cs[0, 1, 0]                                  # step 1's control instead of step 2's
    with pytest.raises(AssertionError, match='frame 0 pixel 3 column 34'):
        K.check_gru(bad, before, wp.numpy(), cs.numpy(), 2, col0)
