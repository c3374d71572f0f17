"""Camera-branch and Look-module kernels at the full thinktwice.py shapes against float64 references: the fused lift-splat
(tt_lift_splat), Look projection + ordered compaction (tt_look_project) and query rebatching with the 4-level bilinear FPN
gather (tt_look_rebatch), the deformable-conv column builder (tt_dcn_im2col) and the GRU input plane (tt_gru_input).  Every
shape comes from configs/thinktwice.py through the product's LSS / ThinkTwiceDecoder._look_meta; the full model is not built.
The checks and their bounds are in tests/camera_look_checks.py; tests/test_camera_look_cpu.py shows that each of them rejects a
corrupted result.  Each test prints the largest error-to-bound ratio it saw."""
import numpy as np
import pytest
import torch

import camera_look_checks as K

pytestmark = pytest.mark.gpu
DCN_GROUPS = 4           # DeformConv2dPack groups (lss.py: conv_group_gemms(..., groups=4))
OFF_LD = 32              # the offset conv's 18 channels padded to 32 (lss.py: conv(..., cout_pad=32))
GRU_LD, GRU_COL = 40, 32  # SpatialGRU planes [state 32 | x_t 6 | 0 0] (ThinkTwiceDecoder._gru)


@pytest.fixture(scope='module')
def cfg():
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    return Config.fromfile(DEFAULT_CONFIG)


@pytest.fixture(scope='module')
def geo(cfg):
    return K.lift_geometry(cfg)


def _metas(geo, B):
    from thinktwice_b200.synthetic import rig_metas
    return [rig_metas(geo['final_dim'], geo['queue_len']) for _ in range(B)]


def _inputs(geo, B, seed, C_=None):
    gen = torch.Generator().manual_seed(seed)
    BN = B * geo['N']
    dl = K.depth_logits(gen, BN, geo['fH'], geo['fW'], geo['D'])
    ctx = torch.randn(BN, geo['fH'], geo['fW'], C_ or geo['C'], generator=gen)
    return dl, ctx


def _bev(B, geo, ld):
    return torch.full((B, geo['Y'], geo['X'], ld), float('nan'), device='cuda')


# ---------------------------------------------------------------------------------------------------------- lift-splat
def test_lift_splat_full_batch_both_sweeps_workspace_reuse_and_run_to_run(geo):
    """B = 16 at the model's layout: both sweeps write their half of one [B][21][21][2C] buffer (history first, through a
    pointer offset as LSS passes the concat slice), then B = 1 and B = 16 again in the same workspace.  K3 places the runs with
    integer atomics, so the order of the sums in a cell changes from run to run: two runs agree within the bound, not bitwise."""
    B, Cc, N = 16, geo['C'], geo['N']
    metas = _metas(geo, B)
    refs, ins = {}, {}
    for s in (1, 0):
        s2e, intr, ida = K.sweep_mats(metas, N, s)
        mats = K.kernel_mats(s2e, intr, ida)
        dl, ctx = _inputs(geo, B, 10 + s)
        refs[s] = K.ref_lift(dl.numpy(), ctx.numpy(), s2e, intr, ida, mats, geo)
        ins[s] = (dl.cuda(), ctx.cuda(), mats.cuda())
        frac = refs[s]['in_bins'] / refs[s]['bins']
        print(f'[lift] sweep {s}: {refs[s]["bins"]} bins, {frac:.1%} in the grid, {refs[s]["amb_bins"]} ambiguous, '
              f'{int(refs[s]["reached"].sum())} of {refs[s]["reached"].size} cells reached')
        assert 0.05 < frac < 0.95
    d = K.lift_desc(geo, B, Cc, geo['D'], 0, Cc, 0, 2 * Cc, 0)
    ws = K.lift_workspace(d, 'cuda')
    bev = _bev(B, geo, 2 * Cc)
    ratios = []
    before = bev.cpu().numpy()
    K.run_lift(d, geo, *ins[1], bev, bev_ptr_off=Cc, ws=ws)                     # history half first, as history_device does
    after = bev.cpu().numpy()
    ratios.append(K.check_lift(after, before, refs[1], geo, Cc, name='lift_splat sweep 1'))
    K.run_lift(d, geo, *ins[0], bev, ws=ws)
    key = bev.cpu().numpy()
    ratios.append(K.check_lift(key, after, refs[0], geo, 0, name='lift_splat sweep 0'))
    # B = 1 in the B = 16 workspace: frame 0 of sweep 0 (frames are independent)
    d1 = K.lift_desc(geo, 1, Cc, geo['D'], 0, Cc, 0, Cc, 0)
    one = _bev(1, geo, Cc)
    dl, ctx, mats = ins[0]
    K.run_lift(d1, geo, dl[:N].contiguous(), ctx[:N].contiguous(), mats[:N].contiguous(), one, ws=ws)
    r1 = dict(refs[0], val=refs[0]['val'][:1], bound=refs[0]['bound'][:1])
    ratios.append(K.check_lift(one.cpu().numpy(), np.full_like(one.cpu().numpy(), np.nan), r1, geo, 0, name='lift_splat B=1 reused ws'))
    again = _bev(B, geo, Cc)
    K.run_lift(K.lift_desc(geo, B, Cc, geo['D'], 0, Cc, 0, Cc, 0), geo, *ins[0], again, ws=ws)
    a2 = again.cpu().numpy()
    ratios.append(K.check_lift(a2, np.full_like(a2, np.nan), refs[0], geo, 0, name='lift_splat B=16 after B=1'))
    diff = np.abs(a2.astype(np.float64) - key[..., :Cc]).reshape(B, -1, Cc)
    over = diff > refs[0]['bound']
    assert not over.any(), f'lift_splat run to run: frame/cell/channel {np.argwhere(over)[0].tolist()} differs by more than the bound'
    print(f'[lift] run to run: {int((diff > 0).sum())} of {diff.size} elements differ, largest {diff.max():.2e}')
    print(f'[lift] B=16 largest err/bound {max(ratios):.4f}')


def _crafted_mats(geo, B):
    """(s2e, intrin, ida) for crafted rays: ida swaps rows 2 and 3 and intrin = I, so p = (u, v, 1, d) and every bin of a
    pixel lands on one point g = Mc (u, v, 1): a = size / (pixel step) turns pixel column i into t = i + 0.5.
      frame 0 cam 0: pixel (i, j) -> cell (x i, y j): pixels with i, j < 21 alone in their cell, the others off the grid
      frame 0 cam 1: t_x in (-0.9, -0.1) and t_z = -0.5 (the truncation band: cell x 0, z 0), t_y = j + 0.5
      frame 0 cam 2 / cam 3: t_z = -3 / t_x = 25.5: every ray misses the grid
      frame 1: every camera misses (a frame with an empty BEV)
      frames >= 2: the rig."""
    N, X = geo['N'], geo['X']
    lower, size = geo['lower'].astype(np.float64), geo['size'].astype(np.float64)
    su = float(geo['fu'][1] - geo['fu'][0])
    sv = float(geo['fv'][1] - geo['fv'][0])
    s2e, intr, ida = K.sweep_mats(_metas(geo, B), N, 0)
    s2e, intr, ida = s2e.clone(), intr.clone(), ida.clone()
    P = torch.eye(4)[[0, 1, 3, 2]]
    umax = float(geo['fu'][-1])

    def mc(tx, ty, tz):                                           # each t as (coef of u, coef of v, constant)
        m = torch.zeros(4, 4, dtype=torch.float64)
        for r, (cu, cv, c0) in enumerate((tx, ty, tz)):
            m[r, 0], m[r, 1], m[r, 2] = cu * size[r], cv * size[r], lower[r] + c0 * size[r]
        m[3, 3] = 1
        return m.float()
    cams = {(0, 0): mc((1 / su, 0, 0.5), (0, 1 / sv, 0.5), (0, 0, 0.5)),
            (0, 1): mc((0.8 / umax, 0, -0.9), (0, 1 / sv, 0.5), (0, 0, -0.5)),
            (0, 2): mc((1 / su, 0, 0.5), (0, 1 / sv, 0.5), (0, 0, -3.0)),
            (0, 3): mc((0, 0, X + 4.5), (0, 1 / sv, 0.5), (0, 0, 0.5))}
    for n in range(N):
        cams[(1, n)] = mc((0, 0, -5.5), (0, 1 / sv, 0.5), (0, 0, 0.5))
    for (b, n), m in cams.items():
        s2e[b, n], intr[b, n], ida[b, n] = m, torch.eye(4), P
    return s2e, intr, ida


@pytest.mark.parametrize('Cc', [80, 264, 512])
@pytest.mark.parametrize('anti', [0, 1])
def test_lift_splat_crafted_rays_strided_layouts_and_channel_passes(geo, Cc, anti):
    """crafted rays (one cell per pixel, the truncation band, rays and a whole frame off the grid) next to a rig frame, with
    the logits at d_coff 8 of a wider depth buffer (NaN elsewhere), the context at c_coff 8 of a wider buffer (NaN
    elsewhere) and the BEV at bev_coff 8.  C = 80 leaves lanes idle in the first channel pass, 264 and 512 need a second
    pass (C / 4 > 64); anti_transpose stores the rot90(flip) layout."""
    B, N, D, fH, fW = 3, geo['N'], geo['D'], geo['fH'], geo['fW']
    s2e, intr, ida = _crafted_mats(geo, B)
    mats = K.kernel_mats(s2e, intr, ida)
    dl, ctx = _inputs(geo, B, 20 + Cc, Cc)
    ref = K.ref_lift(dl.numpy(), ctx.numpy(), s2e, intr, ida, mats, geo)
    X = geo['X']
    # what the crafted rays must produce: a lone pixel's cell is its context row; frame 1 is empty; cell x 0 gets the band
    r, c = 5, 7
    lone = ctx[0, r, c].double().numpy()
    assert np.allclose(ref['val'][0, r * X + c], lone, rtol=1e-12, atol=0)
    assert not ref['reached'][1].any() and ref['reached'][2].any()
    band = ref['W'][0 * X * X + 3 * X + 0].toarray().reshape(B * N, fH, fW)
    assert band[1].sum() > 0                                      # camera 1's truncation-band pixels reach cell (y 3, x 0)
    dpad, cpad, bpad = 8, 8, 8
    dbuf = torch.full((B * N, fH, fW, D + 2 * dpad), float('nan'))
    dbuf[..., dpad:dpad + D] = dl
    cbuf = torch.full((B * N, fH, fW, Cc + 2 * cpad), float('nan'))
    cbuf[..., cpad:cpad + Cc] = ctx
    bev = torch.full((B, geo['Y'], X, Cc + 2 * bpad), K.SENT, device='cuda')
    bev[..., bpad:bpad + Cc] = float('nan')
    before = bev.cpu().numpy()
    d = K.lift_desc(geo, B, Cc, D + 2 * dpad, dpad, Cc + 2 * cpad, cpad, Cc + 2 * bpad, bpad, anti)
    K.run_lift(d, geo, dbuf.cuda(), cbuf.cuda(), mats.cuda(), bev)
    ratio = K.check_lift(bev.cpu().numpy(), before, ref, geo, bpad, anti=bool(anti), name=f'lift_splat C={Cc} anti={anti}')
    print(f'[lift] crafted C={Cc} anti={anti}: largest err/bound {ratio:.4f}')


# ---------------------------------------------------------------------------------------------------------- Look module
def _look_inputs(cfg, d, B):
    """rig lidar2img / ida with crafted cameras and waypoints (see the test docstring)."""
    from thinktwice_b200.lss import LSS
    from thinktwice_b200.synthetic import rig_metas
    H, W = cfg.model['decoder']['config']['img_size']
    metas = [rig_metas((H, W), 2) for _ in range(B)]
    l2i = torch.stack([m[-1]['lidar2img'] for m in metas]).float().clone()
    ida = LSS.build_mats(metas, d.num_cams)['ida_mats'][:, -1].clone().float()
    gen = torch.Generator().manual_seed(3)
    T = d.T
    wp = torch.stack([torch.randn(B, T, generator=gen) * 8 + 6, torch.randn(B, T, generator=gen) * 4], -1)
    I = torch.eye(4)

    def cam(rows):
        m = torch.zeros(4, 4)
        m[:3] = torch.tensor(rows, dtype=torch.float32)
        m[3, 3] = 1
        return m
    # frame 1 cam 2: the comb: x = 64 py + 320 (py = -5 -> x = 0 exactly: invalid), y = 20 (z + 4) (z = -4 -> y = 0: invalid),
    # so the valid queries are the waypoints / static points with py > -5 at z levels 1..14
    l2i[1, 2], ida[1, 2] = cam([[0, 64, 0, 320], [0, 0, 20, 80], [0, 0, 0, 1]]), I
    wp[1, :, 1] = torch.tensor([-5.0, -5.0, 0.0, -5.0])
    # frame 2 cam 0 sees nothing, frame 3 cam 1 sees every query
    l2i[2, 0], ida[2, 0] = cam([[0, 0, 0, 0], [0, 0, 0, 0], [0, 0, 0, 0]]), I
    l2i[3, 1], ida[3, 1] = cam([[0, 0, 0, W / 2], [0, 0, 0, H / 2], [0, 0, 0, 1]]), I
    # frames 4, 5 cam 3: x = px / W, y = py / H; their waypoints sample the outer half pixel of the FPN levels
    # (frame 4: every level, frame 5: only the coarse ones)
    for b, f in ((4, 0.3 / d.lvl_w[0]), (5, 0.4 / d.lvl_w[3])):
        l2i[b, 3], ida[b, 3] = cam([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1]]), I
        fy = f * W / H if b == 5 else f
        wp[b] = torch.tensor([[f * W, H / 2], [W - f * W, H / 2], [W / 2, fy * H], [W / 2, H - fy * H]])
    return wp.float().contiguous(), l2i.reshape(B, -1, 16).contiguous(), ida.reshape(B, -1, 16).contiguous()


def test_look_project_and_rebatch_full_batch(cfg):
    """B = 16 with the rig's lidar2img / ida, random waypoints and crafted cameras: a comb whose valid queries sit on both
    sides of every 32-query chunk edge (31/32, 63/64, 95/96) and at 119, with exact ties x = 0 and y = 0 (invalid), a camera
    that sees no query and one that sees all 120, queries behind the rig cameras, and samples in the outer half pixel of the
    FPN levels (x0 = -1, x0 + 1 = W, the same in y).  Project runs twice, first with every camera seeing every query: the
    counts and max_len must be those of the second call.  The rebatch writes rows of width 1543 into rows_ld = 1552 (tail
    columns hold sentinels, the rows start as NaN)."""
    B = 16
    d, lv = K.look_desc(cfg, B)
    N, Q, cap = d.num_cams, d.num_query, d.max_len_cap
    wp, l2i, ida = _look_inputs(cfg, d, B)
    ref = K.ref_project(wp.numpy(), l2i.view(B, N, 4, 4).numpy(), ida.view(B, N, 4, 4).numpy(), d.img_w, d.img_h)
    assert (ref['depth'] < 0).any() and ref['valid'][1, 2][[31, 32, 63, 64, 95, 96, 119]].all()
    assert ref['valid'][3, 1].all() and not ref['maybe'][2, 0].any()
    print(f'[look] {int(ref["valid"].sum())} surely valid, {int((ref["maybe"] & ~ref["valid"]).sum())} ambiguous of {ref["valid"].size} queries')
    allv = torch.zeros(B, N, 4, 4)
    allv[..., 0, 3], allv[..., 1, 3], allv[..., 2, 3], allv[..., 3, 3] = d.img_w / 2, d.img_h / 2, 1, 1
    proj = K.run_project(d, wp.cuda(), allv.reshape(B, N, 16).cuda(), torch.eye(4).repeat(B, N, 1, 1).reshape(B, N, 16).cuda())
    assert int(proj['max_len'][0]) == Q
    K.run_project(d, wp.cuda(), l2i.cuda(), ida.cuda(), out=proj)
    ph = K.host(proj)
    r_proj = K.check_project(ph, ref)
    comb = ph['order'][1, 2, :ph['counts'][1, 2]]
    want = [t * 15 + z for t in (2, 4, 6, 7) for z in range(1, 15)]
    assert comb.tolist() == want, f'look_project: (b 1, cam 2): order {comb.tolist()}, expected {want}'
    assert ph['counts'][2, 0] == 0 and ph['counts'][3, 1] == Q
    # rebatch
    gen = torch.Generator().manual_seed(4)
    T, E = d.T, d.emb_dim
    ctrl_sp = torch.nn.functional.softplus(torch.randn(B, T, 4, generator=gen))
    temb, semb = torch.randn(T, E, generator=gen), torch.randn(4, E, generator=gen)
    meas, flat = torch.randn(B, d.meas_dim, generator=gen), torch.randn(B, d.flat_dim, generator=gen)
    levels = [torch.randn(B * N, h, w, d.C, device='cuda') for h, w in lv]
    width, rows_ld = d.q_dim + d.levels * d.C, 1552
    assert width == 1543
    rows = torch.full((B * N * cap, rows_ld), K.SENT, device='cuda')
    rows[:, :width] = float('nan')
    ref_re = torch.full((B * N * cap, 2), float('nan'), device='cuda')
    before = rows.cpu().numpy()
    dev = lambda t: t.cuda().contiguous()
    K.run_rebatch(d, dev(wp), dev(ctrl_sp), dev(temb), dev(semb), dev(meas), dev(flat), levels, proj, rows, rows_ld, ref_re)
    qrows = K.query_rows(d, wp.numpy(), ctrl_sp.numpy(), temb.numpy(), semb.numpy(), meas.numpy(), flat.numpy())
    # the crafted border samples are there: x0 = -1 / x0 + 1 = W on every level (frame 4) and on the coarse ones only (frame 5)
    for b in (4, 5):
        xy = ph['ref_cam'][b, 3, ph['order'][b, 3, :ph['counts'][b, 3]]]
        for l, (h, w) in enumerate(lv):
            px, py = xy[:, 0] * w - 0.5, xy[:, 1] * h - 0.5
            edge = (np.floor(px) == -1).any() and (np.floor(px) + 1 == w).any() and (np.floor(py) == -1).any() and (np.floor(py) + 1 == h).any()
            assert edge == (b == 4 or l == 3), (b, l)
    r_re = K.check_rebatch(rows.cpu().numpy(), before, ref_re.cpu().numpy(), d, ph, qrows, levels, rows_ld)
    print(f'[look] project: largest ref_cam err/bound {r_proj:.4f}; rebatch: largest sample err/bound {r_re:.4f}; '
          f'max_len {int(ph["max_len"][0])}')


# ---------------------------------------------------------------------------------------------------------- DCN columns
def test_dcn_im2col_depth_net_shape(geo):
    """the depth net's DCN: BN = 64 images of 28 x 56 x 512, 4 groups, offsets in an OFF_LD-wide buffer whose pad channels
    hold NaN.  Offsets ~ N(0, 3); images 0 and 1 carry crafted positions (integer, (-1, 0), (H-1, H), exactly -1 and H / W).
    Every column element of every image (1.85 GB in fp32) is compared with the float64 reference, image by image on the GPU."""
    B = 16
    BN, H, W, Cc = B * geo['N'], geo['fH'], geo['fW'], geo['mid']
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(BN, H, W, Cc, generator=gen).cuda()
    off = torch.full((BN, H, W, OFF_LD), float('nan'), device='cuda')
    off[..., :18] = (torch.randn(BN, H, W, 18, generator=gen) * 3).cuda()
    for n in (0, 1):
        K.craft_dcn_offsets(off, H, W, n, gen)
    h, w = K.dcn_positions(off[:2], H, W)
    for what, m in (('h = -1', h == -1), ('h = H', h == H), ('w = W', w == W), ('h in (-1, 0)', (h > -1) & (h < 0)),
                    ('h in (-1, -0.5)', (h > -1) & (h < -0.5)), ('h in (H-1, H)', (h > H - 1) & (h < H)),
                    ('w in (-1, 0)', (w > -1) & (w < 0)), ('w in (W-1, W)', (w > W - 1) & (w < W)), ('integer h', h == torch.round(h))):
        assert int(m.sum()) > 100, what
    col = torch.full((BN * H * W * 9 * Cc,), float('nan'), device='cuda')
    K.run_dcn(x, off, OFF_LD, col, DCN_GROUPS)
    ratio = K.check_dcn(x, off, col, DCN_GROUPS, range(BN))
    print(f'[dcn] largest err/bound {ratio:.4f}')


# ---------------------------------------------------------------------------------------------------------- GRU input
def test_gru_input_columns_and_sentinels(cfg):
    dec = cfg.model['decoder']
    B, T, Hb, Wb = 16, dec['config']['pred_len'], dec['bev_h'], dec['bev_w']
    gen = torch.Generator().manual_seed(8)
    wp, ctrl_sp = torch.randn(B, T, 2, generator=gen), torch.randn(B, T, 4, generator=gen)
    buf = torch.full((B, Hb, Wb, GRU_LD), K.SENT, device='cuda')
    for t in range(T):
        before = buf.cpu().numpy().reshape(B, -1, GRU_LD)
        K.run_gru(wp.cuda(), ctrl_sp.cuda(), t, buf, GRU_COL)
        K.check_gru(buf.cpu().numpy().reshape(B, -1, GRU_LD), before, wp.numpy(), ctrl_sp.numpy(), t, GRU_COL)
    print('[gru_input] exact')
