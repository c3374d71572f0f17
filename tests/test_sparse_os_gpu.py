"""Output-stationary sparse convolution (tt_sparse_conv_os_f16s) on neighbour tables the encoder's clouds do not produce: tiles
whose rows all lack the same taps, rows with only the centre tap, a tile that uses no tap at all, a count that ends inside a tile
with stale table rows and NaN input rows past it, and the 128- and 32-column outputs.  The kernel walks only the taps (tap pairs
when Cin = 32) that some row of a 128-row tile uses and runs 128-column tiles for Cout >= 128; every case is compared with a
float64 reference within the per-element bound of tests/lidar_sparse_checks.py, and the rows past the count must keep their
sentinels."""
import numpy as np
import pytest
import torch

import lidar_sparse_checks as L

pytestmark = pytest.mark.gpu
FORCE_BN64 = 0x400000
SUBM = ((3, 3, 3), (1, 1, 1), (1, 1, 1), True)
WIDTHS = [(32, 64), (64, 64), (64, 32), (32, 128), (128, 128)]


@pytest.fixture(scope='module')
def eng():
    from thinktwice_b200.engine import Engine
    return Engine('cuda:0', impl=4)


def split_rows(x):
    """[2][rows * C] split planes of fp32 rows x (rows, C) on the device, and their float64 value on the host."""
    from thinktwice_b200.weights import f16s_split
    hi, lo = f16s_split(x.cpu())
    return torch.stack([hi.reshape(-1), lo.reshape(-1)]).cuda(), L.split_round(x).numpy()


def operands(n_in, cin, cout, kvol, seed, cap_in=None):
    """input rows (n_in real rows, NaN rows up to cap_in), weights (Cout, kvol, Cin) and bias."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(cap_in or n_in, cin, generator=g)
    x[n_in:] = float('nan')
    w = torch.randn(cout, kvol, cin, generator=g) / np.sqrt(cin * kvol)
    b = torch.randn(cout, generator=g) * 0.1
    x_s, x64 = split_rows(x)
    return x_s, x64[:n_in], w, b


def ref_nbr(x64, nbr, w):
    """float64 conv over a neighbour table nbr (rows, kvol): the dict lidar_sparse_checks.expected() takes."""
    Cout, kvol, Cin = w.shape
    w = w.double().numpy()
    acc, mag = np.zeros((len(nbr), Cout)), np.zeros((len(nbr), Cout))
    for t in range(kvol):
        r = np.nonzero(nbr[:, t] >= 0)[0]
        acc[r] += x64[nbr[r, t]] @ w[:, t].T
        mag[r] += np.abs(x64[nbr[r, t]]) @ np.abs(w[:, t]).T
    return dict(acc=acc, mag=mag, K=Cin * (nbr >= 0).sum(1))


def table_rule(nbr, count, cap):
    """a rulebook dict for Engine.sparse_conv from a host neighbour table nbr (cap, kvol)."""
    return dict(nbr=torch.as_tensor(nbr, dtype=torch.int32).cuda(), count=torch.tensor([count], dtype=torch.int32).cuda(), cap=cap,
                kvol=nbr.shape[1])


def check(out, out_s, y, bnd, n, cout, name):
    g, r = L.check_conv(out.cpu().numpy()[:n], y, bnd, name)
    g2, r2 = L.check_conv(L.planes_value(out_s, n, cout), y, bnd + L.SPLIT * np.abs(y), f'{name} planes')
    L.check_untouched(out, n, cout, name)
    L.check_untouched(out_s, n, cout, f'{name} planes')
    print(f'{name}: max err {max(g, g2):.2e} of max |ref|, {max(r, r2):.3f} of the bound')
    return out.cpu().numpy()[:n]


def site_case(eng, coords, shape, cin, cout, seed, name):
    """SubM 3x3x3 conv over the sites `coords` (n, 4) through the product's rulebook; returns (rule, tap occupancy)."""
    n = len(coords)
    c = torch.as_tensor(coords, dtype=torch.int32).cuda()
    rb = L.rulebook(eng, name, 1, c, torch.tensor([n], dtype=torch.int32).cuda(), n, shape, *SUBM, 'nbr')
    ref_rb = L.ref_rulebook(coords, shape, *SUBM)
    L.check_rulebook(L.rulebook_host(rb), ref_rb, name)
    x_s, x64, w, b = operands(n, cin, cout, 27, seed)
    ref = L.ref_sparse_conv(x64, coords, shape, 1, w.numpy(), *SUBM, ref_rb)
    y, bnd = L.expected(ref, b.numpy(), act=1)
    out, out_s = L.run_conv(eng, rb, x_s, L.pack(w.cuda(), b.cuda()), act=1)
    check(out, out_s, y, bnd, n, cout, name)
    return ref_rb['nbr'] >= 0


@pytest.mark.parametrize('cin,cout', WIDTHS)
def test_every_row_of_the_tiles_lacks_the_same_taps(eng, cin, cout):
    # 20 x 20 sites on one z plane: no row has a neighbour under the 18 taps with dz != 0 (and, at Cin = 32, tap pairs 0..3 and
    # 9..12 are empty for every tile)
    yy, xx = np.meshgrid(np.arange(4, 24), np.arange(6, 26), indexing='ij')
    coords = np.stack([np.zeros(400), np.full(400, 3), yy.ravel(), xx.ravel()], 1).astype(np.int64)
    occ = site_case(eng, coords, (8, 32, 32), cin, cout, 1, f'plane {cin}->{cout}')
    dz = np.arange(27) // 9
    assert not occ[:, dz != 1].any() and occ[:, dz == 1].all(0).sum() == 1 and occ[:, 13].all()


@pytest.mark.parametrize('cin,cout', WIDTHS)
def test_rows_with_only_the_centre_tap(eng, cin, cout):
    # sites two cells apart on every axis: each row's only neighbour is itself
    z, y, x = np.meshgrid(np.arange(0, 12, 2), np.arange(0, 16, 2), np.arange(0, 16, 2), indexing='ij')
    coords = np.stack([np.zeros(z.size), z.ravel(), y.ravel(), x.ravel()], 1).astype(np.int64)
    occ = site_case(eng, coords, (12, 16, 16), cin, cout, 2, f'isolated {cin}->{cout}')
    assert occ[:, 13].all() and not np.delete(occ, 13, 1).any()


@pytest.mark.parametrize('cout', [64, 128])
def test_a_down_conv_tile_that_uses_no_tap_writes_bias_activation_and_residual(eng, cout):
    # a 27-tap table of 400 output rows where rows 128..255 (one whole tile) have no input at all: that tile's K walk is empty,
    # its rows are act(bias + residual)
    g = np.random.default_rng(3)
    n_in, n, cin = 900, 400, 64
    nbr = np.where(g.random((n, 27)) < 0.3, g.integers(0, n_in, (n, 27)), -1)
    nbr[128:256] = -1
    x_s, x64, w, b = operands(n_in, cin, cout, 27, 4)
    res = torch.randn(n, cout, generator=torch.Generator().manual_seed(5))
    y, bnd = L.expected(ref_nbr(x64, nbr, w), b.numpy(), res=res.double().numpy(), act=1)
    rb = table_rule(nbr, n, n)
    pw = L.pack(w.cuda(), b.cuda())
    out, out_s = L.run_conv(eng, rb, x_s, pw, act=1, res=res.cuda())
    got = check(out, out_s, y, bnd, n, cout, f'empty tile ->{cout}')
    np.testing.assert_allclose(got[128:256], np.maximum(b.numpy() + res.numpy()[128:256], 0), rtol=1e-6, atol=1e-6)
    # the same with the residual given as split planes
    r_s, r64 = split_rows(res)
    y, bnd = L.expected(ref_nbr(x64, nbr, w), b.numpy(), res=r64, act=1)
    out, out_s = L.run_conv(eng, rb, x_s, pw, act=1, res_s=r_s)
    check(out, out_s, y, bnd, n, cout, f'empty tile ->{cout} split residual')


@pytest.mark.parametrize('cin,cout', WIDTHS)
def test_a_count_that_ends_inside_a_tile_ignores_the_stale_rows_past_it(eng, cin, cout):
    # capacity 512 rows, count 200: rows 200.. of the table are stale and point at NaN input rows (and at real ones), as an
    # earlier, larger cloud leaves them; they must neither be gathered into the live rows nor written
    g = np.random.default_rng(6)
    n_in, cap_in, n, cap = 700, 1000, 200, 512
    nbr = np.where(g.random((cap, 27)) < 0.4, g.integers(0, n_in, (cap, 27)), -1)
    nbr[n:] = np.where(g.random((cap - n, 27)) < 0.5, g.integers(n_in, cap_in, (cap - n, 27)), g.integers(0, n_in, (cap - n, 27)))
    x_s, x64, w, b = operands(n_in, cin, cout, 27, 7, cap_in=cap_in)
    y, bnd = L.expected(ref_nbr(x64, nbr[:n], w), b.numpy(), act=1)
    out, out_s = L.run_conv(eng, table_rule(nbr, n, cap), x_s, L.pack(w.cuda(), b.cuda()), act=1)
    check(out, out_s, y, bnd, n, cout, f'count mid-tile {cin}->{cout}')


# knobs the output-stationary kernel reads besides 0x200000 / 0x400000: the register fold every 4 / 1 executed stages, and an SM
# reserve that leaves one CTA to walk every tile ('one-cta': bits 8..15 = SMs - 1, from the device)
KNOBS = [(0, ''), (0x20000, '-fold4'), (0x40000, '-fold1'), ('one-cta', '-one-cta')]


@pytest.mark.parametrize('cin,cout,knobs', [pytest.param(ci, co, k, id=f'{ci}-{co}{tag}') for k, tag in KNOBS for ci, co in WIDTHS])
def test_wide_and_narrow_outputs_on_a_random_table_with_more_tiles_than_sms(eng, cin, cout, knobs):
    # 20000 rows (157 tiles) of a 27-tap table with mixed occupancy; Cout = 128 runs 128-column tiles, and must agree with the
    # 64-column tiles debug bit 0x400000 forces; Cout = 32 leaves half of a 64-column tile dead.  The bound does not depend on the fold
    if knobs == 'one-cta':
        knobs = (torch.cuda.get_device_properties(0).multi_processor_count - 1) << 8
    g = np.random.default_rng(8)
    n_in, n = 30000, 20000
    dens = np.repeat(g.choice([0.0, 0.05, 0.3, 0.9], n // 128 + 1), 128)[:n, None]
    nbr = np.where(g.random((n, 27)) < dens, g.integers(0, n_in, (n, 27)), -1)
    x_s, x64, w, b = operands(n_in, cin, cout, 27, 9)
    y, bnd = L.expected(ref_nbr(x64, nbr, w), b.numpy(), act=1)
    rb, pw = table_rule(nbr, n, n), L.pack(w.cuda(), b.cuda())
    out, out_s = L.run_conv(eng, rb, x_s, pw, act=1, flags=knobs)
    a = check(out, out_s, y, bnd, n, cout, f'random {cin}->{cout} knobs {knobs:#x}')
    out, out_s = L.run_conv(eng, rb, x_s, pw, act=1, flags=knobs | FORCE_BN64)
    f = check(out, out_s, y, bnd, n, cout, f'random {cin}->{cout} knobs {knobs:#x} BN 64')
    L.check_conv(a, f.astype(np.float64), 2 * bnd, f'random {cin}->{cout} BN 128 vs 64')
