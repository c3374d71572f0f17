"""The checker of tests/conv_contract.py on the emulated C ABI (tests/emu_lib.py): the small cases of the descriptor matrix pass it,
the case list reaches every regime of tt_conv2d_f16s at an H100's 132 SMs, and each seeded bug below is rejected by the check meant
for it."""
import math

import pytest
import torch

import conv_contract as K
import emu_lib
from emu_lib import Ptr, _desc, _pix_view, _res_view, conv_store, y_region

CPU_F16S = [c for c in K.f16s_cases() if c.cpu]
CPU_POINTWISE = [c for c in K.pointwise_cases() if c.cpu]


def run(emu, c, kind='f16s'):
    return K.run_case(K.Buffers(K.Backend(emu, False), c, kind))


def named(name):
    return next(c for c in K.f16s_cases() if c.name == name)


def test_the_case_list_reaches_every_regime_at_132_sms():
    table = K.regime_table(K.f16s_cases(), 132)
    assert K.REQUIRED_REGIMES <= set(table), K.REQUIRED_REGIMES - set(table)
    # the schedules the knobs force (the GPU file asserts their launch counts against tt_launch_count)
    assert K.schedule(named('splitk'), 132).launches == 2 and K.schedule(named('splitk-finish'), 132).launches == 3
    assert K.schedule(named('splitk'), 132, K.NO_SPLITK).launches == 1
    assert K.schedule(named('wide-flat'), 132).wide and not K.schedule(named('wide-flat'), 132, K.BN64).wide
    assert K.schedule(named('wide-tiled'), 132, K.reserve(132)).ctas == 1


def test_fold_aware_bound_is_the_census_bound_at_the_default_fold():
    from thinktwice_b200.lib import ConvDesc
    from kernel_census import conv_c
    d = ConvDesc()
    for k in (8, 72, 128, 129, 576, 4608):
        assert conv_c('tt_conv2d_f16s', d, k) == 72 + 4 * math.ceil(k / 128)
        assert conv_c('tt_conv2d_f16s', d, k, 1) == 40 + 4 * math.ceil(k / 64)
        assert conv_c('tt_conv2d_f16s', d, k, 4) == 136 + 4 * math.ceil(k / 256)


@pytest.mark.parametrize('c', CPU_F16S + CPU_POINTWISE, ids=lambda c: c.name)
def test_the_emulated_abi_passes(c):
    worst, found, _ = run(emu_lib.Emu(), c, 'pointwise' if c in CPU_POINTWISE else 'f16s')
    assert not found, '\n'.join(f.text for f in found)
    assert worst < 1


# ---------------------------------------------------------------------------------------------------------- seeded bugs
class Seeded(emu_lib.Emu):
    """the emulated tt_conv2d_f16s with one bug: mutate(emu, d, io) runs the call its buggy way."""

    def __init__(self, mutate):
        super().__init__()
        self.mutate = mutate

    def tt_conv2d_f16s(self, d, io, stream):
        return self.mutate(super().tt_conv2d_f16s, _desc(d), io)


def drop_last_k_slab(call, d, io):
    """the last 64-channel K slab of every tap skipped (a Cin tail lost)."""
    w = io.w_split.t.clone()
    c8 = -(-d.Cin // 8) * 8
    n = 2 * d.Cout * d.KH * d.KW * c8
    w[io.w_split.off:io.w_split.off + n].view(2, d.Cout, d.KH * d.KW, c8)[..., (d.Cin - 1) // 64 * 64:] = 0
    io.w_split = Ptr(w, io.w_split.off)
    return call(d, io, None)


def write_ld_padding(call, d, io):
    """one store past Cout into the y_ld padding."""
    rc = call(d, io, None)
    io.y.t[io.y.off + d.y_coff + d.Cout] = 0.0
    return rc


def wrong_phase(call, d, io):
    """a scatter phase written at the other oy_add."""
    d.oy_add = 1 - d.oy_add
    try:
        return call(d, io, None)
    finally:
        d.oy_add = 1 - d.oy_add


def lo_plane_off_by_one(call, d, io):
    """the lo' half of the first output element one unit in the last place off."""
    rc = call(d, io, None)
    t = io.y_split.t.view(torch.int16)
    t[io.y_split.off + io.y_plane + d.y_coff] += 1
    return rc


def bias_row_n(call, d, io):
    """the bias row taken as n instead of n % bias_n_mod (a table of N rows)."""
    k = d.bias_n_mod
    d.bias_n_mod = d.N
    try:
        return call(d, io, None)
    finally:
        d.bias_n_mod = k


def _restore(d, io, out):
    conv_store(d, io.y, io.y_split, io.y_plane, out.float())


def up2_rounded(call, d, io):
    """the UP2 residual's source pixel rounded, floor(o res / O + 1/2), instead of floored."""
    rc = call(d, io, None)
    r = _res_view(d, io.res, io.res_split, io.res_plane, d.N, d.res_H, d.res_W, d.res_ld, d.res_coff)
    pick = lambda O, R, f: torch.clamp(f(torch.arange(O, dtype=torch.float64) * R / O).long(), max=R - 1)
    fh, fw = pick(d.OH, d.res_H, torch.floor), pick(d.OW, d.res_W, torch.floor)
    rh, rw = pick(d.OH, d.res_H, lambda v: torch.floor(v + 0.5)), pick(d.OW, d.res_W, lambda v: torch.floor(v + 0.5))
    assert not (torch.equal(fh, rh) and torch.equal(fw, rw))
    y = y_region(d, io.y).double() + r[:, rh][:, :, rw] - r[:, fh][:, :, fw]
    _restore(d, io, y)
    return rc


def nan_pad_channel(call, d, io):
    """channel Cin of each input pixel (a NaN pad channel of x_ld) read into the sum of its 1x1 output."""
    rc = call(d, io, None)
    assert d.KH == d.KW == 1 and d.stride == 1 and d.x_ld > d.Cin
    pad = _pix_view(io.x_split, d.N, d.H, d.W, d.x_ld, C=d.Cin + 1)[..., d.Cin:].double()
    _restore(d, io, y_region(d, io.y).double() + 0.0 * pad)
    return rc


SEEDED = [
    ('drop-last-k-slab', drop_last_k_slab, 'flat-m-tail', 'value'),
    ('write-ld-padding', write_ld_padding, 'up2-odd-concat', 'outside'),
    ('wrong-oy_add', wrong_phase, 'k2s2-scatter', 'outside'),
    ('lo-plane-ulp', lo_plane_off_by_one, 'flat-m-tail', 'planes'),
    ('bias-row-n', bias_row_n, 'pad3-bias-table', 'value'),
    ('up2-rounded', up2_rounded, 'up2-odd-concat', 'value'),
    ('nan-pad-channel', nan_pad_channel, 'flat-m-tail', 'value'),
]


@pytest.mark.parametrize('bug,mutate,name,check', SEEDED, ids=[s[0] for s in SEEDED])
def test_a_seeded_bug_is_rejected_by_its_check(bug, mutate, name, check):
    _, found, _ = run(Seeded(mutate), named(name))
    print(bug, [(f.check, f.text) for f in found])
    assert check in {f.check for f in found}, found
