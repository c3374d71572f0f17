"""The kernel census (tests/kernel_census.py) on the emulated C ABI at the plumbing size: a B = 2 forward passes it unmodified, and
each mutated emulator entry below is rejected by the check meant for it, with a message naming the call (index, entry, layer)."""
import pytest
import torch

import emu_frames
import emu_lib
import kernel_census as KC
from emu_lib import Ptr, _desc, _pix_view


@pytest.fixture
def plumbing(emulated, monkeypatch):
    from oracle.model import EncoderDecoder as Oracle, calibrate_bn, init_oracle_weights
    from thinktwice_b200.config import Config, PLUMBING_CONFIG
    from thinktwice_b200.registry import build_model
    from thinktwice_b200.synthetic import make_batch
    emu_frames.install(emulated)
    emu_lib._by_addr.clear()                                           # tensors earlier emulated forwards left reachable
    cfg = Config.fromfile(PLUMBING_CONFIG)
    for c in (cfg.model.decoder.config, cfg.model.train_cfg, cfg.model.test_cfg):
        c['refine_num'] = 2                                            # two Look layers: the second reads the value tensor at value_coff 256
    o = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'})
    init_oracle_weights(o, 1)
    batch = make_batch(cfg, 2, seed=1, num_points=1500)
    calibrate_bn(o, batch)
    m = build_model(cfg.model)
    m.load_state_dict(o.state_dict())
    m.prepare('cpu', impl=4)

    def run(B, independent=False, census=None):
        m.enable_independent_frames(independent)
        census = KC.install(monkeypatch, census or KC.Census(m.eng))
        m.forward_inference({k: v[:B] for k, v in batch.items()})
        KC.inverse_softplus(m.eng)
        return census
    yield emulated, m, run
    emu_lib._by_addr.clear()


def test_plumbing_b2_forward_passes_the_census(plumbing):
    emu, m, run = plumbing
    for independent in (False, True):
        census = run(2, independent)
        print(census.table())
        census.assert_clean()
        assert census.stats['tt_conv2d_f16s'][0] > 100 and census.stats['tt_split_f16'][0] > 10
        assert {'tt_conv2d', 'tt_copy2d', 'tt_eltwise', 'tt_layernorm'} <= set(census.stats)
        assert ('tt_msda_forward_frames' if independent else 'tt_msda_forward') in census.stats
    # the B = 16 form: convolutions on windows of images, other entries skipped above a working-set cap (1 MB here)
    census = run(2, census=KC.Census(m.eng, outside=False, window=True, cap=1 << 20))
    print(census.table())
    census.assert_clean()
    assert census.skipped and census.stats['tt_conv2d_f16s'][0] > 100


def test_conv_windows_cover_every_bias_residue_and_256_rows():
    from thinktwice_b200.lib import ConvDesc
    d = ConvDesc()
    d.N, d.OH, d.OW, d.bias_n_mod = 64, 64, 128, 4                   # look.value at B = 16: N = B x cams, bias row n % cams
    assert KC.conv_windows(d, True) == [(0, 4), (60, 4)]
    d.N, d.OH, d.OW, d.bias_n_mod = 30, 1, 1, 0                       # a linear of 30 rows: too few to window
    assert KC.conv_windows(d, True) == [(0, 30)]
    d.N = 7056                                                        # a linear of 16 x 21 x 21 rows
    assert KC.conv_windows(d, True) == [(0, 256), (6800, 256)]
    d.N, d.bias_n_mod = 66, 4                                         # N not a multiple of the residue count: the end window runs on
    d.OH = d.OW = 8
    assert KC.conv_windows(d, True) == [(0, 4), (60, 6)]
    assert KC.conv_windows(d, False) == [(0, 66)]


# ---------------------------------------------------------------------------------------------------------- mutants
# Every call is compared with a reference computed from the operands that call received, so a corrupted output upstream does not
# make a downstream call fail: all the mutants run in ONE forward, each on calls of its own, and each failure is attributed to the
# mutant by the call index it names.
class Mutants:
    def __init__(self, emu, monkeypatch):
        self.emu, self.mp = emu, monkeypatch
        self.census = None
        self.hits = {}                                                 # mutant -> call indices it altered
        self.claimed = set()

    def now(self):
        return self.census.calls - 1

    def claim(self, mutant, ok=True, once=True):
        """record the current call for `mutant` when ok and (once: the mutant has no call yet; no other mutant took this call)."""
        i = self.now()
        if not ok or i in self.claimed or (once and self.hits.get(mutant)):
            return False
        self.claimed.add(i)
        self.hits.setdefault(mutant, []).append(i)
        return True

    def wrap(self, entry, make):
        self.mp.setattr(self.emu, entry, make(getattr(self.emu, entry)), raising=False)


def mut_k_slab(M):
    """the last 64-channel K slab of one deep conv dropped (its weights read as zero)."""
    def make(orig):
        def f(d, io, stream):
            dd = _desc(d)
            if M.claim('k_slab_dropped', dd.KH * dd.KW * dd.Cin >= 256 and dd.Cin % 64 == 0):
                taps, c8 = dd.KH * dd.KW, -(-dd.Cin // 8) * 8
                w = io.w_split.flat()[:2 * dd.Cout * taps * c8].clone().view(2, dd.Cout, taps, c8)
                w[:, :, -1, dd.Cin - 64:dd.Cin] = 0
                io.w_split = Ptr(w)
            return orig(d, io, stream)
        return f
    M.wrap('tt_conv2d_f16s', make)


def mut_past_concat(M):
    """one channel written past a concat slice: the next channel of the first output pixel, inside the row pitch."""
    def make(orig):
        def f(d, io, stream):
            dd = _desc(d)
            h = M.claim('channel_past_concat_slice', bool(io.y) and dd.y_ld > dd.Cout)
            rc = orig(d, io, stream)
            if h:
                io.y.flat()[dd.Cout] += 1.0
            return rc
        return f
    M.wrap('tt_conv2d_f16s', make)


def mut_lo_unwritten(M):
    """the lo' plane left as it was."""
    def make(orig):
        def f(d, io, stream):
            h = M.claim('lo_plane_unwritten', bool(io.y_split))
            keep = io.y_split.t.clone() if h else None
            rc = orig(d, io, stream)
            if h:
                n = io.y_split.t.numel() // 2
                io.y_split.t.reshape(-1)[n:] = keep.reshape(-1)[n:]
            return rc
        return f
    M.wrap('tt_conv2d_f16s', make)


def mut_bias_n_mod(M):
    """the per-image bias table ignored: row 0 for every image."""
    def make(orig):
        def f(d, io, stream):
            dd = _desc(d)
            if not M.claim('bias_n_mod_ignored', dd.bias_n_mod > 1):
                return orig(d, io, stream)
            k, dd.bias_n_mod = dd.bias_n_mod, 0
            try:
                return orig(d, io, stream)
            finally:
                dd.bias_n_mod = k
        return f
    M.wrap('tt_conv2d_f16s', make)


def mut_res_up2(M):
    """RES_UP2 taken as same-size: output pixel (y, x) adds residual pixel (y, x) (clamped to the residual map)."""
    def make(orig):
        def f(d, io, stream):
            dd = _desc(d)
            if not M.claim('res_up2_as_same_size', dd.res_mode == 2):
                return orig(d, io, stream)
            ih, iw = torch.arange(dd.OH).clamp(max=dd.res_H - 1), torch.arange(dd.OW).clamp(max=dd.res_W - 1)
            io2 = emu_lib.IO()
            io2.__dict__.update(io.__dict__)
            n = dd.N * dd.OH * dd.OW * dd.Cout
            if io.res:
                io2.res = Ptr(_pix_view(io.res, dd.N, dd.res_H, dd.res_W, dd.res_ld, C=dd.Cout)[:, ih][:, :, iw].contiguous())
            else:
                planes = torch.empty(2, n, dtype=torch.float16)
                for i, pl in enumerate((0, io.res_plane)):
                    v = _pix_view(Ptr(io.res_split.t, io.res_split.off + pl), dd.N, dd.res_H, dd.res_W, dd.res_ld, C=dd.Cout)
                    planes[i] = v[:, ih][:, :, iw].reshape(-1)
                io2.res_split, io2.res_plane = Ptr(planes), n
            saved = dd.res_mode, dd.res_ld
            dd.res_mode, dd.res_ld = 1, dd.Cout
            try:
                return orig(d, io2, stream)
            finally:
                dd.res_mode, dd.res_ld = saved
        return f
    M.wrap('tt_conv2d_f16s', make)


def mut_value_coff(M):
    """the MSDA reads the first layer's value projection whatever value_coff says."""
    def make(orig):
        def f(d, value, off, logits, ref, max_len, out, stream):
            dd = _desc(d)
            if not M.claim('value_coff_ignored', dd.value_coff != 0):
                return orig(d, value, off, logits, ref, max_len, out, stream)
            k, dd.value_coff = dd.value_coff, 0
            try:
                return orig(d, value, off, logits, ref, max_len, out, stream)
            finally:
                dd.value_coff = k
        return f
    M.wrap('tt_msda_forward', make)


def mut_eltwise_swap(M):
    """eltwise op 2 with b and c swapped: (1 - a) c + a b."""
    def make(orig):
        def f(op, act, a, a_ld, b, b_ld, c, c_ld, y, y_ld, rows, cols, stream):
            if M.claim('eltwise_op2_b_c_swapped', emu_lib._v(op) == 2):
                b, b_ld, c, c_ld = c, c_ld, b, b_ld
            return orig(op, act, a, a_ld, b, b_ld, c, c_ld, y, y_ld, rows, cols, stream)
        return f
    M.wrap('tt_eltwise', make)


def mut_upsample_half_pixel(M):
    """the 2x bilinear upsample (both entries) with align_corners=False."""
    emu = M.emu

    def up(x, N, H, W, Cc):
        o = torch.nn.functional.interpolate(_pix_view(x, N, H, W, Cc).permute(0, 3, 1, 2).float(), scale_factor=2, mode='bilinear',
                                            align_corners=False)
        return o.permute(0, 2, 3, 1).contiguous()

    def f(x, y, N, H, W, Cc, stream):
        M.claim('upsample_align_corners_false', once=False)
        emu.launches += 1
        o = up(x, N, H, W, Cc)
        y.flat()[:o.numel()].copy_(o.reshape(-1))
        return 0

    def fs(x, y_split, y_plane, N, H, W, Cc, stream):
        M.claim('upsample_align_corners_false', once=False)
        emu.launches += 1
        o = up(x, N, H, W, Cc)
        hi, lo = emu_lib._split_f16(o)
        y_split.flat()[:o.numel()].copy_(hi.reshape(-1))
        Ptr(y_split.t, y_split.off + emu_lib._v(y_plane)).flat()[:o.numel()].copy_(lo.reshape(-1))
        return 0
    M.wrap('tt_upsample2x_bilinear_ac', lambda orig: f)
    M.wrap('tt_upsample2x_bilinear_ac_split', lambda orig: fs)


def mut_se_pool_mean(M):
    """se_pool as the mean only."""
    emu = M.emu

    def f(x, s, N, HW, Cc, stream):
        M.claim('se_pool_mean_only', once=False)
        emu.launches += 1
        xv = x.flat()[:N * HW * Cc].view(N, HW, Cc)
        s.flat()[:N * Cc].view(N, Cc).copy_(xv.double().mean(1))
        return 0
    M.wrap('tt_se_pool', lambda orig: f)


# mutant -> (installer, the entry its failure names, the words of the check that must reject it)
MUTANTS = {
    'k_slab_dropped': (mut_k_slab, 'tt_conv2d_f16s', 'beyond the bound'),
    'channel_past_concat_slice': (mut_past_concat, 'tt_conv2d_f16s', 'write outside the destination'),
    'lo_plane_unwritten': (mut_lo_unwritten, 'tt_conv2d_f16s', 'io.y_split:'),
    'bias_n_mod_ignored': (mut_bias_n_mod, 'tt_conv2d_f16s', 'beyond the bound'),
    'res_up2_as_same_size': (mut_res_up2, 'tt_conv2d_f16s', 'beyond the bound'),
    'value_coff_ignored': (mut_value_coff, 'tt_msda_forward', 'beyond the bound'),
    'eltwise_op2_b_c_swapped': (mut_eltwise_swap, 'tt_eltwise', 'beyond the bound'),
    'upsample_align_corners_false': (mut_upsample_half_pixel, 'tt_upsample2x_bilinear_ac', 'beyond the bound'),
    'se_pool_mean_only': (mut_se_pool_mean, 'tt_se_pool', 'beyond the bound'),
}


def test_each_mutant_is_rejected_by_its_check_and_named(plumbing, monkeypatch):
    emu, m, run = plumbing
    M = Mutants(emu, monkeypatch)
    for install, _, _ in MUTANTS.values():
        install(M)
    M.census = KC.Census(m.eng)
    run(1, census=M.census)
    fails = M.census.failures
    by_call = {}
    for f in fails:
        by_call.setdefault(int(f.split()[1].lstrip('#')), []).append(f)
    for mutant, (_, entry, what) in MUTANTS.items():
        assert M.hits.get(mutant), f'{mutant}: the plumbing forward makes no call it applies to'
        msgs = [f for i in M.hits[mutant] for f in by_call.get(i, [])]
        print(mutant, '->', msgs[0] if msgs else None)
        assert any(entry in f and what in f for f in msgs), (mutant, msgs)
        assert all('[?]' not in f and '[outside the arena]' not in f for f in msgs), msgs
    hit = {i for v in M.hits.values() for i in v}
    assert set(by_call) <= hit, [f for i, v in by_call.items() if i not in hit for f in v]      # nothing else fails
