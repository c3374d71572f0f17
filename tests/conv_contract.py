"""The dense convolution contract (include/tt_b200.h (2) / (2b)) as a fixed, seeded descriptor matrix — TEST HARNESS ONLY.

Every case calls the C ABI directly (tt_conv2d_f16s, tt_pointwise_f16s, tt_conv2d), not through Engine, so it reaches descriptors the
engine never builds.  Each case names the corner of the contract it exercises.  Buffers are laid out so that a kernel which reads or
writes outside its contract is caught:
  * every input buffer holds NaN (fp32) or a NaN half (both split planes) wherever the descriptor does not read: channels in
    [Cin, x_ld) and before x_coff, pixels past W within x_hstride, rows between images within x_nstride, the gap between the two planes
    and a guard region before and after the buffer (the row-packed stem form reads whole rows: only its guards and gaps are NaN);
  * every output buffer, both planes included, starts filled with a sentinel, guards included.
The checks follow the kernel census (tests/kernel_census.py):
  * value: each output element within act_bound(conv_c(...)) of emu_lib.conv_ref(..., magnitude=True) in float64;
  * planes: the split planes bitwise _split_f16 of the same call's fp32 output, or, for a planes-only output, their decoded value
    within the bound + SPLIT |y| + SPLIT_ABS;
  * outside: every element outside y_region bitwise unchanged (other scatter phases, concat neighbours, y_ld padding, y_nstride gaps,
    rows past *m_count, guards);
  * saturation: tt_f16s_saturation_count unchanged; launches: the tt_launch_count delta the host schedule implies (GPU only).

The host decisions of tt_conv2d_f16s (flat / tiled A operand and tile shape, 64- / 128-column tiles, split-K, finish kernel, fold
length, persistent grid) are restated in `schedule`, so that the case list can be shown to reach every regime at a given SM count.
The same module drives the emulated ABI (tests/emu_lib.py) on the CPU, where seeded bugs show that each check rejects what it is for.
"""
import ctypes as C
import math
from types import SimpleNamespace

import torch

from emu_lib import IO, NULL, Ptr, _split_f16, conv_ref, y_region
from kernel_census import SPLIT, SPLIT_ABS, act_bound, conv_c

GUARD = 64                      # elements of poison / sentinel before and after every buffer (a 16-byte multiple for halves and fp32)
PLANE_GAP = 24                  # halves between the end of a hi plane's body and its lo' plane (a multiple of 8)
Y_SENTINEL = -1234.5            # fp32 outputs start as this ...
H_SENTINEL = -0.3125            # ... split-plane outputs as this half
NAN = float('nan')

ERR_INVALID, ERR_UNSUPPORTED = -1, -3
NO_SPLITK, FOLD4, FOLD1, BN64, SPARSE_ONE_TAP = 128, 0x20000, 0x40000, 0x400000, 0x200000
KNOWN_KNOBS = NO_SPLITK | 0xFF00 | FOLD4 | FOLD1 | SPARSE_ONE_TAP | BN64


def reserve(num_sms):
    """debug bits 8..15 leaving all SMs but one free: one CTA walks every work item."""
    return (num_sms - 1) << 8


def knob_matrix(num_sms):
    """(label, tt_debug_set flags): every bit the dense tensor-core convolutions read."""
    one = reserve(num_sms)
    return [('default', 0), ('no-splitk', NO_SPLITK), ('bn64', BN64), ('fold4', FOLD4), ('fold1', FOLD1), ('one-cta', one),
            ('bn64+fold4+one-cta', BN64 | FOLD4 | one)]


def fold_stages(flags):
    """K stages (64 halves each) the f16s / 3xTF32 register accumulator runs before it is folded into the fp32 sums."""
    return 1 if flags & FOLD1 else 4 if flags & FOLD4 else 2


# ---------------------------------------------------------------------------------------------------------- cases
def case(name, corner, **kw):
    """one descriptor of the matrix; the fields not given take the defaults below.  Geometry: K = KH x KW taps, OH / OW from H, W,
    pad, dil and stride.  Layout: x_ld / y_ld (None = Cin rounded up to 8 / Cout), x_coff, row_gap (pixels past W in each input row),
    img_gap (elements between input images), y_gap (between output images), y_coff.  Epilogue: bias (None, 'vec' or a table of
    bias_n_mod rows), res / res2 (None, 'f32' or 'split'), res_mode, res_hw (UP2 residual map size), act, out ('both', 'f32',
    'planes').  scatter: the four k2s2 phases into one buffer.  packed: the row-packed stem form (x_ld < Cin).  m_count: rows of
    an impl 1 call.  junk: taps / M set although a dense call ignores them."""
    c = dict(name=name, corner=corner, N=1, H=8, W=8, Cin=16, Cout=32, KH=1, KW=1, stride=1, pad=0, dil=1, groups=1, x_ld=None,
             x_coff=0, row_gap=0, img_gap=0, y_ld=None, y_coff=0, y_gap=0, scatter=False, act=0, bias=None, bias_n_mod=0,
             res=None, res_mode=1, res_hw=None, res_ld=None, res_coff=0, res2=None, res2_ld=None, res2_coff=0, out='both',
             packed=False, m_count=None, junk=False, seed=0, cpu=False)
    unknown = set(kw) - set(c)
    assert not unknown, unknown
    c.update(kw)
    c = SimpleNamespace(**c)
    c.seed = c.seed or sum(map(ord, name))
    c.x_ld = c.x_ld or -(-(c.x_coff + c.Cin) // 8) * 8
    c.y_ld = c.y_ld or c.y_coff + c.Cout
    c.OH = (c.H + 2 * c.pad - c.dil * (c.KH - 1) - 1) // c.stride + 1
    c.OW = (c.W + 2 * c.pad - c.dil * (c.KW - 1) - 1) // c.stride + 1
    c.res_ld = c.res_ld or c.res_coff + c.Cout
    c.res2_ld = c.res2_ld or c.res2_coff + c.Cout
    return c


def f16s_cases():
    """the descriptors tt_conv2d_f16s runs (their fp32 twins go through tt_conv2d).  cpu=True: small enough for the emulated ABI."""
    return [
        case('flat-m-tail', '1x1 flat A operand, 130 pixels (an M tail of 2 rows), Cin 72 (a second K slab of 8), Cout 40 (an N '
             'tail), x_ld 88 > Cin with the channels at x_coff 8, bias, relu, both outputs',
             H=10, W=13, Cin=72, x_coff=8, x_ld=88, Cout=40, bias='vec', act=1, cpu=True),
        case('cin8-pad', '3x3 tiled, Cin 13 (Cin8 = 16 zero-padded weights, channels 13..15 of x NaN), rows with 3 NaN pixels past W '
             'and 40 NaN elements between images, gelu, fp32 only; taps / M set to values a dense call ignores',
             N=2, H=9, W=11, KH=3, KW=3, pad=1, Cin=13, Cout=36, row_gap=3, img_gap=40, act=2, out='f32', junk=True, cpu=True),
        case('stride2-odd', '3x3 stride 2 on 15 x 17 (odd H / W), sigmoid, planes-only output',
             H=15, W=17, KH=3, KW=3, pad=1, stride=2, Cin=32, Cout=64, act=3, out='planes', cpu=True),
        case('dilated-halo', '3x3 dilation 6 (a 12-pixel halo, larger than the 8 x 8 map and its tile), pad 6, softplus',
             N=2, H=8, W=8, KH=3, KW=3, pad=6, dil=6, Cin=16, Cout=32, act=4, bias='vec'),
        case('pad3-bias-table', '3x3 pad 3 > (k - 1) / 2, a bias table of 3 rows over N = 4 images (row n % 3), gaps of 20 floats '
             'between output images, clamped softplus',
             N=4, H=7, W=10, KH=3, KW=3, pad=3, Cin=24, Cout=28, bias='table', bias_n_mod=3, y_gap=20, act=5, cpu=True),
        case('up2-odd-concat', '1x1, RES_UP2 from a 5 x 6 fp32 map onto a 9 x 11 output (floor(o res / O)) at res_coff 4 of '
             'res_ld 40, res2 as split planes at res2_coff 4 of 36, output at y_coff 8 of y_ld 48 (a concat slice), both outputs',
             N=2, H=9, W=11, Cin=24, Cout=32, res='f32', res_mode=2, res_hw=(5, 6), res_coff=4, res_ld=40, res2='split',
             res2_coff=4, res2_ld=36, y_coff=8, y_ld=48, cpu=True),
        case('same-res-split', '3x3, a SAME residual as split planes at res_coff 8 of 72, res2 in fp32, relu, both outputs',
             H=12, W=12, KH=3, KW=3, pad=1, Cin=40, Cout=64, res='split', res_coff=8, res_ld=72, res2='f32', act=1),
        case('k2s2-scatter', 'a k2s2 transposed conv: four 1x1 calls scattered into one 2H x 2W buffer (oy_mul = ox_mul = 2), bias, '
             'both outputs',
             N=2, H=5, W=7, Cin=32, Cout=48, bias='vec', scatter=True, cpu=True),
        case('stem-packed', 'the row-packed stem: x_ld 8 < Cin 56 (7 pixels of 8 channels per K slab), 7 x 1 taps, stride 2 over a '
             '26 x 28 padded frame, relu, both outputs',
             N=2, H=26, W=22, Cin=56, x_ld=8, KH=7, KW=1, stride=2, packed=True, Cout=64, act=1, bias='vec', cpu=True),
        case('splitk', 'split-K without a finish kernel: 2 tiles, Cin 96 (K tail of 32 in every tap), SAME fp32 residual, bias, '
             'fp32 only',
             H=16, W=16, KH=3, KW=3, pad=1, Cin=96, Cout=64, res='f32', bias='vec', out='f32'),
        case('splitk-finish', 'split-K with a finish kernel (relu, planes): Cout 96 on 64-column tiles (an N tail of 32), res2 as '
             'split planes',
             H=12, W=12, KH=3, KW=3, pad=1, Cin=64, Cout=96, res2='split', act=1),
        case('wide-flat', '128-column tiles on the flat path: 144 M tiles, Cout 96 (one partial 128-column tile), bias, relu',
             N=2, H=96, W=96, Cin=24, Cout=96, bias='vec', act=1),
        case('wide-tiled', '128-column tiles on the tiled path: 3x3 over 2 x 96 x 96, Cout 192 (a full and a half tile), SAME fp32 '
             'residual, fp32 only',
             N=2, H=96, W=96, KH=3, KW=3, pad=1, Cin=16, Cout=192, res='f32', out='f32'),
    ]


def pointwise_cases():
    """tt_pointwise_f16s over its Cin, Cout <= 64 range."""
    return [
        case('pw-thin', 'Cin 13 (channels 13..15 of x NaN), Cout 12 (one 16-column pass, a partial one), sigmoid, fp32 only',
             N=2, H=9, W=15, Cin=13, Cout=12, act=3, out='f32', cpu=True),
        case('pw-64', 'Cin 64, Cout 64 (two 32-column passes), bias, relu, both outputs at y_coff 8 of y_ld 80',
             H=12, W=20, Cin=64, Cout=64, bias='vec', act=1, y_coff=8, y_ld=80, cpu=True),
        case('pw-planes', 'Cin 40, Cout 16, planes only at y_coff 4 of y_ld 20 (rows start 8-byte, not 16-byte, aligned), gelu',
             N=3, H=7, W=11, Cin=40, Cout=16, act=2, out='planes', y_coff=4, cpu=True),
    ]


def simt_cases():
    """descriptors only the SIMT engine (impl 1) takes."""
    return [
        case('grouped', 'groups 4: the DCN grouped GEMM (1x1, Cin = 9 x 8 sampled columns per group), bias',
             H=10, W=10, Cin=72, Cout=32, groups=4, bias='vec', out='f32'),
        case('m-count', 'm_count = 100 ending inside a 64-row tile: rows 100.. of the 144 stay untouched, relu',
             H=12, W=12, KH=3, KW=3, pad=1, Cin=16, Cout=32, act=1, out='f32', m_count=100),
    ]


# ---------------------------------------------------------------------------------------------------------- host decisions
def cdiv(a, b):
    return -(-a // b)


def tile_shape(OH, OW, stride):
    """tt_conv2d_f16s / tt_conv2d_tc: the TH x TW <= 128 rectangle that wastes the fewest rows."""
    best, bt = -1.0, (1, 1)
    for tw in range(1, 129):
        if tw * stride > 256:
            break
        th = 128 // tw
        cover = OW * OH / (cdiv(OW, tw) * tw * cdiv(OH, th) * th)
        eff = cover * (tw * th) / 128.0
        if eff > best + 1e-9:
            best, bt = eff, (th, tw)
    return bt


def geometry(c):
    """(flat, TH, TW, m_tiles) of the A operand, as tt_conv2d_f16s and tt_conv2d_tc choose it."""
    d = desc(c, 4)
    xhs = d.x_hstride or d.W * d.x_ld
    xns = d.x_nstride or d.H * xhs
    flat = d.KH * d.KW == 1 and d.pad == 0 and d.stride == 1 and xhs == d.W * d.x_ld and xns == d.H * xhs
    if flat:
        return True, 1, 128, cdiv(d.N * d.H * d.W, 128)
    th, tw = tile_shape(d.OH, d.OW, d.stride)
    return False, th, tw, cdiv(d.OW, tw) * cdiv(d.OH, th) * d.N


def schedule(c, num_sms, flags=0):
    """tt_conv2d_f16s's host decisions for case c (phase 0 of a scatter) at num_sms SMs and knobs `flags`."""
    flat, th, tw, m_tiles = geometry(c)
    taps = c.KH * c.KW
    wide = c.Cout > 64 and not flags & BN64 and m_tiles * cdiv(c.Cout, 128) >= num_sms
    bn = 128 if wide else 64
    n_tiles = cdiv(c.Cout, bn)
    k_iters = taps * cdiv(c.Cin, 64)
    splits = 1
    plain = c.out != 'planes' and not c.scatter and c.res_mode != 2 and not c.bias_n_mod and not flags & NO_SPLITK
    if plain and m_tiles * n_tiles <= num_sms // 2 and k_iters >= 8:
        sp = min(cdiv(num_sms, m_tiles * n_tiles), k_iters // 4, 32)
        if sp >= 2:
            splits = cdiv(k_iters, cdiv(k_iters, sp))
    finish = splits > 1 and (c.act != 0 or c.out != 'f32')
    items = m_tiles * n_tiles * splits
    ctas = max(1, min(items, num_sms - ((flags >> 8) & 0xFF)))
    ragged = not flat and (c.OH % th != 0 or c.OW % tw != 0)
    return SimpleNamespace(flat=flat, TH=th, TW=tw, m_tiles=m_tiles, wide=wide, bn=bn, n_tiles=n_tiles, k_iters=k_iters,
                           splits=splits, finish=finish, chunk=fold_stages(flags), ctas=ctas, items=items, ragged=ragged,
                           launches=1 + (splits > 1) + finish)


def regimes(c, num_sms):
    """the corners of section (2b) case c reaches at knob 0 on num_sms SMs."""
    s = schedule(c, num_sms)
    r = {'flat' if s.flat else 'tiled', 'wide' if s.wide else 'narrow'}
    if s.ragged:
        r.add('ragged tiles')
    if s.flat and (c.N * c.H * c.W) % 128:
        r.add('M tail')
    if c.Cout % s.bn:
        r.add('N tail')
    if s.wide and c.Cout % 128:
        r.add('partial wide tile')
    if c.Cin % 64:
        r.add('K tail')
    if c.Cin % 8:
        r.add('Cin8 padding')
    if s.splits > 1:
        r.add('split-K + finish' if s.finish else 'split-K')
    return r


REQUIRED_REGIMES = {'flat', 'tiled', 'ragged tiles', 'M tail', 'N tail', 'partial wide tile', 'K tail', 'Cin8 padding', 'narrow',
                    'wide', 'split-K', 'split-K + finish'}


def regime_table(cases, num_sms):
    """{regime: [case names]} over the case list at num_sms SMs."""
    out = {}
    for c in cases:
        for r in regimes(c, num_sms):
            out.setdefault(r, []).append(c.name)
    return out


def tc_supported(c):
    """tt_conv2d's impl >= 2 predicate (csrc/gemm_conv_tc.cu tt_conv2d_tc_supported, with the buffers of `Buffers` aligned)."""
    d = desc(c, 3)
    if c.m_count is not None or d.groups != 1 or d.stride not in (1, 2):
        return False
    if any(v % 4 for v in (d.Cin, d.Cout, d.x_ld, d.x_coff, d.y_ld, d.y_coff, d.x_nstride, d.y_nstride, d.x_hstride)):
        return False
    if (d.res_mode and (d.res_ld % 4 or d.res_coff % 4)) or d.res2_ld % 4 or d.res2_coff % 4:
        return False
    return True


def tc_launches(c, num_sms, flags):
    """tt_conv2d_tc's launches: split-K init + kernel + finish when act != 0."""
    flat, th, tw, m_tiles = geometry(c)
    tiles = m_tiles * cdiv(c.Cout, 64)
    k_iters = c.KH * c.KW * cdiv(c.Cin, 32)
    plain = not c.scatter and c.res_mode != 2 and not c.bias_n_mod and not flags & NO_SPLITK
    splits = 1
    if plain and tiles <= num_sms // 2 and k_iters >= 16:
        sp = min(cdiv(num_sms, tiles), k_iters // 8, 32)
        if sp >= 2:
            splits = cdiv(k_iters, cdiv(k_iters, sp))
    return 1 + (splits > 1) * (1 + (c.act != 0))


# ---------------------------------------------------------------------------------------------------------- descriptors
def phases(c):
    """(oy_add, ox_add) of each call of the case."""
    return [(i, j) for i in range(2) for j in range(2)] if c.scatter else [(0, 0)]


def row_pixels(c):
    """pixels of an input row the descriptor reads (the row-packed form reads Cin / x_ld - 1 pixels past its W positions)."""
    return c.W + (c.Cin // c.x_ld - 1 if c.packed else 0)


def x_strides(c):
    """(x_hstride, x_nstride) in elements; 0 where the dense value applies."""
    hs = (row_pixels(c) + c.row_gap) * c.x_ld
    ns = c.H * hs + c.img_gap
    dense_hs = c.W * c.x_ld
    return (0 if hs == dense_hs else hs), (0 if ns == c.H * dense_hs else ns)


def desc(c, impl, phase=(0, 0)):
    from thinktwice_b200.lib import ConvDesc
    d = ConvDesc()
    for k in ('N', 'H', 'W', 'Cin', 'x_ld', 'Cout', 'KH', 'KW', 'stride', 'pad', 'dil', 'groups', 'OH', 'OW', 'y_ld', 'y_coff', 'act',
              'bias_n_mod'):
        setattr(d, k, getattr(c, k))
    d.x_coff = c.x_coff if impl != 4 else 0                            # f16s: x_split points at the channel offset already
    d.x_hstride, d.x_nstride = x_strides(c)
    m = 2 if c.scatter else 1
    d.yH, d.yW = c.OH * m, c.OW * m
    d.oy_mul = d.ox_mul = m
    d.oy_add, d.ox_add = phase
    d.y_nstride = d.yH * d.yW * d.y_ld + c.y_gap if c.y_gap else 0
    if c.res:
        d.res_mode, d.res_ld, d.res_coff = c.res_mode, c.res_ld, c.res_coff
        if c.res_mode == 2:
            d.res_H, d.res_W = c.res_hw
    if c.res2:
        d.res2_ld, d.res2_coff = c.res2_ld, c.res2_coff
    if c.junk:
        d.taps, d.M = 5, 3
    d.impl = impl
    return d


# ---------------------------------------------------------------------------------------------------------- buffers
class Backend:
    """the C ABI a case runs on: the real library (pointers are addresses) or the emulated one (pointers are emu_lib.Ptr)."""

    def __init__(self, lib, cuda):
        self.lib, self.cuda = lib, cuda
        self.dev = torch.device('cuda:0' if cuda else 'cpu')

    @classmethod
    def gpu(cls):
        from thinktwice_b200 import lib
        return cls(lib.load(), True)

    def p(self, t, off=0):
        if t is None:
            return C.c_void_p(0) if self.cuda else NULL
        return C.c_void_p(t.data_ptr() + off * t.element_size()) if self.cuda else Ptr(t, off)

    def byref(self, s):
        return C.byref(s) if self.cuda else s

    def new_io(self):
        from thinktwice_b200.lib import F16sIO
        return F16sIO() if self.cuda else IO()

    def stream(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream) if self.cuda else None

    def sync(self):
        if self.cuda:
            torch.cuda.synchronize()

    def launches(self):
        return int(self.lib.tt_launch_count())

    def saturations(self):
        v = C.c_uint()
        rc = self.lib.tt_f16s_saturation_count(self.byref(v), 0, self.stream())
        assert rc == 0, rc
        return int(v.value)

    def num_sms(self):
        return torch.cuda.get_device_properties(0).multi_processor_count if self.cuda else 132

    def debug_set(self, flags):
        return int(self.lib.tt_debug_set(flags))


def _poisoned(n, dtype, dev, fill=NAN):
    """a flat buffer of GUARD + n + GUARD elements (body at offset GUARD)."""
    return torch.full((GUARD + n + GUARD,), fill, dtype=dtype, device=dev)


def _grid(t, off, N, H, W, ld, C, hs=0, ns=0, coff=0):
    """(N, H, W, C) strided view of channels [coff, coff + C) of a channels-last grid at element `off` of flat t."""
    hs = hs or W * ld
    ns = ns or H * hs
    return torch.as_strided(t, (N, H, W, C), (ns, hs, ld, 1), off + coff)


def _split_planes(v):
    hi, lo = _split_f16(v)
    return hi, lo


class Buffers:
    """the operand and destination buffers of one case for one engine ('f16s', 'pointwise', 'simt' or 'tc'), poisoned / sentinel
    filled as the module docstring says.  Values are seeded by the case; the same case gives the fp32 twin the same fp32 operand
    values (its split planes carry them to 2^-22)."""

    def __init__(self, be, c, kind):
        self.be, self.c, self.kind = be, c, kind
        dev, g = be.dev, torch.Generator().manual_seed(c.seed)
        split = kind in ('f16s', 'pointwise')
        taps, cg = c.KH * c.KW, c.Cin // c.groups
        # ---- input
        hs, ns = x_strides(c)
        hs = hs or c.W * c.x_ld
        ns = ns or c.H * hs
        body = c.N * ns
        rw, rc = row_pixels(c), (c.x_ld if c.packed else c.Cin)
        xv = torch.randn(c.N, c.H, rw, rc, generator=g)
        xv[..., :rc] *= torch.exp(torch.randn(1, 1, 1, rc, generator=g))            # per-channel scales: small elements matter too
        if split:
            self.x_plane = body + PLANE_GAP
            self.x = _poisoned(2 * self.x_plane, torch.float16, dev)
            hi, lo = _split_f16(xv)
            for pl, v in ((0, hi), (self.x_plane, lo)):
                _grid(self.x, GUARD + pl, c.N, c.H, rw, c.x_ld, rc, hs, ns, c.x_coff).copy_(v)
            self.x_off = GUARD + c.x_coff                                  # x_split points at the channel offset
        else:
            self.x_plane = 0
            self.x = _poisoned(body, torch.float32, dev)
            _grid(self.x, GUARD, c.N, c.H, rw, c.x_ld, rc, hs, ns, c.x_coff).copy_(xv)
            self.x_off = GUARD
        # ---- weights: (Cout, taps, Cin_g) values in the engine's packing
        w = torch.randn(c.Cout, taps, cg, generator=g) / math.sqrt(taps * cg)
        if kind == 'f16s':
            c8 = cdiv(c.Cin, 8) * 8
            wp = torch.zeros(c.Cout, taps, c8)
            wp[..., :c.Cin] = w
            hi, lo = _split_f16(wp)
            self.w = _poisoned(2 * wp.numel(), torch.float16, dev)
            self.w[GUARD:GUARD + 2 * wp.numel()] = torch.cat([hi.reshape(-1), lo.reshape(-1)]).to(dev)
        elif kind == 'tc':
            from thinktwice_b200.weights import tf32_split
            hi, lo = tf32_split(w)
            self.w = _poisoned(2 * w.numel(), torch.float32, dev)
            self.w[GUARD:GUARD + 2 * w.numel()] = torch.cat([hi.reshape(-1), lo.reshape(-1)]).to(dev)
        else:                                                          # [taps * Cin_g][Cout] (impl 1, and pointwise's K-major)
            wk = w.permute(1, 2, 0).reshape(-1)
            self.w = _poisoned(wk.numel(), torch.float32, dev)
            self.w[GUARD:GUARD + wk.numel()] = wk.to(dev)
        # ---- bias
        self.bias = None
        if c.bias:
            rows = c.bias_n_mod if c.bias == 'table' else 1
            self.bias = _poisoned(rows * c.Cout, torch.float32, dev)
            self.bias[GUARD:GUARD + rows * c.Cout] = (torch.randn(rows * c.Cout, generator=g) * 0.5).to(dev)
        # ---- residuals
        self.res = self.res_s = self.res2 = self.res2_s = None
        self.res_plane = self.res2_plane = 0
        for which, form, ld, coff in (('res', c.res, c.res_ld, c.res_coff), ('res2', c.res2, c.res2_ld, c.res2_coff)):
            if not form:
                continue
            rh, rw_ = c.res_hw if which == 'res' and c.res_mode == 2 else (c.OH, c.OW)
            n = c.N * rh * rw_ * ld
            v = torch.randn(c.N, rh, rw_, c.Cout, generator=g)
            if form == 'f32' or not split:
                t = _poisoned(n, torch.float32, dev)
                _grid(t, GUARD, c.N, rh, rw_, ld, c.Cout, coff=coff).copy_(v)
                setattr(self, which, t)
            else:
                plane = n + PLANE_GAP
                t = _poisoned(2 * plane, torch.float16, dev)
                hi, lo = _split_f16(v)
                for pl, vv in ((0, hi), (plane, lo)):
                    _grid(t, GUARD + pl, c.N, rh, rw_, ld, c.Cout, coff=coff).copy_(vv)
                setattr(self, which + '_s', t)
                setattr(self, which + '_plane', plane)
        # ---- outputs
        d = desc(c, 1)
        self.y_body = (d.y_nstride or d.yH * d.yW * d.y_ld) * c.N
        self.y = _poisoned(self.y_body, torch.float32, dev, Y_SENTINEL) if (c.out != 'planes' or not split) else None
        self.y_plane = 0
        self.ys = None
        if split and c.out != 'f32':
            self.y_plane = self.y_body + PLANE_GAP
            self.ys = _poisoned(2 * self.y_plane, torch.float16, dev, H_SENTINEL)
        self.m_count = torch.tensor([c.m_count], dtype=torch.int32, device=dev) if c.m_count is not None else None

    def outputs(self):
        return {k: getattr(self, k) for k in ('y', 'ys') if getattr(self, k) is not None}

    # ------------------------------------------------------------------ the calls
    def io(self, emu_ptrs=False):
        """the tt_f16s_io of a call (emu_ptrs: emu_lib.IO of Ptrs, what conv_ref takes)."""
        be = self.be
        io = IO() if emu_ptrs else be.new_io()
        p = (lambda t, off=GUARD: Ptr(t, off) if t is not None else NULL) if emu_ptrs else \
            (lambda t, off=GUARD: be.p(t, off) if t is not None else be.p(None))
        io.x_split, io.x_plane = p(self.x, self.x_off), self.x_plane
        io.w_split, io.bias = p(self.w), p(self.bias)
        io.res, io.res2 = p(self.res), p(self.res2)
        io.res_split, io.res_plane = p(self.res_s), self.res_plane
        io.res2_split, io.res2_plane = p(self.res2_s), self.res2_plane
        io.y, io.y_split, io.y_plane = p(self.y), p(self.ys), self.y_plane
        return io

    def run(self, d, workspace=None):
        be = self.be
        if self.kind == 'f16s':
            return int(be.lib.tt_conv2d_f16s(be.byref(d), be.byref(self.io()), be.stream()))
        if self.kind == 'pointwise':
            return int(be.lib.tt_pointwise_f16s(be.byref(d), be.byref(self.io()), be.p(self.w, GUARD), be.stream()))
        q = lambda t: be.p(t, GUARD) if t is not None else be.p(None)
        return int(be.lib.tt_conv2d(be.byref(d), be.p(self.x, self.x_off), q(self.w), q(self.bias), q(self.res), q(self.res2),
                                    be.p(None), be.p(self.m_count) if self.m_count is not None else be.p(None), q(self.y),
                                    be.p(workspace) if workspace is not None else be.p(None), be.stream()))

    def reference(self, d):
        """(value, magnitude) of the call in float64 on the buffers' device."""
        io = self.io(emu_ptrs=True)
        if self.kind == 'pointwise':
            return conv_ref(d, io.x_split, io.w_split, io.bias, NULL, NULL, io, kmajor_w=True, magnitude=True)
        if self.kind == 'f16s':
            return conv_ref(d, io.x_split, io.w_split, io.bias, io.res, io.res2, io, magnitude=True)
        x = Ptr(self.x, self.x_off + self.c.x_coff)                   # tt_conv2d reads channel x_coff + c of each pixel
        return conv_ref(d, x, io.w_split, io.bias, io.res, io.res2, magnitude=True)


# ---------------------------------------------------------------------------------------------------------- checks
class Finding(SimpleNamespace):
    """one failed check: check in ('value', 'planes', 'outside', 'saturation', 'launches', 'status'), text."""


def _bits(t):
    return t.view({4: torch.int32, 2: torch.int16}[t.element_size()])


def _ratio(got, want, bound):
    err = (got.double() - want).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return torch.nan_to_num(r, nan=math.inf, posinf=math.inf)


def engine_name(kind):
    return {'f16s': 'tt_conv2d_f16s', 'pointwise': 'tt_pointwise_f16s'}.get(kind, 'tt_conv2d')


def rows_mask(d, rows):
    """(N, OH, OW, Cout) 0/1 mask of the first `rows` output rows (all when rows is None)."""
    m = torch.ones(d.N * d.OH * d.OW, d.Cout, dtype=torch.bool)
    if rows is not None:
        m[rows:] = False
    return m.view(d.N, d.OH, d.OW, d.Cout)


def check_call(bufs, d, before, ref, chunk=2):
    """the checks of one call whose destinations were `before` (clones of bufs.outputs()) and whose float64 reference is `ref`:
    returns (worst err / bound ratio, [Finding])."""
    c, found = bufs.c, []
    val, mag = ref
    K = d.KH * d.KW * (d.Cin // d.groups)
    bound = act_bound(d.act, conv_c(engine_name(bufs.kind), d, K, chunk), mag, val)
    keep = rows_mask(d, c.m_count).to(val.device)
    worst = 0.0

    def judge(check, got, want, bnd, what):
        nonlocal worst
        r = _ratio(got, want, bnd)[keep]
        if not r.numel():
            return
        rm = float(r.max())
        if check == 'value':
            worst = max(worst, rm)
        if not rm < 1:
            found.append(Finding(check=check, text=f'{c.name} {what}: {int((r >= 1).sum())} elements beyond the bound '
                                                   f'(worst ratio {rm:.3g})'))
    y32 = None
    if bufs.y is not None:
        y32 = y_region(d, Ptr(bufs.y, GUARD))
        judge('value', y32, val, bound, 'fp32 y')
    if bufs.ys is not None:
        hi = y_region(d, Ptr(bufs.ys, GUARD))
        lo = y_region(d, Ptr(bufs.ys, GUARD + bufs.y_plane))
        if y32 is not None:
            h, l = _split_f16(y32)
            same = (_bits(hi) == _bits(h)) & (_bits(lo) == _bits(l))
            bad = ~same & keep
            if bool(bad.any()):
                found.append(Finding(check='planes', text=f'{c.name}: {int(bad.sum())} plane elements are not _split_f16 of fp32 y'))
        else:
            judge('value', hi.double() + lo.double() / 2048.0, val, bound + SPLIT * val.abs() + SPLIT_ABS, 'planes')
    for k, t in bufs.outputs().items():
        m = torch.zeros(t.shape, dtype=torch.float32, device=t.device)
        for pl in ((0, bufs.y_plane) if k == 'ys' else (0,)):
            y_region(d, Ptr(m, GUARD + pl))[...] = keep.float()
        bad = (_bits(t) != _bits(before[k])) & (m == 0)
        if bool(bad.any()):
            i = int(bad.nonzero()[0])
            found.append(Finding(check='outside', text=f'{c.name}: {int(bad.sum())} elements of {k} outside the region changed '
                                                       f'(first at flat index {i})'))
    return worst, found


def run_checked(bufs, d, ref, flags=0, workspace=None, expect_launches=None):
    """one call through the checks: (worst ratio, [Finding]).  The outputs are NOT reset: a scatter's later phases see the earlier
    ones, and a check of a repeated call sees the previous result outside its region."""
    be = bufs.be
    before = {k: t.clone() for k, t in bufs.outputs().items()}
    be.sync()
    sat0, l0 = be.saturations(), be.launches()
    rc = bufs.run(d, workspace)
    be.sync()
    if rc != 0:
        return math.inf, [Finding(check='status', text=f'{bufs.c.name}: returned {rc}')]
    launches = be.launches() - l0
    worst, found = check_call(bufs, d, before, ref, fold_stages(flags))
    if be.saturations() != sat0:
        found.append(Finding(check='saturation', text=f'{bufs.c.name}: an epilogue saturated a split plane'))
    if expect_launches is not None and launches != expect_launches:
        found.append(Finding(check='launches', text=f'{bufs.c.name}: {launches} launches, the host schedule implies {expect_launches}'))
    return worst, found


def reset_outputs(bufs):
    if bufs.y is not None:
        bufs.y.fill_(Y_SENTINEL)
    if bufs.ys is not None:
        bufs.ys.fill_(H_SENTINEL)


def run_case(bufs, flags=0, workspace=None, launches=None, refs=None):
    """every phase of a case from sentinel-filled outputs: (worst ratio, [Finding], refs).  refs: the float64 references of the
    phases (computed on the first run and passed back in to save the work)."""
    reset_outputs(bufs)
    impl = {'f16s': 4, 'pointwise': 4, 'simt': 1, 'tc': 3}[bufs.kind]
    worst, found, out = 0.0, [], []
    for i, ph in enumerate(phases(bufs.c)):
        d = desc(bufs.c, impl, ph)
        ref = refs[i] if refs else bufs.reference(d)
        out.append(ref)
        w, f = run_checked(bufs, d, ref, flags, workspace, launches)
        worst, found = max(worst, w), found + f
    return worst, found, out
