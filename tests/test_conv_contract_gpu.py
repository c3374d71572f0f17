"""The dense convolution engines against float64 on the descriptor matrix of tests/conv_contract.py, under every schedule the host
can choose: each tt_conv2d_f16s case under each tt_debug_set knob setting (default, no split-K, 64-column tiles, fold every 4 / 1
slabs, one CTA walking every work item, and the three combined), the fp32 twins through tt_conv2d impl 1 (without and with the
split-K workspace) and impl 3 (under the knobs its kernel reads), tt_pointwise_f16s, and one refusal case per term of each `ok`
predicate.  Every call is checked per element (value, planes, outside its region, saturation) and its launch count against the host
schedule conv_contract.schedule restates.  Prints, per engine and knob setting, the largest error-to-bound ratio and the regimes
reached."""
import ctypes as C

import pytest
import torch

import conv_contract as K

pytestmark = pytest.mark.gpu
WORST = {}                                                             # (engine, knob label) -> worst err / bound ratio


@pytest.fixture(scope='module')
def be():
    b = K.Backend.gpu()
    yield b
    b.debug_set(0)


def set_knobs(be, flags):
    assert be.debug_set(flags) == 0, flags


def note(engine, label, ratio):
    WORST[(engine, label)] = max(WORST.get((engine, label), 0.0), ratio)


def outputs(bufs):
    return {k: t.clone() for k, t in bufs.outputs().items()}


def assert_bitwise(a, b, what):
    for k in a:
        same = K._bits(a[k]) == K._bits(b[k])
        assert bool(same.all()), f'{what}: {int((~same).sum())} elements of {k} differ'


def by_name(cases):
    return {c.name: c for c in cases}


F16S = by_name(K.f16s_cases())
POINTWISE = by_name(K.pointwise_cases())
SIMT_ONLY = by_name(K.simt_cases())


def test_the_case_list_reaches_every_regime_at_the_device_sm_count(be):
    n = be.num_sms()
    table = K.regime_table(F16S.values(), n)
    print(f'\nregimes at {n} SMs:')
    for r in sorted(table):
        print(f'  {r:18s} {", ".join(table[r])}')
    assert K.REQUIRED_REGIMES <= set(table), K.REQUIRED_REGIMES - set(table)


@pytest.mark.parametrize('name', list(F16S))
def test_f16s_under_every_knob_setting(be, name):
    c, n = F16S[name], be.num_sms()
    bufs = K.Buffers(be, c, 'f16s')
    refs, outs = None, {}
    try:
        for label, flags in K.knob_matrix(n):
            set_knobs(be, flags)
            s = K.schedule(c, n, flags)
            worst, found, refs = K.run_case(bufs, flags, launches=s.launches, refs=refs)
            assert not found, f'{label}: ' + '\n'.join(f.text for f in found)
            note('tt_conv2d_f16s', label, worst)
            outs[label] = outputs(bufs)
            print(f'{name:16s} {label:20s} splits {s.splits} bn {s.bn} fold {s.chunk} ctas {s.ctas:3d}  worst err/bound {worst:.3g}')
    finally:
        set_knobs(be, 0)
    # outside split-K the persistent loop must not carry state from one work item to the next: the SM reserve and the tile width
    # change which CTA computes an element, not how
    one = K.reserve(n)
    pairs = [('one-cta', 0, 'default', 0), ('bn64', K.BN64, 'default', 0), ('bn64+fold4+one-cta', K.BN64 | K.FOLD4 | one, 'fold4', K.FOLD4)]
    for a, fa, b, fb in pairs:
        if K.schedule(c, n, fa).splits == 1 and K.schedule(c, n, fb).splits == 1:
            assert_bitwise(outs[a], outs[b], f'{name}: {a} vs {b}')


@pytest.mark.parametrize('name', list(POINTWISE))
def test_pointwise(be, name):
    c = POINTWISE[name]
    bufs = K.Buffers(be, c, 'pointwise')
    worst, found, _ = K.run_case(bufs, launches=K.cdiv(c.Cout, 32))
    assert not found, '\n'.join(f.text for f in found)
    note('tt_pointwise_f16s', 'default', worst)
    print(f'{name}: worst err/bound {worst:.3g}')


@pytest.mark.parametrize('name', list(F16S) + list(SIMT_ONLY))
def test_simt_twin_with_and_without_workspace(be, name):
    c = F16S.get(name) or SIMT_ONLY[name]
    bufs = K.Buffers(be, c, 'simt')
    worst, found, refs = K.run_case(bufs, launches=1)
    assert not found, '\n'.join(f.text for f in found)
    note('tt_conv2d impl 1', 'default', worst)
    need = int(be.lib.tt_conv2d_workspace_bytes(C.byref(K.desc(c, 1))))
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device=be.dev)
    runs = []
    for _ in range(2):
        w2, found, _ = K.run_case(bufs, workspace=ws, launches=2 if need else 1, refs=refs)
        assert not found, '\n'.join(f.text for f in found)
        runs.append(outputs(bufs))
        note('tt_conv2d impl 1', 'workspace', w2)
    assert_bitwise(runs[0], runs[1], f'{name}: two impl 1 calls')
    print(f'{name}: worst err/bound {worst:.3g}, with a workspace of {need} bytes {w2:.3g}')


TC_KNOBS = ('default', 'no-splitk', 'fold4', 'fold1', 'one-cta')


@pytest.mark.parametrize('name', list(F16S))
def test_3xtf32_twin_under_its_knobs(be, name):
    c, n = F16S[name], be.num_sms()
    bufs = K.Buffers(be, c, 'tc')
    if not K.tc_supported(c):
        l0 = be.launches()
        assert bufs.run(K.desc(c, 3)) == K.ERR_UNSUPPORTED and be.launches() == l0
        pytest.skip('outside the impl 3 predicate: refused, nothing launched')
    refs = None
    try:
        for label, flags in K.knob_matrix(n):
            if label not in TC_KNOBS:
                continue
            set_knobs(be, flags)
            worst, found, refs = K.run_case(bufs, flags, launches=K.tc_launches(c, n, flags), refs=refs)
            assert not found, f'{label}: ' + '\n'.join(f.text for f in found)
            note('tt_conv2d impl 3', label, worst)
            print(f'{name:16s} {label:12s} worst err/bound {worst:.3g}')
    finally:
        set_knobs(be, 0)


# ---------------------------------------------------------------------------------------------------------- refusals
SLACK = 1 << 16                                                        # elements each refusal buffer holds past its pointer
BASE_OFF = 4096                                                        # element offset of every base pointer


class Refusal:
    """real, sentinel-filled buffers much larger than any refused descriptor could address, and the pointers / plane strides of a
    valid base call that each refusal case changes in one term."""

    def __init__(self, be, c, impl):
        self.be, self.c, self.impl = be, c, impl
        dev = be.dev
        half = impl == 4
        mk = lambda dt: torch.full((BASE_OFF + 4 * SLACK,), 0.25, dtype=dt, device=dev)
        self.t = {k: mk(torch.float16 if half and k in ('x', 'w', 'ys', 'res_s', 'res2_s') else torch.float32)
                  for k in ('x', 'w', 'bias', 'res', 'res2', 'res_s', 'res2_s', 'y', 'ys')}
        self.t['y'].fill_(K.Y_SENTINEL)
        self.t['ys'].fill_(K.H_SENTINEL)
        self.off = {k: BASE_OFF for k in self.t}
        self.plane = {'x': SLACK, 'res': SLACK, 'res2': SLACK, 'y': SLACK}
        self.use = {'x', 'w', 'bias', 'res', 'res2', 'y'} | ({'ys'} if half else set())
        self.d = K.desc(c, impl)

    def call(self, w_kmajor=False):
        be, p = self.be, lambda k: be.p(self.t[k], self.off[k]) if k in self.use else be.p(None)
        if self.impl == 4:
            io = be.new_io()
            io.x_split, io.x_plane, io.w_split, io.bias = p('x'), self.plane['x'], p('w'), p('bias')
            io.res, io.res_split, io.res_plane = p('res'), p('res_s'), self.plane['res']
            io.res2, io.res2_split, io.res2_plane = p('res2'), p('res2_s'), self.plane['res2']
            io.y, io.y_split, io.y_plane = p('y'), p('ys'), self.plane['y']
            if w_kmajor:
                return int(be.lib.tt_pointwise_f16s(C.byref(self.d), C.byref(io), be.p(self.t['bias'], BASE_OFF), be.stream()))
            return int(be.lib.tt_conv2d_f16s(C.byref(self.d), C.byref(io), be.stream()))
        gather = be.p(self.gather) if getattr(self, 'gather', None) is not None else be.p(None)
        m_count = be.p(self.m_count) if getattr(self, 'm_count', None) is not None else be.p(None)
        return int(be.lib.tt_conv2d(C.byref(self.d), p('x'), p('w'), p('bias'), p('res'), p('res2'), gather, m_count, p('y'), be.p(None),
                                    be.stream()))


def _geom(d, stride):
    d.stride = stride
    d.OH = (d.H + 2 * d.pad - d.dil * (d.KH - 1) - 1) // stride + 1
    d.OW = (d.W + 2 * d.pad - d.dil * (d.KW - 1) - 1) // stride + 1
    d.yH, d.yW = d.OH, d.OW


def _set(**kw):
    def f(r):
        for k, v in kw.items():
            setattr(r.d, k, v)
    return f


def _ptr(k, by):
    def f(r):
        r.off[k] += by
    return f


def _plane(k, by):
    def f(r):
        r.plane[k] += by
    return f


def _split_res(k, by):
    """residual k given as split planes, its plane stride off by `by` (0: only the pointer moves to the split form)."""
    def f(r):
        r.use.discard(k)
        r.use.add(k + '_s')
        r.plane[k] += by
    return f


def _both(*fs):
    def f(r):
        for g in fs:
            g(r)
    return f


REFUSAL_BASE = K.case('refusal-base', '3x3 pad 1, Cin 16 in x_ld 24, Cout 32 at y_ld 40, bias, both residuals', H=8, W=8, KH=3,
                      KW=3, pad=1, Cin=16, x_ld=24, Cout=32, y_ld=40, bias='vec', res='f32', res_ld=40, res2='f32', res2_ld=40)
POINTWISE_BASE = K.case('pointwise-base', '1x1, Cin 16 in x_ld 16, Cout 32 at y_ld 40, bias', H=8, W=8, Cin=16, x_ld=16, Cout=32,
                        y_ld=40, bias='vec')

# one entry per term of tt_conv2d_f16s's `ok` (csrc/gemm_conv_f16s.cu): each breaks that term only
F16S_REFUSALS = {
    'groups': _set(groups=2), 'stride': lambda r: _geom(r.d, 3), 'Cout % 4': _set(Cout=30), 'x_ld % 8': _set(x_ld=20),
    'x_hstride % 8': _set(x_hstride=8 * 24 + 4), 'x_nstride % 8': _set(x_nstride=8 * 8 * 24 + 4), 'x_plane % 8': _plane('x', 4),
    'y_ld % 4': _set(y_ld=42), 'y_coff % 4': _set(y_coff=2), 'y_nstride % 4': _set(y_nstride=8 * 8 * 40 + 2),
    'y_plane % 4': _plane('y', 2), 'res_ld % 4': _set(res_ld=42), 'res_coff % 4': _set(res_coff=2),
    'res2_ld % 4': _set(res2_ld=42), 'res2_coff % 4': _set(res2_coff=2), 'res_plane % 4': _split_res('res', 2),
    'res2_plane % 4': _split_res('res2', 2), 'x_split 16-byte': _ptr('x', 4), 'w_split 16-byte': _ptr('w', 4),
    'y 16-byte': _ptr('y', 1), 'res 16-byte': _ptr('res', 1), 'res2 16-byte': _ptr('res2', 1), 'bias 16-byte': _ptr('bias', 1),
    'y_split 8-byte': _ptr('ys', 2), 'res_split 8-byte': _both(_split_res('res', 0), _ptr('res_s', 2)),
    'res2_split 8-byte': _both(_split_res('res2', 0), _ptr('res2_s', 2)), 'OH': _set(OH=7, yH=7), 'OW': _set(OW=9, yW=9),
}
# ... of tt_pointwise_f16s's `ok`
POINTWISE_REFUSALS = {
    'KH': _set(KH=3), 'KW': _set(KW=3), 'stride': _set(stride=2), 'pad': _set(pad=1), 'groups': _set(groups=2),
    'Cin <= 64': _set(Cin=72, x_ld=72), 'Cout <= 64': _set(Cout=68, y_ld=72), 'Cout % 4': _set(Cout=30), 'x_ld % 8': _set(x_ld=20),
    'Cin8 <= x_ld': _set(Cin=13, x_ld=8), 'y_ld % 4': _set(y_ld=42), 'y_coff % 4': _set(y_coff=2), 'x_plane % 8': _plane('x', 4),
    'y_plane % 4': _plane('y', 2), 'x_hstride dense': _set(x_hstride=8 * 16 + 8), 'x_nstride dense': _set(x_nstride=8 * 8 * 16 + 8),
    'y_nstride 0': _set(y_nstride=8 * 8 * 40 + 4), 'oy_mul': _set(oy_mul=2), 'ox_mul': _set(ox_mul=2), 'oy_add': _set(oy_add=1),
    'ox_add': _set(ox_add=1), 'yH': _set(yH=9), 'yW': _set(yW=9), 'OH == H': _set(OH=7, yH=7), 'OW == W': _set(OW=7, yW=7),
    'res_mode': _set(res_mode=1), 'res': lambda r: r.use.add('res'), 'res_split': lambda r: r.use.add('res_s'),
    'res2': lambda r: r.use.add('res2'), 'res2_split': lambda r: r.use.add('res2_s'), 'bias_n_mod': _set(bias_n_mod=2),
    'x_split 16-byte': _ptr('x', 4), 'y 16-byte': _ptr('y', 1), 'y_split 8-byte': _ptr('ys', 2),
}
# ... of tt_conv2d's impl >= 2 path (csrc/api.cu and tt_conv2d_tc_supported)
TC_REFUSALS = {
    'groups': _set(groups=2), 'stride': lambda r: _geom(r.d, 3), 'Cin % 4': _set(Cin=18), 'Cout % 4': _set(Cout=30),
    'x_ld % 4': _set(x_ld=22), 'x_coff % 4': _set(x_coff=2), 'y_ld % 4': _set(y_ld=42), 'y_coff % 4': _set(y_coff=2),
    'x_nstride % 4': _set(x_nstride=8 * 8 * 24 + 2), 'y_nstride % 4': _set(y_nstride=8 * 8 * 40 + 2),
    'x_hstride % 4': _set(x_hstride=8 * 24 + 2), 'res_ld % 4': _set(res_ld=42), 'res_coff % 4': _set(res_coff=2),
    'res2_ld % 4': _set(res2_ld=42), 'res2_coff % 4': _set(res2_coff=2), 'x 16-byte': _ptr('x', 1), 'w 16-byte': _ptr('w', 1),
    'y 16-byte': _ptr('y', 1), 'res 16-byte': _ptr('res', 1), 'res2 16-byte': _ptr('res2', 1), 'bias 16-byte': _ptr('bias', 1),
    'OH': _set(OH=7, yH=7), 'OW': _set(OW=9, yW=9),
    'gather': lambda r: (setattr(r, 'gather', torch.zeros(4096, dtype=torch.int32, device=r.be.dev)), setattr(r.d, 'taps', 1)),
    'm_count': lambda r: setattr(r, 'm_count', torch.tensor([10], dtype=torch.int32, device=r.be.dev)),
}


def _refusal(be, base, impl, mutate, pointwise=False):
    r = Refusal(be, base, impl)
    if pointwise:
        r.use = {'x', 'bias', 'y', 'ys'}
    mutate(r)
    before = {k: t.clone() for k, t in r.t.items()}
    torch.cuda.synchronize()
    l0 = be.launches()
    rc = r.call(w_kmajor=pointwise)
    torch.cuda.synchronize()
    assert rc == K.ERR_UNSUPPORTED, rc
    assert be.launches() == l0, 'a refused call launched a kernel'
    for k, t in r.t.items():
        assert bool((K._bits(t) == K._bits(before[k])).all()), f'a refused call changed {k}'


def test_the_refusal_bases_are_accepted(be):
    """each base call runs (so that every refusal below is caused by the one term it changes)."""
    for base, impl, pw in ((REFUSAL_BASE, 4, False), (POINTWISE_BASE, 4, True), (REFUSAL_BASE, 3, False)):
        r = Refusal(be, base, impl)
        if pw:
            r.use = {'x', 'bias', 'y', 'ys'}
        assert r.call(w_kmajor=pw) == 0, (base.name, impl, be.lib.tt_last_error())
    torch.cuda.synchronize()


@pytest.mark.parametrize('term', list(F16S_REFUSALS))
def test_f16s_refuses(be, term):
    _refusal(be, REFUSAL_BASE, 4, F16S_REFUSALS[term])


@pytest.mark.parametrize('term', list(POINTWISE_REFUSALS))
def test_pointwise_refuses(be, term):
    _refusal(be, POINTWISE_BASE, 4, POINTWISE_REFUSALS[term], pointwise=True)


@pytest.mark.parametrize('term', list(TC_REFUSALS))
def test_3xtf32_refuses(be, term):
    _refusal(be, REFUSAL_BASE, 3, TC_REFUSALS[term])


def test_unknown_debug_bits_are_refused_and_keep_the_previous_knobs(be):
    c = F16S['splitk']
    assert K.schedule(c, be.num_sms()).splits > 1
    bufs = K.Buffers(be, c, 'f16s')
    try:
        set_knobs(be, K.NO_SPLITK)
        for bad in (1, 0x10000, 0x80000, 0x800000, 1 << 30):
            assert bad & ~K.KNOWN_KNOBS
            assert be.debug_set(bad) == K.ERR_INVALID, hex(bad)
        _, found, _ = K.run_case(bufs, K.NO_SPLITK, launches=1)             # still no split-K: one launch
        assert not found, '\n'.join(f.text for f in found)
    finally:
        set_knobs(be, 0)


def test_split_rows_follow_rn_f16_for_nan_inf_and_out_of_range_values(be):
    """tt_split_f16 also sweeps arena rows no kernel has written, whose bits may be anything: its planes must be _split_f16 of the
    rows (the restatement the census checks it against), NaN included, and infinities and |x| > 65504 saturate."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(64, 40, generator=g) * torch.tensor([1e-8, 1.0, 3e4, 1e6]).repeat(10)
    x[::5, ::7] = float('nan')
    x[1::7, 3] = float('inf')
    x[2::7, 5] = -float('inf')
    xd = x.to(be.dev)
    ys = torch.full((2 * 64 * 48,), K.H_SENTINEL, dtype=torch.float16, device=be.dev)
    assert be.lib.tt_split_f16(be.p(xd), C.c_longlong(40), be.p(ys), C.c_longlong(64 * 48), C.c_longlong(48), C.c_longlong(64), 40,
                               be.p(None), be.stream()) == 0
    torch.cuda.synchronize()
    got = ys.view(2, 64, 48)[:, :, :40].cpu()
    hi, lo = K._split_f16(x)
    want = torch.stack([hi, lo])
    assert bool(((got == want) | (got.isnan() & want.isnan())).all())
    assert bool((ys.view(2, 64, 48)[:, :, 40:] == K.H_SENTINEL).all())


def test_report():
    """the worst err / bound ratio per engine and knob setting over this file's cases (printed; each call already passed)."""
    print(f'\n{torch.cuda.get_device_name(0)}, {torch.cuda.get_device_properties(0).multi_processor_count} SMs')
    for (eng, label), r in sorted(WORST.items()):
        print(f'  {eng:20s} {label:20s} worst err/bound {r:.3g}')
    assert all(r < 1 for r in WORST.values())
