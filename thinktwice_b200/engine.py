"""Host-side op layer: channels-last feature-map handles, a persistent buffer arena and one Python
method per C-ABI op.  No arithmetic happens here — every method ends in a libtt_b200 call.

Buffers are allocated once per (name, shape) and reused on every forward, so a steady-state forward
performs no allocation (CUDA-graph capturable) and keeps activations resident in HBM.
"""
import ctypes as C
import os

import torch

from . import lib
from .lib import ConvDesc, _p, _stream


class FMap:
    """A logical (N, H, W, C) fp32 tensor stored channels-last inside a buffer whose pixels hold `ld`
    floats; the C channels start at `coff`.  Concat = several FMaps viewing one buffer.
    `s` (optional) is the buffer's scaled-split fp16 companion: two half planes (hi, lo') over the SAME element grid as
    `t` (csrc/gemm_conv_f16s.cu), kept in step with `t` by whichever Engine op writes the map."""
    __slots__ = ('t', 'N', 'H', 'W', 'C', 'ld', 'coff', 's')

    def __init__(self, t, N, H, W, C, ld=None, coff=0, s=None):
        self.t, self.N, self.H, self.W, self.C = t, N, H, W, C
        self.ld = ld if ld is not None else C
        self.coff = coff
        self.s = s

    def slice(self, coff, C):
        return FMap(self.t, self.N, self.H, self.W, C, self.ld, self.coff + coff, self.s)

    def view(self, N, H, W, C, ld=None, coff=None):
        """another geometry over the same storage (fp32 buffer and split companion)."""
        return FMap(self.t, N, H, W, C, ld if ld is not None else C, self.coff if coff is None else coff, self.s)

    def rows(self):
        return self.N * self.H * self.W

    def as_rows(self):
        """view as a (rows, 1, 1, C) map (for Linear layers)."""
        return FMap(self.t, self.rows(), 1, 1, self.C, self.ld, self.coff, self.s)

    def dense(self):
        """contiguous (N, H, W, C) torch view/copy of the logical tensor (debug / tests / outputs)."""
        if self.t is None:                                         # split-only tensor: hi + lo' / 2048 (debug / test path)
            n = self.N * self.H * self.W * self.ld
            hi, lo = self.s[0].view(-1)[:n], self.s[1].view(-1)[:n]
            full = (hi.float() + lo.float() / 2048.0).view(self.N, self.H, self.W, self.ld)
            return full[..., self.coff:self.coff + self.C]
        v = self.t.view(self.N, self.H, self.W, self.ld)[..., self.coff:self.coff + self.C]
        return v

    def nchw(self):
        return self.dense().permute(0, 3, 1, 2)


def _t(fm):
    """the fp32 tensor of a map, or a loud error when the map is stored as split planes only."""
    if fm.t is None:
        raise lib.TTError('this kernel reads / writes fp32 but the map is stored as split planes only (fmt="s")')
    return fm.t


def _ps(fm):
    """device pointer of the hi plane of `fm`'s split companion at the map's channel offset (+ the plane stride in halves)."""
    return _p(fm.s, fm.coff), fm.s.numel() // 2


class PackedConv:
    """weights of one conv / linear in kernel layout: w [taps*Cin_g][Cout] (BatchNorm folded), bias [Cout]|None."""
    __slots__ = ('w', 'bias', 'Cin', 'Cout', 'KH', 'KW', 'groups', 'w_tc', 'w_h', 'alg_k')

    def __init__(self, w, bias, Cin, Cout, KH=1, KW=1, groups=1, w_tc=None, w_h=None):
        self.w, self.bias, self.Cin, self.Cout, self.KH, self.KW, self.groups = w, bias, Cin, Cout, KH, KW, groups
        self.w_tc = w_tc            # [2][Cout][taps][Cin] TF32 hi / lo planes for the tensor-core 3xTF32 path (or None)
        self.w_h = w_h              # [2][Cout][taps][Cin8] scaled-split fp16 planes for the tensor-core f16s path (or None)
        self.alg_k = None           # algorithmic K per output (row-packed convs carry zero-weight padding)


class _SideBranch:
    def __init__(self, eng):
        self.eng = eng

    def __enter__(self):
        e = self.eng
        # serial when profiling per-launch events (overlapped kernels would inflate each other's timings) or off-GPU
        self.active = e.overlap and e.prof is None and e.device.type == 'cuda' and torch.cuda.is_available()
        if not self.active:
            return self
        if e._side is None:
            e._side = torch.cuda.Stream(device=e.device)
        self.main = torch.cuda.current_stream()
        fork = torch.cuda.Event()
        fork.record(self.main)
        e._side.wait_event(fork)
        self.ctx = torch.cuda.stream(e._side)
        self.ctx.__enter__()
        e.lane = 1
        return self

    def __exit__(self, *exc):
        e = self.eng
        if not self.active:
            return False
        e.lane = 0
        self.done = torch.cuda.Event()
        self.done.record(e._side)
        self.ctx.__exit__(*exc)
        return False

    def join(self):
        """make the current (main) stream wait for the side branch."""
        if self.active:
            torch.cuda.current_stream().wait_event(self.done)


class Engine:
    def __init__(self, device, impl=lib.IMPL_AUTO):
        self.device = torch.device(device)
        self.impl = impl
        self.bufs = {}
        self.last_buf = {}
        self.cur = {}                 # name -> the buffer the latest upload(name, ...) went to (shape-keyed arena: see static())
        self.conv_ws = {}             # per lane: grow-only conv workspace (split-K partial sums of the SIMT kernel)
        self._ws_retired = []         # outgrown workspaces stay alive: CUDA graphs captured earlier still point at them
        self._scratch, self._tmp_maps = {}, set()
        self.lane = 0               # 0 = main stream; 1 = side stream (independent branch running concurrently)
        self._side = None
        self._copy = None           # upload stream of the pipelined forward (EncoderDecoder._pipelined_forward)
        self.overlap = True         # run independent branches (side_branch) concurrently
        self.marks = None           # bench.py: list of (segment name, event) recorded by mark() in a serial eager step
        self.tc_min_rows = 512
        self.thin_min_rows = 1 << 16   # rows from which a thin (Cin, Cout <= 64) 1x1 conv runs as a per-pixel mat-vec
        self.tc_strides = (1, 2)
        self.split = impl == lib.IMPL_F16S   # feature maps carry a scaled-split fp16 companion (gemm_conv_f16s.cu)
        self.stats = {'late_split': 0}
        self._cur_name = None
        self.force_fs = set(filter(None, os.environ.get('TT_FORCE_FS', '').split(',')))   # debugging: maps kept in both formats
        self.prof = None            # bench.py: list of (name, flops, start_event, end_event) per conv launch
        lib.load()

    def mark(self, name):
        """segment boundary for bench.py's per-segment timing (no-op unless `marks` is a list)."""
        if self.marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.marks.append((name, ev))

    # ------------------------------------------------------------------ streams
    def side_branch(self):
        """context manager: kernels issued inside run on a side stream forked from the current one (an independent
        branch of the forward, e.g. the LiDAR encoder beside the camera encoder); `join()` on exit.  Works eagerly and
        under CUDA-graph capture (fork / join become graph dependencies)."""
        return _SideBranch(self)

    # ------------------------------------------------------------------ buffers
    def buf(self, name, shape, dtype=torch.float32, zero=False):
        key = (name, tuple(shape), dtype)
        t = self.bufs.get(key)
        if t is None:
            t = (torch.zeros if zero else torch.empty)(tuple(shape), dtype=dtype, device=self.device)
            self.bufs[key] = t
        self.last_buf[name] = t
        return t

    def static_named(self, name):
        """the buffer most recently requested under `name` (tests / debugging: a name can exist in several shapes)."""
        return self.last_buf[name]

    def upload(self, name, t):
        """copy a host (or device) tensor into the persistent device buffer `name` (static address: graph-safe)."""
        b = self.buf(name, t.shape, t.dtype)
        b.copy_(t, non_blocking=True)
        self.cur[name] = b
        return b

    def static(self, name):
        """the buffer of the LATEST upload under `name`.  Buffers are keyed by (name, shape, dtype), so when an input
        changes shape between forwards (batch size, LiDAR point count) a stale sibling of the same name exists too."""
        try:
            return self.cur[name]
        except KeyError:
            raise KeyError(f'static buffer {name} has not been staged') from None

    def fmap(self, name, N, H, W, C, ld=None, zero=False, split=None, fmt=None):
        """feature-map buffer `name`.  fmt (scaled-split engine only): 'fs' fp32 + split companion (default), 'f' fp32 only (nobody
        feeds it to a tensor-core conv), 's' split planes only (ONLY convolutions read it: operands and residuals come from the
        companion, no fp32 copy is stored).  's' is honoured when the map can feed the tensor-core kernel at all (row pitch a
        multiple of 8 halves, >= tc_min_rows rows); otherwise it degrades to 'f' and consumers convert late."""
        ld = ld if ld is not None else C
        if split is not None:
            fmt = 'fs' if split else 'f'
        if not self.split:
            fmt = 'f'
        elif fmt is None or name in self.force_fs or '*' in self.force_fs:
            fmt = 'fs'
        rows = N * H * W
        if fmt == 's' and not (ld % 8 == 0 and ld >= 32 and rows >= self.tc_min_rows):
            fmt = 'f'
        # a tensor-core conv needs >= 128 GEMM rows: smaller maps only ever feed the SIMT kernels
        if 's' in fmt and not (ld % 4 == 0 and ld >= 32 and rows >= 128):
            fmt = 'f'
        t = self.buf(name, (N, H, W, ld), zero=zero) if 'f' in fmt else None
        sc = self.buf(name + '#s', (2, rows * ld), torch.float16, zero=True) if 's' in fmt else None
        return FMap(t, N, H, W, C, ld, 0, sc)

    def scratch_f32(self, numel):
        """per-lane fp32 scratch (grow-only; outgrown buffers stay alive for already captured graphs): the fp32 side of an
        operation whose result is kept as split planes only."""
        sb = self._scratch.get(self.lane)
        if sb is None or sb.numel() < numel:
            if sb is not None:
                self._ws_retired.append(sb)
            sb = self._scratch[self.lane] = torch.empty(int(numel), dtype=torch.float32, device=self.device)
        return sb

    def out_map(self, name, N, H, W, C, fmt=None, ld=None):
        """output map of a NON-convolution kernel (they write fp32): for fmt 's' the fp32 side lives in the lane's scratch just long
        enough to be converted (finish_out)."""
        fm = self.fmap(name, N, H, W, C, ld, fmt=fmt)
        if fm.t is None:
            n = N * H * W * fm.ld
            fm.t = self.scratch_f32(n)[:n].view(N, H, W, fm.ld)
            self._tmp_maps.add(id(fm))
        return fm

    def finish_out(self, fm):
        self.sync_split(fm)
        if id(fm) in self._tmp_maps:
            self._tmp_maps.discard(id(fm))
            fm.t = None                                             # the scratch is free again: only the planes persist
        return fm

    def need_f32(self, fm, what):
        if fm.t is None:
            raise lib.TTError(f'{what}: the input map is stored as split planes only (fmt="s") but this kernel reads fp32')
        return fm

    def wrap(self, t, C=None):
        """wrap an existing contiguous (N, H, W, ld) tensor."""
        N, H, W, ld = t.shape
        return FMap(t, N, H, W, C if C is not None else ld, ld, 0)

    # ------------------------------------------------------------------ scaled-split companions
    def sync_split(self, fm):
        """bring the split companion of `fm` in step with its fp32 values (after a non-convolution kernel wrote them)."""
        if fm.s is None:
            return fm
        # the converter works on 4-column groups: widen the column range to the enclosing groups (the companion mirrors the
        # fp32 buffer element for element, so converting a neighbour's columns as well is always consistent)
        c0 = fm.coff // 4 * 4                                     # (coff may exceed ld: an element offset into the buffer)
        w = -(-(fm.coff - c0 + fm.C) // 4) * 4
        w = min(w, fm.ld - c0 % fm.ld) if fm.ld >= 4 else w
        if fm.ld % 4 or w % 4 or w <= 0:
            raise lib.TTError(f'split companion of a map with C={fm.C} coff={fm.coff} ld={fm.ld}: row pitch must be a multiple of 4')
        lib.call('tt_split_f16', _p(fm.t, c0), C.c_longlong(fm.ld), _p(fm.s, c0), C.c_longlong(fm.s.numel() // 2), C.c_longlong(fm.ld),
                 C.c_longlong(fm.rows()), w, None)
        return fm

    def merge_split(self, fm):
        """fp32 values of `fm` rebuilt from its split planes (hi + lo' / 2048), for maps that keep both representations."""
        if (fm.C | fm.coff | fm.ld) % 4:
            raise lib.TTError('merge_split: needs 4-column alignment')
        lib.call('tt_merge_f16', _p(fm.s, fm.coff), C.c_longlong(fm.s.numel() // 2), C.c_longlong(fm.ld), _p(fm.t, fm.coff), C.c_longlong(fm.ld),
                 C.c_longlong(fm.rows()), fm.C)
        return fm

    def with_split(self, fm):
        """`fm` with a valid split companion: its own, or a late one (allocated per underlying buffer, converted now)."""
        if fm.s is not None:
            return fm
        key = ('late#s', fm.t.data_ptr(), fm.t.numel())
        sc = self.bufs.get(key)
        if sc is None:
            sc = self.bufs[key] = torch.zeros((2, fm.t.numel()), dtype=torch.float16, device=self.device)
        self.stats['late_split'] += 1
        self.stats.setdefault('late_names', []).append(self._cur_name)
        return self.sync_split(FMap(fm.t, fm.N, fm.H, fm.W, fm.C, fm.ld, fm.coff, sc))

    # ------------------------------------------------------------------ conv / linear
    def conv(self, x, pw, out=None, name=None, stride=1, pad=0, dil=1, act=0, res=None, res_mode=0, res2=None,
             scatter=None, out_ld=None, impl=None, x_nstride=0, y_nstride=0, n_images=None, bias_n_mod=0, x_hstride=0, fmt=None):
        """y = act(conv(x) + bias + res + res2).  `out` (FMap) selects the destination (concat slice / scatter
        target); otherwise a buffer `name` is created.  scatter = (oy_mul, oy_add, ox_mul, ox_add)."""
        assert x.C == pw.Cin, (x.C, pw.Cin, name)
        OH = (x.H + 2 * pad - dil * (pw.KH - 1) - 1) // stride + 1
        OW = (x.W + 2 * pad - dil * (pw.KW - 1) - 1) // stride + 1
        if out is None:
            out = self.fmap(name, x.N, OH, OW, pw.Cout, out_ld, fmt=fmt)
        d = ConvDesc()
        d.N, d.H, d.W, d.Cin, d.x_ld, d.x_coff = (n_images or x.N), x.H, x.W, x.C, x.ld, 0
        d.x_nstride, d.y_nstride, d.x_hstride = x_nstride, y_nstride, x_hstride
        d.Cout, d.KH, d.KW, d.stride, d.pad, d.dil, d.groups = pw.Cout, pw.KH, pw.KW, stride, pad, dil, pw.groups
        d.OH, d.OW = OH, OW
        d.y_ld, d.y_coff, d.yH, d.yW = out.ld, 0, out.H, out.W
        if scatter is None:
            assert out.H == OH and out.W == OW and out.C == pw.Cout, (name, out.H, OH, out.W, OW)
            d.oy_mul, d.oy_add, d.ox_mul, d.ox_add = 1, 0, 1, 0
        else:
            d.oy_mul, d.oy_add, d.ox_mul, d.ox_add = scatter
        d.act = act
        d.bias_n_mod = bias_n_mod
        d.res_mode = res_mode if res is not None else 0
        if res is not None:
            if d.res_mode == 0:
                d.res_mode = lib.RES_SAME
            d.res_ld, d.res_coff, d.res_H, d.res_W = res.ld, 0, res.H, res.W
            assert res.C == pw.Cout
        if res2 is not None:
            d.res2_ld, d.res2_coff = res2.ld, 0
        impl = self.impl if impl is None else impl
        # tensor-core paths: dense convs with enough work to fill 128-row tiles; everything else stays SIMT fp32
        big = (d.N * OH * OW >= self.tc_min_rows or (d.N * OH * OW >= 128 and pw.KH * pw.KW * pw.Cin >= 2048))   # thin M: only with a long K (split-K)
        common = (stride in self.tc_strides and pw.groups == 1 and out.ld % 4 == 0 and out.coff % 4 == 0
                  and (res is None or (res.ld % 4 == 0 and res.coff % 4 == 0)) and (res2 is None or (res2.ld % 4 == 0 and res2.coff % 4 == 0))
                  and y_nstride % 4 == 0 and big and pw.Cout >= 32)
        split_only = x.t is None or out.t is None or (res is not None and res.t is None) or (res2 is not None and res2.t is None)
        h_ok = (impl == lib.IMPL_F16S and pw.w_h is not None and stride in (1, 2) and pw.groups == 1 and out.ld % 4 == 0 and out.coff % 4 == 0
                and (res is None or (res.ld % 4 == 0 and res.coff % 4 == 0)) and (res2 is None or (res2.ld % 4 == 0 and res2.coff % 4 == 0))
                and y_nstride % 4 == 0 and x.ld % 8 == 0 and x.coff % 8 == 0 and x_nstride % 8 == 0
                and x_hstride % 8 == 0 and (x.s is not None or (x.C % 4 == 0 and x.t is not None)))
        use_h = h_ok and (common or split_only)                    # split-only operands exist only in the tensor-core format
        if split_only and not use_h:
            raise lib.TTError(f'conv {name}: an operand is stored as split planes only but the layer cannot run on the f16s kernel')
        use_tc = (impl in (lib.IMPL_TF32, lib.IMPL_3XTF32) and pw.w_tc is not None and common and x.ld % 4 == 0 and x.coff % 4 == 0
                  and x_nstride % 4 == 0 and x_hstride % 4 == 0)
        d.impl = impl if (use_tc or use_h) else lib.IMPL_SIMT
        if use_h:
            self._cur_name = name
            xs = self.with_split(x)
        ws = None
        need = 0 if use_h else lib.load().tt_conv2d_workspace_bytes(C.byref(d))    # SIMT: split-K partials; tensor cores: 0
        if need:
            ws = self.conv_ws.get(self.lane)
            if ws is None or ws.numel() < need:
                if ws is not None:
                    self._ws_retired.append(ws)
                ws = self.conv_ws[self.lane] = torch.empty(int(need * 1.25), dtype=torch.uint8, device=self.device)
        if self.prof is not None:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        # thin 1x1 heads over large maps: per-pixel fp32 mat-vec instead of 128-row tensor-core tiles (tt_pointwise_f16s)
        thin = (use_h and pw.KH == 1 and pw.KW == 1 and stride == 1 and pad == 0 and pw.Cin <= 64 and pw.Cout <= 64 and res is None and res2 is None
                and scatter is None and not x_nstride and not x_hstride and not y_nstride and not bias_n_mod and xs.ld >= -(-pw.Cin // 8) * 8
                and d.N * OH * OW >= self.thin_min_rows)
        if use_h:
            io = lib.F16sIO()
            io.x_split, io.x_plane = _ps(xs)[0], xs.s.numel() // 2
            io.w_split, io.bias = _p(pw.w_h), _p(pw.bias)
            for r, f32, sp, pl in ((res, 'res', 'res_split', 'res_plane'), (res2, 'res2', 'res2_split', 'res2_plane')):
                if r is None:
                    continue
                if r.t is not None:
                    setattr(io, f32, _p(r.t, r.coff))
                else:
                    setattr(io, sp, _p(r.s, r.coff)); setattr(io, pl, r.s.numel() // 2)
            if out.t is not None:
                io.y = _p(out.t, out.coff)
            elif out.s.numel() // 2 <= (1 << 24):
                # small split-only output: lend the kernel an fp32 workspace with the same element grid so that under-filled
                # layers can still run split-K (partial sums are red.add-ed in fp32, the finish pass writes the planes)
                io.y = _p(self.scratch_f32(out.s.numel() // 2), out.coff)
            if out.s is not None:
                io.y_split, io.y_plane = _p(out.s, out.coff), out.s.numel() // 2
            if thin:
                lib.check(lib.load().tt_pointwise_f16s(C.byref(d), lib.ref(io), _p(pw.w), _stream()), f'tt_pointwise_f16s[{name}]')
            else:
                lib.check(lib.load().tt_conv2d_f16s(C.byref(d), lib.ref(io), _stream()), f'tt_conv2d_f16s[{name}]')
        else:
            pres = _p(res.t, res.coff) if res is not None else None
            pres2 = _p(res2.t, res2.coff) if res2 is not None else None
            lib.check(lib.load().tt_conv2d(
                C.byref(d), _p(x.t, x.coff), _p(pw.w_tc if use_tc else pw.w), _p(pw.bias), pres, pres2,
                None, None, _p(out.t, out.coff), _p(ws), _stream()), f'tt_conv2d[{name}]')
            if out.s is not None:
                if y_nstride or scatter is not None:                  # strided / scattered rows: refresh the whole buffer's companion
                    self.sync_split(FMap(out.t, out.t.numel() // out.ld, 1, 1, out.ld, out.ld, 0, out.s))
                else:
                    self.sync_split(out)
        if self.prof is not None:
            ev1.record()
            flops = 2.0 * d.N * OH * OW * (pw.alg_k or pw.KH * pw.KW * pw.Cin // pw.groups) * pw.Cout
            self.prof.append((name, flops, ev0, ev1))
        return out

    def linear(self, x, pw, out=None, name=None, act=0, res=None):
        """x: FMap with H=W=1 (rows in N) or any FMap (flattened over pixels)."""
        xr = x.as_rows()
        if out is None:
            out = self.fmap(name, xr.N, 1, 1, pw.Cout)
        else:
            out = out.as_rows()
        return self.conv(xr, pw, out=out, name=name, act=act, res=res.as_rows() if res is not None else None)

    def sparse_feats(self, name, rows, Cc, f32=True):
        """(fp32 rows [rows][C] or None, split companion [2][rows*C] or None) for a sparse feature matrix.  f32=False: rows that only
        the output-stationary f16s convolutions read (operands and residuals from the planes) keep no fp32 copy."""
        sc = self.buf(name + '#s', (2, rows * Cc), torch.float16, zero=True) if self.split and Cc % 8 == 0 and Cc >= 32 else None
        t = self.buf(name, (rows, Cc)) if (f32 or sc is None) else None
        return t, sc

    def sparse_conv(self, feats, pw, rule, out, act=0, res=None, name=None, feats_s=None, out_s=None, res_s=None):
        """sparse conv over a rulebook `rule` (dict from LidarNet._rulebook): feats [cap_in][Cin] -> out [cap_out][Cout].
        feats_s / out_s / res_s: scaled-split companions of the input / output / residual rows (f16s engine); with the output-
        stationary form any of the fp32 tensors may be None (planes only)."""
        d = lib.SparseConvDesc()
        d.Cin, d.Cout, d.kvol = pw.Cin, pw.Cout, rule['kvol']
        d.in_ld, d.out_ld = pw.Cin, pw.Cout                         # sparse feature matrices are dense rows
        d.res_ld = pw.Cout if (res is not None or res_s is not None) else 0
        d.cap_out, d.pair_cap, d.act = rule['cap'], rule['cap'], act
        wide = pw.Cin >= 32 and pw.Cout >= 32 and rule['kvol'] <= 32
        use_h = (self.impl == lib.IMPL_F16S and pw.w_h is not None and feats_s is not None and wide and pw.Cin % 8 == 0 and d.in_ld % 8 == 0
                 and d.out_ld % 4 == 0)
        use_tc = (self.impl in (lib.IMPL_TF32, lib.IMPL_3XTF32) and pw.w_tc is not None and wide
                  and pw.Cin % 4 == 0 and d.in_ld % 4 == 0 and d.out_ld % 4 == 0)
        d.impl = self.impl if (use_tc or use_h) else lib.IMPL_SIMT
        if self.prof is not None:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        if use_h and rule.get('nbr') is not None:                  # output-stationary form: one launch, fused epilogue, no atomics
            io = lib.F16sIO()
            io.x_split, io.x_plane = _p(feats_s), feats_s.numel() // 2
            io.w_split, io.bias = _p(pw.w_h), _p(pw.bias)
            if res is not None:
                io.res = _p(res)
            elif res_s is not None:
                io.res_split, io.res_plane = _p(res_s), res_s.numel() // 2
            if out is not None:
                io.y = _p(out)
            if out_s is not None:
                io.y_split, io.y_plane = _p(out_s), out_s.numel() // 2
            lib.check(lib.load().tt_sparse_conv_os_f16s(C.byref(d), lib.ref(io), _p(rule['nbr']), _p(rule['count']), _stream()),
                      f'tt_sparse_conv_os_f16s[{name}]')
        elif feats is None or out is None or (res is None and res_s is not None):
            raise lib.TTError(f'sparse conv {name}: planes-only rows need the output-stationary f16s form')
        elif use_h:
            lib.check(lib.load().tt_sparse_conv_f16s(C.byref(d), _p(feats_s), C.c_longlong(feats_s.numel() // 2), _p(pw.w_h), _p(pw.bias), _p(res),
                                                     _p(rule['pairs_in']), _p(rule['pairs_out']), _p(rule['pair_count']), _p(rule['count']), _p(out),
                                                     _p(out_s), C.c_longlong(out_s.numel() // 2 if out_s is not None else 0), _stream()),
                      f'tt_sparse_conv_f16s[{name}]')
        else:
            lib.check(lib.load().tt_sparse_conv(C.byref(d), _p(feats), _p(pw.w_tc if use_tc else pw.w), _p(pw.bias), _p(res), _p(rule['pairs_in']),
                                                _p(rule['pairs_out']), _p(rule['pair_count']), _p(rule['count']), _p(out),
                                                _stream()), f'tt_sparse_conv[{name}]')
            if out_s is not None:                                    # rows produced by the SIMT kernel: convert the first *count of them
                lib.call('tt_split_f16', _p(out), C.c_longlong(out.shape[1]), _p(out_s), C.c_longlong(out_s.numel() // 2), C.c_longlong(out.shape[1]),
                         C.c_longlong(out.shape[0]), out.shape[1], _p(rule['count']))
        if self.prof is not None:
            ev1.record()
            self.prof.append((f'sparse.{name}', 0.0, ev0, ev1))    # data-dependent work: algorithmic FLOPs not counted
        return out

    # ------------------------------------------------------------------ memory-bound ops
    def nchw_to_nhwc(self, x, name, cpad=None):
        N, Cc, H, W = x.shape
        cpad = cpad or Cc
        out = self.fmap(name, N, H, W, cpad)
        lib.call('tt_nchw_to_nhwc', _p(x), _p(_t(out)), N, Cc, H, W, out.ld, 0, cpad)
        return self.sync_split(out)

    def nchw_to_nhwc_padded(self, x, name, cpad, top, bottom, left, right):
        """NCHW -> channels-last inside a zero-bordered [N][top+H+bottom][left+W+right][cpad] buffer (zeroed once at
        allocation; the border is never written afterwards).  Returns the raw buffer."""
        N, Cc, H, W = x.shape
        out = self.buf(name, (N, top + H + bottom, left + W + right, cpad), zero=True)
        lib.call('tt_nchw_to_nhwc_padded', _p(x), _p(out), N, Cc, H, W, cpad, cpad, top + H + bottom, left + W + right, top, left)
        return out

    def nhwc_to_nchw(self, x, name):
        out = self.buf(name, (x.N, x.C, x.H, x.W))
        lib.call('tt_nhwc_to_nchw', _p(_t(x), x.coff), x.ld, 0, _p(out), x.N, x.C, x.H, x.W)
        return out

    def maxpool3x3s2(self, x, name, fmt=None):
        assert x.ld == x.C and x.coff == 0
        self.need_f32(x, 'maxpool3x3s2')
        out = self.out_map(name, x.N, (x.H + 2 - 3) // 2 + 1, (x.W + 2 - 3) // 2 + 1, x.C, fmt)
        lib.call('tt_maxpool3x3s2', _p(_t(x)), _p(_t(out)), x.N, x.H, x.W, x.C)
        return self.finish_out(out)

    def upsample2x(self, x, name, fmt=None):
        assert x.ld == x.C and x.coff == 0
        self.need_f32(x, 'upsample2x')
        if fmt == 's' and self.split:
            out = self.fmap(name, x.N, 2 * x.H, 2 * x.W, x.C, fmt='s')
            if out.t is None:                                        # planes only: written directly, no fp32 copy of the 4x larger map
                lib.call('tt_upsample2x_bilinear_ac_split', _p(x.t), _p(out.s), C.c_longlong(out.s.numel() // 2), x.N, x.H, x.W, x.C)
                return out
        out = self.out_map(name, x.N, 2 * x.H, 2 * x.W, x.C, fmt)
        lib.call('tt_upsample2x_bilinear_ac', _p(_t(x)), _p(_t(out)), x.N, x.H, x.W, x.C)
        return self.finish_out(out)

    def global_avgpool(self, x, name):
        out = self.fmap(name, x.N, 1, 1, x.C)
        lib.call('tt_global_avgpool', _p(_t(x), x.coff), x.ld, 0, _p(_t(out)), x.N, x.H * x.W, x.C)
        return self.sync_split(out)

    def broadcast_rows(self, v, out):
        lib.call('tt_broadcast_rows', _p(_t(v), v.coff), _p(_t(out), out.coff), out.N, out.H * out.W, out.C, out.ld, 0)
        return self.sync_split(out)

    def se_gate(self, x, g, name, fmt=None):
        assert x.ld == x.C and x.coff == 0 and g.ld == g.C
        self.need_f32(x, 'se_gate')
        out = self.out_map(name, x.N, x.H, x.W, x.C, fmt)
        lib.call('tt_se_gate', _p(_t(x)), _p(_t(g)), _p(_t(out)), x.N, x.H * x.W, x.C)
        return self.finish_out(out)

    def se_pool(self, x, name):
        assert x.ld == x.C and x.coff == 0
        out = self.fmap(name, x.N, 1, 1, x.C)
        lib.call('tt_se_pool', _p(_t(x)), _p(_t(out)), x.N, x.H * x.W, x.C)
        return self.sync_split(out)

    def se_apply(self, x, g, shortcut, out=None, name=None):
        assert x.ld == x.C and x.coff == 0
        if out is None:
            out = self.fmap(name, x.N, x.H, x.W, x.C)
        lib.call('tt_se_apply', _p(_t(x)), _p(_t(g)), _p(_t(shortcut), shortcut.coff), shortcut.ld, 0, _p(_t(out), out.coff),
                 out.ld, 0, x.N, x.H * x.W, x.C)
        return self.sync_split(out)

    def anti_transpose(self, x, name):
        assert x.ld == x.C and x.coff == 0 and x.H == x.W
        out = self.fmap(name, x.N, x.H, x.W, x.C)
        lib.call('tt_anti_transpose', _p(_t(x)), _p(_t(out)), x.N, x.H, x.C)
        return self.sync_split(out)

    def copy_cols(self, src, dst, rdiv=1, rmod=None):
        """dst rows r (all pixels of dst) <- src row (r // rdiv) % rmod; copies src.C columns."""
        rows = dst.rows()
        rmod = rmod if rmod is not None else max(src.rows(), 1)
        assert src.C == dst.C
        if dst.t is None and src.t is not None and src.s is None and rdiv == 1 and rmod >= rows:
            if (src.C | src.coff | src.ld | dst.coff | dst.ld) % 4:
                raise lib.TTError('copy_cols: fp32 -> split planes needs 4-column alignment')
            lib.call('tt_split_f16', _p(src.t, src.coff), C.c_longlong(src.ld), _p(dst.s, dst.coff), C.c_longlong(dst.s.numel() // 2),
                     C.c_longlong(dst.ld), C.c_longlong(rows), src.C, None)
            return dst
        if dst.t is None or src.t is None:
            # plane-to-plane copy (both maps are stored as split planes): two halves travel as one 4-byte word
            if src.s is None or dst.s is None or (src.C | src.ld | src.coff | dst.ld | dst.coff) % 2:
                raise lib.TTError('copy_cols: a split-only map can only be copied from / to split planes (even offsets)')
            for pl_s, pl_d in ((0, 0), (src.s.numel() // 2, dst.s.numel() // 2)):
                lib.call('tt_copy2d', _p(src.s, src.coff + pl_s), src.ld // 2, _p(dst.s, dst.coff + pl_d), dst.ld // 2, rows, src.C // 2, rdiv, rmod)
            if dst.t is not None:                                   # the destination also keeps an fp32 copy: rebuild it from its planes
                self.merge_split(dst)
            return dst
        lib.call('tt_copy2d', _p(_t(src), src.coff), src.ld, _p(_t(dst), dst.coff), dst.ld, rows, src.C, rdiv, rmod)
        return self.sync_split(dst)

    def layernorm(self, x, gamma, beta, out=None, name=None, out_ld=None, row_count=None):
        xr = x.as_rows()
        if out is None:
            out = self.fmap(name, xr.N, 1, 1, xr.C, out_ld, zero=True)
        lib.call('tt_layernorm', _p(_t(xr), xr.coff), xr.ld, _p(gamma), _p(beta), _p(_t(out), out.coff), out.ld, xr.N, xr.C,
                 _p(row_count))
        return self.sync_split(out)

    def eltwise(self, op, a, b=None, c=None, out=None, name=None, act=0):
        a_, b_, c_ = a.as_rows(), (b.as_rows() if b is not None else None), (c.as_rows() if c is not None else None)
        if out is None:
            out = self.fmap(name, a.N, a.H, a.W, a.C)
        o_ = out.as_rows()
        lib.call('tt_eltwise', op, act, _p(_t(a_), a_.coff), a_.ld, _p(_t(b_), b_.coff) if b_ else None, b_.ld if b_ else 0,
                 _p(_t(c_), c_.coff) if c_ else None, c_.ld if c_ else 0, _p(_t(o_), o_.coff), o_.ld, a_.N, a_.C)
        return self.sync_split(out)

    def fill(self, t, v=0.0):
        lib.call('tt_fill', _p(t), C.c_float(v), C.c_longlong(t.numel()))
        return t
