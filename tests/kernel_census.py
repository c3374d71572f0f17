"""A shadow harness for the C ABI — TEST HARNESS ONLY.  `install()` wraps `lib.load()` in a proxy: every kernel entry the product
calls is intercepted, its operands and destination buffers are snapshotted, the real entry runs, and its output is compared element
by element with a float64 reference computed from the snapshot on the same device.  The reference is the contract as tests/emu_lib.py
restates it (the convolutions through `emu_lib.conv_ref`, the other entries by running the emulated entry on float64 copies of the
operands), so the emulator and the census share one restatement.

Per call the harness synchronises, snapshots, runs the entry, synchronises again and checks:
  * the elements the contract says are written, against the reference within a per-element bound (or bitwise);
  * every other element of each destination buffer, bitwise unchanged (concat neighbours, pad columns of `ld`, scatter holes, rows of
    a `y_nstride` buffer that belong to other steps);
  * for the f16s convolutions, that the split planes they write decode to their own fp32 output;
  * for the two loss entries (the open-loop validation forward), that every operand they read is bitwise unchanged.
Entries that have full-shape checkers of their own are listed in COVERED_ELSEWHERE and only counted; an entry that is in neither map is
reported, so a new kernel cannot slip in unchecked.

On the GPU the synchronisation serialises the side streams; that changes timing, not results (CUDA graphs stay off): every access across
streams is ordered by an event (the audit of tests/test_stream_order_gpu.py), and adversarial schedules match the serial forward.
"""
import ctypes as C
import inspect
import math
from collections import defaultdict

import torch

import emu_camera_losses
import emu_frames
import emu_lib
import emu_losses
from emu_lib import IO, NULL, Ptr, _desc, _pix_view, _split_f16, conv_ref, y_region

U = 2.0 ** -24                       # unit roundoff of round-to-nearest fp32
U64 = 2.0 ** -53                     # ... of fp64 (the loss kernels accumulate in fp64)
SPLIT = 2.0 ** -22                   # hi + lo'/2048 carries an fp32 value to 2^-22 relative ...
SPLIT_ABS = 2.0 ** -35               # ... down to the fp16 subnormal step of lo' (2^-24 / 2048)
MSDA_TOL = 2e-5                      # tests/test_independent_frames_gpu.py: fp32 sample positions, relative to max |ref| of the call

COVERED_ELSEWHERE = {
    'tt_lift_splat': 'tests/test_camera_look_gpu.py::test_lift_splat_full_batch_both_sweeps_workspace_reuse_and_run_to_run',
    'tt_look_project': 'tests/test_camera_look_gpu.py::test_look_project_and_rebatch_full_batch',
    'tt_look_rebatch': 'tests/test_camera_look_gpu.py::test_look_project_and_rebatch_full_batch',
    'tt_dcn_im2col': 'tests/test_camera_look_gpu.py::test_dcn_im2col_depth_net_shape',
    'tt_gru_input': 'tests/test_camera_look_gpu.py::test_gru_input_columns_and_sentinels',
    'tt_voxelize_mean': 'tests/test_lidar_sparse_gpu.py::test_voxelize_matches_hard_voxelize_and_the_fp64_mean_of_the_first_points',
    'tt_sparse_rulebook': 'tests/test_lidar_sparse_gpu.py::test_rulebooks_match_the_reference',
    'tt_sparse_conv': 'tests/test_lidar_sparse_gpu.py::test_encoder_layer_by_layer_matches_the_fp64_oracle',   # the 16-channel blocks
    'tt_sparse_conv_f16s': 'tests/test_lidar_sparse_gpu.py::test_f16s_sparse_conv_matches_fp64',
    'tt_sparse_conv_os_f16s': 'tests/test_lidar_sparse_gpu.py::test_f16s_sparse_conv_matches_fp64',
    'tt_sparse_to_bev': 'tests/test_lidar_sparse_gpu.py::test_encoder_layer_by_layer_matches_the_fp64_oracle',
    'tt_preprocess_u8': 'tests/test_preprocess_gpu.py::test_stem_planes_at_the_agent_shape',
}
NOT_KERNELS = {'tt_version', 'tt_last_error', 'tt_launch_count', 'tt_debug_set', 'tt_f16s_saturation_count'}

# destination arguments of each checked entry (names of the emulated entry's parameters; `io.*` = fields of the tt_f16s_io)
OUTPUTS = {
    'tt_conv2d': ('y',), 'tt_conv2d_f16s': ('io.y', 'io.y_split'), 'tt_pointwise_f16s': ('io.y', 'io.y_split'),
    'tt_split_f16': ('y_split',), 'tt_merge_f16': ('y',), 'tt_image_to_split8': ('y_split',), 'tt_upsample2x_bilinear_ac_split': ('y_split',),
    'tt_copy2d': ('dst',), 'tt_anti_transpose': ('y',), 'tt_nchw_to_nhwc': ('y',), 'tt_nchw_to_nhwc_padded': ('y',), 'tt_nhwc_to_nchw': ('y',),
    'tt_broadcast_rows': ('y',), 'tt_fill': ('y',), 'tt_maxpool3x3s2': ('y',), 'tt_upsample2x_bilinear_ac': ('y',),
    'tt_global_avgpool': ('y',), 'tt_se_pool': ('s',), 'tt_se_gate': ('y',), 'tt_se_apply': ('y',), 'tt_layernorm': ('y',),
    'tt_eltwise': ('y',), 'tt_msda_forward': ('out',), 'tt_msda_forward_frames': ('out',), 'tt_look_reduce': ('out',),
    'tt_look_reduce_frames': ('out',), 'tt_loss_reduce': ('out',), 'tt_camera_loss': ('out',),
}
IO_FIELDS = ('x_split', 'w_split', 'bias', 'res', 'res_split', 'res2', 'res2_split', 'y', 'y_split')
CONVS = ('tt_conv2d', 'tt_conv2d_f16s', 'tt_pointwise_f16s')
KEEP_DTYPE = {'tt_copy2d'}           # moves 4-byte words (a pair of halves is one word): its operands keep their dtype


class CensusError(AssertionError):
    pass


def _bits(t):
    return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16}[t.element_size()])


# ---------------------------------------------------------------------------------------------------------- activations
# (Lipschitz constant L, evaluation error in units of U times the pre-activation magnitude, ... times |result|) of csrc/common.cuh
# tt_act.  GELU = 0.5 v (1 + erff(v / sqrt 2)): |gelu'| <= 1.13; erff is within 2 ulp and the three fp32 operations add at most 8 U |v|.
# SIGMOID = 1 / (1 + expf(-v)): |s'| <= 1/4; expf within 2 ulp (4 U relative), 1 + e and the division: <= 8 U |result|.  SOFTPLUS =
# log1pf(expf(v)): slope <= 1; a relative error d of expf moves the result by d e / (1 + e) <= d log1p(e), log1pf adds 2 U: <= 8 U |result|.
ACT_ERR = {0: (1.0, 0, 0), 1: (1.0, 0, 0), 2: (1.13, 8, 0), 3: (0.25, 0, 8), 4: (1.0, 0, 8), 5: (1.0, 0, 8)}


def act_bound(act, c, mag, ref):
    """|got - ref| bound of act(sum) when the fp32 sum is within c U mag of the exact one, rounded once more to fp32."""
    L, a_mag, a_ref = ACT_ERR[act]
    return (L * c + a_mag) * U * mag + (1 + a_ref) * U * ref.abs()


def conv_c(name, d, K, chunk=2):
    """c of the conv bound |y - ref| <= act_bound(c, magnitude), magnitude = conv(|x|, |w|) + |bias| + |res| + |res2|.

    tt_conv2d_f16s (csrc/gemm_conv_f16s.cu): the reference reads the decoded split operands, so the only operand error is the
    dropped lo'·lo' product, |lo'_x lo'_w| / 2048^2 <= 2^-11 |x| 2^-11 |w| = 4 U |x||w|.  The register accumulator is folded every
    `chunk` K stages of 64 (2 by default; 1 / 4 under the debug bits 0x40000 / 0x20000): a fold of 64 chunk K is 4 chunk wgmma
    k16 steps into an accumulator that is not rounded to nearest: count 2 ulp (4 U) of the fold's magnitude per step, doubled for
    the correction accumulator and its 2^-11 scaling: 32 chunk U per fold, so 32 chunk U of the whole magnitude.  The fp32 register
    sums add main + 2^-11 corr once per fold (two roundings) over nc = ceil(K / (64 chunk)) folds, and split-K red.add-s at most
    nc partial sums: 4 nc U.  Bias, two residuals and the fp32 store: 4 U.  So c = 4 + 32 chunk + 4 nc + 4 (72 + 4 nc at chunk 2).
    tt_pointwise_f16s: the input decoded in fp32 (1 U) and a K-term fp32 FMA chain: c = K + 4.
    tt_conv2d impl 0/1 (SIMT FFMA): K FMA roundings, plus a deterministic split-K reduction of at most K partial sums: c = 2 K + 8;
    impl 2/3 (TF32 pairs) also round the activation operand to 2^-22 (4 U): c = 2 K + 16."""
    if name == 'tt_conv2d_f16s':
        return 8 + 32 * chunk + 4 * math.ceil(K / (64 * chunk))
    if name == 'tt_pointwise_f16s':
        return K + 4
    return 2 * K + (16 if d.impl >= 2 else 8)


# ---------------------------------------------------------------------------------------------------------- one call
class Call:
    def __init__(self, census, idx, name, args):
        self.census, self.idx, self.name = census, idx, name
        self.fn = getattr(census.ref, name)
        params = list(inspect.signature(self.fn).parameters)
        self.a = dict(zip(params, args))
        self.d = _desc(self.a['d']) if 'd' in self.a else None
        self.p = {}                                                    # argument name -> Ptr of the real buffer
        self.planes, self.null = {}, set()
        for k, v in self.a.items():
            if k == 'io':
                io = _desc(v)
                for f in IO_FIELDS:
                    r = census.resolve(getattr(io, f), f'io.{f}')
                    if r:
                        self.p[f'io.{f}'] = r
                self.planes = {f: int(getattr(io, f)) for f in ('x_plane', 'res_plane', 'res2_plane', 'y_plane')}
            elif k not in ('d', 'stream'):
                r = census.resolve(v, k)
                if isinstance(r, Ptr):
                    if r:
                        self.p[k] = r
                    else:
                        self.null.add(k)
        self.decoded = {}                                              # argument name -> fmap -> the argument the reference runs on
        if name in DECODE:                                             # operands behind pointers inside a table or descriptor
            DECODE[name](self)
        self.outs = [k for k in OUTPUTS[name] if k in self.p]
        names = [census.namer(self.p[k].t) for k in self.outs]
        self.layer = next((n for n in names if n != 'scratch'), names[0] if names else '?')
        self.launches, self.ratio, self.where, self.planes_ratio = 0, 0.0, '', 0.0
        keep = name in KEEP_DTYPE
        self.dt = lambda t: t.dtype if keep or not t.is_floating_point() else torch.float64
        self.src = {}                                                  # (id(tensor), map tag) -> fp64 copy taken before the call
        self.skip = False
        if name in CONVS:                                              # fp64 copies of the operand windows only (conv_snapshot)
            self.win = conv_snapshot(self)
            self.snap = {k: self.p[k].t.clone() for k in self.outs} if census.outside else {}
        else:
            tensors = {id(p.t): p.t for k, p in self.p.items() if k not in self.outs}
            # fp64 source copies; per destination element the snapshot, two fp64 reference runs and the fill of the second, the
            # written mask, the gathered got / want / bound / ratio and their indices: about 80 bytes
            need = sum(t.numel() * 8 for t in tensors.values()) + sum(self.p[k].t.numel() * 80 for k in self.outs)
            if census.cap is not None and need > census.cap:           # no window for this entry: counted as skipped in the table
                self.skip = True
                return
            for t in tensors.values():
                self.src[(id(t), None)] = t.to(self.dt(t), copy=True)
            self.snap = {k: self.p[k].t.clone() for k in self.outs}

    # ------------------------------------------------------------------ reference runs
    def src_ptr(self, k, fmap=None):
        p = self.p[k]
        key = (id(p.t), k if fmap and k in fmap else None)
        if key not in self.src:
            self.src[key] = fmap[k](self.src[(id(p.t), None)])
        return Ptr(self.src[key], p.off)

    def io(self):
        """the tt_f16s_io of the call with its operands pointing at the snapshot (outputs NULL)."""
        io = IO()
        for f in IO_FIELDS:
            k = f'io.{f}'
            if k in self.p and k not in self.outs:
                setattr(io, f, self.src_ptr(k))
        for f, v in self.planes.items():
            setattr(io, f, v)
        return io

    def run_ref(self, fill=None, fmap=None):
        """the emulated entry on fp64 copies of the snapshot: {destination: its fp64 copy after the call}.  Sources are read from
        their own copies, so a destination that shares a buffer with a source (concat, in place) reads the pre-call values."""
        dest, args = {}, []
        for k in self.outs:
            t = self.snap[k].to(self.dt(self.snap[k]), copy=True)
            dest[k] = fill(t) if fill is not None else t
        for k, v in self.a.items():
            if k in self.outs:
                args.append(Ptr(dest[k], self.p[k].off))
            elif k in self.decoded:
                args.append(self.decoded[k](fmap))
            elif k in self.p:
                args.append(self.src_ptr(k, fmap))
            elif k in self.null:
                args.append(NULL)
            elif k == 'stream':
                args.append(None)
            else:
                args.append(v)
        self.fn(*args)
        return dest

    def reference(self):
        """(reference destinations, written masks): an element is written when two runs that start from different destination
        contents agree on it bitwise."""
        a = self.run_ref()
        b = self.run_ref(fill=lambda t: torch.where(t == 0.5, torch.full_like(t, 0.25), torch.full_like(t, 0.5)))
        return a, {k: _bits(a[k]) == _bits(b[k]) for k in a}

    # ------------------------------------------------------------------ comparisons
    def where_str(self, k, flat_idx):
        t = self.p[k].t
        pos = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat_idx), tuple(t.shape)))
        return f'{k} element {pos} of {tuple(t.shape)}'

    def fail(self, what):
        msg = (f'call #{self.idx} {self.name} [{self.layer}] (launches {self.launches}, impl {getattr(self.d, "impl", "-")}): {what}')
        self.census.failures.append(msg)
        if self.census.stop:
            raise CensusError(msg)

    def check_outside(self, k, mask):
        if not self.census.outside or self.census.is_scratch(self.p[k].t):
            return
        got = self.p[k].t.reshape(-1)
        bad = (_bits(got) != _bits(self.snap[k].reshape(-1))) & ~mask.reshape(-1)
        if bool(bad.any()):
            i = int(bad.nonzero()[0])
            self.fail(f'write outside the destination: {int(bad.sum())} elements changed, first {self.where_str(k, i)} '
                      f'got {float(got[i]):.8g} was {float(self.snap[k].reshape(-1)[i]):.8g}')

    def compare(self, k, got, want, bound, where, planes=False):
        """got / want / bound: same-shape tensors of the written elements; bound None = bitwise.  where(i) names element i.
        planes: the check that split planes encode the call's own fp32 output (its own column of the table)."""
        got, want = got.reshape(-1).double(), want.reshape(-1).double()
        if bound is None:
            ok = (got == want) | (torch.isnan(got) & torch.isnan(want))
            ratio = torch.where(ok, torch.zeros_like(got), torch.full_like(got, math.inf))
        else:
            bound = bound.reshape(-1)
            err = (got - want).abs()
            ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
            ratio = torch.nan_to_num(ratio, nan=math.inf)
        if not ratio.numel():
            return
        i = int(ratio.argmax())
        r = float(ratio[i])
        if planes:
            self.planes_ratio = max(self.planes_ratio, r)
        elif r > self.ratio:
            self.ratio, self.where = r, where(i)
        if not r < 1:
            b = 'bitwise' if bound is None else f'{float(bound[i]):.3g}'
            self.fail(f'{k}: {int((ratio >= 1).sum())} elements beyond the bound, worst at {where(i)}: got {float(got[i]):.9g} '
                      f'want {float(want[i]):.9g} bound {b} (ratio {r:.3g})')

    def compare_written(self, k, want, mask, bound=None):
        idx = mask.reshape(-1).nonzero().squeeze(1)
        self.compare(k, self.p[k].t.reshape(-1)[idx], want.reshape(-1)[idx], None if bound is None else bound.reshape(-1)[idx],
                     lambda i: self.where_str(k, int(idx[i])))
        self.check_outside(k, mask)


# ---------------------------------------------------------------------------------------------------------- entry checks
def _conv_strides(d):
    """elements between consecutive images of x, res, res2 and y."""
    sx = d.x_nstride or d.H * (d.x_hstride or d.W * d.x_ld)
    sr = (d.res_H * d.res_W if d.res_mode == 2 else d.OH * d.OW) * d.res_ld
    return sx, sr, d.OH * d.OW * d.res2_ld, d.y_nstride or d.yH * d.yW * d.y_ld


def conv_windows(d, window):
    """[(first image, images)] a call is checked on: all N, or (window) the first w images and the images from the last multiple of
    bias_n_mod at or below N - w to the end: w is a multiple of bias_n_mod (every residue in each window, and each window's image i
    takes bias row i % bias_n_mod) and covers >= 256 output rows (a linear is N images of 1 x 1)."""
    if not window:
        return [(0, d.N)]
    k = max(d.bias_n_mod, 1)
    w = max(k, -(-256 // max(d.OH * d.OW, 1)))
    w = -(-w // k) * k
    n1 = (d.N - w) // k * k
    return [(0, d.N)] if w >= n1 else [(0, w), (n1, d.N - n1)]


def _window(p, start, length, plane=None):
    """fp64 copy of `length` elements from `start` past p (and of the same range of the lo' plane `plane` elements further):
    (Ptr to the copy, its plane stride)."""
    flat, a = p.t.reshape(-1), p.off + start
    if plane is None:
        return Ptr(flat[a:a + length].to(torch.float64)), 0
    n = min(length, flat.numel() - plane - a)
    return Ptr(torch.cat([flat[a:a + n], flat[a + plane:a + plane + n]]).to(torch.float64)), n


def conv_snapshot(c):
    """before the call: per window (conv_windows), a descriptor for its images and fp64 copies of the input and residual images it
    reads.  Weights and bias are read in place (the forward never writes them)."""
    d, f16s = c.d, c.name != 'tt_conv2d'
    sx, sr, s2, _ = _conv_strides(d)
    g = lambda k: c.p.get(k, NULL)
    wins = []
    for n0, w in conv_windows(d, c.census.window):
        dw = type(d).from_buffer_copy(d)
        dw.N = w
        bias = g('io.bias' if f16s else 'bias')
        if f16s:
            io = IO()
            io.x_split, io.x_plane = _window(c.p['io.x_split'], n0 * sx, w * sx, c.planes['x_plane'])
            io.w_split, io.bias = g('io.w_split'), bias
            for f, s_ in (('res', sr), ('res2', s2)):
                if f'io.{f}' in c.p:
                    setattr(io, f, _window(c.p[f'io.{f}'], n0 * s_, w * s_)[0])
                if f'io.{f}_split' in c.p:
                    ptr, n = _window(c.p[f'io.{f}_split'], n0 * s_, w * s_, c.planes[f'{f}_plane'])
                    setattr(io, f'{f}_split', ptr)
                    setattr(io, f'{f}_plane', n)
            ops = (io,)
        else:
            win = lambda k, s_: _window(c.p[k], n0 * s_, w * s_)[0] if k in c.p else NULL
            ops = (win('x', sx), g('w'), bias, win('res', sr), win('res2', s2))
        wins.append((n0, dw, ops))
    return wins


def check_conv(c):
    """per window: y against conv_ref within the conv bound, and the split planes bitwise the _split_f16 of the call's own fp32 y (or,
    for a planes-only output, their value within the bound + 2^-22); then, over the whole buffers, nothing outside the region."""
    d, f16s = c.d, c.name != 'tt_conv2d'
    K = d.KH * d.KW * (d.Cin // d.groups)
    sy = _conv_strides(d)[3]
    yk, sk = ('y', None) if not f16s else ('io.y', 'io.y_split')
    y, ys = c.p.get(yk), c.p.get(sk) if sk else None
    plane = c.planes.get('y_plane', 0)
    for n0, dw, ops in c.win:
        if c.name == 'tt_pointwise_f16s':
            io = ops[0]
            val, mag = conv_ref(dw, io.x_split, c.p['w_kmajor'], io.bias, NULL, NULL, io, kmajor_w=True, magnitude=True)
        elif f16s:
            io = ops[0]
            val, mag = conv_ref(dw, io.x_split, io.w_split, io.bias, io.res, io.res2, io, magnitude=True)
        else:
            val, mag = conv_ref(dw, *ops, magnitude=True)
        bound = act_bound(d.act, conv_c(c.name, d, K), mag, val)
        del mag

        def pos(i):
            n, oy, ox, ch = (int(v) for v in torch.unravel_index(torch.tensor(i % val.numel()), tuple(val.shape)))
            return f'(image {n0 + n}, y {oy}, x {ox}, channel {ch}) of ({d.N}, {d.OH}, {d.OW}, {d.Cout})'
        y32 = None
        if y:
            y32 = y_region(dw, Ptr(y.t, y.off + n0 * sy))
            c.compare(yk, y32, val, bound, pos)
        if ys:
            hi = y_region(dw, Ptr(ys.t, ys.off + n0 * sy))
            lo = y_region(dw, Ptr(ys.t, ys.off + plane + n0 * sy))
            if y32 is not None and not c.census.is_scratch(y.t):
                h, l = _split_f16(y32)
                c.compare(sk, torch.stack([hi, lo]), torch.stack([h, l]), None, lambda i: f'plane {i // val.numel()} {pos(i)}', planes=True)
            else:
                dec = hi.double() + lo.double() / 2048.0
                c.compare(sk, dec, val, bound + SPLIT * val.abs() + SPLIT_ABS, pos)
        del val, bound
    if c.census.outside:
        for k, planes in ((yk, (0,)), (sk, (0, plane))):               # the descriptor's region, as a mask of each buffer
            if k and k in c.p:
                m = torch.zeros(c.p[k].t.shape, dtype=torch.float32, device=c.p[k].t.device)
                for pl in planes:
                    y_region(d, Ptr(m, c.p[k].off + pl))[...] = 1.0
                c.check_outside(k, m != 0)


def check_exact(c):
    ref, mask = c.reference()
    for k in c.outs:
        c.compare_written(k, ref[k], mask[k])


def bounded(bound_fn):
    """bound_fn(call, reference destinations, written masks) -> {destination: per-element bound over the whole destination}."""
    def check(c):
        ref, mask = c.reference()
        bounds = bound_fn(c, ref, mask)
        for k in c.outs:
            c.compare_written(k, ref[k], mask[k], bounds[k])
    return check


def _abs_of(*names):
    return {k: torch.abs for k in names}


def _upsample_dims(c):
    return tuple(int(emu_lib._v(c.a[k])) for k in ('N', 'H', 'W', 'Cc'))


def _upsample_bound(c):
    """bilinear, align_corners: the source position o (H - 1) / (2H - 1) is formed in fp32 (absolute error <= 2 U H), so the lerp
    weights are off by <= 2 U (H + W) in sum, each multiplied by a corner difference <= the sum S of the 4 corner magnitudes; the
    4 products and 3 sums add 8 U S: U (2H + 2W + 8) S, (N, 2H, 2W, C)."""
    N, H, W, Cc = _upsample_dims(c)
    x = _pix_view(c.src_ptr('x'), N, H, W, Cc).abs()
    iy = (torch.arange(2 * H, device=x.device) * (H - 1)) // max(2 * H - 1, 1)
    ix = (torch.arange(2 * W, device=x.device) * (W - 1)) // max(2 * W - 1, 1)
    iy1, ix1 = (iy + 1).clamp(max=H - 1), (ix + 1).clamp(max=W - 1)
    S = x[:, iy][:, :, ix] + x[:, iy1][:, :, ix] + x[:, iy][:, :, ix1] + x[:, iy1][:, :, ix1]
    return U * (2 * H + 2 * W + 8) * S


def bound_upsample(c, ref, mask):
    """_upsample_bound + U |ref| for the fp32 store."""
    N, H, W, Cc = _upsample_dims(c)
    out = torch.zeros_like(ref['y'])
    view = lambda t: _pix_view(Ptr(t, c.p['y'].off), N, 2 * H, 2 * W, Cc)
    view(out)[...] = _upsample_bound(c) + U * view(ref['y']).abs()
    return {'y': out}


def check_upsample_split(c):
    """the planes must be exactly _split_f16 of the fp32 upsample tt_upsample2x_bilinear_ac computes from the same input, and that
    fp32 upsample must be within bound_upsample of the fp64 one."""
    N, H, W, Cc = _upsample_dims(c)
    n = N * 4 * H * W * Cc
    plane = int(emu_lib._v(c.a['y_plane']))
    ys, x = c.p['y_split'], c.p['x']
    y32 = torch.empty(n, dtype=torch.float32, device=x.t.device)
    c.census.real_entry('tt_upsample2x_bilinear_ac')(c.census.pointer(Ptr(c.src[(id(x.t), None)].float(), x.off)),
                                                      c.census.pointer(Ptr(y32)), N, H, W, Cc, c.census.stream())
    c.census.sync()
    hi, lo = _split_f16(y32)
    got = torch.cat([ys.flat()[:n], ys.flat()[plane:plane + n]])
    c.compare('y_split', got, torch.cat([hi, lo]), None, lambda i: f'plane {i // n} element {i % n} of [{N}][{2 * H}][{2 * W}][{Cc}]')
    exact = torch.nn.functional.interpolate(_pix_view(c.src_ptr('x'), N, H, W, Cc).permute(0, 3, 1, 2), scale_factor=2, mode='bilinear',
                                            align_corners=True).permute(0, 2, 3, 1).reshape(-1)
    c.compare('y_split', y32, exact, _upsample_bound(c).reshape(-1) + U * exact.abs(), lambda i: f'fp32 upsample element {i}')
    m = torch.zeros(ys.t.numel(), dtype=torch.bool, device=ys.t.device)
    for pl in (0, plane):
        m[ys.off + pl:ys.off + pl + n] = True
    c.check_outside('y_split', m)


def bound_pool(c, ref, mask):
    """pool_hw_kernel (csrc/elementwise.cu): each of 8 lanes sums ceil(HW / 8) pixels serially, lane 0 adds the 7 other sums,
    divides by HW and scales (se_pool: 0.5 mean + 0.5 max, two more roundings).  gamma_n with n = ceil(HW / 8) + 7 of the mean of
    |x|, + 4 U: bound = (ceil(HW / 8) + 11) U M, M = the same pool of |x| (>= the mean of |x| and >= |ref|)."""
    HW = int(emu_lib._v(c.a['HW']))
    M = c.run_ref(fmap=_abs_of('x'))
    return {k: (math.ceil(HW / 8) + 11) * U * M[k] for k in c.outs}


def bound_se_gate(c, ref, mask):
    """y = x sigmoid(g): sigmoid within 8 U relative (ACT_ERR), the product 1 U: bound = 10 U |x| sigmoid(g)."""
    M = c.run_ref(fmap=_abs_of('x'))
    return {'y': 10 * U * M['y']}


def bound_se_apply(c, ref, mask):
    """y = relu(x sigmoid(g) + sc): 10 U |x sigmoid(g)| (se_gate) + U |sum|: bound = 11 U (|x| sigmoid(g) + |sc|)."""
    M = c.run_ref(fmap=_abs_of('x', 'sc'))
    return {'y': 11 * U * M['y']}


def bound_look_reduce(c, ref, mask):
    """a sum of at most cap rows (then / B): gamma_{cap + 1} of the same reduce of |rows|."""
    cap = int(emu_lib._v(c.a['cap']))
    M = c.run_ref(fmap=_abs_of('rows'))
    return {'out': (cap + 2) * U * M['out']}


def bound_msda(c, ref, mask):
    """the sampling positions are fp32 (about 1e-6 px at 56 px, tests/test_independent_frames_gpu.py): MSDA_TOL of max |ref| over the
    rows this call writes (rows at or past max_len keep other values)."""
    r = ref['out']
    w = r[mask['out']]
    scale = float(torch.nan_to_num(w, nan=0.0).abs().max()) if w.numel() else 0.0
    return {'out': torch.full_like(r, MSDA_TOL * max(scale, 1e-30))}


def bound_layernorm(c, ref, mask):
    """layernorm_kernel: one warp per row, lane sums of ceil(D / 32) elements + a 5-level shuffle tree, n = ceil(D / 32) + 5.
      mean: |dmu| <= (n + 1) U mean|x|;  x - mu: + U |x - mu|;  variance: relative (n + 3) U (the dmu term cancels to first order,
      sum (x - mu) = 0);  + eps: U;  rsqrtf: 2 ulp (4 U).  So rstd is within ((n + 4) / 2 + 4) U relative, and
      |dy| <= |g| rstd (n + 1) U mean|x| + |g t| ((n + 4) / 2 + 5) U + 3 U (|g t| + |b|),   t = (x - mu) rstd."""
    a = c.a
    rows, D, x_ld, y_ld = (int(emu_lib._v(a[k])) for k in ('rows', 'D', 'x_ld', 'y_ld'))
    n = rows if 'row_count' not in c.p else min(rows, int(c.src_ptr('row_count').flat()[0]))
    x = torch.as_strided(c.src_ptr('x').flat(), (rows, D), (x_ld, 1))[:n]
    g, b = c.src_ptr('gamma').flat()[:D], c.src_ptr('beta').flat()[:D]
    mu = x.mean(1, keepdim=True)
    rstd = ((x - mu).pow(2).mean(1, keepdim=True) + 1e-5).rsqrt()
    t = (x - mu) * rstd
    nn = math.ceil(D / 32) + 5
    bnd = U * (g.abs() * rstd * (nn + 1) * x.abs().mean(1, keepdim=True) + (g * t).abs() * ((nn + 4) / 2 + 8) + 3 * b.abs())
    out = torch.zeros_like(ref['y'])
    torch.as_strided(Ptr(out, c.p['y'].off).flat(), (rows, D), (y_ld, 1))[:n] = bnd
    return {'y': out}


def bound_eltwise(c, ref, mask):
    """csrc/elementwise.cu eltwise_kernel, the pre-activation value v and its error in units of U times a magnitude M:
      op 0  a + b                    one rounding                          M = |a| + |b|,              c = 1
      op 1  (1 - a) b                two                                   M = (1 + |a|) |b|,          c = 2
      op 2  (1 - a) b + a c          four                                  M = (1 + |a|) |b| + |a||c|, c = 4
      op 3  a                        none                                  M = |a|,                    c = 0
      op 4  a + logf(-expm1f(-a))    expm1f 1 ulp moves the log by 2 U, logf and the sum round:  M = |a| + |log| + 1, c = 4
    then the activation (act_bound)."""
    a = c.a
    op, act, rows, cols = (int(emu_lib._v(a[k])) for k in ('op', 'act', 'rows', 'cols'))
    v = lambda k: torch.as_strided(c.src_ptr(k).flat(), (rows, cols), (int(emu_lib._v(a[k + '_ld'])), 1))
    A = v('a')
    if op == 0:
        M, cc = A.abs() + v('b').abs(), 1
    elif op == 1:
        M, cc = (1 + A.abs()) * v('b').abs(), 2
    elif op == 2:
        M, cc = (1 + A.abs()) * v('b').abs() + A.abs() * v('c').abs(), 4
    elif op == 4:
        M, cc = A.abs() + torch.log(-torch.expm1(-A)).abs() + 1, 4
    else:
        M, cc = A.abs(), 0
    y_ld = int(emu_lib._v(a['y_ld']))
    yref = torch.as_strided(Ptr(ref['y'], c.p['y'].off).flat(), (rows, cols), (y_ld, 1))
    out = torch.zeros_like(ref['y'])
    torch.as_strided(Ptr(out, c.p['y'].off).flat(), (rows, cols), (y_ld, 1))[...] = act_bound(act, cc, M, yref)
    return {'y': out}


# ---------------------------------------------------------------------------------------------------------- the loss entries
# tt_loss_reduce and tt_camera_loss read their operands through pointers inside a term table / a descriptor.  DECODE resolves each of
# those pointers through the census's pointer table (the GPU: an address lib._p handed out since the last checked call; the emulated
# ABI: the Ptr itself) into an entry of Call.p named after its place ('terms[3].gt', 'd.seg_logits'), so that the operand is
# snapshotted in fp64 before the call like any other, and rebuilds the table / descriptor over those snapshots for the reference.  A
# pointer made before an earlier checked call is not in the table any more: the census raises instead of reading a stale buffer.
LOSS_PTRS = ('pred', 'pred2', 'gt', 'gt2')
CAM_PTRS = ('seg_logits', 'seg_gt', 'depth_logits', 'depth_gt')


def _operand(c, v, what):
    """a pointer field (an address on the GPU, a Ptr on the emulated ABI) -> its key in c.p, or None for NULL."""
    r = c.census.resolve(v if isinstance(v, Ptr) else C.c_void_p(v or 0), what)
    if not r:
        return None
    c.p[what] = r
    return what


def decode_loss_terms(c):
    """tt_loss_reduce: the tt_loss_term array lib.pack_loss_terms built (or, emulated, the term dicts themselves) -> c.terms, term
    dicts whose pointer fields are keys of c.p; the reference reads them as emu_losses does."""
    terms = []
    for i in range(int(emu_lib._v(c.a['n_terms']))):
        t = c.a['terms'][i]
        if isinstance(t, dict):
            d = {k: v for k, v in t.items() if k not in LOSS_PTRS}
        else:
            nd = t.ndim
            d = dict(kind=t.kind, slot=t.slot, aux=t.aux, scale=t.scale, shape=list(t.shape[:nd]), pred_stride=list(t.pred_stride[:nd]),
                     gt_stride=list(t.gt_stride[:nd]))
        for f in LOSS_PTRS:
            d[f] = _operand(c, t[f] if isinstance(t, dict) else getattr(t, f), f'terms[{i}].{f}')
        terms.append(d)
    c.terms = terms
    c.decoded['terms'] = lambda fmap: [dict(t, **{f: c.src_ptr(t[f], fmap) if t[f] else NULL for f in LOSS_PTRS}) for t in terms]


def decode_camera_desc(c):
    """tt_camera_loss: the tt_camera_loss_desc -> a namespace of its fields for emu_camera_losses, pointers over the snapshots.  The
    ground truth stays fp32 (the kernel bins depths in fp32: an fp64 copy would move values at the bin edges)."""
    from types import SimpleNamespace
    from thinktwice_b200 import lib
    fields = {n: getattr(c.d, n, 0) for n, _ in lib.CameraLossDesc._fields_}
    keys = {f: _operand(c, fields[f], f'd.{f}') for f in CAM_PTRS}
    # a logit map is snapshotted as the (pixels, classes) block the kernel reads, not as its whole buffer (a wide map at B = 16 would
    # pass the working-set cap): the reference reads that block with ld = classes, coff = 0
    for half, n_cls in (('seg', 'seg_classes'), ('depth', 'depth_bins')):
        k = keys[f'{half}_logits']
        if k:
            rows = fields['BN'] * fields[f'{half}_h'] * fields[f'{half}_w']
            ld, coff, n = fields[f'{half}_ld'], fields[f'{half}_coff'], fields[n_cls]
            c.p[k] = Ptr(c.p[k].flat()[:rows * ld].view(rows, ld)[:, coff:coff + n])
            fields[f'{half}_ld'], fields[f'{half}_coff'] = n, 0
    fp32 = {k: torch.Tensor.float for f, k in keys.items() if k and f.endswith('_gt')}
    c.decoded['d'] = lambda fmap: SimpleNamespace(**dict(fields, **{f: c.src_ptr(k, {**fp32, **(fmap or {})}) if k else NULL
                                                                    for f, k in keys.items()}))


DECODE = {'tt_loss_reduce': decode_loss_terms, 'tt_camera_loss': decode_camera_desc}


def _digamma_err(x):
    """|digamma_pos(x) - psi(x)| of csrc/losses.cu, plus the error of the fp64 reference's torch.digamma, for x > 0.
    digamma_pos takes s = ceil(6 - x) recurrence steps r -= 1 / (x + j) to x' = x + s in [6, 7), then ln x' - 1 / (2x') and the
    asymptotic series cut after its x'^-10 term.  The series' remainder is smaller than its first dropped term, 691 / (32760 x'^12)
    (9.7e-12 at x' = 6).  Rounding: the s divisions and subtractions, log, the halving and the 5-term Horner chain in fp64, a few
    roundings of the magnitude |r| + |ln x'| + 1 each; torch.digamma rounds about as often: 32 u64 of that magnitude."""
    s = (6.0 - x).ceil().clamp(min=0)
    xs = x + s
    mag = xs.log().abs() + 1
    for j in range(7):
        mag = mag + torch.where(j < s, 1.0 / (x + j), torch.zeros_like(x))
    return 691.0 / (32760.0 * xs ** 12) + 32 * U64 * mag


def _beta_kl_err(t):
    """per-element |kernel - reference| bound of a BETA_KL term, both in fp64 (csrc/losses.cu beta_kl; torch's _kl_beta_beta is the same
    formula): KL = t1 - t2 + (a1 - a2) psi(a1) + (b1 - b2) psi(b1) + (s2 - s1) psi(s1), t1 = lg a2 + lg b2 + lg s1, t2 = lg a1 + lg b1 + lg s2.
      lgamma: CUDA's is within 4 ulp for x > 0, the reference's about as close; t1 - t2 cancels, so the six lgamma errors and the five
        sums count as an absolute term in the lgamma magnitudes: 24 u64 (sum |lg| + 6), the + 6 standing for the absolute error an
        ulp count does not cover near the zeros of lgamma (x = 1, 2);
      s1 = a1 + b1, s2 = a2 + b2 round once: lgamma moves by |psi(s)| u64 s, psi(s1) by psi'(s1) u64 s1 <= u64 (1 + 1 / s1);
      each psi: _digamma_err, times the difference it multiplies; the three differences, three products and four sums: 8 u64 of
      sum |difference psi| and of |KL|."""
    P, G, P2, G2 = emu_losses.term_operands(t)
    a1, b1, a2, b2 = G, G2, P, P2
    s1, s2 = a1 + b1, a2 + b2
    err = 24 * U64 * (sum(torch.lgamma(x).abs() for x in (a1, b1, s1, a2, b2, s2)) + 6)
    err = err + U64 * (s1 * torch.digamma(s1).abs() + s2 * torch.digamma(s2).abs()) + (s2 - s1).abs() * U64 * (1 + 1 / s1)
    for dlt, x in ((a1 - a2, a1), (b1 - b2, b1), (s2 - s1, s1)):
        err = err + dlt.abs() * (_digamma_err(x) + 8 * U64 * torch.digamma(x).abs())
    return err


def bound_loss_reduce(c, ref, mask):
    """csrc/losses.cu loss_reduce_kernel, per term of n elements: values v_i in fp64; 16 CTAs of 256 threads each sum ceil(n / 4096)
    values serially, then an 8-level tree and the 16 range sums serially: a summation depth of ceil(n / 4096) + 24.  The reference's
    torch sum has depth <= n.  So the two sums differ by at most (ceil(n / 4096) + 24 + n) u64 sum |v_i|, plus sum_i e_i, e_i the
    two evaluations' error on element i:
      SMOOTH_L1 (and the clamped form, 1-Lipschitz) / L1: the fp64 |p - g| of two fp32 values (one rounding when their exponents are far
        apart), 0.5 a a or a - 0.5: 4 u64 |v| each side, 8 u64 |v|;
      BETA_KL: _beta_kl_err;
      ACTION_L1: evaluated in fp32 by both as thinktwice_decoder.py:623-636 does (no FMA can change it: x * 2 is exact), and |x1 - x2| in
        fp64: equal per element, e_i = 0.
    Then scale * sum and the serial sum over the m terms of the slot: (m + 2) u64 of sum |scale| sum |v|; the slot's fp32 store:
    U |ref|.  Every slot below n_slots is written (0 when no term names it): the reference's written mask; what is past it must not
    change."""
    from thinktwice_b200 import lib
    n_slots = int(emu_lib._v(c.a['n_slots']))
    terms = c.decoded['terms'](None)
    per_slot = defaultdict(int)
    for t in terms:
        per_slot[t['slot']] += 1
    b = torch.zeros(n_slots, dtype=torch.float64, device=ref['out'].device)
    for t in terms:
        v = emu_losses.term_values(t)
        n, A = v.numel(), v.abs().sum()
        if t['kind'] in (lib.LOSS_SMOOTH_L1, lib.LOSS_SMOOTH_L1_CLAMP, lib.LOSS_L1):
            e = 8 * U64 * A
        elif t['kind'] == lib.LOSS_BETA_KL:
            e = _beta_kl_err(t).sum() + 8 * U64 * A
        else:
            e = 0.0
        b[t['slot']] += abs(t['scale']) * ((math.ceil(n / 4096) + 24 + n + per_slot[t['slot']] + 2) * U64 * A + e)
    out = torch.zeros_like(ref['out'])
    o = Ptr(out, c.p['out'].off).flat()
    o[:n_slots] = b + U * Ptr(ref['out'], c.p['out'].off).flat()[:n_slots].abs()
    return {'out': out}


def bound_camera_loss(c, ref, mask):
    """csrc/losses.cu camera_loss_kernel against emu_camera_losses, both fp64 up to the final fp32 store.
    seg_loss: per pixel of C classes, CE = m + log(sum_c exp(q_c - m)) - q_l with the sum in [1, C]: exp and log within 1 ulp, C sums,
      three more roundings: (C + 8) u64 (2Q + ln C), Q = max_c |q_c|; the N pixels' CEs summed (thread, CTA tree, CTA fold: depth <= N);
      torch's logsumexp and sum on the reference side the same: |dS| <= 2 (C + N + 8) u64 sum_pixels (2Q + ln C).  ce = S / n rounds
      once: dce = |dS| / n + u64 ce.  The finish f(ce) = alpha w ce (1 - e^-ce)^gamma (utils.py:43-46) moves by |f'(ce)| dce, doubled
      for the variation of f' over [ce - dce, ce + dce] (dce / ce is ~1e-12); exp, pow (2 ulp) and four products: 16 u64 |f|.
    depth_loss: per bin, max(x, 0) - y x + log1p(exp(-|x|)) of magnitude <= 2|x| + 1, within 4 u64 of it; summed over at most
      BN h w D bins (any order) on either side: |dS| <= 2 (BN h w D + 8) u64 sum_all_bins (2|x| + 1); / max(1, n): + u64 |ref|.
    Then the fp32 store of each: U |ref|."""
    d = c.decoded['d'](None)
    sums = emu_camera_losses.camera_terms(d)
    r = Ptr(ref['out'], c.p['out'].off).flat()
    out = torch.zeros_like(ref['out'])
    o = Ptr(out, c.p['out'].off).flat()
    if 'seg' in sums:
        s, n, _, _, _ = sums['seg']
        BN, h, w, C = d.BN, d.seg_h, d.seg_w, d.seg_classes
        q = torch.as_strided(d.seg_logits.flat(), (BN, h, w, C), (h * w * d.seg_ld, w * d.seg_ld, d.seg_ld, 1), d.seg_coff)
        dS = 2 * (C + BN * h * w + 8) * U64 * float((2 * torch.maximum(q.amax(-1), -q.amin(-1)) + math.log(C)).sum())
        ce = float(s) / max(n, 1)
        dce = dS / max(n, 1) + U64 * ce
        g, em = float(d.seg_gamma), math.exp(-ce)
        fp = float(d.seg_alpha) * float(d.seg_weight) * (1 - em) ** (g - 1) * ((1 - em) + g * ce * em)
        o[0] = 2 * abs(fp) * dce + (16 * U64 + U) * r[0].abs()
    if 'depth' in sums:
        _, n = sums['depth']
        BN, h, w, D = d.BN, d.depth_h, d.depth_w, d.depth_bins
        x = torch.as_strided(d.depth_logits.flat(), (BN, h, w, D), (h * w * d.depth_ld, w * d.depth_ld, d.depth_ld, 1), d.depth_coff)
        dS = 2 * (x.numel() + 8) * U64 * float((2 * x.abs() + 1).sum())
        o[1] = dS / max(n, 1) + (U64 + U) * r[1].abs()
    return {'out': out}


def check_operands_unchanged(c):
    """a loss launch may write its destination and its workspace only: every operand it reads is bitwise what it was."""
    seen = set()
    for k, p in c.p.items():
        if k in c.outs or k == 'ws' or id(p.t) in seen:
            continue
        seen.add(id(p.t))
        was = c.src[(id(p.t), None)]
        now = p.t.to(was.dtype)
        bad = (now != was) & ~(now.isnan() & was.isnan()) if was.is_floating_point() else now != was
        if bool(bad.any()):
            i = int(bad.reshape(-1).nonzero()[0])
            c.fail(f'{k}: the call changed an operand it only reads: {int(bad.sum())} elements, first {c.where_str(k, i)}')


def check_loss(bound_fn):
    inner = bounded(bound_fn)

    def check(c):
        inner(c)
        check_operands_unchanged(c)
    return check


CHECKS = {
    'tt_conv2d': check_conv, 'tt_conv2d_f16s': check_conv, 'tt_pointwise_f16s': check_conv,
    **{k: check_exact for k in ('tt_split_f16', 'tt_merge_f16', 'tt_image_to_split8', 'tt_copy2d', 'tt_anti_transpose', 'tt_nchw_to_nhwc',
                                'tt_nchw_to_nhwc_padded', 'tt_nhwc_to_nchw', 'tt_broadcast_rows', 'tt_fill', 'tt_maxpool3x3s2')},
    'tt_upsample2x_bilinear_ac_split': check_upsample_split,
    'tt_upsample2x_bilinear_ac': bounded(bound_upsample),
    'tt_global_avgpool': bounded(bound_pool), 'tt_se_pool': bounded(bound_pool),
    'tt_se_gate': bounded(bound_se_gate), 'tt_se_apply': bounded(bound_se_apply),
    'tt_layernorm': bounded(bound_layernorm), 'tt_eltwise': bounded(bound_eltwise),
    'tt_msda_forward': bounded(bound_msda), 'tt_msda_forward_frames': bounded(bound_msda),
    'tt_look_reduce': bounded(bound_look_reduce), 'tt_look_reduce_frames': bounded(bound_look_reduce),
    'tt_loss_reduce': check_loss(bound_loss_reduce), 'tt_camera_loss': check_loss(bound_camera_loss),
}
assert set(CHECKS) == set(OUTPUTS)


def inverse_softplus(eng):
    """tt_eltwise op 4 (the teacher-forced decoder pass's inverse softplus, not part of the inference forward) through the engine, on
    values from 1e-3 to 30: run inside a census to have it checked."""
    from thinktwice_b200 import lib
    from thinktwice_b200.engine import FMap
    a = eng.buf('census.softplus', (64, 1, 1, 4))
    a.copy_(torch.linspace(1e-3, 30.0, 256).view(64, 1, 1, 4))
    return eng.eltwise(lib.ELT_INV_SOFTPLUS, FMap(a, 64, 1, 1, 4), name='census.inv_softplus')


# ---------------------------------------------------------------------------------------------------------- the census
class Census:
    """stop: raise CensusError at the first failing call (else collect every failure in `failures`).  outside: check that nothing
    outside each destination's written region changed.  eng: the product's Engine, to name layers by their buffers."""

    def __init__(self, eng=None, stop=False, outside=True, window=False, cap=None):
        """window: check each convolution on conv_windows (the first and the last images of its N) instead of all of N.  cap: bytes
        of fp64 copies above which a call of another entry is counted as skipped instead of checked."""
        # the loss entries without their lib monkeypatches: the product keeps packing real tt_loss_term arrays / descriptors
        self.ref = emu_camera_losses.install(emu_losses.install(emu_frames.install(emu_lib.Emu())))
        self.eng, self.stop, self.outside, self.window, self.cap = eng, stop, outside, window, cap
        self.skipped = defaultdict(int)
        self.peak = (0, -1, '')                                        # (bytes, call, entry): the largest working set of one check
        self.max_allocated = 0                                         # device bytes allocated at most before the latest checked call
        self.calls = 0
        self.stats = {}                                                # entry -> [calls checked, worst ratio, where]
        self.layers = {}                                               # (entry, layer) -> [calls checked, worst ratio]
        self.failures, self.unchecked, self.covered = [], defaultdict(int), defaultdict(int)
        self.cuda = False
        self._table = None
        self._real = None

    # ------------------------------------------------------------------ plumbing (set by install)
    def sync(self):
        if self.cuda:
            torch.cuda.synchronize()

    def stream(self):
        from thinktwice_b200 import lib
        return lib._stream()

    def resolve(self, v, what):
        if isinstance(v, Ptr) or v is None:
            return v
        if isinstance(v, C.c_void_p) or (what.startswith('io.') and isinstance(v, int)):
            addr = v.value if isinstance(v, C.c_void_p) else v
            if not addr:
                return NULL
            if addr not in self._table:
                raise CensusError(f'{what}: device pointer {addr:#x} was not handed out by lib._p')
            t, off = self._table[addr]
            return Ptr(t, off)
        return v

    def pointer(self, p):
        """a Ptr as the real entry takes it."""
        if not self.cuda:
            return p
        from thinktwice_b200 import lib
        return lib._p(p.t, p.off)

    def real_entry(self, name):
        return getattr(self._real, name)

    def _storages(self, t):
        return t.untyped_storage().data_ptr()

    def is_scratch(self, t):
        if self.eng is None:
            return False
        s = self._storages(t)
        return any(self._storages(b) == s for b in self.eng._scratch.values())

    def namer(self, t):
        if self.eng is None:
            return '?'
        s = self._storages(t)
        for key, b in self.eng.bufs.items():
            if self._storages(b) == s:
                return key[0] if key[0] != 'late#s' else 'late split companion'
        return 'scratch' if self.is_scratch(t) else 'outside the arena'

    # ------------------------------------------------------------------ interception
    def wrap(self, name, fn, launch_count):
        if name in NOT_KERNELS or name.endswith('_workspace_bytes'):
            return fn

        def call(*args):
            idx = self.calls
            self.calls += 1
            if name in COVERED_ELSEWHERE:
                self.covered[name] += 1
                return fn(*args)
            if name not in CHECKS:
                self.unchecked[name] += 1
                return fn(*args)
            try:
                return checked(idx, *args)
            finally:
                if self._table is not None:                            # pointers live from lib._p to the call they are made for
                    self._table.clear()

        def checked(idx, *args):
            self.sync()
            base = 0
            if self.cuda:
                self.max_allocated = max(self.max_allocated, torch.cuda.max_memory_allocated())
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
            c = Call(self, idx, name, args)
            if c.skip:
                self.skipped[name] += 1
                return fn(*args)
            sat0 = self.saturations()
            l0 = launch_count()
            rc = fn(*args)
            self.sync()
            if rc != 0:
                return rc
            c.launches = launch_count() - l0
            sat = self.saturations() - sat0
            if sat:
                c.fail(f'{sat} epilogue threads saturated a split plane at +-65504')
            CHECKS[name](c)
            st = self.stats.setdefault(name, [0, 0.0, '', 0.0])
            st[0] += 1
            st[3] = max(st[3], c.planes_ratio)
            if c.ratio >= st[1]:
                st[1], st[2] = c.ratio, f'call #{idx} [{c.layer}] {c.where}'
            ls = self.layers.setdefault((name, c.layer), [0, 0.0])
            ls[0] += 1
            ls[1] = max(ls[1], c.ratio)
            del c
            if self.cuda:
                ws = torch.cuda.max_memory_allocated() - base
                if ws > self.peak[0]:
                    self.peak = (ws, idx, name)
            return rc
        return call

    def saturations(self):
        """the f16s epilogues' saturation counter (it synchronises)."""
        v = C.c_uint()
        from thinktwice_b200 import lib
        lib.check(self._real.tt_f16s_saturation_count(C.byref(v), 0, self.stream()), 'tt_f16s_saturation_count')
        return int(v.value)

    def table(self):
        """per entry: calls checked, calls skipped (working set over the cap), the worst err / bound ratio (with where it was) and,
        for the f16s convs, the worst ratio of the bitwise split-plane check (0 = every plane element is _split_f16 of fp32 y)."""
        lines = [f'{"entry":34s} {"calls":>6s} {"skipped":>7s} {"worst err/bound":>16s} {"planes":>7s}  where']
        for k in sorted(set(self.stats) | set(self.skipped)):
            n, r, w, pr = self.stats.get(k, (0, 0.0, '', 0.0))
            lines.append(f'{k:34s} {n:6d} {self.skipped.get(k, 0):7d} {r:16.3g} {pr:7.3g}  {w}')
        for k in sorted(self.covered):
            lines.append(f'{k:34s} {self.covered[k]:6d} {"elsewhere":>16s}  {COVERED_ELSEWHERE[k]}')
        for k in sorted(self.unchecked):
            lines.append(f'{k:34s} {self.unchecked[k]:6d} {"UNCHECKED":>16s}')
        return '\n'.join(lines)

    def layer_table(self, prefix):
        """per (entry, destination buffer) whose buffer name starts with `prefix`: calls checked and the worst err / bound ratio."""
        lines = [f'{"entry":34s} {"buffer":24s} {"calls":>6s} {"worst err/bound":>16s}']
        for (k, layer), (n, r) in sorted(self.layers.items()):
            if layer.startswith(prefix):
                lines.append(f'{k:34s} {layer:24s} {n:6d} {r:16.3g}')
        return '\n'.join(lines)

    def assert_clean(self):
        assert not self.unchecked, f'entries called by the forward that neither the census nor COVERED_ELSEWHERE checks: {dict(self.unchecked)}'
        assert not self.failures, '\n'.join(self.failures[:20])
        assert self.stats, 'no call was checked'


class _Proxy:
    def __init__(self, real, census):
        self._real, self._census, self._cache = real, census, {}

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if not name.startswith('tt_'):
            return fn
        if name not in self._cache:
            self._cache[name] = self._census.wrap(name, fn, lambda: int(self._real.tt_launch_count()))
        return self._cache[name]


def install(monkeypatch, census):
    """route every C ABI call of the product through `census`.  On the GPU `lib._p` (and the copies the product modules imported)
    is wrapped to record which tensor and element offset each device pointer it hands out belongs to; on the emulated ABI (the
    `emulated` fixture) the pointers are emu_lib.Ptr objects already."""
    from thinktwice_b200 import lib
    import thinktwice_b200.encoder_decoder_framework as fw
    import thinktwice_b200.engine as engine
    import thinktwice_b200.lidarnet as lidarnet
    import thinktwice_b200.lss as lss
    import thinktwice_b200.preprocess as pre
    import thinktwice_b200.thinktwice_decoder as dec
    real = lib.load()
    census._real = real
    census.cuda = isinstance(real, C.CDLL)
    if census.cuda:
        census._table = table = {}
        orig = lib._p

        def _p(t, off=0):
            r = orig(t, off)
            if t is not None:
                table[r.value] = (t, off)
            return r
        monkeypatch.setattr(lib, '_p', _p)
        for mod in (engine, lss, lidarnet, dec, fw, pre):
            monkeypatch.setattr(mod, '_p', _p, raising=False)
    proxy = _Proxy(real, census)
    monkeypatch.setattr(lib, 'load', lambda: proxy)
    return census
