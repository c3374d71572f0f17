"""A torch-on-CPU emulation of the libtt_b200 C ABI — TEST HARNESS ONLY (never imported by the product).

tests/test_host_emulated_cpu.py swaps it in for `thinktwice_b200.lib.load()` and runs the PRODUCT's host code (weight
repacking, BatchNorm folding, buffer / concat / scatter layout, descriptor filling, the whole forward orchestration) on the CPU,
comparing the outputs with the oracle.  Every entry point below follows the contract written in include/tt_b200.h; the
arithmetic is plain torch (fp64 inside the contractions), so what is under test is everything ABOVE the C ABI.  The CUDA
kernels themselves are the GPU suite's job.
"""
import ctypes as C

import torch
import torch.nn.functional as F


class Ptr:
    """what `lib._p` hands to the emulated entry points: a tensor and an element offset into its flat storage."""
    __slots__ = ('t', 'off')

    def __init__(self, t, off=0):
        self.t, self.off = t, off

    def flat(self):
        return self.t.reshape(-1)[self.off:]

    def __bool__(self):
        return self.t is not None


NULL = Ptr(None)


class IO:
    """stand-in for lib.F16sIO (tt_f16s_io): same field names, Ptr objects instead of addresses."""

    def __init__(self):
        self.x_split = self.w_split = self.bias = self.res = self.res_split = self.res2 = self.res2_split = self.y = self.y_split = NULL
        self.x_plane = self.res_plane = self.res2_plane = self.y_plane = 0
_by_addr = {}


def make_p():
    def _p(t, off=0):
        if t is None:
            return NULL
        assert t.is_contiguous()
        _by_addr[t.data_ptr()] = t
        return Ptr(t, off)
    return _p


def _v(a):
    """plain python value of a ctypes scalar argument."""
    return a.value if hasattr(a, 'value') else a


def _desc(a):
    return a._obj if hasattr(a, '_obj') else a


def _act(v, act):
    if act == 0:
        return v
    if act == 1:
        return F.relu(v)
    if act == 2:
        return F.gelu(v)
    if act == 3:
        return torch.sigmoid(v)
    if act == 4:
        return F.softplus(v)
    if act == 5:
        return F.softplus(v).clamp_min(1e-3)
    raise NotImplementedError(f'act {act}')


def _split_f16(v):
    """fp32 -> (hi, lo') halves exactly as csrc/gemm_conv_f16s.cu split_h (saturating)."""
    c = v.float().clamp(-65504.0, 65504.0)
    hi = c.half()
    return hi, ((c - hi.float()) * 2048.0).half()


def _pix_view(p, N, H, W, ld, nstride=0, hstride=0, C=None):
    """(N, H, W, C) strided view of a channels-last buffer starting at pointer p."""
    hs = hstride or W * ld
    ns = nstride or H * hs
    return torch.as_strided(p.flat(), (N, H, W, C if C is not None else ld), (ns, hs, ld, 1))


def conv_ref(d, x, w, bias, res, res2, f16s=None, kmajor_w=False, magnitude=False):
    """include/tt_b200.h (2) / (2b) in fp64 on the operands' device: (value, magnitude), both (N, OH, OW, Cout).  value =
    act(conv(x, w) + bias + res + res2) from exactly what the kernel reads (split operands decoded as hi + lo' / 2048);
    magnitude (only when asked, else None) = conv(|x|, |w|) + |bias| + |res| + |res2|, the pre-activation scale a rounding
    bound is proportional to."""
    taps = d.KH * d.KW
    cg = d.Cin // d.groups
    dev = (x.t if x else w.t).device

    def xview(C_):                                                     # (N, H, W, C_) fp64 view of the input
        Wv = d.W if C_ == d.Cin else d.x_hstride // d.x_ld
        if f16s is None:
            return _pix_view(x, d.N, d.H, Wv, d.x_ld, d.x_nstride, d.x_hstride, C_).double()
        hi = _pix_view(x, d.N, d.H, Wv, d.x_ld, d.x_nstride, d.x_hstride, C_).double()
        lo = _pix_view(Ptr(x.t, x.off + f16s.x_plane), d.N, d.H, Wv, d.x_ld, d.x_nstride, d.x_hstride, C_).double()
        return hi + lo / 2048.0
    if f16s is not None and not kmajor_w:                              # [2][Cout][taps][Cin8] scaled-split half planes
        c8 = -(-d.Cin // 8) * 8
        planes = w.flat()[:2 * d.Cout * taps * c8].view(2, d.Cout, taps, c8).double()
        wt = (planes[0] + planes[1] / 2048.0)[..., :d.Cin].reshape(d.Cout, d.KH, d.KW, d.Cin).permute(0, 3, 1, 2)
        assert d.groups == 1
    elif d.impl >= 2 and not kmajor_w:                                 # [2][Cout][taps][Cin] hi / lo planes
        planes = w.flat()[:2 * d.Cout * taps * d.Cin].view(2, d.Cout, taps, d.Cin).double()
        wt = (planes[0] + planes[1]).view(d.Cout, d.KH, d.KW, d.Cin).permute(0, 3, 1, 2)
        assert d.groups == 1
    else:                                                              # [taps * Cin_g][Cout]
        wt = w.flat()[:taps * cg * d.Cout].view(d.KH, d.KW, cg, d.Cout).permute(3, 2, 0, 1).double()
    if d.x_ld < d.Cin:                                                 # row-packed input: channels run on into the next pixels
        assert d.KW == 1 and d.pad == 0 and d.groups == 1
        px = d.Cin // d.x_ld                                           # pixels per K slab
        xin = xview(d.x_ld).permute(0, 3, 1, 2)
        wt = wt.reshape(d.Cout, px, d.x_ld, d.KH).permute(0, 2, 3, 1)                      # (Cout, c, kh, kw)
        contract = lambda a, b: F.conv2d(a, b, stride=d.stride)
    else:
        xin = xview(d.Cin).permute(0, 3, 1, 2)
        contract = lambda a, b: F.conv2d(a, b, stride=d.stride, padding=d.pad, dilation=d.dil, groups=d.groups)

    def terms(f):                                                      # the summands of the epilogue, f = identity or abs
        out = contract(f(xin), f(wt))
        assert out.shape[2] >= d.OH and out.shape[3] >= d.OW, (tuple(out.shape), d.OH, d.OW)
        out = out[..., :d.OH, :d.OW].permute(0, 2, 3, 1)               # (N, OH, OW, Cout)
        if bias:
            if d.bias_n_mod:
                tab = bias.flat()[:d.bias_n_mod * d.Cout].view(d.bias_n_mod, d.Cout).double()
                out = out + f(tab[torch.arange(d.N, device=dev) % d.bias_n_mod][:, None, None, :])
            else:
                out = out + f(bias.flat()[:d.Cout].double())
        rs_, rp_ = (f16s.res_split, f16s.res_plane) if f16s is not None else (NULL, 0)
        r2s_, r2p_ = (f16s.res2_split, f16s.res2_plane) if f16s is not None else (NULL, 0)
        if d.res_mode == 1:
            out = out + f(_res_view(d, res, rs_, rp_, d.N, d.OH, d.OW, d.res_ld, d.res_coff))
        elif d.res_mode == 2:                                          # nearest-upsampled residual (PAFPN top-down)
            r = _res_view(d, res, rs_, rp_, d.N, d.res_H, d.res_W, d.res_ld, d.res_coff)
            ih = (torch.arange(d.OH, device=dev) * d.res_H) // d.OH
            iw = (torch.arange(d.OW, device=dev) * d.res_W) // d.OW
            out = out + f(r[:, ih][:, :, iw])
        if res2 or r2s_:
            out = out + f(_res_view(d, res2, r2s_, r2p_, d.N, d.OH, d.OW, d.res2_ld, d.res2_coff))
        return out
    return _act(terms(lambda v: v), d.act), (terms(torch.abs) if magnitude else None)


def _res_view(d, p32, psplit, plane, N_, H_, W_, ld_, coff_):
    """(N_, H_, W_, Cout) fp64 residual, from fp32 or from split planes."""
    if p32:
        return _pix_view(p32, N_, H_, W_, ld_, C=d.Cout + coff_)[..., coff_:].double()
    hi = _pix_view(psplit, N_, H_, W_, ld_, C=d.Cout + coff_)[..., coff_:].double()
    lo = _pix_view(Ptr(psplit.t, psplit.off + plane), N_, H_, W_, ld_, C=d.Cout + coff_)[..., coff_:].double()
    return hi + lo / 2048.0


def y_region(d, p):
    """the (N, OH, OW, Cout) elements of a conv output buffer (fp32 or one split plane, pointer p) that output rows go to."""
    yv = _pix_view(p, d.N, d.yH, d.yW, d.y_ld, d.y_nstride, 0, d.Cout + d.y_coff)[..., d.y_coff:]
    return yv[:, d.oy_add::d.oy_mul, d.ox_add::d.ox_mul][:, :d.OH, :d.OW]


def conv_store(d, y, y_split, y_plane, out):
    """write the fp32 result `out` (N, OH, OW, Cout) to y and / or the split planes, as the conv epilogue does."""
    if y:
        y_region(d, y)[...] = out
    if y_split:
        hi, lo = _split_f16(out)
        for plane, val in ((0, hi), (y_plane, lo)):
            y_region(d, Ptr(y_split.t, y_split.off + plane))[...] = val


class Emu:
    def __init__(self):
        self.launches = 0
        self.error = b'emulated'

    # ------------------------------------------------------------------ bookkeeping
    def tt_version(self):
        return 1

    def tt_last_error(self):
        return self.error

    def tt_launch_count(self):
        return self.launches

    def tt_debug_set(self, flags):
        return 0

    def __getattr__(self, name):
        if name.endswith('_workspace_bytes'):
            return lambda *a: 64
        raise NotImplementedError(f'emu_lib: {name}')

    # ------------------------------------------------------------------ conv / linear
    def tt_conv2d(self, d, x, w, bias, res, res2, gather, m_count, y, ws, stream, f16s=None, kmajor_w=False):
        d = _desc(d)
        self.launches += 1
        assert not gather and not m_count
        out, _ = conv_ref(d, x, w, bias, res, res2, f16s, kmajor_w)
        conv_store(d, y, f16s.y_split if f16s is not None else NULL, f16s.y_plane if f16s is not None else 0, out.float())
        return 0

    def tt_conv2d_f16s(self, d, io, stream):
        """include/tt_b200.h (2b): operands are read from the split planes (x = hi + lo' / 2048), residuals from fp32 or split
        planes, outputs written as fp32 and / or split."""
        assert io.x_split.t.dtype == torch.float16 and io.w_split.t.dtype == torch.float16
        assert io.y or io.y_split
        return self.tt_conv2d(d, io.x_split, io.w_split, io.bias, io.res, io.res2, NULL, NULL, io.y, NULL, stream, f16s=io)

    def tt_pointwise_f16s(self, d, io, w_kmajor, stream):
        """thin 1x1 conv: split-plane input, fp32 K-major weights [Cin][Cout]."""
        dd = _desc(d)
        assert dd.KH == 1 and dd.KW == 1 and dd.Cin <= 64 and dd.Cout <= 64 and not io.res and not io.res_split
        old = dd.impl
        dd.impl = 1                                                    # weights in the SIMT layout
        io2 = IO()
        io2.__dict__.update(io.__dict__)
        rc = self.tt_conv2d(d, io.x_split, w_kmajor, io.bias, NULL, NULL, NULL, NULL, io.y, NULL, stream, f16s=io2, kmajor_w=True)
        dd.impl = old
        return rc

    def tt_split_f16(self, x, x_ld, y_split, y_plane, y_ld, rows, cols, row_count, stream):
        self.launches += 1
        x_ld, y_plane, y_ld, rows = _v(x_ld), _v(y_plane), _v(y_ld), _v(rows)
        n = min(rows, int(row_count.flat()[0])) if row_count else rows
        src = torch.as_strided(x.flat(), (n, cols), (x_ld, 1))
        hi, lo = _split_f16(src)
        torch.as_strided(y_split.flat(), (n, cols), (y_ld, 1)).copy_(hi)
        torch.as_strided(Ptr(y_split.t, y_split.off + y_plane).flat(), (n, cols), (y_ld, 1)).copy_(lo)
        return 0

    def tt_image_to_split8(self, x, y_split, y_plane, N, Cc, H, W, out_H, out_W, top, left, stream):
        self.launches += 1
        y_plane = _v(y_plane)
        img = x.flat()[:N * Cc * H * W].view(N, Cc, H, W).permute(0, 2, 3, 1)
        hi, lo = _split_f16(img)
        for plane, val in ((0, hi), (y_plane, lo)):
            dst = Ptr(y_split.t, y_split.off + plane).flat()[:N * out_H * out_W * 8].view(N, out_H, out_W, 8)
            dst[:, top:top + H, left:left + W, :Cc] = val
            dst[:, top:top + H, left:left + W, Cc:] = 0
        return 0

    def tt_preprocess_u8(self, d, raw, map_grid, out_nchw, out_split8, split_plane, stream):
        """include/tt_b200.h section 8: uint8 HWC frames -> grid_sample -> bilinear resize -> crop -> / div -> (x - mean) / std, written as
        fp32 NCHW and / or the stem's split planes (plain torch ops: the semantics, not the kernel's operation order)."""
        d = _desc(d)
        n, H, W = d.n_img, d.H, d.W
        if out_split8 and n * d.pad_H * d.pad_W * 8 > _v(split_plane):
            self.error = b'tt_preprocess_u8: n_img stem slots exceed the stem-plane capacity split_plane'
            return -1
        self.launches += 1
        x = raw.flat()[:n * H * W * 3].view(n, H, W, 3).float().permute(0, 3, 1, 2)
        if d.undistort:
            g = map_grid.flat()[:H * W * 2].view(1, H, W, 2).expand(n, H, W, 2)
            x = F.grid_sample(x, g, mode='bilinear', padding_mode='zeros', align_corners=False)
        x = F.interpolate(x, size=(d.newH, d.newW), mode='bilinear', align_corners=False, antialias=False)
        x = x[:, :, d.crop_y:d.crop_y + d.outH, d.crop_x:d.crop_x + d.outW]
        mean = torch.tensor(list(d.mean)).view(1, 3, 1, 1)
        std = torch.tensor(list(d.std)).view(1, 3, 1, 1)
        x = (x / d.div - mean) / std
        if out_nchw:
            out_nchw.flat()[:x.numel()].copy_(x.reshape(-1))
        if out_split8:
            plane = _v(split_plane)
            hi, lo = _split_f16(x.permute(0, 2, 3, 1))
            for off, val in ((0, hi), (plane, lo)):
                dst = Ptr(out_split8.t, out_split8.off + off).flat()[:n * d.pad_H * d.pad_W * 8].view(n, d.pad_H, d.pad_W, 8)
                dst[:, d.pad_top:d.pad_top + d.outH, d.pad_left:d.pad_left + d.outW, :3] = val
                dst[:, d.pad_top:d.pad_top + d.outH, d.pad_left:d.pad_left + d.outW, 3:] = 0
        return 0

    def tt_upsample2x_bilinear_ac_split(self, x, y_split, y_plane, N, H, W, Cc, stream):
        self.launches += 1
        y_plane = _v(y_plane)
        xin = x.flat()[:N * H * W * Cc].view(N, H, W, Cc).permute(0, 3, 1, 2)
        up = F.interpolate(xin, scale_factor=2, mode='bilinear', align_corners=True).permute(0, 2, 3, 1).contiguous()
        hi, lo = _split_f16(up)
        y_split.flat()[:up.numel()].copy_(hi.reshape(-1))
        Ptr(y_split.t, y_split.off + y_plane).flat()[:up.numel()].copy_(lo.reshape(-1))
        return 0

    def tt_merge_f16(self, x_split, x_plane, x_ld, y, y_ld, rows, cols, stream):
        self.launches += 1
        x_plane, x_ld, y_ld, rows = _v(x_plane), _v(x_ld), _v(y_ld), _v(rows)
        hi = torch.as_strided(x_split.flat(), (rows, cols), (x_ld, 1)).float()
        lo = torch.as_strided(Ptr(x_split.t, x_split.off + x_plane).flat(), (rows, cols), (x_ld, 1)).float()
        torch.as_strided(y.flat(), (rows, cols), (y_ld, 1)).copy_(hi + lo / 2048.0)
        return 0

    def tt_f16s_saturation_count(self, out_host, reset, stream):
        _desc(out_host).value = 0
        return 0

    # ------------------------------------------------------------------ LiDAR: voxelise, rulebooks, sparse conv, densify
    def tt_voxelize_mean(self, d, points, feats, coords, count, ws, stream):
        d = _desc(d)
        self.launches += 1
        pts = points.flat()[:d.B * d.P * d.F].view(d.B, d.P, d.F)
        lower, vs, grid = torch.tensor(list(d.lower)), torch.tensor(list(d.vsize)), torch.tensor(list(d.grid))
        fo, co = feats.flat().view(-1, d.F), coords.flat().view(-1, 4)
        n = 0
        for b in range(d.B):
            c = torch.floor((pts[b, :, :3] - lower) / vs).long()                      # (x, y, z)
            ok = ((c >= 0) & (c < grid)).all(1) & (c[:, 2] < d.zmax)
            idx = torch.nonzero(ok).squeeze(1)
            c = c[idx]
            key = (c[:, 2] * grid[1] + c[:, 1]) * grid[0] + c[:, 0]
            uniq, inv = torch.unique(key, return_inverse=True)
            assert uniq.numel() <= d.max_voxels
            order = torch.argsort(inv, stable=True)                                  # points grouped by voxel, input order kept
            sv = inv[order]
            start = torch.zeros(uniq.numel() + 1, dtype=torch.long)
            start[1:] = torch.cumsum(torch.bincount(sv, minlength=uniq.numel()), 0)
            slot = torch.arange(sv.numel()) - start[sv]
            sel = slot < d.max_points
            acc = torch.zeros(uniq.numel(), d.F, dtype=torch.float64).index_add_(0, sv[sel], pts[b, idx[order][sel]].double())
            cnt = torch.bincount(sv[sel], minlength=uniq.numel()).double()
            m = uniq.numel()
            fo[n:n + m] = (acc / cnt[:, None]).float()
            z, rem = uniq // (grid[1] * grid[0]), uniq % (grid[1] * grid[0])
            co[n:n + m] = torch.stack([torch.full_like(z, b), z, rem // grid[0], rem % grid[0]], 1).int()
            n += m
        count.flat()[0] = n
        return 0

    def tt_sparse_rulebook(self, d, in_coords, in_count, out_coords, out_count, nbr, pairs_in, pairs_out, pair_count, ws, stream):
        d = _desc(d)
        self.launches += 1
        n_in = int(in_count.flat()[0])
        ic = in_coords.flat().view(-1, 4)[:n_in].long()
        k, s, p, ishape, oshape = (list(getattr(d, n)) for n in ('k', 's', 'p', 'in_shape', 'out_shape'))
        kvol = k[0] * k[1] * k[2]
        taps = [(a, b, c) for a in range(k[0]) for b in range(k[1]) for c in range(k[2])]

        def key(cc, shape):
            return ((cc[:, 0] * shape[0] + cc[:, 1]) * shape[1] + cc[:, 2]) * shape[2] + cc[:, 3]
        if d.subm:
            oc = ic.clone()
        else:                                                          # every output site reached by an input (spconv SparseConv3d)
            outs = []
            for t in taps:
                num = ic[:, 1:] + torch.tensor(p) - torch.tensor(t)
                ok = (num % torch.tensor(s) == 0).all(1)
                o = num // torch.tensor(s)
                ok &= ((o >= 0) & (o < torch.tensor(oshape))).all(1)
                outs.append(torch.cat([ic[ok, :1], o[ok]], 1))
            allo = torch.cat(outs)
            uk = torch.unique(key(allo, oshape))
            sp = oshape[0] * oshape[1] * oshape[2]
            b, r = uk // sp, uk % sp
            oc = torch.stack([b, r // (oshape[1] * oshape[2]), (r // oshape[2]) % oshape[1], r % oshape[2]], 1)
        n_out = oc.shape[0]
        assert n_out <= d.cap_out
        out_coords.flat().view(-1, 4)[:n_out] = oc.int()
        out_count.flat()[0] = n_out
        ikeys = key(ic, ishape)
        srt, perm = torch.sort(ikeys)
        pin = pairs_in.flat().view(kvol, -1) if pairs_in else None
        pout = pairs_out.flat().view(kvol, -1) if pairs_out else None
        for ti, t in enumerate(taps):
            if d.subm:
                src = oc[:, 1:] + torch.tensor(t) - torch.tensor([kk // 2 for kk in k])
            else:
                src = oc[:, 1:] * torch.tensor(s) - torch.tensor(p) + torch.tensor(t)
            ok = ((src >= 0) & (src < torch.tensor(ishape))).all(1)
            sk = key(torch.cat([oc[:, :1], src], 1), ishape)
            pos = torch.searchsorted(srt, sk).clamp_max(max(srt.numel() - 1, 0))
            hit = ok & (srt[pos] == sk) if srt.numel() else ok & False
            rows_out = torch.nonzero(hit).squeeze(1)
            m = rows_out.numel()
            if pin is not None:
                pin[ti, :m] = perm[pos[hit]].int()
                pout[ti, :m] = rows_out.int()
                pair_count.flat()[ti] = m
            if nbr:
                nb = nbr.flat().view(-1, kvol)
                nb[:n_out, ti] = -1
                nb[rows_out, ti] = perm[pos[hit]].int()
        return 0

    def tt_sparse_conv(self, d, feats_in, w, bias, res, pairs_in, pairs_out, pair_count, out_count, feats_out, stream):
        d = _desc(d)
        self.launches += 3
        n_out = int(out_count.flat()[0])
        fi = feats_in.flat().view(-1, d.in_ld)[:, :d.Cin].double()
        if d.impl >= 2:
            planes = w.flat()[:2 * d.Cout * d.kvol * d.Cin].view(2, d.Cout, d.kvol, d.Cin).double()
            wt = (planes[0] + planes[1]).permute(1, 2, 0)              # (kvol, Cin, Cout)
        else:
            wt = w.flat()[:d.kvol * d.Cin * d.Cout].view(d.kvol, d.Cin, d.Cout).double()
        out = torch.zeros(n_out, d.Cout, dtype=torch.float64)
        if bias:
            out += bias.flat()[:d.Cout].double()
        pin, pout = pairs_in.flat().view(d.kvol, -1), pairs_out.flat().view(d.kvol, -1)
        for t in range(d.kvol):
            m = int(pair_count.flat()[t])
            if m:
                out.index_add_(0, pout[t, :m].long(), fi[pin[t, :m].long()] @ wt[t])
        if res:
            out += res.flat().view(-1, d.res_ld)[:n_out, :d.Cout].double()
        feats_out.flat().view(-1, d.out_ld)[:n_out, :d.Cout] = _act(out, d.act).float()
        return 0

    def tt_sparse_conv_f16s(self, d, feats_in_split, in_plane, w_split, bias, res, pairs_in, pairs_out, pair_count, out_count, feats_out,
                            out_split, out_plane, stream):
        d = _desc(d)
        self.launches += 3
        in_plane, out_plane = _v(in_plane), _v(out_plane)
        n_out = int(out_count.flat()[0])
        fi = (feats_in_split.flat().view(-1, d.in_ld)[:in_plane // d.in_ld, :d.Cin].double() +
              Ptr(feats_in_split.t, feats_in_split.off + in_plane).flat().view(-1, d.in_ld)[:in_plane // d.in_ld, :d.Cin].double() / 2048.0)
        c8 = -(-d.Cin // 8) * 8
        planes = w_split.flat()[:2 * d.Cout * d.kvol * c8].view(2, d.Cout, d.kvol, c8).double()
        wt = (planes[0] + planes[1] / 2048.0)[..., :d.Cin].permute(1, 2, 0)   # (kvol, Cin, Cout)
        out = torch.zeros(n_out, d.Cout, dtype=torch.float64)
        if bias:
            out += bias.flat()[:d.Cout].double()
        pin, pout = pairs_in.flat().view(d.kvol, -1), pairs_out.flat().view(d.kvol, -1)
        for t in range(d.kvol):
            m = int(pair_count.flat()[t])
            if m:
                out.index_add_(0, pout[t, :m].long(), fi[pin[t, :m].long()] @ wt[t])
        if res:
            out += res.flat().view(-1, d.res_ld)[:n_out, :d.Cout].double()
        o = _act(out, d.act).float()
        feats_out.flat().view(-1, d.out_ld)[:n_out, :d.Cout] = o
        if out_split:
            hi, lo = _split_f16(o)
            out_split.flat().view(-1, d.out_ld)[:n_out, :d.Cout] = hi
            Ptr(out_split.t, out_split.off + out_plane).flat().view(-1, d.out_ld)[:n_out, :d.Cout] = lo
        return 0

    def tt_sparse_conv_os_f16s(self, d, io, nbr, out_count, stream):
        """output-stationary form: out[m] = act(sum_tap W[tap] . in[nbr[m][tap]] + bias + res[m]), one launch."""
        d = _desc(d)
        self.launches += 1
        n_out = int(out_count.flat()[0])
        rows_in = io.x_plane // d.in_ld
        fi = (io.x_split.flat().view(-1, d.in_ld)[:rows_in, :d.Cin].double() +
              Ptr(io.x_split.t, io.x_split.off + io.x_plane).flat().view(-1, d.in_ld)[:rows_in, :d.Cin].double() / 2048.0)
        c8 = -(-d.Cin // 8) * 8
        planes = io.w_split.flat()[:2 * d.Cout * d.kvol * c8].view(2, d.Cout, d.kvol, c8).double()
        wt = (planes[0] + planes[1] / 2048.0)[..., :d.Cin].permute(1, 2, 0)   # (kvol, Cin, Cout)
        nb = nbr.flat().view(-1, d.kvol)[:n_out].long()
        out = torch.zeros(n_out, d.Cout, dtype=torch.float64)
        for t in range(d.kvol):
            ok = nb[:, t] >= 0
            if ok.any():
                out[ok] += fi[nb[ok, t]] @ wt[t]
        if io.bias:
            out += io.bias.flat()[:d.Cout].double()
        if io.res:
            out += io.res.flat().view(-1, d.res_ld)[:n_out, :d.Cout].double()
        elif io.res_split:
            out += (io.res_split.flat().view(-1, d.res_ld)[:n_out, :d.Cout].double() +
                    Ptr(io.res_split.t, io.res_split.off + io.res_plane).flat().view(-1, d.res_ld)[:n_out, :d.Cout].double() / 2048.0)
        o = _act(out, d.act).float()
        if io.y:
            io.y.flat().view(-1, d.out_ld)[:n_out, :d.Cout] = o
        if io.y_split:
            hi, lo = _split_f16(o)
            io.y_split.flat().view(-1, d.out_ld)[:n_out, :d.Cout] = hi
            Ptr(io.y_split.t, io.y_split.off + io.y_plane).flat().view(-1, d.out_ld)[:n_out, :d.Cout] = lo
        return 0

    def tt_sparse_to_bev(self, feats, coords, count, cap, Cc, D, H, W, anti, dense, stream):
        self.launches += 1
        n = int(count.flat()[0])
        f = feats.flat().view(-1, Cc)[:n]
        c = coords.flat().view(-1, 4)[:n].long()
        dv = dense.flat()
        B = dv.numel() // (H * W * Cc * D)
        out = dv[:B * H * W * Cc * D].view(B, H, W, Cc, D)            # channel = c * D + z, channels-last
        assert not anti
        out[c[:, 0], c[:, 2], c[:, 3], :, c[:, 1]] = f
        return 0

    def tt_fill(self, y, v, n, stream):
        self.launches += 1
        y.flat()[:_v(n)] = _v(v)
        return 0

    def tt_anti_transpose(self, x, y, N, S, Cc, stream):
        self.launches += 1
        xv = x.flat()[:N * S * S * Cc].view(N, S, S, Cc)
        y.flat()[:N * S * S * Cc].view(N, S, S, Cc).copy_(xv.flip(1).flip(2).transpose(1, 2))   # out[i, j] = x[S-1-j, S-1-i]
        return 0

    # ------------------------------------------------------------------ layout / elementwise
    def tt_nchw_to_nhwc_padded(self, x, y, N, Cc, H, W, y_ld, cpad, out_H, out_W, top, left, stream):
        self.launches += 1
        src = x.flat()[:N * Cc * H * W].view(N, Cc, H, W)
        dst = torch.as_strided(y.flat(), (N, out_H, out_W, y_ld), (out_H * out_W * y_ld, out_W * y_ld, y_ld, 1))
        dst[:, top:top + H, left:left + W, :Cc] = src.permute(0, 2, 3, 1)
        dst[:, top:top + H, left:left + W, Cc:cpad] = 0
        return 0

    def tt_nchw_to_nhwc(self, x, y, N, Cc, H, W, y_ld, y_coff, cpad, stream):
        self.launches += 1
        src = x.flat()[:N * Cc * H * W].view(N, Cc, H, W)
        dst = _pix_view(y, N, H, W, y_ld, C=y_coff + cpad)
        dst[..., y_coff:y_coff + Cc] = src.permute(0, 2, 3, 1)
        dst[..., y_coff + Cc:] = 0
        return 0

    def tt_nhwc_to_nchw(self, x, x_ld, x_coff, y, N, Cc, H, W, stream):
        self.launches += 1
        y.flat()[:N * Cc * H * W].view(N, Cc, H, W).copy_(_pix_view(x, N, H, W, x_ld, C=x_coff + Cc)[..., x_coff:].permute(0, 3, 1, 2))
        return 0

    def tt_maxpool3x3s2(self, x, y, N, H, W, Cc, stream):
        self.launches += 1
        o = F.max_pool2d(_pix_view(x, N, H, W, Cc).permute(0, 3, 1, 2), 3, stride=2, padding=1)
        y.flat()[:o.numel()].view(N, o.shape[2], o.shape[3], Cc).copy_(o.permute(0, 2, 3, 1))
        return 0

    def tt_upsample2x_bilinear_ac(self, x, y, N, H, W, Cc, stream):
        self.launches += 1
        o = F.interpolate(_pix_view(x, N, H, W, Cc).permute(0, 3, 1, 2), scale_factor=2, mode='bilinear', align_corners=True)
        y.flat()[:o.numel()].view(N, 2 * H, 2 * W, Cc).copy_(o.permute(0, 2, 3, 1))
        return 0

    def tt_global_avgpool(self, x, x_ld, x_coff, y, N, HW, Cc, stream):
        self.launches += 1
        v = torch.as_strided(x.flat()[x_coff:], (N, HW, Cc), (HW * x_ld, x_ld, 1))
        y.flat()[:N * Cc].view(N, Cc).copy_(v.double().mean(1))
        return 0

    def tt_broadcast_rows(self, v, y, N, HW, Cc, y_ld, y_coff, stream):
        self.launches += 1
        torch.as_strided(y.flat()[y_coff:], (N, HW, Cc), (HW * y_ld, y_ld, 1)).copy_(v.flat()[:N * Cc].view(N, 1, Cc).expand(N, HW, Cc))
        return 0

    def tt_se_gate(self, x, g, y, N, HW, Cc, stream):
        self.launches += 1
        xv, gv = x.flat()[:N * HW * Cc].view(N, HW, Cc), g.flat()[:N * Cc].view(N, 1, Cc)
        y.flat()[:N * HW * Cc].view(N, HW, Cc).copy_(xv * torch.sigmoid(gv))
        return 0

    def tt_se_pool(self, x, s, N, HW, Cc, stream):
        self.launches += 1
        xv = x.flat()[:N * HW * Cc].view(N, HW, Cc)
        s.flat()[:N * Cc].view(N, Cc).copy_(0.5 * xv.double().mean(1) + 0.5 * xv.amax(1).double())
        return 0

    def tt_se_apply(self, x, g, sc, sc_ld, sc_coff, y, y_ld, y_coff, N, HW, Cc, stream):
        self.launches += 1
        xv, gv = x.flat()[:N * HW * Cc].view(N, HW, Cc), g.flat()[:N * Cc].view(N, 1, Cc)
        scv = torch.as_strided(sc.flat()[sc_coff:], (N, HW, Cc), (HW * sc_ld, sc_ld, 1))
        torch.as_strided(y.flat()[y_coff:], (N, HW, Cc), (HW * y_ld, y_ld, 1)).copy_(F.relu(xv * torch.sigmoid(gv) + scv))
        return 0

    def tt_copy2d(self, src, src_ld, dst, dst_ld, rows, cols, rdiv, rmod, stream):
        self.launches += 1
        if src.t.dtype == torch.float16:                            # the C ABI moves 4-byte words: a pair of halves is one word
            assert dst.t.dtype == torch.float16 and src.off % 2 == 0 and dst.off % 2 == 0
            src = Ptr(src.t.reshape(-1).view(torch.float32), src.off // 2)
            dst = Ptr(dst.t.reshape(-1).view(torch.float32), dst.off // 2)
        r = (torch.arange(rows, device=dst.t.device) // rdiv) % rmod
        n_src = int(r.max()) + 1
        sv = torch.as_strided(src.flat(), (n_src, cols), (src_ld, 1))
        torch.as_strided(dst.flat(), (rows, cols), (dst_ld, 1)).copy_(sv[r])
        return 0

    def tt_layernorm(self, x, x_ld, gamma, beta, y, y_ld, rows, D, row_count, stream):
        self.launches += 1
        n = rows if not row_count else min(rows, int(row_count.flat()[0]))
        xv = torch.as_strided(x.flat(), (rows, D), (x_ld, 1))[:n].double()
        o = F.layer_norm(xv, (D,), gamma.flat()[:D].double(), beta.flat()[:D].double(), 1e-5)
        torch.as_strided(y.flat(), (rows, D), (y_ld, 1))[:n] = o
        return 0

    def tt_eltwise(self, op, act, a, a_ld, b, b_ld, c, c_ld, y, y_ld, rows, cols, stream):
        self.launches += 1
        op, act = _v(op), _v(act)
        v = lambda p, ld: torch.as_strided(p.flat(), (rows, cols), (ld, 1))
        A = v(a, a_ld)
        if op == 0:
            o = A + v(b, b_ld)
        elif op == 1:
            o = (1 - A) * v(b, b_ld)
        elif op == 2:
            o = (1 - A) * v(b, b_ld) + A * v(c, c_ld)
        elif op == 4:                                                  # inverse softplus (a > 0)
            o = A + torch.log(-torch.expm1(-A))
        else:
            o = A
        v(y, y_ld).copy_(_act(o, act))
        return 0

    def tt_gru_input(self, wp, ctrl_sp, t, T, buf, ld, B, HW, stream):
        self.launches += 1
        w = wp.flat()[:B * T * 2].view(B, T, 2)[:, t]
        c = ctrl_sp.flat()[:B * T * 4].view(B, T, 4)[:, t]
        torch.as_strided(buf.flat(), (B, HW, 6), (HW * ld, ld, 1)).copy_(torch.cat([w, c], 1)[:, None, :].expand(B, HW, 6))
        return 0

    # ------------------------------------------------------------------ DCN columns, lift-splat
    def tt_dcn_im2col(self, x, offset, off_ld, col, N, H, W, Cc, groups, stream):
        from torchvision.ops import deform_conv2d
        self.launches += 1
        xv = _pix_view(x, N, H, W, Cc).permute(0, 3, 1, 2).contiguous()
        off = _pix_view(offset, N, H, W, off_ld, C=18).permute(0, 3, 1, 2).contiguous()
        cg = Cc // groups
        out = torch.zeros(N, H, W, groups, 9, cg)
        eye = torch.zeros(9 * cg, cg, 3, 3)                            # output channel (tap, c) = input channel c sampled at tap
        for k in range(9):
            eye[k * cg:(k + 1) * cg, :, k // 3, k % 3] = torch.eye(cg)
        for g in range(groups):
            o = deform_conv2d(xv[:, g * cg:(g + 1) * cg], off, eye, padding=1)          # (N, 9 * cg, H, W)
            out[:, :, :, g] = o.permute(0, 2, 3, 1).reshape(N, H, W, 9, cg)
        col.flat()[:out.numel()].copy_(out.reshape(-1))
        return 0

    def tt_lift_splat(self, d, depth_logits, context, mats, fu, fv, fd, bev, ws, stream):
        d = _desc(d)
        self.launches += 1
        BN = d.B * d.N
        dl = _pix_view(depth_logits, BN, d.fH, d.fW, d.ld_d, C=d.d_coff + d.D)[..., d.d_coff:].double()
        cx = _pix_view(context, BN, d.fH, d.fW, d.ld_c, C=d.c_coff + d.C)[..., d.c_coff:].double()
        prob = dl.softmax(-1)                                          # (BN, fH, fW, D)
        m = mats.flat()[:BN * 32].view(BN, 2, 4, 4)
        u, v, dd = fu.flat()[:d.fW], fv.flat()[:d.fH], fd.flat()[:d.D]
        pts = torch.stack([u.view(1, 1, -1).expand(d.D, d.fH, d.fW), v.view(1, -1, 1).expand(d.D, d.fH, d.fW),
                           dd.view(-1, 1, 1).expand(d.D, d.fH, d.fW), torch.ones(d.D, d.fH, d.fW)], -1)       # (D, fH, fW, 4)
        p = torch.einsum('nij,dhwj->ndhwi', m[:, 0], pts)
        p = torch.cat([p[..., :2] * p[..., 2:3], p[..., 2:]], -1)
        g = torch.einsum('nij,ndhwj->ndhwi', m[:, 1], p)[..., :3]
        idx = ((g - torch.tensor(list(d.lower))) / torch.tensor(list(d.size))).int().long()                      # trunc toward zero
        ok = (idx[..., 0] >= 0) & (idx[..., 0] < d.X) & (idx[..., 1] >= 0) & (idx[..., 1] < d.Y) & (idx[..., 2] >= 0) & (idx[..., 2] < d.Z)
        out = torch.zeros(d.B, d.Y * d.X, d.C, dtype=torch.float64)
        feat = prob.permute(0, 3, 1, 2)[..., None] * cx[:, None]      # (BN, D, fH, fW, C)
        for b in range(d.B):
            sl = slice(b * d.N, (b + 1) * d.N)
            k = ok[sl]
            out[b].index_add_(0, (idx[sl][..., 1] * d.X + idx[sl][..., 0])[k], feat[sl][k])
        out = out.view(d.B, d.Y, d.X, d.C)
        if d.anti_transpose:
            out = out.flip(1).flip(2).transpose(1, 2)
        _pix_view(bev, d.B, d.Y, d.X, d.bev_ld, C=d.bev_coff + d.C)[..., d.bev_coff:] = out.float()
        return 0

    # ------------------------------------------------------------------ Look module, MSDA
    @staticmethod
    def _look_points(d, wp):
        B, T = d.B, d.T
        w = wp.flat()[:B * T * 2].view(B, T, 2)
        static = torch.tensor([[5.0, 0.0], [0.0, -5.0], [0.0, 5.0], [-5.0, 0.0]])[None].repeat(B, 1, 1)
        look = torch.cat([w, static], 1)
        z = torch.linspace(-4, 10, 15, dtype=torch.float64)[None, None, :, None].repeat(B, look.shape[1], 1, 1)
        return torch.cat([look.unsqueeze(2).repeat(1, 1, 15, 1), z], -1).view(B, -1, 3).to(w.dtype)           # (B, Q, 3)

    def tt_look_project(self, d, wp, lidar2img, ida, ref_cam, order, counts, max_len, stream):
        d = _desc(d)
        self.launches += 1
        B, N, Q = d.B, d.num_cams, d.num_query
        look3d = self._look_points(d, wp)
        assert look3d.shape[1] == Q
        ref = torch.cat([look3d, torch.ones_like(look3d[..., :1])], -1).view(B, 1, Q, 4, 1)
        l2i = lidar2img.flat()[:B * N * 16].view(B, N, 1, 4, 4)
        idm = ida.flat()[:B * N * 16].view(B, N, 1, 4, 4)
        cam = torch.matmul(l2i, ref).squeeze(-1)                        # (B, N, Q, 4)
        eps = 1e-5
        cam2 = cam.clone()
        cam2[..., 0:2] = cam[..., 0:2] / torch.maximum(cam[..., 2:3], torch.ones_like(cam[..., 2:3]) * eps)
        cam = torch.matmul(idm, cam2.unsqueeze(-1)).squeeze(-1)
        mask = cam[..., 2] > eps
        xy = cam[..., :2].clone()
        xy[..., 0] /= d.img_w
        xy[..., 1] /= d.img_h
        mask = mask & (xy[..., 1] > 0.0) & (xy[..., 1] < 1.0) & (xy[..., 0] < 1.0) & (xy[..., 0] > 0.0)
        ref_cam.flat()[:B * N * Q * 2].view(B, N, Q, 2).copy_(xy)
        ov, cv = order.flat()[:B * N * Q].view(B, N, Q), counts.flat()[:B * N].view(B, N)
        ml = 0
        for b in range(B):
            for i in range(N):
                ix = mask[b, i].nonzero().squeeze(-1)
                ov[b, i, :len(ix)] = ix.int()
                cv[b, i] = len(ix)
                ml = max(ml, len(ix))
        max_len.flat()[0] = ml
        return 0

    def tt_look_rebatch(self, d, wp, ctrl_sp, temb, semb, meas, flat, mlvl, ref_cam, order, counts, rows, rows_ld, ref_re, stream):
        d = _desc(d)
        self.launches += 1
        B, N, Q, T, L, Cc, cap = d.B, d.num_cams, d.num_query, d.T, d.levels, d.C, d.max_len_cap
        look3d = self._look_points(d, wp)
        cs = ctrl_sp.flat()[:B * T * 4].view(B, T, 4)
        in_ctrl = torch.cat([cs.unsqueeze(2).repeat(1, 1, 15, 1).view(B, -1, 4), torch.zeros(B, 4 * 15, 4)], 1)
        te, se = temb.flat()[:T * d.emb_dim].view(T, d.emb_dim), semb.flat()[:4 * d.emb_dim].view(4, d.emb_dim)
        emb = torch.cat([te[None, :, None].repeat(B, 1, 15, 1).view(B, -1, d.emb_dim), se[None, :, None].repeat(B, 1, 15, 1).view(B, -1, d.emb_dim)], 1)
        me = meas.flat()[:B * d.meas_dim].view(B, d.meas_dim)
        fl = flat.flat()[:B * d.flat_dim].view(B, d.flat_dim)
        q = torch.cat([in_ctrl, look3d, emb, me.unsqueeze(1).repeat(1, Q, 1), fl.unsqueeze(1).repeat(1, Q, 1)], -1)   # (B, Q, 519)
        assert q.shape[-1] == d.q_dim
        xy = ref_cam.flat()[:B * N * Q * 2].view(B, N, Q, 2)
        grid = xy.reshape(B * N, Q, 1, 2) * 2 - 1.0
        sampled = []
        for l in range(L):
            t = _by_addr[mlvl[l]]
            feat = t.reshape(-1)[:B * N * d.lvl_h[l] * d.lvl_w[l] * Cc].view(B * N, d.lvl_h[l], d.lvl_w[l], Cc).permute(0, 3, 1, 2)
            sampled.append(F.grid_sample(feat, grid, align_corners=False).view(B, N, Cc, Q))                       # (B, N, C, Q)
        samp = torch.stack(sampled, -1).permute(0, 3, 1, 2, 4).reshape(B, Q, N, Cc * L)                           # feature index c * L + l
        ov, cv = order.flat()[:B * N * Q].view(B, N, Q), counts.flat()[:B * N].view(B, N)
        rv = torch.as_strided(rows.flat(), (B * N, cap, d.q_dim + Cc * L), (cap * rows_ld, rows_ld, 1))
        rr = ref_re.flat()[:B * N * cap * 2].view(B * N, cap, 2)
        rv.zero_()
        rr.zero_()
        for b in range(B):
            for i in range(N):
                n = int(cv[b, i])
                ix = ov[b, i, :n].long()
                rv[b * N + i, :n] = torch.cat([q[b, ix], samp[b, ix, i]], -1)
                rr[b * N + i, :n] = xy[b, i, ix]
        return 0

    def tt_msda_forward(self, d, value, off, logits, ref, max_len, out, stream):
        from oracle.decoder import msda_pytorch                       # mmcv's published pure-torch formulation
        d = _desc(d)
        self.launches += 1
        BN, cap, Hh, L, P, dh = d.BN, d.rows_cap, d.heads, d.levels, d.points, d.dh
        shapes = [(d.lvl_h[l], d.lvl_w[l]) for l in range(L)]
        VL = d.value_ld or Hh * dh
        v = value.flat()[:BN * d.num_keys * VL].view(BN, d.num_keys, VL)[..., d.value_coff:d.value_coff + Hh * dh].reshape(BN, d.num_keys, Hh, dh)
        o = off.flat()[:BN * cap * Hh * L * P * 2].view(BN, cap, Hh, L, P, 2)
        lg = logits.flat()[:BN * cap * Hh * L * P].view(BN, cap, Hh, L * P)
        r = ref.flat()[:BN * cap * 2].view(BN, cap, 1, 1, 1, 2)
        norm = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float32, device=o.device)
        loc = r + o / norm[None, None, None, :, None, :]
        aw = lg.softmax(-1).view(BN, cap, Hh, L, P)
        res = msda_pytorch(v, torch.tensor(shapes), loc, aw)
        n = min(cap, int(max_len.flat()[0])) if max_len else cap     # rows at or past *max_len are not written
        out.flat()[:BN * cap * Hh * dh].view(BN, cap, Hh * dh)[:, :n] = res[:, :n]
        return 0

    def tt_look_reduce(self, rows, B, cams, cap, Cc, max_len, out, stream):
        self.launches += 1
        ml = int(max_len.flat()[0])
        r = rows.flat()[:B * cams * cap * Cc].view(B, cams, cap, Cc)
        out.flat()[:B * cams * Cc].view(B, cams * Cc).copy_((r[:, :, B:ml].double().sum(2) / B).float().reshape(B, cams * Cc))
        return 0
